"""Plain-torch restatement of kornia 0.6.3's `inverse_depth_smoothness_loss` and `ssim_loss` (window 11), in kornia's
order of operations: image gradients by slicing, and SSIM's window sums as F.pad(mode='reflect') followed by a full
2-D depthwise conv2d.  Written from kornia's published definitions, not from its source.  Every function works in the
dtype of its inputs, so the tests run it in float64 as the truth and in float32 as kornia's own arithmetic.

It lives with the tests rather than under oracle/, the yardstick of the rendering path, which these losses do not
touch; sinnerf_b200.losses is the GPU implementation checked against it."""
import torch
import torch.nn.functional as F


def _gradient_x(t):
    return t[:, :, :, :-1] - t[:, :, :, 1:]


def _gradient_y(t):
    return t[:, :, :-1, :] - t[:, :, 1:, :]


def inverse_depth_smoothness_loss(idepth, image):
    idepth_dx, idepth_dy = _gradient_x(idepth), _gradient_y(idepth)
    image_dx, image_dy = _gradient_x(image), _gradient_y(image)
    weights_x = torch.exp(-torch.mean(torch.abs(image_dx), dim=1, keepdim=True))
    weights_y = torch.exp(-torch.mean(torch.abs(image_dy), dim=1, keepdim=True))
    smoothness_x = torch.abs(idepth_dx * weights_x)
    smoothness_y = torch.abs(idepth_dy * weights_y)
    return torch.mean(smoothness_x) + torch.mean(smoothness_y)


def gaussian_1d(window_size=11, sigma=1.5, dtype=torch.float64, device=None):
    """exp(-x^2 / (2 sigma^2)) for x = -(ws // 2) .. ws // 2, normalised to sum 1 (odd window sizes)."""
    x = torch.arange(window_size, dtype=dtype, device=device) - window_size // 2
    g = torch.exp(-x.pow(2.0) / (2 * sigma ** 2))
    return g / g.sum()


def gaussian_2d(window_size=11, sigma=1.5, dtype=torch.float64, device=None):
    g = gaussian_1d(window_size, sigma, dtype, device)
    return torch.matmul(g.unsqueeze(-1), g.unsqueeze(-1).t())


def filter2d(x, kernel):
    """kornia filter2d with border_type='reflect': reflect-pad by ws // 2 on every side, then a depthwise
    correlation of every channel with the same 2-D kernel."""
    b, c, h, w = x.shape
    kh, kw = kernel.shape
    xp = F.pad(x, [kw // 2, kw // 2, kh // 2, kh // 2], mode="reflect")
    weight = kernel.to(x.dtype).expand(c, 1, kh, kw)
    return F.conv2d(xp, weight, groups=c, padding=0, stride=1)


def ssim_map(img1, img2, window_size=11, max_val=1.0, eps=1e-12):
    kernel = gaussian_2d(window_size, 1.5, img1.dtype, img1.device)
    C1 = (0.01 * max_val) ** 2
    C2 = (0.03 * max_val) ** 2
    mu1 = filter2d(img1, kernel)
    mu2 = filter2d(img2, kernel)
    mu1_sq, mu2_sq, mu1_mu2 = mu1 ** 2, mu2 ** 2, mu1 * mu2
    sigma1_sq = filter2d(img1 ** 2, kernel) - mu1_sq
    sigma2_sq = filter2d(img2 ** 2, kernel) - mu2_sq
    sigma12 = filter2d(img1 * img2, kernel) - mu1_mu2
    num = (2.0 * mu1_mu2 + C1) * (2.0 * sigma12 + C2)
    den = (mu1_sq + mu2_sq + C1) * (sigma1_sq + sigma2_sq + C2)
    return num / (den + eps)


def ssim_loss(img1, img2, window_size=11, max_val=1.0, eps=1e-12):
    loss = torch.clamp((1.0 - ssim_map(img1, img2, window_size, max_val, eps)) / 2, min=0, max=1)
    return torch.mean(loss)
