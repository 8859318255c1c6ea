"""The semantic-loss kernels (csrc/vit.cu) stage by stage against float64.

tests/test_gpu_vit.py holds the 384-float CLS feature and the image gradient to the float64 oracle end to end; twelve
residual blocks summarised in one vector hide a defect in one 64-row tile, one K tail or one head.  Here the kernels
run through the C ABI with a workspace and a weight image this file allocates (the workspace filled with NaN first),
and every stage the buffers bracket is recomputed in float64 from the kernel's OWN saved inputs, with the GEMM
operands rounded the way the kernel rounds them (tests/vit_emulation.py), so errors do not compound.  The per-element
error is |y - y_ref| / (sum_k |a_k||b_k| + |bias| + |residual|); worst and rms are held to the per-stage bars of
vit_emulation.BARS and printed beside the error against the unrounded float64 product.

Also: the im2col gather bit for bit, the fold against float64 with exact zeros where the nearest map sends nothing,
image sizes from 1 x 1 to 378 x 504 in three memory layouts, n = 8 passes of mixed images equal to n = 1 passes bit
for bit, the upstream-gradient scale at magnitudes 2^-147 ... 2^120, and the packed weight planes bit for bit.
"""
import ctypes as C

import pytest
import torch

from sinnerf_b200 import _lib, synthetic
from sinnerf_b200.vit import _kernel_params, load_dino_weights
from tests import vit_emulation as ve
from tests import vit_oracle as vo
from tests._common import rel_l2

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
NAN = float("nan")
MODE_LIST = list(ve.MODES)
# the n = 8 pass: eight sizes (up- and downsampling, 1-pixel sides, exactly 224) in three layouts; n = 1, 2 take the
# first ones
BATCH = [((64, 64), "nchw"), ((63, 84), "rays"), ((225, 300), "cl_odd"), ((1, 61), "nchw"), ((56, 70), "rays"),
         ((5, 7), "cl_odd"), ((224, 224), "nchw"), ((378, 504), "rays")]
EDGE_SIZES = [(1, 1), (1, 61), (5, 7), (224, 224), (225, 300), (400, 400), (378, 504)]


# --------------------------------------------------------------------------------------------------------------------
# driving the C ABI
# --------------------------------------------------------------------------------------------------------------------
def placed(x, layout):
    """(3, h, w) values -> a (1, 3, h, w) GPU view holding them in `layout`: contiguous NCHW, the '(b p q) c -> b c p q'
    view of a ray-major tensor, or channels-last inside a padded buffer (strides 1, 5 (w + 1), 5; 4-byte offset)."""
    c, h, w = x.shape
    if layout == "nchw":
        return x.to(DEV).reshape(1, c, h, w).contiguous()
    if layout == "rays":
        return x.permute(1, 2, 0).reshape(h * w, c).contiguous().to(DEV).view(1, h, w, c).permute(0, 3, 1, 2)
    assert layout == "cl_odd"
    v = torch.zeros(h, w + 1, 5, device=DEV)[:, :w, 1:4].permute(2, 0, 1).unsqueeze(0)
    v.copy_(x.to(DEV).unsqueeze(0))
    return v


def image(hw, seed):
    return torch.rand(3, *hw, generator=torch.Generator().manual_seed(seed))


def _arrays(ts):
    n = len(ts)
    return ((C.c_void_p * n)(*[t.data_ptr() for t in ts]), (C.c_int64 * (3 * n))(*[s for t in ts for s in t.stride()[1:]]),
            (C.c_int * (2 * n))(*[s for t in ts for s in t.shape[2:]]))


def vit_forward(packed, mode, imgs):
    """(out, workspace) of snb_vit_forward with save = 1 on a NaN-filled workspace"""
    lib, n = _lib.load(), len(imgs)
    ws = torch.full((lib.snb_vit_workspace_bytes(n, 1) // 4,), NAN, device=DEV)
    out = torch.full((n, ve.DIM), NAN, device=DEV)
    p, s, z = _arrays(imgs)
    _lib.check(lib.snb_vit_forward(_lib.ptr(packed), ve.MODES[mode], p, s, z, n, 1, _lib.ptr(out), _lib.ptr(ws),
                                   _lib.stream_ptr(DEV)), "snb_vit_forward")
    return out, ws


def vit_backward(packed, mode, ws, d_out, layouts, sizes):
    """image gradients (NaN-filled views in the given layouts) written by snb_vit_backward"""
    lib = _lib.load()
    grads = [placed(torch.full((3, *hw), NAN), lay) for hw, lay in zip(sizes, layouts)]
    p, s, z = _arrays(grads)
    _lib.check(lib.snb_vit_backward(_lib.ptr(packed), ve.MODES[mode], z, len(grads), _lib.ptr(d_out.contiguous()), p,
                                    s, _lib.ptr(ws), _lib.stream_ptr(DEV)), "snb_vit_backward")
    return grads


@pytest.fixture(scope="module")
def ext():
    return load_dino_weights(synthetic.dino_vits16_state_dict(0)).to(DEV)


@pytest.fixture(scope="module")
def P(ext):
    return {k: v.detach() for k, v in ext.model.state_dict().items()}


def run(ext, mode, n):
    """forward (save) + backward of the first n BATCH images.  Not cached: a pass takes milliseconds, and each test
    frees its workspace (0.36 GB at n = 8) when it returns."""
    packed = ext.packed(DEV, ve.MODES[mode])
    xs = [image(hw, 100 + i) for i, (hw, _) in enumerate(BATCH[:n])]
    imgs = [placed(x, lay) for x, (_, lay) in zip(xs, BATCH)]
    out, ws = vit_forward(packed, mode, imgs)
    col_fwd = ve.workspace_views(ws, n, 1)["col"].clone()
    d_out = torch.randn(n, ve.DIM, generator=torch.Generator().manual_seed(n)).to(DEV)
    grads = vit_backward(packed, mode, ws, d_out, [lay for _, lay in BATCH[:n]], [hw for hw, _ in BATCH[:n]])
    torch.cuda.synchronize()
    return dict(xs=xs, imgs=imgs, out=out, ws=ws, w=ve.workspace_views(ws, n, 1), col_fwd=col_fwd, d_out=d_out,
                grads=grads)


# --------------------------------------------------------------------------------------------------------------------
# references of the gather and the fold
# --------------------------------------------------------------------------------------------------------------------
def gather_ref(img):
    """col of one (1, 3, h, w) image in fp32, as torch computes (x[iy][:, ix] - mean) / std"""
    x = img[0].cpu()
    iy, ix = (torch.from_numpy(vo.nearest_index(s)) for s in x.shape[1:])
    mean = torch.tensor(ve.MEAN, dtype=torch.float32).view(3, 1, 1)
    std = torch.tensor(ve.STD, dtype=torch.float32).view(3, 1, 1)
    return ve.im2col((x[:, iy][:, :, ix] - mean) / std)


def check_fold(grad, col, inv, hw):
    """grad (1, 3, h, w) from the kernel against the float64 fold of its own col: every pixel written, exact zeros where
    the nearest map sends nothing, and elsewhere within the recursive-summation bound (terms + 2) 2^-24 of the sum of
    |terms| (an fp32 sum of the terms, one division by std, one exact power-of-two scale).  -> worst e / bound"""
    h, w = hw
    g224 = ve.col2im(col.double())
    iy, ix = (torch.from_numpy(vo.nearest_index(s)).to(DEV) for s in hw)
    idx = (iy[:, None] * w + ix[None, :]).flatten()
    ref = torch.zeros(3, h * w, dtype=torch.float64, device=DEV).index_add_(1, idx, g224.reshape(3, -1))
    mag = torch.zeros(3, h * w, dtype=torch.float64, device=DEV).index_add_(1, idx, g224.abs().reshape(3, -1))
    cnt = torch.bincount(idx, minlength=h * w).double()
    std = torch.tensor(ve.STD, dtype=torch.float32, device=DEV).double().view(3, 1)
    ref, mag = (ref / std * inv).view(3, h, w), (mag / std * inv).view(3, h, w)
    g = grad[0]
    assert not torch.isnan(g).any()
    empty = (cnt == 0).view(1, h, w).expand(3, h, w)
    assert torch.equal(g[empty], torch.zeros_like(g[empty]))
    bound = (cnt.view(1, h, w) + 2) * 2.0 ** -24 * mag
    e = ((g.double() - ref).abs() / bound.clamp_min(1e-300))[~empty]
    worst = float(e.max()) if e.numel() else 0.0
    assert worst <= 1.0, worst
    return worst


# --------------------------------------------------------------------------------------------------------------------
# stage by stage
# --------------------------------------------------------------------------------------------------------------------
class Stages:
    """per stage: the largest worst and the largest rms over the stage's GEMMs (one per block), against the emulation
    and against the exact product.  The rms is per GEMM so that a defect in one block is not averaged away."""

    def __init__(self):
        self.e, self.chains = {}, set()

    def add(self, stage, y, emu, exact, scale):
        """exact None: a chain of several products, compared with the emulation only"""
        assert not torch.isnan(y).any(), stage
        if exact is None:
            self.chains.add(stage)
            exact = emu
        old = self.e.get(stage, (0.0,) * 4)
        new = ve.stats(ve.err(y, emu, scale)) + ve.stats(ve.err(y, exact, scale))
        self.e[stage] = tuple(max(a, b) for a, b in zip(old, new))

    def check(self, mode, what):
        bad = []
        for stage, (w, r, wx, rx) in self.e.items():
            bw, br = ve.BARS[mode].get(stage, (0.0, 0.0))
            exact = f" | vs exact product: worst {wx:.2e} rms {rx:.2e}" if stage not in self.chains else ""
            print(f"vit layerwise {what} {mode:5s} {stage:6s}: worst {w:.2e} rms {r:.2e} (bars {bw:.0e} {br:.0e})"
                  + exact)
            if not (w <= bw and r <= br):
                bad.append((stage, w, r))
        assert not bad, bad


def blk_w(P, l):
    p = f"blocks.{l}."
    return {k: P[p + v] for k, v in (("n1w", "norm1.weight"), ("n1b", "norm1.bias"), ("Wqkv", "attn.qkv.weight"),
                                      ("bqkv", "attn.qkv.bias"), ("Wp", "attn.proj.weight"), ("bp", "attn.proj.bias"),
                                      ("n2w", "norm2.weight"), ("n2b", "norm2.bias"), ("W1", "mlp.fc1.weight"),
                                      ("b1", "mlp.fc1.bias"), ("W2", "mlp.fc2.weight"), ("b2", "mlp.fc2.bias"))}


@pytest.mark.parametrize("n", [1, 2, 8])
@pytest.mark.parametrize("mode", MODE_LIST)
def test_forward_stages(ext, P, mode, n):
    R = run(ext, mode, n)
    w, st = R["w"], Stages()
    for i, img in enumerate(R["imgs"]):
        assert torch.equal(R["col_fwd"][i].cpu(), gather_ref(img)), i
    Wpe = P["patch_embed.proj.weight"].reshape(ve.DIM, ve.PATCHK)
    st.add("embed", w["blk0.x_in"][:, 1:], *ve.linear_ref(R["col_fwd"], Wpe, P["patch_embed.proj.bias"], mode,
                                                          resid=P["pos_embed"][0, 1:]))
    cls = (P["cls_token"][0, 0] + P["pos_embed"][0, 0]).expand(n, -1)
    assert torch.equal(w["blk0.x_in"][:, 0], cls)
    for l in range(ve.BLOCKS - 1):
        B, x_in, qkv, x_mid = blk_w(P, l), w[f"blk{l}.x_in"], w[f"blk{l}.qkv"], w[f"blk{l}.x_mid"]
        st.add("qkv", qkv, *ve.linear_ref(ve.ln64(x_in, B["n1w"], B["n1b"]).float(), B["Wqkv"], B["bqkv"], mode))
        q, k, v = (ve.heads(qkv[..., j * ve.DIM:(j + 1) * ve.DIM]) for j in range(3))
        lse, lse_x, sc, Pm = ve.scores_ref(q, k, mode)
        st.add("lse", w[f"blk{l}.lse"], lse, lse_x, sc)
        st.add("pv", ve.heads(w[f"blk{l}.O"]), *ve.pv_ref(Pm, v, mode))
        st.add("proj", x_mid, *ve.linear_ref(w[f"blk{l}.O"], B["Wp"], B["bp"], mode, resid=x_in))
        st.add("fc1", w[f"blk{l}.pre"], *ve.linear_ref(ve.ln64(x_mid, B["n2w"], B["n2b"]).float(), B["W1"], B["b1"], mode))
        st.add("fc2", w[f"blk{l + 1}.x_in"], *ve.linear_ref(ve.gelu64(w[f"blk{l}.pre"]).float(), B["W2"], B["b2"], mode,
                                                            resid=x_mid))
    # block 11, pruned: K and V of every token, Q and the rest at the CLS rows only
    B, x_in, qkv = blk_w(P, 11), w["blk11.x_in"], w["blk11.qkv"]
    ln1 = ve.ln64(x_in, B["n1w"], B["n1b"]).float()
    D = ve.DIM
    st.add("qkv", qkv[..., D:], *ve.linear_ref(ln1, B["Wqkv"][D:], B["bqkv"][D:], mode))
    st.add("qkv", qkv[:, :1, :D], *ve.linear_ref(ln1[:, :1], B["Wqkv"][:D], B["bqkv"][:D], mode))
    assert torch.isnan(qkv[:, 1:, :D]).all()          # Q of the other tokens is never computed
    q, k, v = ve.heads(qkv[:, :1, :D]), ve.heads(qkv[..., D:2 * D]), ve.heads(qkv[..., 2 * D:])
    lse, lse_x, sc, Pm = ve.scores_ref(q, k, mode)
    st.add("lse", w["lse_c"].view(n, ve.HEADS, 1), lse, lse_x, sc)
    st.add("pv", ve.heads(w["O_c"].view(n, 1, D)), *ve.pv_ref(Pm, v, mode))
    st.add("proj", w["xmid_c"], *ve.linear_ref(w["O_c"], B["Wp"], B["bp"], mode, resid=x_in[:, 0]))
    st.add("fc1", w["pre_c"], *ve.linear_ref(ve.ln64(w["xmid_c"], B["n2w"], B["n2b"]).float(), B["W1"], B["b1"], mode))
    st.add("fc2", R["out"], *ve.linear_ref(ve.gelu64(w["pre_c"]).float(), B["W2"], B["b2"], mode, resid=w["xmid_c"]))
    st.check(mode, f"forward n={n}")


@pytest.mark.parametrize("n", [1, 2, 8])
@pytest.mark.parametrize("mode", MODE_LIST)
def test_backward_stages(ext, P, mode, n):
    R = run(ext, mode, n)
    w, st, D = R["w"], Stages(), ve.DIM
    # c0: the upstream gradient times s = 2^(1 - e), max |g| = f 2^e, bit for bit
    m = R["d_out"].abs().amax(1)
    s = (2.0 ** (1 - torch.frexp(m).exponent).double()).float()
    assert torch.equal(w["c0"], R["d_out"] * s[:, None]) and torch.equal(w["inv"], 1.0 / s)
    # block 11 (CLS rows): fc2 dgrad + GELU derivative, fc1 dgrad + LN2 backward + residual, proj dgrad
    B = blk_w(P, 11)
    e, x, a = ve.dgrad_ref(w["c0"], B["W2"], mode)
    gg = ve.gelu_grad64(w["pre_c"])
    st.add("dfc2", w["ch"], e * gg, x * gg, a * ve.gelu_grad64(w["pre_c"], magnitude=True))
    e, x, a = ve.dgrad_ref(w["ch"], B["W1"], mode)
    dx, sc = ve.ln_bwd64(w["xmid_c"], B["n2w"], e, a)
    dxx, _ = ve.ln_bwd64(w["xmid_c"], B["n2w"], x)
    st.add("dfc1", w["c2"], dx + w["c0"].double(), dxx + w["c0"].double(), sc + w["c0"].double().abs())
    st.add("dproj", w["c1"], *ve.dgrad_ref(w["c2"], B["Wp"], mode))
    # block 0's attention half, from dx2 (the gradient at x_mid) to dx (at x_in)
    B = blk_w(P, 0)
    st.add("dproj", w["dO"], *ve.dgrad_ref(w["dx2"], B["Wp"], mode))
    qkv = w["blk0.qkv"]
    q, k, v = (ve.heads(qkv[..., j * D:(j + 1) * D]) for j in range(3))
    Pk, dSk = w["S"][..., :ve.TOK], w["dP"][..., :ve.TOK]
    pr = ve.Prod(q, k, mode)
    lse = w["blk0.lse"].double()[..., None]
    pe, px = torch.exp(ve.ALPHA * pr.emu - lse), torch.exp(ve.ALPHA * pr.exact - lse)
    st.add("P", Pk, pe, px, pe * ve.ALPHA * pr.abs)
    dO, O = ve.heads(w["dO"]), ve.heads(w["blk0.O"])
    pr = ve.Prod(dO, v, mode)
    Dr = (dO.double() * O.double()).sum(-1, keepdim=True)
    Da = (dO.double() * O.double()).abs().sum(-1, keepdim=True)
    c = ve.ALPHA * Pk.double()
    st.add("dS", dSk, c * (pr.emu - Dr), c * (pr.exact - Dr), c * (pr.abs + Da))
    for j, (A_, B_) in enumerate([(dSk, k.transpose(-1, -2)), (dSk.transpose(-1, -2), q.transpose(-1, -2)),
                                  (Pk.transpose(-1, -2), dO.transpose(-1, -2))]):
        pr = ve.Prod(A_, B_, mode)
        st.add("dqkv", ve.heads(w["dqkv"][..., j * D:(j + 1) * D]), pr.emu, pr.exact, pr.abs)
    st.add("dqkvW", w["dln"], *ve.dgrad_ref(w["dqkv"], B["Wqkv"], mode))
    dx, sc = ve.ln_bwd64(w["blk0.x_in"], B["n1w"], w["dln"])
    st.add("dln1", w["dx"], dx + w["dx2"].double(), dx + w["dx2"].double(), sc + w["dx2"].double().abs())
    # patch-embedding dgrad into im2col rows, then the fold
    Wpe = P["patch_embed.proj.weight"].reshape(D, ve.PATCHK)
    st.add("dembed", w["col"], *ve.dgrad_ref(w["dx"][:, 1:], Wpe, mode))
    st.check(mode, f"backward n={n}")
    for i, (hw, _) in enumerate(BATCH[:n]):
        check_fold(R["grads"][i], w["col"][i], float(w["inv"][i]), hw)


def block11_token_grad(w, P, mode, n):
    """float64 (gradient, error scale) at block 11's input, all 197 n token rows, from the kernel's c2 (the gradient at
    the CLS rows of x_mid) and c1 (dO of the CLS rows) and block 11's saved state: the q_rows = 1 attention backward
    (P from the saved lse, dS, dQ = dS K at M = 1, dK = dS^T Q and dV = P^T dO at K = 1), the qkv dgrad over every
    token row, then the LN1 backward plus c2 at the CLS rows.  Each intermediate is rounded to fp32 where the kernel
    stores it; the scale carries sum |a||b| of every product through the chain."""
    B, D = blk_w(P, 11), ve.DIM
    qkv = w["blk11.qkv"]
    q, k, v = ve.heads(qkv[:, :1, :D]), ve.heads(qkv[..., D:2 * D]), ve.heads(qkv[..., 2 * D:])
    dO, O = ve.heads(w["c1"].view(n, 1, D)), ve.heads(w["O_c"].view(n, 1, D))
    Pm = torch.exp(ve.ALPHA * ve.Prod(q, k, mode).emu - w["lse_c"].double().view(n, ve.HEADS, 1, 1))
    dp = ve.Prod(dO, v, mode)
    Dr = (dO.double() * O.double()).sum(-1, keepdim=True)
    Da = (dO.double() * O.double()).abs().sum(-1, keepdim=True)
    dS, sdS = ve.ALPHA * Pm * (dp.emu - Dr), ve.ALPHA * Pm * (dp.abs + Da)
    dSf, Pf = dS.float(), Pm.float()
    dqkv = torch.zeros(n, ve.TOK, ve.QKV, dtype=torch.float64, device=DEV)
    sqkv = torch.zeros_like(dqkv)
    dqkv[:, :1, :D] = ve.unheads(ve.Prod(dSf, k.transpose(-1, -2), mode).emu)
    sqkv[:, :1, :D] = ve.unheads(sdS @ k.double().abs())
    dqkv[..., D:2 * D] = ve.unheads(ve.Prod(dSf.transpose(-1, -2), q.transpose(-1, -2), mode).emu)
    sqkv[..., D:2 * D] = ve.unheads(sdS.transpose(-1, -2) @ q.double().abs())
    pv = ve.Prod(Pf.transpose(-1, -2), dO.transpose(-1, -2), mode)
    dqkv[..., 2 * D:], sqkv[..., 2 * D:] = ve.unheads(pv.emu), ve.unheads(pv.abs)
    dln = ve.Prod(dqkv.float(), B["Wqkv"].t(), mode).emu
    sln = sqkv @ B["Wqkv"].double().abs()
    dx, sc = ve.ln_bwd64(w["blk11.x_in"], B["n1w"], dln, sln)
    dx[:, 0] += w["c2"].double()
    sc[:, 0] += w["c2"].double().abs()
    return dx, sc


def zeroed(sd, blocks):
    """the state dict with every tensor of the given blocks set to zero: such a block passes activations and gradients
    through exactly (LN output 0, every product +0, x + 0 = x, and the LN backward of dy = 0 is 0)"""
    return {k: torch.zeros_like(v) if any(k.startswith(f"blocks.{b}.") for b in blocks) else v for k, v in sd.items()}


@pytest.mark.parametrize("n", [1, 8])
@pytest.mark.parametrize("mode", MODE_LIST)
def test_backward_through_zero_blocks(mode, n):
    """The stages no buffer brackets in a full pass, isolated with zero-weight blocks.
    - Blocks 0-10 zero: the final dx is block 11's input gradient, checked against float64 from c2 and block 11's
      saved state ('b11tok': the q_rows = 1 attention backward, the qkv dgrad, the res_cls LN1 backward).
    - Blocks 1-10 zero: block 0 receives that gradient.  Its dh (fc2 dgrad + GELU derivative over all 197 n rows,
      'dh0') is checked against the float64 chain through block 11, and its dx2 (fc1 dgrad over all rows, LN2
      backward and the residual, 'dx2_0') from the kernel's dh and the chain.  Their scales carry block 11's error."""
    sd = synthetic.dino_vits16_state_dict(0)
    st = Stages()
    for zero in (range(0, 11), range(1, 11)):
        ext = load_dino_weights(zeroed(sd, zero)).to(DEV)
        P = {k: v.detach() for k, v in ext.model.state_dict().items()}
        R = run(ext, mode, n)
        w = R["w"]
        assert torch.equal(w["blk11.x_in"], w[f"blk{zero.start}.x_in"])       # the zero blocks pass x exactly
        dx11, sc11 = block11_token_grad(w, P, mode, n)
        if zero.start == 0:
            st.add("b11tok", w["dx"], dx11, None, sc11)
        else:
            B = blk_w(P, 0)
            gg = ve.gelu_grad64(w["blk0.pre"])
            st.add("dh0", w["dh"], ve.Prod(dx11.float(), B["W2"].t(), mode).emu * gg, None,
                   (sc11 @ B["W2"].double().abs()) * ve.gelu_grad64(w["blk0.pre"], magnitude=True))
            e, _, a = ve.dgrad_ref(w["dh"], B["W1"], mode)
            dx, sc = ve.ln_bwd64(w["blk0.x_mid"], B["n2w"], e, a)
            st.add("dx2_0", w["dx2"], dx + dx11, None, sc + sc11)
        del R, w, ext
    st.check(mode, f"zero blocks n={n}")


# --------------------------------------------------------------------------------------------------------------------
# edges
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hw,layout", [(hw, lay) for hw in EDGE_SIZES for lay in ("nchw", "rays")] +
                         [((225, 300), "cl_odd")], ids=lambda s: "x".join(map(str, s)) if isinstance(s, tuple) else s)
def test_image_sizes(ext, P, hw, layout):
    """gather bit for bit, fold against float64, feature and gradient against the oracle at test_gpu_vit's split bars"""
    x = image(hw, hw[0] * 1000 + hw[1])
    img = placed(x, layout)
    packed = ext.packed(DEV, ve.MODES["split"])
    out, ws = vit_forward(packed, "split", [img])
    w = ve.workspace_views(ws, 1, 1)
    assert torch.equal(w["col"][0].cpu(), gather_ref(img))
    wvec = torch.randn(1, ve.DIM, generator=torch.Generator().manual_seed(3)).to(DEV)
    (g,) = vit_backward(packed, "split", ws, wvec, [layout], [hw])
    worst = check_fold(g, w["col"][0], float(w["inv"][0]), hw)
    x64 = x.to(DEV, torch.float64)[None].requires_grad_(True)
    f = vo.cls_feature(P, x64)
    (f * wvec[0].double()).sum().backward()
    ef, eg = rel_l2(out[0].cpu(), f.detach().cpu()), rel_l2(g.cpu(), x64.grad.cpu())
    print(f"vit sizes {hw} {layout}: feature {ef:.2e} gradient {eg:.2e} fold {worst:.2f} of its bound")
    assert ef <= 1e-4 and eg <= 1e-3, (ef, eg)


@pytest.mark.parametrize("mode", MODE_LIST)
def test_batch_of_8_equals_single_passes(ext, mode):
    """DESIGN 4.5: a row's result does not depend on which other images share the pass"""
    R = run(ext, mode, 8)
    packed = ext.packed(DEV, ve.MODES[mode])
    for i, (hw, lay) in enumerate(BATCH):
        out, ws = vit_forward(packed, mode, [R["imgs"][i]])
        (g,) = vit_backward(packed, mode, ws, R["d_out"][i:i + 1], [lay], [hw])
        assert torch.equal(out[0], R["out"][i]), (i, hw)
        assert torch.equal(g, R["grads"][i]), (i, hw)


@pytest.mark.parametrize("mode", MODE_LIST)
def test_upstream_gradient_scale(ext, mode):
    """The power-of-two scale of the upstream gradient is exact: grad(f (c w)) == c grad(f w) bit for bit wherever
    c grad is a normal fp32; a zero upstream gives exact zeros, and an upstream whose largest element is subnormal
    gives the right subnormal gradient."""
    packed = ext.packed(DEV, ve.MODES[mode])
    hw, lay = (63, 84), "rays"
    _, ws = vit_forward(packed, mode, [placed(image(hw, 7), lay)])
    wvec = torch.randn(1, ve.DIM, generator=torch.Generator().manual_seed(8)).to(DEV)
    (g1,) = vit_backward(packed, mode, ws, wvec, [lay], [hw])
    assert torch.isfinite(g1).all() and float(g1.abs().max()) > 0
    for k in (-120, -60, 0, 60, 120):
        (gk,) = vit_backward(packed, mode, ws, wvec * 2.0 ** k, [lay], [hw])
        want = g1 * 2.0 ** k
        normal = torch.isfinite(want) & (want.abs() >= 2.0 ** -126)
        assert bool(normal.any()), k
        assert torch.equal(gk[normal], want[normal]), k
        assert torch.isfinite(gk[torch.isfinite(want)]).all(), k
    (g0,) = vit_backward(packed, mode, ws, torch.zeros_like(wvec), [lay], [hw])
    assert torch.equal(g0, torch.zeros_like(g0))
    # Upstreams whose largest element is subnormal.  A scale s = 2^(1 - e) formed as a float overflows to inf there and
    # 1 / s to 0 (NaN gradients in bf16, exact zeros in the fp16 modes).  Scaled exactly, the chain sees the same c0 as
    # for the same upstream scaled up by 2^-k (exact: the subnormal upstream is itself rounded, so w 2^k would not do),
    # and only the fold's last multiply differs: the gradient is that one's times 2^k, rounded once, bit for bit.
    ulp = 2.0 ** -149
    for k in (-127 - int(torch.frexp(wvec.abs().max()).exponent), -140, -147):
        sub = wvec * 2.0 ** k
        assert 0 < float(sub.abs().max()) < 2.0 ** -126, k
        (gs,) = vit_backward(packed, mode, ws, sub, [lay], [hw])
        (gu,) = vit_backward(packed, mode, ws, sub * 2.0 ** 64 * 2.0 ** (-k - 64), [lay], [hw])   # fp32 factors
        want = (gu.double() * 2.0 ** k).float()
        print(f"vit upstream 2^{k} {mode}: max |grad| {float(want.abs().max()) / ulp:.3g} ulps, "
              f"{int((gs != want).sum())} elements differ")
        assert float(want.abs().max()) >= 8 * ulp, k
        assert torch.equal(gs, want), (k, float((gs.double() - want.double()).abs().max()) / ulp)


@pytest.mark.parametrize("mode", MODE_LIST)
def test_pack_bitwise(mode):
    """snb_vit_pack: fp32 vectors copied, every matrix's plane(s) equal to the emulation's bit for bit, with entries
    beyond +-65504 (clamped before the fp16 rounding) and below 2^-14 (fp16 subnormal hi and lo words)"""
    sd = synthetic.dino_vits16_state_dict(1)
    special = torch.tensor([1e5, -7e4, 65504.0, 65519.0, 65520.0, -3e38, 3e-6, -1e-7, 6e-5, 2.0 ** -14, 2.0 ** -24,
                            2.0 ** -25, 1e-9, 0.0, -0.0, 0.2, 0.1234567, -1.0e-3, 5.96e-8, 65503.9])
    for key in ("patch_embed.proj.weight", "blocks.0.attn.qkv.weight", "blocks.11.mlp.fc2.weight"):
        t = sd[key].clone()
        t.view(-1)[:special.numel()] = special
        t.view(-1)[-special.numel():] = -special
        sd[key] = t
    ps = [p.detach().to(DEV) for p in _kernel_params(load_dino_weights(sd).model)]
    lib = _lib.load()
    prec = ve.MODES[mode]
    assert lib.snb_vit_pack_bytes(prec) == ve.pack_bytes(mode)
    img = torch.zeros(ve.pack_bytes(mode), dtype=torch.uint8, device=DEV)
    _lib.check(lib.snb_vit_pack((C.c_void_p * len(ps))(*[p.data_ptr() for p in ps]), prec, _lib.ptr(img),
                                _lib.stream_ptr(DEV)), "snb_vit_pack")
    L = ve.pack_layout(mode)
    f = img[:L["n_floats"] * 4].view(torch.float32)
    h = img[L["n_floats"] * 4:].view(torch.int16)
    # (offset, tensor, is a matrix) in the C ABI's tensor order
    pieces = [(L["cls"], False), (L["pos"], False), (L["pe"], True), (L["pe_b"], False)]
    for B in L["blk"]:
        pieces += [(B[k], k in ("qkv", "proj", "fc1", "fc2")) for k in ("n1w", "n1b", "qkv", "qkv_b", "proj", "proj_b",
                                                                        "n2w", "n2b", "fc1", "fc1_b", "fc2", "fc2_b")]
    for i, ((off, is_mat), t) in enumerate(zip(pieces, ps)):
        t = t.flatten()
        if not is_mat:
            assert torch.equal(f[off:off + t.numel()], t), i
            continue
        for j, plane in enumerate(ve.packed_planes(t, mode)):
            got = h[off + j * t.numel():off + (j + 1) * t.numel()]
            assert torch.equal(got, plane), (i, j, int((got != plane).sum()))
