"""`Embedding` and `NeRF` with the reference's constructor signatures, attributes and state-dict
(reference models/nerf.py:7-41, :46-148), executing on libsinnerf_b200's sm_90a kernels.

The modules are parameter containers: `nn.Linear` leaves with the reference's names
(`xyz_encoding_{1..8}.0.{weight,bias}`, `xyz_encoding_final.*`, `dir_encoding.0.*`, `sigma.*`,
`rgb.0.*`) so `utils.load_ckpt`, optimizers, DDP and Lightning checkpoints keep working
(reference utils/__init__.py:60-83, train.py:25-30).  `forward` never runs the nn.Linear
modules; it calls the fused CUDA kernels through the C ABI.
"""
from __future__ import annotations

import ctypes as C

import torch
from torch import nn

from . import _lib
from . import config


class ShiftedSoftplus(nn.Module):
    """Marker for reference models/activations.py:54-71; evaluated inside the fused kernels."""

    def forward(self, x):  # pragma: no cover - never on the hot path
        raise RuntimeError("activation is fused into the sm_90a field kernel; call NeRF.forward")


class WidenedSigmoid(ShiftedSoftplus):
    """Marker for reference models/activations.py:38-51."""


class Embedding(nn.Module):
    def __init__(self, in_channels, N_freqs, logscale=True):
        """Embeds x to (x, sin(2^k x), cos(2^k x), ...)  -- reference models/nerf.py:8-22."""
        super().__init__()
        self.N_freqs = N_freqs
        self.in_channels = in_channels
        self.funcs = [torch.sin, torch.cos]
        self.out_channels = in_channels * (len(self.funcs) * N_freqs + 1)
        if logscale:
            self.freq_bands = 2 ** torch.linspace(0, N_freqs - 1, N_freqs)
        else:
            self.freq_bands = torch.linspace(1, 2 ** (N_freqs - 1), N_freqs)
        self._logscale = bool(logscale)

    def forward(self, x):
        """x (B, in_channels) -> (B, out_channels)  -- reference models/nerf.py:24-41."""
        if not self._logscale:
            raise NotImplementedError("sinnerf_b200.Embedding: only logscale=True bands (the ones SinNeRF "
                                      "uses, models/sinnerf.py:131-132) have a kernel")
        _lib.require_device(x, "Embedding.forward")
        if torch.is_grad_enabled() and x.requires_grad:
            raise NotImplementedError("sinnerf_b200.Embedding.forward is not differentiable in its input (the reference "
                                      "never differentiates it either: rays carry no grad, models/sinnerf.py:171-193); "
                                      "call it under torch.no_grad() or detach the input")
        if x.dim() != 2 or x.shape[1] != self.in_channels:
            raise ValueError(f"Embedding.forward: expected (B, {self.in_channels}), got {tuple(x.shape)}")
        xc = x.detach().to(torch.float32).contiguous()
        out = torch.empty(xc.shape[0], self.out_channels, device=x.device, dtype=torch.float32)
        with torch.cuda.device(x.device):
            _lib.check(_lib.load().snb_embed(_lib.ptr(xc), xc.shape[0], self.in_channels, self.N_freqs,
                                             _lib.ptr(out), _lib.stream_ptr(x.device)), "snb_embed")
        return out


class NeRF(nn.Module):
    def __init__(self, D=8, W=256, in_channels_xyz=63, in_channels_dir=27, skips=[4], use_new_activation=False):
        """Same arguments and parameter names as reference models/nerf.py:47-103."""
        super().__init__()
        self.D, self.W = D, W
        self.in_channels_xyz, self.in_channels_dir = in_channels_xyz, in_channels_dir
        self.skips = skips
        self.use_new_activation = bool(use_new_activation)
        for i in range(D):
            if i == 0:
                layer = nn.Linear(in_channels_xyz, W)
            elif i in skips:
                layer = nn.Linear(W + in_channels_xyz, W)
            else:
                layer = nn.Linear(W, W)
            setattr(self, f"xyz_encoding_{i + 1}", nn.Sequential(layer, nn.ReLU(True)))
        self.xyz_encoding_final = nn.Linear(W, W)
        if use_new_activation:
            self.dir_encoding = nn.Sequential(nn.Linear(W + in_channels_dir, W // 2), ShiftedSoftplus())
            self.sigma = nn.Linear(W, 1)
            self.rgb = nn.Sequential(nn.Linear(W // 2, 3), WidenedSigmoid())
        else:
            self.dir_encoding = nn.Sequential(nn.Linear(W + in_channels_dir, W // 2), nn.ReLU(True))
            self.sigma = nn.Linear(W, 1)
            self.rgb = nn.Sequential(nn.Linear(W // 2, 3), nn.Sigmoid())
        self._packed = {}  # (precision id, device) -> uint8 device tensor
        self._fast = {}    # precision id -> validated pointer table of packed_weights()
        self._last_stream = {}   # precision id -> the stream the image was last refreshed / read on
        self._last_prec = None   # precision id of the last pass (the image a fused optimiser re-packs under 'autocast')

    # ------------------------------------------------------------------ kernels' weight image
    def _check_shape(self):
        if (self.D, self.W, self.in_channels_xyz, self.in_channels_dir, list(self.skips)) != (8, 256, 63, 27, [4]):
            raise NotImplementedError(
                "sinnerf_b200 kernels are specialised for NeRF(D=8, W=256, in_channels_xyz=63, "
                "in_channels_dir=27, skips=[4]) -- the shape SinNeRF instantiates (models/sinnerf.py:137,140)")

    def _param_list(self):
        """The 24 parameter tensors in state-dict order.  Walks the module dicts directly (three dict lookups per
        tensor, ~5 us in all; `getattr` chains through nn.Module.__getattr__ cost 19 us) and always returns the
        CURRENT Parameter objects, so replaced parameters / sub-modules are seen."""
        mods = self._modules
        ps = []
        for i in range(self.D):
            lp = mods[f"xyz_encoding_{i + 1}"]._modules["0"]._parameters
            ps.append(lp["weight"])
            ps.append(lp["bias"])
        for name, sub in (("xyz_encoding_final", None), ("dir_encoding", "0"), ("sigma", None), ("rgb", "0")):
            m = mods[name] if sub is None else mods[name]._modules[sub]
            lp = m._parameters
            ps.append(lp["weight"])
            ps.append(lp["bias"])
        return ps

    def packed_weights(self, precision=None) -> torch.Tensor:
        """Device image of the weights in the layout the kernels stream, brought up to date on the current
        stream (C ABI snb_refresh_weights).  The image buffer is allocated once per (precision, device);
        every call enqueues a check kernel that compares a checksum of the parameter VALUES with the one the
        image was packed from and re-packs on the device only when they differ -- so optimizer steps,
        `load_state_dict` and in-place updates through `p.data` (which do not bump `_version`; reference
        utils/optimizers.py:98,180,268) are all seen, with no host synchronisation.

        Host cost matters here: a render starts with two of these calls while the GPU idles (a 5 292-ray patch is
        0.9 ms in all).  The validated pointer table is therefore cached and reused for as long as the 24 storage
        addresses are the ones it was built from (a dtype / device / layout change re-allocates and is re-validated):
        ~10 us per call instead of ~70."""
        prec = config.resolve_precision(precision)
        self._last_prec = prec
        ps = self._param_list()
        ptrs = [p.data_ptr() for p in ps]
        fast = self._fast.get(prec)
        if fast is None or fast[0] != ptrs:
            dev = ps[0].device
            srcs = []
            for p in ps:
                if p.dtype != torch.float32 or p.device != dev:
                    raise ValueError("NeRF parameters must be fp32 tensors on one CUDA device")
                srcs.append(p.detach().contiguous())
            image = self.packed_image_buffer(prec)
            arr = (C.c_void_p * len(srcs))(*[s.data_ptr() for s in srcs])
            fast = (ptrs, arr, image, dev, _lib.ptr(image), int(self.use_new_activation))
            # cache only when the kernels read the parameters' own storage (a non-contiguous parameter is copied per call)
            self._fast[prec] = fast if all(s.data_ptr() == q for s, q in zip(srcs, ptrs)) else None
        _, arr, image, dev, image_ptr, new_act = fast
        lib = _lib.load()
        # the image (and its header's check scratch) is shared by every stream that renders with this model: when the
        # stream changes, the new one first waits for what the previous one had enqueued (ADVICE r1: the image used to be
        # packed on the stream of first use and read from others with no ordering)
        stream = torch.cuda.current_stream(dev)
        last = self._last_stream.get(prec)
        if last is not None and last != stream:
            stream.wait_stream(last)
        self._last_stream[prec] = stream
        sp = C.c_void_p(stream.cuda_stream)
        if torch.cuda.current_device() == dev.index:
            _lib.check(lib.snb_refresh_weights(arr, prec, new_act, image_ptr, sp), "snb_refresh_weights")
        else:
            with torch.cuda.device(dev):
                _lib.check(lib.snb_refresh_weights(arr, prec, new_act, image_ptr, sp), "snb_refresh_weights")
        return image

    def packed_image_buffer(self, prec: int) -> torch.Tensor:
        """The (precision, device) image buffer, allocated zero-filled on first use; its CONTENT is brought up
        to date by packed_weights() / the fused optimisers' step()."""
        self._check_shape()
        ps = self._param_list()
        dev = ps[0].device
        _lib.require_device(ps[0], "NeRF")
        key = (prec, str(dev))
        image = self._packed.get(key)
        if image is None:
            nbytes = _lib.load().snb_packed_weights_bytes(prec)
            if nbytes == 0:
                raise NotImplementedError(f"precision mode {prec} is not available in this build")
            image = torch.zeros(nbytes, dtype=torch.uint8, device=dev)
            self._packed = {k: v for k, v in self._packed.items() if k[1] == str(dev)}   # drop images of old devices
            self._packed[key] = image
        return image

    def invalidate_packed(self) -> None:
        """Forget every packed image (they are rebuilt on the next pass).  Never needed for correctness --
        packed_weights() checks the parameter values itself -- only to release the buffers."""
        self._packed = {}
        self._fast = {}
        self._last_stream = {}

    def __getstate__(self):
        # the cached pointer table holds ctypes pointers (not picklable / meaningless in a copy): copy.deepcopy and
        # torch.save(model) get a module that re-validates on first use
        d = self.__dict__.copy()
        d["_fast"] = {}
        d["_last_stream"] = {}
        return d

    # ------------------------------------------------------------------ forward
    def forward(self, x, sigma_only=False):
        """x (B, 63(+27)) embedded position (and direction) -> (B,4) [rgb, sigma], or (B,1) sigma
        -- reference models/nerf.py:105-148."""
        _lib.require_device(x, "NeRF.forward")
        if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in self.parameters())):
            raise NotImplementedError(
                "sinnerf_b200.NeRF.forward runs the inference kernels and builds no autograd graph; gradients are "
                "wired through render_rays (the only differentiated caller in the reference, models/sinnerf.py:171-193). "
                "Call model(x) under torch.no_grad(), or train through render_rays.")
        need = self.in_channels_xyz if sigma_only else self.in_channels_xyz + self.in_channels_dir
        if x.dim() != 2 or x.shape[1] != need:
            raise ValueError(f"NeRF.forward: expected (B, {need}), got {tuple(x.shape)}")
        prec = config.resolve_precision()
        image = self.packed_weights(prec)
        xc = x.detach().to(torch.float32).contiguous()
        out = torch.empty(xc.shape[0], 1 if sigma_only else 4, device=x.device, dtype=torch.float32)
        with torch.cuda.device(x.device):
            _lib.check(_lib.load().snb_mlp_forward(_lib.ptr(image), prec, _lib.ptr(xc), xc.shape[1], xc.shape[0],
                                                   int(bool(sigma_only)), _lib.ptr(out),
                                                   _lib.stream_ptr(x.device)), "snb_mlp_forward")
        return out
