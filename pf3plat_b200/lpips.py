"""LPIPS-VGG on the device (csrc/gs_lpips.cu): a drop-in for `from lpips import LPIPS` at PF3plat's
src/loss/loss_lpips.py:6 and src/evaluation/metrics.py:6.

`LPIPS(net="vgg", weights=None)` computes the `lpips` 0.1 package's LPIPS(net="vgg") distance (lpips=True,
spatial=False) with hand-written sm_90a kernels: TF32 tensor-core convolutions, fp32 everywhere else.  It is
differentiable in both inputs (the weights are constants, as PF3plat's convert_to_buffer makes them).

Weights: `weights` is a state dict or a path to one under the package's key names (`scaling_layer.{shift,scale}`,
`net.slice{k}.{i}.{weight,bias}`, `lin{k}.model.1.weight` or `lins.{k}.model.1.weight`).  With None they are taken from
the installed `lpips` package, as the reference does.  The module holds them under those names, so `.to()`,
`load_state_dict` and convert_to_buffer keep working; they are packed into the kernels' layouts lazily, once per device,
and packed again whenever a weight tensor is replaced or modified in place.  Inputs must be float32 CUDA tensors of at
least 16 x 16 pixels; there is no CPU fallback.
"""
from __future__ import annotations

import ctypes
import functools

import torch
from torch import nn

from . import _capi
from .losses import _layout

# VGG16 features[0:30]: (feature index, cin, cout) of the 13 convolutions; slices [0:4] [4:9] [9:16] [16:23] [23:30]
_CONVS = ((0, 3, 64), (2, 64, 64), (5, 64, 128), (7, 128, 128), (10, 128, 256), (12, 256, 256), (14, 256, 256),
          (17, 256, 512), (19, 512, 512), (21, 512, 512), (24, 512, 512), (26, 512, 512), (28, 512, 512))
_SLICE_ENDS = (4, 9, 16, 23, 30)
_TAP_CHANNELS = (64, 128, 256, 512, 512)
_SHIFT = (-.030, -.088, -.188)
_SCALE = (.458, .448, .450)


def _slice_of(idx: int) -> int:
    return next(k for k, end in enumerate(_SLICE_ENDS) if idx < end) + 1


CONV_KEYS = tuple((f"net.slice{_slice_of(i)}.{i}.weight", f"net.slice{_slice_of(i)}.{i}.bias") for i, _, _ in _CONVS)
LIN_KEYS = tuple(f"lin{k}.model.1.weight" for k in range(5))


class _Conv(nn.Module):
    def __init__(self, cin, cout):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(cout, cin, 3, 3))
        self.bias = nn.Parameter(torch.empty(cout))


class _Weight(nn.Module):
    def __init__(self, *shape):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(*shape))


class _Lin(nn.Module):  # the package's NetLinLayer: model = [Dropout, Conv2d(c, 1, 1, bias=False)]
    def __init__(self, c):
        super().__init__()
        self.model = nn.ModuleDict({"1": _Weight(1, c, 1, 1)})


class _Scaling(nn.Module):
    def __init__(self):
        super().__init__()
        self.register_buffer("shift", torch.tensor(_SHIFT).reshape(1, 3, 1, 1))
        self.register_buffer("scale", torch.tensor(_SCALE).reshape(1, 3, 1, 1))


def _package_state_dict() -> dict:
    try:
        import lpips as lpips_package
    except ImportError as e:
        raise ImportError("pf3plat_b200.lpips.LPIPS(weights=None) takes the pretrained weights of the `lpips` package, "
                          "which is not installed: pass weights= a state dict (or a path to one) under the package's "
                          "key names") from e
    return lpips_package.LPIPS(net="vgg", version="0.1", verbose=False).state_dict()


def canonical_state_dict(sd: dict) -> dict:
    """The package's key names in every spelling it uses: `lins.{k}.*` and `lin{k}.*` are the same tensors, and a dict
    without the scaling layer gets the package's constants."""
    sd = dict(sd)
    for k in range(5):
        a, b = f"lin{k}.model.1.weight", f"lins.{k}.model.1.weight"
        if a not in sd and b in sd:
            sd[a] = sd[b]
        if b not in sd and a in sd:
            sd[b] = sd[a]
    sd.setdefault("scaling_layer.shift", torch.tensor(_SHIFT).reshape(1, 3, 1, 1))
    sd.setdefault("scaling_layer.scale", torch.tensor(_SCALE).reshape(1, 3, 1, 1))
    return sd


class _Pack:
    """Packed weights on one device (gs_lpips_weights_create); freed with the object."""

    def __init__(self, tensors, device):
        L = _capi.lib()
        # float32 copies on the device; packing is stream-ordered, so they may be freed once it is enqueued
        src = [t.detach().to(device, torch.float32).contiguous() for t in tensors]
        ptrs = [t.data_ptr() for t in src]
        cw = (ctypes.c_void_p * 13)(*ptrs[0:26:2])
        cb = (ctypes.c_void_p * 13)(*ptrs[1:26:2])
        lin = (ctypes.c_void_p * 5)(*ptrs[26:31])
        handle = ctypes.c_void_p()
        with torch.cuda.device(device):
            _capi.check(L.gs_lpips_weights_create(cw, cb, lin, ptrs[31], ptrs[32],
                                                  torch.cuda.current_stream(device).cuda_stream, ctypes.byref(handle)))
        self.handle = handle.value

    def __del__(self):
        if getattr(self, "handle", None):
            _capi.lib().gs_lpips_weights_destroy(self.handle)
            self.handle = None


class _LpipsFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, in0, in1, pack, normalize, grads):
        a, n, chw, sa = _layout(in0)
        b, _, _, sb = _layout(in1)
        _, h, w = chw
        cfg = _capi.GsLpipsConfig(batch=n, height=h, width=w, normalize=int(bool(normalize)), in0_stride=sa, in1_stride=sb,
                                  grads=grads)
        dev = in0.device
        L = _capi.lib()
        out = torch.empty((n,), dtype=torch.float32, device=dev)
        ws = None
        if n:
            with torch.cuda.device(dev):
                nbytes = int(L.gs_lpips_workspace_bytes(ctypes.byref(cfg)))
                ws = torch.empty((nbytes,), dtype=torch.uint8, device=dev)
                _capi.check(L.gs_lpips_forward(pack.handle, ctypes.byref(cfg), a.data_ptr(), b.data_ptr(), ws.data_ptr(),
                                               out.data_ptr(), torch.cuda.current_stream(dev).cuda_stream))
        ctx.cfg, ctx.pack, ctx.ws = cfg, pack, (ws if grads else None)
        ctx.shapes = (in0.shape, in1.shape)
        ctx.set_materialize_grads(False)
        return out

    @staticmethod
    def backward(ctx, dout):
        need0, need1 = ctx.needs_input_grad[:2]
        if dout is None or not (need0 or need1):
            return None, None, None, None, None
        cfg, dev = ctx.cfg, dout.device
        n, h, w = cfg.batch, cfg.height, cfg.width
        g0 = torch.empty((n, 3, h, w), dtype=torch.float32, device=dev) if need0 else None
        g1 = torch.empty((n, 3, h, w), dtype=torch.float32, device=dev) if need1 else None
        if n:
            d = dout.to(torch.float32).contiguous()  # a device array (the grad of .mean() is an expanded view)
            ptr = lambda t: t.data_ptr() if t is not None else None
            with torch.cuda.device(dev):
                _capi.check(_capi.lib().gs_lpips_backward(ctx.pack.handle, ctypes.byref(cfg), d.data_ptr(), ctx.ws.data_ptr(),
                                                          ptr(g0), ptr(g1), torch.cuda.current_stream(dev).cuda_stream))
        s0, s1 = ctx.shapes
        return (g0.reshape(s0) if g0 is not None else None), (g1.reshape(s1) if g1 is not None else None), None, None, None


class LPIPS(nn.Module):
    """LPIPS(net="vgg") of the `lpips` package on the device.  forward(in0, in1, retPerLayer=False, normalize=False)
    -> (N, 1, 1, 1) for (N, 3, H, W) inputs ((B, V, 1, 1, 1) for (B, V, 3, H, W))."""

    def __init__(self, net: str = "vgg", weights=None, **unused_package_options):
        super().__init__()
        if net != "vgg":
            raise NotImplementedError(f"only net='vgg' is implemented, got {net!r}")
        self.scaling_layer = _Scaling()
        self.net = nn.Module()
        for k in range(1, 6):
            setattr(self.net, f"slice{k}", nn.Module())
        for i, cin, cout in _CONVS:
            getattr(self.net, f"slice{_slice_of(i)}").add_module(str(i), _Conv(cin, cout))
        for k, c in enumerate(_TAP_CHANNELS):
            setattr(self, f"lin{k}", _Lin(c))
        self.lins = nn.ModuleList([getattr(self, f"lin{k}") for k in range(5)])
        if weights is None:
            weights = _package_state_dict()
        elif isinstance(weights, (str, bytes)) or hasattr(weights, "__fspath__"):
            weights = torch.load(weights, map_location="cpu")
        with torch.no_grad():
            self.load_state_dict(canonical_state_dict(weights), strict=True)
        self._packs = {}

    def _tensors(self):
        get = lambda key: functools.reduce(getattr, key.split("."), self)
        keys = [k for pair in CONV_KEYS for k in pair] + list(LIN_KEYS) + ["scaling_layer.shift", "scaling_layer.scale"]
        return [get(k) for k in keys]

    def _pack(self, device) -> _Pack:
        """The packed weights for `device`, packed again if any weight tensor was replaced or changed in place (the
        cache holds the tensors it packed, so identity and version counter decide)."""
        tensors = self._tensors()
        sig = [(t, t._version) for t in tensors]
        hit = self._packs.get(device)
        if hit is not None and len(hit[0]) == len(sig) and all(a is b and va == vb for (a, va), (b, vb) in zip(hit[0], sig)):
            return hit[1]
        pack = _Pack(tensors, device)
        self._packs[device] = (sig, pack)
        return pack

    def forward(self, in0: torch.Tensor, in1: torch.Tensor, retPerLayer: bool = False, normalize: bool = False):
        if retPerLayer:
            raise NotImplementedError("retPerLayer=True is not implemented")
        if not (torch.is_tensor(in0) and torch.is_tensor(in1)) or in0.shape != in1.shape or in0.dim() not in (4, 5):
            raise ValueError("LPIPS expects two tensors of the same (n, 3, h, w) or (b, v, 3, h, w) shape")
        if in0.device.type != "cuda" or in1.device != in0.device:
            raise RuntimeError("pf3plat_b200.lpips needs both images on the same CUDA device (there is no CPU fallback)")
        if in0.dtype != torch.float32 or in1.dtype != torch.float32:
            raise TypeError(f"pf3plat_b200.lpips needs float32 images, got {in0.dtype} and {in1.dtype}")
        c, h, w = in0.shape[-3:]
        if c != 3 or h < 16 or w < 16:
            raise ValueError(f"LPIPS needs 3-channel images of at least 16 x 16 pixels, got {tuple(in0.shape)}")
        # which input gradients the backward may be asked for decides what the forward keeps
        grads = (int(in0.requires_grad) | 2 * int(in1.requires_grad)) if torch.is_grad_enabled() else 0
        out = _LpipsFn.apply(in0, in1, self._pack(in0.device), normalize, grads)
        return out.reshape(tuple(in0.shape[:-3]) + (1, 1, 1))
