"""PF3plat's encoder depth glue between UniDepth and the networks and losses that read its output, on the device
(csrc/gs_encoder_depth.cu).

- `depth_update(depth, scale_shift, intrinsics, near, far, grid)` is encoder_costvolume.py:265, :285-287 (with
  `get_scaleshift`, :167-172) and the unprojections :304-307 / :506-528: the clamped depth plus the upsampled,
  clamped shift, clamped again, and its unprojection.  Forward and backward (into `scale_shift`).
- `mono_cue(depths, near, far, b, v)` is the one-hot mono cue of :292-298 (forward only; the reference detaches it).
- `pdf_peak(logits, upscale_factor)` is depth_predictor_multiview.py:379-384: max over D of softmax over D,
  nearest-upsampled.  Forward and backward; the [items, D, h, w] softmax is never stored.

None of them synchronises the device with the host, and every backward is a fixed-order gather without atomics, so it
is bit-reproducible with or without `torch.use_deterministic_algorithms`.  Inputs must be float32 CUDA tensors; there is
no CPU fallback.

Ties: `pdf_peak` takes the lowest index among equal maxima (PyTorch's CUDA `max(dim)` does not specify its choice;
only the gradient depends on it), and `mono_cue` the first smallest distance, as `torch.argmin` does.
"""
from __future__ import annotations

import torch

from . import _capi
from .poses import _check_cuda_float, _stream

MONO_CUE_BINS = _capi.GS_MONO_CUE_BINS
_LIN = {}  # device -> (pinned host table, device table, event recorded after the upload)


def _linspace_table(dev):
    """torch.linspace(0, 1, 128) as the CPU computes it, uploaded once per device without blocking the host; every
    later call's stream waits on the upload's event."""
    if dev not in _LIN:
        host = torch.linspace(0.0, 1.0, MONO_CUE_BINS).pin_memory()
        table = host.to(dev, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(dev))
        _LIN[dev] = (host, table, ev)
    _, table, ev = _LIN[dev]
    torch.cuda.current_stream(dev).wait_event(ev)
    return table


def _du_structs(depth, scale_shift, intrinsics, near, far, b, v, h, w, grid):
    return (_capi.GsDepthUpdateConfig(batch=b, views=v, height=h, width=w, grid_height=grid[0], grid_width=grid[1]),
            _capi.GsDepthUpdateInputs(depth=depth.data_ptr(), scale_shift=scale_shift.data_ptr(),
                                      intrinsics=intrinsics.data_ptr(), near_=near.data_ptr(), far_=far.data_ptr()))


class _DepthUpdate(torch.autograd.Function):
    @staticmethod
    def forward(ctx, scale_shift, depth, intrinsics, near, far, grid):
        b, v = near.shape
        h, w = depth.shape[-2:]
        dev = depth.device
        cfg, ins = _du_structs(depth, scale_shift, intrinsics, near, far, b, v, h, w, grid)
        depths = torch.empty_like(depth)
        xyz = torch.empty((b, v, 3, h, w), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _capi.check(_capi.lib().gs_depth_update_forward(cfg, ins, depths.data_ptr(), xyz.data_ptr(), _stream(dev)))
        ctx.save_for_backward(scale_shift, depth, intrinsics, near, far)
        ctx.grid = grid
        ctx.set_materialize_grads(False)
        return depths, xyz

    @staticmethod
    def backward(ctx, g_depths, g_xyz):
        if g_depths is None and g_xyz is None:
            return (None,) * 6
        scale_shift, depth, intrinsics, near, far = ctx.saved_tensors
        b, v = near.shape
        h, w = depth.shape[-2:]
        dev = depth.device
        cfg, ins = _du_structs(depth, scale_shift, intrinsics, near, far, b, v, h, w, ctx.grid)
        gd = g_depths.to(torch.float32).contiguous() if g_depths is not None else None
        gx = g_xyz.to(torch.float32).contiguous() if g_xyz is not None else None
        d_ss = torch.empty_like(scale_shift)
        grads = _capi.GsDepthUpdateGrads(dL_ddepths=gd.data_ptr() if gd is not None else None,
                                         dL_dxyz=gx.data_ptr() if gx is not None else None,
                                         dL_dscale_shift=d_ss.data_ptr())
        with torch.cuda.device(dev):
            _capi.check(_capi.lib().gs_depth_update_backward(cfg, ins, grads, _stream(dev)))
        return d_ss, None, None, None, None, None


def depth_update(depth: torch.Tensor, scale_shift: torch.Tensor, intrinsics: torch.Tensor, near: torch.Tensor,
                 far: torch.Tensor, grid):
    """encoder_costvolume.py:265, :285-287 and :304-307 / :506-528.  depth: UniDepth's predictions["depth"]
    [(b v), 1, h, w] (frozen: it must not require grad); scale_shift: the head's raw output [b, v, h_d w_d, 2] with
    grid = (h_d, w_d); intrinsics [b, v, 3, 3] normalised; near, far [b, v].  Returns (depths, xyz): depths
    [(b v), 1, h, w] is `depths` of :287 and, bit for bit, `depths_final` of :528; xyz [b, v, 3, h, w] is both
    `xyz_up_h` and `xyz_refine`.  Gradients from either output reach scale_shift (its channel 0, the unused scale,
    gets 0)."""
    _check_cuda_float("depth_update: depth", depth)
    dev = depth.device
    for name, t in (("scale_shift", scale_shift), ("intrinsics", intrinsics), ("near", near), ("far", far)):
        _check_cuda_float(f"depth_update: {name}", t, dev)
    gh, gw = (int(x) for x in grid)
    if near.dim() != 2 or tuple(far.shape) != tuple(near.shape) or near.shape[0] < 1 or near.shape[1] < 1:
        raise ValueError(f"depth_update needs near and far [b, v], got {tuple(near.shape)}, {tuple(far.shape)}")
    b, v = near.shape
    if depth.dim() != 4 or depth.shape[0] != b * v or depth.shape[1] != 1 or depth.shape[2] < 1 or depth.shape[3] < 1:
        raise ValueError(f"depth_update needs depth [(b v), 1, h, w] with b v = {b * v}, got {tuple(depth.shape)}")
    if gh < 1 or gw < 1 or tuple(scale_shift.shape) != (b, v, gh * gw, 2):
        raise ValueError(f"depth_update needs scale_shift [b, v, h_d w_d, 2] = [{b}, {v}, {gh * gw}, 2] for grid "
                         f"{(gh, gw)}, got {tuple(scale_shift.shape)}")
    if tuple(intrinsics.shape) != (b, v, 3, 3):
        raise ValueError(f"depth_update needs intrinsics [b, v, 3, 3], got {tuple(intrinsics.shape)}")
    if depth.requires_grad:
        raise ValueError("depth_update: depth must not require grad (UniDepth is frozen)")
    if intrinsics.requires_grad or near.requires_grad or far.requires_grad:
        raise ValueError("depth_update: intrinsics, near and far must not require grad")
    return _DepthUpdate.apply(scale_shift.contiguous(), depth.contiguous(), intrinsics.contiguous(), near.contiguous(),
                              far.contiguous(), (gh, gw))


def mono_cue(depths: torch.Tensor, near: torch.Tensor, far: torch.Tensor, b: int, v: int) -> torch.Tensor:
    """encoder_costvolume.py:292-298: depths [(b v), 1, h, w] (h and w multiples of 4), near and far [b, v].
    Returns the detached one-hot [(v b), 128, h/4, w/4] over the hypotheses 1/far + linspace(0, 1, 128) (1/near -
    1/far) of scene 0, view 0, compared against the ÷4 bilinear downsample of depths, as the reference writes it."""
    _check_cuda_float("mono_cue: depths", depths)
    dev = depths.device
    _check_cuda_float("mono_cue: near", near, dev)
    _check_cuda_float("mono_cue: far", far, dev)
    b, v = int(b), int(v)
    if b < 1 or v < 1 or tuple(near.shape) != (b, v) or tuple(far.shape) != (b, v):
        raise ValueError(f"mono_cue needs near and far [b, v] = [{b}, {v}], got {tuple(near.shape)}, "
                         f"{tuple(far.shape)}")
    if depths.dim() != 4 or depths.shape[0] != b * v or depths.shape[1] != 1:
        raise ValueError(f"mono_cue needs depths [(b v), 1, h, w] with b v = {b * v}, got {tuple(depths.shape)}")
    h, w = depths.shape[-2:]
    if h < 4 or w < 4 or h % 4 or w % 4:
        raise ValueError(f"mono_cue needs h and w to be positive multiples of 4 (the exact ÷4 downsample), got {h} x {w}")
    d = depths.detach().contiguous()
    out = torch.empty((v * b, MONO_CUE_BINS, h // 4, w // 4), dtype=torch.float32, device=dev)
    cfg = _capi.GsMonoCueConfig(batch=b, views=v, height=h, width=w)
    with torch.cuda.device(dev):
        lin = _linspace_table(dev)
        nr, fr = near.detach().contiguous(), far.detach().contiguous()
        _capi.check(_capi.lib().gs_mono_cue(cfg, d.data_ptr(), nr.data_ptr(), fr.data_ptr(), lin.data_ptr(),
                                            out.data_ptr(), _stream(dev)))
    return out


class _PdfPeak(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, s):
        n, D, h, w = logits.shape
        dev = logits.device
        cfg = _capi.GsPdfPeakConfig(items=n, depth_candidates=D, height=h, width=w, upscale=s)
        out = torch.empty((n, 1, h * s, w * s), dtype=torch.float32, device=dev)
        peak = torch.empty((n, h, w), dtype=torch.float32, device=dev)
        arg = torch.empty((n, h, w), dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            _capi.check(_capi.lib().gs_pdf_peak_forward(cfg, logits.data_ptr(), out.data_ptr(), peak.data_ptr(),
                                                        arg.data_ptr(), _stream(dev)))
        ctx.save_for_backward(logits, peak, arg)
        ctx.s = s
        ctx.mark_non_differentiable(peak, arg)
        ctx.set_materialize_grads(False)
        return out

    @staticmethod
    def backward(ctx, g_out):
        if g_out is None:
            return None, None
        logits, peak, arg = ctx.saved_tensors
        n, D, h, w = logits.shape
        dev = logits.device
        cfg = _capi.GsPdfPeakConfig(items=n, depth_candidates=D, height=h, width=w, upscale=ctx.s)
        g = g_out.to(torch.float32).contiguous()
        d_logits = torch.empty_like(logits)
        with torch.cuda.device(dev):
            _capi.check(_capi.lib().gs_pdf_peak_backward(cfg, logits.data_ptr(), peak.data_ptr(), arg.data_ptr(),
                                                         g.data_ptr(), d_logits.data_ptr(), _stream(dev)))
        return d_logits, None


def pdf_peak(logits: torch.Tensor, upscale_factor: int = 4) -> torch.Tensor:
    """depth_predictor_multiview.py:379-384: logits [items, D, h, w] (depth_head_lowres's output) -> pdf_max
    [items, 1, h s, w s] = nearest-upsampled max over D of softmax over D, with s = upscale_factor (a positive
    integer).  Differentiable in logits; the argmax ties to the lowest index."""
    _check_cuda_float("pdf_peak: logits", logits)
    s = int(upscale_factor)
    if s != upscale_factor or s < 1:
        raise ValueError(f"pdf_peak needs a positive integer upscale_factor, got {upscale_factor!r}")
    if logits.dim() != 4 or min(logits.shape) < 1:
        raise ValueError(f"pdf_peak needs logits [items, D, h, w], got {tuple(logits.shape)}")
    return _PdfPeak.apply(logits.contiguous(), s)
