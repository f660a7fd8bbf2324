"""PF3plat's photometric training loss on the device (csrc/gs_losses.cu).

Every PF3plat training config trains with `loss: [lpips, mse, multissim, pose]`.  This module covers the two
photometric terms:
  * `ssim`  -- drop-in for `ssim` of PF3plat's src/loss/loss_multissim.py:57-65 (one scale of SSIM despite the module's
               name: zero-padded 11x11 Gaussian window, sigma 1.5, population covariance, no clipping);
  * `photometric_loss` -- `LossMse` (loss_mse.py:35) + `LossMultiSSIM` (loss_multissim.py:41-43) in one forward and one
               backward kernel, each term already weighted as the reference logs it (`loss/mse`, `loss/MultiSSIM`).
Both are differentiable with respect to both images.  LPIPS is `pf3plat_b200.lpips.LPIPS`; the pose loss (encoder side)
is not here.  Inputs must be float32 CUDA tensors; there is no CPU fallback.
"""
from __future__ import annotations

import torch

from . import _capi

_WINDOW = 11


def _layout(t: torch.Tensor):
    """-> (tensor to read, n images, (c, h, w), floats between images).  (n,c,h,w) or (b,v,c,h,w) inputs whose (c,h,w)
    blocks are contiguous and whose batch dimensions collapse to one stride (e.g. color[:, 1:-1] with b == 1, or any
    contiguous tensor) are read in place; anything else is copied to a contiguous tensor first."""
    if t.dim() not in (4, 5):
        raise ValueError(f"expected a (n, c, h, w) or (b, v, c, h, w) tensor, got shape {tuple(t.shape)}")
    lead, chw = t.shape[:-3], t.shape[-3:]
    n = 1
    for s in lead:
        n *= s
    if n == 0:
        return t, 0, tuple(chw), 0
    numel = chw[0] * chw[1] * chw[2]
    block_ok = t[(0,) * len(lead)].is_contiguous()
    dims = [(s, st) for s, st in zip(lead, t.stride()[:-3]) if s != 1]
    stride = dims[-1][1] if dims else numel
    collapses = all(dims[i][1] == dims[i + 1][0] * dims[i + 1][1] for i in range(len(dims) - 1))
    if not (block_ok and collapses and stride >= numel):
        t = t.contiguous()
        stride = numel
    return t, n, tuple(chw), stride


def _check(a: torch.Tensor, b: torch.Tensor):
    if not (torch.is_tensor(a) and torch.is_tensor(b)) or a.shape != b.shape or a.dim() not in (4, 5):
        raise ValueError("expected two tensors of the same (n, c, h, w) or (b, v, c, h, w) shape")
    if a.device.type != "cuda" or b.device != a.device:
        raise RuntimeError("pf3plat_b200.losses needs both images on the same CUDA device (there is no CPU fallback)")
    if a.dtype != torch.float32 or b.dtype != torch.float32:
        raise TypeError(f"pf3plat_b200.losses needs float32 images, got {a.dtype} and {b.dtype}")


def _config(n, chw, sp, sg):
    c, h, w = chw
    return _capi.GsLossConfig(batch=n, channels=c, height=h, width=w, pred_stride=sp, gt_stride=sg, with_mse=1)


class _Photometric(torch.autograd.Function):
    """(pred, gt) -> per-image (ssim, mse), each (n,); one forward and one backward kernel for both."""

    @staticmethod
    def forward(ctx, pred, gt):
        p, n, chw, sp = _layout(pred)
        g, _, _, sg = _layout(gt)
        cfg = _config(n, chw, sp, sg)
        L = _capi.lib()
        dev = pred.device
        ssim = torch.empty((n,), dtype=torch.float32, device=dev)
        mse = torch.empty((n,), dtype=torch.float32, device=dev)
        if n:
            with torch.cuda.device(dev):
                nbytes = int(L.gs_photometric_scratch_bytes(cfg))
                scratch = torch.empty((max(1, nbytes // 8),), dtype=torch.float64, device=dev)
                _capi.check(L.gs_photometric_forward(cfg, p.data_ptr(), g.data_ptr(), scratch.data_ptr(), ssim.data_ptr(),
                                                     mse.data_ptr(), torch.cuda.current_stream(dev).cuda_stream))
        ctx.save_for_backward(pred, gt)
        ctx.set_materialize_grads(False)
        return ssim, mse

    @staticmethod
    def backward(ctx, d_ssim, d_mse):
        pred, gt = ctx.saved_tensors
        need_p, need_g = ctx.needs_input_grad[:2]
        if not (need_p or need_g) or (d_ssim is None and d_mse is None):
            return None, None
        p, n, chw, sp = _layout(pred)
        g, _, _, sg = _layout(gt)
        cfg = _config(n, chw, sp, sg)
        dev = pred.device
        # incoming gradients go to the kernel as device arrays (an expanded grad of .mean() has stride 0)
        ds = d_ssim.to(torch.float32).contiguous() if d_ssim is not None else None
        dm = d_mse.to(torch.float32).contiguous() if d_mse is not None else None
        gp = torch.empty(pred.shape, dtype=torch.float32, device=dev) if need_p else None
        gg = torch.empty(gt.shape, dtype=torch.float32, device=dev) if need_g else None
        if n:
            ptr = lambda t: t.data_ptr() if t is not None else None
            with torch.cuda.device(dev):
                _capi.check(_capi.lib().gs_photometric_backward(cfg, p.data_ptr(), g.data_ptr(), ptr(ds), ptr(dm), ptr(gp),
                                                                ptr(gg), None, torch.cuda.current_stream(dev).cuda_stream))
        return gp, gg


def _per_image(img1, img2):
    _check(img1, img2)
    s, m = _Photometric.apply(img1, img2)
    lead = img1.shape[:-3]
    return s.reshape(lead), m.reshape(lead)


def ssim(img1: torch.Tensor, img2: torch.Tensor, window_size: int = 11, size_average: bool = True) -> torch.Tensor:
    """`ssim` of loss_multissim.py:57-65: the mean SSIM over (n, c, h, w) if size_average, else the mean per image,
    shape (n,) (or (b, v) for (b, v, c, h, w) inputs).  Differentiable with respect to both images."""
    if window_size != _WINDOW:
        raise ValueError(f"only window_size=11 is implemented (the reference's default), got {window_size}")
    s, _ = _per_image(img1, img2)
    return s.mean() if size_average else s


def photometric_loss(prediction: torch.Tensor, target: torch.Tensor, mse_weight: float = 1.0, ssim_weight: float = 0.1):
    """-> (mse_term, ssim_term) = (mse_weight * mean((prediction - target)^2), ssim_weight * (1 - ssim(prediction, target))),
    i.e. LossMse and LossMultiSSIM of PF3plat with its default weights (config/loss/mse.yaml, multissim.yaml).  Pass
    `color[:, 1:-1]` and `image[:, 1:-1]` as the reference's losses do."""
    s, m = _per_image(prediction, target)
    return mse_weight * m.mean(), ssim_weight * (1.0 - s.mean())
