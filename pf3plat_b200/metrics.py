"""Image metrics of the evaluation path (SURVEY.md section 8(f).4).

`compute_psnr`, `compute_lpips` and `compute_ssim` have the signatures and semantics of the reference's
(PF3plat's src/evaluation/metrics.py:11-19, :27-33, :38-54) and run on the device (gs_metrics.cu, gs_lpips.cu); the
reference's SSIM loops over images on the CPU through scikit-image.  `compute_lpips` takes the pretrained VGG weights
of the installed `lpips` package, as the reference does (pf3plat_b200.lpips.LPIPS)."""
from __future__ import annotations

import functools

import torch

from . import _capi
from .lpips import LPIPS


@torch.no_grad()
def compute_psnr(ground_truth: torch.Tensor, predicted: torch.Tensor) -> torch.Tensor:
    """(batch, channel, height, width) x 2 -> (batch,) PSNR in dB; inputs are clipped to [0, 1] (a NaN stays NaN, so
    an image holding one gets a NaN PSNR).  Computed in float32 and returned in torch.result_type(gt, pred), as the
    reference's tensor arithmetic returns it."""
    if ground_truth.shape != predicted.shape or ground_truth.dim() < 2:
        raise ValueError("compute_psnr expects two tensors of the same (batch, ...) shape")
    if predicted.device.type != "cuda":
        raise RuntimeError("pf3plat_b200.metrics needs CUDA tensors (there is no CPU fallback)")
    gt = ground_truth.detach().to(predicted.device, torch.float32).contiguous()
    pr = predicted.detach().to(torch.float32).contiguous()
    b = pr.shape[0]
    n = pr[0].numel() if b else 1
    L = _capi.lib()
    out = torch.empty((b,), dtype=torch.float32, device=pr.device)
    with torch.cuda.device(pr.device):
        scratch = torch.empty((max(1, int(L.gs_psnr_scratch_floats(b, n))),), dtype=torch.float32, device=pr.device)
        _capi.check(L.gs_psnr(gt.data_ptr(), pr.data_ptr(), b, n, scratch.data_ptr(), out.data_ptr(),
                              torch.cuda.current_stream(pr.device).cuda_stream))
    return out.to(torch.result_type(ground_truth, predicted))


@functools.cache
def get_lpips(device: torch.device) -> LPIPS:
    """One LPIPS-VGG module per device (metrics.py:22-24), in TF32 whatever lpips.set_precision says: a reported metric
    does not depend on a training-speed setting."""
    return LPIPS(net="vgg", precision="tf32").to(device)


@torch.no_grad()
def compute_lpips(ground_truth: torch.Tensor, predicted: torch.Tensor) -> torch.Tensor:
    """(batch, 3, height, width) x 2 -> (batch,) LPIPS-VGG distance, inputs in [0, 1] (normalize=True)."""
    value = get_lpips(predicted.device).forward(ground_truth, predicted, normalize=True)
    return value[:, 0, 0, 0]


@torch.no_grad()
def compute_ssim(ground_truth: torch.Tensor, predicted: torch.Tensor) -> torch.Tensor:
    """(batch, channel, height, width) x 2 -> (batch,) mean SSIM (Gaussian window, sigma 1.5, 11 taps, data range 1)."""
    if ground_truth.shape != predicted.shape or ground_truth.dim() != 4:
        raise ValueError("compute_ssim expects two (batch, channel, height, width) tensors of the same shape")
    if predicted.device.type != "cuda":
        raise RuntimeError("pf3plat_b200.metrics needs CUDA tensors (there is no CPU fallback)")
    gt = ground_truth.detach().to(predicted.device, torch.float32).contiguous()
    pr = predicted.detach().to(torch.float32).contiguous()
    b, c, h, w = pr.shape
    L = _capi.lib()
    out = torch.empty((b,), dtype=torch.float32, device=pr.device)
    with torch.cuda.device(pr.device):
        n = max(2, int(L.gs_ssim_scratch_floats(b, c, h, w)))
        scratch = torch.empty(((n + 1) // 2,), dtype=torch.float64, device=pr.device)
        _capi.check(L.gs_ssim(gt.data_ptr(), pr.data_ptr(), b, c, h, w, scratch.data_ptr(), out.data_ptr(),
                              torch.cuda.current_stream(pr.device).cuda_stream))
    return out.to(predicted.dtype)
