"""fp64 restatement of PF3plat's photometric training loss, for the parity tests of pf3plat_b200.losses.

TEST INFRASTRUCTURE ONLY (imported by tests/, never by the product path).

Semantics of src/loss/loss_multissim.py:45-86 and loss_mse.py:35, written independently here: per image and channel
plane, a zero-padded 11x11 Gaussian filter (sigma 1.5) with a full H x W output gives the local moments
  ux = w*x, uy = w*y, vx = w*(x^2) - ux^2, vy = w*(y^2) - uy^2, vxy = w*(xy) - ux uy      (population covariance)
and S = (2 ux uy + C1)(2 vxy + C2) / ((ux^2 + uy^2 + C1)(vx + vy + C2)), C1 = 0.01^2, C2 = 0.03^2, no clipping.
ssim per image = mean of S over (c, h, w); mse per image = mean of (x - y)^2.

Two windows:
  * the default is the exact Gaussian, applied as a separable filter (what the kernels compute);
  * `reference_window()` is the 11x11 window the reference builds (create_window, :50-55): 1-D taps rounded to float32,
    normalised in float32, their outer product rounded to float32, and only then cast to the input's dtype
    (`window.type_as(img1)`).  Passing it reproduces the reference's fp64 run to rounding, as the golden fixture
    comparison needs; it differs from the exact window by ~1e-7 relative.
Gradients come from autograd through these ops, or from `closed_form_backward` (the formulas gs_losses.cu implements).
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

WIN, RADIUS, SIGMA = 11, 5, 1.5
C1, C2 = 0.01 ** 2, 0.03 ** 2


def gaussian_taps(dtype=torch.float64) -> torch.Tensor:
    k = torch.arange(WIN, dtype=torch.float64) - RADIUS
    g = torch.exp(-k * k / (2 * SIGMA ** 2))
    return (g / g.sum()).to(dtype)


def reference_window() -> torch.Tensor:
    """(11, 11) float64 holding the float32 values of the reference's window."""
    g = torch.tensor([math.exp(-((x - RADIUS) ** 2) / (2 * SIGMA ** 2)) for x in range(WIN)], dtype=torch.float32)
    g = g / g.sum()
    return (g[:, None] * g[None, :]).to(torch.float64)


def filt(a: torch.Tensor, window: torch.Tensor | None = None) -> torch.Tensor:
    """Zero-padded 'same' filter over the last two dims: separable with the exact taps, or direct with a 2-D window."""
    h, w = a.shape[-2:]
    p = F.pad(a, (RADIUS, RADIUS, RADIUS, RADIUS))
    if window is None:
        g = gaussian_taps(a.dtype).to(a.device)
        rows = sum(g[k] * p[..., :, k:k + w] for k in range(WIN))
        return sum(g[k] * rows[..., k:k + h, :] for k in range(WIN))
    window = window.to(a.dtype).to(a.device)
    return sum(window[i, j] * p[..., i:i + h, j:j + w] for i in range(WIN) for j in range(WIN))


def moments(x, y, window=None):
    ux, uy = filt(x, window), filt(y, window)
    vx = filt(x * x, window) - ux * ux
    vy = filt(y * y, window) - uy * uy
    vxy = filt(x * y, window) - ux * uy
    return ux, uy, vx, vy, vxy


def ssim_map(x: torch.Tensor, y: torch.Tensor, window=None) -> torch.Tensor:
    ux, uy, vx, vy, vxy = moments(x, y, window)
    return ((2 * ux * uy + C1) * (2 * vxy + C2)) / ((ux * ux + uy * uy + C1) * (vx + vy + C2))


def ssim_per_image(x, y, window=None) -> torch.Tensor:
    """(n, c, h, w) x 2 -> (n,)  (= ssim(..., size_average=False))"""
    return ssim_map(x, y, window).flatten(1).mean(1)


def mse_per_image(x, y) -> torch.Tensor:
    return ((x - y) ** 2).flatten(1).mean(1)


def _t(a):
    return a if torch.is_tensor(a) else torch.as_tensor(np.asarray(a))


def per_image_with_grads(x, y, d_ssim=None, d_mse=None, window=None):
    """fp64 values and autograd gradients of L = sum(d_ssim * ssim_i) + sum(d_mse * mse_i).
    -> (ssim (n,), mse (n,), dL/dx, dL/dy) as float64 tensors."""
    x = _t(x).to(torch.float64).clone().requires_grad_(True)
    y = _t(y).to(torch.float64).clone().requires_grad_(True)
    s, m = ssim_per_image(x, y, window), mse_per_image(x, y)
    loss = 0.0
    if d_ssim is not None:
        loss = loss + (s * _t(d_ssim).to(torch.float64)).sum()
    if d_mse is not None:
        loss = loss + (m * _t(d_mse).to(torch.float64)).sum()
    gx, gy = torch.autograd.grad(loss, (x, y), allow_unused=True) if torch.is_tensor(loss) else (None, None)
    z = lambda g, t: torch.zeros_like(t) if g is None else g
    return s.detach(), m.detach(), z(gx, x).detach(), z(gy, y).detach()


def closed_form_backward(x, y, d_ssim, d_mse=None, window=None):
    """The backward gs_losses.cu implements, in fp64.  g = d_ssim / (c h w) per map pixel:
      alpha = -g S / B2, beta = 2 g A1 / (B1 B2), gamma_x = g S (2 uy / A1 - 2 ux / B1) - 2 ux alpha - uy beta
      dL/dx = w*gamma_x + 2x (w*alpha) + y (w*beta)   (x <-> y for dL/dy),  plus 2 (x - y) d_mse / (c h w).
    The maps live on the image only (zero outside it before the back-filter): filt() zero-pads them."""
    x, y = _t(x).to(torch.float64), _t(y).to(torch.float64)
    n = x[0].numel()
    g = (_t(d_ssim).to(torch.float64) / n).reshape(-1, 1, 1, 1)
    ux, uy, vx, vy, vxy = moments(x, y, window)
    A1, A2 = 2 * ux * uy + C1, 2 * vxy + C2
    B1, B2 = ux * ux + uy * uy + C1, vx + vy + C2
    S = A1 * A2 / (B1 * B2)
    alpha = -g * S / B2
    beta = 2 * g * A1 / (B1 * B2)
    t1 = 2 * g * A2 / (B1 * B2)           # g S 2/A1 without dividing by A1 (which may vanish off [0, 1])
    gx = t1 * uy - 2 * g * S * ux / B1 - 2 * ux * alpha - uy * beta
    gy = t1 * ux - 2 * g * S * uy / B1 - 2 * uy * alpha - ux * beta
    # the window is symmetric, so the adjoint of the filter is the filter itself
    wa, wb = filt(alpha, window), filt(beta, window)
    dx = filt(gx, window) + 2 * x * wa + y * wb
    dy = filt(gy, window) + 2 * y * wa + x * wb
    if d_mse is not None:
        m = (2 * _t(d_mse).to(torch.float64) / n).reshape(-1, 1, 1, 1) * (x - y)
        dx, dy = dx + m, dy - m
    return dx, dy
