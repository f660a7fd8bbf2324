"""LPIPS-VGG restated in torch from F.conv2d / F.max_pool2d (no torchvision): the checker of csrc/gs_lpips.cu.

This restates the published `lpips` 0.1 package (LPIPS(net="vgg"), version "0.1", lpips=True, spatial=False).  That
package is not a dependency, so the definition is pinned only where it is importable (tests/test_lpips_cpu.py compares
against it live there):
  x <- 2x - 1 if normalize;  x <- (x - shift) / scale
  VGG16 features[0:30]: conv3x3 (pad 1, bias) + ReLU, 2x2/2 max-pools (floor); taps at relu1_2, relu2_2, relu3_3,
  relu4_3, relu5_3 (feature indices 3, 8, 15, 22, 29; slices [0:4] [4:9] [9:16] [16:23] [23:30])
  n = f / (sqrt(sum_c f^2) + 1e-10);  out = sum_l mean_{h,w} sum_c lin_l[c] (n0 - n1)^2      -> (N,)
Weights are a state dict under the package's key names.  Run it in float64 for the reference values; autograd gives
the gradients.  In float32 on a GPU (cudnn.allow_tf32 on or off) it is the op sequence PyTorch runs for the package.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

# torchvision vgg16().features[0:30]: "C" = conv3x3 + ReLU (2 entries), "M" = max-pool (1 entry)
VGG16_CFG = (64, 64, "M", 128, 128, "M", 256, 256, 256, "M", 512, 512, 512, "M", 512, 512, 512)
SLICES = ((0, 4), (4, 9), (9, 16), (16, 23), (23, 30))
TAP_INDICES = (3, 8, 15, 22, 29)           # the ReLU ending each slice
TAP_CHANNELS = (64, 128, 256, 512, 512)
EPS = 1e-10
SHIFT = (-.030, -.088, -.188)
SCALE = (.458, .448, .450)


def conv_layers():
    """-> [(feature index, cin, cout)] of the 13 convolutions of features[0:30]."""
    out, idx, cin = [], 0, 3
    for v in VGG16_CFG:
        if v == "M":
            idx += 1
        else:
            out.append((idx, cin, v))
            cin = v
            idx += 2
    return out


def _slice_of(idx):
    return next(k for k, (a, b) in enumerate(SLICES) if a <= idx < b)


def conv_keys():
    """State-dict keys of the 13 convolutions: [(weight key, bias key)] ("net.slice{k}.{feature index}.*")."""
    return [(f"net.slice{_slice_of(i) + 1}.{i}.weight", f"net.slice{_slice_of(i) + 1}.{i}.bias") for i, _, _ in conv_layers()]


def lin_keys():
    return [f"lin{k}.model.1.weight" for k in range(5)]


def random_state_dict(seed: int, bias_scale: float = 0.05) -> dict:
    """Seeded He-scaled conv weights (std sqrt(2 / (9 cin))), small biases, non-negative lin weights (as trained ones
    are), float32.  numpy's PCG64 stream, so the same seed gives the same weights on every machine."""
    rng = np.random.default_rng(seed)
    sd = {}
    for (wk, bk), (_, cin, cout) in zip(conv_keys(), conv_layers()):
        sd[wk] = torch.from_numpy((rng.standard_normal((cout, cin, 3, 3)) * np.sqrt(2.0 / (9 * cin))).astype(np.float32))
        sd[bk] = torch.from_numpy((rng.standard_normal(cout) * bias_scale).astype(np.float32))
    for k, c in zip(lin_keys(), TAP_CHANNELS):
        sd[k] = torch.from_numpy((rng.random(c) * 2.0 / c).astype(np.float32).reshape(1, c, 1, 1))
    sd["scaling_layer.shift"] = torch.tensor(SHIFT, dtype=torch.float32).reshape(1, 3, 1, 1)
    sd["scaling_layer.scale"] = torch.tensor(SCALE, dtype=torch.float32).reshape(1, 3, 1, 1)
    return sd


def features(x, sd):
    """Scaled input -> the five tap activations."""
    taps, convs, k = [], conv_keys(), 0
    idx = 0
    for v in VGG16_CFG:
        if v == "M":
            x = F.max_pool2d(x, 2, 2)
            idx += 1
            continue
        wk, bk = convs[k]
        x = F.relu(F.conv2d(x, sd[wk].to(x), sd[bk].to(x), padding=1))
        k += 1
        idx += 2
        if idx - 1 in TAP_INDICES:
            taps.append(x)
    return taps


def lpips(in0, in1, sd, normalize=False):
    """(N, 3, H, W) x 2 -> (N,), in the inputs' dtype and device; differentiable in both inputs."""
    if normalize:
        in0, in1 = 2 * in0 - 1, 2 * in1 - 1
    shift = sd["scaling_layer.shift"].to(in0).reshape(1, 3, 1, 1)
    scale = sd["scaling_layer.scale"].to(in0).reshape(1, 3, 1, 1)
    f0 = features((in0 - shift) / scale, sd)
    f1 = features((in1 - shift) / scale, sd)
    total = 0
    for a, b, lk in zip(f0, f1, lin_keys()):
        na = a / (torch.sqrt((a * a).sum(dim=1, keepdim=True)) + EPS)
        nb = b / (torch.sqrt((b * b).sum(dim=1, keepdim=True)) + EPS)
        d = F.conv2d((na - nb) ** 2, sd[lk].to(a).reshape(1, -1, 1, 1))
        total = total + d.mean(dim=(2, 3))
    return total[:, 0]


def with_grads(in0, in1, sd, normalize=False, dout=None, device=None, dtype=torch.float64):
    """-> (value (N,), dL/din0, dL/din1) for L = sum(dout * value) (dout = ones by default), computed in `dtype` on
    `device` (default: the inputs' device); results on the CPU."""
    device = device or in0.device
    a = in0.detach().to(device, dtype).requires_grad_(True)
    b = in1.detach().to(device, dtype).requires_grad_(True)
    v = lpips(a, b, sd, normalize)
    w = torch.ones_like(v) if dout is None else dout.to(v)
    ga, gb = torch.autograd.grad((v * w).sum(), (a, b))
    return v.detach().cpu(), ga.cpu(), gb.cpu()
