"""Times PF3plat's photometric training loss (LossMse + LossMultiSSIM), forward + backward, on one GPU: the fused
kernels of pf3plat_b200.losses against the reference's PyTorch op sequence (loss_multissim.py:45-86 + loss_mse.py:35:
a host-built window copied to the device on every call, five depthwise 11x11 conv2d, the SSIM map, autograd
backward) with cudnn.allow_tf32 on (PyTorch's default) and off.  The three variants alternate within one run.

Usage:  python scripts/bench_losses.py [--steps 50] [--warmup 10] [--repeats 5] [--out DIR]
Writes DIR/bench_losses.json (default: a temporary directory) and prints it.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys
import tempfile

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pf3plat_b200 import losses  # noqa: E402

SHAPES = {  # name: (images, channels, h, w)
    "pf3plat_train_14x3x256": (14, 3, 256, 256),   # color[:, 1:-1] of 14 scenes x 3 target views
    "val_video_60x3x256": (60, 3, 256, 256),
    "large_32x3x512": (32, 3, 512, 512),
}
# per element: the separable filter's FMAs -- forward 5 moments x 2 passes x 11 taps, backward the 4 maps back-filtered
# (4 x 2 x 11); the backward's recomputation of the moments is not counted (it is a choice, not a need)
FMA_PER_ELEMENT = 5 * 2 * 11 + 4 * 2 * 11
BYTES_PER_ELEMENT = 4 * (2 + 2 + 2)   # forward reads 2 images; backward reads 2 and writes 2 gradients


def torch_sequence(pred, gt):
    """The reference's loss as PyTorch ops (what PF3plat runs today), mse and 1 - ssim with weights 1.0 and 0.1."""
    c = pred.shape[-3]
    g = torch.tensor([math.exp(-((k - 5) ** 2) / (2 * 1.5 ** 2)) for k in range(11)])
    g = g / g.sum()
    win = (g[:, None] @ g[None, :]).expand(c, 1, 11, 11).contiguous().to(pred.device).type_as(pred)
    conv = lambda t: F.conv2d(t, win, padding=5, groups=c)
    mu1, mu2 = conv(pred), conv(gt)
    s11 = conv(pred * pred) - mu1 * mu1
    s22 = conv(gt * gt) - mu2 * mu2
    s12 = conv(pred * gt) - mu1 * mu2
    C1, C2 = 0.01 ** 2, 0.03 ** 2
    smap = ((2 * mu1 * mu2 + C1) * (2 * s12 + C2)) / ((mu1 * mu1 + mu2 * mu2 + C1) * (s11 + s22 + C2))
    return ((pred - gt) ** 2).mean(), 0.1 * (1 - smap.mean())


def ours(pred, gt):
    return losses.photometric_loss(pred, gt)


def card_info():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit_and_max_sm_clock"] = out
    except (OSError, subprocess.SubprocessError) as e:
        info["power_limit_and_max_sm_clock"] = f"unavailable: {e}"
    return info


def time_variant(fn, pred, gt, steps):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        pred.grad = None
        m, s = fn(pred, gt)
        (m + s).backward()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_losses.py needs a CUDA device")
    dev = torch.device("cuda:0")
    result = {"card": card_info(), "steps": args.steps, "repeats": args.repeats, "shapes": {}}
    variants = {"ours": (ours, None), "torch_tf32": (torch_sequence, True), "torch_fp32": (torch_sequence, False)}
    for name, (n, c, h, w) in SHAPES.items():
        g = torch.Generator(device=dev).manual_seed(0)
        gt = torch.rand(n, c, h, w, device=dev, generator=g)
        pred = (gt + 0.1 * torch.randn(n, c, h, w, device=dev, generator=g)).requires_grad_(True)
        # agreement of what is timed: ours against the fp32 PyTorch sequence
        torch.backends.cudnn.allow_tf32 = False
        m0, s0 = torch_sequence(pred, gt)
        (m0 + s0).backward()
        g0 = pred.grad.clone()
        pred.grad = None
        m1, s1 = ours(pred, gt)
        (m1 + s1).backward()
        agree = {"mse_abs": abs(float(m1.detach() - m0.detach())), "ssim_term_abs": abs(float(s1.detach() - s0.detach())),
                 "grad_max_abs": float((pred.grad - g0).abs().max()), "grad_max_ref": float(g0.abs().max())}
        times = {k: [] for k in variants}
        for k, (fn, tf32) in variants.items():   # warm every variant (cuDNN picks its algorithms here)
            if tf32 is not None:
                torch.backends.cudnn.allow_tf32 = tf32
            time_variant(fn, pred, gt, args.warmup)
        for _ in range(args.repeats):
            for k, (fn, tf32) in variants.items():
                if tf32 is not None:
                    torch.backends.cudnn.allow_tf32 = tf32
                times[k].append(time_variant(fn, pred, gt, args.steps))
        torch.backends.cudnn.allow_tf32 = True
        elems = n * c * h * w
        med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
        result["shapes"][name] = {
            "shape": [n, c, h, w], "ms_per_fwd_bwd_median": med, "ms_all": times,
            "speedup_vs_torch_tf32": med["torch_tf32"] / med["ours"], "speedup_vs_torch_fp32": med["torch_fp32"] / med["ours"],
            "compulsory_bytes": elems * BYTES_PER_ELEMENT, "filter_fmas": elems * FMA_PER_ELEMENT,
            "ours_GBps_compulsory": elems * BYTES_PER_ELEMENT / (med["ours"] * 1e6),
            "agreement_vs_torch_fp32": agree,
        }
        print(name, json.dumps(result["shapes"][name]["ms_per_fwd_bwd_median"]), flush=True)
    out = args.out or tempfile.mkdtemp(prefix="bench_losses_")
    os.makedirs(out, exist_ok=True)
    with open(os.path.join(out, "bench_losses.json"), "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
