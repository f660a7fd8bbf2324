"""Times LPIPS-VGG's BF16 path on one GPU against our TF32 path and PyTorch, on bench_lpips.py's shapes.  Four variants
alternate within one run:
  ours_tf32           LPIPS(precision="tf32"): TF32 mma.sync convolutions, fp32 activations (the default)
  ours_bf16           LPIPS(precision="bf16"): BF16 wgmma convolutions, BF16 activations and inter-layer gradients
  torch_autocast_bf16 the `lpips` package's op sequence (oracle/lpips_oracle.py) under torch.autocast(bfloat16): cuDNN
  torch_tf32          the same sequence in float32 with cudnn.allow_tf32 (PyTorch's default)
For each: median ms, TFLOP/s on bench_lpips.py's FLOP count, peak memory above the inputs, and for ours the time per
kernel of one profiled step.  The card's name, power limit and clocks are recorded in the same run.

Usage:  python scripts/bench_lpips_bf16.py [--steps 20] [--warmup 5] [--repeats 5] [--shapes a,b] [--out DIR]
Writes DIR/bench_lpips_bf16.json (default: a temporary directory) and prints a summary.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import bench_lpips as bl  # noqa: E402
from oracle import lpips_oracle as lo  # noqa: E402
from pf3plat_b200 import lpips as pl  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--shapes", default=",".join(bl.SHAPES))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lpips_bf16.py needs a CUDA device")
    dev = torch.device("cuda:0")
    sd = lo.random_state_dict(0)
    m32 = pl.LPIPS(weights=sd, precision="tf32").to(dev)
    m16 = pl.LPIPS(weights=sd, precision="bf16").to(dev)
    sd_dev = {k: v.to(dev) for k, v in sd.items()}
    torch_seq = lambda a, b: lo.lpips(a, b, sd_dev, normalize=True)

    def autocast_seq(a, b):
        with torch.autocast("cuda", dtype=torch.bfloat16):
            return torch_seq(a, b)

    variants = {  # name: (fn, cudnn.allow_tf32)
        "ours_tf32": (lambda a, b: m32(a, b, normalize=True), True),
        "ours_bf16": (lambda a, b: m16(a, b, normalize=True), True),
        "torch_autocast_bf16": (autocast_seq, True),
        "torch_tf32": (torch_seq, True),
    }
    result = {"card": bl.card_info(), "steps": args.steps, "repeats": args.repeats, "shapes": {}}
    prev_tf32 = torch.backends.cudnn.allow_tf32
    for name in args.shapes.split(","):
        n, h, w, backward = bl.SHAPES[name]
        g = torch.Generator(device=dev).manual_seed(0)
        x1 = torch.rand(n, 3, h, w, device=dev, generator=g)
        x0 = (x1 + 0.1 * torch.randn(n, 3, h, w, device=dev, generator=g)).clamp(0, 1).requires_grad_(backward)
        times, peaks = {k: [] for k in variants}, {}
        for k, (fn, tf32) in variants.items():  # warm every variant (cuDNN picks its algorithms here)
            torch.backends.cudnn.allow_tf32 = tf32
            bl.time_variant(fn, x0, x1, backward, args.warmup)
            peaks[k] = bl.peak_bytes(fn, x0, x1, backward)
        for _ in range(args.repeats):
            for k, (fn, tf32) in variants.items():
                torch.backends.cudnn.allow_tf32 = tf32
                times[k].append(bl.time_variant(fn, x0, x1, backward, args.steps))
        torch.backends.cudnn.allow_tf32 = prev_tf32
        with torch.no_grad():
            v32, v16 = m32(x0, x1, normalize=True).reshape(-1), m16(x0, x1, normalize=True).reshape(-1)
        med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
        f = bl.flops(n, h, w, backward)
        result["shapes"][name] = {
            "pairs_h_w": [n, h, w], "backward": backward, "ms_median": med, "ms_all": times,
            "bf16_speedup_vs_ours_tf32": med["ours_tf32"] / med["ours_bf16"],
            "bf16_speedup_vs_torch_autocast_bf16": med["torch_autocast_bf16"] / med["ours_bf16"],
            "conv_tflop": f / 1e12, "achieved_tflops": {k: f / (v * 1e9) for k, v in med.items()},
            "peak_bytes_above_inputs": peaks,
            "bf16_vs_tf32_value_max_abs": float((v16 - v32).abs().max()), "value_max": float(v32.abs().max()),
            "kernels_one_step": {k: bl.kernel_breakdown(variants[k][0], x0, x1, backward) for k in ("ours_tf32", "ours_bf16")},
        }
        print(name, json.dumps(med), flush=True)
    out = args.out or tempfile.mkdtemp(prefix="bench_lpips_bf16_")
    os.makedirs(out, exist_ok=True)
    with open(os.path.join(out, "bench_lpips_bf16.json"), "w") as fh:
        json.dump(result, fh, indent=1)
    print(json.dumps({"card": result["card"], **{k: {kk: v[kk] for kk in ("ms_median", "achieved_tflops", "peak_bytes_above_inputs")}
                                                 for k, v in result["shapes"].items()}}))


if __name__ == "__main__":
    main()
