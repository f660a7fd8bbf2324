"""Times LPIPS-VGG on one GPU: the kernels of pf3plat_b200.lpips against the PyTorch op sequence the `lpips` package
runs (oracle/lpips_oracle.py in float32: cuDNN convolutions, NCHW, autograd backward), with cudnn.allow_tf32 on
(PyTorch's default) and off.  The three variants alternate within one run.  Seeded weights: the time does not depend
on their values.

Shapes: PF3plat's training step (LossLpips on color[:, 1:-1] of 14 scenes x 3 target views: forward of 14 pairs,
gradient of the prediction only), evaluation batches (forward only, no grad), and a large training-like batch.  For
ours, one extra profiled step per shape gives the time per kernel (the stage breakdown).

Usage:  python scripts/bench_lpips.py [--steps 20] [--warmup 5] [--repeats 5] [--out DIR]
Writes DIR/bench_lpips.json (default: a temporary directory) and prints it.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import lpips_oracle as lo  # noqa: E402
from pf3plat_b200 import lpips as pl  # noqa: E402

SHAPES = {  # name: (pairs, h, w, backward)
    "pf3plat_train_14x3x256": (14, 256, 256, True),
    "eval_3x3x256": (3, 256, 256, False),
    "eval_60x3x256": (60, 256, 256, False),
    "large_32x3x512": (32, 512, 512, True),
}
GMAC_PER_256SQ_IMAGE = 20.0   # VGG16 features up to relu5_3 (the convolutions; pools and head are not counted)


def flops(n, h, w, backward):
    """Forward of 2n images; the backward's data gradient of n images costs one more forward's convolutions."""
    images = 2 * n + (n if backward else 0)
    return 2 * GMAC_PER_256SQ_IMAGE * 1e9 * images * (h * w) / 65536.0


def card_info():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader",
                              "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit_max_sm_clock_sm_clock"] = out
    except (OSError, subprocess.SubprocessError) as e:
        info["power_limit_max_sm_clock_sm_clock"] = f"unavailable: {e}"
    return info


def step(fn, x0, x1, backward):
    if backward:
        x0.grad = None
        fn(x0, x1).sum().backward()
    else:
        with torch.no_grad():
            fn(x0, x1)


def time_variant(fn, x0, x1, backward, steps):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        step(fn, x0, x1, backward)
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / steps


def peak_bytes(fn, x0, x1, backward):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    step(fn, x0, x1, backward)
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def kernel_breakdown(fn, x0, x1, backward):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step(fn, x0, x1, backward)
        torch.cuda.synchronize()
    rows = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if t > 0:
            rows[e.key] = {"ms": t / 1e3, "calls": e.count}
    return dict(sorted(rows.items(), key=lambda kv: -kv[1]["ms"]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lpips.py needs a CUDA device")
    dev = torch.device("cuda:0")
    sd = lo.random_state_dict(0)
    model = pl.LPIPS(weights=sd).to(dev)
    sd_dev = {k: v.to(dev) for k, v in sd.items()}
    ours = lambda a, b: model(a, b, normalize=True)
    torch_seq = lambda a, b: lo.lpips(a, b, sd_dev, normalize=True)
    variants = {"ours": (ours, None), "torch_tf32": (torch_seq, True), "torch_fp32": (torch_seq, False)}
    result = {"card": card_info(), "steps": args.steps, "repeats": args.repeats, "shapes": {}}
    for name in args.shapes.split(","):
        n, h, w, backward = SHAPES[name]
        g = torch.Generator(device=dev).manual_seed(0)
        x1 = torch.rand(n, 3, h, w, device=dev, generator=g)
        x0 = (x1 + 0.1 * torch.randn(n, 3, h, w, device=dev, generator=g)).clamp(0, 1).requires_grad_(backward)
        # agreement of what is timed: ours against the fp32 PyTorch sequence
        torch.backends.cudnn.allow_tf32 = False
        v_ref = torch_seq(x0, x1).detach()
        v_ours = ours(x0, x1).detach().reshape(-1)
        agree = {"value_max_abs": float((v_ours - v_ref).abs().max()), "value_ref_max": float(v_ref.abs().max())}
        times, peaks = {k: [] for k in variants}, {}
        for k, (fn, tf32) in variants.items():   # warm every variant (cuDNN picks its algorithms here)
            if tf32 is not None:
                torch.backends.cudnn.allow_tf32 = tf32
            time_variant(fn, x0, x1, backward, args.warmup)
            peaks[k] = peak_bytes(fn, x0, x1, backward)
        for _ in range(args.repeats):
            for k, (fn, tf32) in variants.items():
                if tf32 is not None:
                    torch.backends.cudnn.allow_tf32 = tf32
                times[k].append(time_variant(fn, x0, x1, backward, args.steps))
        torch.backends.cudnn.allow_tf32 = True
        med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
        f = flops(n, h, w, backward)
        result["shapes"][name] = {
            "pairs_h_w": [n, h, w], "backward": backward, "ms_median": med, "ms_all": times,
            "speedup_vs_torch_tf32": med["torch_tf32"] / med["ours"], "speedup_vs_torch_fp32": med["torch_fp32"] / med["ours"],
            "conv_tflop": f / 1e12, "achieved_tflops": {k: f / (v * 1e9) for k, v in med.items()},
            "peak_bytes_above_inputs": peaks, "agreement_vs_torch_fp32": agree,
            "ours_kernels_one_step": kernel_breakdown(ours, x0, x1, backward),
        }
        print(name, json.dumps(med), flush=True)
    out = args.out or tempfile.mkdtemp(prefix="bench_lpips_")
    os.makedirs(out, exist_ok=True)
    with open(os.path.join(out, "bench_lpips.json"), "w") as fh:
        json.dump(result, fh, indent=1)
    print(json.dumps({k: {kk: v[kk] for kk in ("ms_median", "achieved_tflops", "peak_bytes_above_inputs")}
                      for k, v in result["shapes"].items()}))


if __name__ == "__main__":
    main()
