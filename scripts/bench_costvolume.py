"""Times PF3plat's plane-sweep cost volume on one GPU: pf3plat_b200.costvolume.plane_sweep_cost_volume (the kernels of
csrc/gs_costvolume.cu) against the reference's PyTorch op sequence (depth_predictor_multiview.py:309-343 with
prepare_feat_proj_data_lists and warp_with_pose_depth_candidates, restated in tests/test_gpu_costvolume.py).

For each shape, forward alone and forward + backward are timed for three variants that alternate within one run:
the reference's ops, ours, and ours under torch.use_deterministic_algorithms(True).  A round is --steps calls between
two device synchronisations, timed with CUDA events; the median over --rounds rounds is reported with the rounds' spread
((max - min) / median).  Also reported: the peak allocation of one forward + backward above the inputs, whether
PyTorch's route raises under the deterministic flag, and the card, its power limit and its maximum SM clock.

Usage:  python scripts/bench_costvolume.py [--steps 5] [--warmup 3] [--rounds 7] [--out DIR]
Writes DIR/bench_costvolume.json (default: a temporary directory) and prints it.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pf3plat_b200.costvolume import plane_sweep_cost_volume  # noqa: E402
from tests.test_gpu_costvolume import reference_ops, seeded_case  # noqa: E402

SHAPES = {  # name: (b, v, C, h, w, D)
    "pf3plat_train_b14_v2_c256_64x64_d32": (14, 2, 256, 64, 64, 32),
    "b6_v3_c256_64x64_d32": (6, 3, 256, 64, 64, 32),
}


def step(fn, args, cot, backward):
    f = args[0].detach().requires_grad_(backward)
    out = fn(f, *args[1:])
    if backward:
        torch.autograd.grad(out, f, cot)


# name: (function, run under torch.use_deterministic_algorithms(True))
VARIANTS = {"reference_ops": (reference_ops, False), "ours": (plane_sweep_cost_volume, False),
            "ours_deterministic": (plane_sweep_cost_volume, True)}


def timed_round(fn, det, args, cot, backward, steps):
    torch.use_deterministic_algorithms(det)
    try:
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        for _ in range(steps):
            step(fn, args, cot, backward)
        b.record()
        torch.cuda.synchronize()
    finally:
        torch.use_deterministic_algorithms(False)
    return a.elapsed_time(b) / steps


def peak_above_inputs(fn, det, args, cot):
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    torch.use_deterministic_algorithms(det)
    try:
        step(fn, args, cot, True)
    finally:
        torch.use_deterministic_algorithms(False)
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def pytorch_route_raises_when_deterministic(args, cot):
    torch.use_deterministic_algorithms(True)
    try:
        step(reference_ops, args, cot, True)
        torch.cuda.synchronize()
        return "no error"
    except RuntimeError as e:
        return f"raises: {str(e).splitlines()[0][:160]}"
    finally:
        torch.use_deterministic_algorithms(False)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_costvolume needs a CUDA device")
    info = {"device": torch.cuda.get_device_name(0)}
    try:
        info["power_limit_and_max_sm_clock"] = subprocess.run(
            ["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
            capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError) as e:
        info["power_limit_and_max_sm_clock"] = f"unavailable: {e}"
    result = {"info": info, "shapes": {}}
    for name, (b, v, C, h, w, D) in SHAPES.items():
        f, K, E, near, far, D, cot = seeded_case(b, v, C, h, w, D, seed=1)
        args = (f, K, E, near, far, D)
        res = {"pytorch_route_deterministic": pytorch_route_raises_when_deterministic(args, cot)}
        for backward in (False, True):
            times = {k: [] for k in VARIANTS}
            for k, (fn, det) in VARIANTS.items():
                timed_round(fn, det, args, cot, backward, a.warmup)
            for _ in range(a.rounds):
                for k, (fn, det) in VARIANTS.items():
                    times[k].append(timed_round(fn, det, args, cot, backward, a.steps))
            tag = "fwd_bwd" if backward else "fwd"
            for k, t in times.items():
                med = statistics.median(t)
                res[f"{tag}_ms_{k}"] = round(med, 3)
                res[f"{tag}_spread_{k}"] = round((max(t) - min(t)) / med, 3)
            res[f"{tag}_speedup"] = round(res[f"{tag}_ms_reference_ops"] / res[f"{tag}_ms_ours"], 2)
        for k, (fn, det) in VARIANTS.items():
            res[f"peak_mb_above_inputs_{k}"] = round(peak_above_inputs(fn, det, args, cot), 1)
        result["shapes"][name] = res
        print(name, json.dumps(res), flush=True)
    out_dir = a.out or tempfile.mkdtemp()
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "bench_costvolume.json"), "w") as fh:
        json.dump(result, fh, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
