"""Times PF3plat's Gaussian head on one GPU: pf3plat_b200.gaussian_head (the kernels of csrc/gs_gaussian_head.cu)
against the route an INTEGRATION.md section 4 user runs today: the reference's glue statements
(depth_predictor_multiview.py:398-415, encoder_costvolume.py:509-540 and :556-573) around the repository's fused
GaussianAdapter (tests/gaussian_head_route.py).  Both routes are followed by decoder_forward's input handling (the
harmonics made contiguous in the rasterizer's layout, the 6-entry covariance gather), so that a harmonics copy is counted
where one happens.

The forward + backward step adds a loss on all four outputs and its backward into the two convolution outputs, the
depths and c2w.  Shapes: PF3plat's training step, b = 14, 256 x 256, d_sh = 25, two depth-predictor views, V = 2 or 3
context views.  The routes alternate within one run; a round is --steps steps between two device synchronisations,
timed with CUDA events, and the median over --rounds rounds is reported with the spread ((max - min) / median).  Also
per route: the peak allocation above the inputs, the kernel launches of one step (torch.profiler), and the synchronising
calls of one step, counted under torch.cuda.set_sync_debug_mode("warn").  Also reported: the card, its power limit and
its maximum SM clock, and the extra bytes the existing route's harmonics copy moves.

Usage:  python scripts/bench_gaussian_head.py [--steps 10] [--warmup 3] [--rounds 9] [--out DIR]
Writes DIR/bench_gaussian_head.json (default: a temporary directory) and prints it.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import warnings

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pf3plat_b200.adapter import GaussianAdapterCfg  # noqa: E402
from pf3plat_b200.gaussian_head import gaussian_head  # noqa: E402
from tests.gaussian_head_route import decoder_inputs, existing_route  # noqa: E402

SHAPES = {  # name: (b, V, h, w, sh_degree)
    "pf3plat_train_b14_v2_256_dsh25": (14, 2, 256, 256, 4),
    "pf3plat_train_b14_v3_256_dsh25": (14, 3, 256, 256, 4),
}
CFG = GaussianAdapterCfg(gaussian_scale_min=0.5, gaussian_scale_max=15.0, sh_degree=4)


def ours(raw, logits, depths, c2w, K, h, w):
    g = gaussian_head(raw, logits, depths, c2w, K, CFG, (h, w))
    return decoder_inputs(g.means, g.covariances, g.harmonics, g.opacities)


def existing(raw, logits, depths, c2w, K, h, w):
    return decoder_inputs(*existing_route(raw, logits, depths, c2w, K, CFG, h, w))


ROUTES = {"existing_route": existing, "ours": ours}


def seeded_inputs(b, V, h, w, deg, dev, seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)
    d_sh = (deg + 1) ** 2
    raw = torch.randn((2 * b, 9 + 3 * d_sh, h, w), generator=g, device=dev)
    logits = torch.randn((2 * b, 2, h, w), generator=g, device=dev)
    depths = 1.0 + 9.0 * torch.rand((b * V, 1, h, w), generator=g, device=dev)
    q = torch.nn.functional.normalize(torch.randn((b * V, 4), generator=g, device=dev), dim=-1)
    r, x, y, z = q.unbind(-1)
    rot = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                       2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                       2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1).reshape(b, V, 3, 3)
    c2w = torch.eye(4, device=dev).repeat(b, V, 1, 1)
    c2w[..., :3, :3] = rot
    c2w[..., :3, 3] = torch.randn((b, V, 3), generator=g, device=dev)
    K = torch.tensor([[1.0, 0.0, 0.5], [0.0, 1.0, 0.5], [0.0, 0.0, 1.0]], device=dev).expand(b, V, 3, 3).contiguous()
    G = 2 * h * w
    cot = [torch.randn(s, generator=g, device=dev) for s in ((b, G, 3), (b, G, 6), (b, G, d_sh, 3), (b, G))]
    return raw, logits, depths, c2w, K, h, w, cot


def step(route, inp, backward):
    raw0, logits0, depths0, c2w0, K, h, w, cot = inp
    leaves = [t.detach().requires_grad_(backward) for t in (raw0, logits0, depths0, c2w0)]
    outs = ROUTES[route](*leaves, K, h, w)
    if backward:
        sum((o * c).sum() for o, c in zip(outs, cot)).backward()
    return outs


def timed_round(route, inp, backward, steps):
    a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(steps):
        step(route, inp, backward)
    e.record()
    torch.cuda.synchronize()
    return a.elapsed_time(e) / steps


def count_syncs(route, inp, backward):
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            step(route, inp, backward)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    return sum("synchroniz" in str(x.message) for x in caught)


def count_launches(route, inp, backward):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step(route, inp, backward)
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type.name == "CUDA" and "memcpy" not in e.name.lower()
               and "memset" not in e.name.lower())


def peak_mib(route, inp, backward):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = step(route, inp, backward)
    torch.cuda.synchronize()
    del out
    return round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=9)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_gaussian_head.py needs a CUDA device")
    dev = torch.device("cuda:0")
    info = {"device": torch.cuda.get_device_name(dev)}
    try:
        info["power_limit_and_max_sm_clock"] = subprocess.run(
            ["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
            capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError) as e:
        info["power_limit_and_max_sm_clock"] = f"unavailable: {e}"
    results = {}
    for name, (b, V, h, w, deg) in SHAPES.items():
        inp = seeded_inputs(b, V, h, w, deg, dev)
        for route in ROUTES:
            for backward in (False, True):
                for _ in range(args.warmup):
                    step(route, inp, backward)
        torch.cuda.synchronize()
        ref = [t.detach() for t in step("existing_route", inp, False)]
        got = [t.detach() for t in step("ours", inp, False)]
        res = {"max_abs_diff": {k: float((r - o).abs().max()) for k, r, o in
                                zip(("means", "covariances6", "harmonics", "opacities"), ref, got)}}
        del ref, got
        with torch.no_grad():
            g = existing_route(*inp[:5], CFG, h, w)
            res["existing_route_harmonics_view_contiguous"] = bool(g[2].transpose(-1, -2).is_contiguous())
            res["harmonics_mib"] = round(g[2].numel() * 4 / 2 ** 20, 1)
            del g
        for label, backward in (("forward", False), ("forward_backward", True)):
            times = {r: [] for r in ROUTES}
            for _ in range(args.rounds):
                for r in ROUTES:
                    times[r].append(timed_round(r, inp, backward, args.steps))
            for r, ts in times.items():
                med = statistics.median(ts)
                res[f"{label}_{r}_ms"] = round(med, 4)
                res[f"{label}_{r}_spread"] = round((max(ts) - min(ts)) / med, 3)
            res[f"{label}_speedup"] = round(res[f"{label}_existing_route_ms"] / res[f"{label}_ours_ms"], 2)
            for r in ROUTES:
                res[f"{label}_{r}_sync_calls"] = count_syncs(r, inp, backward)
                res[f"{label}_{r}_launches"] = count_launches(r, inp, backward)
                res[f"{label}_{r}_peak_mib_above_inputs"] = peak_mib(r, inp, backward)
        results[name] = res
        del inp
        torch.cuda.empty_cache()
    out = {"bench": "gaussian_head", **info, "torch": torch.__version__, "steps": args.steps, "rounds": args.rounds,
           "shapes": results}
    out_dir = args.out or tempfile.mkdtemp(prefix="bench_gaussian_head_")
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "bench_gaussian_head.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
