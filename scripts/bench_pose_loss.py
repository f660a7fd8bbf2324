"""Times PF3plat's correspondence (pose) loss, forward + backward, on one GPU: pf3plat_b200.losses.pose_loss (the kernels
of csrc/gs_pose_loss.cu) against the reference's PyTorch op sequence (Losspose.forward, loss_pose.py:29-129, restated
below op for op: a dense projection of every pixel for the absolute and the relative pose of every pair, torch.inverse,
then a Python loop over scenes x pairs with gathers, Huber, norms and an L1-normalised weighting; the relative-pose terms
are computed and discarded as there).  The two variants alternate within one run.  Each round of a variant runs as many
steps as fill --round-s seconds (calibrated once after the warm-up), so that a round is long enough not to measure the
host's scheduler; the median over the rounds is reported with the rounds' spread ((max - min) / median), and the
speedup of each round (both variants' step time is set by the host, whose load drifts between rounds, so the ratio
within a round is the steadier comparison).  Garbage collection is off while timing.  Also reported,
from one profiled step of a separate pass: CUDA kernels and copies per step, their summed device time ("device busy":
what the step would take if the host never made the GPU wait), and the peak allocation of one step.

Usage:  python scripts/bench_pose_loss.py [--round-s 1.0] [--warmup 10] [--rounds 7] [--out DIR]
Writes DIR/bench_pose_loss.json (default: a temporary directory) and prints it.
"""
from __future__ import annotations

import argparse
import gc
import json
import os
import statistics
import subprocess
import sys
import tempfile

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pf3plat_b200 import losses  # noqa: E402
from tests.pose_loss_cases import pairs_of, seeded_case  # noqa: E402

SHAPES = {  # name: (b, v, h, w, min matches, max matches) per (scene, pair)
    "pf3plat_train_b14_v3_256": (14, 3, 256, 256, 500, 2047),
    "b4_v4_256": (4, 4, 256, 256, 500, 2047),
}


def _project(xy, d, Ki, Kj, T):
    """batch_project_to_other_img as the reference writes it: [b, hw, 2] pixels, [b, hw] depth."""
    ones = torch.ones_like(xy[..., :1])
    X = torch.cat([xy, ones], -1) @ torch.inverse(Ki).transpose(-1, -2)
    X = X * d[..., None]
    Q = torch.cat([X, torch.ones_like(X[..., :1])], -1) @ T.transpose(-1, -2)
    P = Q[..., :-1] / (Q[..., -1:] + 1e-6)
    u = P @ Kj.transpose(-1, -2)
    return u[..., :-1] / (u[..., -1:] + 1e-6)


def torch_sequence(batch, c2w, depth, corr, xyz_h, weight_2d=0.005, weight_3d=0.025):
    b, v, _, h, w = batch["context"]["image"].shape
    pairs = pairs_of(v)
    relpose, abspose = c2w
    corre, trans_conf = corr[0], corr[2]
    K = batch["target"]["intrinsics"]
    ys, xs = torch.meshgrid(torch.arange(h, device=abspose.device), torch.arange(w, device=abspose.device), indexing="ij")
    xy = torch.stack([(xs + 0.5) / w, (ys + 0.5) / h], -1).reshape(1, h * w, 2).expand(b, -1, -1)
    d = depth[0].reshape(b, v, h * w)
    rel_T = lambda A, C: C @ A.inverse()
    pts, pts_rel = {}, {}
    for idx, (a, c) in enumerate(pairs):
        T = abspose[:, c] if a == 0 else rel_T(abspose[:, a], abspose[:, c])
        pts[(a, c)] = _project(xy, d[:, a], K[:, a], K[:, c], T)
        pts_rel[(a, c)] = _project(xy, d[:, a], K[:, a], K[:, c], relpose[:, idx])
    l3, l2 = [], []
    for i in range(b):
        for idx, (a, c) in enumerate(pairs):
            id_a, id_c, wt = corre[(a, c)][i]
            wn = F.normalize(wt, p=1, dim=-1)
            xa = xyz_h[i, a].flatten(-2, -1).T[id_a]
            xc = xyz_h[i, c].flatten(-2, -1).T[id_c]
            q = xy[i][id_c]
            e2 = (pts[(a, c)][i][id_a] - q).norm(dim=-1)
            e2r = (pts_rel[(a, c)][i][id_a] - q).norm(dim=-1)
            l2.append((F.huber_loss(e2, torch.zeros_like(e2), reduction="none", delta=0.01) / 0.01).sum())
            _ = (F.huber_loss(e2r, torch.zeros_like(e2r), reduction="none", delta=0.01) / 0.01).sum()
            T = abspose[i, c] if a == 0 else rel_T(abspose[i, a], abspose[i, c])
            e3 = (xa @ T[:3, :3].T + T[:3, 3] - xc).norm(dim=-1)
            e3r = (xa @ relpose[i, idx, :3, :3].T + relpose[i, idx, :3, 3] - xc).norm(dim=-1)
            l3.append((wn * e3).sum() * trans_conf[(a, c)][i])
            _ = (wn * e3r).sum() * trans_conf[(a, c)][i]
    return torch.stack(l3).mean() * weight_3d + torch.stack(l2).mean() * weight_2d


def ours(batch, c2w, depth, corr, xyz_h):
    return losses.pose_loss(batch, c2w, depth, corr, xyz_h)


def card_info():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit_and_max_sm_clock"] = out
    except (OSError, subprocess.SubprocessError) as e:
        info["power_limit_and_max_sm_clock"] = f"unavailable: {e}"
    return info


def make_inputs(b, v, h, w, nmin, nmax, dev):
    case = seeded_case(b, v, h, w, nmin, nmax, seed=0).to(dev)
    leaves = [case.abspose.clone().requires_grad_(True), case.depth.clone().requires_grad_(True),
              case.xyz.clone().requires_grad_(True)]
    corre, conf = case.matches()
    img = torch.zeros(b, v, 3, h, w, device=dev)
    batch = {"context": {"image": img}, "target": {"image": img, "intrinsics": case.K}}
    relpose = torch.eye(4, device=dev).repeat(b, len(pairs_of(v)), 1, 1)
    return leaves, (batch, (relpose, leaves[0]), (leaves[1],), (corre, None, conf), leaves[2]), int(case.counts.sum())


def step(fn, leaves, args):
    for t in leaves:
        t.grad = None
    fn(*args).backward()


def time_variant(fn, leaves, args, steps):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        step(fn, leaves, args)
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / steps


def profiled(fn, leaves, args):
    """-> (CUDA kernels and copies in one step, their summed device time in ms)."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step(fn, leaves, args)
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type.name == "CUDA"]
    return len(ev), sum(e.time_range.elapsed_us() for e in ev) / 1e3


def peak_bytes(fn, leaves, args):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    step(fn, leaves, args)
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--round-s", type=float, default=1.0, help="seconds per timed round of each variant")
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pose_loss.py needs a CUDA device")
    dev = torch.device("cuda:0")
    result = {"card": card_info(), "round_s": args.round_s, "rounds": args.rounds, "shapes": {}}
    variants = {"ours": ours, "torch_sequence": torch_sequence}
    for name, shape in SHAPES.items():
        leaves, inputs, M = make_inputs(*shape, dev)
        # agreement of what is timed
        step(torch_sequence, leaves, inputs)
        ref = [t.grad.clone() for t in leaves]
        l_ref = float(torch_sequence(*inputs).detach())
        step(ours, leaves, inputs)
        l_ours = float(ours(*inputs).detach())
        agree = {"loss_abs": abs(l_ours - l_ref), "loss": l_ref}
        for k, t, r in zip(("abspose", "depth", "xyz"), leaves, ref):
            agree[f"grad_{k}_max_abs"] = float((t.grad - r).abs().max())
            agree[f"grad_{k}_max_ref"] = float(r.abs().max())
        steps = {}
        for k, fn in variants.items():   # warm up, then size each variant's round to about round_s seconds
            ms = time_variant(fn, leaves, inputs, args.warmup)
            steps[k] = max(5, int(round(args.round_s * 1e3 / ms)))
        times = {k: [] for k in variants}
        gc.collect()
        gc.disable()   # a collection inside a round would be charged to whichever variant it lands in
        try:
            for _ in range(args.rounds):
                for k, fn in variants.items():
                    times[k].append(time_variant(fn, leaves, inputs, steps[k]))
        finally:
            gc.enable()
        med = {k: statistics.median(v) for k, v in times.items()}
        spread = {k: (max(v) - min(v)) / med[k] for k, v in times.items()}
        # the host's load drifts between rounds and both variants are host-bound: compare within a round
        ratios = sorted(t / o for t, o in zip(times["torch_sequence"], times["ours"]))
        prof = {k: profiled(fn, leaves, inputs) for k, fn in variants.items()}
        result["shapes"][name] = {
            "b_v_h_w_matches": [*shape[:4], M], "steps_per_round": steps, "ms_per_fwd_bwd_median": med,
            "round_spread_rel": spread, "ms_all": times,
            "speedup_vs_torch_sequence": med["torch_sequence"] / med["ours"],
            "speedup_per_round_min_median_max": [ratios[0], statistics.median(ratios), ratios[-1]],
            "cuda_kernels_and_copies_per_step": {k: p[0] for k, p in prof.items()},
            "device_busy_ms_per_step": {k: p[1] for k, p in prof.items()},
            "peak_alloc_bytes_per_step": {k: peak_bytes(fn, leaves, inputs) for k, fn in variants.items()},
            "agreement_vs_torch_sequence": agree,
        }
        print(name, json.dumps({"median": med, "spread": spread, "speedup_per_round": ratios,
                                "device_busy_ms": result["shapes"][name]["device_busy_ms_per_step"]}), flush=True)
    out = args.out or tempfile.mkdtemp(prefix="bench_pose_loss_")
    os.makedirs(out, exist_ok=True)
    with open(os.path.join(out, "bench_pose_loss.json"), "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
