"""Times PF3plat's pose path on one GPU: pf3plat_b200.poses (camera_synchronization, refine_poses, plucker_rays; the
kernels of csrc/gs_poses.cu) against the reference's PyTorch op sequence, restated below (`reference_*`, pinned to
tests/golden/poses.npz by tests/test_poses_cpu.py).

One step is the encoder's stretch: synchronise the pairwise poses, take the 9-vector, build the Plücker rays, refine
the poses and invert them.  The forward + backward step adds a loss on both refined outputs and its backward into
delta and gamma.  The two routes alternate within one run; a round is --steps steps between two device
synchronisations, timed with CUDA events, and the median over --rounds rounds is reported with the spread
((max - min) / median).  Each route's synchronising calls are counted once under torch.cuda.set_sync_debug_mode("warn").
Also reported: the card, its power limit and its maximum SM clock.

Usage:  python scripts/bench_poses.py [--steps 20] [--warmup 5] [--rounds 9] [--out DIR]
Writes DIR/bench_poses.json (default: a temporary directory) and prints it.
"""
from __future__ import annotations

import argparse
import itertools
import json
import math
import os
import statistics
import subprocess
import sys
import tempfile
import warnings

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pf3plat_b200 import poses  # noqa: E402

SHAPES = {  # name: (b, N, Plücker h, w)
    "pf3plat_train_b14_n3_64x64": (14, 3, 64, 64),
    "pf3plat_eval_b1_n3_64x64": (1, 3, 64, 64),
}


# ---- the reference's op sequence (src/flow_util.py, encoder_costvolume.py, src/geometry/projection.py) ----

def reference_se3_inverse(P):
    R_inv = P[..., :3, :3].transpose(-2, -1)
    t_inv = -1 * R_inv @ P[..., :3, 3:4]
    return torch.cat((torch.cat((R_inv, t_inv), dim=-1), P[..., 3:4, :]), dim=-2)


def reference_chaining(Ps, N):
    batch = Ps[(0, 1)].shape[0]
    L = [torch.eye(4, device=Ps[(0, 1)].device)[None].expand(batch, 4, 4)]
    for i in range(N - 1):
        L.append(Ps[(i, i + 1)].float() @ L[-1].float())
    return torch.stack(L, 1)


def reference_sync(Ps, confidence, N):
    if N == 2:
        return reference_chaining(Ps, N)
    first = next(iter(Ps.values()))
    batch, device, dt = first.shape[0], first.device, first.dtype
    zero = torch.zeros(batch, device=device, dtype=dt)
    conf = [[zero for _ in range(N)] for _ in range(N)]
    for i, j in Ps:
        c = confidence[(i, j)]
        conf[i][j] = c
        conf[j][i] = c
        conf[i][i] = conf[i][i] + c / 2
        conf[j][j] = conf[j][j] + c / 2
    conf = torch.stack([torch.stack(row, dim=1) for row in conf], dim=1)
    conf = conf / conf.sum(dim=1, keepdim=True).clamp(min=1e-9)
    zP = torch.zeros(batch, 4, 4, device=device, dtype=dt)
    eye = torch.eye(4, device=device, dtype=dt)[None].expand(batch, 4, 4)
    L = [[zP for _ in range(N)] for _ in range(N)]
    for i in range(N):
        L[i][i] = conf[:, i, i, None, None] * eye
    for i, j in Ps:
        L[i][j] = conf[:, i, j, None, None] * reference_se3_inverse(Ps[(i, j)])
        L[j][i] = conf[:, j, i, None, None] * Ps[(i, j)]
    L = torch.cat([torch.cat(row, dim=2) for row in L], dim=1).double()
    for _ in range(10):
        L = L @ L
    L = L.view(batch, N, 4, N, 4)[:, :, :, 0, :]
    mass = L[:, :, 3:, 3:]
    if mass.min().item() == 0:
        return reference_chaining(Ps, N)
    L = L / mass.clamp(min=1e-9)
    U, _, V = torch.svd(L[:, :, :3, :3])
    V_t = V.transpose(-1, -2)
    S = torch.det(U @ V_t)
    S = torch.cat([torch.ones(*S.shape, 1, 2, device=device), S[..., None, None]], -1)
    R = (U * S.double()) @ V_t
    L = torch.cat([torch.cat([R, L[:, :, :3, 3:]], 3), L[:, :, 3:]], 2)
    return L.float()


def reference_r6d2mat(d6):
    a1, a2 = d6[..., :3], d6[..., 3:]
    b1 = F.normalize(a1, dim=-1)
    b2 = F.normalize(a2 - (b1 * a2).sum(-1, keepdim=True) * b1, dim=-1)
    return torch.stack((b1, b2, torch.cross(b1, b2, dim=-1)), dim=-2)


def reference_refine(pred_pose_enc, delta, gamma):
    pred_pose = pred_pose_enc[:, 1:] + delta[:, 1:] * gamma
    x = torch.cat([pred_pose_enc[:, :1], pred_pose], dim=1)
    Rt = torch.cat([reference_r6d2mat(x[:, :, :6]), x[:, :, 6:][..., None]], dim=-1)
    pad = torch.zeros_like(Rt[..., 2:3, :])
    pad[..., -1] = 1.0
    A = torch.cat((Rt, pad), dim=-2)
    return A, A.inverse()


def reference_plucker(abspose, intrinsics, h, w):
    b, v = abspose.shape[:2]
    dev, dt = abspose.device, abspose.dtype
    ys, xs = torch.meshgrid((torch.arange(h, device=dev) + 0.5).to(dt) / h, (torch.arange(w, device=dev) + 0.5).to(dt) / w,
                            indexing="ij")
    xy = torch.stack([xs, ys], -1).reshape(1, 1, h * w, 2)
    c2w = abspose.inverse()[:, :, None]                  # [b, v, 1, 4, 4]
    d = torch.cat([xy, torch.ones_like(xy[..., :1])], -1)
    d = torch.einsum("bvnij,bvpj->bvpi", intrinsics.inverse()[:, :, None], d.expand(b, v, h * w, 3))
    d = d / d.norm(dim=-1, keepdim=True)
    d = torch.cat([d, torch.zeros_like(d[..., :1])], -1)
    d = torch.einsum("bvnij,bvpj->bvpi", c2w, d)[..., :-1]
    o = c2w[..., :-1, -1].broadcast_to(d.shape)
    out = torch.cat((d, torch.cross(o, d, dim=-1)), dim=-1)
    return out.reshape(b * v, h, w, 6).permute(0, 3, 1, 2)


def matrix_to_rotation_6d(m):
    return m[..., :2, :].clone().reshape(*m.shape[:-2], 6)


# ---- the step ----

def seeded_inputs(b, N, h, w, dev, seed=0):
    g = torch.Generator().manual_seed(seed)

    def rigid(rot, trans):
        k = torch.randn(3, generator=g, dtype=torch.float64)
        k = k / k.norm()
        a = rot * float(torch.rand(1, generator=g)) + 0.05
        Kx = torch.tensor([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]], dtype=torch.float64)
        P = torch.eye(4, dtype=torch.float64)
        P[:3, :3] = torch.eye(3, dtype=torch.float64) + math.sin(a) * Kx + (1 - math.cos(a)) * Kx @ Kx
        P[:3, 3] = torch.randn(3, generator=g, dtype=torch.float64) * trans
        return P

    keys = list(itertools.combinations(range(N), 2))
    Ps = {k: torch.zeros(b, 4, 4, dtype=torch.float64) for k in keys}
    conf = {k: torch.zeros(b) for k in keys}
    for s in range(b):
        W = [torch.eye(4, dtype=torch.float64)] + [rigid(0.3, 0.3) for _ in range(N - 1)]
        for i, j in keys:
            Ps[(i, j)][s] = W[j] @ torch.linalg.inv(W[i]) @ rigid(0.03, 0.03)
            c = 0.55 + 0.4 * float(torch.rand(1, generator=g))
            conf[(i, j)][s] = max(c - 0.5, 0.0) / 0.5 if abs(i - j) > 1 else c
    K = torch.tensor([[1.0, 0.0, 0.5], [0.0, 1.0, 0.5], [0.0, 0.0, 1.0]]).expand(b, N, 3, 3).contiguous()
    return ({k: v.float().to(dev) for k, v in Ps.items()}, {k: v.to(dev) for k, v in conf.items()}, K.to(dev),
            (torch.randn(b, N, 9, generator=g) * 0.05).to(dev), torch.randn(b, N, 4, 4, generator=g).to(dev),
            torch.randn(b, N, 4, 4, generator=g).to(dev))


ROUTES = {
    "reference_ops": (reference_sync, reference_plucker, reference_refine),
    "ours": (poses.camera_synchronization, poses.plucker_rays, poses.refine_poses),
}


def step(route, inp, N, h, w, backward):
    sync, plucker, refine = ROUTES[route]
    Ps, conf, K, delta0, g1, g2 = inp
    abspose = sync(Ps, conf, N)
    rays = plucker(abspose, K, h, w)
    enc = torch.cat([matrix_to_rotation_6d(abspose[:, :, :3, :3]), abspose[:, :, :3, 3]], dim=-1)
    delta = delta0.detach().requires_grad_(backward)
    gamma = torch.ones((), device=enc.device, requires_grad=backward)
    A, Ai = refine(enc, delta, gamma)
    if backward:
        ((A * g1).sum() + (Ai * g2).sum()).backward()
    return rays, A, Ai


def timed_round(route, inp, shape, backward, steps):
    b, N, h, w = shape
    a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(steps):
        step(route, inp, N, h, w, backward)
    e.record()
    torch.cuda.synchronize()
    return a.elapsed_time(e) / steps


def count_syncs(route, inp, shape, backward):
    b, N, h, w = shape
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            step(route, inp, N, h, w, backward)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    return sum("synchroniz" in str(x.message) for x in caught)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=9)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_poses.py needs a CUDA device")
    dev = torch.device("cuda:0")
    info = {"device": torch.cuda.get_device_name(dev)}
    try:
        info["power_limit_and_max_sm_clock"] = subprocess.run(
            ["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
            capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError) as e:
        info["power_limit_and_max_sm_clock"] = f"unavailable: {e}"
    results = {}
    for name, shape in SHAPES.items():
        inp = seeded_inputs(*shape, dev)
        for route in ROUTES:
            for backward in (False, True):
                for _ in range(args.warmup):
                    step(route, inp, shape[1], shape[2], shape[3], backward)
        torch.cuda.synchronize()
        # the two routes' outputs on the same inputs
        ref = [t.detach() for t in step("reference_ops", inp, *shape[1:], False)]
        got = [t.detach() for t in step("ours", inp, *shape[1:], False)]
        res = {"max_abs_diff": {k: float((r - o).abs().max()) for k, r, o in zip(("plucker", "abspose", "abspose_inv"),
                                                                                 ref, got)}}
        for label, backward in (("forward", False), ("forward_backward", True)):
            times = {r: [] for r in ROUTES}
            for _ in range(args.rounds):
                for r in ROUTES:
                    times[r].append(timed_round(r, inp, shape, backward, args.steps))
            for r, ts in times.items():
                med = statistics.median(ts)
                res[f"{label}_{r}_ms"] = round(med, 4)
                res[f"{label}_{r}_spread"] = round((max(ts) - min(ts)) / med, 3)
            res[f"{label}_speedup"] = round(res[f"{label}_reference_ops_ms"] / res[f"{label}_ours_ms"], 2)
            for r in ROUTES:
                res[f"{label}_{r}_sync_calls"] = count_syncs(r, inp, shape, backward)
        results[name] = res
    out = {"bench": "poses", **info, "steps": args.steps, "rounds": args.rounds, "shapes": results}
    out_dir = args.out or tempfile.mkdtemp(prefix="bench_poses_")
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "bench_poses.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
