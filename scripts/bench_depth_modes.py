"""What the fused depth channel saves in the depth modes other than "depth": for "disparity", "relative_disparity" and
"log", decoder_forward(depth_mode=m) -- one gs_forward call compositing f(z) next to the colour -- against the reference's
two-pass route (a colour render, then render_depth's second render of the Gaussians repeated per view with f(z) as their
colour), the two routes alternating in one process, medians over rounds.  Prints one JSON line with the card's name and
power limit, read in the same run.
  * PF3plat's training shape: b = 14 scenes x v = 3 views, 131072 Gaussians per scene (2 x 256 x 256), 256x256, the
    Gaussians and the extrinsics requiring grad, loss = MSE on the colour + a depth term: forward, forward + backward,
    and per step the peak torch allocation and the library pool's reservation;
  * the validation-video shape: b = 1 scene x v = 60 views, forward only (no grad).
Usage: python scripts/bench_depth_modes.py [--steps K] [--warmup W] [--rounds R] [--modes m1,m2]"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pf3plat_b200.rasterizer import last_stats  # noqa: E402
from pf3plat_b200.render import decoder_forward, render_depth, render_views  # noqa: E402
from pf3plat_b200.synthetic import make_pixel_aligned_scene, make_target  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [s.strip() for s in out.split(",")]
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def two_pass(means, cov, harm, opa, ext, intr, near, far, hw, bg, mode):
    """The reference's route: colour render, then render_depth's second render."""
    b, v = ext.shape[:2]
    flat = lambda t: t.reshape(b * v, *t.shape[2:])
    color = render_views(flat(ext), flat(intr), flat(near), flat(far), hw, bg.reshape(1, 3).expand(b * v, 3), means,
                         cov, harm, opa)
    return color.reshape(b, v, *color.shape[1:]), render_depth(means, cov, opa, ext, intr, near, far, hw, mode)


def fused(means, cov, harm, opa, ext, intr, near, far, hw, bg, mode):
    return decoder_forward(means, cov, harm, opa, ext, intr, near, far, hw, bg, depth_mode=mode)


ROUTES = {"fused": fused, "two_pass": two_pass}


def scenes(b, v, seed, dev):
    scs = [make_pixel_aligned_scene(256, 256, v, seed=seed + k) for k in range(b)]
    st = lambda n: torch.stack([getattr(s, n) for s in scs]).to(dev)
    return st("means"), st("covariances"), st("harmonics"), st("opacities"), st("extrinsics"), st("intrinsics")


def median(xs):
    return sorted(xs)[len(xs) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--modes", default="disparity,relative_disparity,log")
    args = ap.parse_args()
    modes = args.modes.split(",")
    dev = torch.device("cuda:0")
    name, limit = card()
    res = {"card": name, "power_limit": limit, "steps": args.steps, "rounds": args.rounds}
    hw = (256, 256)
    bg = torch.zeros(3, device=dev)

    # ---- PF3plat's training shape ----
    b, v = 14, 3
    means, cov, harm, opa, ext0, intr = scenes(b, v, 30, dev)
    near, far = torch.full((b, v), 1.0, device=dev), torch.full((b, v), 100.0, device=dev)
    tgt = make_target(b * v, *hw).to(dev).reshape(b, v, 3, *hw)
    L = [t.clone().requires_grad_(True) for t in (means, cov, harm, opa)]
    ext = ext0.clone().requires_grad_(True)
    train = {m: {r: {"fwd": [], "fwd_bwd": [], "peak_alloc_mb": [], "pool_reserved_mb": []} for r in ROUTES}
             for m in modes}
    for _ in range(args.rounds):
        for m in modes:
            for r, route in ROUTES.items():
                def fwd():
                    return route(*L, ext, intr, near, far, hw, bg, m)

                def step():
                    col, dep = fwd()
                    (((col - tgt) ** 2).mean() + 1e-3 * dep.mean()).backward()
                t = train[m][r]
                t["fwd"].append(timed(fwd, args.steps, args.warmup))
                t["fwd_bwd"].append(timed(step, args.steps, args.warmup))
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats(dev)
                base = torch.cuda.memory_allocated(dev)
                step()
                torch.cuda.synchronize()
                t["peak_alloc_mb"].append((torch.cuda.max_memory_allocated(dev) - base) / 2 ** 20)
                t["pool_reserved_mb"].append(last_stats(dev)["pool_reserved_bytes"] / 2 ** 20)
    res["training_shape"] = {"b": b, "v": v, "gaussians_per_scene": int(means.shape[1]), "hw": list(hw),
                             "ms_and_mb_median": {m: {r: {k: median(x) for k, x in train[m][r].items()} for r in ROUTES}
                                                  for m in modes}}
    del L, ext, means, cov, harm, opa
    torch.cuda.empty_cache()

    # ---- validation-video shape: forward only ----
    b, v = 1, 60
    means, cov, harm, opa, ext, intr = scenes(b, v, 60, dev)
    near, far = torch.full((b, v), 1.0, device=dev), torch.full((b, v), 100.0, device=dev)
    video = {m: {r: [] for r in ROUTES} for m in modes}
    with torch.no_grad():
        for _ in range(args.rounds):
            for m in modes:
                for r, route in ROUTES.items():
                    video[m][r].append(timed(lambda: route(means, cov, harm, opa, ext, intr, near, far, hw, bg, m),
                                             args.steps, args.warmup))
    res["video_shape"] = {"b": b, "v": v, "gaussians": int(means.shape[1]), "hw": list(hw),
                          "fwd_ms_median": {m: {r: median(video[m][r]) for r in ROUTES} for m in modes}}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
