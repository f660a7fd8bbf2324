"""PF3plat-shaped decoder timing (BASELINE.json configs[4] geometry without the encoder): b scenes x v views,
131072 Gaussians per scene (2 x 256 x 256 pixel-aligned Gaussians), 256x256, colour + depth.
  (1) the reference's call pattern: per-view GaussianRasterizer calls on v-fold repeated Gaussians + a second
      pass for depth (tests/ref_callsite.py restates cuda_splatting.py / decoder_splatting_cuda.py);
  (2) pf3plat_b200.render.decoder_forward: one batched call, depth fused.
Prints one JSON line; both run OUR kernels -- this measures what the batched entry (SURVEY.md section 8(f).1) buys.

GS_POSE=1 runs the leg PF3plat trains through instead (b defaults to 14): target extrinsics that require grad
(predicted poses), loss = MSE on color[:, 1:-1] + a depth term.  It compares the two-pass route decoder_forward took for
that case before the fused depth channel carried the camera gradient (render_views + render_depth) with
decoder_forward, alternating, each on a stream (hence a rasterizer context and memory pool) of its own: forward,
forward + backward, torch's peak allocation and the context pool's reservation, with the card's name and power limit."""
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pf3plat_b200.render import decoder_forward, render_depth, render_views  # noqa: E402
from pf3plat_b200.synthetic import make_scene, make_target  # noqa: E402
from tests.ref_callsite import render_depth_like_reference, render_like_reference  # noqa: E402

POSE = os.environ.get("GS_POSE") == "1"
b, v, P, hw = int(os.environ.get("GS_B", 14 if POSE else 2)), int(os.environ.get("GS_V", 3)), 131072, (256, 256)
steps = int(os.environ.get("GS_STEPS", 10))
dev = torch.device("cuda:0")
scs = [make_scene(P, v, *hw, seed=30 + k).to(dev) for k in range(b)]
st = lambda n: torch.stack([getattr(s, n) for s in scs])
means, cov, sh, opac, ext, intr = st("means"), st("covariances"), st("harmonics"), st("opacities"), st("extrinsics"), st("intrinsics")
near = torch.full((b, v), 1.0, device=dev)
far = torch.full((b, v), 100.0, device=dev)
bg = torch.zeros(3, device=dev)
target = make_target(b * v, *hw).to(dev).reshape(b, v, 3, *hw)
flat = lambda t: t.reshape(b * v, *t.shape[2:])
rep = lambda t: t.repeat_interleave(v, dim=0)


def ref_fwd(grad):
    L = [t.clone().requires_grad_(grad) for t in (means, cov, sh, opac)]
    c = render_like_reference(flat(ext), flat(intr), flat(near), flat(far), hw, bg[None].expand(b * v, 3), *[rep(t) for t in L])
    d = render_depth_like_reference(flat(ext), flat(intr), flat(near), flat(far), hw, rep(L[0]), rep(L[1]), rep(L[3]))
    if grad:
        (((c.reshape(b, v, 3, *hw) - target) ** 2).mean() + 1e-3 * d.mean()).backward()
    return c


def ours_fwd(grad):
    L = [t.clone().requires_grad_(grad) for t in (means, cov, sh, opac)]
    c, d = decoder_forward(*L, ext, intr, near, far, hw, bg, depth_mode="depth")
    if grad:
        (((c - target) ** 2).mean() + 1e-3 * d.mean()).backward()
    return c


def timeit(fn, grad):
    from pf3plat_b200.rasterizer import last_stats
    for _ in range(3):
        fn(grad)
    torch.cuda.synchronize()
    per = []
    t0 = time.perf_counter()
    for _ in range(steps):
        t1 = time.perf_counter()
        fn(grad)
        if os.environ.get("GS_VERBOSE"):
            torch.cuda.synchronize()
            per.append((round(1e3 * (time.perf_counter() - t1), 3), last_stats(dev)["speculative"], last_stats(dev)["overflow_redos"]))
    torch.cuda.synchronize()
    if per:
        sys.stderr.write(f"{fn.__name__} grad={grad}: {per}\n")
    return 1e3 * (time.perf_counter() - t0) / steps


def two_pass_route(grad):
    e = ext.clone().requires_grad_(True)
    L = [t.clone().requires_grad_(grad) for t in (means, cov, sh, opac)]
    c = render_views(flat(e), flat(intr), flat(near), flat(far), hw, bg[None].expand(b * v, 3), *L).reshape(b, v, 3, *hw)
    d = render_depth(L[0], L[1], L[3], e, intr, near, far, hw)
    if grad:
        (((c[:, 1:-1] - target[:, 1:-1]) ** 2).mean() + 1e-3 * d.mean()).backward()
    return c


def fused_route(grad):
    e = ext.clone().requires_grad_(True)
    L = [t.clone().requires_grad_(grad) for t in (means, cov, sh, opac)]
    c, d = decoder_forward(*L, e, intr, near, far, hw, bg, depth_mode="depth")
    if grad:
        (((c[:, 1:-1] - target[:, 1:-1]) ** 2).mean() + 1e-3 * d.mean()).backward()
    return c


def pose_leg(rounds=3):
    from pf3plat_b200.rasterizer import last_stats
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    streams = {fn.__name__: torch.cuda.Stream(dev) for fn in (two_pass_route, fused_route)}
    res = {k: {"fwd": [], "fwd_bwd": [], "peak_torch_mb": 0.0, "pool_reserved_mb": 0.0} for k in streams}
    for _ in range(rounds):
        for fn in (two_pass_route, fused_route):
            name = fn.__name__
            with torch.cuda.stream(streams[name]):
                res[name]["fwd"].append(timeit(fn, False))
                torch.cuda.reset_peak_memory_stats(dev)
                res[name]["fwd_bwd"].append(timeit(fn, True))
                res[name]["peak_torch_mb"] = max(res[name]["peak_torch_mb"], torch.cuda.max_memory_allocated(dev) / 2**20)
                res[name]["pool_reserved_mb"] = max(res[name]["pool_reserved_mb"],
                                                    last_stats(dev)["pool_reserved_bytes"] / 2**20)
    out = {"config": f"GS_POSE: {b} scenes x {v} views, {P} Gaussians/scene, 256x256, extrinsics requiring grad, "
                     f"loss MSE(color[:, 1:-1]) + 1e-3 mean(depth)", "steps": steps, "rounds (alternating)": rounds,
           "device": torch.cuda.get_device_name(dev), "nvidia-smi name, power.limit": q.stdout.strip()}
    for name, r in res.items():
        out[name + "_ms"] = {k: {"median": sorted(r[k])[len(r[k]) // 2], "all": [round(x, 3) for x in r[k]]}
                             for k in ("fwd", "fwd_bwd")}
        out[name + "_memory_mb"] = {k: round(r[k], 1) for k in ("peak_torch_mb", "pool_reserved_mb")}
    print(json.dumps(out))


if POSE:
    pose_leg()
    sys.exit(0)

out = {"config": f"{b} scenes x {v} views, {P} Gaussians/scene, 256x256, colour+depth", "steps": steps,
       "reference_call_pattern_ms": {"fwd": timeit(ref_fwd, False), "fwd_bwd": timeit(ref_fwd, True)},
       "batched_decoder_forward_ms": {"fwd": timeit(ours_fwd, False), "fwd_bwd": timeit(ours_fwd, True)}}
out["speedup"] = {k: out["reference_call_pattern_ms"][k] / out["batched_decoder_forward_ms"][k] for k in ("fwd", "fwd_bwd")}
print(json.dumps(out))
