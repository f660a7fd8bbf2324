"""Times PF3plat's encoder depth glue on one GPU: pf3plat_b200.encoder_depth (depth_update, mono_cue, pdf_peak; the
kernels of csrc/gs_encoder_depth.cu) against the reference's PyTorch op sequence, restated below (`reference_*`; the
mono cue's restatement is pinned to the reference's own lines by tests/test_encoder_depth_cpu.py).

One step is encoder_costvolume.py:265-307 and :506-528 (clamp, the upsampled shift, the updated depth, the mono cue and
both unprojections) plus depth_predictor_multiview.py:379-384 (pdf_max).  The forward + backward step adds a loss on
depths, both unprojections and pdf_max and its backward into the scale-shift head's output and the logits.  Shape:
PF3plat's training step, b = 14, v = 3 (the target joins the context), 256 x 256, D = 128 (re10k.yaml).  The
feature grid the scale-shift head runs on is set by UniDepth's resize, which is not recorded here: 28 x 28 and
42 x 42 are assumptions.  The routes alternate within one run; a round is --steps steps between two device
synchronisations, timed with CUDA events, and the median over --rounds rounds is reported with the spread
((max - min) / median).  Also per route: the peak allocation above the inputs, the kernel launches of one step
(torch.profiler), and the synchronising calls of one step, counted under torch.cuda.set_sync_debug_mode("warn").
Also reported: the card, its power limit and its maximum SM clock.

Usage:  python scripts/bench_encoder_depth.py [--steps 10] [--warmup 3] [--rounds 9] [--out DIR]
Writes DIR/bench_encoder_depth.json (default: a temporary directory) and prints it.
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
import torch.nn.functional as F
from einops import rearrange, repeat

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pf3plat_b200 import encoder_depth  # noqa: E402

SHAPES = {  # name: (b, v, h, w, grid, D)
    "pf3plat_train_b14_v3_256_grid28": (14, 3, 256, 256, (28, 28), 128),
    "pf3plat_train_b14_v3_256_grid42": (14, 3, 256, 256, (42, 42), 128),
}


# ---- the reference's op sequence (encoder_costvolume.py, depth_predictor_multiview.py, projection.py) ----

def sample_image_grid(h, w, device):
    ys, xs = torch.meshgrid((torch.arange(h, device=device) + 0.5) / h, (torch.arange(w, device=device) + 0.5) / w,
                            indexing="ij")
    return torch.stack([xs, ys], -1)


def unproject(coordinates, z, intrinsics):
    coordinates = torch.cat([coordinates, torch.ones_like(coordinates[..., :1])], dim=-1)
    ray_directions = torch.einsum("...ij,...j->...i", intrinsics.inverse(), coordinates)
    return ray_directions * z[..., None]


def reference_route(depth, scale_shift, K, near, far, grid, logits):
    b, v = near.shape
    h, w = depth.shape[-2:]
    gh, gw = grid
    nf = lambda t: rearrange(t, "b v -> (b v) () () ()")  # noqa: E731
    depths = depth.clamp(nf(near), nf(far))
    ss = rearrange(F.interpolate(rearrange(scale_shift, "b v (h w) c -> (b v) c h w", h=gh, w=gw), (h, w),
                                 mode="bilinear"), "(b v) c h w -> b v (h w) c", v=v)
    scale, shift = torch.chunk(ss, 2, dim=-1)
    scale = scale.exp()
    shift = rearrange(shift.clamp(min=-5, max=5), "b v (h w) 1 -> (b v) 1 h w", h=h, w=w)
    depths = (depths + shift).clamp(nf(near), nf(far))
    disparity_down = F.interpolate(depths, (h // 4, w // 4), mode="bilinear")
    hyp = ((1.0 / far)[0, 0].item() + torch.linspace(0.0, 1.0, 128).unsqueeze(0).to(depths.device)
           * ((1.0 / near)[0, 0].item() - (1.0 / far)[0, 0].item())).view(1, -1, 1, 1).expand(
        b * v, -1, h // 4, w // 4).detach()
    idx = torch.argmin(torch.abs(disparity_down - hyp), dim=1, keepdim=True)
    cue = rearrange(hyp.new_zeros(hyp.shape).scatter_(dim=1, index=idx, src=hyp.new_ones(hyp.shape)).detach(),
                    "(b v) c h w -> (v b) c h w", b=b, v=v)
    grid_up = repeat(sample_image_grid(h, w, depth.device), "h w c -> b h w c", b=b).permute(0, 3, 1, 2)
    coords = repeat(grid_up.flatten(-2, -1), "b c N -> (b v) c N", v=v).permute(0, 2, 1)
    Kr = rearrange(K, "b v c k -> (b v) 1 c k")
    xyz_up_h = rearrange(unproject(coords, rearrange(depths.flatten(-2, -1), "(b v) 1 N -> (b v) N", b=b, v=v), Kr),
                         "(b v) (h w) c -> b v c h w", b=b, v=v, h=h, w=w)
    depths_refine = rearrange(depths, "(b v) 1 h w -> b v (h w) 1", b=b, v=v).unsqueeze(-1).clamp(
        rearrange(near, "b v -> b v () () ()"), rearrange(far, "b v -> b v () () ()"))
    xyz_refine = rearrange(unproject(coords, rearrange(depths_refine.squeeze(-1), "b v N 1 -> (b v) N"), Kr),
                           "(b v) (h w) c -> b v c h w", b=b, v=v, h=h, w=w)
    depths_final = rearrange(depths_refine, "b v (h w) c 1 -> (b v) c h w", h=h, w=w)
    pdf = F.softmax(logits, dim=1)
    pdf_max = F.interpolate(torch.max(pdf, dim=1, keepdim=True)[0], scale_factor=4)
    return depths_final, xyz_up_h, xyz_refine, cue, pdf_max


def ours_route(depth, scale_shift, K, near, far, grid, logits):
    b, v = near.shape
    depths, xyz = encoder_depth.depth_update(depth, scale_shift, K, near, far, grid)
    cue = encoder_depth.mono_cue(depths, near, far, b, v)
    return depths, xyz, xyz, cue, encoder_depth.pdf_peak(logits, 4)


ROUTES = {"reference_ops": reference_route, "ours": ours_route}


def seeded_inputs(b, v, h, w, grid, D, dev, seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)
    near = 0.5 + torch.rand((b, v), generator=g, device=dev)
    far = near + 50.0 + 50.0 * torch.rand((b, v), generator=g, device=dev)
    depth = (0.2 + torch.rand((b * v, 1, h, w), generator=g, device=dev)) * 40.0
    ss = torch.randn((b, v, grid[0] * grid[1], 2), generator=g, device=dev) * 3.0
    K = torch.tensor([[1.0, 0.0, 0.5], [0.0, 1.0, 0.5], [0.0, 0.0, 1.0]], device=dev).expand(b, v, 3, 3).contiguous()
    logits = torch.randn((v * b, D, h // 4, w // 4), generator=g, device=dev) * 2.0
    cot = [torch.randn(s, generator=g, device=dev) for s in ((b * v, 1, h, w), (b, v, 3, h, w), (v * b, 1, h, w))]
    return near, far, depth, ss, K, logits, grid, cot


def step(route, inp, backward):
    near, far, depth, ss0, K, logits0, grid, (gd, gx, gp) = inp
    ss = ss0.detach().requires_grad_(backward)
    logits = logits0.detach().requires_grad_(backward)
    depths, xa, xb, cue, peak = ROUTES[route](depth, ss, K, near, far, grid, logits)
    if backward:
        ((depths * gd).sum() + (xa * gx).sum() + (xb * gx).sum() + (peak * gp).sum()).backward()
    return depths, xa, cue, peak


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
        raise SystemExit("bench_encoder_depth.py needs a CUDA device")
    dev = torch.device("cuda:0")
    info = {"device": torch.cuda.get_device_name(dev)}
    try:
        info["power_limit_and_max_sm_clock"] = subprocess.run(
            ["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
            capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError) as e:
        info["power_limit_and_max_sm_clock"] = f"unavailable: {e}"
    results = {}
    for name, (b, v, h, w, grid, D) in SHAPES.items():
        inp = seeded_inputs(b, v, h, w, grid, D, dev)
        for route in ROUTES:
            for backward in (False, True):
                for _ in range(args.warmup):
                    step(route, inp, backward)
        torch.cuda.synchronize()
        ref = [t.detach() for t in step("reference_ops", inp, False)]
        got = [t.detach() for t in step("ours", inp, False)]
        res = {"max_abs_diff": {k: float((r - o).abs().max()) for k, r, o in
                                zip(("depths", "xyz", "mono_cue", "pdf_max"), ref, got)},
               "mono_cue_equal": bool(torch.equal(ref[2], got[2]))}
        del ref, got
        for label, backward in (("forward", False), ("forward_backward", True)):
            times = {r: [] for r in ROUTES}
            for _ in range(args.rounds):
                for r in ROUTES:
                    times[r].append(timed_round(r, inp, backward, args.steps))
            for r, ts in times.items():
                med = statistics.median(ts)
                res[f"{label}_{r}_ms"] = round(med, 4)
                res[f"{label}_{r}_spread"] = round((max(ts) - min(ts)) / med, 3)
            res[f"{label}_speedup"] = round(res[f"{label}_reference_ops_ms"] / res[f"{label}_ours_ms"], 2)
            for r in ROUTES:
                res[f"{label}_{r}_sync_calls"] = count_syncs(r, inp, backward)
                res[f"{label}_{r}_launches"] = count_launches(r, inp, backward)
                res[f"{label}_{r}_peak_mib_above_inputs"] = peak_mib(r, inp, backward)
        results[name] = res
    x = torch.randn(6, 2, 28, 28, device=dev, requires_grad=True)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        F.interpolate(x, (256, 256), mode="bilinear").sum().backward()
        verdict = "runs"
    except RuntimeError as e:
        verdict = "raises: " + str(e).splitlines()[0]
    finally:
        torch.use_deterministic_algorithms(prev)
    out = {"bench": "encoder_depth", **info, "torch": torch.__version__, "steps": args.steps, "rounds": args.rounds,
           "reference_bilinear_backward_under_deterministic_algorithms": verdict, "shapes": results}
    out_dir = args.out or tempfile.mkdtemp(prefix="bench_encoder_depth_")
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "bench_encoder_depth.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
