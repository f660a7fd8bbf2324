"""What the fused accumulated opacity costs, against the route without it: a second full render of the same Gaussians with
colours 1 on a black background, whose channel 0 is 1 - T_final.  Three routes alternate in one process, medians over
rounds: "none" (colour only, no alpha), "fused" (alpha from the colour pass: gs_forward_ex / gs_backward_ex) and
"two_pass".  Prints one JSON line with the card's name and power limit, read in the same run.
  * PF3plat's training shape: b = 14 scenes x v = 3 views, 131072 Gaussians per scene (2 x 256 x 256), 256x256,
    decoder_forward with the Gaussians requiring grad, loss = MSE on the colour + 0.1 x mean alpha: forward, forward +
    backward;
  * C2: 500k Gaussians x 8 views x 256x256, M = 25, loss = <W, colour> + 0.1 x mean alpha: forward, forward + backward.
Usage: python scripts/bench_alpha.py [--steps K] [--warmup W] [--rounds R]"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pf3plat_b200.cameras import make_view_batch  # noqa: E402
from pf3plat_b200.rasterizer import BatchSettings, rasterize_batch  # noqa: E402
from pf3plat_b200.render import decoder_forward, render_views  # noqa: E402
from pf3plat_b200.synthetic import make_pixel_aligned_scene, make_scene, make_target  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit, clock = [s.strip() for s in out.split(",")]
        return name, limit, clock
    except Exception:
        return torch.cuda.get_device_name(0), "unknown", "unknown"


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


def median(xs):
    return sorted(xs)[len(xs) // 2]


ROUTES = ("none", "fused", "two_pass")


def training_shape(args, dev):
    b, v, hw = 14, 3, (256, 256)
    scs = [make_pixel_aligned_scene(256, 256, v, seed=30 + k) for k in range(b)]
    st = lambda n: torch.stack([getattr(s, n) for s in scs]).to(dev)
    L = [st(n).clone().requires_grad_(True) for n in ("means", "covariances", "harmonics", "opacities")]
    ext, intr = st("extrinsics"), st("intrinsics")
    near, far = torch.full((b, v), 1.0, device=dev), torch.full((b, v), 100.0, device=dev)
    bg = torch.zeros(3, device=dev)
    tgt = make_target(b * v, *hw).to(dev).reshape(b, v, 3, *hw)
    ones = torch.ones(b, L[0].shape[1], 3, 1, device=dev)
    flat = lambda t: t.reshape(b * v, *t.shape[2:])

    def fwd(route):
        if route == "fused":
            color, _, alpha = decoder_forward(*L, ext, intr, near, far, hw, bg, return_alpha=True)
            return color, alpha
        color, _ = decoder_forward(*L, ext, intr, near, far, hw, bg)
        if route == "none":
            return color, None
        cover = render_views(flat(ext), flat(intr), flat(near), flat(far), hw, torch.zeros(b * v, 3, device=dev), L[0],
                             L[1], ones, L[3], use_sh=False)
        return color, cover[:, 0].reshape(b, v, *hw)

    def step(route):
        color, alpha = fwd(route)
        loss = ((color - tgt) ** 2).mean()
        if alpha is not None:
            loss = loss + 0.1 * alpha.mean()
        loss.backward()

    out = {r: {"fwd": [], "fwd_bwd": []} for r in ROUTES}
    for _ in range(args.rounds):
        for r in ROUTES:
            with torch.no_grad():
                out[r]["fwd"].append(timed(lambda: fwd(r), args.steps, args.warmup))
            out[r]["fwd_bwd"].append(timed(lambda: step(r), args.steps, args.warmup))
    return {"b": b, "v": v, "gaussians_per_scene": int(L[0].shape[1]), "hw": list(hw),
            "ms_median": {r: {k: median(x) for k, x in out[r].items()} for r in ROUTES}}


def c2(args, dev):
    sc = make_scene(500_000, 8, 256, 256, seed=0)
    vb = make_view_batch(sc.extrinsics, sc.intrinsics, sc.near, sc.far)
    c = sc.covariances
    cov6 = torch.stack([c[:, 0, 0], c[:, 0, 1], c[:, 0, 2], c[:, 1, 1], c[:, 1, 2], c[:, 2, 2]], -1)
    leaves = [t[None].to(dev).contiguous().requires_grad_(True)
              for t in (sc.means, sc.opacities, sc.harmonics.permute(0, 2, 1), cov6)]
    W = make_target(8, 256, 256).to(dev)
    cams = dict(viewmatrix=vb.viewmatrix.to(dev), projmatrix=vb.projmatrix.to(dev), campos=vb.campos.to(dev),
                bg=sc.background.to(dev), tanfov=vb.tanfov.to(dev), view_scale=vb.scale.to(dev))
    bs = BatchSettings(image_height=256, image_width=256, sh_degree=4, **cams)
    ones = torch.ones(8, leaves[0].shape[1], 3, device=dev)
    black = torch.zeros(8, 3, device=dev)

    def fwd(route):
        if route == "fused":
            color, _, alpha = rasterize_batch(bs._replace(with_alpha=True), leaves[0], leaves[1], shs=leaves[2],
                                              cov3D_precomp=leaves[3])
            return color, alpha
        color, _ = rasterize_batch(bs, leaves[0], leaves[1], shs=leaves[2], cov3D_precomp=leaves[3])
        if route == "none":
            return color, None
        cover, _ = rasterize_batch(bs._replace(bg=black), leaves[0], leaves[1], colors_precomp=ones,
                                   cov3D_precomp=leaves[3])
        return color, cover[:, 0]

    def step(route):
        color, alpha = fwd(route)
        loss = (color * W).sum()
        if alpha is not None:
            loss = loss + 0.1 * alpha.mean()
        loss.backward()

    out = {r: {"fwd": [], "fwd_bwd": []} for r in ROUTES}
    for _ in range(args.rounds):
        for r in ROUTES:
            with torch.no_grad():
                out[r]["fwd"].append(timed(lambda: fwd(r), args.steps, args.warmup))
            out[r]["fwd_bwd"].append(timed(lambda: step(r), args.steps, args.warmup))
    return {"gaussians": int(leaves[0].shape[1]), "views": 8, "hw": [256, 256],
            "ms_median": {r: {k: median(x) for k, x in out[r].items()} for r in ROUTES}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    name, limit, clock = card()
    res = {"card": name, "power_limit": limit, "max_sm_clock": clock, "steps": args.steps, "rounds": args.rounds}
    res["training_shape"] = training_shape(args, dev)
    torch.cuda.empty_cache()
    res["c2"] = c2(args, dev)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
