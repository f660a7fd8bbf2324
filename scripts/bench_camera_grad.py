"""What the camera gradient (gs_backward_cam_tanfov) costs.  Forward + backward with the setting off, on for the
extrinsics, and on for the extrinsics and the intrinsics, alternated in one process, medians over rounds; besides the times, every stage of the library (gs_get_stage_ms, in a separate profiled pass)
and what is left of the step outside the library.  Prints one JSON line with the card's name, power limit and clock, read in the same run.
  * PF3plat's training shape: b = 14 scenes x v = 3 views, 131072 Gaussians per scene (2 x 256 x 256), 256x256,
    decoder_forward(depth_mode="depth") on poses that require grad, loss = MSE on the colour + mean depth (off: the depth
    channel's z column reaches the poses; on: the full gradient; with the intrinsics: they require grad too);
  * C2: 500k Gaussians x 8 views x 256x256, M = 25, loss = <W, colour>, the three camera inputs requiring grad (and
    tanfov, with the intrinsics).
Usage: python scripts/bench_camera_grad.py [--steps K] [--warmup W] [--rounds R]"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pf3plat_b200.cameras import make_view_batch  # noqa: E402
from pf3plat_b200.rasterizer import BatchSettings, rasterize_batch, set_profiling, stage_ms  # noqa: E402
from pf3plat_b200.render import decoder_forward  # noqa: E402
from pf3plat_b200.synthetic import make_pixel_aligned_scene, make_scene, make_target  # noqa: E402
from scripts.bench_alpha import card, median, timed  # noqa: E402

# (name, camera gradients on, intrinsics / tanfov requiring grad)
SETTINGS = (("off", False, False), ("extrinsics", True, False), ("extrinsics+intrinsics", True, True))


def _measure(step, dev, args):
    out = {name: [] for name, _, _ in SETTINGS}
    for _ in range(args.rounds):
        for name, on, intr in SETTINGS:
            out[name].append(timed(lambda: step(on, intr), args.steps, args.warmup))
    stages = {}
    for name, on, intr in SETTINGS:   # stage times in a pass of their own (profiling synchronises every stage)
        set_profiling(True, dev)
        ms = []
        for _ in range(args.steps):
            step(on, intr)
            torch.cuda.synchronize()
            ms.append(stage_ms(dev))
        set_profiling(False, dev)
        stages[name] = {k: median([m[k] for m in ms]) for k in ms[0]}
        stages[name]["library_total"] = sum(stages[name].values())
    # the rest of a step is outside the library: the torch glue (make_view_batch's straight-through expressions and their
    # backward, autograd, the loss), measured here as the step time less the library's stages
    med = {n: median(x) for n, x in out.items()}
    outside = {n: med[n] - stages[n]["library_total"] for n in med}
    return {"fwd_bwd_ms_median": med, "stage_ms_median": stages, "outside_library_ms": outside}


def training_shape(args, dev):
    b, v, hw = 14, 3, (256, 256)
    scs = [make_pixel_aligned_scene(256, 256, v, seed=30 + k) for k in range(b)]
    st = lambda n: torch.stack([getattr(s, n) for s in scs]).to(dev)
    L = [st(n).clone().requires_grad_(True) for n in ("means", "covariances", "harmonics", "opacities")]
    ext = st("extrinsics").clone().requires_grad_(True)
    intr = st("intrinsics")
    intr_g = intr.clone().requires_grad_(True)
    near, far = torch.full((b, v), 1.0, device=dev), torch.full((b, v), 100.0, device=dev)
    bg = torch.zeros(3, device=dev)
    tgt = make_target(b * v, *hw).to(dev).reshape(b, v, 3, *hw)

    def step(on, with_intr):
        color, depth = decoder_forward(*L, ext, intr_g if with_intr else intr, near, far, hw, bg, depth_mode="depth",
                                       camera_gradients=on)
        (((color - tgt) ** 2).mean() + depth.mean()).backward()

    return {"b": b, "v": v, "gaussians_per_scene": int(L[0].shape[1]), "hw": list(hw), **_measure(step, dev, args)}


def c2(args, dev):
    sc = make_scene(500_000, 8, 256, 256, seed=0)
    vb = make_view_batch(sc.extrinsics, sc.intrinsics, sc.near, sc.far)
    c = sc.covariances
    cov6 = torch.stack([c[:, 0, 0], c[:, 0, 1], c[:, 0, 2], c[:, 1, 1], c[:, 1, 2], c[:, 2, 2]], -1)
    leaves = [t[None].to(dev).contiguous().requires_grad_(True)
              for t in (sc.means, sc.opacities, sc.harmonics.permute(0, 2, 1), cov6)]
    W = make_target(8, 256, 256).to(dev)
    cams = dict(viewmatrix=vb.viewmatrix.to(dev).requires_grad_(True), projmatrix=vb.projmatrix.to(dev).requires_grad_(True),
                campos=vb.campos.to(dev).requires_grad_(True), bg=sc.background.to(dev), tanfov=vb.tanfov.to(dev),
                view_scale=vb.scale.to(dev))
    bs = BatchSettings(image_height=256, image_width=256, sh_degree=4, **cams)
    tan_g = cams["tanfov"].clone().requires_grad_(True)

    def step(on, with_intr):
        b = bs._replace(camera_gradients=on, tanfov=tan_g if with_intr else bs.tanfov)
        out = rasterize_batch(b, leaves[0], leaves[1], shs=leaves[2], cov3D_precomp=leaves[3])
        (out[0] * W).sum().backward()

    return {"gaussians": int(leaves[0].shape[1]), "views": 8, "hw": [256, 256], **_measure(step, dev, args)}


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
