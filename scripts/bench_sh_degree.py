"""What the opt-in degree-4 SH evaluation (sh_eval_max_degree = 4) costs against the default degree 3, on the same inputs,
the two degrees alternating in one process.  Prints one JSON line with the card's name and power limit.
  * C2: 500k Gaussians x 8 views x 256x256, M = 25: forward, forward + backward, and the preprocess / preprocess-backward
    stage times (CUDA events of the library's profiling mode);
  * PF3plat's training shape: b = 14 scenes x v = 3 views, 131072 Gaussians per scene (2 x 256 x 256), 256x256,
    decoder_forward(depth_mode="depth") on poses that require grad, forward + backward.
The scenes carry band-4 coefficients of the same order as the other bands, so both degrees see the same non-zero inputs.
Usage: python scripts/bench_sh_degree.py [--steps K] [--warmup W] [--skip-decoder]"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pf3plat_b200 import rasterizer  # noqa: E402
from pf3plat_b200.cameras import make_view_batch  # noqa: E402
from pf3plat_b200.rasterizer import BatchSettings, rasterize_batch  # noqa: E402
from pf3plat_b200.render import decoder_forward  # noqa: E402
from pf3plat_b200.synthetic import make_pixel_aligned_scene, make_scene, make_target  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [s.strip() for s in out.split(",")]
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def band4(harmonics, seed):
    g = torch.Generator().manual_seed(seed)
    h = harmonics.clone()
    h[..., 16:25] = 0.05 * torch.randn(*h.shape[:-1], 9, generator=g)
    return h


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--skip-decoder", action="store_true")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    name, limit = card()
    res = {"card": name, "power_limit": limit, "steps": args.steps, "rounds": args.rounds}

    # ---- C2 ----
    sc = make_scene(500_000, 8, 256, 256, seed=0)
    vb = make_view_batch(sc.extrinsics, sc.intrinsics, sc.near, sc.far)
    c = sc.covariances
    cov6 = torch.stack([c[:, 0, 0], c[:, 0, 1], c[:, 0, 2], c[:, 1, 1], c[:, 1, 2], c[:, 2, 2]], -1)
    means = sc.means[None].to(dev).contiguous()
    opac = sc.opacities[None].to(dev).contiguous()
    shs = band4(sc.harmonics, 1).permute(0, 2, 1)[None].to(dev).contiguous()
    cov6 = cov6[None].to(dev).contiguous()
    W = make_target(8, 256, 256).to(dev)
    cams = dict(viewmatrix=vb.viewmatrix.to(dev), projmatrix=vb.projmatrix.to(dev), campos=vb.campos.to(dev),
                bg=sc.background.to(dev), tanfov=vb.tanfov.to(dev), view_scale=vb.scale.to(dev))
    leaves = [t.clone().requires_grad_(True) for t in (means, opac, shs, cov6)]
    c2 = {3: {"fwd": [], "fwd_bwd": [], "preprocess": [], "preprocess_bwd": []},
          4: {"fwd": [], "fwd_bwd": [], "preprocess": [], "preprocess_bwd": []}}
    for _ in range(args.rounds):
        for deg in (3, 4):
            bs = BatchSettings(image_height=256, image_width=256, sh_degree=4, sh_eval_max_degree=deg, **cams)
            with torch.no_grad():
                c2[deg]["fwd"].append(timed(lambda: rasterize_batch(bs, means, opac, shs=shs, cov3D_precomp=cov6),
                                            args.steps, args.warmup))

            def fb():
                col, _ = rasterize_batch(bs, *leaves[:2], shs=leaves[2], cov3D_precomp=leaves[3])
                (col * W).sum().backward()
            c2[deg]["fwd_bwd"].append(timed(fb, args.steps, args.warmup))
            rasterizer.set_profiling(True)
            fb()
            torch.cuda.synchronize()
            ms = rasterizer.stage_ms()
            rasterizer.set_profiling(False)
            c2[deg]["preprocess"].append(ms["preprocess"])
            c2[deg]["preprocess_bwd"].append(ms["preprocess_bwd"])
    res["c2_ms_median"] = {str(d): {k: sorted(v)[len(v) // 2] for k, v in c2[d].items()} for d in (3, 4)}
    del leaves, means, opac, shs, cov6
    torch.cuda.empty_cache()

    # ---- PF3plat's training shape ----
    if not args.skip_decoder:
        b, v, hw = 14, 3, (256, 256)
        scs = [make_pixel_aligned_scene(256, 256, v, seed=30 + k) for k in range(b)]
        st = lambda n: torch.stack([getattr(s, n) for s in scs]).to(dev)
        mean, cov, opa = st("means"), st("covariances"), st("opacities")
        harm = band4(st("harmonics").cpu(), 2).to(dev)
        ext0, intr = st("extrinsics"), st("intrinsics")
        near = torch.full((b, v), 1.0, device=dev)
        far = torch.full((b, v), 100.0, device=dev)
        bgc = torch.zeros(3, device=dev)
        tgt = make_target(b * v, *hw).to(dev).reshape(b, v, 3, *hw)
        dec = {3: [], 4: []}
        h = harm.clone().requires_grad_(True)
        ext = ext0.clone().requires_grad_(True)
        for _ in range(args.rounds):
            for deg in (3, 4):
                def step():
                    col, dep = decoder_forward(mean, cov, h, opa, ext, intr, near, far, hw, bgc, depth_mode="depth",
                                               sh_eval_max_degree=deg)
                    (((col - tgt) ** 2).mean() + 1e-3 * dep.mean()).backward()
                dec[deg].append(timed(step, max(args.steps // 2, 3), args.warmup))
        res["pf3plat_decoder_fwd_bwd_ms_median"] = {str(d): sorted(dec[d])[len(dec[d]) // 2] for d in (3, 4)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
