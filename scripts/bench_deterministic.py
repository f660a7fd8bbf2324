"""Cost of the deterministic backward (torch.use_deterministic_algorithms(True) -> GS_FLAG_DETERMINISTIC /
GS_ADAPTER_DETERMINISTIC) against the default one, alternating the two in one process:

  1. C2 (500k Gaussians x 8 views x 256x256, SH 25 coefficients, MSE loss): the backward alone (CUDA events around
     loss.backward(), and the library's own stage timers of its two backward kernels).
  2. PF3plat's training shape, b = 14 scenes x 3 target views (2 context views of 256x256 each: 131072 Gaussians per
     scene): adapter -> decoder_forward(depth_mode="depth") on target extrinsics that require grad -> photometric_loss
     -> backward, the whole step; and the rasterizer context's pool reservation.

Prints the card's name and power limit, then one JSON line.  Usage: python scripts/bench_deterministic.py [--steps N]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # the numbers below still stand; say that the card could not be queried
        q = f"{torch.cuda.get_device_name(0)}, power limit unknown ({e})"
    return q


def alternate(fn, steps, warmup):
    """fn(det) -> ms; runs det and default alternately; medians."""
    out = {True: [], False: []}
    for i in range(warmup + steps):
        for det in (i % 2 == 0, i % 2 != 0):
            torch.use_deterministic_algorithms(det)
            ms = fn(det)
            if i >= warmup:
                out[det].append(ms)
    torch.use_deterministic_algorithms(False)
    return {("deterministic" if k else "default"): statistics.median(v) for k, v in out.items()}


def c2(steps, warmup):
    from pf3plat_b200.cameras import make_view_batch
    from pf3plat_b200.rasterizer import BatchSettings, rasterize_batch, set_profiling, stage_ms
    from pf3plat_b200.synthetic import make_scene, make_target
    P, V, HW = 500_000, 8, 256
    dev = torch.device("cuda:0")
    sc = make_scene(P, V, HW, HW, seed=0)
    vb = make_view_batch(sc.extrinsics, sc.intrinsics, sc.near, sc.far, scale_invariant=True)
    c = sc.covariances
    ins = {"means3D": sc.means.reshape(1, P, 3), "opacities": sc.opacities.reshape(1, P),
           "shs": sc.harmonics.permute(0, 2, 1).contiguous().reshape(1, P, -1, 3),
           "cov3D_precomp": torch.stack([c[:, 0, 0], c[:, 0, 1], c[:, 0, 2], c[:, 1, 1], c[:, 1, 2], c[:, 2, 2]],
                                        -1).reshape(1, P, 6)}
    leaves = {k: v.to(dev).contiguous().requires_grad_(True) for k, v in ins.items()}
    bs = BatchSettings(image_height=HW, image_width=HW, viewmatrix=vb.viewmatrix.to(dev), projmatrix=vb.projmatrix.to(dev),
                       campos=vb.campos.to(dev), bg=sc.background.to(dev), sh_degree=4, tanfov=vb.tanfov.to(dev))
    target = make_target(V, HW, HW, seed=1).to(dev)
    kernels = {True: [], False: []}
    set_profiling(True, dev)

    def step(det):
        for t in leaves.values():
            t.grad = None
        color, _ = rasterize_batch(bs, **leaves)
        loss = ((color - target) ** 2).mean()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        loss.backward()
        b.record()
        b.synchronize()
        st = stage_ms(dev)
        kernels[det].append(st["composite_bwd"] + st["preprocess_bwd"])
        return a.elapsed_time(b)

    res = alternate(step, steps, warmup)
    set_profiling(False, dev)
    res["kernels_deterministic"] = statistics.median(kernels[True][warmup:])
    res["kernels_default"] = statistics.median(kernels[False][warmup:])
    return {k: round(v, 4) for k, v in res.items()}


def chain(steps, warmup):
    from pf3plat_b200.adapter import GaussianAdapter, GaussianAdapterCfg
    from pf3plat_b200.losses import photometric_loss
    from pf3plat_b200.rasterizer import last_stats
    from pf3plat_b200.render import decoder_forward
    from pf3plat_b200.synthetic import make_target
    from tests.chain_oracle import make_chain_inputs
    dev = torch.device("cuda:0")
    b, vc, vt, chw, hw, deg = 14, 2, 3, (256, 256), (256, 256), 4
    inp = make_chain_inputs(5, b, vc, chw, vt, deg, 1.0)
    G = vc * chw[0] * chw[1]
    adapter = GaussianAdapter(GaussianAdapterCfg(gaussian_scale_min=0.5, gaussian_scale_max=15.0, sh_degree=deg)).to(dev)
    target = make_target(b * vt, *hw, seed=2).to(dev).reshape(b, vt, 3, *hw)
    bg = torch.zeros(3, device=dev)
    d = {k: v.to(dev) for k, v in inp.items()}
    pool = {}

    def step(det):
        L = {k: d[k].clone().requires_grad_(True) for k in ("extrinsics", "intrinsics", "coordinates", "depths",
                                                            "opacities", "raw_gaussians", "target_extrinsics")}
        a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        g = adapter.forward(L["extrinsics"][:, :, None], L["intrinsics"][:, :, None], L["coordinates"], L["depths"],
                            L["opacities"], L["raw_gaussians"], chw)
        color, depth = decoder_forward(g.means.reshape(b, G, 3), g.covariances.reshape(b, G, 3, 3),
                                       g.harmonics.reshape(b, G, 3, -1), g.opacities.reshape(b, G),
                                       L["target_extrinsics"], d["target_intrinsics"], d["near"], d["far"], hw, bg,
                                       depth_mode="depth")
        mse, ssim = photometric_loss(color, target)
        (mse + ssim + 1e-3 * depth.mean()).backward()
        e.record()
        e.synchronize()
        pool[det] = max(pool.get(det, 0), last_stats(dev)["pool_reserved_bytes"])
        return a.elapsed_time(e)

    res = alternate(step, steps, warmup)
    res = {k: round(v, 3) for k, v in res.items()}
    res["pool_reserved_mb"] = round(max(pool.values()) / 2 ** 20, 1)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU (no CPU fallback exists)"
    gpu = card()
    print(f"card: {gpu}", flush=True)
    out = {"card": gpu, "c2_backward_ms": c2(args.steps, args.warmup),
           "training_chain_step_ms": chain(max(args.steps // 2, 4), args.warmup)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
