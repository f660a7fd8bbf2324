"""k_preprocess on the steady-state speculative path (fused bucket emission into per-view depth strata, the path the bench
runs) against the exact-capacity path (k_preprocess counting, then k_emit_buckets from the stored rects and records), on
identical inputs: images, radii and depths bit for bit, and the deterministic backward's gradients bit for bit (they are
computed from the records, meta, point_list and ranges the forward kept).  Shapes: the bench's C2, the pixel-aligned C5
shape, SH with M = 9, and two scenes of eleven views each (two camera chunks per scene)."""
import numpy as np
import pytest
import torch

from pf3plat_b200.synthetic import make_pixel_aligned_scene, make_scene, make_target
from tests.batch_oracle import scene_batch_args
from tests.regimes import stacked_views_cameras

pytestmark = pytest.mark.gpu


def _dev():
    assert torch.cuda.is_available(), "GPU test needs CUDA"
    return torch.device("cuda:0")


def _single_scene(sc, dev):
    from pf3plat_b200.cameras import make_view_batch
    d = sc.to(dev)
    vb = make_view_batch(d.extrinsics, d.intrinsics, d.near, d.far, scale_invariant=True)
    c = d.covariances
    cams = {"viewmatrix": vb.viewmatrix, "projmatrix": vb.projmatrix, "campos": vb.campos, "bg": d.background,
            "tanfov": vb.tanfov, "view_scale": vb.scale}
    ins = {"means3D": d.means[None], "opacities": d.opacities[None], "shs": d.harmonics.permute(0, 2, 1).contiguous()[None],
           "cov3D_precomp": torch.stack([c[:, 0, 0], c[:, 0, 1], c[:, 0, 2], c[:, 1, 1], c[:, 1, 2], c[:, 2, 2]], -1)[None]}
    return cams, ins, tuple(sc.image_shape)


def _case(name, dev):
    if name == "c2":
        return _single_scene(make_scene(500_000, 8, 256, 256, seed=0), dev)
    if name == "c5_aligned":
        return _single_scene(make_pixel_aligned_scene(128, 128, 4, seed=0), dev)
    if name == "m9":
        return _single_scene(make_scene(30_000, 5, 96, 128, seed=3, d_sh=9), dev)
    # two scenes x eleven views: two camera chunks per scene, per-view view_scale
    S, VPS, hw = 2, 11, (48, 64)
    scenes = [stacked_views_cameras(make_scene(4000, VPS, *hw, seed=70 + k)) for k in range(S)]
    cams, ins = scene_batch_args(scenes, near=1.0 / np.tile(np.linspace(0.8, 1.25, VPS), S), device=dev)
    return cams, {k: ins[k] for k in ("means3D", "opacities", "shs", "cov3D_precomp")}, hw


def _call(cams, ins, hw, tuning, target):
    from pf3plat_b200.rasterizer import BatchSettings, last_stats, rasterize_batch
    bs = BatchSettings(image_height=hw[0], image_width=hw[1], viewmatrix=cams["viewmatrix"], projmatrix=cams["projmatrix"],
                       campos=cams["campos"], bg=cams["bg"], sh_degree=4, tanfov=cams["tanfov"],
                       view_scale=cams["view_scale"], with_depth=True, tuning=tuning)
    leaves = {k: v.detach().clone().requires_grad_(True) for k, v in ins.items()}
    color, radii, depth = rasterize_batch(bs, **leaves)
    spec = last_stats(bs.viewmatrix.device)["speculative"]
    ((color - target) ** 2).mean().add(1e-3 * depth.mean()).backward()
    return [color.detach(), radii, depth.detach()], {k: t.grad for k, t in leaves.items()}, spec


@pytest.mark.parametrize("name", ["c2", "c5_aligned", "m9", "two_scenes_vps11"])
def test_speculative_preprocess_matches_exact_path(name):
    from pf3plat_b200._capi import GS_TUNE_NO_SPECULATION
    dev = _dev()
    cams, ins, hw = _case(name, dev)
    V = cams["viewmatrix"].shape[0]
    target = make_target(V, *hw, seed=5).to(dev)
    stream = torch.cuda.Stream(dev)          # a context of its own: the shape's speculation starts from scratch
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        with torch.cuda.stream(stream):
            ref_out, ref_grads, _ = _call(cams, ins, hw, GS_TUNE_NO_SPECULATION, target)
            states = []
            for _ in range(4):               # the exact reference call learned the capacities: trial, then stratified
                out, grads, spec = _call(cams, ins, hw, 0, target)
                states.append(spec)
            stream.synchronize()
    finally:
        torch.use_deterministic_algorithms(prev)
    print(f"[equiv] {name}: speculative per call {states}")
    assert states[-1] > 0, f"{name}: the last call did not run on the speculative path ({states})"
    for label, a, b in zip(("color", "radii", "depth"), out, ref_out):
        assert torch.equal(a, b), f"{name}: {label} differs from the exact path"
    for k in ref_grads:
        assert torch.equal(grads[k], ref_grads[k]), f"{name}: dL/d{k} differs from the exact path"
