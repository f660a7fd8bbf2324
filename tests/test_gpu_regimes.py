"""GPU parity in the regimes the ordinary synthetic scenes never reach, against the CPU oracle through the batched oracle
(tests/batch_oracle.py): more views per scene than one camera chunk (8) of the preprocess kernels and than one staging
chunk (64) of k_sh_colour; every input combination of the batched operator with per-view view_scale != 1; centres far
outside the frustum (clamped projection Jacobian); splats at the near plane; opaque stacks where alpha clamps at 0.99
and pixels terminate early.

Criteria are tests/util.py's (1e-4 abs RGB outside fragile pixels, element-wise 1e-3 gradient rule per tensor and per SH
band) unless a test derives another.  Every test also asserts, on the oracle's intermediates, that its regime was reached,
and prints the numbers as "[regime]" lines next to the usual "[parity]" reports."""
import ctypes

import numpy as np
import pytest
import torch

from pf3plat_b200.synthetic import make_scene, make_target
from tests.batch_oracle import oracle_batch, scene_batch_args
from tests.regimes import near_plane_scene, offscreen_scene, opaque_stack_scene, stacked_views_cameras
from tests.util import SH_BANDS, affected_gaussians, check_grad, check_image_strict

pytestmark = pytest.mark.gpu


def _dev():
    assert torch.cuda.is_available(), "GPU test needs CUDA"
    return torch.device("cuda:0")


def _settings(cams, hw, sh_degree=4, scale_modifier=1.0, with_depth=False, tuning=0):
    from pf3plat_b200.rasterizer import BatchSettings
    return BatchSettings(image_height=hw[0], image_width=hw[1], viewmatrix=cams["viewmatrix"],
                         projmatrix=cams["projmatrix"], campos=cams["campos"], bg=cams["bg"], sh_degree=sh_degree,
                         tanfov=cams["tanfov"], view_scale=cams["view_scale"], scale_modifier=scale_modifier,
                         with_depth=with_depth, tuning=tuning)


def _loss_grads(ob, seed=1, depth_weight=1e-3):
    """dL/dcolor (and dL/ddepth) of an MSE against a seeded target plus a small depth term, from the oracle's images, so
    that the GPU and the oracle are handed identical incoming gradients."""
    V, _, H, W = ob.color.shape
    target = make_target(V, H, W, seed=seed).numpy()
    dL = (2 * (ob.color - target) / target.size).astype(np.float32)
    dLd = np.full((V, H, W), depth_weight / (V * H * W), np.float32) if ob.with_depth else None
    return dL, dLd


def _run(bs, ins, dL=None, dLd=None, means2D=False):
    """rasterize_batch on device copies of `ins` (leaves requiring grad); the backward with the given incoming gradients.
    Returns (outputs, {name: grad})."""
    from pf3plat_b200.rasterizer import rasterize_batch
    dev = bs.viewmatrix.device
    leaves = {k: v.to(dev).clone().requires_grad_(dL is not None) for k, v in ins.items()}
    V, P = bs.viewmatrix.shape[0], ins["means3D"].shape[1]
    if means2D:
        leaves["means2D"] = torch.zeros(V, P, 3, device=dev, requires_grad=True)
    out = rasterize_batch(bs, **leaves)
    if dL is None:
        return [o.detach() for o in out], None
    outs, grads = [out[0]], [torch.as_tensor(dL, device=dev)]
    if dLd is not None:
        outs.append(out[2])
        grads.append(torch.as_tensor(dLd, device=dev))
    torch.autograd.backward(outs, grads)
    return [o.detach() for o in out], {k: t.grad for k, t in leaves.items()}


def _check_images(color, ob, label, max_fragile_frac=0.03, depth=None):
    for v, r in enumerate(ob.views):
        check_image_strict(color[v], r, max_fragile_frac, label=f"{label} view {v}")
        if depth is not None:
            derr = np.abs(depth[v].cpu().numpy() - r.depth)[~r.px_fragile].max()
            assert derr <= 1e-3, (label, v, derr)      # depths reach ~40: 1e-3 abs is ~3e-5 relative


def _check_radii(radii, ob, label):
    r = radii.cpu().numpy()
    for v, orc in enumerate(ob.views):
        ok = (r[v] == orc.radii) | orc.geom_fragile
        assert ok.all(), f"{label} view {v}: {(~ok).sum()} radii differ on non-fragile Gaussians"


def _check_grads(label, grads, gref, aff, VPS, names=None):
    """Every gradient the operator returned, against the batched oracle's: per-scene tensors over S*P Gaussians, per-view
    ones (means2D, colors_precomp) over V*P (a Gaussian of view v is affected if it is affected in its scene)."""
    S, P = aff.shape
    aff_v = np.repeat(aff, VPS, axis=0).reshape(-1)
    for name, t in grads.items():
        if names is not None and name not in names:
            continue
        ref = gref[name]
        if name in ("means2D", "colors_precomp"):
            check_grad(f"{label} dL/d{name}", t.reshape(-1, 3), ref.reshape(-1, 3), aff_v)
        elif name == "shs":
            M = ref.shape[2]
            bands = [b for b in SH_BANDS if b[1].start < M]
            check_grad(f"{label} dL/dshs", t.reshape(S * P, M, 3), ref.reshape(S * P, M, 3), aff.reshape(-1), bands=bands)
        else:
            check_grad(f"{label} dL/d{name}", t.reshape(S * P, -1), ref.reshape(S * P, -1), aff.reshape(-1))


# ---------------------------------------------------------------------------------------------------------------------
# 1. many views per scene
# ---------------------------------------------------------------------------------------------------------------------
def _many_view_batch(dev, S=2, VPS=19, P=2500, hw=(32, 48)):
    """S scenes x VPS views (chunks of 8 + 8 + 3); the chunks of a scene stand 8 units apart along the optical axis, and
    every view has its own near plane (view_scale 0.8 .. 1.25)."""
    scenes = [stacked_views_cameras(make_scene(P, VPS, *hw, seed=50 + k)) for k in range(S)]
    near = 1.0 / np.tile(np.linspace(0.8, 1.25, VPS), S)
    cams, ins = scene_batch_args(scenes, near=near, device=dev)
    ins = {k: ins[k] for k in ("means3D", "opacities", "shs", "cov3D_precomp")}
    return cams, ins, hw


def test_many_views_per_scene_forward_backward_matches_oracle():
    from pf3plat_b200._capi import GS_TUNE_BWD_V1, GS_TUNE_PBWD_2PHASE
    dev = _dev()
    cams, ins, hw = _many_view_batch(dev)
    S, VPS = 2, 19
    ob = oracle_batch(_settings(cams, hw, with_depth=True), **ins)
    assert ob.VPS > 8 and ob.VPS % 8 != 0
    vis = (ob.radii > 0).mean(axis=1)
    zs = [float(np.median(r.depths[r.radii > 0])) for r in ob.views]
    print(f"[regime] many views: S={ob.S} VPS={ob.VPS} P={ob.P}; visible fraction per view {vis.min():.3f}..{vis.max():.3f}; "
          f"median depth of views 0/8/16: {zs[0]:.2f}/{zs[8]:.2f}/{zs[16]:.2f}")
    assert vis.min() > 0.3
    assert zs[8] > zs[0] + 4 and zs[16] > zs[8] + 4         # each camera chunk sees its own depth range
    dL, dLd = _loss_grads(ob)
    gref = ob.backward(dL, dLd)
    aff = ob.affected()
    for tuning, label in ((0, "default"), (GS_TUNE_PBWD_2PHASE, "2-phase preprocess bwd"), (GS_TUNE_BWD_V1, "bwd v1")):
        (color, radii, depth), grads = _run(_settings(cams, hw, with_depth=True, tuning=tuning), ins, dL, dLd)
        _check_images(color, ob, f"VPS=19 {label}", depth=depth)
        _check_radii(radii, ob, label)
        _check_grads(f"VPS=19 {label}", grads, gref, aff, VPS)


def test_many_views_per_scene_speculative_strata():
    """Three calls of the same shape on a fresh context: exact, per-view strata trial, stratified.  Both speculative calls
    must take the per-view strata (a trial that overflowed would be redone exactly and report 0; per-tile boundaries are
    only tried after that) and give the pixels of the exact path."""
    from pf3plat_b200._capi import GS_TUNE_NO_SPECULATION
    from pf3plat_b200.rasterizer import last_stats
    dev = _dev()
    cams, ins, hw = _many_view_batch(dev)
    stream = torch.cuda.Stream(dev)          # a context of its own: this shape has no history there
    with torch.cuda.stream(stream):
        states, outs = [], []
        for _ in range(3):
            out, _ = _run(_settings(cams, hw, with_depth=True), ins)
            st = last_stats(dev)
            states.append(st["speculative"])
            outs.append(out)
        ref, _ = _run(_settings(cams, hw, with_depth=True, tuning=GS_TUNE_NO_SPECULATION), ins)
        stream.synchronize()
    print(f"[regime] speculation on VPS=19: speculative per call {states}, stats of the third call {st}")
    assert states == [0, 2, 2], states
    for out in outs:
        for a, b in zip(out, ref):
            assert torch.equal(a, b)


def test_host_entry_beyond_one_sh_colour_chunk():
    """gs_render_host, 70 views of one scene (k_sh_colour stages 64 cameras at a time), pinned M = 25 SH block, per-view
    view_scale: the split pipeline (k_sh_colour on its own stream) and the fused preprocess give the device entry's bytes;
    the device entry matches the oracle on views either side of the 64-view boundary."""
    from pf3plat_b200 import _capi, rasterizer
    from pf3plat_b200.rasterizer import last_stats
    dev = _dev()
    V, P, hw = 70, 3000, (48, 48)
    sc = make_scene(P, V, *hw, seed=60)
    near = 1.0 / np.linspace(0.8, 1.25, V)
    cams, ins = scene_batch_args([sc], near=near)
    ins = {k: ins[k] for k in ("means3D", "opacities", "shs", "cov3D_precomp")}
    assert ins["shs"].shape[2] == 25
    dcams = {k: v.to(dev) for k, v in cams.items()}
    (c_dev, r_dev), _ = _run(_settings(dcams, hw), ins)
    ob = oracle_batch(_settings(cams, hw), **ins)
    print(f"[regime] host entry: VPS={V} (> 64 staged by k_sh_colour), M={ins['shs'].shape[2]}")
    assert V > 64
    for v in (0, 63, 64, 69):
        check_image_strict(c_dev[v], ob.views[v], 0.03, label=f"VPS=70 device entry view {v}")
    _check_radii(r_dev, ob, "VPS=70 device entry")

    host = {k: v.contiguous().float().pin_memory() for k, v in {**ins, **cams}.items()}
    cfg = _capi.GsConfig()
    cfg.P, cfg.S, cfg.V, cfg.M, cfg.sh_degree = P, 1, V, 25, 4
    cfg.image_height, cfg.image_width, cfg.scale_modifier = hw[0], hw[1], 1.0
    for k in ("viewmatrix", "projmatrix", "campos", "bg", "tanfov", "view_scale"):
        setattr(cfg, k, host[k].data_ptr())
    gin = _capi.GsInputs(means3D=host["means3D"].data_ptr(), opacities=host["opacities"].data_ptr(),
                         shs=host["shs"].data_ptr(), cov3D_precomp=host["cov3D_precomp"].data_ptr())
    color = torch.empty(V, 3, *hw).pin_memory()
    radii = torch.empty(V, P, dtype=torch.int32).pin_memory()
    gout = _capi.GsOutputs(color=color.data_ptr(), radii=radii.data_ptr(), depth=None)
    ctx = rasterizer.current_context(dev)
    launches = {}
    for tuning in (0, _capi.GS_TUNE_NO_SPLIT_COLOUR):
        cfg.tuning = tuning
        for _ in range(3):     # exact, strata trial, stratified
            color.zero_(); radii.zero_()
            _capi.check(_capi.lib().gs_render_host(ctx, ctypes.byref(cfg), ctypes.byref(gin), ctypes.byref(gout),
                                                   torch.cuda.current_stream(dev).cuda_stream))
            assert torch.equal(color, c_dev.cpu()) and torch.equal(radii, r_dev.cpu()), tuning
        launches[tuning] = last_stats(dev)["kernel_launches"]
    print(f"[regime] host entry kernel launches (split pipeline, fused): {launches[0]}, "
          f"{launches[_capi.GS_TUNE_NO_SPLIT_COLOUR]}")
    assert launches[0] == launches[_capi.GS_TUNE_NO_SPLIT_COLOUR] + 1     # k_sh_colour ran in the split pipeline


# ---------------------------------------------------------------------------------------------------------------------
# 2. the batched operator's inputs
# ---------------------------------------------------------------------------------------------------------------------
_NEAR4 = [1.25, 0.8, 1 / 1.7, 1 / 0.6]          # view_scale 0.8, 1.25, 1.7, 0.6


def _operator_inputs(colour, geometry, d_sh=25, P=2000, hw=(48, 64), mod=1.0):
    """S = 2 scenes x 2 views with per-view view_scale.  colour: "shs" | "colors" (per-view distinct colors_precomp);
    geometry: "cov3D" | "scalerot" (scales given so that mod * scales is the scene's scale; quaternions scaled to norms
    0.6 .. 1.5 -- the operator does not normalise them, so the covariance changes with the norm)."""
    scenes = [make_scene(P, 2, *hw, seed=80 + k, d_sh=d_sh) for k in range(2)]
    cams, ins = scene_batch_args(scenes, near=_NEAR4)
    out = {"means3D": ins["means3D"], "opacities": ins["opacities"]}
    if colour == "shs":
        out["shs"] = ins["shs"]
    else:
        g = torch.Generator().manual_seed(7)
        out["colors_precomp"] = torch.rand(4, P, 3, generator=g)
    if geometry == "cov3D":
        out["cov3D_precomp"] = ins["cov3D_precomp"]
    else:
        norm = torch.linspace(0.6, 1.5, 2 * P).reshape(2, P, 1)
        out["scales"] = (ins["scales"] / mod).contiguous()
        out["rotations"] = (ins["rotations"] * norm).contiguous()
    return cams, out, hw


@pytest.mark.parametrize("colour", ["shs", "colors"])
@pytest.mark.parametrize("geometry,mod", [("cov3D", 1.0), ("scalerot", 1.0), ("scalerot", 0.7)])
def test_operator_input_matrix_matches_oracle(colour, geometry, mod):
    dev = _dev()
    cams, ins, hw = _operator_inputs(colour, geometry, mod=mod)
    label = f"{colour}/{geometry}/mod={mod}"
    ob = oracle_batch(_settings(cams, hw, scale_modifier=mod), **ins)
    print(f"[regime] {label}: S={ob.S} V={ob.V} view_scale={[round(float(s), 3) for s in ob.s]} "
          f"visible per view {(ob.radii > 0).sum(axis=1).tolist()}")
    assert len(set(np.round(ob.s, 6).tolist())) == 4 and (np.abs(ob.s - 1) > 0.1).all()
    if "colors_precomp" in ins:
        assert not torch.equal(ins["colors_precomp"][0], ins["colors_precomp"][1])
    if "rotations" in ins:
        n = ins["rotations"].norm(dim=-1)
        assert float(n.min()) < 0.7 and float(n.max()) > 1.4
    dL, _ = _loss_grads(ob)
    gref = ob.backward(dL)
    dcams = {k: v.to(dev) for k, v in cams.items()}
    (color, radii), grads = _run(_settings(dcams, hw, scale_modifier=mod), ins, dL, means2D=True)
    _check_images(color, ob, label)
    _check_radii(radii, ob, label)
    assert set(grads) == {k for k in gref if gref[k] is not None}
    _check_grads(label, grads, gref, ob.affected(), ob.VPS)


@pytest.mark.parametrize("d_sh,sh_degree", [(16, 1), (25, 2)])
def test_sh_degree_below_coefficient_count(d_sh, sh_degree):
    """M = 16 evaluated to degree 1, M = 25 to degree 2: the bands that are never evaluated get exactly zero gradient."""
    dev = _dev()
    cams, ins, hw = _operator_inputs("shs", "cov3D", d_sh=d_sh)
    label = f"M={d_sh} sh_degree={sh_degree}"
    ob = oracle_batch(_settings(cams, hw, sh_degree=sh_degree), **ins)
    assert ob.views[0].M == d_sh
    dL, _ = _loss_grads(ob)
    gref = ob.backward(dL)
    dcams = {k: v.to(dev) for k, v in cams.items()}
    (color, radii), grads = _run(_settings(dcams, hw, sh_degree=sh_degree), ins, dL, means2D=True)
    _check_images(color, ob, label)
    _check_grads(label, grads, gref, ob.affected(), ob.VPS)
    used = (sh_degree + 1) ** 2
    unused = grads["shs"][:, :, used:]
    print(f"[regime] {label}: bands 0..{sh_degree} evaluated, max |dL/dsh| beyond coefficient {used}: "
          f"{float(unused.abs().max())}, within: {float(grads['shs'][:, :, :used].abs().max()):.3e}")
    assert float(unused.abs().max()) == 0.0
    assert float(grads["shs"][:, :, used - 1].abs().max()) > 0.0     # the last evaluated band does get gradient


# ---------------------------------------------------------------------------------------------------------------------
# 3.-5. geometry the synthetic distribution excludes
# ---------------------------------------------------------------------------------------------------------------------
def _single_scene(sc, hw, use_sh=True):
    cams, ins = scene_batch_args([sc])
    keep = ("means3D", "opacities", "cov3D_precomp") + (("shs",) if use_sh else ())
    return cams, {k: ins[k] for k in keep}


def _contributing(orc):
    """bool[P]: Gaussians with alpha >= 1/255 at some pixel of the image."""
    return affected_gaussians(orc, np.ones((orc.H, orc.W), bool))


def test_offscreen_centres_match_oracle():
    dev = _dev()
    hw, P, n_off = (48, 64), 1500, 400
    sc = offscreen_scene(P, n_off, 2, *hw, seed=90)
    cams, ins = _single_scene(sc, hw)
    ob = oracle_batch(_settings(cams, hw, with_depth=True), **ins)
    for v, r in enumerate(ob.views):
        # the clamp, recomputed in numpy from the camera: |t.x / t.z| or |t.y / t.z| beyond 1.3 tanfov
        view = np.asarray(cams["viewmatrix"][v], np.float64)
        m = np.asarray(ins["means3D"][0], np.float64)
        t = m @ view[:3, :3] + view[3, :3]
        tan = np.asarray(cams["tanfov"][v], np.float64)
        clamped = (np.abs(t[:, 0] / t[:, 2]) > 1.3 * tan[0]) | (np.abs(t[:, 1] / t[:, 2]) > 1.3 * tan[1])
        visible = r.radii > 0
        contrib = _contributing(r)
        n_vis, n_cl, n_cl_contrib = int(visible.sum()), int((clamped & visible).sum()), int((clamped & contrib).sum())
        print(f"[regime] off-screen view {v}: visible {n_vis}, clamped Jacobian {n_cl} ({n_cl / n_vis:.1%}), "
              f"of which contribute to a pixel {n_cl_contrib}")
        assert n_cl >= 0.01 * n_vis and n_cl_contrib >= 0.01 * n_vis
    dL, dLd = _loss_grads(ob)
    gref = ob.backward(dL, dLd)
    dcams = {k: v.to(dev) for k, v in cams.items()}
    (color, radii, depth), grads = _run(_settings(dcams, hw, with_depth=True), ins, dL, dLd, means2D=True)
    _check_images(color, ob, "off-screen", depth=depth)
    _check_radii(radii, ob, "off-screen")
    _check_grads("off-screen", grads, gref, ob.affected(), ob.VPS)


def test_near_plane_splats_match_oracle():
    from pf3plat_b200.rasterizer import GaussianRasterizationSettings, GaussianRasterizer
    dev = _dev()
    hw = (48, 64)
    sc = near_plane_scene(1500, 150, 60, 60, 2, *hw, seed=100)
    cams, ins = _single_scene(sc, hw)
    ob = oracle_batch(_settings(cams, hw, with_depth=True), **ins)
    z = ins["means3D"][0, :, 2].double().numpy()              # camera-space z in every view (cameras move in x, y)
    dcams = {k: v.to(dev) for k, v in cams.items()}
    for v, r in enumerate(ob.views):
        view = np.asarray(cams["viewmatrix"][v], np.float64)
        zc = np.asarray(ins["means3D"][0], np.float64) @ view[:3, 2] + view[3, 2]
        assert np.allclose(zc, z)
        visible = r.radii > 0
        n_cull = int(((z > 0) & (z < 0.2)).sum())
        n_near_vis = int((visible & (z < 1.5)).sum())
        print(f"[regime] near plane view {v}: culled 0<z<0.2 {n_cull}, behind {int((z <= 0).sum())}, visible z<1.5 "
              f"{n_near_vis} (closest {z[visible].min():.4f}), max radius {int(r.radii.max())} vs image {max(hw)}, "
              f"geom_fragile {int(r.geom_fragile.sum())}")
        assert n_cull > 0 and (z <= 0).any() and n_near_vis > 0 and z[visible].min() < 0.21
        assert not visible[z <= 0.2].any()
        assert r.radii.max() >= max(hw)
        # markVisible against the near-plane cull z > 0.2
        st = GaussianRasterizationSettings(
            image_height=hw[0], image_width=hw[1], tanfovx=float(cams["tanfov"][v, 0]), tanfovy=float(cams["tanfov"][v, 1]),
            bg=dcams["bg"][v], scale_modifier=1.0, viewmatrix=dcams["viewmatrix"][v], projmatrix=dcams["projmatrix"][v],
            sh_degree=4, campos=dcams["campos"][v], prefiltered=False, debug=False)
        present = GaussianRasterizer(st).markVisible(ins["means3D"][0].to(dev)).cpu().numpy().reshape(-1)
        assert np.array_equal(present, zc > 0.2)
    dL, dLd = _loss_grads(ob)
    gref = ob.backward(dL, dLd)
    (color, radii, depth), grads = _run(_settings(dcams, hw, with_depth=True), ins, dL, dLd, means2D=True)
    _check_images(color, ob, "near plane", max_fragile_frac=0.05, depth=depth)
    _check_radii(radii, ob, "near plane")
    _check_grads("near plane", grads, gref, ob.affected(), ob.VPS)


def _termination(orc):
    """Per pixel: whether it terminated early -- a Gaussian later in its tile list than n_contrib still reaches it
    (alpha >= 1/255), so the walk stopped because that Gaussian would have taken T below 1e-4 (final_T is the last
    transmittance above 1e-4, as upstream stores it) -- and the transmittance that Gaussian would have left.  Also, per
    Gaussian, the largest alpha it takes at a pixel centre before the 0.99 clamp."""
    H, W = orc.H, orc.W
    gx = (W + 15) // 16
    xy, co, pl, rg = orc.xy.astype(np.float64), orc.conic_opacity.astype(np.float64), orc.point_list, orc.ranges
    early = np.zeros((H, W), bool)
    t_next = np.full((H, W), np.nan)
    raw_alpha = np.zeros(orc.P)
    for t in range(rg.shape[0]):
        s, e = rg[t]
        ids = pl[s:e]
        if len(ids) == 0:
            continue
        ty, tx = divmod(t, gx)
        ys, xs = np.mgrid[ty * 16:min(H, ty * 16 + 16), tx * 16:min(W, tx * 16 + 16)]
        ys, xs = ys.reshape(-1), xs.reshape(-1)
        dx, dy = xy[ids, 0:1] - xs[None], xy[ids, 1:2] - ys[None]
        power = -0.5 * (co[ids, 0:1] * dx * dx + co[ids, 2:3] * dy * dy) - co[ids, 1:2] * dx * dy
        a = co[ids, 3:4] * np.exp(np.minimum(power, 0.0))
        np.maximum.at(raw_alpha, ids, np.where(power <= 0, a, 0.0).max(axis=1))
        reach = (power <= 0) & (a >= 1 / 255)
        later = np.arange(len(ids))[:, None] >= orc.n_contrib[ys, xs][None]
        hit = reach & later
        first = np.argmax(hit, axis=0)
        ok = hit.any(axis=0)
        early[ys[ok], xs[ok]] = True
        t_next[ys[ok], xs[ok]] = orc.final_T[ys[ok], xs[ok]] * (1 - np.minimum(0.99, a[first[ok], np.nonzero(ok)[0]]))
    return early, t_next, raw_alpha


def test_opaque_stacks_match_fp32_and_fp64_oracles():
    dev = _dev()
    hw = (48, 64)
    sc = opaque_stack_scene(6, 10, 2, *hw, seed=110)
    cams, ins = _single_scene(sc, hw)
    bs = _settings(cams, hw, with_depth=True)
    ob = oracle_batch(bs, **ins)
    ob64 = oracle_batch(bs, dtype=np.float64, **ins)
    for v, r in enumerate(ob.views):
        early, t_next, raw_alpha = _termination(r)
        n_clamp = int((raw_alpha >= 0.99).sum())
        print(f"[regime] opaque stacks view {v}: early-terminated pixels {early.mean():.1%} (T after the stopping "
              f"Gaussian <= {np.nanmax(t_next):.2e}; median n_contrib {int(np.median(r.n_contrib))}, median final_T "
              f"{np.median(r.final_T):.2e}); Gaussians whose alpha reaches the 0.99 clamp: {n_clamp} of {r.P}; "
              f"fragile pixels {r.px_fragile.mean():.2%}")
        assert early.mean() >= 0.3 and np.nanmax(t_next) < 1e-4 and n_clamp > 0
    dL, dLd = _loss_grads(ob)
    gref, gref64 = ob.backward(dL, dLd), ob64.backward(dL, dLd)
    dcams = {k: v.to(dev) for k, v in cams.items()}
    (color, radii, depth), grads = _run(_settings(dcams, hw, with_depth=True), ins, dL, dLd, means2D=True)
    _check_images(color, ob, "opaque fp32", depth=depth)
    _check_images(color, ob64, "opaque fp64")
    _check_radii(radii, ob, "opaque")
    # Every Gaussian is held to the strict 1e-3 rule, fragile pixels or not: what is under test is whether the backward
    # compositor's approximate rcp / ex2 (gs_composite_bwd.cu) stay within it where 1/(1 - alpha) is about 100 and T is
    # rebuilt through dozens of such divisions -- against fp32 arithmetic and against the exact (fp64) result.
    strict = np.zeros((ob.S, ob.P), bool)
    _check_grads("opaque vs fp32 oracle", grads, gref, strict, ob.VPS)
    _check_grads("opaque vs fp64 oracle", grads, gref64, strict, ob.VPS)
