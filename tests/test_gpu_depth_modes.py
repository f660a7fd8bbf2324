"""GPU tests of the fused depth channel in the modes other than "depth" (GsConfig.depth_mode): "disparity",
"relative_disparity" and "log" composite f(z) -- render_depth_cuda's fake colour at the unscaled camera-space depth -- in
the colour pass, with the gradients of the reference's construction.

The oracle is that construction in fp64 (tests/depth_modes_oracle.py): the batched CPU oracle renders colors_precomp = f(z)
on black, and its colour gradient, through f'(z) dz/dz_s, reaches the means and the z column of each view matrix.  Images
use the fragile-pixel rules of tests/util.py, Gaussian gradients the element-wise rule (check_grad), view-matrix gradients
tests/chain_oracle.camera_grad_check.  The loss is a colour term plus a signed per-pixel depth term.  Every test prints
"[regime]" lines and asserts its regime was reached."""
import ctypes

import numpy as np
import pytest
import torch

from pf3plat_b200 import _capi
from pf3plat_b200.synthetic import make_pixel_aligned_scene, make_scene, make_target
from tests.batch_oracle import scene_batch_args
from tests.chain_oracle import camera_grad_check
from tests.depth_modes_oracle import MODES, DepthModeOracle
from tests.regimes import edge_straddle_scene
from tests.test_gpu_backward_paths import PATH_RTOL, _agree, _stream_ctx
from tests.test_gpu_depth_chain import _depth_batch, _depth_field, _leaves, _turned
from tests.test_gpu_regimes import _settings
from tests.util import check_grad

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


@pytest.fixture(autouse=True, scope="module")
def _fresh_contexts():
    """Rasterizer contexts are cached per (device, stream), and torch hands out streams from a small pool: a "fresh"
    stream of a later test can be one of these tests' streams, with the binning history (learned capacities, overflow
    redo count) left there.  Start and end with no cached context."""
    import gc
    from pf3plat_b200.rasterizer import destroy_contexts
    torch.cuda.synchronize()
    destroy_contexts()
    yield
    gc.collect()
    torch.cuda.synchronize()
    destroy_contexts()


def _near_far(cams, far_ratio=100.0):
    """(V,2) unscaled near and far of the views: near = 1 / view_scale, as the camera glue made it."""
    near = 1.0 / cams["view_scale"].double()
    return torch.stack([near, far_ratio * near], -1).float()


def _incoming(V, hw, seed):
    rng = np.random.default_rng(seed)
    dL = rng.standard_normal((V, 3, *hw)) / (hw[0] * hw[1])
    return dL, _depth_field(V, hw, seed + 1)


def _bs(cams_dev, hw, mode, nf, tuning=0, viewmatrix=None, **kw):
    c = dict(cams_dev) if viewmatrix is None else {**cams_dev, "viewmatrix": viewmatrix}
    return _settings(c, hw, with_depth=True, tuning=tuning, **kw)._replace(depth_mode=mode, depth_near_far=nf)


def _gpu(cams_dev, hw, ins, mode, nf, dL, w, tuning=0, view_grad=True):
    """rasterize_batch in `mode` with Gaussians and (view_grad) the view matrix requiring grad; backward of
    <dL, colour> + <w, depth>.  Returns (view-matrix gradient, {input: grad}, outputs)."""
    from pf3plat_b200.rasterizer import rasterize_batch
    vm = cams_dev["viewmatrix"].clone().requires_grad_(view_grad)
    leaves = _leaves(ins, DEV)
    out = rasterize_batch(_bs(cams_dev, hw, mode, nf.to(DEV), tuning, viewmatrix=vm), **leaves)
    f32 = lambda a: torch.as_tensor(a, dtype=torch.float32, device=DEV)
    torch.autograd.backward([out[0], out[2]], [f32(dL), f32(w)])
    return vm.grad, {k: t.grad for k, t in leaves.items()}, [o.detach() for o in out]


def _check(label, orc, go, view_grad, grads, out):
    V, S, VPS = orc.V, orc.S, orc.VPS
    depth = out[2].cpu().double().numpy()
    dd = np.abs(depth - orc.depth)[~orc.frag]
    dmax = float(np.abs(orc.depth).max())
    print(f"[parity] {label}: depth max err (non-fragile) {dd.max():.2e} of max |depth| {dmax:.3f}; fragile pixels "
          f"{orc.frag.mean():.4f}")
    assert dd.max() <= 1e-4 * max(dmax, 1e-3), (label, dd.max(), dmax)
    aff = orc.affected()
    for k, g in grads.items():
        if k == "colors_precomp":
            for v in range(V):
                check_grad(f"{label} dL/dcolors view {v}", g[v], go[k][v], aff[v // VPS])
            continue
        for s in range(S):
            check_grad(f"{label} dL/d{k} scene {s}", g[s].reshape(g.shape[1], -1), go[k][s].reshape(g.shape[1], -1),
                       aff[s])
    assert view_grad is not None and view_grad.shape == (V, 4, 4)
    rest = view_grad.clone()
    rest[:, :, 2] = 0
    assert int(torch.count_nonzero(rest)) == 0, f"{label}: gradient outside the z column"
    if orc.mode == "log":
        # near < far: f = log(far) for every Gaussian, f' = 0 -- no z path, no camera gradient, exactly
        assert not np.any(go["z_path"]) and int(torch.count_nonzero(view_grad)) == 0, label
    else:
        camera_grad_check(f"{label} dL/dviewmatrix_z", view_grad[:, :, 2], go["view_z"], go["view_z_terms"],
                          orc.affected_views())


def _regime(label, orc, go):
    vis = (orc.ob_depth.radii > 0).sum(axis=1)
    zp = np.abs(go["z_path"])
    print(f"[regime] {label}: S={orc.S} VPS={orc.VPS} P={orc.P}, visible per view {vis.min()}..{vis.max()}, f(z) "
          f"{orc.f.min():.3f}..{orc.f.max():.3f}, |dL/dz_s| max {zp.max():.2e}, |dL/dopacity| max "
          f"{np.abs(go['opacities']).max():.2e}")
    assert vis.min() > 0 and np.abs(go["opacities"]).max() > 0
    if orc.mode != "log":
        assert zp.max() > 0 and (np.abs(go["view_z"]).max(axis=1) > 0).all()


def _case(label, cams, ins, hw, mode, seed, tunings=((0, "default"),), nf=None):
    nf = _near_far(cams) if nf is None else nf
    bs = _settings(cams, hw)._replace(depth_mode=mode, depth_near_far=nf)
    orc = DepthModeOracle(bs, ins, mode, nf)
    dL, w = _incoming(orc.V, hw, seed)
    go = orc.backward(dL, w)
    _regime(f"{label} {mode}", orc, go)
    dcams = {k: v.to(DEV) for k, v in cams.items()}
    outs = []
    for tuning, name in tunings:
        vg, grads, out = _gpu(dcams, hw, ins, mode, nf, dL, w, tuning=tuning)
        _check(f"{label} {mode} {name}", orc, go, vg, grads, out)
        outs.append((vg, grads, out))
    return orc, outs


# ---------------------------------------------------------------------------------------------------------------------
# 1. forward and gradients against the oracle under every backward kernel
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("geometry", ["cov3D", "scalerot"])
@pytest.mark.parametrize("mode", MODES)
def test_depth_mode_against_oracle_under_every_backward(mode, geometry):
    """S = 2 scenes x 9 views (camera chunks 8 + 1), view_scale 0.8 .. 1.25, turned cameras; the default backward, the
    round-1 compositor, the 4-CTA compositor, the two-phase preprocess backward."""
    cams, ins, hw = _depth_batch(geometry)
    tunings = ((0, "default"), (_capi.GS_TUNE_BWD_V1, "bwd v1"), (_capi.GS_TUNE_BWD_OCC4, "bwd occ4"),
               (_capi.GS_TUNE_PBWD_2PHASE, "2-phase preprocess bwd"))
    _, outs = _case(f"every backward, {geometry}", cams, ins, hw, mode, seed=61, tunings=tunings)
    for vg, grads, out in outs[1:]:
        for a, b in zip(out, outs[0][2]):
            assert torch.equal(a, b)
    # the colour image does not depend on the mode
    dcams = {k: v.to(DEV) for k, v in cams.items()}
    from pf3plat_b200.rasterizer import rasterize_batch
    plain = rasterize_batch(_settings(dcams, hw), **{k: v.to(DEV) for k, v in ins.items()})
    assert torch.equal(plain[0], outs[0][2][0]) and torch.equal(plain[1], outs[0][2][1])


def test_log_mode_trains_the_opacities_through_alpha_only():
    """A depth-only loss in "log": dL/dopacity is non-zero (the image is log(far) (1 - T_final)), the view matrices get
    an exact zero gradient, and the means' gradient is the alpha path alone (the oracle's, with no z term)."""
    cams, ins, hw = _depth_batch("cov3D")
    nf = _near_far(cams)
    bs = _settings(cams, hw)._replace(depth_mode="log", depth_near_far=nf)
    orc = DepthModeOracle(bs, ins, "log", nf)
    V = orc.V
    dL = np.zeros((V, 3, *hw))
    w = _depth_field(V, hw, 62)
    go = orc.backward(dL, w)
    vg, grads, out = _gpu({k: v.to(DEV) for k, v in cams.items()}, hw, ins, "log", nf, dL, w)
    far = nf[:, 1].double().numpy()
    print(f"[regime] log, depth-only loss: max |dL/dopacity| {float(grads['opacities'].abs().max()):.2e}; depth "
          f"{float(out[2].min()):.3f}..{float(out[2].max()):.3f} (log far {np.log(far).min():.3f})")
    assert float(grads["opacities"].abs().max()) > 0 and int(torch.count_nonzero(vg)) == 0
    assert float(out[2].max()) <= np.log(far).max() * (1 + 1e-6)
    _check("log depth-only", orc, go, vg, grads, out)


# ---------------------------------------------------------------------------------------------------------------------
# 2. every binning path: the same depth bits
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
def test_depth_mode_every_binning_path(mode):
    """2 scenes x 3 views on a context of its own, walked through every binning state; each call's depth image equals
    the exact path's bit for bit and its gradients meet the oracle."""
    from pf3plat_b200.rasterizer import last_stats
    c = _capi
    hw = (32, 48)
    scenes = [make_scene(2500, 3, *hw, seed=70 + k) for k in range(2)]
    cams, ins = scene_batch_args(scenes, near=1.0 / np.tile(np.linspace(0.8, 1.25, 3), 2))
    ins = {k: ins[k] for k in ("means3D", "opacities", "shs", "cov3D_precomp")}
    nf = _near_far(cams)
    orc = DepthModeOracle(_settings(cams, hw)._replace(depth_mode=mode, depth_near_far=nf), ins, mode, nf)
    dL, w = _incoming(orc.V, hw, 63)
    go = orc.backward(dL, w)
    dcams = {k: v.to(DEV) for k, v in cams.items()}
    sequence = [("exact", c.GS_TUNE_NO_SPECULATION, 0), ("per-view strata trial", 0, 2), ("stratified", 0, 2),
                ("stratified, k_emit_buckets", c.GS_TUNE_SEPARATE_EMIT, 2),
                ("exact, re-learn unstratified", c.GS_TUNE_NO_STRATA | c.GS_TUNE_NO_SPECULATION, 0),
                ("whole-tile", c.GS_TUNE_NO_STRATA, 1), ("radix fallback", c.GS_TUNE_FORCE_RADIX_BINNING, 0),
                ("warp-specialised compositor", c.GS_TUNE_FWD_WS | c.GS_TUNE_NO_SPECULATION, 0)]
    stream = _stream_ctx(DEV)
    states, first = [], None
    with torch.cuda.stream(stream):
        for label, tuning, want in sequence:
            vg, grads, out = _gpu(dcams, hw, ins, mode, nf, dL, w, tuning=tuning)
            st = last_stats(DEV)
            states.append(st["speculative"])
            assert st["speculative"] == want and st["overflow_redos"] == 0, (label, st)
            _check(f"binning {label} {mode}", orc, go, vg, grads, out)
            if first is None:
                first = out
            for a, b in zip(out, first):
                assert torch.equal(a, b), label
        stream.synchronize()
    print(f"[regime] {mode} binning paths: speculative per call {states}")


def _depth_only(bs, ins):
    from pf3plat_b200.rasterizer import rasterize_batch
    with torch.no_grad():
        return rasterize_batch(bs, **{k: v.to(DEV) for k, v in ins.items()})


@pytest.mark.parametrize("mode", MODES)
def test_depth_mode_per_tile_strata_and_overflow_redo(mode):
    """The pixel-aligned cloud (per-view strata trial overflows, then per-(view, tile) strata) and a sparse-then-dense
    sequence (speculative capacities overflow, exact redo): every call's depth equals the exact path's."""
    from pf3plat_b200.rasterizer import last_stats
    sc = make_pixel_aligned_scene(128, 128, 3, seed=2)
    hw = sc.image_shape
    cams, ins = scene_batch_args([sc])
    ins = {k: ins[k] for k in ("means3D", "opacities", "shs", "cov3D_precomp")}
    dcams = {k: v.to(DEV) for k, v in cams.items()}
    nf = _near_far(cams).to(DEV)
    ref = _depth_only(_bs(dcams, hw, mode, nf, _capi.GS_TUNE_NO_SPECULATION), ins)
    stream = _stream_ctx(DEV)
    states, redos = [], []
    with torch.cuda.stream(stream):
        for _ in range(5):
            out = _depth_only(_bs(dcams, hw, mode, nf), ins)
            st = last_stats(DEV)
            states.append(st["speculative"])
            redos.append(st["overflow_redos"])
            for a, b in zip(out, ref):
                assert torch.equal(a, b), (states, redos)
        stream.synchronize()
    print(f"[regime] {mode} per-tile strata: speculative per call {states}, overflow redos {redos}")
    assert states == [0, 0, 2, 2, 2] and redos == [0, 1, 1, 1, 1]

    hw = (48, 64)
    sparse = make_scene(3000, 2, *hw, seed=73)
    kw = dict(sparse.__dict__)
    kw["means"] = sparse.means * torch.tensor([0.63, 0.63, 1.0])
    dense = type(sparse)(**kw)
    cams, ins_s = scene_batch_args([sparse])
    _, ins_d = scene_batch_args([dense])
    keep = ("means3D", "opacities", "shs", "cov3D_precomp")
    ins_s, ins_d = ({k: i[k] for k in keep} for i in (ins_s, ins_d))
    dcams = {k: v.to(DEV) for k, v in cams.items()}
    nf = _near_far(cams).to(DEV)
    ref = _depth_only(_bs(dcams, hw, mode, nf, _capi.GS_TUNE_NO_SPECULATION), ins_d)
    stream = _stream_ctx(DEV)
    with torch.cuda.stream(stream):
        for _ in range(3):
            _depth_only(_bs(dcams, hw, mode, nf), ins_s)
        before = last_stats(DEV)
        out = _depth_only(_bs(dcams, hw, mode, nf), ins_d)
        after = last_stats(DEV)
        stream.synchronize()
    print(f"[regime] {mode} overflow: redos {before['overflow_redos']} -> {after['overflow_redos']}")
    assert after["overflow_redos"] == before["overflow_redos"] + 1 and after["speculative"] == 0
    for a, b in zip(out, ref):
        assert torch.equal(a, b)


# ---------------------------------------------------------------------------------------------------------------------
# 3. deterministic backward, SH degree 4, the host entry
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
def test_depth_mode_deterministic_backward(mode):
    cams, ins, hw = _depth_batch("cov3D")
    nf = _near_far(cams)
    dcams = {k: v.to(DEV) for k, v in cams.items()}
    dL, w = _incoming(cams["viewmatrix"].shape[0], hw, 64)
    plain = _gpu(dcams, hw, ins, mode, nf, dL, w)
    torch.use_deterministic_algorithms(True)
    try:
        runs = [_gpu(dcams, hw, ins, mode, nf, dL, w) for _ in range(2)]
    finally:
        torch.use_deterministic_algorithms(False)
    assert torch.equal(runs[0][0], runs[1][0])
    for k in runs[0][1]:
        assert torch.equal(runs[0][1][k], runs[1][1][k]), k
    worst = _agree(f"{mode} deterministic vs default", runs[0][1], plain[1])
    scale = float(plain[0].abs().max())
    err = float((runs[0][0] - plain[0]).abs().max())
    print(f"[regime] {mode} deterministic: two runs bit-identical; vs default {worst:.2e} (Gaussians), view-matrix "
          f"{err:.2e} of {scale:.2e}")
    assert err <= 1e-4 * scale + 1e-30


@pytest.mark.parametrize("mode", MODES)
def test_depth_mode_at_sh_degree4(mode):
    """Degree 4 (the B4 kernels): the depth image and the depth-only gradients are those of degree 3."""
    from tests.sh4_oracle import with_band4
    sc = with_band4(make_scene(4000, 3, 48, 64, seed=11))
    hw = sc.image_shape
    cams, ins = scene_batch_args([sc])
    ins = {k: ins[k] for k in ("means3D", "opacities", "shs", "cov3D_precomp")}
    nf = _near_far(cams)
    dcams = {k: v.to(DEV) for k, v in cams.items()}
    from pf3plat_b200.rasterizer import rasterize_batch
    res = {}
    for deg in (3, 4):
        vm = dcams["viewmatrix"].clone().requires_grad_(True)
        leaves = _leaves(ins, DEV)
        bs = _bs(dcams, hw, mode, nf.to(DEV), viewmatrix=vm)._replace(sh_eval_max_degree=deg)
        out = rasterize_batch(bs, **leaves)
        out[2].backward(torch.as_tensor(_depth_field(3, hw, 65), dtype=torch.float32, device=DEV))
        res[deg] = (out[0].detach(), out[2].detach(), vm.grad, {k: t.grad for k, t in leaves.items()})
    assert (res[4][0] - res[3][0]).abs().max() > 1e-3            # band 4 changes the colour ...
    assert torch.equal(res[4][1], res[3][1])                      # ... not the depth
    grads3 = {k: v for k, v in res[3][3].items() if k != "shs"}
    worst = _agree(f"{mode} degree 4 vs 3, depth-only gradients", {k: res[4][3][k] for k in grads3}, grads3)
    assert float(res[4][3]["shs"].abs().max()) == 0.0
    scale = float(res[3][2].abs().max())
    assert float((res[4][2] - res[3][2]).abs().max()) <= PATH_RTOL * scale
    print(f"[regime] {mode} degree 4: depth bit-identical to degree 3, gradients within {worst:.2e}")


@pytest.mark.parametrize("mode", MODES)
def test_depth_mode_host_entry_matches_device_entry(mode):
    """Every feed of gs_render_host (pageable upload; pinned zero-copy with the split colour pipeline, with the fused
    preprocess, and without zero copy) returns the device entry's colour, radii and depth bytes."""
    from pf3plat_b200 import rasterizer
    P, V, hw = 20000, 3, (64, 80)
    sc = make_scene(P, V, *hw, seed=12)
    cams, ins = scene_batch_args([sc])
    ins = {k: ins[k] for k in ("means3D", "opacities", "shs", "cov3D_precomp")}
    nf = _near_far(cams)
    dcams = {k: v.to(DEV) for k, v in cams.items()}
    c_dev, r_dev, d_dev = _depth_only(_bs(dcams, hw, mode, nf.to(DEV)), ins)
    host = {k: v[0].contiguous() for k, v in ins.items()}
    M = host["shs"].shape[1]
    cfg = _capi.GsConfig()
    cfg.P, cfg.S, cfg.V, cfg.M, cfg.sh_degree = P, 1, V, M, 4
    cfg.image_height, cfg.image_width, cfg.scale_modifier = hw[0], hw[1], 1.0
    cfg.flags, cfg.depth_mode = _capi.GS_FLAG_DEPTH, _capi.DEPTH_MODES[mode]
    hc = {k: v.contiguous() for k, v in cams.items()}
    for k, t in hc.items():
        setattr(cfg, k, t.data_ptr())
    nf_h = nf.contiguous()
    cfg.depth_near_far = nf_h.data_ptr()
    ctx = rasterizer.current_context(DEV)
    color = torch.empty(V, 3, *hw).pin_memory()
    radii = torch.empty(V, P, dtype=torch.int32).pin_memory()
    depth = torch.empty(V, *hw).pin_memory()
    gout = _capi.GsOutputs(color=color.data_ptr(), radii=radii.data_ptr(), depth=depth.data_ptr())
    pin = {k: v.pin_memory() for k, v in host.items()}
    runs = 0
    for src in (host, pin):
        gin = _capi.GsInputs(means3D=src["means3D"].data_ptr(), opacities=src["opacities"].data_ptr(),
                             shs=src["shs"].data_ptr(), cov3D_precomp=src["cov3D_precomp"].data_ptr())
        for tuning in ((0,) if src is host else (0, _capi.GS_TUNE_NO_SPLIT_COLOUR, _capi.GS_TUNE_NO_ZERO_COPY)):
            cfg.tuning = tuning
            color.zero_(); radii.zero_(); depth.zero_()
            _capi.check(_capi.lib().gs_render_host(ctx, ctypes.byref(cfg), ctypes.byref(gin), ctypes.byref(gout),
                                                   torch.cuda.current_stream(DEV).cuda_stream))
            assert torch.equal(color, c_dev.cpu()) and torch.equal(radii, r_dev.cpu()), tuning
            assert torch.equal(depth, d_dev.cpu()), tuning
            runs += 1
    print(f"[regime] {mode} host entry: M = {M}, {runs} feeds bit-identical to the device entry")
    assert M > 16 and runs == 4


# ---------------------------------------------------------------------------------------------------------------------
# 4. regimes: near plane, views per scene, ragged frame
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
def test_depth_mode_splats_near_the_near_plane(mode):
    """The cloud shrunk to 1/20 of its size (depths 0.075 .. 1) with near 0.05: splats down to 1.5 near from the camera,
    disparities up to ~13."""
    hw = (32, 48)
    sc = make_scene(1500, 3, *hw, seed=520)
    kw = dict(sc.__dict__)
    kw["means"] = sc.means * 0.05
    kw["covariances"] = sc.covariances * 0.0025
    kw["extrinsics"] = sc.extrinsics.clone()
    kw["extrinsics"][:, :3, 3] *= 0.05
    sc = type(sc)(**kw)
    cams, ins = scene_batch_args([sc], near=np.full(3, 0.05))
    ins = {k: ins[k] for k in ("means3D", "opacities", "shs", "cov3D_precomp")}
    orc, _ = _case("near plane", cams, ins, hw, mode, seed=66)
    vis = orc.ob_depth.radii > 0
    zmin = float(orc.z[vis].min())
    print(f"[regime] near plane {mode}: nearest visible splat at z = {zmin:.4f} (near 0.05), disparity up to "
          f"{1 / zmin:.1f}")
    assert 1 / zmin > 5


@pytest.mark.parametrize("vps", [1, 3, 9, 19])
@pytest.mark.parametrize("mode", MODES)
def test_depth_mode_views_per_scene(mode, vps):
    hw = (32, 48)
    scenes = [_turned(make_scene(1200, vps, *hw, seed=400 + 10 * vps + k), seed=450 + k) for k in range(2)]
    cams, ins = scene_batch_args(scenes, near=1.0 / np.tile(np.linspace(0.8, 1.25, vps), 2))
    ins = {k: ins[k] for k in ("means3D", "opacities", "shs", "cov3D_precomp")}
    _case(f"{vps} views per scene", cams, ins, hw, mode, seed=67 + vps)


@pytest.mark.parametrize("mode", MODES)
def test_depth_mode_ragged_frame(mode):
    hw = (33, 250)
    sc = _turned(edge_straddle_scene(600, 120, 2, *hw, seed=77), seed=78)
    cams, ins = scene_batch_args([sc])
    ins = {k: ins[k] for k in ("means3D", "opacities", "shs", "cov3D_precomp")}
    _case("33 x 250 frame", cams, ins, hw, mode, seed=68)


# ---------------------------------------------------------------------------------------------------------------------
# 5. decoder_forward(depth_mode=m) on predicted poses: one render, the two-pass route's results
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
def test_decoder_forward_depth_mode_is_one_render_and_matches_the_two_pass_route(mode, monkeypatch):
    from pf3plat_b200 import render
    from pf3plat_b200.rasterizer import last_stats
    b, v, P, hw = 2, 3, 1500, (48, 64)
    scs = [_turned(make_scene(P, v, *hw, seed=700 + k), seed=710 + k) for k in range(b)]
    st = lambda name: torch.stack([getattr(s, name) for s in scs]).to(DEV)
    ext, intr = st("extrinsics"), st("intrinsics")
    nr, fr = torch.full((b, v), 0.5, device=DEV), torch.full((b, v), 50.0, device=DEV)
    bg = torch.tensor([0.3, 0.2, 0.1], device=DEV)
    names = ("means", "covariances", "harmonics", "opacities")
    V = b * v
    dL = torch.as_tensor(make_target(V, *hw, seed=8).numpy() - 0.5, device=DEV).reshape(b, v, 3, *hw) / V
    w = torch.as_tensor(_depth_field(V, hw, seed=69), dtype=torch.float32, device=DEV).reshape(b, v, *hw)
    flat = lambda t: t.reshape(V, *t.shape[2:])

    def run(route):
        e = ext.clone().requires_grad_(True)
        L = [st(n).clone().requires_grad_(True) for n in names]
        if route == "fused":
            # on a context of its own (a fresh shape history), so that its launch count can be compared below
            calls = []
            inner = render.rasterize_batch
            monkeypatch.setattr(render, "rasterize_batch",
                                lambda bs, *a, **k: calls.append(bs.depth_mode) or inner(bs, *a, **k))
            stream = _stream_ctx(DEV)
            stream.wait_stream(torch.cuda.current_stream(DEV))
            with torch.cuda.stream(stream):
                color, depth = render.decoder_forward(*L, e, intr, nr, fr, hw, bg, depth_mode=mode)
                launches = last_stats(DEV)["kernel_launches"]
                torch.autograd.backward([color, depth], [dL, w])
            torch.cuda.current_stream(DEV).wait_stream(stream)
            monkeypatch.undo()
            assert calls == [mode], calls
        else:
            launches = None
            color = render.render_views(flat(e), flat(intr), flat(nr), flat(fr), hw, bg.reshape(1, 3).expand(V, 3), *L)
            color = color.reshape(b, v, 3, *hw)
            depth = render.render_depth(L[0], L[1], L[3], e, intr, nr, fr, hw, mode)
            torch.autograd.backward([color, depth], [dL, w])
        return color.detach(), depth.detach(), e.grad, [t.grad for t in L], launches

    new, old = run("fused"), run("two-pass")
    # one forward's launches: those of a colour-only call of the same shape on a fresh context
    stream = _stream_ctx(DEV)
    stream.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(stream):
        plain, none = render.decoder_forward(*[st(n) for n in names], ext, intr, nr, fr, hw, bg, depth_mode=None)
        launches_plain = last_stats(DEV)["kernel_launches"]
    torch.cuda.current_stream(DEV).wait_stream(stream)
    assert none is None and torch.equal(plain, new[0]) and torch.equal(new[0], old[0])
    assert new[4] == launches_plain, (new[4], launches_plain)
    dmax = float(old[1].abs().max())
    derr = float((new[1] - old[1]).abs().max())
    print(f"[regime] decoder {mode}: one operator call of {V} views ({new[4]} kernel launches, as a colour-only call); "
          f"colour bit-identical; max |depth fused - two-pass| {derr:.2e} of {dmax:.3f}")
    assert derr <= 1e-4 * max(dmax, 1e-3)
    for k, n in enumerate(names):
        scale = float(old[3][k].abs().max())
        err = float((new[3][k] - old[3][k]).abs().max())
        print(f"[regime] decoder {mode} dL/d{n}: max |fused - two-pass| {err:.2e} of {scale:.2e}")
        assert scale > 0 and err <= 1e-3 * scale, (n, err, scale)
    assert new[2] is not None and old[2] is not None
    if mode == "log":
        assert int(torch.count_nonzero(new[2])) == 0 and int(torch.count_nonzero(old[2])) == 0
    else:
        a, r = new[2].double(), old[2].double()
        rms = float(r.pow(2).mean().sqrt())
        ratio = float(((a - r).abs() / (r.abs() + rms)).max())
        print(f"[regime] decoder {mode} dL/dextrinsics: rms {rms:.3e}, worst |fused - two-pass| / (|two-pass| + rms) "
              f"{ratio:.2e}")
        assert rms > 0 and ratio <= 1e-3, ratio


def test_backward_needs_near_far_for_the_modes_that_read_it():
    """gs_backward of a "relative_disparity" forward refuses a call without depth_near_far."""
    from pf3plat_b200.rasterizer import _context, _make_config, rasterize_batch
    hw = (16, 16)
    cams, ins = scene_batch_args([make_scene(200, 1, *hw, seed=630)])
    dcams = {k: v.to(DEV) for k, v in cams.items()}
    leaves = _leaves({k: ins[k] for k in ("means3D", "opacities", "shs", "cov3D_precomp")}, DEV)
    bs = _bs(dcams, hw, "relative_disparity", _near_far(cams).to(DEV))
    color, _, depth = rasterize_batch(bs, **leaves)
    node = color.grad_fn
    keep = []
    S, P, V, M, H, W = node.dims
    cfg = _make_config(bs._replace(depth_near_far=None), S, P, M, keep)
    gin = _capi.GsInputs(**{k: None if t is None else t.data_ptr() for k, t in node.ins.items()})
    dcol = torch.zeros(V, 3, H, W, device=DEV)
    out = torch.empty(S * P * M * 3 + S * P * 10, device=DEV)
    ig = _capi.GsInGrads(dL_dmeans3D=out.data_ptr())
    og = _capi.GsOutGrads(dcol.data_ptr(), dcol.data_ptr())
    stream = torch.cuda.current_stream(DEV).cuda_stream
    rc = _capi.lib().gs_backward(_context(DEV, stream), ctypes.byref(cfg), ctypes.byref(gin), node.handle.ptr,
                                 ctypes.byref(og), ctypes.byref(ig), stream)
    assert rc == -1 and b"depth_near_far" in _capi.lib().gs_last_error()
