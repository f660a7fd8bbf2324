"""GPU tests of the accumulated opacity (BatchSettings.with_alpha, gs_forward_ex / gs_backward_ex / gs_render_host_ex):
alpha = 1 - T_final of the colour pass, and its gradient through the background term of every dL/dalpha_i.

The oracle is tests/alpha_oracle.py: the fp64 batched oracle rendering colours 1 on black, its backward with dL/dC =
(dL/dalpha, 0, 0), added to the colour (and depth) render's backward.  Images use the fragile-pixel rules of tests/util.py,
gradients the element-wise rule (check_grad).  Every test prints "[regime]" lines and asserts its regime was reached."""
import ctypes

import numpy as np
import pytest
import torch

from pf3plat_b200 import _capi
from pf3plat_b200.synthetic import make_pixel_aligned_scene, make_scene, make_target
from tests.alpha_oracle import AlphaOracle
from tests.batch_oracle import oracle_batch, scene_batch_args
from tests.regimes import edge_straddle_scene, long_list_scene, near_plane_scene, offscreen_scene, opaque_stack_scene
from tests.test_gpu_backward_paths import _agree, _stream_ctx
from tests.test_gpu_depth_chain import _depth_batch, _depth_field, _leaves, _turned
from tests.test_gpu_regimes import _settings
from tests.util import FRAGILE_RGB_TOL, RGB_TOL, check_grad

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
KEEP = ("means3D", "opacities", "shs", "cov3D_precomp")


@pytest.fixture(autouse=True, scope="module")
def _fresh_contexts():
    """Contexts are cached per (device, stream) and torch reuses streams: start and end with none cached."""
    import gc
    from pf3plat_b200.rasterizer import destroy_contexts
    torch.cuda.synchronize()
    destroy_contexts()
    yield
    gc.collect()
    torch.cuda.synchronize()
    destroy_contexts()


class _Det:
    def __enter__(self):
        torch.use_deterministic_algorithms(True)

    def __exit__(self, *exc):
        torch.use_deterministic_algorithms(False)


def _f32(a):
    return torch.as_tensor(np.asarray(a), dtype=torch.float32, device=DEV)


def _gpu(bs, ins, dA=None, dL=None, w=None, view_grad=False):
    """rasterize_batch with bs (device cameras); backward of <dA, alpha> + <dL, colour> + <w, depth> (None: left out of
    the loss).  Returns ({input: grad}, outputs, view-matrix grad)."""
    from pf3plat_b200.rasterizer import rasterize_batch
    vm = bs.viewmatrix.clone().requires_grad_(view_grad)
    leaves = _leaves(ins, DEV)
    out = rasterize_batch(bs._replace(viewmatrix=vm), **leaves)
    names = ["color", "radii"] + (["depth"] if bs.with_depth else []) + (["alpha"] if bs.with_alpha else [])
    o = dict(zip(names, out))
    ts, gs = [], []
    for key, g in (("alpha", dA), ("color", dL), ("depth", w)):
        if g is not None:
            ts.append(o[key])
            gs.append(_f32(g))
    if ts:
        torch.autograd.backward(ts, gs)
    return {k: t.grad for k, t in leaves.items()}, {k: v.detach() for k, v in o.items()}, vm.grad


def _check_alpha(label, alpha, orc, max_fragile=0.02):
    a = alpha.cpu().double().numpy()
    err = np.abs(a - orc.alpha)
    frag = orc.frag
    worst = float(err[~frag].max()) if (~frag).any() else 0.0
    print(f"[parity] {label}: alpha max err non-fragile {worst:.2e}, fragile {float(err[frag].max()) if frag.any() else 0:.2e}"
          f" ({frag.mean():.4f} of pixels); alpha {orc.alpha.min():.3f}..{orc.alpha.max():.3f}")
    assert frag.mean() <= max_fragile and worst <= RGB_TOL
    assert not frag.any() or float(err[frag].max()) <= FRAGILE_RGB_TOL
    empty = orc.final_T == 1.0
    assert torch.all(alpha.cpu()[torch.as_tensor(empty)] == 0.0)   # no contributor: exactly 0


def _check_grads(label, grads, go, aff, VPS):
    for k, g in grads.items():
        if k == "colors_precomp":
            for v in range(g.shape[0]):
                check_grad(f"{label} dL/dcolors view {v}", g[v], go[k][v], aff[v // VPS])
        elif k == "shs" and go.get(k) is None:
            continue
        else:
            for s in range(g.shape[0]):
                check_grad(f"{label} dL/d{k} scene {s}", g[s].reshape(g.shape[1], -1), go[k][s].reshape(g.shape[1], -1),
                           aff[s])


def _two_pass_alpha(bs, ins):
    """The route without the feature: a second render of the same Gaussians, colours 1 on black; its channel 0."""
    from pf3plat_b200.rasterizer import rasterize_batch
    V = bs.viewmatrix.shape[0]
    P = ins["means3D"].shape[1]
    geo = {k: v.to(DEV) for k, v in ins.items() if k not in ("shs", "colors_precomp")}
    with torch.no_grad():
        out = rasterize_batch(bs._replace(bg=torch.zeros(V, 3, device=DEV), with_depth=False, with_alpha=False),
                              colors_precomp=torch.ones(V, P, 3, device=DEV), **geo)
    return out[0][:, 0]


# ---------------------------------------------------------------------------------------------------------------------
# 1. against the oracles, under every compositor
# ---------------------------------------------------------------------------------------------------------------------
TUNINGS = ((0, "default"), (_capi.GS_TUNE_BWD_V1, "bwd v1"), (_capi.GS_TUNE_BWD_OCC4, "bwd occ4"),
           (_capi.GS_TUNE_FWD_WS, "warp-specialised fwd"), (_capi.GS_TUNE_PBWD_2PHASE, "2-phase preprocess bwd"))


@pytest.mark.parametrize("geometry", ["cov3D", "scalerot"])
def test_alpha_against_oracle_under_every_compositor(geometry):
    """S = 2 scenes x 9 views, view_scale 0.8 .. 1.25, turned cameras.  An alpha-only loss and alpha + colour MSE +
    depth, under both forward compositors and every backward compositor; colour, depth and radii are those of a call
    without alpha, bit for bit; alpha is the two-pass route's within 1e-4."""
    cams, ins, hw = _depth_batch(geometry)
    V, S = cams["viewmatrix"].shape[0], 2
    bs_cpu = _settings(cams, hw, with_depth=True)
    orc = AlphaOracle(bs_cpu, ins, base=oracle_batch(bs_cpu, dtype=np.float64, **ins))
    rng = np.random.default_rng(71)
    dA = rng.standard_normal((V, *hw)) / (hw[0] * hw[1])
    target = make_target(V, *hw, seed=3).numpy()
    dL = 2 * (orc.color - target) / target.size
    w = _depth_field(V, hw, 72)
    go_a = orc.backward(dA)
    go_all = orc.backward(dA, dL, w)
    aff = orc.affected()
    print(f"[regime] {geometry}: V={V}, covered pixels {(orc.alpha > 0).mean():.3f}, |dL/dopacity| of the alpha-only loss "
          f"max {np.abs(go_a['opacities']).max():.2e}")
    assert np.abs(go_a["opacities"]).max() > 0 and (orc.alpha > 0).mean() > 0.5 and (orc.alpha < 0.99).any()
    dcams = {k: v.to(DEV) for k, v in cams.items()}
    plain_g, plain, _ = _gpu(_settings(dcams, hw, with_depth=True), ins, dL=dL, w=w)
    for tuning, name in TUNINGS:
        bs = _settings(dcams, hw, with_depth=True, tuning=tuning)._replace(with_alpha=True)
        grads, out, _ = _gpu(bs, ins, dA=dA)
        _check_alpha(f"{geometry} {name}", out["alpha"], orc)
        for k in ("color", "radii", "depth"):
            assert torch.equal(out[k], plain[k]), (name, k)
        if geometry == "cov3D":
            assert float(grads["shs"].abs().max()) == 0.0
        else:
            assert float(grads["colors_precomp"].abs().max()) == 0.0
        _check_grads(f"{geometry} {name} alpha-only", {k: g for k, g in grads.items() if k not in ("shs", "colors_precomp")},
                     go_a, aff, V // S)
        grads, out, _ = _gpu(bs, ins, dA=dA, dL=dL, w=w)
        _check_grads(f"{geometry} {name} alpha + colour + depth", grads, go_all, aff, V // S)
        if tuning == 0:
            two = _two_pass_alpha(bs, ins)
            diff = float((two - out["alpha"]).abs().max())
            print(f"[parity] {geometry}: max |fused alpha - two-pass alpha| {diff:.2e}")
            assert diff <= 1e-4


# ---------------------------------------------------------------------------------------------------------------------
# 2. binning paths: the same bits
# ---------------------------------------------------------------------------------------------------------------------
def test_alpha_every_binning_path():
    """2 scenes x 3 views on a context of its own, walked through every binning state: alpha and the deterministic
    gradients of alpha + colour are the exact path's bit for bit."""
    from pf3plat_b200.rasterizer import last_stats
    c = _capi
    hw = (32, 48)
    scenes = [make_scene(2500, 3, *hw, seed=80 + k) for k in range(2)]
    cams, ins = scene_batch_args(scenes, near=1.0 / np.tile(np.linspace(0.8, 1.25, 3), 2))
    ins = {k: ins[k] for k in KEEP}
    dcams = {k: v.to(DEV) for k, v in cams.items()}
    V = 6
    rng = np.random.default_rng(81)
    dA, dL = rng.standard_normal((V, *hw)) / 1536, rng.standard_normal((V, 3, *hw)) / 1536
    sequence = [("exact", c.GS_TUNE_NO_SPECULATION, 0), ("per-view strata trial", 0, 2), ("stratified", 0, 2),
                ("stratified, k_emit_buckets", c.GS_TUNE_SEPARATE_EMIT, 2),
                ("exact, re-learn unstratified", c.GS_TUNE_NO_STRATA | c.GS_TUNE_NO_SPECULATION, 0),
                ("whole-tile", c.GS_TUNE_NO_STRATA, 1), ("radix fallback", c.GS_TUNE_FORCE_RADIX_BINNING, 0)]
    stream = _stream_ctx(DEV)
    states, first = [], None
    with torch.cuda.stream(stream), _Det():
        for label, tuning, want in sequence:
            bs = _settings(dcams, hw, tuning=tuning)._replace(with_alpha=True)
            grads, out, _ = _gpu(bs, ins, dA=dA, dL=dL)
            st = last_stats(DEV)
            states.append(st["speculative"])
            assert st["speculative"] == want and st["overflow_redos"] == 0, (label, st)
            if first is None:
                first = (grads, out)
            assert torch.equal(out["alpha"], first[1]["alpha"]), label
            for k in grads:
                assert torch.equal(grads[k], first[0][k]), (label, k)
        stream.synchronize()
    print(f"[regime] alpha binning paths: speculative per call {states}")


def test_alpha_per_tile_strata_and_overflow_redo():
    """The pixel-aligned cloud (per-view strata trial overflows, then per-(view, tile) strata) and a sparse-then-dense
    sequence (speculative capacities overflow, exact redo): alpha and the deterministic gradients equal the exact path's."""
    from pf3plat_b200.rasterizer import last_stats
    sc = make_pixel_aligned_scene(128, 128, 3, seed=2)
    hw = sc.image_shape
    cams, ins = scene_batch_args([sc])
    ins = {k: ins[k] for k in KEEP}
    dcams = {k: v.to(DEV) for k, v in cams.items()}
    dA = np.random.default_rng(82).standard_normal((3, *hw)) / (hw[0] * hw[1])
    bs = lambda tuning=0: _settings(dcams, hw, tuning=tuning)._replace(with_alpha=True)
    with _Det():
        ref_g, ref, _ = _gpu(bs(_capi.GS_TUNE_NO_SPECULATION), ins, dA=dA)
        stream = _stream_ctx(DEV)
        states, redos = [], []
        with torch.cuda.stream(stream):
            for _ in range(5):
                grads, out, _ = _gpu(bs(), ins, dA=dA)
                st = last_stats(DEV)
                states.append(st["speculative"])
                redos.append(st["overflow_redos"])
                assert torch.equal(out["alpha"], ref["alpha"]), states
                for k in grads:
                    assert torch.equal(grads[k], ref_g[k]), (states, k)
            stream.synchronize()
    print(f"[regime] alpha per-tile strata: speculative per call {states}, overflow redos {redos}")
    assert states == [0, 0, 2, 2, 2] and redos == [0, 1, 1, 1, 1]

    hw = (48, 64)
    sparse = make_scene(3000, 2, *hw, seed=83)
    kw = dict(sparse.__dict__)
    kw["means"] = sparse.means * torch.tensor([0.63, 0.63, 1.0])
    dense = type(sparse)(**kw)
    cams, ins_s = scene_batch_args([sparse])
    _, ins_d = scene_batch_args([dense])
    ins_s, ins_d = ({k: i[k] for k in KEEP} for i in (ins_s, ins_d))
    dcams = {k: v.to(DEV) for k, v in cams.items()}
    bs = lambda tuning=0: _settings(dcams, hw, tuning=tuning)._replace(with_alpha=True)
    ref = _gpu(bs(_capi.GS_TUNE_NO_SPECULATION), ins_d)[1]
    stream = _stream_ctx(DEV)
    with torch.cuda.stream(stream):
        for _ in range(3):
            _gpu(bs(), ins_s)
        before = last_stats(DEV)
        out = _gpu(bs(), ins_d)[1]
        after = last_stats(DEV)
        stream.synchronize()
    print(f"[regime] alpha overflow: redos {before['overflow_redos']} -> {after['overflow_redos']}")
    assert after["overflow_redos"] == before["overflow_redos"] + 1 and after["speculative"] == 0
    for k in ("color", "radii", "alpha"):
        assert torch.equal(out[k], ref[k]), k


# ---------------------------------------------------------------------------------------------------------------------
# 3. no leakage into SH, colours or cameras; an alpha that is requested but unused
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("geometry", ["cov3D", "scalerot"])
def test_alpha_gives_sh_colours_and_cameras_nothing(geometry):
    """Deterministic mode: the SH or colour gradient, and the view-matrix gradient of a depth term, are torch.equal with
    and without an added alpha term; the geometry gradients do change."""
    cams, ins, hw = _depth_batch(geometry)
    V = cams["viewmatrix"].shape[0]
    dcams = {k: v.to(DEV) for k, v in cams.items()}
    rng = np.random.default_rng(73)
    dA, dL = rng.standard_normal((V, *hw)) / 1536, rng.standard_normal((V, 3, *hw)) / 1536
    w = _depth_field(V, hw, 74)
    bs = _settings(dcams, hw, with_depth=True)._replace(with_alpha=True)
    with _Det():
        g0, _, v0 = _gpu(bs, ins, dL=dL, w=w, view_grad=True)
        g1, _, v1 = _gpu(bs, ins, dA=dA, dL=dL, w=w, view_grad=True)
    key = "shs" if geometry == "cov3D" else "colors_precomp"
    assert torch.equal(g0[key], g1[key]) and float(g0[key].abs().max()) > 0
    assert v0 is not None and torch.equal(v0, v1) and float(v0.abs().max()) > 0
    assert not torch.equal(g0["opacities"], g1["opacities"]) and not torch.equal(g0["means3D"], g1["means3D"])
    print(f"[regime] {geometry}: {key} and view-matrix gradients bit-identical with and without dL/dalpha")


@pytest.mark.parametrize("tuning", [0, _capi.GS_TUNE_BWD_OCC4])
def test_requested_but_unused_alpha_changes_no_gradient(tuning):
    cams, ins, hw = _depth_batch("cov3D")
    V = cams["viewmatrix"].shape[0]
    dcams = {k: v.to(DEV) for k, v in cams.items()}
    dL = np.random.default_rng(75).standard_normal((V, 3, *hw)) / 1536
    bs = _settings(dcams, hw, tuning=tuning)
    with _Det():
        g0, o0, _ = _gpu(bs, ins, dL=dL)
        g1, o1, _ = _gpu(bs._replace(with_alpha=True), ins, dL=dL)
    assert o1["alpha"] is not None and torch.equal(o0["color"], o1["color"])
    for k in g0:
        assert torch.equal(g0[k], g1[k]), k
    print(f"[regime] unused alpha (tuning {tuning}): every gradient bit-identical to a call without alpha")


# ---------------------------------------------------------------------------------------------------------------------
# 4. option combinations: SH degree 4 and every depth mode
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["depth", "disparity", "relative_disparity", "log"])
def test_alpha_with_degree4_and_every_depth_mode(mode):
    """Alpha does not depend on the SH degree or the depth channel: the same bits as a degree-3 call without depth, and
    the same alpha-only gradients (to the backward-path tolerance); the colour of degree 4 differs."""
    from tests.sh4_oracle import with_band4
    sc = with_band4(make_scene(4000, 3, 48, 64, seed=13))
    hw = sc.image_shape
    cams, ins = scene_batch_args([sc])
    ins = {k: ins[k] for k in KEEP}
    dcams = {k: v.to(DEV) for k, v in cams.items()}
    near = 1.0 / dcams["view_scale"]
    nf = torch.stack([near, 100 * near], -1)
    dA = np.random.default_rng(76).standard_normal((3, *hw)) / (hw[0] * hw[1])
    g3, o3, _ = _gpu(_settings(dcams, hw)._replace(with_alpha=True, sh_eval_max_degree=3), ins, dA=dA)
    bs = _settings(dcams, hw, with_depth=True)._replace(with_alpha=True, sh_eval_max_degree=4, depth_mode=mode,
                                                         depth_near_far=nf)
    g4, o4, _ = _gpu(bs, ins, dA=dA)
    assert torch.equal(o4["alpha"], o3["alpha"]) and torch.equal(o4["radii"], o3["radii"])
    assert float((o4["color"] - o3["color"]).abs().max()) > 1e-3
    assert float(g4["shs"].abs().max()) == 0.0
    worst = _agree(f"alpha degree 4 + {mode}", {k: g4[k] for k in g3 if k != "shs"}, {k: g3[k] for k in g3 if k != "shs"})
    # and with every term in the loss, the alpha term is the same linear addition on top of colour + depth
    rng = np.random.default_rng(77)
    dL, w = rng.standard_normal((3, 3, *hw)) / 3072, _depth_field(3, hw, 78)
    with _Det():
        ga, _, _ = _gpu(bs, ins, dA=dA, dL=dL, w=w)
        gb, _, _ = _gpu(bs, ins, dL=dL, w=w)
        gc, _, _ = _gpu(bs, ins, dA=dA)
    assert torch.equal(ga["shs"], gb["shs"])
    for k in ("means3D", "opacities", "cov3D_precomp"):
        scale = float(ga[k].abs().max())
        assert float((ga[k] - gb[k] - gc[k]).abs().max()) <= 1e-4 * scale, k
    print(f"[regime] alpha at degree 4 with depth mode {mode}: bit-identical to degree 3, gradients within {worst:.2e}")


# ---------------------------------------------------------------------------------------------------------------------
# 5. the host entry
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("with_depth", [False, True])
def test_host_entry_returns_the_device_entry_bytes(with_depth):
    """Every feed of gs_render_host_ex (pageable upload; pinned zero-copy with the split colour pipeline, with the fused
    pull, through the copy engine; direct output into pinned buffers) returns the device entry's colour, radii, depth
    and alpha bytes."""
    from pf3plat_b200 import rasterizer
    P, V, hw = 20000, 3, (64, 80)
    sc = make_scene(P, V, *hw, seed=14)
    cams, ins = scene_batch_args([sc])
    ins = {k: ins[k] for k in KEEP}
    dcams = {k: v.to(DEV) for k, v in cams.items()}
    ref = _gpu(_settings(dcams, hw, with_depth=with_depth)._replace(with_alpha=True), ins)[1]
    host = {k: v[0].contiguous() for k, v in ins.items()}
    M = host["shs"].shape[1]
    cfg = _capi.GsConfig()
    cfg.P, cfg.S, cfg.V, cfg.M, cfg.sh_degree = P, 1, V, M, 4
    cfg.image_height, cfg.image_width, cfg.scale_modifier = hw[0], hw[1], 1.0
    cfg.flags = _capi.GS_FLAG_DEPTH if with_depth else 0
    hc = {k: v.contiguous() for k, v in cams.items()}
    for k, t in hc.items():
        setattr(cfg, k, t.data_ptr())
    ctx = rasterizer.current_context(DEV)
    color = torch.empty(V, 3, *hw).pin_memory()
    radii = torch.empty(V, P, dtype=torch.int32).pin_memory()
    depth = torch.empty(V, *hw).pin_memory()
    alpha = torch.empty(V, *hw).pin_memory()
    gout = _capi.GsOutputs(color=color.data_ptr(), radii=radii.data_ptr(), depth=depth.data_ptr() if with_depth else None)
    req = _capi.GsAlpha(alpha.data_ptr(), None)
    pin = {k: v.pin_memory() for k, v in host.items()}
    runs = 0
    for src in (host, pin):
        gin = _capi.GsInputs(means3D=src["means3D"].data_ptr(), opacities=src["opacities"].data_ptr(),
                             shs=src["shs"].data_ptr(), cov3D_precomp=src["cov3D_precomp"].data_ptr())
        feeds = (0, _capi.GS_TUNE_DIRECT_OUTPUT) if src is host else \
            (0, _capi.GS_TUNE_NO_SPLIT_COLOUR, _capi.GS_TUNE_NO_ZERO_COPY, _capi.GS_TUNE_DIRECT_OUTPUT)
        for tuning in feeds:
            cfg.tuning = tuning
            color.zero_(); radii.zero_(); depth.zero_(); alpha.fill_(-1.0)
            _capi.check(_capi.lib().gs_render_host_ex(ctx, ctypes.byref(cfg), ctypes.byref(gin), ctypes.byref(gout),
                                                      ctypes.byref(req), torch.cuda.current_stream(DEV).cuda_stream))
            assert torch.equal(color, ref["color"].cpu()) and torch.equal(radii, ref["radii"].cpu()), tuning
            assert torch.equal(alpha, ref["alpha"].cpu()), tuning
            if with_depth:
                assert torch.equal(depth, ref["depth"].cpu()), tuning
            runs += 1
    print(f"[regime] host entry (depth {with_depth}): M = {M}, {runs} feeds bit-identical to the device entry")
    assert M > 16 and runs == 6


# ---------------------------------------------------------------------------------------------------------------------
# 6. edge cases: thin and ragged frames, empty tiles, opaque stacks, off-screen and near-plane Gaussians
# ---------------------------------------------------------------------------------------------------------------------
def _edge_case(label, sc, dev_tuning=0, max_fragile=0.02):
    hw = sc.image_shape
    cams, ins = scene_batch_args([sc])
    ins = {k: ins[k] for k in KEEP}
    V = cams["viewmatrix"].shape[0]
    orc = AlphaOracle(_settings(cams, hw), ins)
    dA = np.random.default_rng(79).standard_normal((V, *hw)) / (hw[0] * hw[1])
    go = orc.backward(dA)
    dcams = {k: v.to(DEV) for k, v in cams.items()}
    grads, out, _ = _gpu(_settings(dcams, hw, tuning=dev_tuning)._replace(with_alpha=True), ins, dA=dA)
    _check_alpha(label, out["alpha"], orc, max_fragile)
    _check_grads(f"{label} alpha-only", {k: g for k, g in grads.items() if k != "shs"}, go, orc.affected(), V)
    return orc, out


@pytest.mark.parametrize("hw", [(1, 40), (33, 250)])
def test_alpha_thin_and_ragged_frames(hw):
    sc = _turned(edge_straddle_scene(600, 120, 2, *hw, seed=90), seed=91)
    orc, _ = _edge_case(f"{hw[0]} x {hw[1]} frame", sc)
    print(f"[regime] {hw}: covered pixels {(orc.alpha > 0).mean():.3f}")
    assert (orc.alpha > 0).any()


def test_alpha_is_exactly_zero_on_empty_tiles():
    """All splats inside one corner box of the frame: every other tile has an empty list and alpha exactly 0 there."""
    sc = long_list_scene(800, 1, 64, 96, box=(2, 2, 30, 28), seed=92)
    orc, out = _edge_case("empty tiles", sc)
    a = out["alpha"].cpu()
    empty_tiles = a[:, 32:, :].abs().max() == 0 and a[:, :, 48:].abs().max() == 0
    print(f"[regime] empty tiles: covered pixels {(orc.alpha > 0).mean():.3f}, alpha outside the box "
          f"{float(a[:, 32:, :].abs().max())}")
    assert empty_tiles and (orc.alpha > 0).any()


@pytest.mark.parametrize("tuning", [0, _capi.GS_TUNE_FWD_WS | _capi.GS_TUNE_BWD_V1])
def test_alpha_of_opaque_stacks_that_stop_early(tuning):
    sc = opaque_stack_scene(6, 12, 2, 48, 64, seed=93)
    orc, out = _edge_case("opaque stack", sc, dev_tuning=tuning, max_fragile=0.2)
    T = orc.final_T
    saturated = float((T < 1e-3).mean())
    print(f"[regime] opaque stack: pixels with T_final < 1e-3 {saturated:.3f}; alpha max {float(out['alpha'].max()):.6f}")
    assert saturated > 0.3 and float(out["alpha"].max()) < 1.0


def test_alpha_with_offscreen_and_near_plane_gaussians():
    sc = offscreen_scene(1500, 200, 2, 48, 64, seed=94)
    _edge_case("off-screen", sc)
    sc = near_plane_scene(1500, 40, 40, 40, 2, 48, 64, seed=95)
    _edge_case("near plane, culled and behind the camera", sc, max_fragile=0.05)


# ---------------------------------------------------------------------------------------------------------------------
# 7. the drop-in and the decoder
# ---------------------------------------------------------------------------------------------------------------------
def test_dropin_return_alpha():
    from pf3plat_b200.rasterizer import GaussianRasterizationSettings, GaussianRasterizer, rasterize_batch
    hw = (48, 64)
    sc = make_scene(3000, 1, *hw, seed=96)
    cams, ins = scene_batch_args([sc])
    c = {k: v.to(DEV) for k, v in cams.items()}
    rs = GaussianRasterizationSettings(image_height=hw[0], image_width=hw[1], tanfovx=float(c["tanfov"][0, 0]),
                                       tanfovy=float(c["tanfov"][0, 1]), bg=c["bg"][0], scale_modifier=1.0,
                                       viewmatrix=c["viewmatrix"][0], projmatrix=c["projmatrix"][0], sh_degree=4,
                                       campos=c["campos"][0], prefiltered=False, debug=False)
    r = GaussianRasterizer(rs)
    m = ins["means3D"][0].to(DEV)
    kw = dict(means3D=m, means2D=torch.zeros_like(m), opacities=ins["opacities"][0].to(DEV),
              shs=ins["shs"][0].to(DEV), cov3D_precomp=ins["cov3D_precomp"][0].to(DEV))
    two = r(**kw)
    three = r(**kw, return_alpha=True)
    four = r(**kw, return_depth=True, return_alpha=True)
    assert len(two) == 2 and len(three) == 3 and len(four) == 4
    assert torch.equal(two[0], three[0]) and torch.equal(three[2], four[3]) and three[2].shape == hw
    bs = _settings({**c, "view_scale": None}, hw)._replace(with_alpha=True, tanfov=None,
                                                            tanfovx=float(c["tanfov"][0, 0]), tanfovy=float(c["tanfov"][0, 1]))
    with torch.no_grad():
        batched = rasterize_batch(bs, **{k: v.to(DEV) for k, v in ins.items() if k in KEEP})
    assert torch.equal(batched[2][0], three[2])
    print(f"[regime] drop-in: alpha {float(three[2].min()):.3f}..{float(three[2].max()):.3f}")


def test_decoder_forward_return_alpha():
    """Alpha-only loss: the extrinsics (requiring grad) get None, the opacities a gradient.  With a depth loss, the
    extrinsics' gradient is bit-equal with and without an added alpha term (deterministic mode)."""
    from pf3plat_b200 import render
    b, v, P, hw = 2, 3, 1500, (48, 64)
    scs = [_turned(make_scene(P, v, *hw, seed=720 + k), seed=730 + k) for k in range(b)]
    st = lambda name: torch.stack([getattr(s, name) for s in scs]).to(DEV)
    ext, intr = st("extrinsics"), st("intrinsics")
    nr, fr = torch.full((b, v), 0.5, device=DEV), torch.full((b, v), 50.0, device=DEV)
    bg = torch.tensor([0.3, 0.2, 0.1], device=DEV)
    names = ("means", "covariances", "harmonics", "opacities")
    dA = torch.as_tensor(np.random.default_rng(97).standard_normal((b, v, *hw)) / 3072, dtype=torch.float32, device=DEV)
    w = torch.as_tensor(_depth_field(b * v, hw, 98), dtype=torch.float32, device=DEV).reshape(b, v, *hw)

    e = ext.clone().requires_grad_(True)
    L = [st(n).clone().requires_grad_(True) for n in names]
    color, depth, alpha = render.decoder_forward(*L, e, intr, nr, fr, hw, bg, return_alpha=True)
    assert depth is None and alpha.shape == (b, v, *hw)
    plain, _ = render.decoder_forward(*[st(n) for n in names], ext, intr, nr, fr, hw, bg)
    assert torch.equal(plain, color.detach())
    alpha.backward(dA)
    assert e.grad is None and float(L[3].grad.abs().max()) > 0 and float(L[2].grad.abs().max()) == 0.0

    def depth_run(with_alpha_term):
        e = ext.clone().requires_grad_(True)
        L = [st(n).clone().requires_grad_(True) for n in names]
        color, depth, alpha = render.decoder_forward(*L, e, intr, nr, fr, hw, bg, depth_mode="depth", return_alpha=True)
        ts, gs = [depth], [w]
        if with_alpha_term:
            ts.append(alpha)
            gs.append(dA)
        torch.autograd.backward(ts, gs)
        return e.grad, L[3].grad

    with _Det():
        e0, o0 = depth_run(False)
        e1, o1 = depth_run(True)
    assert e0 is not None and float(e0.abs().max()) > 0 and torch.equal(e0, e1)
    assert not torch.equal(o0, o1)
    print(f"[regime] decoder: alpha {float(alpha.detach().min()):.3f}..{float(alpha.detach().max()):.3f}; extrinsics gradient "
          f"bit-identical with and without the alpha term")
