"""The rasterizer's gradients against the fp64 oracles under the strict rule of tests/strict_parity.py: the cotangent is zero
at the oracle's fragile pixels, and every Gaussian -- except the few whose own radius, near-plane cull, SH clamp or
anti-aliasing clamp is undecided -- is held to |a - b| <= 1e-3 (|b| + rms(b)) per tensor and per SH band.

The scenes, oracles and calls are the ones the loose-rule tests use (test_gpu_parity, test_gpu_regimes,
test_gpu_backward_paths, test_gpu_steady_state, test_gpu_alpha, test_gpu_antialias, test_gpu_depth_modes,
test_gpu_sh_degree4, test_gpu_config_sizes), imported rather than rebuilt.  Each case prints its masked pixel fraction,
its per-Gaussian exemption count and the worst ratio of every gradient tensor ("[strict]" lines)."""
import numpy as np
import pytest
import torch

from pf3plat_b200 import _capi
from pf3plat_b200.synthetic import make_pixel_aligned_scene, make_scene, make_target
from tests.aa_oracle import AAOracle
from tests.alpha_oracle import AlphaOracle
from tests.batch_oracle import oracle_batch, scene_batch_args
from tests.depth_modes_oracle import DepthModeOracle
from tests.regimes import near_plane_scene, offscreen_scene, opaque_stack_scene
from tests.sh4_oracle import SH_BANDS4, ShOracleBatch, with_band4
from tests.strict_parity import (check_exempt, check_grad_strict, check_masked_regime, early_terminated, fragile_pixels,
                                 masked_cotangent, per_gaussian_decisions)
from tests.test_gpu_alpha import _Det
from tests.test_gpu_antialias import _gpu, _shrink
from tests.test_gpu_backward_paths import _incoming, _squeezed
from tests.test_gpu_depth_chain import _depth_batch, _depth_field
from tests.test_gpu_depth_modes import _near_far
from tests.test_gpu_regimes import _many_view_batch, _operator_inputs, _settings

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
KEEP = ("means3D", "opacities", "shs", "cov3D_precomp")
PER_VIEW = ("means2D", "colors_precomp")


@pytest.fixture(autouse=True, scope="module")
def _fresh_contexts():
    """Contexts are cached per (device, stream) and torch reuses streams: start and end with none cached."""
    import gc
    from pf3plat_b200.rasterizer import destroy_contexts
    torch.cuda.synchronize()
    destroy_contexts()
    yield
    torch.use_deterministic_algorithms(False)
    gc.collect()
    torch.cuda.synchronize()
    destroy_contexts()


# ---------------------------------------------------------------------------------------------------------------------
# the engine
# ---------------------------------------------------------------------------------------------------------------------
def _compare(label, grads, gref, exempt, VPS):
    """Every gradient the call returned that the oracle has, strictly.  Per-scene tensors over S*P Gaussians, per-view ones
    (means2D, colors_precomp) over V*P, a Gaussian of view v exempt if it is exempt in its scene."""
    S, P = exempt.shape
    ex_v = np.repeat(exempt, VPS, axis=0).reshape(-1)
    worst = {}
    for name, t in grads.items():
        ref = gref.get(name)
        if ref is None or t is None:
            continue
        if name in PER_VIEW:
            rep = check_grad_strict(f"{label} dL/d{name}", t.reshape(-1, 3), np.asarray(ref).reshape(-1, 3), ex_v)
        elif name == "shs":
            M = ref.shape[2]
            rep = check_grad_strict(f"{label} dL/dshs", t.reshape(S * P, M, 3), np.asarray(ref).reshape(S * P, M, 3),
                                    exempt.reshape(-1), bands=[b for b in SH_BANDS4 if b[1].start < M])
        else:
            rep = check_grad_strict(f"{label} dL/d{name}", t.reshape(S * P, -1), np.asarray(ref).reshape(S * P, -1),
                                    exempt.reshape(-1))
        worst[name] = rep["worst_ratio"]
    print(f"[strict] {label}: worst ratio per tensor {({k: float(f'{v:.2e}') for k, v in worst.items()})}")
    return worst


def _strict(label, orc, cots, runs, max_fragile=0.03, early=False, refs=()):
    """orc: a batched oracle; cots: its backward's arguments (full cotangents, [V,...] or None); runs: {label: fn(masked
    cotangents) -> GPU gradients}.  Masks, checks the regime guard and the exemptions, then every run against the oracle
    (and against every extra oracle in `refs`, e.g. the fp32 one, under the same masked cotangent)."""
    frag = fragile_pixels(orc)
    for r in refs:
        frag = frag | fragile_pixels(r)
    masked = [None if c is None else masked_cotangent(np.asarray(c, np.float32), frag) for c in cots]
    gref = orc.backward(*masked)
    full = [None if c is None else np.asarray(c, np.float32) for c in cots]
    check_masked_regime(label, frag, max_fragile, gref, orc.backward(*full),
                        early_terminated(orc) if early else None)
    exempt = per_gaussian_decisions(orc)
    for r in refs:
        exempt = exempt | per_gaussian_decisions(r)
    check_exempt(label, exempt)
    worst = {}
    for run_label, fn in runs.items():
        grads = fn(masked)
        for k, g in [("", gref)] + [(f" vs {r.dtype if hasattr(r, 'dtype') else 'ref'} oracle", r.backward(*masked))
                                    for r in refs]:
            w = _compare(f"{label} {run_label}{k}", grads, g, exempt, orc.VPS)
            for n, x in w.items():
                worst[n] = max(worst.get(n, 0.0), x)
    return worst


def _batch_run(bs, ins, det=False):
    """fn(masked [dL, dLd?]) -> gradients of rasterize_batch (with a means2D sink) under bs (device cameras)."""
    def fn(masked):
        dL, dLd = masked[0], (masked[1] if len(masked) > 1 else None)
        if det:
            with _Det():
                return _gpu(bs, ins, dL=dL, w=dLd)[0]
        return _gpu(bs, ins, dL=dL, w=dLd)[0]
    return fn


def _case(label, cams, ins, hw, cots=None, seed=1, with_depth=True, tunings=((0, "default"),), max_fragile=0.03,
          early=False, fp32=False, **settings):
    """One batched call against oracle_batch in fp64 (and fp32 if asked), under each tuning."""
    bs_cpu = _settings(cams, hw, with_depth=with_depth, **settings)
    ob = oracle_batch(bs_cpu, dtype=np.float64, **ins)
    refs = (oracle_batch(bs_cpu, dtype=np.float32, **ins),) if fp32 else ()
    if cots is None:
        dL, dLd = _incoming(ob.V, hw, seed)
        cots = [dL, dLd if with_depth else None]
    dcams = {k: v.to(DEV) for k, v in cams.items()}
    runs = {}
    for tuning, name in tunings:
        det = tuning == "det"
        bs = _settings(dcams, hw, with_depth=with_depth, tuning=0 if det else tuning, **settings)
        runs[name] = _batch_run(bs, ins, det)
    return _strict(label, ob, cots, runs, max_fragile, early, refs)


def _single(sc):
    cams, ins = scene_batch_args([sc])
    return cams, {k: ins[k] for k in KEEP}


def _mse(ob_color, seed=1):
    V, _, H, W = ob_color.shape
    target = make_target(V, H, W, seed=seed).numpy()
    return 2 * (ob_color - target) / target.size


TUNINGS = ((0, "default"), (_capi.GS_TUNE_BWD_OCC4, "bwd occ4"), (_capi.GS_TUNE_BWD_V1, "bwd v1"),
           ("det", "deterministic"))


# ---------------------------------------------------------------------------------------------------------------------
# 1. test_gpu_parity's scenes
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["sh_cov", "rgb_cov", "sh_scalerot"])
def test_input_modes(mode):
    sc = make_scene(4000, 2, 48, 64, seed=3)
    cams, ins = scene_batch_args([sc])
    keep = {"means3D": ins["means3D"], "opacities": ins["opacities"]}
    if mode.startswith("sh"):
        keep["shs"] = ins["shs"]
    else:
        keep["colors_precomp"] = ins["shs"][:, :, 0].expand(2, -1, -1).contiguous()
    if mode.endswith("scalerot"):
        keep["scales"], keep["rotations"] = ins["scales"], ins["rotations"]
    else:
        keep["cov3D_precomp"] = ins["cov3D_precomp"]
    _case(mode, cams, keep, sc.image_shape, seed=3)


def test_batched_views_with_depth():
    sc = make_scene(6000, 3, 64, 64, seed=4)
    _case("batched 3 views + depth", *_single(sc), sc.image_shape, seed=4)


@pytest.mark.parametrize("blow_up", [25.0, 400.0])
def test_huge_footprints(blow_up):
    sc = make_scene(24, 2, 48, 80, seed=17)
    sc.covariances.mul_(blow_up)
    _case(f"x{blow_up:g} footprints", *_single(sc), sc.image_shape, seed=17, max_fragile=0.1)


@pytest.mark.parametrize("d_sh,P", [(1, 1000), (4, 1001), (9, 777), (16, 1300), (16, 129), (25, 1301), (25, 63)])
def test_sh_coefficient_counts(d_sh, P):
    sc = make_scene(P, 2, 48, 48, seed=40 + d_sh, d_sh=d_sh)
    _case(f"d_sh={d_sh} P={P}", *_single(sc), sc.image_shape, seed=40)


def test_pixel_aligned_cloud():
    sc = make_pixel_aligned_scene(128, 128, 3, seed=2)
    _case("pixel-aligned 128x128", *_single(sc), sc.image_shape, seed=2)


# ---------------------------------------------------------------------------------------------------------------------
# 2. test_gpu_regimes' regimes, and every backward kernel
# ---------------------------------------------------------------------------------------------------------------------
def test_opaque_stacks_every_backward_kernel():
    """Early termination at T < 1e-4 behind alpha clamped at 0.99, against the fp64 and the fp32 oracle, under every
    backward kernel and the deterministic backward."""
    hw = (48, 64)
    sc = opaque_stack_scene(6, 10, 2, *hw, seed=110)
    _case("opaque stacks", *_single(sc), hw, seed=110, tunings=TUNINGS, early=True, fp32=True, max_fragile=0.2)


def test_dense_scene_every_backward_kernel():
    sc = make_scene(40000, 3, 80, 112, seed=12)
    _case("dense 40k", *_single(sc), sc.image_shape, seed=12, tunings=TUNINGS)


def test_near_plane_splats():
    hw = (48, 64)
    sc = near_plane_scene(1500, 150, 60, 60, 2, *hw, seed=100)
    _case("near plane", *_single(sc), hw, seed=100, early=True, max_fragile=0.05)


def test_offscreen_centres():
    hw = (48, 64)
    sc = offscreen_scene(1500, 400, 2, *hw, seed=90)
    _case("off-screen", *_single(sc), hw, seed=90)


def test_many_views_per_scene():
    cams, ins, hw = _many_view_batch("cpu")
    _case("VPS=19", cams, ins, hw, seed=50,
          tunings=((0, "default"), (_capi.GS_TUNE_PBWD_2PHASE, "2-phase preprocess bwd"), (_capi.GS_TUNE_BWD_V1, "bwd v1")))


@pytest.mark.parametrize("colour", ["shs", "colors"])
@pytest.mark.parametrize("geometry,mod", [("cov3D", 1.0), ("scalerot", 1.0), ("scalerot", 0.7)])
def test_operator_input_matrix(colour, geometry, mod):
    cams, ins, hw = _operator_inputs(colour, geometry, mod=mod)
    _case(f"{colour}/{geometry}/mod={mod}", cams, ins, hw, seed=80, scale_modifier=mod)


# ---------------------------------------------------------------------------------------------------------------------
# 3. every binning path (test_gpu_backward_paths) and lazily sorted strata (test_gpu_steady_state)
# ---------------------------------------------------------------------------------------------------------------------
def _sequence_runs(bs, ins, sequence, setup=None):
    """One run per (label, tuning, expected speculative state), each doing its forward + backward in turn on one stream
    (a context) of its own, after `setup` (forward-only calls) has run there.  tuning "det": the deterministic backward."""
    from pf3plat_b200.rasterizer import last_stats
    stream = torch.cuda.Stream(DEV)
    with torch.cuda.stream(stream):
        for extra in setup or ():
            _gpu(bs._replace(tuning=extra[0]), extra[1])
        stream.synchronize()

    def run(tuning, want, label):
        def fn(masked):
            with torch.cuda.stream(stream):
                if tuning == "det":
                    with _Det():
                        g = _gpu(bs, ins, dL=masked[0], w=masked[1])[0]
                else:
                    g = _gpu(bs._replace(tuning=tuning), ins, dL=masked[0], w=masked[1])[0]
                st = last_stats(DEV)
                stream.synchronize()
            print(f"[strict] {label}: speculative {st['speculative']}, overflow redos {st['overflow_redos']}")
            assert want is None or st["speculative"] == want, (label, st)
            return g
        return fn
    return {label: run(tuning, want, label) for label, tuning, want in sequence}


def test_every_binning_state():
    from pf3plat_b200._capi import (GS_TUNE_FORCE_RADIX_BINNING, GS_TUNE_NO_SPECULATION, GS_TUNE_NO_STRATA,
                                    GS_TUNE_SEPARATE_EMIT)
    hw = (32, 48)
    scenes = [make_scene(2500, 3, *hw, seed=70 + k) for k in range(2)]
    cams, ins = scene_batch_args(scenes, near=1.0 / np.tile(np.linspace(0.8, 1.25, 3), 2))
    ins = {k: ins[k] for k in KEEP}
    ob = oracle_batch(_settings(cams, hw, with_depth=True), dtype=np.float64, **ins)
    dcams = {k: v.to(DEV) for k, v in cams.items()}
    bs = _settings(dcams, hw, with_depth=True)
    sequence = [("exact", GS_TUNE_NO_SPECULATION, 0), ("per-view strata trial", 0, 2), ("stratified", 0, 2),
                ("stratified, k_emit_buckets", GS_TUNE_SEPARATE_EMIT, 2),
                ("exact, re-learn unstratified", GS_TUNE_NO_STRATA | GS_TUNE_NO_SPECULATION, 0),
                ("whole-tile", GS_TUNE_NO_STRATA, 1), ("radix fallback", GS_TUNE_FORCE_RADIX_BINNING, 0)]
    _strict("binning paths", ob, list(_incoming(ob.V, hw, seed=71)), _sequence_runs(bs, ins, sequence))


def test_per_tile_strata():
    sc = make_pixel_aligned_scene(128, 128, 3, seed=2)
    hw = sc.image_shape
    cams, ins = _single(sc)
    ob = oracle_batch(_settings(cams, hw, with_depth=True), dtype=np.float64, **ins)
    bs = _settings({k: v.to(DEV) for k, v in cams.items()}, hw, with_depth=True)
    runs = _sequence_runs(bs, ins, [("per-tile strata", 0, 2)], setup=[(0, ins)] * 5)
    _strict("per-tile strata", ob, list(_incoming(ob.V, hw, seed=72)), runs)


def test_overflow_redo():
    hw = (48, 64)
    sparse = make_scene(3000, 2, *hw, seed=73)
    dense = _squeezed(sparse, 0.63)
    cams, ins_s = _single(sparse)
    _, ins_d = _single(dense)
    ob = oracle_batch(_settings(cams, hw, with_depth=True), dtype=np.float64, **ins_d)
    bs = _settings({k: v.to(DEV) for k, v in cams.items()}, hw, with_depth=True)
    runs = _sequence_runs(bs, ins_d, [("overflow redo", 0, 0)], setup=[(0, ins_s)] * 3)
    _strict("overflow redo", ob, list(_incoming(ob.V, hw, seed=74)), runs)


def test_lazily_sorted_strata_in_the_steady_state():
    """A saturating shape (7.5 Gaussians per pixel, as C2) on a context of its own: exact, trial, then lazily sorted
    strata -- the fourth call's backward reads the lists the compositor extended."""
    hw = (64, 96)
    sc = make_scene(46_000, 2, *hw, seed=130)
    cams, ins = _single(sc)
    ob = oracle_batch(_settings(cams, hw, with_depth=True), dtype=np.float64, **ins)
    bs = _settings({k: v.to(DEV) for k, v in cams.items()}, hw, with_depth=True)
    runs = _sequence_runs(bs, ins, [("lazy strata, call 4", 0, 2), ("lazy strata, call 5, deterministic", "det", 2)],
                          setup=[(0, ins)] * 3)
    _strict("steady state", ob, list(_incoming(ob.V, hw, seed=131)), runs, max_fragile=0.05)


# ---------------------------------------------------------------------------------------------------------------------
# 4. features: alpha, anti-aliasing, depth modes, SH degree 4
# ---------------------------------------------------------------------------------------------------------------------
def test_alpha():
    cams, ins, hw = _depth_batch("cov3D")
    V = cams["viewmatrix"].shape[0]
    bs_cpu = _settings(cams, hw, with_depth=True)
    orc = AlphaOracle(bs_cpu, ins, base=oracle_batch(bs_cpu, dtype=np.float64, **ins))
    orc.VPS = orc.base.VPS
    dA = np.random.default_rng(71).standard_normal((V, *hw)) / (hw[0] * hw[1])
    bs = _settings({k: v.to(DEV) for k, v in cams.items()}, hw, with_depth=True)._replace(with_alpha=True)
    run = lambda m: _gpu(bs, ins, dA=m[0], dL=m[1], w=m[2])[0]
    _strict("alpha", orc, [dA, _mse(orc.color), _depth_field(V, hw, 72)], {"default": run})


def test_antialiasing():
    cams, ins, hw = _depth_batch("cov3D")
    ins = _shrink(ins)
    V = cams["viewmatrix"].shape[0]
    bs_cpu = _settings(cams, hw, with_depth=True)._replace(antialiasing=True)
    orc = AAOracle(bs_cpu, ins)
    vis = orc.radii.reshape(V, -1) > 0
    print(f"[strict] anti-aliasing: rho of visible pairs {orc.rho[vis].min():.4f}..{orc.rho[vis].max():.4f}, "
          f"Gaussians at the clamp {int((orc.near_clamp & vis).sum())}")
    assert orc.rho[vis].min() < 0.05
    bs = _settings({k: v.to(DEV) for k, v in cams.items()}, hw, with_depth=True)._replace(antialiasing=True)
    run = lambda m: _gpu(bs, ins, dL=m[0], w=m[1])[0]
    _strict("anti-aliasing", orc, [_mse(orc.color), _depth_field(V, hw, 72)], {"default": run})


def test_antialiasing_at_the_clamp():
    """Sub-pixel splats whose ratio det0 / det1 reaches the 2.5e-5 floor of the compensation (rho's derivative jumps
    there): the clamped ones must get the strict gradient, only those within 1e-3 of the floor are exempt."""
    sc = make_pixel_aligned_scene(32, 48, 2, seed=21)
    cams, ins = _single(sc)
    ins = _shrink(ins, every=2, factor=300.0)
    hw = sc.image_shape
    V = cams["viewmatrix"].shape[0]
    orc = AAOracle(_settings(cams, hw)._replace(antialiasing=True), ins)
    from tests.aa_oracle import RATIO_MIN
    vis = orc.radii.reshape(V, -1) > 0
    n_clamped = int(((orc.ratio < RATIO_MIN) & vis).sum())
    print(f"[strict] anti-aliasing clamp: visible pairs {int(vis.sum())}, clamped {n_clamped}, "
          f"within 1e-3 of the clamp {int((orc.near_clamp & vis).sum())}")
    assert n_clamped > 0
    bs = _settings({k: v.to(DEV) for k, v in cams.items()}, hw)._replace(antialiasing=True)
    run = lambda m: _gpu(bs, ins, dL=m[0])[0]
    _strict("anti-aliasing clamp", orc, [_mse(orc.color)], {"default": run}, max_fragile=0.05)


@pytest.mark.parametrize("mode", ["depth", "disparity", "relative_disparity", "log"])
def test_depth_modes(mode):
    hw = (40, 56)
    scenes = [make_scene(2500, 3, *hw, seed=140 + k) for k in range(2)]
    cams, ins = scene_batch_args(scenes, near=1.0 / np.tile(np.linspace(0.8, 1.25, 3), 2))
    ins = {k: ins[k] for k in KEEP}
    nf = _near_far(cams)
    orc = DepthModeOracle(_settings(cams, hw)._replace(depth_mode=mode, depth_near_far=nf), ins, mode, nf)
    dL, w = _incoming(orc.V, hw, 141)
    # "depth" composites the rescaled s * z (test_gpu_steady_state._oracle): the oracle's weight on z is s times the call's
    s = cams["view_scale"].numpy().astype(np.float64)[:, None, None] if mode == "depth" else 1.0
    bs = _settings({k: v.to(DEV) for k, v in cams.items()}, hw, with_depth=True)._replace(
        depth_mode=mode, depth_near_far=nf.to(DEV))
    run = lambda m: _gpu(bs, ins, dL=m[0], w=m[1] / s)[0]
    _strict(f"depth mode {mode}", orc, [dL, w * s], {"default": run})


def test_sh_degree4():
    sc = with_band4(make_scene(4000, 3, 48, 64, seed=13))
    hw = sc.image_shape
    cams, ins = _single(sc)
    bs_cpu = _settings(cams, hw, with_depth=True)._replace(sh_eval_max_degree=4)
    orc = ShOracleBatch(bs_cpu, ins["means3D"], ins["opacities"], ins["shs"], deg=4, cov3D_precomp=ins["cov3D_precomp"])
    dL, dLd = _incoming(orc.V, hw, 14)
    bs = _settings({k: v.to(DEV) for k, v in cams.items()}, hw, with_depth=True)._replace(sh_eval_max_degree=4)
    run = lambda m: _gpu(bs, ins, dL=m[0], w=m[1])[0]
    worst = _strict("SH degree 4", orc, [dL, dLd], {"default": run})
    assert "shs" in worst


# ---------------------------------------------------------------------------------------------------------------------
# 5. the C5 shape: 131 072 pixel-aligned Gaussians at 256 x 256
# ---------------------------------------------------------------------------------------------------------------------
def test_c5_shape():
    sc = make_pixel_aligned_scene(256, 256, 2, seed=5)
    assert sc.means.shape[0] == 2 * 256 * 256
    cams, ins = _single(sc)
    hw = sc.image_shape
    ob = oracle_batch(_settings(cams, hw), dtype=np.float64, **ins)
    bs = _settings({k: v.to(DEV) for k, v in cams.items()}, hw)
    _strict("C5 shape", ob, [_mse(ob.color, seed=1)], {"default": _batch_run(bs, ins)}, max_fragile=0.05)
