"""The deterministic backward (torch.use_deterministic_algorithms(True) -> GS_FLAG_DETERMINISTIC and
GS_ADAPTER_DETERMINISTIC): gradients that are bit-identical from run to run, on every binning path and kernel variant,
that still match the fp64 oracle, that scale exactly with the incoming gradient, and that turn non-finite exactly where
the default path's do.  Every test runs with torch's flag set by the fixture below and restores it afterwards."""
import os

# torch's glue may run cuBLAS matmuls; under the flag they need a fixed workspace (set before the first CUDA use)
os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")

import numpy as np  # noqa: E402
import pytest  # noqa: E402
import torch  # noqa: E402

from pf3plat_b200.synthetic import make_scene, make_target  # noqa: E402
from tests import adapter_util as au  # noqa: E402
from tests.batch_oracle import oracle_batch, scene_batch_args  # noqa: E402
from tests.chain_oracle import make_chain_inputs  # noqa: E402
from tests.test_gpu_backward_paths import _incoming  # noqa: E402
from tests.test_gpu_regimes import _check_grads, _operator_inputs, _settings  # noqa: E402
from tests.util import grad_report  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def deterministic():
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(was, warn_only=warn)


def _dev():
    assert torch.cuda.is_available(), "GPU test needs CUDA"
    return torch.device("cuda:0")


def _unrelated_work(dev):
    """Something else on the stream between two backwards: a sort and a reduction of a few million floats."""
    x = torch.randn(1 << 22, device=dev)
    torch.sort(x)
    return float(x.abs().sum())


def _grads(bs, ins, dL, dLd=None, view_grad=False):
    """rasterize_batch (means2D requested) and its backward; {name: grad}, "viewmatrix" included when view_grad."""
    from pf3plat_b200.rasterizer import rasterize_batch
    dev = bs.viewmatrix.device
    leaves = {k: v.to(dev).clone().requires_grad_(True) for k, v in ins.items()}
    V, P = bs.viewmatrix.shape[0], ins["means3D"].shape[1]
    leaves["means2D"] = torch.zeros(V, P, 3, device=dev, requires_grad=True)
    if view_grad:
        bs = bs._replace(viewmatrix=bs.viewmatrix.detach().clone().requires_grad_(True))
    out = rasterize_batch(bs, **leaves)
    outs, gs = [out[0]], [torch.as_tensor(dL, device=dev)]
    if dLd is not None:
        outs.append(out[2])
        gs.append(torch.as_tensor(dLd, device=dev))
    torch.autograd.backward(outs, gs)
    grads = {k: t.grad.detach().clone() for k, t in leaves.items()}
    if view_grad:
        grads["viewmatrix"] = bs.viewmatrix.grad.detach().clone()
    return grads


def _assert_equal(label, a, b):
    assert set(a) == set(b), label
    for k in a:
        assert torch.equal(a[k], b[k]), (label, k, float((a[k] - b[k]).abs().max()))


def _default_path(fn):
    torch.use_deterministic_algorithms(False)
    try:
        return fn()
    finally:
        torch.use_deterministic_algorithms(True)


# ---------------------------------------------------------------------------------------------------------------------
# 1. repeated runs, on one stream and on a second one (a second context), against the oracle
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("colour,geometry,depth", [("shs", "cov3D", False), ("colors", "scalerot", False),
                                                   ("shs", "scalerot", True), ("colors", "cov3D", True)])
def test_repeated_runs_are_bit_identical_and_match_oracle(colour, geometry, depth):
    dev = _dev()
    cams, ins, hw = _operator_inputs(colour, geometry, mod=0.8)
    label = f"{colour}/{geometry}/{'colour+depth' if depth else 'colour'}"
    ob = oracle_batch(_settings(cams, hw, scale_modifier=0.8, with_depth=depth), dtype=np.float64, **ins)
    dL, dLd = _incoming(ob.V, hw, seed=91)
    dLd = dLd if depth else None
    gref = ob.backward(dL, dLd)
    bs = _settings({k: v.to(dev) for k, v in cams.items()}, hw, scale_modifier=0.8, with_depth=depth)
    runs = []
    for _ in range(3):
        runs.append(_grads(bs, ins, dL, dLd, view_grad=depth))
        _unrelated_work(dev)
    stream = torch.cuda.Stream(dev)
    with torch.cuda.stream(stream):
        runs.append(_grads(bs, ins, dL, dLd, view_grad=depth))
        stream.synchronize()
    for k, r in enumerate(runs[1:]):
        _assert_equal(f"{label} run {k + 1}", r, runs[0])
    det = runs[0]
    if depth:
        assert float(det["viewmatrix"].abs().max()) > 0
    names = [k for k in det if k != "viewmatrix"]
    _check_grads(label + " deterministic", {k: det[k] for k in names}, gref, ob.affected(), ob.VPS)
    dflt = _default_path(lambda: _grads(bs, ins, dL, dLd, view_grad=depth))
    for k in names:
        ref = gref[k].reshape(det[k].shape[0] * det[k].shape[1], -1) if k in ("means2D", "colors_precomp") else \
            gref[k].reshape(ob.S * ob.P, -1)
        rd = grad_report(k, det[k].reshape(ref.shape[0], -1), ref, None)
        rf = grad_report(k, dflt[k].reshape(ref.shape[0], -1), ref, None)
        print(f"[determinism] {label} dL/d{k}: worst ratio to the fp64 oracle, deterministic {rd['worst_ratio_unaffected']:.2e}"
              f" vs default {rf['worst_ratio_unaffected']:.2e}")
    if depth:
        # the default path's view-matrix gradient is pinned to the oracle by the depth-chain tests
        scale = float(dflt["viewmatrix"].abs().max())
        err = float((det["viewmatrix"] - dflt["viewmatrix"]).abs().max())
        print(f"[determinism] {label} dL/dviewmatrix: max |deterministic - default| = {err:.2e} of max-abs {scale:.2e}")
        assert err <= 2e-5 * scale


# ---------------------------------------------------------------------------------------------------------------------
# 2. every binning path: one set of bits
# ---------------------------------------------------------------------------------------------------------------------
def _binning_sequence():
    from pf3plat_b200._capi import (GS_TUNE_FORCE_RADIX_BINNING, GS_TUNE_NO_SPECULATION, GS_TUNE_NO_STRATA,
                                    GS_TUNE_SEPARATE_EMIT)
    return [("exact", GS_TUNE_NO_SPECULATION, 0), ("per-view strata trial", 0, 2), ("stratified", 0, 2),
            ("stratified, k_emit_buckets", GS_TUNE_SEPARATE_EMIT, 2),
            ("exact, re-learn unstratified", GS_TUNE_NO_STRATA | GS_TUNE_NO_SPECULATION, 0),
            ("whole-tile", GS_TUNE_NO_STRATA, 1), ("radix fallback", GS_TUNE_FORCE_RADIX_BINNING, 0)]


def test_every_binning_path_gives_the_same_bits():
    from pf3plat_b200.rasterizer import last_stats
    dev = _dev()
    hw = (32, 48)
    scenes = [make_scene(2500, 3, *hw, seed=70 + k) for k in range(2)]
    cams, ins = scene_batch_args(scenes, near=1.0 / np.tile(np.linspace(0.8, 1.25, 3), 2))
    ins = {k: ins[k] for k in ("means3D", "opacities", "shs", "cov3D_precomp")}
    ob = oracle_batch(_settings(cams, hw, with_depth=True), dtype=np.float64, **ins)
    dL, dLd = _incoming(ob.V, hw, seed=71)
    gref = ob.backward(dL, dLd)
    dcams = {k: v.to(dev) for k, v in cams.items()}
    stream = torch.cuda.Stream(dev)
    first, states = None, []
    with torch.cuda.stream(stream):
        for label, tuning, want in _binning_sequence():
            grads = _grads(_settings(dcams, hw, with_depth=True, tuning=tuning), ins, dL, dLd, view_grad=True)
            st = last_stats(dev)
            states.append(st["speculative"])
            assert st["speculative"] == want and st["overflow_redos"] == 0, (label, st)
            if first is None:
                first = grads
                _check_grads("binning paths, exact", {k: v for k, v in grads.items() if k != "viewmatrix"}, gref,
                             ob.affected(), ob.VPS)
            else:
                _assert_equal(label, grads, first)
        stream.synchronize()
    print(f"[determinism] binning paths {states}: every gradient bit-identical, dL/dviewmatrix_z included")


def test_overflow_redo_gives_the_same_bits():
    """A speculative call that overflows and is redone exactly hands the backward the exact path's lists."""
    from pf3plat_b200._capi import GS_TUNE_NO_SPECULATION
    from pf3plat_b200.rasterizer import last_stats
    from tests.test_gpu_backward_paths import _squeezed
    dev = _dev()
    hw = (48, 64)
    sparse = make_scene(3000, 2, *hw, seed=73)
    dense = _squeezed(sparse, 0.63)
    cams, ins_s = scene_batch_args([sparse])
    _, ins_d = scene_batch_args([dense])
    keep = ("means3D", "opacities", "shs", "cov3D_precomp")
    ins_s, ins_d = ({k: i[k] for k in keep} for i in (ins_s, ins_d))
    dcams = {k: v.to(dev) for k, v in cams.items()}
    dL, dLd = _incoming(2, hw, seed=74)
    stream = torch.cuda.Stream(dev)
    with torch.cuda.stream(stream):
        for _ in range(3):
            _grads(_settings(dcams, hw, with_depth=True), ins_s, dL, dLd)
        redos = last_stats(dev)["overflow_redos"]
        redone = _grads(_settings(dcams, hw, with_depth=True), ins_d, dL, dLd, view_grad=True)
        assert last_stats(dev)["overflow_redos"] == redos + 1
        exact = _grads(_settings(dcams, hw, with_depth=True, tuning=GS_TUNE_NO_SPECULATION), ins_d, dL, dLd,
                       view_grad=True)
        stream.synchronize()
    _assert_equal("overflow redo vs exact", redone, exact)


# ---------------------------------------------------------------------------------------------------------------------
# 3. kernel variants
# ---------------------------------------------------------------------------------------------------------------------
def test_kernel_variants_reproduce_themselves_and_round1_is_refused():
    from pf3plat_b200._capi import GS_TUNE_BWD_OCC4, GS_TUNE_BWD_V1, GS_TUNE_PBWD_2PHASE
    dev = _dev()
    cams, ins, hw = _operator_inputs("shs", "cov3D")
    dcams = {k: v.to(dev) for k, v in cams.items()}
    dL, dLd = _incoming(4, hw, seed=92)
    for tuning, label in ((0, "default"), (GS_TUNE_BWD_OCC4, "OCC4"), (GS_TUNE_PBWD_2PHASE, "two-phase preprocess"),
                          (GS_TUNE_BWD_OCC4 | GS_TUNE_PBWD_2PHASE, "OCC4 + two-phase")):
        bs = _settings(dcams, hw, with_depth=True, tuning=tuning)
        a = _grads(bs, ins, dL, dLd, view_grad=True)
        _unrelated_work(dev)
        _assert_equal(label, _grads(bs, ins, dL, dLd, view_grad=True), a)
    with pytest.raises(ValueError, match="GS_TUNE_BWD_V1"):
        _grads(_settings(dcams, hw, with_depth=True, tuning=GS_TUNE_BWD_V1), ins, dL, dLd)
    _default_path(lambda: _grads(_settings(dcams, hw, tuning=GS_TUNE_BWD_V1), ins, dL))   # still there by default


# ---------------------------------------------------------------------------------------------------------------------
# 4. range and resolution: scaling the incoming gradients by 2^k scales every gradient by exactly 2^k
# ---------------------------------------------------------------------------------------------------------------------
def test_gradients_scale_exactly_with_the_incoming_gradient():
    """Exact as long as every term the compositor adds is a multiple of the 2^-80 resolution before and after scaling,
    i.e. lies in [2^-57, 2^45) (a float32 below 2^-57 has bits below 2^-80 and is rounded).  Positive incoming gradients
    of order one keep the colour terms of every pixel block away from cancellation and inside that band for
    k = -24 .. 24."""
    dev = _dev()
    cams, ins, hw = _operator_inputs("shs", "scalerot")
    dcams = {k: v.to(dev) for k, v in cams.items()}
    bs = _settings(dcams, hw, with_depth=True)
    rng = np.random.default_rng(93)
    dL = rng.uniform(0.5, 1.0, (4, 3, *hw)).astype(np.float32)
    dLd = rng.uniform(0.5, 1.0, (4, *hw)).astype(np.float32) * np.float32(1e-2)
    base = _grads(bs, ins, dL, dLd, view_grad=True)
    top = max(float(t.abs().max()) for t in base.values())
    low = min(float(t[t != 0].abs().min()) for t in base.values() if (t != 0).any())
    for k in (-24, -8, 8, 24):
        s = 2.0 ** k
        got = _grads(bs, ins, dL * np.float32(s), dLd * np.float32(s), view_grad=True)
        for name, t in got.items():
            assert torch.equal(t, base[name] * s), (k, name)
    print(f"[determinism] 2^k scaling exact for k in -24..24 (gradients {low:.1e} .. {top:.1e} at k = 0)")


# ---------------------------------------------------------------------------------------------------------------------
# 5. non-finite incoming gradients
# ---------------------------------------------------------------------------------------------------------------------
def test_nan_reaches_the_same_gradients_as_on_the_default_path():
    dev = _dev()
    cams, ins, hw = _operator_inputs("shs", "cov3D")
    dcams = {k: v.to(dev) for k, v in cams.items()}
    bs = _settings(dcams, hw, with_depth=True)
    dL, dLd = _incoming(4, hw, seed=94)
    dL = dL.copy()
    dL[1, 0, hw[0] // 2, hw[1] // 3] = np.nan
    det = _grads(bs, ins, dL, dLd, view_grad=True)
    dflt = _default_path(lambda: _grads(bs, ins, dL, dLd, view_grad=True))
    bad = 0
    for k in det:
        a, b = torch.isfinite(det[k]), torch.isfinite(dflt[k])
        assert torch.equal(a, b), (k, int((a != b).sum()))
        bad += int((~a).sum())
    assert bad > 0
    print(f"[determinism] one NaN pixel: {bad} non-finite gradient elements, the same set as the default path's")


# ---------------------------------------------------------------------------------------------------------------------
# 6. the adapter's per-camera sums
# ---------------------------------------------------------------------------------------------------------------------
def test_adapter_camera_gradients_are_bit_identical_and_match_oracle():
    import sys
    sys.path.insert(0, au.GOLDEN)
    import make_adapter_golden as mk
    from oracle import adapter_oracle
    from pf3plat_b200.sh_rotation import sh_rotation_blocks
    from tests.test_gpu_adapter import _adapter
    b, v, h, w, deg = 1, 2, 256, 512, 4           # R = 2 * 256^2 Gaussians per camera: 1024 CTAs per camera
    inp = mk.make_inputs(17, b, v, h, w, deg)
    dmat = sh_rotation_blocks(inp["extrinsics"][..., :3, :3].reshape(b, v, 3, 3).double(), (deg + 1) ** 2)
    g = torch.Generator().manual_seed(5)
    lo = {k: t.double().requires_grad_(k != "opacities") for k, t in inp.items()}
    oo = adapter_oracle.adapter_forward(lo["extrinsics"], lo["intrinsics"], lo["coordinates"], lo["depths"],
                                        lo["opacities"], lo["raw_gaussians"], (h, w), deg, 0.5, 15.0,
                                        sh_rotation=dmat[:, :, None, None, None])
    weights = {k: torch.randn(oo[k].shape, generator=g, dtype=torch.float64) for k in au.OUTPUTS}
    sum((weights[k] * oo[k]).sum() for k in au.OUTPUTS).backward()
    dev = _dev()

    def run():
        lk = {k: t.to(dev).requires_grad_(k != "opacities") for k, t in inp.items()}
        ok = _adapter(deg).forward(lk["extrinsics"], lk["intrinsics"], lk["coordinates"], lk["depths"], lk["opacities"],
                                   lk["raw_gaussians"], (h, w), sh_rotation=dmat.float().to(dev))
        sum((weights[k].float().to(dev) * getattr(ok, k)).sum() for k in au.OUTPUTS).backward()
        return {k: lk[k].grad.detach().clone() for k in au.GRADS}

    first = run()
    for _ in range(2):
        _unrelated_work(dev)
        _assert_equal("adapter", run(), first)
    for k in au.GRADS:
        err = au.rel_err(first[k].cpu(), lo[k].grad)
        print(f"[determinism] adapter dL/d{k}: relative error to the fp64 oracle {err:.2e}")
        assert err < 1e-3, (k, err)


@pytest.mark.parametrize("name", au.CASES)
def test_adapter_matches_the_golden_fixtures(name):
    from tests.test_gpu_adapter import _run_kernels
    z, meta = au.load(name)
    _, outs, grads = _run_kernels(z, meta)
    _, _, again = _run_kernels(z, meta)
    for k in au.OUTPUTS:
        assert au.rel_err(outs[k], z["out_" + k]) < 1e-5, k
    for k in au.GRADS:
        assert torch.equal(grads[k], again[k]), k
        assert au.rel_err(grads[k], z["grad_" + k]) < 1e-3, (k, au.rel_err(grads[k], z["grad_" + k]))


# ---------------------------------------------------------------------------------------------------------------------
# 7. the whole training chain
# ---------------------------------------------------------------------------------------------------------------------
def test_training_chain_is_bit_identical():
    """adapter -> decoder_forward(depth_mode="depth") on target poses that require grad -> photometric loss + LPIPS
    with seeded weights -> backward, twice: every leaf gradient identical, nothing raises under the flag."""
    from oracle import lpips_oracle
    from pf3plat_b200 import lpips as pl
    from pf3plat_b200.adapter import GaussianAdapter, GaussianAdapterCfg
    from pf3plat_b200.losses import photometric_loss
    from pf3plat_b200.render import decoder_forward
    dev = _dev()
    b, vc, vt, chw, hw, deg = 1, 2, 3, (64, 64), (64, 64), 4
    inp = make_chain_inputs(62, b, vc, chw, vt, deg, 1.0)
    G = vc * chw[0] * chw[1]
    adapter = GaussianAdapter(GaussianAdapterCfg(gaussian_scale_min=0.5, gaussian_scale_max=15.0, sh_degree=deg)).to(dev)
    lpips = pl.LPIPS(weights=lpips_oracle.random_state_dict(3)).to(dev)
    target = make_target(b * vt, *hw, seed=8).to(dev).reshape(b, vt, 3, *hw)
    bg = torch.tensor([0.3, 0.2, 0.1], device=dev)

    def step():
        L = {k: inp[k].to(dev).requires_grad_(True) for k in ("extrinsics", "intrinsics", "coordinates", "depths",
                                                              "opacities", "raw_gaussians", "target_extrinsics")}
        g = adapter.forward(L["extrinsics"][:, :, None], L["intrinsics"][:, :, None], L["coordinates"], L["depths"],
                            L["opacities"], L["raw_gaussians"], chw)
        color, depth = decoder_forward(g.means.reshape(b, G, 3), g.covariances.reshape(b, G, 3, 3),
                                       g.harmonics.reshape(b, G, 3, -1), g.opacities.reshape(b, G),
                                       L["target_extrinsics"], inp["target_intrinsics"].to(dev), inp["near"].to(dev),
                                       inp["far"].to(dev), hw, bg, depth_mode="depth")
        mse, ssim = photometric_loss(color, target)
        loss = mse + ssim + 0.05 * lpips(color, target).mean() + 1e-3 * depth.mean()
        loss.backward()
        return float(loss), {k: t.grad.detach().clone() for k, t in L.items() if t.grad is not None}

    l0, g0 = step()
    _unrelated_work(dev)
    l1, g1 = step()
    assert l0 == l1
    assert {"extrinsics", "target_extrinsics", "raw_gaussians", "depths"} <= set(g0)
    assert float(g0["target_extrinsics"].abs().max()) > 0 and float(g0["extrinsics"].abs().max()) > 0
    _assert_equal("training chain", g1, g0)
    print(f"[determinism] training chain: loss {l0:.6f}, {len(g0)} leaf gradients bit-identical")


# ---------------------------------------------------------------------------------------------------------------------
# 8. the frame limit of the fixed-point accumulators
# ---------------------------------------------------------------------------------------------------------------------
def test_frame_above_the_term_limit_is_rejected():
    """ceil(H/4) * ceil(W/8) >= 2^21 (8192 x 8192 has exactly 2^21 pixel blocks): GS_ERR_INVALID -> ValueError."""
    dev = _dev()
    hw = (8192, 8192)
    sc = make_scene(64, 1, *hw, seed=95)
    cams, ins = scene_batch_args([sc])
    ins = {k: ins[k] for k in ("means3D", "opacities", "shs", "cov3D_precomp")}
    bs = _settings({k: v.to(dev) for k, v in cams.items()}, hw)
    from pf3plat_b200.rasterizer import rasterize_batch
    leaves = {k: v.to(dev).clone().requires_grad_(True) for k, v in ins.items()}
    color = rasterize_batch(bs, **leaves)[0]
    with pytest.raises(ValueError, match="8x4 pixel blocks"):
        color.sum().backward()
