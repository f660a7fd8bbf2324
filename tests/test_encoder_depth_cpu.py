"""CPU checks of the encoder depth glue: the fp64 oracle (tests/encoder_depth_oracle.py) against the reference's own
code recorded in tests/golden/encoder_depth.npz (make_encoder_depth_golden.py), values and gradients within 1e-10 and
the mono cue's one-hot exactly; the oracle's gradients against central finite differences; the float32 hypothesis table
against the reference's own expression; the regimes the golden cases reach; the C structs' layouts; and the Python
entries' refusals (no device)."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from einops import rearrange

from tests import encoder_depth_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "encoder_depth.npz")


def load_cases():
    z = np.load(GOLDEN)
    return {str(n): {k.split("/", 1)[1]: z[k] for k in z.files if k.startswith(f"{n}/")} for n in z["names"]}


CASES = load_cases()
DEPTH = sorted(n for n in CASES if n.startswith("du_"))
MONO = sorted(n for n in CASES if n.startswith("mono_"))
# every case with a recorded mono cue: the mono cases, and the depth cases whose updated depths were recorded for it
CUES = sorted(n for n in CASES if "mono_bin32" in CASES[n])
PDF = sorted(n for n in CASES if n.startswith("pdf_"))


def f64(a):
    return np.asarray(a, np.float64)


def close(a, b, tol):
    a, b = f64(a), f64(b)
    assert a.shape == b.shape
    assert np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(np.isfinite(a), np.isfinite(b))
    f = np.isfinite(b)
    err = np.abs(a[f] - b[f]) / (np.abs(b[f]) + 1.0)
    assert float(err.max(initial=0.0)) <= tol, float(err.max())


def du_args(c):
    return c["depth"], c["scale_shift"], c["intrinsics"], c["near"], c["far"], tuple(int(x) for x in c["grid"])


def at_pixels(a, c):
    """a [..., h, w] at the recorded pixel sample c["pix"] (flat indices of h w): [..., len(pix)]"""
    a = np.asarray(a)
    return a.reshape(*a.shape[:-2], -1)[..., c["pix"]]


def du_cotangents(c):
    return f64(c["g_depths"]), f64(c["g_xyz_a"]) + f64(c["g_xyz_b"])


@pytest.mark.parametrize("name", DEPTH)
def test_depth_update_oracle_matches_the_reference_record(name):
    c = CASES[name]
    depths, xyz, _ = O.depth_update_forward(*du_args(c))
    close(at_pixels(depths, c), c["depths64"], 1e-10)
    close(at_pixels(xyz, c), c["xyz64"], 1e-10)
    close(O.depth_update_backward(*du_args(c), *du_cotangents(c)), c["d_scale_shift64"], 1e-10)


@pytest.mark.parametrize("name", CUES)
def test_mono_cue_restatement_matches_the_reference_one_hot_exactly(name):
    c = CASES[name]
    b, v = c["near"].shape
    bins = O.mono_bins_f32(c["depths32"] if "depths32" in c else c["depths"], c["near"], c["far"], b, v)
    assert np.array_equal(bins, c["mono_bin32"].astype(np.int64))


@pytest.mark.parametrize("name", PDF)
def test_pdf_peak_oracle_matches_the_reference_record(name):
    c = CASES[name]
    s = int(c["upscale"])
    close(O.pdf_peak_forward(c["logits"], s), c["pdf_max64"], 1e-10)
    close(O.pdf_peak_backward(c["logits"], s, c["g_pdf"]), c["d_logits64"], 1e-10)


def test_golden_cases_reach_their_regimes():
    grids = {tuple(int(x) for x in CASES[n]["grid"]) for n in DEPTH}
    frames = {CASES[n]["depth"].shape[-2:] for n in DEPTH}
    assert {(7, 7), (28, 28), (37, 29)} <= grids and {(64, 64), (48, 80)} <= frames
    assert {CASES[n]["near"].shape for n in DEPTH} >= {(1, 2), (1, 3), (3, 2), (3, 3)}
    crossed = on_bound = across = 0
    for n in DEPTH:
        c = CASES[n]
        sraw = O.upsample_shift(c["scale_shift"], tuple(int(x) for x in c["grid"]), *c["depth"].shape[-2:])
        crossed += int((np.abs(sraw) > 5).sum())
        lo, hi = c["near"].reshape(-1, 1, 1, 1), c["far"].reshape(-1, 1, 1, 1)
        on_bound += int(((c["depth"] == lo) | (c["depth"] == hi)).sum())
        across += int(((c["depth"] < lo) | (c["depth"] > hi)).sum())
    assert crossed > 0 and on_bound > 0 and across > 0
    nan_case = CASES["du_g28_24x40_b1_v3_nan"]
    assert np.isnan(nan_case["depth"]).sum() == 1 and np.isnan(nan_case["depths64"]).sum() == 1  # in the sample
    assert set(MONO) < set(CUES) and any(n in CUES for n in DEPTH)
    for n in DEPTH:  # the sample holds rows 1 and 2, where depths lie on near and far
        h, w = CASES[n]["depth"].shape[-2:]
        assert set(range(w, 3 * w)) <= set(CASES[n]["pix"].tolist())
    for n in MONO:  # depths exactly on hypotheses, on midpoints (ties) and a NaN
        c = CASES[n]
        hyp = O.hypotheses_f32(c["near"][0, 0], c["far"][0, 0])
        dn = O.downsample4_f32(c["depths"])
        assert np.isin(dn, hyp).any() and np.isnan(dn).any()
        d = np.abs(dn[..., None] - hyp).astype(np.float32)
        srt = np.sort(d, axis=-1)
        assert (srt[..., 0] == srt[..., 1]).any()  # an exact tie between two hypotheses
    assert {int(CASES[n]["logits"].shape[1]) for n in PDF} == {32, 128}
    assert {int(CASES[n]["upscale"]) for n in PDF} == {1, 4}
    assert any(np.isnan(CASES[n]["logits"]).any() for n in PDF)


def test_depth_update_oracle_gradient_matches_finite_differences():
    rng = np.random.default_rng(3)
    b, v, h, w, grid = 1, 2, 12, 20, (5, 7)
    near, far = np.array([[1.0, 1.2]]), np.array([[6.0, 7.0]])
    depth = rng.uniform(2.0, 5.0, (b * v, 1, h, w))
    ss = np.stack([rng.normal(size=(b, v, 35)), rng.normal(0.0, 0.5, (b, v, 35))], -1)
    K = np.tile(np.array([[1.0, 0.01, 0.5], [0.0, 1.1, 0.45], [0.0, 0.0, 1.0]]), (b, v, 1, 1))
    gd, gx = rng.normal(size=(b * v, 1, h, w)), rng.normal(size=(b, v, 3, h, w))

    def loss(s):
        d, x, _ = O.depth_update_forward(depth, s, K, near, far, grid)
        return float((d * gd).sum() + (x * gx).sum())

    _, _, (sraw, pre, lo, hi) = O.depth_update_forward(depth, ss, K, near, far, grid)
    assert (np.abs(sraw) < 4.9).all() and (pre > lo + 0.01).all() and (pre < hi - 0.01).all()  # away from the clamps
    got = O.depth_update_backward(depth, ss, K, near, far, grid, gd, gx)
    eps = 1e-6
    for idx in np.ndindex(ss.shape):
        hi_, lo_ = ss.copy(), ss.copy()
        hi_[idx] += eps
        lo_[idx] -= eps
        num = (loss(hi_) - loss(lo_)) / (2 * eps)
        assert abs(num - got[idx]) <= 1e-6 * (1.0 + abs(num)), (idx, num, got[idx])


def test_pdf_peak_oracle_gradient_matches_finite_differences():
    rng = np.random.default_rng(4)
    x0 = rng.normal(0.0, 1.5, (2, 6, 3, 2))
    g = rng.normal(size=(2, 1, 6, 4))
    got = O.pdf_peak_backward(x0, 2, g)
    eps = 1e-6
    for idx in np.ndindex(x0.shape):
        hi, lo = x0.copy(), x0.copy()
        hi[idx] += eps
        lo[idx] -= eps
        num = float(((O.pdf_peak_forward(hi, 2) - O.pdf_peak_forward(lo, 2)) * g).sum() / (2 * eps))
        assert abs(num - got[idx]) <= 1e-6 * (1.0 + abs(num)), (idx, num, got[idx])


def reference_hypotheses(near, far):
    """encoder_costvolume.py:293 in float32 on the CPU, without the expand"""
    near, far = torch.tensor(near, dtype=torch.float32), torch.tensor(far, dtype=torch.float32)
    return ((1.0 / far)[0, 0].item() + torch.linspace(0.0, 1.0, 128).unsqueeze(0)
            * ((1.0 / near)[0, 0].item() - (1.0 / far)[0, 0].item())).view(-1).numpy()


def test_hypothesis_table_is_the_reference_expression_bit_for_bit():
    rng = np.random.default_rng(5)
    pairs = [(1.0, 100.0), (0.5, 1.0), (1e-3, 1e3), (0.1, 0.1000001), (3.0, 3.0)]
    pairs += [(float(a), float(a * m)) for a, m in zip(rng.uniform(0.01, 10.0, 200), rng.uniform(1.0, 1e4, 200))]
    for n, f in pairs:
        near, far = np.full((2, 3), n, np.float32), np.full((2, 3), f, np.float32)
        assert np.array_equal(O.hypotheses_f32(near[0, 0], far[0, 0]).view(np.uint32),
                              reference_hypotheses(near, far).view(np.uint32)), (n, f)


def reference_mono_cue(depths, near, far, b, v):
    """encoder_costvolume.py:292-298, restated (the CPU tests pin it to the reference's own lines)"""
    h, w = depths.shape[-2:]
    disparity_down = F.interpolate(depths, (h // 4, w // 4), mode="bilinear")
    depth_hypothesis = ((1.0 / far)[0, 0].item() + torch.linspace(0.0, 1.0, 128).unsqueeze(0).to(depths.device)
                        * ((1.0 / near)[0, 0].item() - (1.0 / far)[0, 0].item())).view(1, -1, 1, 1).expand(
        b * v, -1, h // 4, w // 4).detach()
    abs_depth_diff = torch.abs(disparity_down - depth_hypothesis)
    min_diff_index = torch.argmin(abs_depth_diff, dim=1, keepdim=True)
    pseudo_cost = depth_hypothesis.new_zeros(depth_hypothesis.shape)
    ones = depth_hypothesis.new_ones(depth_hypothesis.shape)
    return rearrange(pseudo_cost.scatter_(dim=1, index=min_diff_index, src=ones).detach(), "(b v) c h w -> (v b) c h w",
                     b=b, v=v)


@pytest.mark.parametrize("name", CUES)
def test_reference_mono_restatement_matches_the_record(name):
    if True:
        c = CASES[name]
        b, v = c["near"].shape
        d = c["depths32"] if "depths32" in c else c["depths"]
        ref = reference_mono_cue(torch.tensor(d), torch.tensor(c["near"]), torch.tensor(c["far"]), b, v)
        assert np.array_equal(ref.argmax(1).numpy(), c["mono_bin32"].astype(np.int64))


@pytest.fixture(scope="module")
def capi():
    import __graft_entry__ as ge
    ge.build()
    from pf3plat_b200 import _capi
    return _capi


def test_encoder_depth_structs_match_the_header(capi, tmp_path):
    names = ["GsDepthUpdateConfig", "GsDepthUpdateInputs", "GsDepthUpdateGrads", "GsMonoCueConfig", "GsPdfPeakConfig"]
    fields = [("GsDepthUpdateConfig", "grid_width"), ("GsDepthUpdateInputs", "far_"),
              ("GsDepthUpdateGrads", "dL_dxyz"), ("GsDepthUpdateGrads", "dL_dscale_shift"),
              ("GsMonoCueConfig", "width"), ("GsPdfPeakConfig", "upscale")]
    prog = tmp_path / "encoder_depth_sizes.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "gsplat_b200.h"\nint main(void){'
                    + "".join(f'printf("%zu\\n", sizeof({n}));' for n in names)
                    + "".join(f'printf("%zu\\n", offsetof({s}, {f}));' for s, f in fields)
                    + 'printf("%d %d\\n", (int)GS_MONO_CUE_BINS, GS_ABI_VERSION);return 0;}')
    exe = tmp_path / "encoder_depth_sizes"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
    out = [int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert [ctypes.sizeof(getattr(capi, n)) for n in names] == out[:5]
    assert [getattr(getattr(capi, s), f).offset for s, f in fields] == out[5:11]
    assert [capi.GS_MONO_CUE_BINS, capi.ABI_VERSION] == out[11:] == [128, 5]


def test_encoder_depth_abi_refuses_bad_arguments_without_a_device(capi):
    L = capi.lib()
    ins = capi.GsDepthUpdateInputs()
    for bad in (dict(batch=0), dict(views=0), dict(height=0), dict(width=0), dict(grid_height=0), dict(grid_width=0),
                dict(batch=300, views=300)):
        base = dict(batch=1, views=2, height=8, width=8, grid_height=2, grid_width=2)
        base.update(bad)
        cfg = capi.GsDepthUpdateConfig(**base)
        assert L.gs_depth_update_forward(ctypes.byref(cfg), ctypes.byref(ins), None, None, None) == -1, bad
    good = capi.GsDepthUpdateConfig(batch=1, views=2, height=8, width=8, grid_height=2, grid_width=2)
    assert L.gs_depth_update_forward(ctypes.byref(good), ctypes.byref(ins), None, None, None) == -1
    assert b"null" in L.gs_last_error()
    assert L.gs_depth_update_backward(ctypes.byref(good), ctypes.byref(ins), None, None) == -1
    for bad in (dict(height=6), dict(width=10), dict(height=0), dict(batch=0), dict(views=0)):
        base = dict(batch=1, views=2, height=8, width=8)
        base.update(bad)
        cfg = capi.GsMonoCueConfig(**base)
        assert L.gs_mono_cue(ctypes.byref(cfg), None, None, None, None, None, None) == -1, bad
    for bad in (dict(items=0), dict(depth_candidates=0), dict(height=0), dict(width=0), dict(upscale=0),
                dict(items=70000)):
        base = dict(items=2, depth_candidates=4, height=4, width=4, upscale=4)
        base.update(bad)
        cfg = capi.GsPdfPeakConfig(**base)
        assert L.gs_pdf_peak_forward(ctypes.byref(cfg), None, None, None, None, None) == -1, bad
        assert L.gs_pdf_peak_backward(ctypes.byref(cfg), None, None, None, None, None, None) == -1, bad


def test_python_entries_refuse_bad_arguments_before_any_launch():
    from pf3plat_b200 import encoder_depth as E
    nf = torch.ones(1, 2)
    with pytest.raises(RuntimeError, match="CUDA"):
        E.depth_update(torch.ones(2, 1, 8, 8), torch.zeros(1, 2, 4, 2), torch.eye(3).expand(1, 2, 3, 3), nf, nf, (2, 2))
    with pytest.raises(RuntimeError, match="CUDA"):
        E.mono_cue(torch.ones(2, 1, 8, 8), nf, nf, 1, 2)
    with pytest.raises(RuntimeError, match="CUDA"):
        E.pdf_peak(torch.zeros(2, 4, 3, 3))
