"""The Gaussian head's fp64 oracle (tests/gaussian_head_oracle.py) against the reference's own record
(tests/golden/gaussian_head.npz, made by tests/golden/make_gaussian_head_golden.py) and against central finite
differences; the C ABI's new structs against the header; refusals that need no device."""
import ctypes
import hashlib
import os
import subprocess

import numpy as np
import pytest
import torch

from tests import gaussian_head_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "gaussian_head.npz")
Z = np.load(GOLDEN)
NAMES = [str(n) for n in Z["names"]]
CASE_KEYS = ("raw", "logits", "depths", "c2w", "K", "sh_degree", "cot_means", "cot_covariances", "cot_harmonics",
             "cot_opacities")


def case(name):
    return {k: Z[f"{name}/{k}"] for k in CASE_KEYS}


def cotangents(c):
    return {k: c["cot_" + k] for k in O.OUTPUTS}


def recorded(name, key, a):
    """`a` where the record holds it: the harmonics and dL/draw at the record's sampled pixels, the rest in full"""
    pix = Z[f"{name}/pix"]
    h, w = Z[f"{name}/raw"].shape[-2:]
    if key == "harmonics":
        return np.asarray(a)[:, np.concatenate([pix, h * w + pix])]
    if key == "d_raw":
        a = np.asarray(a)
        return a.reshape(a.shape[0], a.shape[1], h * w)[..., pix]
    return a


def close(got, ref, tol=1e-10):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    assert got.shape == ref.shape
    assert np.array_equal(np.isnan(got), np.isnan(ref))
    f = np.isfinite(ref)
    err = np.abs(got[f] - ref[f]) / (np.abs(ref[f]) + 1.0)
    assert err.max(initial=0.0) <= tol, err.max()


@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_the_reference_record(name):
    c = case(name)
    vals, grads = O.run(c, cotangents(c))
    for k in O.OUTPUTS:
        close(recorded(name, k, vals[k]), Z[f"{name}/{k}64"])
    for k in O.INPUTS:
        close(recorded(name, "d_" + k, grads[k]), Z[f"{name}/d_{k}64"])


def test_golden_cases_reach_their_regimes():
    degs = {int(Z[f"{n}/sh_degree"]) for n in NAMES}
    assert degs == {0, 1, 2, 3, 4}
    views = {Z[f"{n}/c2w"].shape[1] for n in NAMES}
    assert views == {2, 3, 4, 5, 6} and {Z[f"{n}/c2w"].shape[0] for n in NAMES} == {1, 2, 3}
    assert any(Z[f"{n}/raw"].shape[-2] == 1 for n in NAMES) and any(Z[f"{n}/raw"].shape[-1] % 4 for n in NAMES)
    # the improper rotation fails the guard: every camera rotates by the identity, so harmonics are the masked raw
    imp = case("b2_v3_4x5_d25_improper")
    rot = imp["c2w"][:, (0, -1), :3, :3].astype(np.float64)
    assert not np.allclose(np.linalg.det(rot), 1.0)
    d_sh = 25
    h, w = imp["raw"].shape[-2:]
    sh = imp["raw"].astype(np.float64).reshape(2, 2, 84, h * w)[:, :, 9:].transpose(1, 0, 3, 2).reshape(2, 2 * h * w, 3, d_sh)
    mask = np.array([1.0] + [0.1 * 0.25 ** l for l in range(1, 5) for _ in range(2 * l + 1)])
    close(recorded("b2_v3_4x5_d25_improper", "harmonics", sh * mask), Z["b2_v3_4x5_d25_improper/harmonics64"],
          tol=1e-8)  # the identity D as fitted
    # the NaN c2w entry (row 1) makes the y of scene 0's slot-0 means NaN, and nothing else of the means
    m = Z["b2_v2_4x4_d9_nan_c2w/means64"]
    assert np.isnan(m[0, :16, 1]).all() and np.isnan(m).sum() == 16
    # saturated sigmoids and NaNs in the extremes case
    e = case("b1_v3_5x6_d25_extremes")
    assert np.isnan(e["raw"]).sum() == 2 and (np.abs(e["raw"]) >= 60).sum() >= 5
    assert np.isnan(Z["b1_v3_5x6_d25_extremes/harmonics64"]).any()
    # every saturating or non-finite input pixel is among the sampled ones
    pix = set(Z["b1_v3_5x6_d25_extremes/pix"].tolist())
    bad = (~np.isfinite(e["raw"]) | (np.abs(e["raw"]) >= 15)).any(axis=(0, 1)).reshape(-1)
    assert set(np.flatnonzero(bad).tolist()) <= pix and len(pix) >= 8
    # the degenerate cases: two or more scenes, five and six views, and in different scenes or slots an exactly zero
    # raw quaternion, one whose float32 squares underflow (|q| = 0 in float32, not in fp64) and a zero depth, each at a
    # recorded pixel; the gradients there are finite, and exactly 0 on the zero quaternion
    seen = {"zero": set(), "tiny": set(), "depth": set()}
    for name in ("b2_v5_6x7_d16_degenerate", "b3_v6_3x5_d25_degenerate"):
        c = case(name)
        b, V = c["c2w"].shape[:2]
        h, w = c["raw"].shape[-2:]
        assert b >= 2 and V >= 5
        pix = set(Z[f"{name}/pix"].tolist())
        q = c["raw"][:, 5:9].reshape(2 * b, 4, h * w)
        zero = (q == 0).all(1)
        tiny = ~zero & ((q * q).sum(1, dtype=np.float32) == 0) & (np.abs(q.astype(np.float64)).max(1) > 0)
        depth = c["depths"].reshape(b * V, h * w) == 0
        assert zero.any() and tiny.any() and depth.any(), name
        for kind, m in (("zero", zero), ("tiny", tiny), ("depth", depth)):
            for i, p in np.argwhere(m):
                assert p in pix, (name, kind, p)
                seen[kind].add((name, int(i)))  # (case, conv item) or (case, scene * V + view)
        d = Z[f"{name}/d_raw64"]
        assert np.isfinite(d).all() and np.isfinite(Z[f"{name}/covariances64"]).all()
        order = Z[f"{name}/pix"].tolist()
        for i, p in np.argwhere(zero):
            assert (d[i, 5:9, order.index(p)] == 0).all()
        for i, p in np.argwhere(tiny):
            assert (d[i, 5:9, order.index(p)] != 0).any()
        # the zero depth: a zero covariance at that Gaussian
        cov = Z[f"{name}/covariances64"]
        for bv, p in np.argwhere(depth):
            bi, v = divmod(int(bv), V)
            if v in (0, V - 1):
                assert (cov[bi, (0 if v == 0 else h * w) + p] == 0).all()
    # different scenes or slots: no two kinds share a (case, item)
    assert len(seen["zero"] & seen["tiny"]) == 0 and all(seen.values())


# sha256 over (name, dtype, shape, bytes) of every array of the first eight cases, in name order, as first recorded
FIRST_CASES_SHA256 = "54c3929f668489c2c13372ba6c5d318d83886af8d87785931ae598347a269104"
FIRST_CASES = ("b1_v2_13x19_d1", "b1_v2_6x8_d25", "b1_v3_5x6_d25_extremes", "b2_v2_4x4_d9_nan_c2w", "b2_v3_1x7_d16",
               "b2_v3_4x5_d25_improper", "b2_v3_5x7_d9", "b3_v4_4x5_d4")


def test_cases_added_later_leave_the_first_cases_byte_identical():
    h = hashlib.sha256()
    keys = sorted(k for k in Z.files if k.split("/")[0] in FIRST_CASES)
    assert len(keys) == 8 * 19
    for k in keys:
        v = Z[k]
        h.update(k.encode())
        h.update(str(v.dtype).encode())
        h.update(str(v.shape).encode())
        h.update(v.tobytes())
    assert h.hexdigest() == FIRST_CASES_SHA256
    assert set(FIRST_CASES) < set(NAMES)


def test_oracle_gradient_matches_finite_differences():
    rng = np.random.default_rng(0)
    c = case("b2_v3_5x7_d9")
    cot = cotangents(c)
    _, grads = O.run(c, cot)

    def loss(cc):
        vals, _ = O.run(cc)
        return sum(float((np.asarray(cot[k], np.float64) * vals[k]).sum()) for k in O.OUTPUTS)

    for key in O.INPUTS:
        base = np.asarray(c[key], np.float64)
        flat = [tuple(int(i) for i in np.unravel_index(j, base.shape)) for j in rng.choice(base.size, 6, replace=False)]
        if key == "c2w":  # the translations: a rotation entry also moves the detached covariance and SH rotation
            flat = [(0, 0, 0, 3), (1, 2, 1, 3), (0, 2, 2, 3), (1, 1, 0, 3)]
        for idx in flat:
            eps = 1e-6 * max(1.0, abs(base[idx]))
            vals = []
            for sgn in (1, -1):
                cc = dict(c)
                a = base.copy()
                a[idx] += sgn * eps
                cc[key] = a
                vals.append(loss(cc))
            fd = (vals[0] - vals[1]) / (2 * eps)
            g = grads[key][idx]
            assert abs(fd - g) <= 1e-5 * (abs(g) + 1.0), (key, idx, fd, g)


def test_gaussian_head_structs_match_the_header(tmp_path):
    from pf3plat_b200 import _capi
    structs = ["GsGaussianHeadConfig", "GsGaussianHeadInputs", "GsGaussianHeadOutputs", "GsGaussianHeadOutGrads",
               "GsGaussianHeadInGrads"]
    fields = [(s, f) for s in structs for f, _ in getattr(_capi, s)._fields_]
    prog = tmp_path / "probe.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "gsplat_b200.h"\nint main(void){'
                    + "".join(f'printf("%zu\\n", sizeof({s}));' for s in structs)
                    + "".join(f'printf("%zu\\n", offsetof({s}, {f}));' for s, f in fields) + "return 0;}\n")
    exe = tmp_path / "probe"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    want = [ctypes.sizeof(getattr(_capi, s)) for s in structs] + [getattr(_capi, s).__dict__[f].offset for s, f in fields]
    assert got == want


def test_gaussian_head_abi_refuses_bad_arguments_without_a_device():
    from pf3plat_b200 import _capi
    L = _capi.lib()
    cfg = _capi.GsGaussianHeadConfig(batch=1, views=2, height=4, width=4, d_sh=9, scale_min=0.5, scale_max=15.0,
                                     eps=1e-8)
    assert L.gs_gaussian_head_scratch_bytes(ctypes.byref(cfg)) == 2 * 1 * 12 * 4
    assert L.gs_gaussian_head_scratch_bytes(None) == -1
    ins, out = _capi.GsGaussianHeadInputs(), _capi.GsGaussianHeadOutputs()
    gout, gin = _capi.GsGaussianHeadOutGrads(), _capi.GsGaussianHeadInGrads()
    assert L.gs_gaussian_head_forward(None, ctypes.byref(ins), ctypes.byref(out), None) == -1
    assert L.gs_gaussian_head_forward(ctypes.byref(cfg), ctypes.byref(ins), ctypes.byref(out), None) == -1  # nulls
    assert L.gs_gaussian_head_backward(ctypes.byref(cfg), ctypes.byref(ins), ctypes.byref(gout), ctypes.byref(gin),
                                       None) == -1
    for field, value in (("d_sh", 8), ("d_sh", 36), ("views", 1), ("batch", 0), ("height", 0), ("flags", 2)):
        bad = _capi.GsGaussianHeadConfig.from_buffer_copy(cfg)
        setattr(bad, field, value)
        assert L.gs_gaussian_head_scratch_bytes(ctypes.byref(bad)) == -1, field


def test_python_entry_refuses_cpu_tensors_before_any_launch():
    from pf3plat_b200.adapter import GaussianAdapterCfg
    from pf3plat_b200.gaussian_head import gaussian_head
    cfg = GaussianAdapterCfg(gaussian_scale_min=0.5, gaussian_scale_max=15.0, sh_degree=1)
    b, V, h, w = 1, 2, 3, 4
    args = (torch.zeros(2 * b, 21, h, w), torch.zeros(2 * b, 2, h, w), torch.ones(b * V, 1, h, w),
            torch.eye(4).repeat(b, V, 1, 1), torch.eye(3).repeat(b, V, 1, 1))
    with pytest.raises(TypeError, match="CUDA"):
        gaussian_head(*args, cfg, (h, w))
