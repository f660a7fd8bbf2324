"""CPU checks of the pose-loss oracle (oracle/pose_loss_oracle.py): it reproduces the reference's own Losspose
(tests/golden/pose_loss.npz, float64 record) to 1e-10, non-finite pattern included, and its gradients agree with central
finite differences.  Also the C ABI's layout and argument checks, without a device."""
import ctypes
import hashlib
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import pose_loss_oracle as po
from tests.pose_loss_cases import GOLDEN_CASES, GRADS, NEW_GOLDEN_CASES, golden_case, load_golden, seeded_case

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# sha256 over (name, dtype, shape, bytes) of every array of the first nine cases, in name order, as first recorded
FIRST_CASES_SHA256 = "f5004fa232bdee47f76336d6cf49990d8daf5df0bb7908b0867b111f62e2b7ae"


def _oracle(case, dtype=torch.float64, eps=po.EPS_N):
    corre, conf = case.matches()
    return po.loss_and_grads(case.abspose, case.depth, case.xyz, case.K, corre, conf, case.h, case.width, dtype=dtype,
                             eps=eps)


def _same(a, b, tol, what):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape, what
    fa, fb = np.isfinite(a), np.isfinite(b)
    assert (fa == fb).all(), f"{what}: non-finite at {np.argwhere(fa != fb)[:5].tolist()}"
    assert (np.isnan(a) == np.isnan(b)).all(), what
    if fa.any():
        err = np.abs(a[fa] - b[fa]) / (np.abs(b[fa]) + 1.0)
        assert err.max() <= tol, f"{what}: worst {err.max():.3e}"


@pytest.mark.parametrize("name", GOLDEN_CASES + NEW_GOLDEN_CASES)
def test_oracle_matches_the_reference_fp64_record(name):
    z = load_golden()
    assert not z[f"{name}/f64/raises"] if f"{name}/f64/raises" in z.files else True
    out = _oracle(golden_case(z, name))
    _same(out["loss"].numpy(), z[f"{name}/f64/loss"], 1e-10, f"{name} loss")
    for k in GRADS:
        _same(out[k].numpy(), z[f"{name}/f64/grad_{k}"].reshape(out[k].shape), 1e-10, f"{name} dL/d{k}")


def test_golden_non_finite_pattern_is_the_one_the_issue_describes():
    z = load_golden()
    n = "v3_b1_nan_depth_unmatched"
    assert np.isfinite(z[f"{n}/f64/loss"])
    gd = z[f"{n}/f64/grad_depth"].reshape(3, -1)
    assert (~np.isfinite(gd)).sum() == 1 and (~np.isfinite(gd[0])).sum() == 1
    ga = z[f"{n}/f64/grad_abspose"][0]
    assert np.isfinite(ga[0]).all() and not np.isfinite(ga[1]).any() and not np.isfinite(ga[2]).any()
    assert np.isfinite(z[f"{n}/f64/grad_xyz"]).all()
    n = "v3_b1_nan_xyz_unmatched"
    assert all(np.isfinite(z[f"{n}/f64/grad_{k}"]).all() for k in GRADS)
    # view v - 1 is never a source: its depth gradient is exactly zero
    for name in GOLDEN_CASES:
        v = int(z[f"{name}/v"])
        gd = z[f"{name}/f64/grad_depth"]
        assert (gd.reshape(int(z[f"{name}/b"]), v, -1)[:, v - 1] == 0).all()


def test_oracle_float32_tracks_the_reference_float32_record():
    z = load_golden()
    for name in ("v3_b2_ragged", "v4_b3_24x24", "v2_b2_edges"):
        out = _oracle(golden_case(z, name), torch.float32)
        _same(out["loss"].numpy(), z[f"{name}/f32/loss"], 1e-5, f"{name} f32 loss")


# v2_b2_edges is left out: its point near u_z = -1e-6 is too curved for a finite difference
@pytest.mark.parametrize("name", ["v3_b2_ragged", "v4_b3_24x24", "v4_b1_zero_weights"])
def test_oracle_gradients_match_central_differences(name):
    z = load_golden()
    case = golden_case(z, name)
    out = _oracle(case)
    corre, conf = case.matches()
    b, v = case.b, case.v
    g = torch.Generator().manual_seed(7)

    def loss_with(**over):
        args = dict(abspose=case.abspose.double(), depth=case.depth.double(), xyz=case.xyz.double())
        args.update(over)
        wt = over.get("w", case.w.double())
        cf = over.get("conf", case.conf.double())
        cr, cn = case.matches(w=wt, conf=cf)
        return float(po.pose_loss(args["abspose"], args["depth"], args["xyz"], case.K.double(), cr, cn, case.h,
                                  case.width))

    base = {"abspose": case.abspose.double(), "depth": case.depth.double(), "xyz": case.xyz.double(),
            "w": case.w.double(), "conf": case.conf.double()}
    for k in GRADS:
        t = base[k]
        if t.numel() == 0:
            continue
        # the matched elements carry the gradient: probe those and a few random ones
        nz = torch.nonzero(out[k].reshape(-1)).reshape(-1)
        probe = torch.cat([nz[torch.randperm(len(nz), generator=g)[:6]], torch.randint(0, t.numel(), (2,), generator=g)])
        for j in probe.tolist():
            if k == "w" and float(t.reshape(-1)[j]) == 0.0:
                continue  # |w| has a kink at 0
            eps = 1e-6 * max(1.0, abs(float(t.reshape(-1)[j])))
            tp, tm = t.clone(), t.clone()
            tp.view(-1)[j] += eps
            tm.view(-1)[j] -= eps
            fd = (loss_with(**{k: tp}) - loss_with(**{k: tm})) / (2 * eps)
            an = float(out[k].reshape(-1)[j])
            assert abs(fd - an) <= 1e-5 * max(1.0, abs(an)), f"{name} dL/d{k}[{j}]: fd {fd} vs autograd {an}"


def test_seeded_cases_pack_like_the_reference_order():
    case = seeded_case(2, 3, 8, 10, 0, 5, seed=1)
    corre, conf = case.matches()
    sid, id_a, id_c, w, cf = po.pack(corre, conf, case.b, case.v)
    assert torch.equal(id_a, case.id_a) and torch.equal(id_c, case.id_c)
    assert sid.tolist() == [s for s, n in enumerate(case.counts) for _ in range(n)]
    assert torch.equal(cf, case.conf.reshape(-1))


@pytest.fixture(scope="module")
def capi():
    import __graft_entry__ as ge
    ge.build()
    from pf3plat_b200 import _capi
    return _capi


def test_pose_loss_structs_match_the_header(capi, tmp_path):
    names = ["GsPoseLossConfig", "GsPoseLossInputs", "GsPoseLossGrads"]
    prog = tmp_path / "sizes.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "gsplat_b200.h"\nint main(void){'
                    + "".join(f'printf("%zu\\n", sizeof({n}));' for n in names)
                    + 'printf("%zu\\n", offsetof(GsPoseLossConfig, matches));'
                    + 'printf("%zu\\n", offsetof(GsPoseLossInputs, xyz));return 0;}')
    exe = tmp_path / "sizes"
    subprocess.run(["/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc", "-I", os.path.join(ROOT, "include"),
                    str(prog), "-o", str(exe)], check=True)
    out = [int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert [ctypes.sizeof(getattr(capi, n)) for n in names] == out[:3]
    assert capi.GsPoseLossConfig.matches.offset == out[3] and capi.GsPoseLossInputs.xyz.offset == out[4]


def test_pose_loss_entries_refuse_bad_arguments_without_a_device(capi):
    L = capi.lib()
    assert L.gs_pose_loss_forward(None, None, None, None, None) == -1
    assert L.gs_pose_loss_backward(None, None, None, None, None, None, None) == -1
    bad = capi.GsPoseLossConfig(batch=2, views=3, height=4, width=4, segments=5, matches=0)  # 2 scenes x 3 pairs
    assert L.gs_pose_loss_scratch_bytes(ctypes.byref(bad)) == -1
    good = capi.GsPoseLossConfig(batch=2, views=3, height=4, width=4, segments=6, matches=10)
    assert L.gs_pose_loss_forward(ctypes.byref(good), ctypes.byref(capi.GsPoseLossInputs()), None, None, None) == -1
    assert b"null" in L.gs_last_error()


def test_cases_added_later_leave_the_first_cases_byte_identical():
    z = load_golden()
    h = hashlib.sha256()
    keys = sorted(k for k in z.files if k.split("/")[0] in GOLDEN_CASES)
    assert len(keys) == 225
    for k in keys:
        v = z[k]
        h.update(k.encode())
        h.update(str(v.dtype).encode())
        h.update(str(v.shape).encode())
        h.update(v.tobytes())
    assert h.hexdigest() == FIRST_CASES_SHA256
    assert {k.split("/")[0] for k in z.files} == set(GOLDEN_CASES + NEW_GOLDEN_CASES)
    # the reference's .inverse() of a non-finite pose returns NaN on the CPU rather than raising: every case is recorded
    assert not any(bool(z[f"{n}/{t}/raises"]) for n in NEW_GOLDEN_CASES for t in ("f32", "f64"))


def _seg_weights(z, name):
    off = np.concatenate([[0], np.cumsum(z[f"{name}/counts"])])
    return [z[f"{name}/w"][off[s]:off[s + 1]] for s in range(len(off) - 1)]


def _nonfinite_per_view(z, name, k):
    b, v = int(z[f"{name}/b"]), int(z[f"{name}/v"])
    return (~np.isfinite(z[f"{name}/f64/grad_{k}"].reshape(b, v, -1))).sum(-1).tolist()


def test_new_cases_are_in_the_regime_they_were_built_for():
    z = load_golden()
    fin = lambda n, k: bool(np.isfinite(z[f"{n}/f64/{k}"]).all())  # noqa: E731
    # five and six views: ragged, with an empty and a single-match segment, every record finite
    for n, (b, v) in (("v5_b2_ragged", (2, 5)), ("v6_b1_ragged", (1, 6))):
        assert (int(z[f"{n}/b"]), int(z[f"{n}/v"])) == (b, v)
        assert 0 in z[f"{n}/counts"] and 1 in z[f"{n}/counts"] and len(set(z[f"{n}/counts"].tolist())) > 3
        assert all(fin(n, k) for k in ["loss"] + [f"grad_{g}" for g in GRADS])
    # signed weights: all negative, mixed, a zero among nonzero ones
    w = _seg_weights(z, "v3_b1_signed_weights")
    assert (w[0] < 0).all() and (w[1] < 0).any() and (w[1] > 0).any() and (w[2] == 0).sum() == 1 and (w[2] > 0).sum() > 1
    assert fin("v3_b1_signed_weights", "grad_w") and (z["v3_b1_signed_weights/f64/grad_w"] != 0).all()
    # the clamp: |w| sums exactly at float32(1e-12), at its float32 neighbours, several tiny weights below it
    n = "v3_b2_clamp"
    w = _seg_weights(z, n)
    e = np.float32(1e-12)
    assert [len(x) for x in w[:3]] == [1, 1, 1] and len(w[5]) == 1 and len(w[3]) > 2
    assert w[0][0] == e and w[1][0] == np.nextafter(e, np.float32(1)) and w[2][0] == np.nextafter(e, np.float32(0))
    assert w[5][0] == -e and float(np.abs(w[3].astype(np.float64)).sum()) < 0.2 * float(e) and (w[4] > 0.1).all()
    case = golden_case(z, n)
    corre, _ = case.matches()
    assert not po.clamp_fragile(corre, case.b, case.v).any()
    # NaN and Inf weights and confidences, each in its own segment; segment 5 is clean
    n = "v3_b2_nonfinite_weights_conf"
    w, cf = _seg_weights(z, n), z[f"{n}/conf"].reshape(-1)
    assert np.isnan(w[0]).sum() == 1 and np.isinf(w[1]).sum() == 1 and np.isnan(cf[2]) and np.isinf(cf[3])
    assert cf[4] == 0 and sum((~np.isfinite(x)).sum() for x in w) == 2 and np.isfinite(cf[[0, 1, 4, 5]]).all()
    assert np.isnan(z[f"{n}/f64/loss"]) and fin(n, "grad_depth")
    gw = z[f"{n}/f64/grad_w"]
    off = np.concatenate([[0], np.cumsum(z[f"{n}/counts"])])
    assert np.isnan(gw[:off[4]]).all() and (gw[off[4]:off[5]] == 0).all() and np.isfinite(gw[off[5]:]).all()
    assert np.flatnonzero(~np.isfinite(z[f"{n}/f64/grad_conf"])).tolist() == [0, 1]
    # a non-finite K of the last view, only ever a target: the 2-D term of its pairs, and their dense projection
    n = "v3_b2_nonfinite_K"
    assert not np.isfinite(z[f"{n}/K"][:, 2]).all(axis=(1, 2)).any() and np.isfinite(z[f"{n}/K"][:, :2]).all()
    assert _nonfinite_per_view(z, n, "depth") == [[320, 320, 0]] * 2 and fin(n, "grad_xyz") and fin(n, "grad_w")
    # a non-finite pose of view 0 enters no T: everything finite and its gradient exactly zero
    n = "v3_b2_nonfinite_pose0"
    assert not np.isfinite(z[f"{n}/abspose"][:, 0]).all(axis=(1, 2)).any()
    assert all(fin(n, k) for k in ["loss"] + [f"grad_{g}" for g in GRADS])
    assert (z[f"{n}/f64/grad_abspose"][:, 0] == 0).all()
    # a non-finite pose of view 1 goes through .inverse(): scene 0's pairs through view 1 are NaN, scene 1 is clean
    n = "v3_b2_nonfinite_pose1"
    assert _nonfinite_per_view(z, n, "abspose") == [[0, 16, 16], [0, 0, 0]]
    assert _nonfinite_per_view(z, n, "depth") == [[320, 320, 0], [0, 0, 0]]
    assert np.isfinite(z[f"{n}/f64/grad_xyz"][1]).all() and np.flatnonzero(~np.isfinite(z[f"{n}/f64/grad_conf"])).tolist() == [0, 2]
    for n, hw in (("v3_b1_1x37", (1, 37)), ("v3_b1_37x1", (37, 1))):
        assert (int(z[f"{n}/height"]), int(z[f"{n}/width"])) == hw and fin(n, "grad_depth") and fin(n, "grad_xyz")


def test_the_clamp_is_where_the_float32_and_float64_records_disagree():
    """A single weight of exactly float32(1e-12) passes the float32 clamp (equality) and is clamped in float64, so
    dL/dw there is 0 in the float32 record and ~1e9 in the float64 one.  Everywhere else the records agree; the oracle
    with EPS_N_F32 reproduces the float32 answer there and the float64 record elsewhere."""
    z = load_golden()
    n = "v3_b2_clamp"
    g32, g64 = z[f"{n}/f32/grad_w"].astype(np.float64), z[f"{n}/f64/grad_w"]
    off = np.concatenate([[0], np.cumsum(z[f"{n}/counts"])])
    at = [off[0], off[5]]  # the weights +float32(1e-12) and -float32(1e-12)
    assert (g32[at] == 0).all() and (np.abs(g64[at]) > 1e9).all()
    rest = np.setdiff1d(np.arange(len(g64)), at)
    assert (np.abs(g32[rest] - g64[rest]) <= 1e-5 * np.abs(g64[rest]) + 1e-9).all()
    assert (np.abs(g64[off[2]:off[4]]) > 1e9).all() and g64[off[1]] == 0  # clamped below, unclamped above
    out = _oracle(golden_case(z, n), eps=po.EPS_N_F32)["w"].numpy()
    assert (np.abs(out[at]) <= 1e-3).all()
    # the clamped segments divide by float32(1e-12) instead of 1e-12: 4e-9 apart
    _same(out[rest], g64[rest], 5e-9, f"{n} dL/dw, eps = float32(1e-12)")
    for k in ("abspose", "depth", "xyz", "conf"):
        o = _oracle(golden_case(z, n), eps=po.EPS_N_F32)[k].numpy()
        _same(o, z[f"{n}/f32/grad_{k}"].reshape(o.shape), 1e-5, f"{n} dL/d{k} vs f32")


def test_terms_and_grads_takes_per_segment_cotangents_and_treats_an_absent_term_as_zero():
    z = load_golden()
    case = golden_case(z, "v3_b2_nonfinite_weights_conf")
    corre, conf = case.matches()
    S = case.b * 3
    args = (case.abspose, case.depth, case.xyz, case.K, corre, conf, case.h, case.width)
    g3 = torch.linspace(-1, 2, S, dtype=torch.float64)
    g2 = torch.linspace(3, -0.5, S, dtype=torch.float64)
    full = po.terms_and_grads(*args, g3, g2)
    # the uniform cotangent of the loss's two means is loss_and_grads
    ref = po.loss_and_grads(*args, eps=po.EPS_N_F32)
    uni = po.terms_and_grads(*args, torch.full((S,), 0.025 / S, dtype=torch.float64),
                             torch.full((S,), 0.005 / S, dtype=torch.float64))
    for k in GRADS:
        _same(uni[k].numpy(), ref[k].numpy(), 1e-12, k)
    # gradients are linear in the cotangents, NaN pattern aside
    only3, only2 = po.terms_and_grads(*args, g3, None), po.terms_and_grads(*args, None, g2)
    for k in GRADS:
        a, b = (only3[k] + only2[k]).numpy(), full[k].numpy()
        f = np.isfinite(b)
        assert (np.isfinite(a) == f).all(), k  # an Inf of one term and a NaN of the other are both non-finite
        _same(a[f], b[f], 1e-12, k)
    # an absent term is a zero cotangent through the chain: the NaN-confidence segment's 0 x NaN reaches its weights
    zero3 = po.terms_and_grads(*args, torch.zeros(S, dtype=torch.float64), g2)
    off = np.concatenate([[0], np.cumsum(case.counts)])
    for k in GRADS:
        assert torch.equal(zero3[k].isnan(), only2[k].isnan()), k
        assert torch.equal(torch.nan_to_num(zero3[k]), torch.nan_to_num(only2[k])), k
    assert torch.isnan(only2["w"][off[2]:off[3]]).all() and torch.isfinite(only2["w"][off[4]:]).all()


def test_config_check_refuses_index_widths_past_int32(capi):
    L = capi.lib()
    ok = capi.GsPoseLossConfig(batch=1, views=2, height=4, width=4, segments=1, matches=2 ** 30 - 1)
    big_m = capi.GsPoseLossConfig(batch=1, views=2, height=4, width=4, segments=1, matches=2 ** 30)
    big_px = capi.GsPoseLossConfig(batch=2, views=2, height=32768, width=32768, segments=2, matches=1)  # 2^31 pixels
    edge_px = capi.GsPoseLossConfig(batch=1, views=2, height=32768, width=32767, segments=1, matches=1)
    assert L.gs_pose_loss_scratch_bytes(ctypes.byref(big_m)) == -1
    assert L.gs_pose_loss_scratch_bytes(ctypes.byref(big_px)) == -1
    assert L.gs_pose_loss_forward(ctypes.byref(big_m), None, None, None, None) == -1 and b"Config" in L.gs_last_error()
    assert L.gs_pose_loss_backward(ctypes.byref(big_px), None, None, None, None, None, None) == -1
    # the largest accepted sizes pass the config check and stop at the null inputs instead
    for cfg in (ok, edge_px):
        assert L.gs_pose_loss_forward(ctypes.byref(cfg), ctypes.byref(capi.GsPoseLossInputs()), None, None, None) == -1
        assert b"null" in L.gs_last_error()
