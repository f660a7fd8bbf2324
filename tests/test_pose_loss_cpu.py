"""CPU checks of the pose-loss oracle (oracle/pose_loss_oracle.py): it reproduces the reference's own Losspose
(tests/golden/pose_loss.npz, float64 record) to 1e-10, non-finite pattern included, and its gradients agree with central
finite differences.  Also the C ABI's layout and argument checks, without a device."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import pose_loss_oracle as po
from tests.pose_loss_cases import GOLDEN_CASES, GRADS, golden_case, load_golden, seeded_case

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _oracle(case, dtype=torch.float64):
    corre, conf = case.matches()
    return po.loss_and_grads(case.abspose, case.depth, case.xyz, case.K, corre, conf, case.h, case.width, dtype=dtype)


def _same(a, b, tol, what):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape, what
    fa, fb = np.isfinite(a), np.isfinite(b)
    assert (fa == fb).all(), f"{what}: non-finite at {np.argwhere(fa != fb)[:5].tolist()}"
    assert (np.isnan(a) == np.isnan(b)).all(), what
    if fa.any():
        err = np.abs(a[fa] - b[fa]) / (np.abs(b[fa]) + 1.0)
        assert err.max() <= tol, f"{what}: worst {err.max():.3e}"


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_oracle_matches_the_reference_fp64_record(name):
    z = load_golden()
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
