"""CPU checks of the pose path: the fp64 oracle (tests/poses_oracle.py) and the benchmark's PyTorch restatement of the
reference (scripts/bench_poses.py) against the reference's own functions recorded in tests/golden/poses.npz
(make_poses_golden.py), with the cases recorded first held byte-identical; the oracle's refine_poses gradient against
central finite differences; the regimes the golden cases are meant to reach; the C ABI's struct layouts and argument checks, and the Python entries' refusals (no device)."""
import ctypes
import hashlib
import importlib.util
import os
import subprocess

import numpy as np
import pytest
import torch

from tests import poses_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "poses.npz")


def load_cases():
    z = np.load(GOLDEN)
    return {str(n): {k.split("/", 1)[1]: z[k] for k in z.files if k.startswith(f"{n}/")} for n in z["names"]}


CASES = load_cases()
SYNC = sorted(n for n in CASES if n.startswith("sync"))
# refine cases with cotangents on both outputs; the refine_degenerate_* cases take cotangents on abspose only, and
# record whether the reference's .inverse() raised
REFINE = sorted(n for n in CASES if n.startswith("refine") and "g_inv" in CASES[n])
REFINE_DEGENERATE = sorted(n for n in CASES if n.startswith("refine_degenerate"))
PLUCKER = sorted(n for n in CASES if n.startswith("plucker"))
# the reference chains these (N = 2, or the batch fallback)
CHAINED = {"sync_n2", "sync_all_zero", "sync_one_zero_mass", "sync_chain_n16"}
# synchronised blocks that are not full rank, or masses that are not positive: their regimes are asserted one by one
DEGENERATE_SYNC = {"sync_rank2", "sync_rank0", "sync_negative_conf"}
# sha256 over (name, dtype, shape, bytes) of every array of the first sixteen cases, in name order, as first recorded
FIRST_CASES_SHA256 = "2cff2f0942fcd449bbbc875f312a27787f1adebe26ceb6b13b2cf4b176164c27"
FIRST_CASES = ("plucker_13x22", "plucker_8x8", "refine_gamma0", "refine_gamma1", "refine_v5_large_t", "sync_all_zero",
               "sync_large_t", "sync_n2", "sync_n3", "sync_n4", "sync_n5", "sync_n8", "sync_nan_conf",
               "sync_one_zero_mass", "sync_pnp_fail", "sync_relu_zero_02")


def keys_of(case):
    return [tuple(int(x) for x in k) for k in case["keys"]]


def sync_oracle(case):
    return O.camera_synchronization(keys_of(case), case["Ps"], case["conf"], int(case["N"]))


def close(a, b, tol):
    assert a.shape == b.shape
    assert np.array_equal(np.isfinite(a), np.isfinite(b))
    f = np.isfinite(b)
    err = np.abs(a[f] - b[f]) / (np.abs(b[f]) + 1.0)
    assert float(err.max(initial=0.0)) <= tol, float(err.max())


@pytest.mark.parametrize("name", SYNC)
def test_sync_oracle_matches_the_reference_record(name):
    case = CASES[name]
    if case["raises64"]:
        assert case["raises32"]  # the reference raises from torch.svd; the oracle defines NaN for that scene instead
        out = sync_oracle(case)
        bad = ~np.isfinite(case["conf"]).all(axis=0)
        assert np.isnan(out[bad]).all() and np.isfinite(out[~bad]).all()
        return
    close(sync_oracle(case), case["value64"], 1e-10)


@pytest.mark.parametrize("name", REFINE)
def test_refine_oracle_matches_the_reference_record(name):
    c = CASES[name]
    A, Ai, _ = O.refine_forward(c["pose_enc"], c["delta"], c["gamma"])
    close(A, c["abspose64"], 1e-10)
    close(Ai, c["abspose_inv64"], 1e-10)
    gp, gd, gg = O.refine_backward(c["pose_enc"], c["delta"], c["gamma"], c["g_abs"], c["g_inv"])
    close(gp, c["d_pose_enc64"], 1e-10)
    close(gd, c["d_delta64"], 1e-10)
    close(np.array(gg), c["d_gamma64"], 1e-10)


def singular_items(c):
    """[b, v] True where the refined abspose is exactly singular (a zero 6-d half: b1 or b2 is 0)"""
    _, _, f = O.refine_forward(c["pose_enc"], c["delta"], c["gamma"])
    return (f["n1"][..., 0] == 0) | (f["n2"][..., 0] == 0)


@pytest.mark.parametrize("name", REFINE_DEGENERATE)
def test_refine_oracle_matches_the_reference_record_on_degenerate_encodings(name):
    c = CASES[name]
    A, Ai, _ = O.refine_forward(c["pose_enc"], c["delta"], c["gamma"])
    close(A, c["abspose64"], 1e-10)
    sing = singular_items(c)
    assert bool(c["raises64"]) == bool(c["raises32"]) == bool(sing.any())
    if c["raises64"]:  # the reference's .inverse() raises; the oracle's inverse is NaN on the singular items only
        assert np.isnan(Ai[sing]).all() and np.isfinite(Ai[~sing]).all()
    else:
        close(Ai, c["abspose_inv64"], 1e-10)
    # gradients near the eps clamp are ~1e12 and cancel to ~0 in places: held relative to |ref| + rms ref
    gp, gd, gg = O.refine_backward(c["pose_enc"], c["delta"], c["gamma"], c["g_abs"], None)
    for got, ref in ((gp, c["d_pose_enc64"]), (gd, c["d_delta64"]), (np.array(gg), c["d_gamma64"])):
        assert got.shape == ref.shape and np.isfinite(got).all() and np.isfinite(ref).all()
        rms = float(np.sqrt((ref ** 2).mean()))
        assert (np.abs(got - ref) <= 1e-10 * (np.abs(ref) + rms) + 1e-300).all(), name


def test_cases_added_later_leave_the_first_cases_byte_identical():
    z = np.load(GOLDEN)
    h = hashlib.sha256()
    keys = sorted(k for k in z.files if k.split("/")[0] in FIRST_CASES)
    assert len(keys) == 145
    for k in keys:
        v = z[k]
        h.update(k.encode())
        h.update(str(v.dtype).encode())
        h.update(str(v.shape).encode())
        h.update(v.tobytes())
    assert h.hexdigest() == FIRST_CASES_SHA256
    assert set(FIRST_CASES) < set(CASES)


@pytest.mark.parametrize("name", PLUCKER)
def test_plucker_oracle_matches_the_reference_record(name):
    c = CASES[name]
    close(O.plucker_rays(c["abspose"], c["intrinsics"], int(c["h"]), int(c["w"])), c["value64"], 1e-10)


def load_bench():
    spec = importlib.util.spec_from_file_location("bench_poses", os.path.join(ROOT, "scripts", "bench_poses.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_bench_restatement_matches_the_reference_record():
    B = load_bench()
    d = torch.float64
    for name in SYNC:
        c = CASES[name]
        if c["raises64"]:
            continue
        keys = keys_of(c)
        Ps = {k: torch.tensor(c["Ps"][q], dtype=d) for q, k in enumerate(keys)}
        conf = {k: torch.tensor(c["conf"][q], dtype=d) for q, k in enumerate(keys)}
        # the reference's op sequence ends in float32 (and chains in float32); the record is float64 throughout
        close(B.reference_sync(Ps, conf, int(c["N"])).numpy(), c["value64"], 1e-6)
    for name in REFINE:
        c = CASES[name]
        A, Ai = B.reference_refine(*(torch.tensor(c[k], dtype=d) for k in ("pose_enc", "delta", "gamma")))
        close(A.numpy(), c["abspose64"], 1e-10)
        close(Ai.numpy(), c["abspose_inv64"], 1e-10)
    for name in PLUCKER:
        c = CASES[name]
        out = B.reference_plucker(torch.tensor(c["abspose"], dtype=d), torch.tensor(c["intrinsics"], dtype=d),
                                  int(c["h"]), int(c["w"]))
        close(out.numpy(), c["value64"], 1e-10)


@pytest.mark.parametrize("name", REFINE)
def test_refine_oracle_gradient_matches_finite_differences(name):
    c = CASES[name]
    p0, d0, g0 = (np.asarray(c[k], dtype=np.float64) for k in ("pose_enc", "delta", "gamma"))
    ga, gi = np.asarray(c["g_abs"], np.float64), np.asarray(c["g_inv"], np.float64)

    def loss(p, d, g):
        A, Ai, _ = O.refine_forward(p, d, g)
        return float((A * ga).sum() + (Ai * gi).sum())

    gp, gd, gg = O.refine_backward(p0, d0, g0, ga, gi)
    eps = 1e-6
    for arr, grad in ((p0, gp), (d0, gd)):
        for idx in np.ndindex(arr.shape):
            hi, lo = arr.copy(), arr.copy()
            hi[idx] += eps
            lo[idx] -= eps
            args_hi = (hi, d0, g0) if arr is p0 else (p0, hi, g0)
            args_lo = (lo, d0, g0) if arr is p0 else (p0, lo, g0)
            num = (loss(*args_hi) - loss(*args_lo)) / (2 * eps)
            assert abs(num - grad[idx]) <= 1e-5 * (1.0 + abs(num)), (idx, num, grad[idx])
    num = (loss(p0, d0, g0 + eps) - loss(p0, d0, g0 - eps)) / (2 * eps)
    assert abs(num - gg) <= 1e-5 * (1.0 + abs(num))


def test_golden_cases_reach_their_regimes():
    Ns = {int(CASES[n]["N"]) for n in SYNC}
    assert {2, 3, 4, 5, 8} <= Ns
    for name in SYNC:
        c = CASES[name]
        keys, N = keys_of(c), int(c["N"])
        if N == 2 or c["raises64"]:
            continue
        blk, bad = O.power_column_block(keys, np.asarray(c["Ps"], np.float64), np.asarray(c["conf"], np.float64), N)
        mass = blk[..., 3, 3]
        if name in CHAINED:
            assert np.min(mass) == 0  # the batch falls back to chaining
            continue
        if name in DEGENERATE_SYNC:
            continue
        assert np.min(mass) > 0 and not bad.any()
        # the polar factor is unique: full rank, and an improper block's smallest singular value is not repeated
        M = blk[..., :3, :3] / mass[..., None, None]
        sv = np.linalg.svd(M, compute_uv=False)
        assert (sv[..., 2] > 1e-3 * sv[..., 0]).all(), name
        improper = np.linalg.det(M) < 0
        assert (sv[..., 1] - sv[..., 2] > 1e-3 * sv[..., 0])[improper].all(), name
    # PnP failures are identity pairs; the relu rescale zeroes a (0, 2) confidence
    assert np.array_equal(CASES["sync_pnp_fail"]["Ps"][0, 0], np.eye(4))
    assert (CASES["sync_relu_zero_02"]["conf"][keys_of(CASES["sync_relu_zero_02"]).index((0, 2))] == 0).all()
    # all-zero confidences chain the batch; one zero-mass scene chains the healthy ones next to it too
    assert (CASES["sync_all_zero"]["conf"] == 0).all()
    c = CASES["sync_one_zero_mass"]
    assert (c["conf"][:, 1] == 0).all() and (c["conf"][:, [0, 2]] > 0).all()
    chained = O.camera_chaining(keys_of(c), np.asarray(c["Ps"], np.float64), 3)
    close(c["value64"], chained, 1e-10)
    # NaN confidence: the reference raises in both precisions
    assert CASES["sync_nan_conf"]["raises64"] and np.isnan(CASES["sync_nan_conf"]["conf"]).any()
    assert np.abs(CASES["sync_large_t"]["Ps"][..., :3, 3]).max() > 100
    assert float(CASES["refine_gamma0"]["gamma"]) == 0.0 and float(CASES["refine_gamma1"]["gamma"]) == 1.0
    assert not CASES["refine_gamma0"]["d_delta64"].any()  # gamma 0: no gradient reaches delta
    assert np.abs(CASES["refine_v5_large_t"]["pose_enc"][..., 6:]).max() > 100
    assert (CASES["plucker_13x22"]["h"], CASES["plucker_13x22"]["w"]) == (13, 22)


def sync_regime(name, l_dtype=np.float64):
    c = CASES[name]
    keys, N = keys_of(c), int(c["N"])
    blk, bad = O.power_column_block(keys, c["Ps"], c["conf"], N, l_dtype=l_dtype)
    return c, keys, N, blk, bad


def test_cases_added_later_reach_their_regimes():
    # pair graphs: only the chain; the chain and one pair with i > j; every pair in a shuffled order, some reversed
    c, keys, N, _, _ = sync_regime("sync_sparse_path_n6")
    assert N == 6 and keys == [(k, k + 1) for k in range(5)] and len(keys) < N * (N - 1) // 2
    c, keys, N, _, _ = sync_regime("sync_sparse_ring_n5")
    assert N == 5 and len(keys) == 5 < N * (N - 1) // 2 and (4, 0) in keys
    for name, N in (("sync_shuffled_n8", 8), ("sync_n16", 16), ("sync_chain_n16", 16)):
        c, keys, n, _, _ = sync_regime(name)
        assert n == N and len(keys) == N * (N - 1) // 2 == len({tuple(sorted(k)) for k in keys})
    for name in ("sync_shuffled_n8", "sync_chain_n16"):  # the chain pairs are not where lexicographic order puts them
        keys = keys_of(CASES[name])
        assert keys != sorted(keys)
        assert [keys.index((k, k + 1)) for k in range(int(CASES[name]["N"]) - 1)] != \
            [sorted(keys).index((k, k + 1)) for k in range(int(CASES[name]["N"]) - 1)]
    assert any(i > j for i, j in keys_of(CASES["sync_shuffled_n8"]))
    # chaining at N = 16: one zero-mass scene, so the healthy scene is chained through 15 pairs too
    c, keys, N, blk, _ = sync_regime("sync_chain_n16")
    mass = blk[..., 3, 3]
    assert (c["conf"][:, 1] == 0).all() and (mass[1] == 0).all() and (mass[0] > 0).all()
    close(c["value64"], O.camera_chaining(keys, np.asarray(c["Ps"], np.float64), N), 1e-10)
    # a NaN scene and a zero-mass scene: the NaN mass keeps the batch from chaining; the reference raises
    c, keys, N, blk, bad = sync_regime("sync_nan_and_zero_mass")
    assert c["raises64"] and c["raises32"] and list(bad) == [False, True, False]
    assert (blk[2, :, 3, 3] == 0).all() and (blk[0, :, 3, 3] > 0).all()
    out = O.camera_synchronization(keys, c["Ps"], c["conf"], N)
    assert np.isnan(out[1]).all() and np.isfinite(out[[0, 2]]).all()
    assert not np.allclose(out[0], O.camera_chaining(keys, np.asarray(c["Ps"], np.float64), N)[0])
    # a negative confidence: one mass ends negative, below the 1e-9 clamp, and the batch is not chained
    for l_dtype in (np.float64, np.float32):
        c, keys, N, blk, bad = sync_regime("sync_negative_conf", l_dtype)
        mass = blk[..., 3, 3]
        assert (c["conf"] < 0).any() and not bad.any() and mass.min() < 0 and (mass[0] > 0).all()
    assert np.isfinite(c["value64"]).all() and np.isfinite(c["value32"]).all()
    # rotation blocks of exact rank 2 (the zeroed axis differs per scene) and exact rank 0, with positive masses
    for name, rank in (("sync_rank2", 2), ("sync_rank0", 0)):
        for l_dtype in (np.float64, np.float32):
            c, keys, N, blk, bad = sync_regime(name, l_dtype)
            mass = blk[..., 3, 3]
            assert (mass > 0).all() and not bad.any()
            sv = np.linalg.svd(blk[..., :3, :3] / mass[..., None, None], compute_uv=False)
            assert (sv[..., 2] == 0).all(), name  # sigma_min == 0 exactly
            assert ((sv[..., 1] > 0.1) if rank == 2 else (sv[..., 0] == 0)).all(), name
    kmin = [np.flatnonzero(np.diag(sync_regime("sync_rank2")[3][s, 1, :3, :3]) == 0) for s in range(3)]
    assert [list(k) for k in kmin] == [[2], [1], [0]]
    assert np.array_equal(CASES["sync_rank0"]["value64"][..., :3, :3], np.broadcast_to(np.eye(3), (2, 4, 3, 3)))
    # degenerate 6-d encodings, each in its own case: at scene 0 view 0 and at the last scene's last view
    n = {}
    for name in REFINE_DEGENERATE:
        c = CASES[name]
        _, _, f = O.refine_forward(c["pose_enc"], c["delta"], c["gamma"])
        b, v = c["pose_enc"].shape[:2]
        n[name] = (f["n1"][..., 0][[0, b - 1], [0, v - 1]], f["n2"][..., 0][[0, b - 1], [0, v - 1]])
        assert "g_inv" not in c
    assert (n["refine_degenerate_a1_zero"][0] == 0).all()
    assert ((n["refine_degenerate_a1_tiny"][0] > 0) & (n["refine_degenerate_a1_tiny"][0] < 1e-12)).all()
    assert (n["refine_degenerate_a2_parallel"][1] == 0).all()  # a2 = 2 a1: c is exactly 0
    assert ((n["refine_degenerate_c_above_eps"][1] > 1e-12) & (n["refine_degenerate_c_above_eps"][1] < 2e-12)).all()
    assert ((n["refine_degenerate_c_below_eps"][1] > 0) & (n["refine_degenerate_c_below_eps"][1] < 1e-12)).all()
    assert CASES["refine_degenerate_v1"]["pose_enc"].shape[1] == 1
    assert float(CASES["refine_degenerate_negative_gamma"]["gamma"]) < 0
    assert [n for n in REFINE_DEGENERATE if CASES[n]["raises64"]] == ["refine_degenerate_a1_zero",
                                                                      "refine_degenerate_a2_parallel"]
    c = CASES["plucker_pixel_units_1x37"]
    assert (int(c["h"]), int(c["w"])) == (1, 37) and (c["intrinsics"][..., 0, 0] > 20).all()


@pytest.fixture(scope="module")
def capi():
    import __graft_entry__ as ge
    ge.build()
    from pf3plat_b200 import _capi
    return _capi


def test_poses_structs_match_the_header(capi, tmp_path):
    names = ["GsPoseSyncConfig", "GsRefinePosesConfig", "GsRefinePosesInputs", "GsRefinePosesGrads", "GsPluckerConfig"]
    fields = [("GsPoseSyncConfig", "pairs"), ("GsPoseSyncConfig", "pair_i"), ("GsPoseSyncConfig", "pair_j"),
              ("GsRefinePosesInputs", "gamma"), ("GsRefinePosesGrads", "dL_dabspose_inv"),
              ("GsRefinePosesGrads", "dL_dgamma"), ("GsPluckerConfig", "width")]
    prog = tmp_path / "poses_sizes.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "gsplat_b200.h"\nint main(void){'
                    + "".join(f'printf("%zu\\n", sizeof({n}));' for n in names)
                    + "".join(f'printf("%zu\\n", offsetof({s}, {f}));' for s, f in fields)
                    + 'printf("%d %d %d\\n", (int)GS_POSES_MAX_VIEWS, (int)GS_POSES_MAX_PAIRS, GS_ABI_VERSION);return 0;}')
    exe = tmp_path / "poses_sizes"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
    out = [int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert [ctypes.sizeof(getattr(capi, n)) for n in names] == out[:5]
    assert [getattr(getattr(capi, s), f).offset for s, f in fields] == out[5:12]
    assert [capi.GS_POSES_MAX_VIEWS, capi.GS_POSES_MAX_PAIRS, capi.ABI_VERSION] == out[12:] == [16, 120, 5]


def sync_cfg(capi, pairs, N=3, b=2):
    cfg = capi.GsPoseSyncConfig(batch=b, views=N, pairs=len(pairs))
    for q, (i, j) in enumerate(pairs):
        cfg.pair_i[q], cfg.pair_j[q] = i, j
    return cfg


def test_poses_abi_refuses_bad_arguments_without_a_device(capi):
    L = capi.lib()
    good = sync_cfg(capi, [(0, 1), (0, 2), (1, 2)])
    assert L.gs_pose_sync_scratch_bytes(ctypes.byref(good)) == 1024  # [2, 3, 16] doubles, then [2] doubles
    assert L.gs_pose_sync_scratch_bytes(None) == -1
    for pairs, N, b in (([(0, 1), (0, 2), (1, 2)], 17, 2), ([(0, 1)], 1, 2), ([(0, 1), (1, 2)], 3, 0),
                        ([(0, 1), (1, 0), (1, 2)], 3, 2),   # a pair in both orders
                        ([(0, 1), (0, 1), (1, 2)], 3, 2),   # a repeat
                        ([(0, 1), (1, 1), (1, 2)], 3, 2),   # i == j
                        ([(0, 1), (1, 3)], 3, 2),           # out of range
                        ([(0, 1), (0, 2)], 3, 2),           # the chain misses (1, 2)
                        ([(0, 1), (1, 2)], 4, 2)):          # view 3 in no pair
        cfg = sync_cfg(capi, pairs, N, b)
        assert L.gs_pose_sync_scratch_bytes(ctypes.byref(cfg)) == -1, (pairs, N, b)
        assert L.gs_pose_sync(ctypes.byref(cfg), None, None, None, None, None) == -1
    assert L.gs_pose_sync(ctypes.byref(good), None, None, None, None, None) == -1
    assert b"null" in L.gs_last_error()
    rc, ri = capi.GsRefinePosesConfig(batch=2, views=3), capi.GsRefinePosesInputs()
    assert L.gs_refine_poses_forward(ctypes.byref(rc), ctypes.byref(ri), None, None, None) == -1
    assert L.gs_refine_poses_backward(ctypes.byref(rc), ctypes.byref(ri), None, None) == -1
    assert L.gs_refine_poses_forward(ctypes.byref(capi.GsRefinePosesConfig(batch=0, views=3)), None, None, None,
                                     None) == -1
    for bad in (dict(batch=0), dict(views=0), dict(height=0), dict(width=0), dict(batch=300, views=300)):
        base = dict(batch=1, views=1, height=4, width=4)
        base.update(bad)
        assert L.gs_plucker_rays(ctypes.byref(capi.GsPluckerConfig(**base)), None, None, None, None) == -1, bad


def test_python_entries_refuse_bad_arguments_before_any_launch():
    from pf3plat_b200 import poses
    eye = torch.eye(4).expand(2, 4, 4).contiguous()
    Ps = {(0, 1): eye, (0, 2): eye, (1, 2): eye}
    conf = {k: torch.ones(2) for k in Ps}
    with pytest.raises(ValueError, match="supports only"):
        poses.camera_synchronization(Ps, conf, 3, squares=8)
    with pytest.raises(ValueError, match="supports only"):
        poses.camera_synchronization(Ps, conf, 3, center_first_camera=False)
    with pytest.raises(ValueError, match="N <= 16"):
        poses.camera_synchronization(Ps, conf, 17)
    with pytest.raises(ValueError, match="2 <= N"):
        poses.camera_synchronization(Ps, conf, 1)
    with pytest.raises(AssertionError):
        poses.camera_synchronization({(0, 1): eye, (1, 0): eye, (1, 2): eye}, conf, 3)
    with pytest.raises(AssertionError):
        poses.camera_synchronization({(0, 1): eye, (1, 2): eye}, {(0, 1): conf[(0, 1)]}, 3)  # no confidence
    with pytest.raises(AssertionError):
        poses.camera_synchronization({(0, 1): eye, (0, 2): eye}, conf, 3)  # the chain misses (1, 2)
    with pytest.raises(RuntimeError, match="CUDA"):
        poses.camera_synchronization(Ps, conf, 3)
    with pytest.raises(RuntimeError, match="CUDA"):
        poses.refine_poses(torch.zeros(1, 2, 9), torch.zeros(1, 2, 9), torch.ones(()))
    with pytest.raises(RuntimeError, match="CUDA"):
        poses.plucker_rays(eye[None], torch.eye(3).expand(1, 2, 3, 3), 4, 4)
