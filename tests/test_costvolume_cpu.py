"""CPU checks of the plane-sweep cost volume: the fp64 oracle (tests/costvolume_oracle.py) against the reference's own
functions recorded in tests/golden/costvolume.npz (make_costvolume_golden.py) and against central finite differences;
the regimes the golden cases are meant to reach; the C ABI's struct layouts and argument checks (no device)."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from tests import costvolume_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "costvolume.npz")


def load_cases():
    z = np.load(GOLDEN)
    return {str(n): {k.split("/", 1)[1]: z[k] for k in z.files if k.startswith(f"{n}/")} for n in z["names"]}


CASES = load_cases()


def oracle(case, features=None, dtype=torch.float64):
    f = torch.tensor(case["features"], dtype=dtype) if features is None else features
    args = [torch.tensor(case[k], dtype=dtype) for k in ("intrinsics", "extrinsics", "near", "far")]
    return O.cost_volume(f, *args, int(case["D"]))


def close_with_pattern(a, b, tol):
    fa, fb = np.isfinite(a), np.isfinite(b)
    assert np.array_equal(fa, fb), "non-finite pattern differs"
    assert np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(a[np.isinf(a)], b[np.isinf(b)])
    scale = max(1.0, float(np.abs(b[fb]).max()) if fb.any() else 1.0)
    err = float(np.abs(a[fa] - b[fb]).max()) if fa.any() else 0.0
    assert err <= tol * scale, err


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_the_reference_record(name):
    case = CASES[name]
    f = torch.tensor(case["features"], dtype=torch.float64, requires_grad=True)
    cost = oracle(case, f)
    (cost * torch.tensor(case["cotangent"], dtype=torch.float64)).sum().backward()
    close_with_pattern(cost.detach().numpy(), case["value64"], 1e-10)
    close_with_pattern(f.grad.numpy(), case["grad64"], 1e-10)


@pytest.mark.parametrize("name", ["v2_skew_pp", "v4_b3_c1_k4x4", "v3_b2_2x2_d1", "v2_behind_source"])
def test_oracle_gradient_matches_finite_differences(name):
    case = CASES[name]
    g = torch.tensor(case["cotangent"], dtype=torch.float64)
    f0 = torch.tensor(case["features"], dtype=torch.float64, requires_grad=True)
    (oracle(case, f0) * g).sum().backward()
    rng = np.random.default_rng(7)
    flat = f0.detach().reshape(-1)
    eps = 1e-6
    for i in rng.choice(flat.numel(), size=min(40, flat.numel()), replace=False):
        fp, fm = flat.clone(), flat.clone()
        fp[i] += eps
        fm[i] -= eps
        num = ((oracle(case, fp.reshape(f0.shape)) - oracle(case, fm.reshape(f0.shape))) * g).sum() / (2 * eps)
        assert abs(float(num) - float(f0.grad.reshape(-1)[i])) < 1e-6 * max(1.0, abs(float(num)))


def coords(case):
    f = torch.tensor(case["features"], dtype=torch.float64)
    b, v, C, h, w = f.shape
    K = O.unnormalised_intrinsics(torch.tensor(case["intrinsics"]), h, w)
    depth = O.depth_candidates(torch.tensor(case["near"]), torch.tensor(case["far"]), int(case["D"]))
    poses = O.relative_poses(torch.tensor(case["extrinsics"]))
    return [O.sample_coordinates(K, p, depth, h, w) for p in poses], (h, w)


def test_golden_cases_reach_their_regimes():
    cs, (h, w) = coords(CASES["v2_out_of_bounds"])
    ix, iy = cs[0]
    out = (ix < -1) | (ix > w) | (iy < -1) | (iy > h)
    assert float(out.double().mean()) > 0.5
    # the source camera 3 ahead: some candidate points lie behind it and are divided by 1e-3
    c = CASES["v2_behind_source"]
    f = torch.tensor(c["features"], dtype=torch.float64)
    K = O.unnormalised_intrinsics(torch.tensor(c["intrinsics"]), *f.shape[-2:])
    pose = O.relative_poses(torch.tensor(c["extrinsics"]))[0]
    depth = O.depth_candidates(torch.tensor(c["near"]), torch.tensor(c["far"]), int(c["D"]))
    z = depth[0, -1] * (pose[0, 2, :3] @ torch.linalg.inv(K[0]) @ torch.tensor([4.0, 4.0, 1.0], dtype=torch.float64)) \
        + pose[0, 2, 3]
    assert float(z) < 1e-3
    # identity pose: every sample within 1e-9 of its own pixel, the last row and column included
    cs, (h, w) = coords(CASES["v2_identity"])
    ix, iy = cs[0]
    xs = torch.arange(w, dtype=torch.float64).repeat(h)
    assert float((ix - xs).abs().max()) < 1e-9 and float(ix.max()) > w - 1 - 1e-9
    # skew and off-centre principal points
    K = CASES["v2_skew_pp"]["intrinsics"]
    assert (np.abs(K[..., 0, 1]) > 0).all() and (np.abs(K[..., :2, 2] - 0.5) > 1e-3).any()
    assert CASES["v4_b3_c1_k4x4"]["intrinsics"].shape[-1] == 4
    assert len(np.unique(CASES["v2_skew_pp"]["near"])) == 4 and len(np.unique(CASES["v2_skew_pp"]["far"])) == 4
    for name in ("v2_nonfinite", "v2_c300_nonfinite"):
        v = CASES[name]["value64"]
        assert np.isnan(v).any() and not np.isfinite(CASES[name]["grad64"]).all()
    # The kernels hold 256 channels (64 float4 chunks) per pass; the poison mask has one 32-bit word per 32 channels.
    shapes = {n: c["features"].shape for n, c in CASES.items()}  # [b, v, C, h, w]
    cp4 = {n: (s[2] + 3) // 4 for n, s in shapes.items()}
    assert {n for n, s in shapes.items() if s[2] > 256} == {"v2_c300_nonfinite", "v2_c257_d2"}
    assert cp4["v2_c257_d2"] == 64 + 1  # the second pass is one chunk, three of its four channels padding
    assert {n for n, s in shapes.items() if s[2] % 4 and cp4[n] > 1} >= {"v8_c5_d3", "v5_b2_c130", "v2_c257_d2"}
    assert shapes["v5_b2_c130"][:2] == (2, 5) and CASES["v5_b2_c130"]["intrinsics"].shape[-1] == 4
    assert shapes["v8_c5_d3"][1] == 8
    # non-finite features at channels in poison words 1, 8 and 9, in both views, and non-finite gradients at each of
    # those channels: in view 0 where it samples view 1's +-Inf, in view 1 where view 0's NaN reaches it
    c = CASES["v2_c300_nonfinite"]
    bad = {(int(i[1]), int(i[2])) for i in np.argwhere(~np.isfinite(c["features"]))}
    assert bad == {(0, 290), (1, 40), (1, 256)}
    assert {ch // 32 for _, ch in bad} == {1, 8, 9}
    gbad = {(int(i[1]), int(i[2])) for i in np.argwhere(~np.isfinite(c["grad64"]))}
    assert gbad == {(0, 40), (0, 256), (1, 290)}


@pytest.fixture(scope="module")
def capi():
    import __graft_entry__ as ge
    ge.build()
    from pf3plat_b200 import _capi
    return _capi


def test_costvolume_structs_match_the_header(capi, tmp_path):
    names = ["GsCostVolumeConfig", "GsCostVolumeInputs", "GsCostVolumeGrads"]
    fields = [("GsCostVolumeConfig", "depth_candidates"), ("GsCostVolumeConfig", "flags"),
              ("GsCostVolumeConfig", "feat_stride"), ("GsCostVolumeInputs", "far_"), ("GsCostVolumeGrads", "dL_dfeatures")]
    prog = tmp_path / "cv_sizes.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "gsplat_b200.h"\nint main(void){'
                    + "".join(f'printf("%zu\\n", sizeof({n}));' for n in names)
                    + "".join(f'printf("%zu\\n", offsetof({s}, {f}));' for s, f in fields)
                    + 'printf("%d\\n", (int)GS_COSTVOLUME_DETERMINISTIC);return 0;}')
    exe = tmp_path / "cv_sizes"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
    out = [int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert [ctypes.sizeof(getattr(capi, n)) for n in names] == out[:3]
    assert [getattr(getattr(capi, s), f).offset for s, f in fields] == out[3:8]
    assert capi.GS_COSTVOLUME_DETERMINISTIC == out[8]


def _cfg(capi, **kw):
    base = dict(batch=2, views=2, channels=256, height=64, width=64, depth_candidates=32, intrinsics_rows=3, flags=0)
    base.update(kw)
    return capi.GsCostVolumeConfig(**base)


def test_costvolume_refuses_bad_arguments_without_a_device(capi):
    L = capi.lib()
    ins = capi.GsCostVolumeInputs()
    assert L.gs_costvolume_forward(None, None, None, None, None) == -1
    assert L.gs_costvolume_backward(None, None, None, None, None) == -1
    assert L.gs_costvolume_scratch_bytes(None, 0) == -1
    good = _cfg(capi)
    # a valid config with null tensors: refused before any launch
    assert L.gs_costvolume_forward(ctypes.byref(good), ctypes.byref(ins), None, None, None) == -1
    assert b"null" in L.gs_last_error()
    assert L.gs_costvolume_backward(ctypes.byref(good), None, None, None, None) == -1
    for bad in (dict(views=1), dict(height=1), dict(width=1), dict(channels=0), dict(depth_candidates=0), dict(batch=0),
                dict(intrinsics_rows=2), dict(flags=2),
                dict(flags=1, views=3, depth_candidates=64, height=128, width=128)):  # deterministic term bound
        cfg = _cfg(capi, **bad)
        assert L.gs_costvolume_scratch_bytes(ctypes.byref(cfg), 1) == -1, bad
        assert L.gs_costvolume_forward(ctypes.byref(cfg), ctypes.byref(ins), None, None, None) == -1, bad
    # the training shape's scratch: the packed features, then in the backward the gradient rows and accumulators
    rows = 2 * 2 * 64 * 64 * 256 * 4
    fwd = L.gs_costvolume_scratch_bytes(ctypes.byref(good), 0)
    bwd = L.gs_costvolume_scratch_bytes(ctypes.byref(good), 1)
    assert rows <= fwd < rows + 65536 and 3 * rows <= bwd < 3 * rows + 65536
    det = L.gs_costvolume_scratch_bytes(ctypes.byref(_cfg(capi, flags=1)), 1)
    assert det >= rows * 8 and det % 256 == 0


def test_python_entry_refuses_bad_arguments_before_any_launch():
    from pf3plat_b200.costvolume import plane_sweep_cost_volume
    f = torch.zeros(1, 2, 3, 4, 4)
    K, E, n = torch.eye(3).expand(1, 2, 3, 3), torch.eye(4).expand(1, 2, 4, 4), torch.ones(1, 2)
    with pytest.raises(RuntimeError, match="CUDA"):
        plane_sweep_cost_volume(f, K, E, n, n * 2, 4)
