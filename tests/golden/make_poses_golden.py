"""Generates tests/golden/poses.npz by running the REFERENCE's own pose functions on small seeded cases, in float32 and
in float64:
- `camera_synchronization` (PF3plat's src/flow_util.py, imported unmodified; its module-level `open3d` and
  `pytorch3d.ops` imports are stubbed, nothing here calls them);
- the refined-pose lines of `EncoderCostVolume.forward` (encoder_costvolume.py:465-473) with the class's own
  `r6d2mat`, then `.inverse()`, with the autograd gradients of sum(abspose * g_abs + abspose_inv * g_inv) (for the
  `refine_degenerate_*` cases of sum(abspose * g_abs) alone, with `raises` recording whether `.inverse()` raised);
- the Plücker lines (:387-392) with projection.py's `sample_image_grid` / `get_world_rays` and the class's own
  `plucker_embedding`.
The three methods use no instance state; they are taken from the class body with `ast` and run with `self = None`, so
the encoder's network imports are never executed.  Each run sets torch's default dtype to its own, so that the constants
the reference creates (zeros, eye, the pixel grid) have the inputs' precision.  The synchronisation ends in `.float()`
and `camera_chaining` calls `.float()` on its operands; in the float64 run `Tensor.float` is the identity for the
duration of the call, so that the float64 record carries float64 all the way.  A case on which the reference raises is
recorded as raising.
Usage:  PF3PLAT_ROOT=<PF3plat checkout> python tests/golden/make_poses_golden.py
"""
import ast
import importlib.util
import itertools
import math
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF_ROOT = os.environ.get("PF3PLAT_ROOT", "")
OUT = os.path.join(HERE, "poses.npz")


def load_module(name, *parts):
    path = os.path.join(REF_ROOT, *parts)
    if not REF_ROOT or not os.path.isfile(path):
        raise SystemExit(f"set PF3PLAT_ROOT to a PF3plat checkout (got {REF_ROOT!r})")
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def load_reference():
    for name in ("open3d", "pytorch3d", "pytorch3d.ops"):
        sys.modules[name] = types.ModuleType(name)
    sys.modules["pytorch3d.ops"].corresponding_points_alignment = None
    flow = load_module("pf3plat_flow_util", "src", "flow_util.py")
    proj = load_module("pf3plat_projection", "src", "geometry", "projection.py")
    path = os.path.join(REF_ROOT, "src", "model", "encoder", "encoder_costvolume.py")
    tree = ast.parse(open(path).read())
    cls = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "EncoderCostVolume")
    wanted = {"r6d2mat", "plucker_embedding", "matrix_to_rotation_6d"}
    fns = [n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name in wanted]
    assert {f.name for f in fns} == wanted
    ns = {"torch": torch, "F": torch.nn.functional}
    exec(compile(ast.Module(body=fns, type_ignores=[]), path, "exec"), ns)
    return flow, proj, {k: ns[k] for k in wanted}


def rotation(axis, angle):
    k = np.asarray(axis, dtype=np.float64)
    k = k / np.linalg.norm(k)
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + math.sin(angle) * Kx + (1 - math.cos(angle)) * Kx @ Kx


def rigid(rng, rot, trans):
    P = np.eye(4)
    P[:3, :3] = rotation(rng.normal(size=3), rot * rng.uniform(0.3, 1.0))
    P[:3, 3] = rng.normal(size=3) * trans
    return P


def sync_case(rng, b, N, trans=0.3, noise=0.03):
    """pairwise poses i -> j of N noisy absolute cameras, every pair i < j in the encoder's order, confidences as the
    matcher's mean scores with the encoder's relu rescale for |i - j| > 1"""
    keys = list(itertools.combinations(range(N), 2))
    Ps = np.zeros((len(keys), b, 4, 4))
    conf = np.zeros((len(keys), b))
    for s in range(b):
        W = [np.eye(4)] + [rigid(rng, 0.3, trans) for _ in range(N - 1)]
        for q, (i, j) in enumerate(keys):
            Ps[q, s] = W[j] @ np.linalg.inv(W[i]) @ rigid(rng, noise, noise)
            c = rng.uniform(0.55, 0.95)
            conf[q, s] = max(c - 0.5, 0.0) / 0.5 if abs(i - j) > 1 else c
    return {"keys": np.array(keys, dtype=np.int64), "Ps": Ps.astype(np.float32), "conf": conf.astype(np.float32),
            "N": np.int64(N)}


def sync_graph(rng, b, N, keys, trans=0.3, noise=0.03):
    """sync_case on any list of keys, in the given order; a key (i, j) with i > j is the transform i -> j all the same"""
    Ps = np.zeros((len(keys), b, 4, 4))
    conf = np.zeros((len(keys), b))
    for s in range(b):
        W = [np.eye(4)] + [rigid(rng, 0.3, trans) for _ in range(N - 1)]
        for q, (i, j) in enumerate(keys):
            Ps[q, s] = W[j] @ np.linalg.inv(W[i]) @ rigid(rng, noise, noise)
            c = rng.uniform(0.55, 0.95)
            conf[q, s] = max(c - 0.5, 0.0) / 0.5 if abs(i - j) > 1 else c
    return {"keys": np.array(keys, dtype=np.int64), "Ps": Ps.astype(np.float32), "conf": conf.astype(np.float32),
            "N": np.int64(N)}


def chain_keys(N):
    return [(k, k + 1) for k in range(N - 1)]


def shuffled_keys(rng, N, reverse_off_chain):
    """every pair once, in a shuffled order; off-chain pairs stored as (j, i) where reverse_off_chain draws True"""
    keys = [(j, i) if j - i > 1 and reverse_off_chain and rng.random() < 0.5 else (i, j)
            for i, j in itertools.combinations(range(N), 2)]
    return [keys[q] for q in rng.permutation(len(keys))]


# 180-degree rotations about the coordinate axes and the identity: a consistent sign gauge per view
AXIS_FLIPS = [np.diag(d).astype(np.float64) for d in ((1, 1, 1), (1, -1, -1), (-1, 1, -1), (-1, -1, 1))]


def sync_degenerate_rotations(rng, b, N, zero_axes):
    """pairwise transforms whose rotation parts are D_j D_i Z with D a per-view axis flip and Z the identity with the
    axes zero_axes[s] zeroed, plus translations: every product along a path is diagonal with entries 0 or +-1, so the
    rotation part of every synchronised block is diagonal, and zero exactly on the zeroed axes (rank 3 - |zero_axes|)"""
    keys = list(itertools.combinations(range(N), 2))
    Ps = np.zeros((len(keys), b, 4, 4))
    conf = rng.uniform(0.55, 0.95, size=(len(keys), b))
    for s in range(b):
        D = [AXIS_FLIPS[0]] + [AXIS_FLIPS[k] for k in rng.integers(0, 4, N - 1)]
        Z = np.eye(3)
        for a in zero_axes[s]:
            Z[a, a] = 0.0
        for q, (i, j) in enumerate(keys):
            Ps[q, s] = np.eye(4)
            Ps[q, s, :3, :3] = D[j] @ D[i] @ Z
            Ps[q, s, :3, 3] = rng.normal(size=3) * 0.3
    return {"keys": np.array(keys, dtype=np.int64), "Ps": Ps.astype(np.float32), "conf": conf.astype(np.float32),
            "N": np.int64(N)}


def refine_case(rng, b, v, gamma, trans=1.0):
    R = [rotation(rng.normal(size=3), rng.uniform(0.1, 1.0)) for _ in range(b * v)]
    enc = np.concatenate([np.stack([r[:2].reshape(6) for r in R]).reshape(b, v, 6), rng.normal(size=(b, v, 3)) * trans],
                         -1)
    return {"pose_enc": enc.astype(np.float32), "delta": (rng.normal(size=(b, v, 9)) * 0.1).astype(np.float32),
            "gamma": np.float32(gamma), "g_abs": rng.normal(size=(b, v, 4, 4)).astype(np.float32),
            "g_inv": rng.normal(size=(b, v, 4, 4)).astype(np.float32)}


def refine_degenerate(rng, b, v, gamma, rot6d):
    """refine_case with abspose-only cotangents and the 6-d rotation rot6d placed in scene 0 at view 0 and, with a zero
    delta on its rotation entries (so x is rot6d exactly), in the last scene at the last view"""
    c = refine_case(rng, b, v, gamma)
    del c["g_inv"]
    for s, u in ((0, 0), (b - 1, v - 1)):
        c["pose_enc"][s, u, :6] = rot6d
        c["delta"][s, u, :6] = 0.0
    return c


def plucker_case(rng, b, v, h, w):
    E = np.stack([rigid(rng, 0.5, 1.0) for _ in range(b * v)]).reshape(b, v, 4, 4)
    K = np.zeros((b, v, 3, 3))
    K[..., 0, 0], K[..., 1, 1] = rng.uniform(0.8, 1.1, (b, v)), rng.uniform(0.8, 1.1, (b, v))
    K[..., 0, 2], K[..., 1, 2], K[..., 2, 2] = rng.uniform(0.45, 0.55, (b, v)), rng.uniform(0.45, 0.55, (b, v)), 1.0
    return {"abspose": E.astype(np.float32), "intrinsics": K.astype(np.float32), "h": np.int64(h), "w": np.int64(w)}


def cases():
    rng = np.random.default_rng(20261018)
    out = {}
    out["sync_n2"] = sync_case(rng, 2, 2)
    out["sync_n3"] = sync_case(rng, 3, 3)
    out["sync_n4"] = sync_case(rng, 2, 4)
    out["sync_n5"] = sync_case(rng, 2, 5)
    out["sync_n8"] = sync_case(rng, 2, 8)
    c = sync_case(rng, 2, 3)  # PnP failures: identity poses for (0, 1) in scene 0 and (1, 2) in scene 1
    c["Ps"][0, 0] = np.eye(4)
    c["Ps"][2, 1] = np.eye(4)
    out["sync_pnp_fail"] = c
    c = sync_case(rng, 2, 3)  # the (0, 2) score below the encoder's 0.5 threshold: relu zeroes it
    c["conf"][1] = 0.0
    out["sync_relu_zero_02"] = c
    c = sync_case(rng, 2, 3)
    c["conf"][:] = 0.0
    out["sync_all_zero"] = c
    c = sync_case(rng, 3, 3)  # scene 1 has zero mass: the whole batch is chained
    c["conf"][:, 1] = 0.0
    out["sync_one_zero_mass"] = c
    c = sync_case(rng, 2, 3)
    c["conf"][0, 1] = np.nan
    out["sync_nan_conf"] = c
    out["sync_large_t"] = sync_case(rng, 2, 4, trans=300.0)
    out["refine_gamma1"] = refine_case(rng, 3, 3, 1.0)
    out["refine_gamma0"] = refine_case(rng, 2, 3, 0.0)
    out["refine_v5_large_t"] = refine_case(rng, 2, 5, 0.7, trans=500.0)
    out["plucker_8x8"] = plucker_case(rng, 2, 3, 8, 8)
    out["plucker_13x22"] = plucker_case(rng, 1, 2, 13, 22)
    # cases added later: each draws from its own generator, so the ones above stay byte-identical
    rng = np.random.default_rng(101)
    out["sync_sparse_path_n6"] = sync_graph(rng, 2, 6, chain_keys(6))  # only the chain pairs
    rng = np.random.default_rng(102)
    out["sync_sparse_ring_n5"] = sync_graph(rng, 2, 5, chain_keys(5) + [(4, 0)])  # one pair stored with i > j
    rng = np.random.default_rng(103)
    out["sync_shuffled_n8"] = sync_graph(rng, 2, 8, shuffled_keys(rng, 8, True))
    rng = np.random.default_rng(104)
    out["sync_n16"] = sync_graph(rng, 2, 16, list(itertools.combinations(range(16), 2)))
    rng = np.random.default_rng(105)
    c = sync_graph(rng, 2, 16, shuffled_keys(rng, 16, False))  # scene 1 has zero mass: 15 chained pairs per view 15
    c["conf"][:, 1] = 0.0
    out["sync_chain_n16"] = c
    rng = np.random.default_rng(106)
    c = sync_graph(rng, 3, 4, list(itertools.combinations(range(4), 2)))
    c["conf"][2, 1] = np.nan  # scene 1: a NaN confidence; scene 2: zero mass, which alone would chain the batch
    c["conf"][:, 2] = 0.0
    out["sync_nan_and_zero_mass"] = c
    rng = np.random.default_rng(107)
    c = sync_graph(rng, 2, 4, chain_keys(4) + [(0, 2), (1, 3)])
    q13, q23 = 4, 2
    c["conf"][q23, 1], c["conf"][q13, 1] = 1e-10, -2e-10  # scene 1, view 3: confidences summing below zero
    out["sync_negative_conf"] = c
    rng = np.random.default_rng(108)
    out["sync_rank2"] = sync_degenerate_rotations(rng, 3, 4, [(2,), (1,), (0,)])
    rng = np.random.default_rng(109)
    out["sync_rank0"] = sync_degenerate_rotations(rng, 2, 4, [(0, 1, 2)] * 2)
    degenerate = {
        "a1_zero": [0.0, 0.0, 0.0, 0.3, -0.8, 0.5],
        "a1_tiny": [3e-13, -4e-13, 1e-13, 0.3, -0.8, 0.5],            # 0 < |a1| < 1e-12
        "a2_parallel": [0.0, -0.25, 0.0, 0.0, -0.5, 0.0],             # a2 = 2 a1 on an axis: c is exactly 0
        "c_above_eps": [0.0, 0.0, 2.0, 1.5e-12, 0.0, 1.0],            # c = (1.5e-12, 0, 0) exactly
        "c_below_eps": [0.0, 0.0, 2.0, 0.5e-12, -0.5e-12, -0.75],     # c = (5e-13, -5e-13, 0) exactly
    }
    for k, (name, rot6d) in enumerate(degenerate.items()):
        rng = np.random.default_rng(110 + k)
        out[f"refine_degenerate_{name}"] = refine_degenerate(rng, 2, 3, 0.8, np.float32(rot6d))
    rng = np.random.default_rng(120)
    out["refine_degenerate_v1"] = refine_degenerate(rng, 3, 1, 0.8, np.float32([1.0, 0.0, 0.0, 0.0, 1.0, 0.0]))
    rng = np.random.default_rng(121)
    out["refine_degenerate_negative_gamma"] = refine_degenerate(rng, 2, 3, -0.7,
                                                                np.float32([0.0, 0.6, 0.8, 1.0, 0.0, 0.0]))
    rng = np.random.default_rng(122)
    c = plucker_case(rng, 1, 2, 1, 37)  # intrinsics in pixel units (rows scaled by w = 37 and h = 1), one pixel high
    c["intrinsics"][..., 0, :] *= 37.0
    out["plucker_pixel_units_1x37"] = c
    return out


def run_sync(flow, case, dtype):
    keys = [tuple(int(x) for x in k) for k in case["keys"]]
    Ps = {k: torch.tensor(case["Ps"][q], dtype=dtype) for q, k in enumerate(keys)}
    conf = {k: torch.tensor(case["conf"][q], dtype=dtype) for q, k in enumerate(keys)}
    orig = torch.Tensor.float
    if dtype == torch.float64:
        torch.Tensor.float = lambda self, *a, **k: self
    try:
        return flow.camera_synchronization(Ps, conf, int(case["N"])).numpy(), False
    except Exception:  # torch.svd on non-finite input raises torch.linalg.LinAlgError
        return np.zeros(0), True
    finally:
        torch.Tensor.float = orig


def run_refine(fns, case, dtype):
    enc = torch.tensor(case["pose_enc"], dtype=dtype, requires_grad=True)
    delta = torch.tensor(case["delta"], dtype=dtype, requires_grad=True)
    gamma = torch.tensor(float(case["gamma"]), dtype=dtype, requires_grad=True)
    pred_pose = enc[:, 1:] + delta[:, 1:] * gamma  # encoder_costvolume.py:465-473
    pred_concat_pose = torch.cat([enc[:, :1], pred_pose], dim=1)
    rot6d = fns["r6d2mat"](None, pred_concat_pose[:, :, :6])
    trans3d = pred_concat_pose[:, :, 6:]
    Rt = torch.cat([rot6d, trans3d[..., None]], dim=-1)
    pad = torch.zeros_like(Rt[..., 2:3, :])
    pad[..., -1] = 1.0
    A = torch.cat((Rt, pad), dim=-2)
    loss = (A * torch.tensor(case["g_abs"], dtype=dtype)).sum()
    try:
        Ai = A.inverse()
    except Exception:  # a singular abspose: torch.linalg.inv raises torch.linalg.LinAlgError
        assert "g_inv" not in case
        Ai = None
    if "g_inv" in case:  # the cases without g_inv take cotangents on abspose only
        loss = loss + (Ai * torch.tensor(case["g_inv"], dtype=dtype)).sum()
    loss.backward()
    Ai = Ai.detach().numpy() if Ai is not None else np.zeros(0)
    return [A.detach().numpy(), Ai] + [t.detach().numpy() for t in (enc.grad, delta.grad, gamma.grad)]


def run_plucker(proj, fns, case, dtype):
    from einops import rearrange, repeat
    E = torch.tensor(case["abspose"], dtype=dtype)
    K = torch.tensor(case["intrinsics"], dtype=dtype)
    b, v = E.shape[:2]
    h, w = int(case["h"]), int(case["w"])
    xy, _ = proj.sample_image_grid((h, w), E.device)  # encoder_costvolume.py:387-392 with (h//4, w//4) -> (h, w)
    xy = repeat(rearrange(xy, "h w xy -> (h w) () xy"), "hw () xy -> b hw xy", b=b * v)
    origins, directions = proj.get_world_rays(rearrange(xy, "(b v) hw xy -> b v () hw () xy", b=b, v=v),
                                              rearrange(E.inverse(), "b v i j -> b v () () () i j"),
                                              rearrange(K, "b v i j -> b v () () () i j"))
    out = fns["plucker_embedding"](None, h, w,
                                   rearrange(origins, "b v 1 hw srf xyz -> (b v) hw srf xyz").squeeze(-2),
                                   rearrange(directions, "b v 1 hw srf xyz -> (b v) hw srf xyz").squeeze(-2))
    return out.numpy()


def main():
    flow, proj, fns = load_reference()
    data = {}
    for name, case in cases().items():
        for k, val in case.items():
            data[f"{name}/{k}"] = val
        for dtype, tag in ((torch.float32, "32"), (torch.float64, "64")):
            torch.set_default_dtype(dtype)
            try:
                if name.startswith("sync"):
                    val, raised = run_sync(flow, case, dtype)
                    data[f"{name}/value{tag}"], data[f"{name}/raises{tag}"] = val, np.bool_(raised)
                elif name.startswith("refine"):
                    for k, val in zip(("abspose", "abspose_inv", "d_pose_enc", "d_delta", "d_gamma"),
                                      run_refine(fns, case, dtype)):
                        data[f"{name}/{k}{tag}"] = val
                    if "g_inv" not in case:
                        data[f"{name}/raises{tag}"] = np.bool_(data[f"{name}/abspose_inv{tag}"].size == 0)
                else:
                    data[f"{name}/value{tag}"] = run_plucker(proj, fns, case, dtype)
            finally:
                torch.set_default_dtype(torch.float32)
        print(name, "raises" if data.get(f"{name}/raises64") else "ok")
    np.savez_compressed(OUT, names=np.array(sorted(cases())), **data)
    print(f"wrote {OUT}")


if __name__ == "__main__":
    main()
