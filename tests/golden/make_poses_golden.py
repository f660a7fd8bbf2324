"""Generates tests/golden/poses.npz by running the REFERENCE's own pose functions on small seeded cases, in float32 and
in float64:
- `camera_synchronization` (PF3plat's src/flow_util.py, imported unmodified; its module-level `open3d` and
  `pytorch3d.ops` imports are stubbed, nothing here calls them);
- the refined-pose lines of `EncoderCostVolume.forward` (encoder_costvolume.py:465-473) with the class's own
  `r6d2mat`, then `.inverse()`, with the autograd gradients of sum(abspose * g_abs + abspose_inv * g_inv);
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


def refine_case(rng, b, v, gamma, trans=1.0):
    R = [rotation(rng.normal(size=3), rng.uniform(0.1, 1.0)) for _ in range(b * v)]
    enc = np.concatenate([np.stack([r[:2].reshape(6) for r in R]).reshape(b, v, 6), rng.normal(size=(b, v, 3)) * trans],
                         -1)
    return {"pose_enc": enc.astype(np.float32), "delta": (rng.normal(size=(b, v, 9)) * 0.1).astype(np.float32),
            "gamma": np.float32(gamma), "g_abs": rng.normal(size=(b, v, 4, 4)).astype(np.float32),
            "g_inv": rng.normal(size=(b, v, 4, 4)).astype(np.float32)}


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
    Ai = A.inverse()
    ((A * torch.tensor(case["g_abs"], dtype=dtype)).sum() + (Ai * torch.tensor(case["g_inv"], dtype=dtype)).sum()).backward()
    return [t.detach().numpy() for t in (A, Ai, enc.grad, delta.grad, gamma.grad)]


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
                else:
                    data[f"{name}/value{tag}"] = run_plucker(proj, fns, case, dtype)
            finally:
                torch.set_default_dtype(torch.float32)
        print(name, "raises" if data.get(f"{name}/raises64") else "ok")
    np.savez_compressed(OUT, names=np.array(sorted(cases())), **data)
    print(f"wrote {OUT}")


if __name__ == "__main__":
    main()
