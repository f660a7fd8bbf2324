"""Generates tests/golden/costvolume.npz by running the REFERENCE's own plane-sweep functions (PF3plat's
src/model/encoder/costvolume/depth_predictor_multiview.py: `prepare_feat_proj_data_lists` and
`warp_with_pose_depth_candidates`, imported unmodified from a PF3plat checkout) with the correlation and mean lines of
`DepthPredictorMultiView.forward` (:309-343) on small seeded cases, in float32 and in float64, and recording the cost
volume and the autograd gradient of sum(cost * cotangent) with respect to the features.  Cases added later draw from a
generator of their own, after the earlier ones, so that regenerating the file reproduces every earlier array byte for
byte.

Needs a PF3plat checkout, named by $PF3PLAT_ROOT.  The module imports its U-Net (.ldm_unet.unet) at module level for
the network around the op; that import is stubbed.  `coords_grid` casts its integer pixel grid to float32 with
`.float()`, which the float64 run cannot multiply with float64 intrinsics; for that run the same integer grid is cast
to float64 instead (integers are exact in both).  Each run sets torch's default dtype to its own, so that the depth
candidates' linspace has the inputs' precision.
Usage:  PF3PLAT_ROOT=<PF3plat checkout> python tests/golden/make_costvolume_golden.py
"""
import importlib.util
import math
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF_ROOT = os.environ.get("PF3PLAT_ROOT", "")
OUT = os.path.join(HERE, "costvolume.npz")


def load_reference():
    path = os.path.join(REF_ROOT, "src", "model", "encoder", "costvolume", "depth_predictor_multiview.py")
    if not REF_ROOT or not os.path.isfile(path):
        raise SystemExit(f"set PF3PLAT_ROOT to a PF3plat checkout (got {REF_ROOT!r})")
    for name in ("src", "src.model", "src.model.encoder", "src.model.encoder.costvolume",
                 "src.model.encoder.costvolume.ldm_unet"):
        m = types.ModuleType(name)
        m.__path__ = [os.path.join(REF_ROOT, *name.split("."))]
        sys.modules[name] = m
    unet = types.ModuleType("src.model.encoder.costvolume.ldm_unet.unet")
    unet.UNetModel = object
    sys.modules[unet.__name__] = unet
    spec = importlib.util.spec_from_file_location("src.model.encoder.costvolume.depth_predictor_multiview", path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[spec.name] = mod
    spec.loader.exec_module(mod)
    return mod


def reference_cost(mod, features, intrinsics, extrinsics, near, far, D):
    """depth_predictor_multiview.py:310-343 up to the torch.cat"""
    b, v, c, h, w = features.shape
    feat_comb_lists, intr_curr, pose_curr_lists, disp_candi_curr = mod.prepare_feat_proj_data_lists(
        features, intrinsics, extrinsics, near, far, num_samples=D)
    feat01 = feat_comb_lists[0]
    lists = []
    for feat10, pose_curr in zip(feat_comb_lists[1:], pose_curr_lists):
        feat01_warped = mod.warp_with_pose_depth_candidates(
            feat10, intr_curr, pose_curr, 1.0 / disp_candi_curr.repeat([1, 1, *feat10.shape[-2:]]),
            warp_padding_mode="zeros")
        lists.append((feat01.unsqueeze(2) * feat01_warped).sum(1) / (c ** 0.5))
    return torch.mean(torch.stack(lists, dim=0), dim=0, keepdim=False)


def run(mod, case, dtype):
    orig = mod.coords_grid
    if dtype == torch.float64:
        mod.coords_grid = lambda *a, **k: orig(*a, **k).to(torch.float64)
    torch.set_default_dtype(dtype)  # the depth candidates' linspace
    try:
        f = torch.tensor(case["features"], dtype=dtype, requires_grad=True)
        args = [torch.tensor(case[k], dtype=dtype) for k in ("intrinsics", "extrinsics", "near", "far")]
        cost = reference_cost(mod, f, *args, int(case["D"]))
        (cost * torch.tensor(case["cotangent"], dtype=dtype)).sum().backward()
    finally:
        mod.coords_grid = orig
        torch.set_default_dtype(torch.float32)
    return cost.detach().numpy(), f.grad.numpy()


def rotation(axis, angle):
    k = np.asarray(axis, dtype=np.float64)
    k = k / np.linalg.norm(k)
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + math.sin(angle) * Kx + (1 - math.cos(angle)) * Kx @ Kx


def make_case(rng, b, v, C, h, w, D, rot=0.08, trans=0.25, skew=0.0, rows=3, near=(1.0, 1.0), far=(8.0, 8.0)):
    E = np.zeros((b, v, 4, 4))
    K = np.zeros((b, v, rows, rows))
    for i in range(b):
        for j in range(v):
            E[i, j, :3, :3] = rotation(rng.normal(size=3), rot * rng.uniform(0.3, 1.0)) if j else np.eye(3)
            E[i, j, :3, 3] = rng.normal(size=3) * trans if j else 0.0
            E[i, j, 3, 3] = 1.0
            fx, fy = rng.uniform(0.8, 1.1), rng.uniform(0.8, 1.1)
            K[i, j, :3, :3] = [[fx, skew * rng.uniform(0.5, 1.0), rng.uniform(0.45, 0.55)],
                               [0.0, fy, rng.uniform(0.45, 0.55)], [0.0, 0.0, 1.0]]
            if rows == 4:
                K[i, j, 3, 3] = 1.0
    return {"features": rng.normal(size=(b, v, C, h, w)).astype(np.float32), "intrinsics": K, "extrinsics": E,
            "near": rng.uniform(*near, size=(b, v)), "far": rng.uniform(*far, size=(b, v)), "D": np.int64(D),
            "cotangent": rng.normal(size=(v * b, D, h, w)).astype(np.float32)}


def cases():
    rng = np.random.default_rng(20261017)
    out = {}
    out["v2_skew_pp"] = make_case(rng, 2, 2, 2, 13, 22, 2, skew=0.05, near=(0.8, 1.5), far=(6.0, 12.0))
    out["v2_c256_d32"] = make_case(rng, 1, 2, 256, 2, 3, 32)
    out["v3_c64_d32"] = make_case(rng, 1, 3, 64, 3, 4, 32, near=(0.8, 1.5), far=(6.0, 12.0))
    out["v4_b3_c1_k4x4"] = make_case(rng, 3, 4, 1, 7, 8, 2, rows=4, near=(0.8, 1.5), far=(6.0, 12.0))
    out["v3_b2_2x2_d1"] = make_case(rng, 2, 3, 3, 2, 2, 1)
    c = make_case(rng, 1, 2, 3, 7, 9, 2)  # identity relative pose: samples on integer pixels, last row and column too
    c["extrinsics"][:, 1] = c["extrinsics"][:, 0]
    c["intrinsics"][:, 1] = c["intrinsics"][:, 0]
    out["v2_identity"] = c
    c = make_case(rng, 1, 2, 3, 9, 12, 2)  # a 60 degree turn: most samples leave the source image
    c["extrinsics"][0, 1, :3, :3] = rotation([0.1, 1.0, 0.0], math.radians(60.0))
    out["v2_out_of_bounds"] = c
    c = make_case(rng, 1, 2, 3, 9, 12, 4, near=(1.0, 1.0), far=(8.0, 8.0))  # source camera 3 ahead: near points behind it
    c["extrinsics"][0, 1, :3, :3] = np.eye(3)
    c["extrinsics"][0, 1, :3, 3] = [0.05, -0.03, 3.0]
    out["v2_behind_source"] = c
    c = make_case(rng, 1, 2, 3, 9, 12, 2)  # NaN in a pixel of view 0, +Inf and -Inf in pixels of view 1
    c["features"][0, 0, 1, 4, 5] = np.nan
    c["features"][0, 1, 0, 3, 7] = np.inf
    c["features"][0, 1, 2, 6, 2] = -np.inf
    out["v2_nonfinite"] = c
    # Past the kernels' first 256-channel pass, past poison word 0, and beyond four views.  These cases draw from their
    # own generator, so the arrays of the cases above stay exactly as they were.
    rng = np.random.default_rng(20261018)
    c = make_case(rng, 1, 2, 300, 3, 4, 3)  # NaN at channel 290 of view 0, +Inf at 40 and -Inf at 256 of view 1
    c["features"][0, 0, 290, 1, 1] = np.nan
    c["features"][0, 1, 40, 1, 2] = np.inf
    c["features"][0, 1, 256, 2, 1] = -np.inf
    out["v2_c300_nonfinite"] = c
    out["v5_b2_c130"] = make_case(rng, 2, 5, 130, 4, 5, 4, rows=4, near=(0.8, 1.5), far=(6.0, 12.0))
    out["v8_c5_d3"] = make_case(rng, 1, 8, 5, 3, 3, 3, near=(0.8, 1.5), far=(6.0, 12.0))
    out["v2_c257_d2"] = make_case(rng, 1, 2, 257, 3, 3, 2)  # second pass: one float4 chunk, three quarters padding
    return out


def main():
    mod = load_reference()
    data = {}
    for name, case in cases().items():
        v32, g32 = run(mod, case, torch.float32)
        v64, g64 = run(mod, case, torch.float64)
        for what, a, b in (("value", v32, v64), ("grad", g32, g64)):
            if not np.array_equal(np.isfinite(a), np.isfinite(b)):
                raise SystemExit(f"{name}: float32 and float64 disagree on which {what}s are finite; move the non-finite "
                                 f"values")
        for k, val in case.items():
            data[f"{name}/{k}"] = val
        data[f"{name}/value64"], data[f"{name}/grad64"] = v64, g64
        data[f"{name}/value32"], data[f"{name}/grad32"] = v32, g32
        print(f"{name}: value {v64.shape}, {int((~np.isfinite(v64)).sum())} non-finite values, "
              f"{int((~np.isfinite(g64)).sum())} non-finite gradients")
    np.savez_compressed(OUT, names=np.array(sorted(cases())), **data)
    print(f"wrote {OUT}")


if __name__ == "__main__":
    main()
