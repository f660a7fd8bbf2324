"""Generates tests/golden/pose_loss.npz by running the REFERENCE's own correspondence loss (PF3plat's
src/loss/loss_pose.py, `Losspose`, imported unmodified from a PF3plat checkout) on small seeded inputs, in float32 and in
float64, and recording the loss and its autograd gradients with respect to the absolute poses, the depth, xyz_h, the match
weights and the per-pair confidences.

Needs a PF3plat checkout, named by $PF3PLAT_ROOT.  loss_pose.py imports src.flow_util, which imports open3d and
pytorch3d.ops at module level for functions the loss never calls: both are stubbed.  The type modules
(src.dataset.types, src.model.decoder.decoder, src.model.types) and the abstract base src.loss.loss are stubbed as in
make_ssim_loss_golden.py; flow_util (cv2, einops) and src.geometry.projection are the reference's.
The float64 run sets torch's default dtype to float64, so that sample_image_grid's pixel grid matches the inputs' dtype.
Usage:  PF3PLAT_ROOT=<PF3plat checkout> python tests/golden/make_pose_loss_golden.py
"""
import importlib.util
import math
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_ssim_loss_golden import REF_ROOT, _stub_loss_base  # noqa: E402

WEIGHT_2D, WEIGHT_3D, DELTA = 0.005, 0.025, 0.01


def load_reference_pose_loss():
    if not REF_ROOT or not os.path.isfile(os.path.join(REF_ROOT, "src/loss/loss_pose.py")):
        raise SystemExit(f"set PF3PLAT_ROOT to a PF3plat checkout (got {REF_ROOT!r})")
    for name in ("src", "src.loss", "src.dataset", "src.model", "src.model.decoder", "src.geometry"):
        m = types.ModuleType(name)
        m.__path__ = [os.path.join(REF_ROOT, *name.split("."))]
        sys.modules[name] = m
    stubs = {"src.dataset.types": {"BatchedExample": dict}, "src.model.decoder.decoder": {"DecoderOutput": object},
             "src.model.types": {"Gaussians": object}, "src.loss.loss": {"Loss": _stub_loss_base()},
             "open3d": {}, "pytorch3d": {}, "pytorch3d.ops": {"corresponding_points_alignment": None}}
    for name, attrs in stubs.items():
        m = types.ModuleType(name)
        for k, v in attrs.items():
            setattr(m, k, v)
        sys.modules[name] = m
    spec = importlib.util.spec_from_file_location("src.loss.loss_pose", os.path.join(REF_ROOT, "src", "loss", "loss_pose.py"))
    mod = importlib.util.module_from_spec(spec)
    sys.modules[spec.name] = mod
    spec.loader.exec_module(mod)
    return mod


def pairs_of(v):
    return [(a, c) for a in range(v) for c in range(a + 1, v)]


def _rotation(g, angle):
    k = torch.randn(3, generator=g, dtype=torch.float64)
    k = k / k.norm()
    K = torch.tensor([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]], dtype=torch.float64)
    return torch.eye(3, dtype=torch.float64) + math.sin(angle) * K + (1 - math.cos(angle)) * K @ K


def _grid(h, w):
    ys, xs = torch.meshgrid(torch.arange(h, dtype=torch.float64), torch.arange(w, dtype=torch.float64), indexing="ij")
    return torch.stack([(xs.reshape(-1) + 0.5) / w, (ys.reshape(-1) + 0.5) / h], -1)


def _project(abspose, K, depth, i, a, c, h, w):
    """fp64 projection of every pixel of (scene i, view a) into view c: [hw, 2]."""
    T = abspose[i, c] if a == 0 else abspose[i, c] @ torch.linalg.inv(abspose[i, a])
    xy = _grid(h, w)
    X = torch.cat([xy, torch.ones(h * w, 1, dtype=torch.float64)], -1) @ torch.linalg.inv(K[i, a]).T
    X = X * depth[i, a].reshape(-1, 1)
    Q = torch.cat([X, torch.ones(h * w, 1, dtype=torch.float64)], -1) @ T.T
    P = Q[:, :3] / (Q[:, 3:] + 1e-6)
    u = P @ K[i, c].T
    return u[:, :2] / (u[:, 2:] + 1e-6)


def base_case(g, b, v, h, w, max_n=14):
    """Random poses (small rotations), intrinsics, depth and xyz, and per-segment matches: half random pairs of pixels,
    half consistent ones (q = the pixel p's projection lands in) so that both Huber regimes appear."""
    u = lambda *s: torch.rand(*s, generator=g, dtype=torch.float64)
    abspose = torch.eye(4, dtype=torch.float64).repeat(b, v, 1, 1)
    for i in range(b):
        for j in range(v):
            abspose[i, j, :3, :3] = _rotation(g, 0.15 * float(u(1)))
            abspose[i, j, :3, 3] = 0.2 * (u(3) - 0.5)
    K = torch.zeros(b, v, 3, 3, dtype=torch.float64)
    K[..., 0, 0] = 0.9 + 0.2 * u(b, v)
    K[..., 1, 1] = 0.9 + 0.2 * u(b, v)
    K[..., 0, 2] = 0.45 + 0.1 * u(b, v)
    K[..., 1, 2] = 0.45 + 0.1 * u(b, v)
    K[..., 2, 2] = 1.0
    depth = 1.5 + 2.5 * u(b, v, h, w)
    xyz = torch.randn(b, v, 3, h, w, generator=g, dtype=torch.float64)
    pairs = pairs_of(v)
    matches = {}
    for i in range(b):
        for pr in pairs:
            n = int(torch.randint(2, max_n + 1, (1,), generator=g))
            p = torch.randint(0, h * w, (n,), generator=g)
            q = torch.randint(0, h * w, (n,), generator=g)
            pi = _project(abspose, K, depth, i, pr[0], pr[1], h, w)[p]
            col = (pi[:, 0] * w).floor().clamp(0, w - 1).long()
            row = (pi[:, 1] * h).floor().clamp(0, h - 1).long()
            half = n // 2
            q[:half] = (row * w + col)[:half]
            matches[(i, pr)] = [p, q, 0.05 + 0.95 * u(n)]
    conf = 0.2 + 0.8 * u(b, len(pairs))
    return dict(abspose=abspose, K=K, depth=depth, xyz=xyz, matches=matches, conf=conf, b=b, v=v, h=h, w=w)


def _unmatched_pixel(c, i, view, sides=("a",)):
    """A pixel of (scene i, view) that no match reads (as a source, or on either side with sides=('a', 'c'))."""
    used = set()
    for (si, (a, cc)), (p, q, _) in c["matches"].items():
        if si == i and a == view and "a" in sides:
            used.update(p.tolist())
        if si == i and cc == view and "c" in sides:
            used.update(q.tolist())
    return next(k for k in range(c["h"] * c["w"]) if k not in used)


def make_case(name, g):
    if name == "v2_b1_16x20":
        return base_case(g, 1, 2, 16, 20)
    if name == "v3_b2_ragged":
        c = base_case(g, 2, 3, 16, 20)
        m = c["matches"]
        m[(1, (0, 2))] = [x[:0] for x in m[(1, (0, 2))]]                 # an empty segment
        m[(0, (1, 2))] = [x[:1] for x in m[(0, (1, 2))]]                 # a single match
        p, q, w = m[(1, (0, 1))]    # duplicated indices within a segment: repeated (p, q) pairs and a repeated p alone
        m[(1, (0, 1))] = [torch.cat([p, p[:3], p[:1]]), torch.cat([q, q[:3], q[1:2]]), torch.cat([w, w[:3] * 0.5, w[:1]])]
        return c
    if name == "v4_b3_24x24":
        return base_case(g, 3, 4, 24, 24)
    if name == "v4_b1_zero_weights":
        c = base_case(g, 1, 4, 24, 24)
        c["matches"][(0, (1, 3))][2] = torch.zeros_like(c["matches"][(0, (1, 3))][2])
        return c
    if name == "v2_b2_edges":
        c = base_case(g, 2, 2, 16, 20)
        h, w = c["h"], c["w"]
        # scene 0: T = I exactly, so a copied xyz gives a 3-D residual of exactly 0; one point with u_z near -1e-6
        c["abspose"][0, 1] = torch.eye(4, dtype=torch.float64)
        p = torch.tensor([5, 37, 90, 151])
        q = torch.tensor([5, 200, 91, 151])
        c["xyz"][0, 1].view(3, -1)[:, 200] = c["xyz"][0, 0].view(3, -1)[:, 37]
        c["depth"][0, 0].view(-1)[151] = -5e-7
        c["matches"][(0, (0, 1))] = [p, q, torch.tensor([0.3, 0.9, 0.5, 0.2], dtype=torch.float64)]
        # scene 1: T = [I | (tx, 0, 0)], q = p, so |pi - xy(q)| = fx tx / d up to 1e-6 relative: below, at, above delta
        tx = 0.02
        c["abspose"][1, 1] = torch.eye(4, dtype=torch.float64)
        c["abspose"][1, 1, 0, 3] = tx
        c["abspose"][1, 0] = torch.eye(4, dtype=torch.float64)
        fx = float(c["K"][1, 0, 0, 0].float())
        c["K"][1, 1] = c["K"][1, 0]
        px = torch.tensor([10, 60, 140, 250, 300])
        for k, ratio in zip(px.tolist(), (0.999, 1.0, 1.001, 0.5, 3.0)):
            c["depth"][1, 0].view(-1)[k] = fx * tx / (DELTA * ratio)
        c["matches"][(1, (0, 1))] = [px, px.clone(), torch.tensor([0.2, 0.4, 0.6, 0.8, 1.0], dtype=torch.float64)]
        return c
    if name == "v3_b1_nan_depth_unmatched":
        c = base_case(g, 1, 3, 16, 20)
        c["depth"][0, 0].view(-1)[_unmatched_pixel(c, 0, 0)] = float("nan")
        return c
    if name == "v3_b1_inf_depth_unmatched":
        c = base_case(g, 1, 3, 16, 20)
        c["depth"][0, 1].view(-1)[_unmatched_pixel(c, 0, 1)] = float("inf")
        c["depth"][0, 0].view(-1)[_unmatched_pixel(c, 0, 0)] = -float("inf")
        return c
    if name == "v3_b2_nonfinite_depth_matched":
        c = base_case(g, 2, 3, 16, 20)
        c["depth"][1, 0].view(-1)[int(c["matches"][(1, (0, 2))][0][0])] = float("nan")
        c["depth"][0, 1].view(-1)[int(c["matches"][(0, (1, 2))][0][0])] = float("inf")
        c["depth"][0, 0].view(-1)[int(c["matches"][(0, (0, 1))][0][0])] = -float("inf")
        return c
    if name == "v3_b1_nan_xyz_unmatched":
        c = base_case(g, 1, 3, 16, 20)
        k = _unmatched_pixel(c, 0, 1, sides=("a", "c"))
        c["xyz"][0, 1, :, k // c["w"], k % c["w"]] = float("nan")
        return c
    if name in ("v5_b2_ragged", "v6_b1_ragged"):
        b, v = (2, 5) if name == "v5_b2_ragged" else (1, 6)
        c = base_case(g, b, v, 12, 14)
        m = c["matches"]
        m[(b - 1, (1, v - 1))] = [x[:0] for x in m[(b - 1, (1, v - 1))]]      # an empty segment
        m[(0, (v - 2, v - 1))] = [x[:1] for x in m[(0, (v - 2, v - 1))]]      # a single match
        return c
    if name == "v3_b1_signed_weights":
        c = base_case(g, 1, 3, 16, 20)
        m = c["matches"]
        m[(0, (0, 1))][2] = -m[(0, (0, 1))][2]                                # all negative
        w = m[(0, (0, 2))][2]
        w[::2] = -w[::2]                                                      # mixed signs
        m[(0, (1, 2))][2][1] = 0.0                                            # a zero among nonzero weights
        return c
    if name == "v3_b2_clamp":
        # the normaliser's clamp max(sum |w|, 1e-12): one weight exactly float32(1e-12) (equality: clamp_min passes the
        # gradient), one at each float32 neighbour of it, its negative, and several tiny weights summing below 1e-12
        c = base_case(g, 2, 3, 16, 20)
        m = c["matches"]
        e = np.float32(1e-12)
        singles = {(0, (0, 1)): e, (0, (0, 2)): np.nextafter(e, np.float32(1)), (0, (1, 2)): np.nextafter(e, np.float32(0)),
                   (1, (1, 2)): -e}
        for key, val in singles.items():
            m[key] = [x[:1] for x in m[key]]
            m[key][2] = torch.tensor([float(val)], dtype=torch.float64)
        n = len(m[(1, (0, 1))][2])
        m[(1, (0, 1))][2] = torch.full((n,), 1e-14, dtype=torch.float64) * (1 + torch.arange(n) % 3)
        return c
    if name == "v3_b2_nonfinite_weights_conf":
        # one non-finite weight or confidence per segment, segment (1, (1, 2)) clean
        c = base_case(g, 2, 3, 16, 20)
        m = c["matches"]
        m[(0, (0, 1))][2][1] = float("nan")
        m[(0, (0, 2))][2][0] = float("inf")
        c["conf"][0, 2] = float("nan")
        c["conf"][1, 0] = float("inf")
        c["conf"][1, 1] = 0.0
        return c
    if name == "v3_b2_nonfinite_K":
        c = base_case(g, 2, 3, 16, 20)
        c["K"][0, 2, 0, 0] = float("inf")     # view 2 is only ever a target: K_c of pairs (0, 2) and (1, 2)
        c["K"][1, 2, 1, 2] = float("nan")
        return c
    if name == "v3_b2_nonfinite_pose0":
        c = base_case(g, 2, 3, 16, 20)
        c["abspose"][0, 0, 0, 3] = float("nan")  # view 0's pose enters no pair's T (T = c2w[c] for a == 0)
        c["abspose"][1, 0, 1, 1] = float("inf")
        return c
    if name == "v3_b2_nonfinite_pose1":
        c = base_case(g, 2, 3, 16, 20)
        c["abspose"][0, 1, 2, 3] = float("nan")  # view 1's pose goes through .inverse() for pair (1, 2)
        return c
    if name in ("v3_b1_1x37", "v3_b1_37x1"):
        return base_case(g, 1, 3, *((1, 37) if name == "v3_b1_1x37" else (37, 1)))
    raise KeyError(name)


CASES = ("v2_b1_16x20", "v3_b2_ragged", "v4_b3_24x24", "v4_b1_zero_weights", "v2_b2_edges",
         "v3_b1_nan_depth_unmatched", "v3_b1_inf_depth_unmatched", "v3_b2_nonfinite_depth_matched",
         "v3_b1_nan_xyz_unmatched",
         "v5_b2_ragged", "v6_b1_ragged", "v3_b1_signed_weights", "v3_b2_clamp", "v3_b2_nonfinite_weights_conf",
         "v3_b2_nonfinite_K", "v3_b2_nonfinite_pose0", "v3_b2_nonfinite_pose1", "v3_b1_1x37", "v3_b1_37x1")
FIRST_CASES = 9  # the cases first recorded; their arrays are held byte-identical (test_pose_loss_cpu.py)


def packed(c):
    """-> (id_a [M], id_c [M], w [M], counts [S]) in the reference's segment order (scene-major, then pair)."""
    trip = [c["matches"][(i, pr)] for i in range(c["b"]) for pr in pairs_of(c["v"])]
    return (torch.cat([t[0] for t in trip]), torch.cat([t[1] for t in trip]), torch.cat([t[2] for t in trip]),
            torch.tensor([len(t[0]) for t in trip]))


def run_reference(mod, arrays, dtype):
    """Losspose.forward on the recorded (float32-representable) inputs, in `dtype`; loss and gradients."""
    b, v, h, w = (int(arrays[k]) for k in ("b", "v", "height", "width"))
    pairs = pairs_of(v)
    t = lambda k: torch.from_numpy(arrays[k]).to(dtype)
    prev = torch.get_default_dtype()
    torch.set_default_dtype(dtype)
    try:
        abspose = t("abspose").requires_grad_(True)
        depth = t("depth").requires_grad_(True)
        xyz = t("xyz").requires_grad_(True)
        W = t("w").requires_grad_(True)
        C = t("conf").requires_grad_(True)
        id_a, id_c = torch.from_numpy(arrays["id_a"]), torch.from_numpy(arrays["id_c"])
        off = np.concatenate([[0], np.cumsum(arrays["counts"])])
        corre = {pr: [] for pr in pairs}
        s = 0
        for i in range(b):
            for pr in pairs:
                o0, o1 = int(off[s]), int(off[s + 1])
                corre[pr].append((id_a[o0:o1], id_c[o0:o1], W[o0:o1]))
                s += 1
        trans_conf = {pr: C[:, k] for k, pr in enumerate(pairs)}
        relpose = torch.eye(4, dtype=dtype).repeat(b, len(pairs), 1, 1)
        img = torch.zeros(b, v, 3, h, w, dtype=dtype)
        batch = {"context": {"image": img}, "target": {"image": img, "intrinsics": t("K")}}
        loss_fn = mod.Losspose(mod.LossposeCfgWrapper(mod.LossposeCfg(weight_2d=WEIGHT_2D, weight_3d=WEIGHT_3D)))
        loss = loss_fn.forward(None, batch, None, 0, (relpose, abspose), (depth.reshape(b * v, 1, h, w),),
                               (corre, None, trans_conf), xyz)
        grads = torch.autograd.grad(loss, (abspose, depth, xyz, W, C))
    finally:
        torch.set_default_dtype(prev)
    out = dict(loss=loss.detach())
    out.update({f"grad_{k}": gr for k, gr in zip(("abspose", "depth", "xyz", "w", "conf"), grads)})
    return {k: x.detach().numpy() for k, x in out.items()}


def main():
    mod = load_reference_pose_loss()
    arrays = {}
    for n, name in enumerate(CASES):
        g = torch.Generator().manual_seed(3000 + n)
        c = make_case(name, g)
        id_a, id_c, w, counts = packed(c)
        rec = {"abspose": c["abspose"].float(), "depth": c["depth"].float(), "xyz": c["xyz"].float(),
               "K": c["K"].float(), "w": w.float(), "conf": c["conf"].float()}
        rec = {k: x.numpy() for k, x in rec.items()}
        rec.update(id_a=id_a.numpy().astype(np.int64), id_c=id_c.numpy().astype(np.int64),
                   counts=counts.numpy().astype(np.int64), b=np.int64(c["b"]), v=np.int64(c["v"]),
                   height=np.int64(c["h"]), width=np.int64(c["w"]))
        for k, x in rec.items():
            arrays[f"{name}/{k}"] = x
        for tag, dt in (("f32", torch.float32), ("f64", torch.float64)):
            try:
                out = run_reference(mod, rec, dt)
            except Exception:  # e.g. .inverse() of a non-finite pose raising torch.linalg.LinAlgError
                if n < FIRST_CASES:
                    raise
                out = {}
            if n >= FIRST_CASES:
                arrays[f"{name}/{tag}/raises"] = np.bool_(not out)
            for k, x in out.items():
                arrays[f"{name}/{tag}/{k}"] = x
        print(name, "b v h w", c["b"], c["v"], c["h"], c["w"], "M", int(counts.sum()), "loss f64",
              arrays.get(f"{name}/f64/loss"), "f32", arrays.get(f"{name}/f32/loss"))
    path = os.path.join(HERE, "pose_loss.npz")
    np.savez_compressed(path, **arrays)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
