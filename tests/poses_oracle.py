"""fp64 NumPy restatement of the pose path of pf3plat_b200.poses (DESIGN.md 5.14), written from PF3plat's own
functions: camera_synchronization / camera_chaining / SE3_inverse (src/flow_util.py), r6d2mat and plucker_embedding
(src/model/encoder/encoder_costvolume.py) and get_world_rays / sample_image_grid (src/geometry/projection.py).

Pairs are given as a list of (i, j) keys with Ps [pairs, b, 4, 4] and conf [pairs, b] in the same order.  Where the
reference raises (non-finite input to the SVD) this returns what the kernels define: NaN in every output of that scene.
"""
import numpy as np


def se3_inverse(P):
    out = np.array(P, dtype=np.float64, copy=True)
    R = P[..., :3, :3]
    out[..., :3, :3] = np.swapaxes(R, -1, -2)
    out[..., :3, 3] = -np.einsum("...ki,...k->...i", R, P[..., :3, 3])
    return out


def camera_chaining(keys, Ps, N):
    b = Ps.shape[1]
    idx = {k: q for q, k in enumerate(keys)}
    out = [np.broadcast_to(np.eye(4), (b, 4, 4))]
    for k in range(N - 1):
        out.append(Ps[idx[(k, k + 1)]] @ out[-1])
    return np.stack(out, 1)


def build_L(keys, Ps, conf, N, dtype=np.float64):
    """the normalised confidence matrix and L [b, 4N, 4N] of camera_synchronization (flow_util.py:660-697), built in
    `dtype` and returned in fp64.  In float32 every operation is rounded in the kernels' order: the confidences in pair
    order with c/2 added on both diagonals, each column summed top to bottom, t_inv = ((-r0 t0) + (-r1 t1)) + (-r2 t2)."""
    Ps, conf = np.asarray(Ps, dtype), np.asarray(conf, dtype)
    b, half = Ps.shape[1], dtype(2)
    C = np.zeros((b, N, N), dtype)
    with np.errstate(all="ignore"):
        for q, (i, j) in enumerate(keys):
            C[:, i, j] = conf[q]
            C[:, j, i] = conf[q]
            C[:, i, i] = C[:, i, i] + conf[q] / half
            C[:, j, j] = C[:, j, j] + conf[q] / half
        for j in range(N):
            s = np.zeros(b, dtype)
            for i in range(N):
                s = s + C[:, i, j]
            s = np.where(s < dtype(1e-9), dtype(1e-9), s)  # clamp(min=1e-9); NaN passes
            C[:, :, j] = C[:, :, j] / s[:, None]
        L = np.zeros((b, N, 4, N, 4), dtype)
        for i in range(N):
            L[:, i, :, i, :] = C[:, i, i, None, None] * np.eye(4, dtype=dtype)
        for q, (i, j) in enumerate(keys):
            P = Ps[q]
            inv = np.array(P, copy=True)
            inv[:, :3, :3] = np.swapaxes(P[:, :3, :3], -1, -2)
            for r in range(3):
                inv[:, r, 3] = ((-P[:, 0, r]) * P[:, 0, 3] + (-P[:, 1, r]) * P[:, 1, 3]) + (-P[:, 2, r]) * P[:, 2, 3]
            L[:, i, :, j, :] = C[:, i, j, None, None] * inv
            L[:, j, :, i, :] = C[:, j, i, None, None] * P
    return C, L.reshape(b, 4 * N, 4 * N).astype(np.float64)


def so3_project(M):
    """U diag(1, 1, det(U V^T)) V^T.  Unique where M has rank >= 2; for rank <= 1 the SVD's basis is arbitrary, and the
    tests pin those blocks to the recorded reference (the zero block: I, from LAPACK's SVD of zeros) or to properties"""
    U, _, Vt = np.linalg.svd(M)
    d = np.linalg.det(U @ Vt)
    return (U * np.stack([np.ones_like(d), np.ones_like(d), d], -1)[..., None, :]) @ Vt


def power_column_block(keys, Ps, conf, N, squares=10, l_dtype=np.float64):
    """L^(2^squares), column block 0, [b, N, 4, 4], and per scene whether L or that block holds a non-finite value"""
    _, L = build_L(keys, Ps, conf, N, l_dtype)
    bad = ~np.isfinite(L).all(axis=(1, 2))
    with np.errstate(all="ignore"):
        for _ in range(squares):
            L = L @ L
    blk = L.reshape(-1, N, 4, N, 4)[:, :, :, 0, :]
    bad |= ~np.isfinite(blk).all(axis=(1, 2, 3))
    return blk, bad


def camera_synchronization(keys, Ps, conf, N, l_dtype=np.float64):
    """l_dtype = np.float64 is the reference run in float64; np.float32 is what the reference and the kernels compute
    from float32 inputs: L built in float32, then squared in fp64.  The synchronised translations are ill-conditioned
    (about 1 / (1 - the rotation blocks' top eigenvalue)), so the two differ by far more than float32 rounding."""
    if N == 2:
        return camera_chaining(keys, np.asarray(Ps, dtype=np.float64), N)
    blk, bad = power_column_block(keys, Ps, conf, N, l_dtype=l_dtype)
    Ps = np.asarray(Ps, dtype=np.float64)
    mass = blk[:, :, 3, 3]
    masses = np.where(bad[:, None], np.nan, mass)
    if np.min(masses) == 0:  # np.min propagates NaN, as torch.min does
        return camera_chaining(keys, Ps, N)
    out = np.full(blk.shape, np.nan)
    good = ~bad
    Lg = blk[good] / np.maximum(mass[good], 1e-9)[..., None, None]
    Lg[..., :3, :3] = so3_project(Lg[..., :3, :3])
    out[good] = Lg
    return out


# ---- refined poses ----

EPS = 1e-12


def refine_forward(pose_enc, delta, gamma):
    """encoder_costvolume.py:465-473, then .inverse(): (abspose, abspose_inv) [b, v, 4, 4] and the intermediates"""
    x = np.array(pose_enc, dtype=np.float64, copy=True)
    x[:, 1:] += np.asarray(delta, dtype=np.float64)[:, 1:] * float(gamma)
    a1, a2 = x[..., :3], x[..., 3:6]
    n1 = np.linalg.norm(a1, axis=-1, keepdims=True)
    b1 = a1 / np.maximum(n1, EPS)
    s = (b1 * a2).sum(-1, keepdims=True)
    c = a2 - s * b1
    n2 = np.linalg.norm(c, axis=-1, keepdims=True)
    b2 = c / np.maximum(n2, EPS)
    b3 = np.cross(b1, b2)
    A = np.zeros(x.shape[:2] + (4, 4))
    A[..., 0, :3], A[..., 1, :3], A[..., 2, :3] = b1, b2, b3
    A[..., :3, 3] = x[..., 6:9]
    A[..., 3, 3] = 1.0
    with np.errstate(all="ignore"):
        Ai = np.linalg.inv(A) if np.isfinite(A).all() and (np.abs(np.linalg.det(A)) > 0).all() else _inv_or_nan(A)
    return A, Ai, dict(x=x, n1=n1, b1=b1, s=s, n2=n2, b2=b2, b3=b3)


def _inv_or_nan(A):
    out = np.full(A.shape, np.nan)
    for idx in np.ndindex(A.shape[:-2]):
        try:
            out[idx] = np.linalg.inv(A[idx])
        except np.linalg.LinAlgError:
            pass
    return out


def _normalize_bwd(y, n, g):
    return np.where(n >= EPS, (g - y * (y * g).sum(-1, keepdims=True)) / np.maximum(n, EPS), g / EPS)


def refine_backward(pose_enc, delta, gamma, g_abs, g_inv):
    """gradients of sum(abspose * g_abs + abspose_inv * g_inv) with respect to (pose_enc, delta, gamma); g_inv None
    leaves the inverse out (its gradient stays finite where abspose is singular)"""
    A, Ai, f = refine_forward(pose_enc, delta, gamma)
    G = np.array(g_abs, dtype=np.float64)
    if g_inv is not None:
        AiT = np.swapaxes(Ai, -1, -2)
        G = G - AiT @ np.asarray(g_inv, dtype=np.float64) @ AiT
    gb1, gb2, gb3 = G[..., 0, :3].copy(), G[..., 1, :3].copy(), G[..., 2, :3]
    gx = np.zeros(f["x"].shape)
    gx[..., 6:9] = G[..., :3, 3]
    gb1 += np.cross(f["b2"], gb3)
    gb2 += np.cross(gb3, f["b1"])
    gc = _normalize_bwd(f["b2"], f["n2"], gb2)
    gcb1 = (gc * f["b1"]).sum(-1, keepdims=True)
    gx[..., 3:6] = gc - gcb1 * f["b1"]
    gb1 += -f["s"] * gc - gcb1 * f["x"][..., 3:6]
    gx[..., :3] = _normalize_bwd(f["b1"], f["n1"], gb1)
    d_delta = gx * float(gamma)
    d_delta[:, 0] = 0.0
    d_gamma = float((gx[:, 1:] * np.asarray(delta, dtype=np.float64)[:, 1:]).sum())
    return gx, d_delta, d_gamma


# ---- Plücker rays ----

def plucker_rays(abspose, intrinsics, h, w):
    """[(b v), 6, h, w]: (d, o x d) with d = c2w[:3, :3] normalise(K^-1 [x, y, 1]) on the pixel-centre grid"""
    abspose = np.asarray(abspose, dtype=np.float64)
    b, v = abspose.shape[:2]
    with np.errstate(all="ignore"):
        c2w = _inv_or_nan(abspose.reshape(-1, 4, 4))
        kinv = _inv_or_nan(np.asarray(intrinsics, dtype=np.float64).reshape(-1, 3, 3))
        ys, xs = np.meshgrid((np.arange(h) + 0.5) / h, (np.arange(w) + 0.5) / w, indexing="ij")
        pix = np.stack([xs, ys, np.ones_like(xs)], -1).reshape(-1, 3)  # [hw, 3], row-major pixels
        d = np.einsum("nij,pj->npi", kinv, pix)
        d = d / np.linalg.norm(d, axis=-1, keepdims=True)
        dh = np.concatenate([d, np.zeros_like(d[..., :1])], -1)
        dw = np.einsum("nij,npj->npi", c2w, dh)[..., :3]
        o = np.broadcast_to(c2w[:, None, :3, 3], dw.shape)
        out = np.concatenate([dw, np.cross(o, dw)], -1)
    return out.reshape(b * v, h, w, 6).transpose(0, 3, 1, 2)
