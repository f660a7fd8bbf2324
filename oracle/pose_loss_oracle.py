"""fp64 restatement of PF3plat's correspondence (pose) loss, for the parity tests of pf3plat_b200.losses.pose_loss.

TEST INFRASTRUCTURE ONLY (imported by tests/, never by the product path).

Semantics of src/loss/loss_pose.py:29-129, written independently here and vectorised over every (scene, pair)
segment.  Pairs [(a, c) for a < c]; segment s = scene * pairs + pair.  Per segment:
  T_s = c2w[c] (a == 0) or c2w[c] @ inverse(c2w[a]),  the grid x(p) = ((p mod w) + 0.5) / w, y(p) = ((p div w) + 0.5) / h
  dense projection of EVERY pixel of the source view a (as the reference computes it, then gathers):
    X = d_a K_a^-1 [x, y, 1],  Q = T_s [X, 1],  P = Q_xyz / (Q_w + 1e-6),  u = K_c P,  pi = u_xy / (u_z + 1e-6)
  L2_s = sum_n huber_0.01(|pi(p_n) - xy(q_n)|) / 0.01
  L3_s = conf_s sum_n (w_n / max(sum |w|, eps)) |R_s xyz_a(p_n) + t_s - xyz_c(q_n)|
  loss = weight_3d mean_s L3_s + weight_2d mean_s L2_s.
The clamp's eps is F.normalize's 1e-12.  The reference trains in float32, where the bound is float32(1e-12) =
9.99999996e-13 < 1e-12: a segment whose |w| sum is exactly float32(1e-12) passes the clamp in float32 (clamp_min passes
its gradient at equality) and is clamped in float64.  `EPS_N` reproduces the float64 record, `EPS_N_F32` the float32
one, which is the truth the kernels follow; `clamp_fragile` names the segments whose sum lies within float32 rounding
of that bound, where no precision's answer is the reference's.
Gradients are autograd's through these ops.  The dense projection is kept on purpose: the zero gradient the gather sends
to an unmatched pixel meets that pixel's projection in the backward, so a non-finite depth there makes dL/ddepth and
dL/dT_s non-finite exactly as in the reference.  Works on any device and dtype (the tests use float64).
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

DELTA = 0.01
EPS_H = 1e-6
EPS_N = 1e-12
EPS_N_F32 = float(np.float32(1e-12))


def pairs_of(v: int):
    return [(a, c) for a in range(v) for c in range(a + 1, v)]


def relative_poses(abspose: torch.Tensor) -> torch.Tensor:
    """[b, v, 4, 4] -> T [b, pairs, 4, 4]."""
    v = abspose.shape[1]
    return torch.stack([abspose[:, c] if a == 0 else abspose[:, c] @ torch.linalg.inv(abspose[:, a])
                        for a, c in pairs_of(v)], dim=1)


def grid(h: int, w: int, dtype=torch.float64, device=None) -> torch.Tensor:
    """[h*w, 2] pixel-centre (x, y), computed in `dtype`."""
    ys, xs = torch.meshgrid(torch.arange(h, device=device), torch.arange(w, device=device), indexing="ij")
    return torch.stack([(xs.reshape(-1).to(dtype) + 0.5) / w, (ys.reshape(-1).to(dtype) + 0.5) / h], dim=-1)


def pack(matches, conf, b, v):
    """Match lists -> (segment id [M], id_a [M], id_c [M], w [M], conf [S]); segments scene-major, then pair."""
    pairs = pairs_of(v)
    trip = [matches[pr][i] for i in range(b) for pr in pairs]
    sid = torch.cat([torch.full((t[0].shape[0],), s, dtype=torch.int64, device=t[0].device) for s, t in enumerate(trip)])
    id_a = torch.cat([t[0].reshape(-1) for t in trip]).long()
    id_c = torch.cat([t[1].reshape(-1) for t in trip]).long()
    w = torch.cat([t[2].reshape(-1) for t in trip])
    cf = torch.stack([conf[pr] for pr in pairs], dim=1).reshape(-1)
    return sid, id_a, id_c, w, cf


def segment_terms(abspose, depth, xyz, K, sid, id_a, id_c, w, cf, h, w_, xy=None, eps=EPS_N):
    """-> (L3 [S], L2 [S]).  abspose [b,v,4,4], depth [b*v,...,h,w], xyz [b,v,3,h,w], K [b,v,3,3]; the packed matches."""
    b, v = abspose.shape[:2]
    pairs = pairs_of(v)
    P, S, hw = len(pairs), b * len(pairs), h * w_
    dt = abspose.dtype
    w, cf = w.to(dt), cf.to(dt)
    if xy is None:
        xy = grid(h, w_, dt, abspose.device)
    T = relative_poses(abspose)                                                   # [b, P, 4, 4]
    pa = [a for a, _ in pairs]
    pc = [c for _, c in pairs]
    Kinv = torch.linalg.inv(K)
    d = depth.reshape(b, v, hw)
    ray = torch.cat([xy, torch.ones_like(xy[:, :1])], -1)                          # [hw, 3]
    X = (ray @ Kinv[:, pa].transpose(-1, -2)) * d[:, pa, :, None]                  # [b, P, hw, 3]
    Q = torch.cat([X, torch.ones_like(X[..., :1])], -1) @ T.transpose(-1, -2)      # [b, P, hw, 4]
    P3 = Q[..., :3] / (Q[..., 3:] + EPS_H)
    u = P3 @ K[:, pc].transpose(-1, -2)
    pi = u[..., :2] / (u[..., 2:] + EPS_H)                                         # [b, P, hw, 2]
    scene = sid // P
    pair = sid % P
    a_n = torch.tensor(pa, device=sid.device)[pair]
    c_n = torch.tensor(pc, device=sid.device)[pair]
    proj = pi.reshape(S * hw, 2)[sid * hw + id_a]
    e2 = (proj - xy[id_c]).norm(dim=-1)
    h2 = F.huber_loss(e2, torch.zeros_like(e2), reduction="none", delta=DELTA) / DELTA
    L2 = torch.zeros(S, dtype=dt, device=h2.device).index_add(0, sid, h2)
    xf = xyz.reshape(b, v, 3, hw)
    xa = xf[scene, a_n, :, id_a]
    xc = xf[scene, c_n, :, id_c]
    Tn = T.reshape(S, 4, 4)[sid]
    e3 = ((Tn[:, :3, :3] @ xa[:, :, None])[..., 0] + Tn[:, :3, 3] - xc).norm(dim=-1)
    D = torch.zeros(S, dtype=dt, device=w.device).index_add(0, sid, w.abs()).clamp_min(eps)
    L3 = cf * torch.zeros(S, dtype=dt, device=w.device).index_add(0, sid, w / D[sid] * e3)
    return L3, L2


def pose_loss(abspose, depth, xyz, K, matches, conf, h, w, weight_2d=0.005, weight_3d=0.025, xy=None):
    """Losspose.forward's value from its inputs (any dtype; autograd flows to abspose, depth, xyz, the weights, conf)."""
    b, v = abspose.shape[:2]
    sid, id_a, id_c, wt, cf = pack(matches, conf, b, v)
    L3, L2 = segment_terms(abspose, depth, xyz, K, sid, id_a, id_c, wt, cf, h, w, xy)
    return L3.mean() * weight_3d + L2.mean() * weight_2d


def loss_and_grads(abspose, depth, xyz, K, matches, conf, h, w, weight_2d=0.005, weight_3d=0.025, dtype=torch.float64,
                   eps=EPS_N):
    """-> dict of the loss and its gradients w.r.t. abspose, depth, xyz, w (packed [M]) and conf ([S]), in `dtype`."""
    b, v = abspose.shape[:2]
    leaf = lambda t: t.detach().to(dtype).clone().requires_grad_(True)
    A, Dp, Xy = leaf(abspose), leaf(depth), leaf(xyz)
    sid, id_a, id_c, wt, cf = pack(matches, conf, b, v)
    wt, cf = leaf(wt), leaf(cf)
    L3, L2 = segment_terms(A, Dp, Xy, K.detach().to(dtype), sid, id_a, id_c, wt, cf, h, w, eps=eps)
    loss = L3.mean() * weight_3d + L2.mean() * weight_2d
    gA, gD, gX, gW, gC = torch.autograd.grad(loss, (A, Dp, Xy, wt, cf))
    return {"loss": loss.detach(), "L3": L3.detach(), "L2": L2.detach(), "abspose": gA, "depth": gD, "xyz": gX,
            "w": gW, "conf": gC}


def terms_and_grads(abspose, depth, xyz, K, matches, conf, h, w, g3, g2, dtype=torch.float64, eps=EPS_N_F32):
    """-> dict of L3 [S], L2 [S] and the gradients of sum(g3 L3) + sum(g2 L2) w.r.t. abspose, depth, xyz, w and conf.

    g3 / g2 are per-segment cotangents [S].  None means the term is absent, and an absent term is a zero cotangent
    through the reference's chain (so 0 x NaN = NaN wherever that chain meets a non-finite value), which is what
    Losspose itself computes with a weight of 0, and what pf3plat_b200.losses.pose_terms gives when only one of its
    outputs reaches the loss."""
    b, v = abspose.shape[:2]
    leaf = lambda t: t.detach().to(dtype).clone().requires_grad_(True)
    A, Dp, Xy = leaf(abspose), leaf(depth), leaf(xyz)
    sid, id_a, id_c, wt, cf = pack(matches, conf, b, v)
    wt, cf = leaf(wt), leaf(cf)
    L3, L2 = segment_terms(A, Dp, Xy, K.detach().to(dtype), sid, id_a, id_c, wt, cf, h, w, eps=eps)
    cot = lambda g, L: torch.zeros_like(L) if g is None else g.detach().to(device=L.device, dtype=dtype)
    gA, gD, gX, gW, gC = torch.autograd.grad((L3, L2), (A, Dp, Xy, wt, cf), (cot(g3, L3), cot(g2, L2)))
    return {"L3": L3.detach(), "L2": L2.detach(), "abspose": gA, "depth": gD, "xyz": gX, "w": gW, "conf": gC}


def clamp_fragile(matches, b, v, eps=EPS_N_F32):
    """-> bool [S]: segments whose sum |w| lies within float32 rounding of the clamp's bound (a float32 sum of n terms
    may be off by (n - 1) 2^-24 of the sum), so that which side of the clamp they fall on depends on the summation.
    A sum of one weight is exact: a single weight at the bound is not fragile."""
    sid, _, _, wt, _ = pack(matches, {pr: torch.zeros(b) for pr in pairs_of(v)}, b, v)
    S = b * len(pairs_of(v))
    wt = wt.detach().double().cpu()
    sid = sid.cpu()
    tot = torch.zeros(S, dtype=torch.float64).index_add(0, sid, wt.abs())
    n = torch.zeros(S, dtype=torch.float64).index_add(0, sid, torch.ones_like(wt))
    return (tot - eps).abs() < (n - 1).clamp_min(0) * 2.0 ** -24 * tot
