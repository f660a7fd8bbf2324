"""The pose path's kernels (csrc/gs_poses.cu) past the inputs PF3plat's training step produces, with every torch.empty
poisoned (tests/poison.py) so that an element a kernel leaves unwritten reads as NaN: every golden case added after the
first sixteen (sparse, ring, shuffled and reversed pair graphs, N = 16, chaining through 15 pairs, a NaN scene next to a
zero-mass scene, a negative mass, rotation blocks of exact rank 2 and 0, degenerate 6-d encodings, pixel-unit
intrinsics); seeded sparse, ring, star-plus-chain and shuffled graphs for N = 3..16; chaining with the zero-mass scene
last of 1000; batches at the ABI's limit checked against the same inputs in chunks; refine_poses at 2^20 items; a rank-1
block; and the Plücker rays at the grid's limit, on frames one pixel high or wide, on a frame of a million pixels and
next to non-finite poses.  Bounds as in test_gpu_poses.py: values within 1e-5 (|ref| + 1), gradients within
1e-3 (|ref| + rms ref), the same non-finite elements; the synchronisation against the oracle with L built in float32,
and against the fp64 record at the bound plus twice the reference float32 route's own distance from it."""
import itertools

import numpy as np
import pytest
import torch

from tests import poses_oracle as O
from tests.poison import poisoned  # noqa: F401  (fixture)
from tests.test_gpu_poses import grad_ratio, refine_run, run_sync, sync_inputs, value_ratio
from tests.test_poses_cpu import CASES, FIRST_CASES, PLUCKER, REFINE_DEGENERATE, SYNC, keys_of, singular_items

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
NEW_SYNC = [n for n in SYNC if n not in FIRST_CASES]
NEW_PLUCKER = [n for n in PLUCKER if n not in FIRST_CASES]


def report(group, **ratios):
    print(f"{group}: " + ", ".join(f"{k} {v:.3f}" for k, v in ratios.items()))


# ---- golden cases ----

@pytest.mark.parametrize("name", NEW_SYNC)
def test_new_sync_cases(name, poisoned):  # noqa: F811
    c = CASES[name]
    keys, N = keys_of(c), int(c["N"])
    got = run_sync(keys, c["Ps"], c["conf"], N)
    r = value_ratio(got, O.camera_synchronization(keys, c["Ps"], c["conf"], N, l_dtype=np.float32))
    if c["raises64"]:  # the reference raises on the NaN scene; the oracle defines the answer
        bad = ~np.isfinite(c["conf"]).all(axis=0)
        assert np.isnan(got[bad]).all() and np.isfinite(got[~bad]).all()
        report(name, oracle=r)
        assert r <= 1.0
        return
    r64 = value_ratio(got, c["value64"])
    ref32 = value_ratio(c["value32"], c["value64"])
    report(name, oracle=r, record64=r64, reference32=ref32)
    assert r <= 1.0 and r64 <= 1.0 + 2.0 * ref32
    if name in ("sync_rank2", "sync_rank0"):  # pinned to the record itself: the projection's basis comes from the SVD
        assert value_ratio(got, c["value32"]) <= 1.0
        R = got[..., :3, :3].astype(np.float64)
        assert np.allclose(R @ np.swapaxes(R, -1, -2), np.eye(3), atol=1e-6)
        assert np.allclose(np.linalg.det(R), 1.0, atol=1e-6)


@pytest.mark.parametrize("name", REFINE_DEGENERATE)
def test_degenerate_encodings(name, poisoned):  # noqa: F811
    """forward, and backward with cotangents on abspose only: |a1| = 0 or below eps, c exactly 0, |c| either side of
    eps, one view, a negative gamma"""
    c = CASES[name]
    A, Ai, gp, gd, gg = refine_run(c["pose_enc"], c["delta"], c["gamma"], c["g_abs"], None)
    oA, oAi, _ = O.refine_forward(c["pose_enc"], c["delta"], c["gamma"])
    op, od, og = O.refine_backward(c["pose_enc"], c["delta"], c["gamma"], c["g_abs"], None)
    sing = singular_items(c)
    rv = max(value_ratio(A, oA), value_ratio(A, c["abspose64"]))
    if c["raises64"]:  # the reference's .inverse() raises: the singular items' inverse is non-finite, the rest kept
        assert not np.isfinite(Ai[sing]).any()
        rv = max(rv, value_ratio(Ai[~sing], oAi[~sing]))
    else:
        rv = max(rv, value_ratio(Ai, oAi), value_ratio(Ai, c["abspose_inv64"]))
    rg = max(grad_ratio(gp, op), grad_ratio(gd, od), grad_ratio(np.array(gg), np.array(og)),
             grad_ratio(gp, c["d_pose_enc64"]), grad_ratio(gd, c["d_delta64"]),
             grad_ratio(np.array(gg), c["d_gamma64"]))
    report(name, values=rv, gradients=rg)
    assert rv <= 1.0 and rg <= 1.0


@pytest.mark.parametrize("name", NEW_PLUCKER)
def test_new_plucker_cases(name, poisoned):  # noqa: F811
    from pf3plat_b200.poses import plucker_rays
    c = CASES[name]
    h, w = int(c["h"]), int(c["w"])
    got = plucker_rays(torch.tensor(c["abspose"], device=DEV), torch.tensor(c["intrinsics"], device=DEV), h, w)
    got = got.cpu().numpy()
    r = max(value_ratio(got, O.plucker_rays(c["abspose"], c["intrinsics"], h, w)), value_ratio(got, c["value64"]))
    report(name, values=r)
    assert r <= 1.0


# ---- seeded pair graphs ----

def rotations(rng, n, max_angle):
    """n Rodrigues rotations about random axes by angles in (0.3, 1) max_angle, vectorised"""
    k = rng.normal(size=(n, 3))
    k /= np.linalg.norm(k, axis=-1, keepdims=True)
    a = max_angle * rng.uniform(0.3, 1.0, size=(n, 1, 1))
    K = np.zeros((n, 3, 3))
    K[:, 0, 1], K[:, 0, 2], K[:, 1, 2] = -k[:, 2], k[:, 1], -k[:, 0]
    K -= np.swapaxes(K, -1, -2)
    return np.eye(3) + np.sin(a) * K + (1 - np.cos(a)) * K @ K


def rigids(rng, n, rot, trans):
    P = np.broadcast_to(np.eye(4), (n, 4, 4)).copy()
    P[:, :3, :3] = rotations(rng, n, rot)
    P[:, :3, 3] = rng.normal(size=(n, 3)) * trans
    return P


def seeded_graph(keys, b, N, seed):
    """as test_gpu_poses.seeded_sync on any keys: noisy pairwise transforms i -> j, the encoder's relu rescale"""
    rng = np.random.default_rng(seed)
    W = np.concatenate([np.broadcast_to(np.eye(4), (b, 1, 4, 4)),
                        rigids(rng, b * (N - 1), 0.3, 0.3).reshape(b, N - 1, 4, 4)], 1)
    Wi = np.linalg.inv(W)
    Ps = np.stack([W[:, j] @ Wi[:, i] @ rigids(rng, b, 0.03, 0.03) for i, j in keys])
    cc = rng.uniform(0.55, 0.95, size=(len(keys), b))
    far = np.array([abs(i - j) > 1 for i, j in keys])[:, None]
    conf = np.where(far, np.maximum(cc - 0.5, 0.0) / 0.5, cc)
    return Ps.astype(np.float32), conf.astype(np.float32)


def graph(kind, N, rng):
    chain = [(k, k + 1) for k in range(N - 1)]
    off = [(i, j) for i, j in itertools.combinations(range(N), 2) if j - i > 1]
    if kind == "sparse":  # the chain and a random third of the other pairs
        keys = chain + [p for p in off if rng.random() < 1 / 3]
    elif kind == "ring":
        keys = chain + ([(N - 1, 0)] if N > 2 else [])
    elif kind == "star_chain":  # the chain and every (0, k), half of them stored as (k, 0)
        keys = chain + [(k, 0) if rng.random() < 0.5 else (0, k) for k in range(2, N)]
    else:  # every pair, shuffled, off-chain pairs reversed at random
        keys = chain + [(j, i) if rng.random() < 0.5 else (i, j) for i, j in off]
    return [keys[q] for q in rng.permutation(len(keys))]


@pytest.mark.parametrize("kind", ["sparse", "ring", "star_chain", "shuffled"])
def test_seeded_graphs(kind, poisoned):  # noqa: F811
    worst = 0.0
    for N in range(3, 17):
        rng = np.random.default_rng(1000 * N + len(kind))
        keys = graph(kind, N, rng)
        Ps, conf = seeded_graph(keys, 3, N, seed=N)
        got = run_sync(keys, Ps, conf, N)
        assert np.isfinite(got).all(), (kind, N)
        r = value_ratio(got, O.camera_synchronization(keys, Ps, conf, N, l_dtype=np.float32))
        assert r <= 1.0, (kind, N, keys, r)
        worst = max(worst, r)
    report(f"{kind} graphs, N = 3..16", oracle=worst)


@pytest.mark.parametrize("N", [4, 8, 16])
def test_chaining_with_the_zero_mass_scene_last_of_1000(N, poisoned):  # noqa: F811
    rng = np.random.default_rng(N)
    keys = graph("shuffled", N, rng)
    Ps, conf = seeded_graph(keys, 1000, N, seed=50 + N)
    healthy = run_sync(keys, Ps, conf, N)
    conf[:, 999] = 0.0
    got = run_sync(keys, Ps, conf, N)
    r = value_ratio(got, O.camera_chaining(keys, Ps.astype(np.float64), N))
    report(f"chaining N = {N}, b = 1000", chained=r)
    assert r <= 1.0
    assert value_ratio(healthy[:64], O.camera_synchronization(keys, Ps[:, :64], conf[:, :64], N,
                                                              l_dtype=np.float32)) <= 1.0
    assert not np.allclose(healthy[0], got[0], atol=1e-3)


@pytest.mark.parametrize("order", ["nan_first", "zero_first"])
def test_a_nan_scene_keeps_a_zero_mass_scene_from_chaining_the_batch(order, poisoned):  # noqa: F811
    N = 5
    keys = graph("shuffled", N, np.random.default_rng(7))
    Ps, conf = seeded_graph(keys, 8, N, seed=7)
    nan_s, zero_s = (1, 6) if order == "nan_first" else (6, 1)
    conf[3, nan_s] = np.nan
    conf[:, zero_s] = 0.0
    got = run_sync(keys, Ps, conf, N)
    oracle = O.camera_synchronization(keys, Ps, conf, N, l_dtype=np.float32)
    r = value_ratio(got, oracle)
    report(f"NaN and zero-mass scenes, {order}", oracle=r)
    assert r <= 1.0
    assert np.isnan(got[nan_s]).all() and np.isfinite(np.delete(got, nan_s, 0)).all()
    # the zero-mass scene is synchronised, not chained: an all-zero block projects to I with a zero translation
    assert np.array_equal(got[zero_s], np.broadcast_to(np.diag([1, 1, 1, 0]).astype(np.float32), (N, 4, 4)))
    chained = O.camera_chaining(keys, Ps.astype(np.float64), N)
    assert not np.allclose(got[0], chained[0], atol=1e-3)


def test_negative_and_tiny_masses(poisoned):  # noqa: F811
    """a view whose confidences sum below zero (its mass ends negative) and a view held by one confidence of 3e-10
    (its mass ends in (0, 1e-9)): both are divided by the clamp's 1e-9, and neither chains the batch"""
    N = 5
    keys = [(0, 1), (1, 2), (2, 3), (3, 4), (0, 2), (2, 4), (1, 4)]
    Ps, conf = seeded_graph(keys, 6, N, seed=11)
    q = {k: i for i, k in enumerate(keys)}
    conf[q[(3, 4)], 1], conf[q[(2, 4)], 1], conf[q[(1, 4)], 1] = 1e-10, -2e-10, 0.0
    conf[q[(3, 4)], 4], conf[q[(2, 4)], 4], conf[q[(1, 4)], 4] = 3e-10, 0.0, 0.0
    blk, bad = O.power_column_block(keys, Ps, conf, N, l_dtype=np.float32)
    mass = blk[..., 3, 3]
    assert not bad.any() and mass[1, 4] < 0 and 0 < mass[4, 4] < 1e-9 and (np.delete(mass, [1, 4], 0) > 1e-3).all()
    got = run_sync(keys, Ps, conf, N)
    r = value_ratio(got, O.camera_synchronization(keys, Ps, conf, N, l_dtype=np.float32))
    report("negative and tiny masses", oracle=r)
    assert r <= 1.0 and np.isfinite(got).all()


def test_a_rank_one_block_projects_to_a_proper_rotation(poisoned):  # noqa: F811
    """pairwise rotation parts D_j D_i diag(1, 0, 0): every synchronised block is diag(+-m, 0, 0).  The SVD's basis of
    the null plane is arbitrary, so the result is held to what any valid answer satisfies: orthonormal, det 1, and R
    maps the block's one singular direction onto its image; translations against the oracle"""
    N, b = 4, 3
    keys = list(itertools.combinations(range(N), 2))
    rng = np.random.default_rng(12)
    flips = [np.diag(d).astype(np.float64) for d in ((1, 1, 1), (1, -1, -1), (-1, 1, -1), (-1, -1, 1))]
    Ps = np.zeros((len(keys), b, 4, 4), np.float32)
    conf = rng.uniform(0.55, 0.95, size=(len(keys), b)).astype(np.float32)
    for s in range(b):
        D = [flips[0]] + [flips[k] for k in rng.integers(0, 4, N - 1)]
        for q, (i, j) in enumerate(keys):
            Ps[q, s] = np.eye(4)
            Ps[q, s, :3, :3] = D[j] @ D[i] @ np.diag([1.0, 0.0, 0.0])
            Ps[q, s, :3, 3] = rng.normal(size=3) * 0.3
    blk, _ = O.power_column_block(keys, Ps, conf, N, l_dtype=np.float32)
    M = blk[..., :3, :3] / blk[..., 3:, 3:]
    assert (np.linalg.svd(M, compute_uv=False)[..., 1:] == 0).all() and (np.abs(M[..., 0, 0]) > 0.1).all()
    got = run_sync(keys, Ps, conf, N)
    assert np.isfinite(got).all()
    R = got[..., :3, :3].astype(np.float64)
    assert np.allclose(R @ np.swapaxes(R, -1, -2), np.eye(3), atol=1e-6)
    assert np.allclose(np.linalg.det(R), 1.0, atol=1e-6)
    assert np.allclose(R[..., 0, 0], np.sign(M[..., 0, 0]), atol=1e-6)  # R e0 = sign(m) e0
    oracle = O.camera_synchronization(keys, Ps, conf, N, l_dtype=np.float32)
    assert value_ratio(got[..., :, 3], oracle[..., :, 3]) <= 1.0


@pytest.mark.parametrize("b,N", [(65535, 3), (4096, 16)])
def test_sync_at_the_batch_limit(b, N, poisoned):  # noqa: F811
    """64 scenes against the oracle; every scene bit for bit against the same inputs run 1024 scenes at a time"""
    from pf3plat_b200.poses import camera_synchronization
    keys = list(itertools.combinations(range(N), 2))
    Ps, conf = seeded_graph(keys, b, N, seed=b + N)
    P, C = sync_inputs(keys, Ps, conf)
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    camera_synchronization(P, C, N)
    start.record()
    got = camera_synchronization(P, C, N)
    end.record()
    torch.cuda.synchronize()
    parts = [camera_synchronization({k: v[s:s + 1024] for k, v in P.items()}, {k: v[s:s + 1024] for k, v in C.items()},
                                    N) for s in range(0, b, 1024)]
    assert torch.equal(got, torch.cat(parts))
    sample = np.sort(np.random.default_rng(b).choice(b, 64, replace=False))
    sample[-1] = b - 1
    got = got.cpu().numpy()
    r = value_ratio(got[sample], O.camera_synchronization(keys, Ps[:, sample], conf[:, sample], N, l_dtype=np.float32))
    report(f"sync b = {b}, N = {N}", oracle=r, ms=start.elapsed_time(end))
    assert r <= 1.0 and np.isfinite(got).all()


# ---- refine_poses and Plücker rays at scale ----

def test_refine_at_a_million_items(poisoned):  # noqa: F811
    from pf3plat_b200.poses import refine_poses
    b, v = 1 << 18, 4
    rng = np.random.default_rng(20)
    R = rotations(rng, b * v, 1.0)
    enc = np.concatenate([R[:, :2].reshape(b, v, 6), rng.normal(size=(b, v, 3))], -1).astype(np.float32)
    delta = (rng.normal(size=(b, v, 9)) * 0.1).astype(np.float32)
    ga, gi = (rng.normal(size=(b, v, 4, 4)).astype(np.float32) for _ in range(2))
    p = torch.tensor(enc, device=DEV, requires_grad=True)
    d = torch.tensor(delta, device=DEV, requires_grad=True)
    g = torch.tensor(0.9, device=DEV, requires_grad=True)
    A, Ai = refine_poses(p, d, g)
    gA, gAi = torch.tensor(ga, device=DEV), torch.tensor(gi, device=DEV)
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    torch.autograd.backward([A, Ai], [gA, gAi])
    end.record()
    torch.cuda.synchronize()
    oA, oAi, _ = O.refine_forward(enc, delta, np.float32(0.9))
    op, od, og = O.refine_backward(enc, delta, np.float32(0.9), ga, gi)
    rv = max(value_ratio(A.detach().cpu().numpy(), oA), value_ratio(Ai.detach().cpu().numpy(), oAi))
    gp, gd = p.grad.cpu().numpy(), d.grad.cpu().numpy()
    rg = max(grad_ratio(gp, op), grad_ratio(gd, od))
    # d_gamma is one fp64 sum over 786 432 items: held to the float32 rounding of the oracle's fp64 sum
    terms = np.abs(op[:, 1:] * delta[:, 1:].astype(np.float64)).sum()
    rgam = abs(float(g.grad) - og) / (1e-6 * terms)
    report("refine b v = 2^20", values=rv, gradients=rg, d_gamma_to_1e6_of_sum_abs=rgam,
           backward_ms=start.elapsed_time(end))
    assert rv <= 1.0 and rg <= 1.0 and rgam <= 1.0


def plucker_inputs(rng, n, pixel_units=None):
    E = rigids(rng, n, 0.5, 1.0)
    K = np.zeros((n, 3, 3))
    K[:, 0, 0], K[:, 1, 1] = rng.uniform(0.8, 1.1, n), rng.uniform(0.8, 1.1, n)
    K[:, 0, 2], K[:, 1, 2], K[:, 2, 2] = rng.uniform(0.45, 0.55, n), rng.uniform(0.45, 0.55, n), 1.0
    if pixel_units:
        K[:, 0] *= pixel_units[1]
        K[:, 1] *= pixel_units[0]
    return E.astype(np.float32), K.astype(np.float32)


@pytest.mark.parametrize("b,v,h,w,pixel_units", [
    (4369, 15, 3, 3, False),   # b v = 65 535, the grid's y limit
    (1, 2, 1, 4099, False), (1, 2, 4099, 1, False),
    (1, 1, 1000, 1003, False),  # h w = 1 003 000, not a multiple of 256
    (2, 3, 24, 40, True),
])
def test_plucker_shapes(b, v, h, w, pixel_units, poisoned):  # noqa: F811
    from pf3plat_b200.poses import plucker_rays
    E, K = plucker_inputs(np.random.default_rng(h * w + b), b * v, (h, w) if pixel_units else None)
    E, K = E.reshape(b, v, 4, 4), K.reshape(b, v, 3, 3)
    got = plucker_rays(torch.tensor(E, device=DEV), torch.tensor(K, device=DEV), h, w).cpu().numpy()
    r = value_ratio(got, O.plucker_rays(E, K, h, w))
    report(f"plucker b = {b}, v = {v}, {h} x {w}{', pixel-unit K' if pixel_units else ''}", values=r)
    assert r <= 1.0


def test_plucker_next_to_non_finite_poses(poisoned):  # noqa: F811
    """a NaN rotation entry, an Inf translation and a NaN translation, each in its own item: that item's output is
    non-finite everywhere, and every other item's bits are those of a run without them"""
    from pf3plat_b200.poses import plucker_rays
    b, v, h, w = 3, 3, 13, 22
    E, K = plucker_inputs(np.random.default_rng(30), b * v)
    E, K = E.reshape(b, v, 4, 4), K.reshape(b, v, 3, 3)
    clean = plucker_rays(torch.tensor(E, device=DEV), torch.tensor(K, device=DEV), h, w).cpu().numpy()
    bad = E.copy()
    bad[0, 1, 0, 1] = np.nan
    bad[1, 0, 2, 3] = np.inf
    bad[2, 2, 1, 3] = np.nan
    got = plucker_rays(torch.tensor(bad, device=DEV), torch.tensor(K, device=DEV), h, w).cpu().numpy()
    items = [0 * v + 1, 1 * v + 0, 2 * v + 2]
    assert not np.isfinite(got[items]).any()
    others = [i for i in range(b * v) if i not in items]
    assert np.array_equal(got[others].view(np.uint32), clean[others].view(np.uint32))
    assert value_ratio(clean, O.plucker_rays(E, K, h, w)) <= 1.0


def test_sync_wall_time_at_b_65535_n16(poisoned):  # noqa: F811
    """the largest synchronisation the ABI takes: every k_pose_sync_finish thread reduces 65 535 masses"""
    from pf3plat_b200.poses import camera_synchronization
    b, N = 65535, 16
    gen = torch.Generator(device=DEV).manual_seed(0)
    P = {k: torch.eye(4, device=DEV) + 0.01 * torch.randn(b, 4, 4, device=DEV, generator=gen)
         for k in itertools.combinations(range(N), 2)}
    for t in P.values():
        t[:, 3] = torch.tensor([0.0, 0.0, 0.0, 1.0], device=DEV)
    C = {k: 0.55 + 0.4 * torch.rand(b, device=DEV, generator=gen) for k in P}
    camera_synchronization(P, C, N)
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    out = camera_synchronization(P, C, N)
    end.record()
    torch.cuda.synchronize()
    report("sync b = 65535, N = 16", ms=start.elapsed_time(end))
    assert torch.isfinite(out).all()
    one = camera_synchronization({k: v[b - 1:] for k, v in P.items()}, {k: v[b - 1:] for k, v in C.items()}, N)
    assert torch.equal(out[b - 1:], one)
