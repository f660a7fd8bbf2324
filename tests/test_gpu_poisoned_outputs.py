"""The cost volume, the pose ops (camera_synchronization, refine_poses, plucker_rays) and the encoder's depth glue
(depth_update, mono_cue, pdf_peak) run once with every torch.empty poisoned (tests/poison.py: NaN, all-ones integers)
and once normally, forward and backward.  An output or gradient element a kernel leaves unwritten shows up as a
difference; otherwise the two runs are bit-identical.  The cost volume's default-mode backward accumulates with float
atomics in no fixed order, so there the non-finite elements must match and the values stay within its usual bound.
Also refine_poses where its single CTA loops: b = 100, v = 4 (400 items over 256 threads) and v = 1 (every delta
gradient 0), against tests/poses_oracle.py."""
import itertools

import numpy as np
import pytest
import torch

from tests import poses_oracle as PO
from tests.poison import poisoning

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def twice(fn):
    """fn() normally and poisoned, each a tuple of tensors; asserts that the poisoned run allocated on autograd's
    thread when it ran a backward"""
    clean = [t.detach().clone() for t in fn()]
    torch.cuda.synchronize()
    with poisoning() as p:
        bad = [t.detach().clone() for t in fn()]
    assert p.calls > 0
    return clean, bad, p


def assert_identical(clean, bad, what):
    for i, (a, b) in enumerate(zip(clean, bad)):
        assert a.shape == b.shape and a.dtype == b.dtype, (what, i)
        assert torch.equal(a, b) or (a.dtype.is_floating_point and torch.equal(a.isnan(), b.isnan())
                                     and torch.equal(torch.nan_to_num(a), torch.nan_to_num(b))), (what, i)


@pytest.mark.parametrize("deterministic", [False, True])
def test_cost_volume(deterministic):
    from tests.test_gpu_costvolume import GRAD_RTOL, run, seeded_case, worst_ratio
    f, K, E, near, far, D, cot = seeded_case(2, 3, 40, 20, 28, 8, seed=61)
    clean, bad, p = twice(lambda: run(f, K, E, near, far, D, cot, deterministic=deterministic))
    assert p.off_thread_calls() > 0
    assert torch.equal(clean[0], bad[0])
    if deterministic:
        assert torch.equal(clean[1], bad[1])
    else:
        r = worst_ratio(bad[1], clean[1], GRAD_RTOL, "cost volume gradient")
        print(f"cost volume default-mode backward, poisoned vs normal: {r:.3f} of the bound")
        assert r <= 1.0


def seeded_poses(b, v, seed):
    rng = np.random.default_rng(seed)
    enc = np.zeros((b, v, 9))
    for i, j in itertools.product(range(b), range(v)):
        a = rng.normal(size=3) * 0.4
        Kx = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
        R = np.eye(3) + np.sin(np.linalg.norm(a)) / np.linalg.norm(a) * Kx + \
            (1 - np.cos(np.linalg.norm(a))) / np.linalg.norm(a) ** 2 * Kx @ Kx
        enc[i, j, :6] = R[:2].reshape(6)
        enc[i, j, 6:] = rng.normal(size=3)
    delta = rng.normal(size=(b, v, 9)) * 0.1
    g_abs, g_inv = rng.normal(size=(b, v, 4, 4)), rng.normal(size=(b, v, 4, 4))
    f32 = lambda a: np.asarray(a, np.float32)  # noqa: E731
    return f32(enc), f32(delta), np.float32(0.7), f32(g_abs), f32(g_inv)


def refine(enc, delta, gamma, g_abs, g_inv):
    from pf3plat_b200.poses import refine_poses
    p = torch.tensor(enc, device=DEV, requires_grad=True)
    d = torch.tensor(delta, device=DEV, requires_grad=True)
    g = torch.tensor(float(gamma), device=DEV, requires_grad=True)
    A, Ai = refine_poses(p, d, g)
    ((A * torch.tensor(g_abs, device=DEV)).sum() + (Ai * torch.tensor(g_inv, device=DEV)).sum()).backward()
    return A, Ai, p.grad, d.grad, g.grad


def test_pose_ops():
    from pf3plat_b200.poses import camera_synchronization, plucker_rays
    from tests.test_gpu_poses import seeded_sync, sync_inputs
    keys, Ps, conf = seeded_sync(14, 4, seed=62)
    P, C = sync_inputs(keys, Ps, conf)
    clean, bad, _ = twice(lambda: (camera_synchronization(P, C, 4),))
    assert_identical(clean, bad, "camera_synchronization")
    K = torch.tensor([[1.0, 0.0, 0.5], [0.0, 1.1, 0.45], [0.0, 0.0, 1.0]], device=DEV).expand(14, 4, 3, 3).contiguous()
    poses = clean[0]
    clean, bad, _ = twice(lambda: (plucker_rays(poses, K, 13, 22),))
    assert_identical(clean, bad, "plucker_rays")
    args = seeded_poses(14, 4, seed=63)
    clean, bad, p = twice(lambda: refine(*args))
    assert p.off_thread_calls() > 0
    assert_identical(clean, bad, "refine_poses")


@pytest.mark.parametrize("b,v", [(100, 4), (3, 1)])
def test_refine_poses_past_one_pass_and_at_one_view(b, v):
    from tests.test_gpu_poses import grad_ratio, value_ratio
    enc, delta, gamma, g_abs, g_inv = seeded_poses(b, v, seed=64 + v)
    clean, bad, p = twice(lambda: refine(enc, delta, gamma, g_abs, g_inv))
    assert p.off_thread_calls() > 0
    assert_identical(clean, bad, "refine_poses")
    A, Ai, gp, gd, gg = (t.cpu().numpy() for t in clean)
    oA, oAi, _ = PO.refine_forward(enc, delta, gamma)
    op, od, og = PO.refine_backward(enc, delta, gamma, g_abs, g_inv)
    r = (value_ratio(A, oA), value_ratio(Ai, oAi), grad_ratio(gp, op), grad_ratio(gd, od),
         grad_ratio(np.array(gg), np.array(og)))
    print(f"refine_poses b={b} v={v}: ratios {['%.3f' % x for x in r]}")
    assert max(r) <= 1.0
    if v == 1:
        assert (gd == 0).all() and float(gg) == 0.0


def test_encoder_depth_ops():
    from tests.test_gpu_encoder_depth import seeded_stretch, stretch
    b, v, h, w, grid = 2, 3, 64, 96, (28, 28)
    inp = seeded_stretch(b, v, h, w, grid, seed=65)
    clean, bad, p = twice(lambda: stretch(inp, b, v, grid))
    assert p.off_thread_calls() > 0
    assert_identical(clean, bad, "depth_update / mono_cue / pdf_peak")
