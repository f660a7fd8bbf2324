"""The device SH rotation (pf3plat_b200.sh_rotation.guarded_sh_rotation_blocks, csrc/gs_sh_rotation.cu) against the
tensor route on the same device (rotations_are_proper's guard, then sh_rotation_blocks' fp64 fit, cast to float32):
every entry within 6e-8 (half a float32 ulp at 1) and exact zeros off the diagonal blocks, under the poison fixture so
that an unwritten element reads NaN.  Also the all-or-nothing guard, the properties of the float32 output, bit
determinism, the Gaussian head against its kernel fed the tensor route's blocks, GaussianAdapter given the device
blocks, and the op's refusals."""
import math

import numpy as np
import pytest
import torch

from pf3plat_b200.sh_rotation import (guarded_sh_rotation_blocks, real_sh_basis, rotations_are_proper,
                                      sh_rotation_blocks)
from tests.poison import poisoned  # noqa: F401  (fixture)
from tests.test_sh_rotation_cpu import near_orthogonal, qr_rotations, singular_rotations

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
D_SHS = (1, 4, 9, 16, 25)
TOL = 6e-8


def route(rot, d_sh):
    """the tensor route on the same device: the reference's guard, then the fit, cast to float32"""
    r = rot[..., :3, :3]
    if not rotations_are_proper(r):
        r = torch.eye(3, device=r.device, dtype=r.dtype).expand(r.shape)
    return sh_rotation_blocks(r, d_sh)


def block_mask(d_sh):
    m = torch.zeros(d_sh, d_sh, dtype=torch.bool, device=DEV)
    for l in range(math.isqrt(d_sh)):
        m[l * l:(l + 1) ** 2, l * l:(l + 1) ** 2] = True
    return m


def assert_parity(got, ref, d_sh):
    """-> how many entries differ from the route at all"""
    assert got.shape == ref.shape and got.dtype == torch.float32
    assert torch.isfinite(got).all()
    assert float((got.double() - ref.double()).abs().max()) <= TOL
    assert (got[..., ~block_mask(d_sh)] == 0).all()
    return int((got != ref).sum())


def f32(a):
    return torch.tensor(np.asarray(a), dtype=torch.float32, device=DEV)


def with_4x4(rot):
    m = torch.zeros(*rot.shape[:-2], 4, 4, dtype=rot.dtype, device=rot.device)
    m[..., :3, :3] = rot
    m[..., :3, 3] = 7.0
    m[..., 3, 3] = 1.0
    return m


@pytest.mark.parametrize("n", [1, 2, 3, 28, 257, 65534])
@pytest.mark.parametrize("d_sh", D_SHS)
def test_qr_rotations_match_the_tensor_route(n, d_sh, poisoned):  # noqa: F811
    rot = f32(qr_rotations(n, n))
    got = guarded_sh_rotation_blocks(rot, d_sh)
    differ = assert_parity(got, route(rot, d_sh), d_sh)
    print(f"n={n} d_sh={d_sh}: {differ} of {got.numel()} entries differ from the route")
    assert poisoned.calls >= 2


@pytest.mark.parametrize("d_sh", D_SHS)
def test_singular_near_orthogonal_and_refined_pose_rotations(d_sh, poisoned):  # noqa: F811
    from pf3plat_b200.poses import refine_poses
    g = torch.Generator(device=DEV).manual_seed(d_sh)
    b, v = 6, 4
    enc = torch.randn((b, v, 9), generator=g, device=DEV)
    _, c2w = refine_poses(enc, 0.1 * torch.randn((b, v, 9), generator=g, device=DEV), torch.ones(1, device=DEV))
    for rot in (f32(singular_rotations()), f32(near_orthogonal(257, 5, 3e-6)), c2w[..., :3, :3]):
        assert rotations_are_proper(rot)
        assert_parity(guarded_sh_rotation_blocks(rot, d_sh), route(rot, d_sh), d_sh)


@pytest.mark.parametrize("V", [2, 3, 4, 5, 6])
def test_strided_views_of_c2w_and_both_matrix_shapes(V, poisoned):  # noqa: F811
    b, d_sh = 7, 25
    c2w = with_4x4(f32(qr_rotations(b * V, 10 + V)).reshape(b, V, 3, 3))
    slots = c2w[:, ::V - 1]
    assert slots.shape == (b, 2, 4, 4) and slots.is_contiguous() == (V == 2)  # views 0 and V - 1, in place
    got = guarded_sh_rotation_blocks(slots, d_sh)
    assert got.shape == (b, 2, d_sh, d_sh) and got.is_contiguous()
    ref = route(slots.contiguous(), d_sh)
    assert_parity(got, ref, d_sh)
    r3 = slots[..., :3, :3].contiguous()
    for other in (r3, slots[..., :3, :3], slots.contiguous()):  # [..., 3, 3], the row-stride-4 view, [..., 4, 4]
        assert torch.equal(guarded_sh_rotation_blocks(other, d_sh), got)
    # no batch dims, one, three (reshaped) and a transposed (non-unit column stride) input
    assert torch.equal(guarded_sh_rotation_blocks(r3[0, 1], d_sh), got[0, 1])
    assert torch.equal(guarded_sh_rotation_blocks(r3.reshape(-1, 3, 3), d_sh), got.reshape(-1, d_sh, d_sh))
    assert torch.equal(guarded_sh_rotation_blocks(r3.reshape(b, 1, 2, 3, 3), d_sh), got.reshape(b, 1, 2, d_sh, d_sh))
    tr = r3.transpose(-1, -2).contiguous().transpose(-1, -2)
    assert torch.equal(guarded_sh_rotation_blocks(tr, d_sh), got)


def scaled_to_det(rot, det):
    return rot * torch.tensor(det, dtype=torch.float64).pow(1 / 3).float().to(rot.device)


@pytest.mark.parametrize("d_sh", [9, 25])
def test_the_guard_is_all_or_nothing(d_sh, poisoned):  # noqa: F811
    base = f32(qr_rotations(257, 3))
    eye = sh_rotation_blocks(torch.eye(3, device=DEV)[None], d_sh)[0]
    for delta in (0.9e-5, -0.9e-5):
        rot = base.clone()
        rot[100] = scaled_to_det(rot[100], 1 + delta)
        assert rotations_are_proper(rot)
        got = guarded_sh_rotation_blocks(rot, d_sh)
        assert_parity(got, route(rot, d_sh), d_sh)
        assert float((got[100] - eye).abs().max()) > 1e-3  # its own matrix
    for delta in (1.2e-5, -1.2e-5):
        rot = base.clone()
        rot[100] = scaled_to_det(rot[100], 1 + delta)
        assert not rotations_are_proper(rot)
        got = guarded_sh_rotation_blocks(rot, d_sh)
        assert_parity(got, route(rot, d_sh), d_sh)
        assert float((got - torch.eye(d_sh, device=DEV)).abs().max()) <= TOL
        assert (got == got[0]).all()
    clean = guarded_sh_rotation_blocks(torch.cat([base[:100], base[101:]]), d_sh)
    assert_parity(clean, route(torch.cat([base[:100], base[101:]]), d_sh), d_sh)
    for bad in ("improper", "nan", "inf", "-inf"):
        rot = base.clone()
        if bad == "improper":
            rot[100, :, 0] *= -1
        else:
            rot[100, 1, 2] = {"nan": math.nan, "inf": math.inf, "-inf": -math.inf}[bad]
        got = guarded_sh_rotation_blocks(rot, d_sh)
        assert torch.isfinite(got).all(), bad
        assert float((got - torch.eye(d_sh, device=DEV)).abs().max()) <= TOL, bad
        assert (got == got[0]).all(), bad
        assert_parity(got, route(rot, d_sh), d_sh)
        # the same set without the bad camera: every other camera gets its own matrix, the same bits as before
        assert torch.equal(guarded_sh_rotation_blocks(torch.cat([rot[:100], rot[101:]]), d_sh), clean), bad


def test_properties_of_the_float32_output():
    d_sh = 25
    n = 512
    r1, r2 = qr_rotations(n, 21), qr_rotations(n, 22)
    D1 = guarded_sh_rotation_blocks(f32(r1), d_sh).double()
    D2 = guarded_sh_rotation_blocks(f32(r2), d_sh).double()
    D12 = guarded_sh_rotation_blocks(f32(r1 @ r2), d_sh).double()
    I = torch.eye(d_sh, dtype=torch.float64, device=DEV)
    assert float((D1.transpose(-1, -2) @ D1 - I).abs().max()) <= 1e-6
    assert float((D12 - D1 @ D2).abs().max()) <= 1e-6
    assert float((D1[:, 1:4, 1:4] - f32(r1).double()).abs().max()) <= 1e-6
    g = torch.Generator().manual_seed(5)
    x = torch.randn(100, 3, generator=g, dtype=torch.float64)
    x = (x / x.norm(dim=-1, keepdim=True)).to(DEV)
    R = f32(r1).double()
    for l in range(5):
        lo, hi = l * l, (l + 1) ** 2
        yx = real_sh_basis(l, x)                                     # (100, 2l+1)
        yrx = real_sh_basis(l, torch.einsum("nij,kj->nki", R, x))    # (n, 100, 2l+1)
        pred = torch.einsum("nij,kj->nki", D1[:, lo:hi, lo:hi], yx)
        assert float((yrx - pred).abs().max()) <= 1e-6, l


def test_bit_determinism_and_no_host_synchronisation():
    d_sh = 25
    rot = f32(qr_rotations(257, 8))
    a = guarded_sh_rotation_blocks(rot, d_sh)
    assert torch.equal(guarded_sh_rotation_blocks(rot, d_sh), a)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        b = guarded_sh_rotation_blocks(rot, d_sh)
    torch.cuda.current_stream().wait_stream(s)
    assert torch.equal(b, a)
    for i in (0, 1, 128, 256):
        assert torch.equal(guarded_sh_rotation_blocks(rot[i:i + 1], d_sh), a[i:i + 1]), i
        assert torch.equal(guarded_sh_rotation_blocks(rot[i], d_sh), a[i]), i
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        c = guarded_sh_rotation_blocks(rot, d_sh)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert torch.equal(c, a)


def test_n_65534_in_one_call_matches_cameras_computed_alone():
    rot = f32(qr_rotations(65534, 4))
    a = guarded_sh_rotation_blocks(rot, 25)
    for i in (0, 1, 32767, 65533):
        assert torch.equal(guarded_sh_rotation_blocks(rot[i:i + 1], 25), a[i:i + 1]), i


def old_slots(c2w, d_sh):
    """the head's former tensor route: stack, det, isclose().all(), where, sh_rotation_blocks"""
    c = c2w.detach()
    rot = torch.stack([c[:, 0, :3, :3], c[:, -1, :3, :3]], 1)
    det = torch.det(rot)
    ok = torch.isclose(det, torch.ones_like(det)).all()
    rot = torch.where(ok, rot, torch.eye(3, dtype=rot.dtype, device=rot.device))
    return sh_rotation_blocks(rot, d_sh).contiguous()


@pytest.mark.parametrize("b,V,h,w,deg,improper", [(2, 3, 16, 24, 4, False), (3, 2, 9, 13, 3, False),
                                                  (2, 4, 8, 8, 4, True), (1, 5, 7, 5, 2, False)])
def test_the_head_against_its_kernel_fed_the_tensor_route(b, V, h, w, deg, improper, poisoned):  # noqa: F811
    from pf3plat_b200.gaussian_head import _GaussianHead, _sh_mask, gaussian_head
    from tests.test_gpu_gaussian_head import KEYS, cfg_for, masked_cotangents, seeded
    c = seeded(b, V, h, w, deg, seed=31 + h)
    if improper:
        c["c2w"][1, V - 1, :, 0] *= -1
    cot = masked_cotangents(c)
    d_sh = (deg + 1) ** 2
    cfg = cfg_for(deg)
    names = ("raw", "logits", "depths", "c2w")

    def leaves():
        return {k: torch.tensor(np.asarray(c[k]), dtype=torch.float32, device=DEV).requires_grad_(True) for k in names}

    K = torch.tensor(np.asarray(c["K"]), dtype=torch.float32, device=DEV)
    t = leaves()
    g = gaussian_head(t["raw"], t["logits"], t["depths"], t["c2w"], K, cfg, (h, w))
    new = {k: getattr(g, k) for k in KEYS}
    sum((torch.tensor(cot[k], dtype=torch.float32, device=DEV) * new[k]).sum() for k in KEYS).backward()
    u = leaves()
    consts = (b, V, h, w, d_sh, float(cfg.gaussian_scale_min), float(cfg.gaussian_scale_max), 1e-8)
    outs = _GaussianHead.apply(u["raw"], u["logits"], u["depths"], u["c2w"], K, old_slots(u["c2w"], d_sh),
                               _sh_mask(deg, DEV), consts)
    old = dict(zip(KEYS, outs))
    old["harmonics"] = old["harmonics"].transpose(-1, -2)
    sum((torch.tensor(cot[k], dtype=torch.float32, device=DEV) * old[k]).sum() for k in KEYS).backward()
    for k in ("means", "covariances", "opacities"):
        assert torch.equal(new[k], old[k]), k
    hn, ho = new["harmonics"].double(), old["harmonics"].double()
    f = torch.isfinite(ho)
    assert torch.equal(torch.isfinite(hn), f)
    assert bool(((hn - ho).abs()[f] <= 1e-6 * (ho.abs()[f] + 1)).all())
    for k in ("logits", "depths", "c2w"):
        assert torch.equal(t[k].grad, u[k].grad), k
    gn, go = t["raw"].grad, u["raw"].grad
    assert torch.equal(gn[:, :9], go[:, :9])
    gn, go = gn[:, 9:].double(), go[:, 9:].double()
    f = torch.isfinite(go)
    assert torch.equal(torch.isfinite(gn), f)
    rms = float(go[f].square().mean().sqrt())
    assert bool(((gn - go).abs()[f] <= 1e-6 * (go.abs()[f] + rms)).all())


def test_the_head_forward_launches_three_kernels_and_never_synchronises():
    from torch.profiler import ProfilerActivity, profile

    from pf3plat_b200.gaussian_head import gaussian_head
    from tests.test_gpu_gaussian_head import cfg_for
    b, V, h, w, deg = 3, 3, 32, 32, 4
    g = torch.Generator(device=DEV).manual_seed(1)
    raw = torch.randn((2 * b, 9 + 3 * 25, h, w), generator=g, device=DEV)
    logits = torch.randn((2 * b, 2, h, w), generator=g, device=DEV)
    depths = 1.0 + torch.rand((b * V, 1, h, w), generator=g, device=DEV)
    c2w = with_4x4(f32(qr_rotations(b * V, 9)).reshape(b, V, 3, 3))
    K = torch.tensor([[1.0, 0.0, 0.5], [0.0, 1.0, 0.5], [0.0, 0.0, 1.0]], device=DEV).expand(b, V, 3, 3).contiguous()
    cfg = cfg_for(deg)
    gaussian_head(raw, logits, depths, c2w, K, cfg, (h, w))  # warm up
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        gaussian_head(raw, logits, depths, c2w, K, cfg, (h, w))
        torch.cuda.synchronize()
    launches = [e.name for e in prof.events() if e.device_type.name == "CUDA"]
    assert len(launches) <= 3, launches
    leaves = [t.clone().requires_grad_(True) for t in (raw, logits, depths, c2w)]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = gaussian_head(*leaves, K, cfg, (h, w))
        (out.means.sum() + out.covariances.sum() + out.harmonics.square().sum() + out.opacities.sum()).backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    for t in leaves:
        assert torch.isfinite(t.grad).all()


@pytest.mark.parametrize("deg", [1, 2, 4])
def test_the_adapter_takes_the_device_blocks(deg):
    from pf3plat_b200.adapter import GaussianAdapter, GaussianAdapterCfg
    d_sh = (deg + 1) ** 2
    ad = GaussianAdapter(GaussianAdapterCfg(gaussian_scale_min=0.5, gaussian_scale_max=15.0, sh_degree=deg)).to(DEV)
    g = torch.Generator(device=DEV).manual_seed(deg)
    V, R = 3, 500
    ext = with_4x4(f32(qr_rotations(V, 40 + deg)))
    K = torch.tensor([[1.1, 0.0, 0.5], [0.0, 0.9, 0.5], [0.0, 0.0, 1.0]], device=DEV).expand(V, 3, 3).contiguous()
    coords = torch.rand((V, R, 2), generator=g, device=DEV)
    depths = 1.0 + 9.0 * torch.rand((V, R), generator=g, device=DEV)
    opac = torch.rand((V, R), generator=g, device=DEV)
    raw0 = torch.randn((V, R, 7 + 3 * d_sh), generator=g, device=DEV)
    w = torch.randn((V, R, 3, d_sh), generator=g, device=DEV)
    results = []
    for sh_rotation in (None, guarded_sh_rotation_blocks(ext.detach(), d_sh)):
        raw = raw0.clone().requires_grad_(True)
        e = ext.clone().requires_grad_(True)
        out = ad.forward(e[:, None], K[:, None], coords, depths, opac, raw, (64, 64), sh_rotation=sh_rotation)
        (out.means.sum() + out.covariances.sum() + (w * out.harmonics).sum()).backward()
        results.append(tuple(t.detach() for t in (out.means, out.covariances, out.harmonics, raw.grad, e.grad)))
    for a, b in zip(results[0][:3], results[1][:3]):  # the adapter tests' bounds: 1e-5 / 1e-3 of the largest magnitude
        assert float((a - b).abs().max()) <= 1e-5 * float(b.abs().max()), a.shape
    for a, b in zip(results[0][3:], results[1][3:]):
        assert float((a - b).abs().max()) <= 1e-3 * float(b.abs().max()), a.shape


def test_refusals():
    rot = f32(qr_rotations(4, 0))
    with pytest.raises(ValueError, match="not differentiable"):
        guarded_sh_rotation_blocks(rot.clone().requires_grad_(True), 9)
    with pytest.raises(TypeError, match="CUDA"):
        guarded_sh_rotation_blocks(rot.cpu(), 9)
    with pytest.raises(TypeError, match="float32"):
        guarded_sh_rotation_blocks(rot.double(), 9)
    for bad in (0, 2, 5, 36, 9.0):
        with pytest.raises(ValueError, match="d_sh"):
            guarded_sh_rotation_blocks(rot, bad)
    for shape in ((4, 3, 4), (4, 2, 2), (3,), (4, 4, 3)):
        with pytest.raises(ValueError, match=r"\[\.\.\., 3, 3\]"):
            guarded_sh_rotation_blocks(torch.zeros(shape, device=DEV), 9)
