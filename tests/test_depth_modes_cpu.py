"""CPU checks of the fused depth modes: the fp64 restatement of each mode's fake colour (tests/depth_modes_oracle.py) against
the fake colours the reference's render_depth_cuda handed its rasterizer (tests/golden/camera_glue.npz), its derivative
against torch autograd and finite differences, the ABI fields that carry the mode, and the requests the library refuses."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from tests.depth_modes_oracle import EPS, fake_depth, fake_depth_grad

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "camera_glue.npz")
ALL_MODES = ("depth", "disparity", "relative_disparity", "log")


@pytest.mark.parametrize("mode", ALL_MODES)
def test_restatement_reproduces_the_reference_fake_colours(mode):
    """The reference rendered its depth for means.abs() + 0.5 (tests/test_camera_cpu.py drives the same call): z from
    extrinsics.inverse(), unscaled, and the recorded colours are f(z) in all three channels."""
    z = np.load(GOLDEN)
    ext = z["extrinsics"].astype(np.float64)
    means = np.abs(z["means"].astype(np.float64)) + 0.5
    near, far = z["near"].astype(np.float64)[:, None], z["far"].astype(np.float64)[:, None]
    w2c = np.linalg.inv(ext)
    zc = np.einsum("bj,bgj->bg", w2c[:, 2, :3], means) + w2c[:, 2, 3:4]
    want = z[f"depth_{mode}_colors"].astype(np.float64)             # (B, G, 3), fp32 as the reference computed it
    got = fake_depth(mode, zc, near, far)
    assert np.all(want[..., 0] == want[..., 1]) and np.all(want[..., 0] == want[..., 2])
    err = np.abs(got - want[..., 0])
    print(f"[regime] {mode}: z {zc.min():.3f}..{zc.max():.3f}, near {near.min():.3f}..{near.max():.3f}, far "
          f"{far.min():.1f}..{far.max():.1f}; max |fp64 - reference fp32| {err.max():.2e}")
    assert np.all(err <= 4 * np.finfo(np.float32).eps * np.maximum(1.0, np.abs(want[..., 0]))), err.max()
    if mode == "log":   # near < far: the clamp as written makes it the constant log(far)
        assert (near < far).all()
        np.testing.assert_array_equal(got, np.broadcast_to(np.log(far), got.shape))


def _reference_torch(mode, z, near, far):
    if mode == "disparity":
        return 1 / z
    if mode == "relative_disparity":
        dn, df, d = 1 / (near + EPS), 1 / (far + EPS), 1 / (z + EPS)
        return 1 - (d - df) / (dn - df + EPS)
    if mode == "log":
        return z.minimum(near).maximum(far).log()
    return z


@pytest.mark.parametrize("mode", ALL_MODES)
def test_derivative_matches_autograd_and_finite_differences(mode):
    rng = np.random.default_rng(3)
    near = rng.uniform(0.2, 2.0, (64, 1))
    far = near * rng.uniform(20.0, 200.0, (64, 1))
    z = near * np.exp(rng.uniform(np.log(0.25), np.log(300.0), (64, 32)))   # in front of near, past far, between
    zt = torch.tensor(z, requires_grad=True)
    _reference_torch(mode, zt, torch.tensor(near), torch.tensor(far)).sum().backward()
    got = fake_depth_grad(mode, z, near, far)
    np.testing.assert_allclose(got, zt.grad.numpy(), rtol=1e-12, atol=0)
    if mode == "log":
        assert np.all(got == 0.0)       # exactly 0 for near < far, as autograd gives it
        return
    h = 1e-6 * z
    fd = (fake_depth(mode, z + h, near, far) - fake_depth(mode, z - h, near, far)) / (2 * h)
    np.testing.assert_allclose(got, fd, rtol=1e-6)


@pytest.fixture(scope="module")
def capi():
    import __graft_entry__ as ge
    ge.build()
    from pf3plat_b200 import _capi
    return _capi


def test_config_offsets_match_the_header(capi, tmp_path):
    prog = tmp_path / "offsets.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "gsplat_b200.h"\nint main(void){'
                    'printf("%zu %zu %zu %d %d %d %d\\n", sizeof(GsConfig), offsetof(GsConfig, depth_mode),'
                    'offsetof(GsConfig, depth_near_far), GS_DEPTH_Z, GS_DEPTH_DISPARITY, GS_DEPTH_RELATIVE_DISPARITY,'
                    'GS_DEPTH_LOG);return 0;}')
    exe = tmp_path / "offsets"
    subprocess.run(["/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc", "-I", os.path.join(ROOT, "include"),
                    str(prog), "-o", str(exe)], check=True)
    out = [int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    C = capi.GsConfig
    assert [ctypes.sizeof(C), C.depth_mode.offset, C.depth_near_far.offset] == out[:3]
    assert [capi.GS_DEPTH_Z, capi.GS_DEPTH_DISPARITY, capi.GS_DEPTH_RELATIVE_DISPARITY, capi.GS_DEPTH_LOG] == out[3:]
    assert capi.DEPTH_MODES == dict(zip(ALL_MODES, out[3:]))
    assert capi.ABI_VERSION == 5 and capi.lib().gs_abi_version() == 5


def _config(capi, mode, flags, near_far):
    """A forward request that is valid in every other respect (device pointers are never dereferenced: validation
    refuses the request before anything is launched or allocated)."""
    fake = 256
    cfg = capi.GsConfig()
    cfg.P, cfg.S, cfg.V, cfg.M, cfg.sh_degree = 16, 1, 1, 0, 0
    cfg.image_height, cfg.image_width, cfg.flags, cfg.scale_modifier = 16, 16, flags, 1.0
    cfg.viewmatrix = cfg.projmatrix = cfg.campos = cfg.bg = fake
    cfg.depth_mode, cfg.depth_near_far = mode, near_far
    gin = capi.GsInputs(means3D=fake, opacities=fake, colors_precomp=fake, cov3D_precomp=fake)
    gout = capi.GsOutputs(color=fake, radii=fake, depth=fake)
    return cfg, gin, gout


@pytest.mark.parametrize("mode,flags,near_far,message", [
    (1, 0, None, b"needs GS_FLAG_DEPTH"),
    (2, 0, 256, b"needs GS_FLAG_DEPTH"),
    (3, 0, 256, b"needs GS_FLAG_DEPTH"),
    (4, 1, 256, b"unknown depth_mode"),
    (-1, 1, 256, b"unknown depth_mode"),
    (2, 1, None, b"needs depth_near_far"),
    (3, 1, None, b"needs depth_near_far"),
])
def test_invalid_combinations_are_rejected(capi, mode, flags, near_far, message):
    L = capi.lib()
    cfg, gin, gout = _config(capi, mode, flags, near_far)
    fake_ctx = ctypes.c_void_p(256)   # never touched: the request is refused first
    for call in (lambda: L.gs_forward(fake_ctx, ctypes.byref(cfg), ctypes.byref(gin), ctypes.byref(gout), None, None),
                 lambda: L.gs_render_host(fake_ctx, ctypes.byref(cfg), ctypes.byref(gin), ctypes.byref(gout), None)):
        assert call() == -1   # GS_ERR_INVALID
        assert message in L.gs_last_error()


def test_unknown_mode_name_is_rejected_by_the_settings(capi):
    from pf3plat_b200.rasterizer import BatchSettings, _make_config
    eye = torch.eye(4).reshape(1, 4, 4)
    bs = BatchSettings(image_height=8, image_width=8, viewmatrix=eye, projmatrix=eye, campos=torch.zeros(1, 3),
                       bg=torch.zeros(1, 3), sh_degree=0, with_depth=True, depth_mode="inverse_depth")
    with pytest.raises(ValueError, match="depth_mode"):
        _make_config(bs, 1, 4, 0, [])
    for name, value in capi.DEPTH_MODES.items():
        cfg = _make_config(bs._replace(depth_mode=name, depth_near_far=torch.ones(1, 2)), 1, 4, 0, [])
        assert cfg.depth_mode == value and bool(cfg.depth_near_far)
