"""CPU checks of the device SH rotation (csrc/gs_sh_rotation.cu, pf3plat_b200.sh_rotation.guarded_sh_rotation_blocks):
the generated fit table csrc/gs_sh_fit.h against pf3plat_b200.sh_rotation._fit_points, an fp64 NumPy restatement of the
kernel's arithmetic (the basis at R x_k for the table's points, times the table's pseudo-inverse) against the tensor
route sh_rotation_blocks, and the C entry's struct layout and argument checks.  No compute calls (no GPU here)."""
import ctypes
import os
import re
import subprocess
from math import isqrt

import numpy as np
import pytest
import torch

from pf3plat_b200.sh_rotation import _fit_points, rotations_are_proper, sh_rotation_blocks

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TABLE = os.path.join(ROOT, "pf3plat_b200", "csrc", "gs_sh_fit.h")
HEADER = os.path.join(ROOT, "include", "gsplat_b200.h")


def parse_table():
    src = open(TABLE).read()
    src = re.sub(r"//[^\n]*", "", src)

    def array(name):
        body = re.search(name + r"\[[^=]*=\s*\{(.*?)\};", src, re.S).group(1)
        return np.array([float.fromhex(v) for v in re.findall(r"-?0x[0-9a-fA-F.]+p[-+]?\d+", body)], np.float64)

    pts = array("GS_SH_FIT_POINTS").reshape(5, 64, 3)
    flat = array("GS_SH_FIT_PINV")
    assert flat.size == 64 * 25
    pinv = [flat[64 * l * l:64 * (l + 1) ** 2].reshape(64, 2 * l + 1) for l in range(5)]
    return pts, pinv


def basis(l, m):
    """(64, 3) -> (2l + 1, 64), statement for statement as the kernel's real_sh_basis"""
    x, y, z = m[:, 2], m[:, 0], m[:, 1]
    xx, yy, zz = x * x, y * y, z * z
    if l == 0:
        return np.full((1, m.shape[0]), 0.28209479177387814)
    if l == 1:
        c = 0.4886025119029199
        return np.stack([c * y, c * z, c * x])
    if l == 2:
        return np.stack([1.0925484305920792 * x * y, 1.0925484305920792 * y * z, 0.31539156525252005 * (2 * zz - xx - yy),
                         1.0925484305920792 * x * z, 0.5462742152960396 * (xx - yy)])
    if l == 3:
        return np.stack([0.5900435899266435 * y * (3 * xx - yy), 2.890611442640554 * x * y * z,
                         0.4570457994644658 * y * (4 * zz - xx - yy), 0.3731763325901154 * z * (2 * zz - 3 * xx - 3 * yy),
                         0.4570457994644658 * x * (4 * zz - xx - yy), 1.445305721320277 * z * (xx - yy),
                         0.5900435899266435 * x * (xx - 3 * yy)])
    rr = xx + yy + zz
    return np.stack([2.5033429417967046 * x * y * (xx - yy), 1.7701307697799304 * y * z * (3 * xx - yy),
                     0.9461746957575601 * x * y * (7 * zz - rr), 0.6690465435572892 * y * z * (7 * zz - 3 * rr),
                     0.10578554691520431 * (35 * zz * zz - 30 * zz * rr + 3 * rr * rr),
                     0.6690465435572892 * x * z * (7 * zz - 3 * rr), 0.47308734787878004 * (xx - yy) * (7 * zz - rr),
                     1.7701307697799304 * x * z * (xx - 3 * yy),
                     0.6258357354491761 * (xx * (xx - 3 * yy) - yy * (3 * xx - yy))])


def kernel_blocks(R, d_sh, table):
    """the kernel's per-camera arithmetic in fp64: R (3, 3) -> (d_sh, d_sh)"""
    pts, pinv = table
    out = np.zeros((d_sh, d_sh))
    for l in range(isqrt(d_sh)):
        moved = pts[l] @ R.T                     # row k: R x_k
        out[l * l:(l + 1) ** 2, l * l:(l + 1) ** 2] = basis(l, moved) @ pinv[l]
    return out


def axis_rotation(axis, angle):
    c, s = np.cos(angle), np.sin(angle)
    i, j = [(1, 2), (2, 0), (0, 1)][axis]
    R = np.eye(3)
    R[i, i], R[i, j], R[j, i], R[j, j] = c, -s, s, c
    return R


def qr_rotations(n, seed):
    rng = np.random.default_rng(seed)
    q, r = np.linalg.qr(rng.standard_normal((n, 3, 3)))
    q = q * np.sign(np.diagonal(r, axis1=1, axis2=2))[:, None, :]
    q[np.linalg.det(q) < 0, :, 0] *= -1
    return q


def singular_rotations():
    """rotations by 0, pi/2 and pi about each axis, and products that put e3nn's beta at 0 or pi (Euler-singular)"""
    out = [axis_rotation(a, t) for a in range(3) for t in (0.0, np.pi / 2, np.pi, -np.pi / 2)]
    out += [axis_rotation(1, 0.3) @ axis_rotation(0, np.pi) @ axis_rotation(1, -1.1),
            axis_rotation(1, 0.7) @ axis_rotation(1, 2.0), axis_rotation(2, np.pi) @ axis_rotation(0, np.pi)]
    return np.stack(out)


def near_orthogonal(n, seed, size):
    """Q (I + E), E ~ size: up to ~size from orthogonal, det within the guard"""
    rng = np.random.default_rng(seed)
    m = qr_rotations(n, seed) @ (np.eye(3) + size * rng.uniform(-1, 1, (n, 3, 3)))
    return m / np.cbrt(np.linalg.det(m))[:, None, None] * np.cbrt(1 + rng.uniform(-0.9e-5, 0.9e-5, n))[:, None, None]


def test_the_table_parses_back_to_the_fit_points():
    pts, pinv = parse_table()
    for l in range(5):
        p, q = _fit_points(l, "cpu")
        assert np.array_equal(pts[l], p.numpy()), l                       # bit-identical points
        ref = q.numpy()
        assert np.abs(pinv[l] - ref).max() <= 1e-13 * np.abs(ref).max(), l


@pytest.mark.parametrize("kind", ["qr", "singular", "near_orthogonal"])
def test_the_kernel_arithmetic_matches_the_tensor_route(kind):
    table = parse_table()
    rots = {"qr": lambda: qr_rotations(40, 1), "singular": singular_rotations,
            "near_orthogonal": lambda: near_orthogonal(40, 2, 3e-6)}[kind]()
    if kind == "near_orthogonal":
        f32 = torch.tensor(rots, dtype=torch.float32)
        assert rotations_are_proper(f32)  # the guard admits them
        assert np.abs(np.einsum("nji,njk->nik", rots, rots) - np.eye(3)).max() > 1e-6
    for d_sh in (1, 4, 9, 16, 25):
        ref = sh_rotation_blocks(torch.tensor(rots, dtype=torch.float64), d_sh).numpy()
        got = np.stack([kernel_blocks(R, d_sh, table) for R in rots])
        assert np.abs(got - ref).max() <= 1e-12, d_sh


@pytest.fixture(scope="module")
def capi():
    import __graft_entry__ as ge
    ge.build()
    from pf3plat_b200 import _capi
    return _capi


def test_the_config_struct_layout_matches_the_header(capi, tmp_path):
    fields = ("outer", "inner", "outer_stride", "inner_stride", "row_stride", "d_sh")
    prog = tmp_path / "sizes.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "gsplat_b200.h"\nint main(void){'
                    'printf("%zu\\n", sizeof(GsShRotationConfig));'
                    + "".join(f'printf("%zu\\n", offsetof(GsShRotationConfig, {f}));' for f in fields)
                    + "return 0;}")
    exe = tmp_path / "sizes"
    subprocess.run(["gcc", "-I", os.path.dirname(HEADER), str(prog), "-o", str(exe)], check=True)
    out = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert ctypes.sizeof(capi.GsShRotationConfig) == out[0]
    for f, off in zip(fields, out[1:]):
        assert getattr(capi.GsShRotationConfig, f).offset == off, f


def test_the_entry_refuses_bad_arguments_without_launching(capi):
    L = capi.lib()
    buf = ctypes.c_void_p(16)  # never dereferenced: every call below fails its checks first

    def cfg(**kw):
        base = dict(outer=2, inner=2, outer_stride=32, inner_stride=16, row_stride=4, d_sh=25)
        base.update(kw)
        return capi.GsShRotationConfig(**base)

    assert L.gs_sh_rotation_workspace_bytes(ctypes.byref(cfg())) >= 4
    assert L.gs_sh_rotation_workspace_bytes(None) == -1
    for bad, word in ((dict(d_sh=5), b"d_sh"), (dict(d_sh=36), b"d_sh"), (dict(d_sh=0), b"d_sh"),
                      (dict(outer=0), b"outer"), (dict(inner=0), b"inner"), (dict(inner=-3), b"inner"),
                      (dict(outer=65536, inner=32768), b"2^31"), (dict(row_stride=5), b"row_stride"),
                      (dict(row_stride=2), b"row_stride")):
        c = cfg(**bad)
        assert L.gs_sh_rotation_workspace_bytes(ctypes.byref(c)) == -1, bad
        assert L.gs_sh_rotation_blocks(ctypes.byref(c), buf, buf, buf, None) == -1, bad
        assert word in L.gs_last_error(), (bad, L.gs_last_error())
    for args in ((None, buf, buf), (buf, None, buf), (buf, buf, None)):
        assert L.gs_sh_rotation_blocks(ctypes.byref(cfg()), *args, None) == -1
        assert b"null" in L.gs_last_error()
    assert L.gs_sh_rotation_blocks(None, buf, buf, buf, None) == -1


def test_the_device_op_refuses_cpu_tensors():
    from pf3plat_b200.sh_rotation import guarded_sh_rotation_blocks
    with pytest.raises(TypeError, match="CUDA"):
        guarded_sh_rotation_blocks(torch.eye(3), 9)
