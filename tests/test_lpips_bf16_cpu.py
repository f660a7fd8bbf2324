"""CPU tests of LPIPS's precision option: the C ABI's GsLpipsConfig.precision and its ctypes mirror, the workspace size
per precision, and the Python setter and keyword (pf3plat_b200/lpips.py)."""
import ctypes
import os
import subprocess

import pytest
import torch

from oracle import lpips_oracle as lo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def capi():
    import __graft_entry__ as ge
    ge.build()
    from pf3plat_b200 import _capi
    return _capi


@pytest.fixture
def restore_precision():
    from pf3plat_b200 import lpips as pl
    prev = pl.get_precision()
    yield pl
    pl.set_precision(prev)


def test_config_layout_and_constants_match_the_header(capi, tmp_path):
    prog = tmp_path / "sizes.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "gsplat_b200.h"\nint main(void){'
                    'printf("%zu %zu %zu %zu %d %d\\n", sizeof(GsLpipsConfig), offsetof(GsLpipsConfig, grads),'
                    ' offsetof(GsLpipsConfig, precision), offsetof(GsLpipsConfig, reserved_),'
                    ' (int)GS_LPIPS_TF32, (int)GS_LPIPS_BF16);return 0;}')
    exe = tmp_path / "sizes"
    subprocess.run(["/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc", "-I", os.path.join(ROOT, "include"),
                    str(prog), "-o", str(exe)], check=True)
    got = tuple(map(int, subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()))
    C = capi.GsLpipsConfig
    assert got[0] == 40
    assert (ctypes.sizeof(C), C.grads.offset, C.precision.offset, C.reserved_.offset, capi.GS_LPIPS_TF32,
            capi.GS_LPIPS_BF16) == got
    cfg = C(precision=capi.GS_LPIPS_BF16)
    assert cfg.reserved_ == capi.GS_LPIPS_BF16 and C().precision == capi.GS_LPIPS_TF32


def test_workspace_depends_on_the_precision_and_bad_values_are_refused(capi):
    L = capi.lib()
    n = 3 * 64 * 64
    for grads in (0, 1, 3):
        tf32 = capi.GsLpipsConfig(batch=2, height=64, width=64, normalize=1, in0_stride=n, in1_stride=n, grads=grads)
        bf16 = capi.GsLpipsConfig.from_buffer_copy(tf32)
        bf16.precision = capi.GS_LPIPS_BF16
        a, b = L.gs_lpips_workspace_bytes(ctypes.byref(tf32)), L.gs_lpips_workspace_bytes(ctypes.byref(bf16))
        assert a > 0 and b > 0 and b < a and b >= a // 2 - 4096
    for bad in (-1, 2, 16):
        cfg = capi.GsLpipsConfig(batch=2, height=64, width=64, normalize=1, in0_stride=n, in1_stride=n, precision=bad)
        assert L.gs_lpips_workspace_bytes(ctypes.byref(cfg)) == -1
    assert L.gs_lpips_weights_pack_bf16(None, None, None) != 0


def test_the_setter_round_trips_and_bad_precisions_are_refused(capi, restore_precision):
    pl = restore_precision
    assert pl.get_precision() == "tf32"
    for p in ("bf16", "tf32", "bf16"):
        pl.set_precision(p)
        assert pl.get_precision() == p
    for bad in ("fp16", "BF16", "float32", "", None, 1):
        with pytest.raises(ValueError, match="precision"):
            pl.set_precision(bad)
        assert pl.get_precision() == "bf16"
    sd = lo.random_state_dict(3)
    for bad in ("fp16", "TF32", 0):
        with pytest.raises(ValueError, match="precision"):
            pl.LPIPS(weights=sd, precision=bad)
    assert pl.LPIPS(weights=sd).precision is None
    assert pl.LPIPS(weights=sd, precision="bf16").precision == "bf16"


def test_inputs_other_than_float32_are_still_refused(capi):
    from pf3plat_b200 import lpips as pl
    m = pl.LPIPS(weights=lo.random_state_dict(3), precision="bf16")
    x = torch.rand(1, 3, 16, 16)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m(x, x)
