"""CPU checks of the sync-free rasterizer path (gs_forward_sync_free / gs_backward_sync_free, DESIGN.md 5.18): the
GsSyncFreeWorkspace layout against the header, the workspace size restated from the layout and compared with
gs_sync_free_workspace_bytes over a spread of shapes and flags, the C entries' refusals before any launch, and the
Python workspace's validation.  No compute calls (no GPU here)."""
import ctypes
import os
import subprocess

import pytest
import torch

from tests.regimes import (DEPTH_PATTERNS, DESIGNED_CASES, PARKED, _at_pixels, designed_case, designed_depths,
                           designed_tile_of, designed_tiles)
from tests.sync_free_layout import regions

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "gsplat_b200.h")


@pytest.fixture(scope="module")
def capi():
    import __graft_entry__ as ge
    ge.build()
    from pf3plat_b200 import _capi
    return _capi


def test_the_workspace_struct_layout_matches_the_header(capi, tmp_path):
    fields = ("base", "bytes", "instance_capacity")
    prog = tmp_path / "sizes.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "gsplat_b200.h"\nint main(void){'
                    'printf("%zu\\n", sizeof(GsSyncFreeWorkspace));'
                    + "".join(f'printf("%zu\\n", offsetof(GsSyncFreeWorkspace, {f}));' for f in fields)
                    + 'printf("%d %d\\n", (int)GS_SYNC_FREE_DETERMINISTIC, (int)GS_SYNC_FREE_CAMERA_GRAD);'
                    + 'printf("%d\\n", GS_ABI_VERSION);return 0;}')
    exe = tmp_path / "sizes"
    subprocess.run(["gcc", "-I", os.path.dirname(HEADER), str(prog), "-o", str(exe)], check=True)
    out = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert ctypes.sizeof(capi.GsSyncFreeWorkspace) == out[0] == 24
    for f, off in zip(fields, out[1:4]):
        assert getattr(capi.GsSyncFreeWorkspace, f).offset == off, f
    assert (capi.GS_SYNC_FREE_DETERMINISTIC, capi.GS_SYNC_FREE_CAMERA_GRAD) == tuple(out[4:6])
    assert out[6] == capi.ABI_VERSION == 5


def expected_bytes(S, V, P, H, W, cap, det, cam):
    """The layout of gs_capi.cu's sf_layout, restated region by region (tests/sync_free_layout.py, whose offsets the
    GPU tests read the tile lists at): status | saved planes | list | max(forward scratch, backward)."""
    return regions(S, V, P, H, W, cap, det, cam)["total"][1]


def test_the_restated_regions_are_aligned_and_disjoint():
    for S, V, P, H, W, cap in SHAPES:
        for det in (False, True):
            reg = regions(S, V, P, H, W, cap, det, True)
            fwd = [(o, n, k) for k, (o, n) in reg.items() if k not in ("total", "backward")]
            assert [k for _, _, k in fwd] == ["status", "rec0", "rec1", "rec2", "meta", "ranges", "final_T", "n_contrib",
                                              "sched", "point_list", "rects", "tile_counts", "cursor", "sub_offsets",
                                              "tile_start", "tile_n", "bucket", "tmp"]
            for (o0, n0, k0), (o1, _, _) in zip(fwd, fwd[1:]):
                assert o0 % 256 == 0 and o0 + n0 <= o1, k0
            assert reg["backward"][0] == reg["rects"][0]          # the backward reuses the forward's scratch
            assert reg["total"][1] >= max(o + n for o, n, _ in fwd)


SHAPES = [(1, 1, 0, 1, 1, 0), (1, 1, 1, 16, 16, 1), (2, 8, 1000, 37, 53, 12345), (14, 42, 131072, 256, 256, 9_000_000),
          (1, 8, 500_000, 256, 256, 2_000_000), (3, 3, 7, 1, 4099, 2**31 - 1), (5, 15, 20000, 256, 256, 0)]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("cam", [False, True])
def test_workspace_bytes_match_the_restated_layout(capi, shape, det, cam):
    from pf3plat_b200.rasterizer import sync_free_workspace_bytes
    S, V, P, H, W, cap = shape
    got = sync_free_workspace_bytes(S, V, P, H, W, cap, deterministic=det, camera_grad=cam)
    assert got == expected_bytes(S, V, P, H, W, cap, det, cam)


def test_workspace_bytes_grow_with_capacity_and_flags(capi):
    from pf3plat_b200.rasterizer import sync_free_workspace_bytes
    base = sync_free_workspace_bytes(2, 6, 50000, 256, 256, 10**6)
    # 20 bytes per instance: the list, the bucket and the long-list sort's second buffer
    assert sync_free_workspace_bytes(2, 6, 50000, 256, 256, 2 * 10**6) - base == 20 * 10**6
    assert sync_free_workspace_bytes(2, 6, 50000, 256, 256, 10**6, deterministic=True) > base


def test_workspace_bytes_refuse_bad_arguments(capi):
    L = capi.lib()
    out = ctypes.c_int64(7)

    def cfg(**kw):
        c = capi.GsConfig()
        c.P, c.S, c.V, c.image_height, c.image_width = 10, 1, 2, 32, 32
        for k, v in kw.items():
            setattr(c, k, v)
        return c

    assert L.gs_sync_free_workspace_bytes(ctypes.byref(cfg()), 5, 0, ctypes.byref(out)) == 0 and out.value > 0
    for bad, cap, needs, word in ((dict(S=0), 5, 0, b"S >= 1"), (dict(V=3, S=2), 5, 0, b"V % S"),
                                  (dict(image_height=0), 5, 0, b"empty image"), (dict(P=-1), 5, 0, b"P >= 0"),
                                  (dict(P=2**30, V=4, S=4), 5, 0, b"2^31-1"), ({}, -1, 0, b"instance_capacity"),
                                  ({}, 2**31, 0, b"instance_capacity"), ({}, 5, 4, b"GS_SYNC_FREE")):
        rc = L.gs_sync_free_workspace_bytes(ctypes.byref(cfg(**bad)), cap, needs, ctypes.byref(out))
        assert rc != 0 and out.value == -1, bad
        assert word in L.gs_last_error(), (bad, L.gs_last_error())
    assert L.gs_sync_free_workspace_bytes(None, 5, 0, ctypes.byref(out)) == -1
    assert L.gs_sync_free_workspace_bytes(ctypes.byref(cfg()), 5, 0, None) == -1


def test_entries_refuse_a_workspace_that_does_not_fit_before_launching(capi):
    """Every pointer below is fake: each call must fail its checks before it launches or dereferences anything."""
    L = capi.lib()
    fake = ctypes.c_void_p(4096)
    cfg = capi.GsConfig()
    cfg.P, cfg.S, cfg.V, cfg.M, cfg.image_height, cfg.image_width = 100, 1, 2, 1, 32, 32
    cfg.viewmatrix = cfg.projmatrix = cfg.campos = 4096
    gin = capi.GsInputs(means3D=4096, opacities=4096, shs=4096, cov3D_precomp=4096)
    gout = capi.GsOutputs(4096, 4096, None)
    need = ctypes.c_int64()
    assert L.gs_sync_free_workspace_bytes(ctypes.byref(cfg), 1000, 0, ctypes.byref(need)) == 0
    saved = ctypes.c_void_p(1234)
    for ws, word in ((capi.GsSyncFreeWorkspace(4096, need.value - 256, 1000), b"smaller"),
                     (capi.GsSyncFreeWorkspace(4096 + 128, need.value, 1000), b"aligned"),
                     (capi.GsSyncFreeWorkspace(4096, need.value, -1), b"instance_capacity"),
                     (capi.GsSyncFreeWorkspace(None, need.value, 1000), b"null")):
        rc = L.gs_forward_sync_free(fake, ctypes.byref(cfg), ctypes.byref(gin), ctypes.byref(gout), None,
                                    ctypes.byref(ws), ctypes.byref(saved), None)
        assert rc == -1 and word in L.gs_last_error(), (word, L.gs_last_error())
        assert saved.value is None
        saved = ctypes.c_void_p(1234)
    rc = L.gs_forward_sync_free(fake, ctypes.byref(cfg), ctypes.byref(gin), ctypes.byref(gout), None, None, None, None)
    assert rc == -1
    og, ig = capi.GsOutGrads(4096, None), capi.GsInGrads()
    rc = L.gs_backward_sync_free(fake, ctypes.byref(cfg), ctypes.byref(gin), fake, ctypes.byref(og), None,
                                 ctypes.byref(ig), None, None, None, None)
    assert rc == -1 and b"same workspace" in L.gs_last_error()


def test_python_workspace_refuses_a_cpu_device_and_checks_calls(capi):
    from pf3plat_b200.rasterizer import SyncFreeWorkspace
    with pytest.raises(ValueError, match="CUDA device"):
        SyncFreeWorkspace("cpu", 1, 2, 100, (32, 32), 1000)
    # the per-call check, on a workspace whose buffer is never touched
    ws = SyncFreeWorkspace.__new__(SyncFreeWorkspace)
    ws.device, ws.dims = torch.device("cuda", 0), (1, 2, 100, 32, 32)
    ws.depth = ws.alpha = ws.camera_grad = False
    ws._check(torch.device("cuda", 0), 1, 2, 100, 32, 32, False, False, False)
    with pytest.raises(ValueError, match="is on cuda:0"):
        ws._check(torch.device("cuda", 1), 1, 2, 100, 32, 32, False, False, False)
    for dims in ((2, 2, 100, 32, 32), (1, 1, 100, 32, 32), (1, 2, 101, 32, 32), (1, 2, 100, 31, 32)):
        with pytest.raises(ValueError, match="sized for"):
            ws._check(torch.device("cuda", 0), *dims, False, False, False)
    for k, name in ((0, "depth"), (1, "alpha"), (2, "camera_grad")):
        flags = [False, False, False]
        flags[k] = True
        with pytest.raises(ValueError, match=f"{name}=True"):
            ws._check(torch.device("cuda", 0), 1, 2, 100, 32, 32, *flags)


def test_entry_points_take_a_workspace_keyword(capi):
    import inspect

    from pf3plat_b200.rasterizer import rasterize_batch
    from pf3plat_b200.render import decoder_forward, render_views
    for fn in (rasterize_batch, decoder_forward, render_views):
        p = inspect.signature(fn).parameters["workspace"]
        assert p.default is None, fn
    assert inspect.signature(rasterize_batch).parameters["workspace"].kind is inspect.Parameter.KEYWORD_ONLY


@pytest.mark.parametrize("name", DESIGNED_CASES)
def test_designed_splats_lie_in_their_tiles(name):
    """Every splat of a designed case (tests/regimes.py: designed_tiles) covers its designated (view, tile) and no other
    tile, by an fp64 restatement of the projection and the 3-sigma rect with a 1 px margin, and is culled in the other
    view: the GPU tests' exact per-tile lengths and D follow from the design."""
    h, w, views, cells = designed_case(name)
    d = designed_tiles(h, w, cells)
    got = designed_tile_of(d, views)
    want = torch.full_like(got, -1)
    want[torch.arange(got.shape[0]), d.view] = d.tile
    bad = (got != want).any(-1).nonzero().flatten()
    assert bad.numel() == 0, [(int(k), got[k].tolist(), want[k].tolist()) for k in bad[:8]]
    assert sum(d.lengths.values()) == d.means.shape[0] == sum(c[3] for c in cells)
    # the parking spot is in front of neither camera
    parked = designed_tiles(h, w, [(0, 0, 0, 1, "random")])
    parked.means = torch.tensor([PARKED])
    assert (designed_tile_of(parked, 2) == -1).all()


def test_the_tile_restatement_sees_a_splat_near_an_edge():
    d = designed_tiles(32, 32, [(0, 0, 0, 3, "random")])
    d.means[1] = _at_pixels(torch.tensor(14.5), torch.tensor(6.0), torch.tensor(4.0), 32, 32)   # 1.5 px from tile 1
    d.means[2] = _at_pixels(torch.tensor(6.0), torch.tensor(6.0), torch.tensor(0.15), 32, 32)   # before the near plane
    assert designed_tile_of(d, 1)[:, 0].tolist() == [0, -2, -1]


@pytest.mark.parametrize("pattern", DEPTH_PATTERNS)
def test_designed_depth_patterns(pattern):
    """Each pattern is in its regime as built; the GPU tests assert the same of the device's own depths."""
    z = designed_depths(pattern, 8193, torch.Generator().manual_seed(0))
    bits = z.view(torch.int32).long() & 0xffffffff
    distinct = bits.unique().numel()
    if pattern == "equal":
        assert distinct == 1
    elif pattern == "ulp":
        assert distinct >= 256 and (bits >> 16).unique().numel() == 1
    elif pattern == "binades":
        assert all(((bits >> (8 * k)) & 255).unique().numel() > 1 for k in range(4))
    elif pattern == "reversed":
        assert (z[1:] < z[:-1]).all()
    assert (z > 0.2).all()
