"""Seeded scenes for the regimes the ordinary synthetic distribution (pf3plat_b200.synthetic.make_scene: centres inside
+-1.05 NDC, depths >= 1.5, opacities U(0.05, 1)) never reaches.  Each is small enough for the CPU oracle and is built from
a make_scene cloud, whose cameras it keeps (view 0 is the identity; the others are displaced in the image plane only, so
camera-space z equals world z in every view)."""
from __future__ import annotations

import math

import torch

from pf3plat_b200.synthetic import FX, Scene, make_cameras, make_scene, quat_to_rotmat

TANFOV = 0.5 / FX


def _with_extra(sc: Scene, means, scales, opac, g) -> Scene:
    """sc plus extra Gaussians (random orientations, SH drawn like make_scene's)."""
    n = means.shape[0]
    q = torch.randn(n, 4, generator=g)
    q = q / q.norm(dim=-1, keepdim=True)
    R = quat_to_rotmat(q)
    cov = R @ torch.diag_embed(scales * scales) @ R.transpose(-1, -2)
    cov = 0.5 * (cov + cov.transpose(-1, -2))
    d_sh = sc.harmonics.shape[-1]
    mask = torch.full((d_sh,), 0.05)
    mask[0] = 1.0
    mask[16:] = 0.0                                              # PF3plat's bands beyond 3 are zero (make_scene)
    sh = torch.randn(n, 3, d_sh, generator=g) * mask
    cat = lambda a, b: torch.cat([a, b]).contiguous()
    return Scene(sc.extrinsics, sc.intrinsics, sc.near, sc.far, sc.image_shape, sc.background, cat(sc.means, means),
                 cat(sc.covariances, cov), cat(sc.harmonics, sh), cat(sc.opacities, opac), cat(sc.scales, scales),
                 cat(sc.rotations, q))


def _U(g, lo, hi, *shape):
    return lo + (hi - lo) * torch.rand(*shape, generator=g)


def offscreen_scene(P: int, n_off: int, views: int, h: int, w: int, seed: int = 0) -> Scene:
    """P ordinary splats plus n_off whose centres lie 1.4-3x tanfov outside the frustum -- left, right, above, below and
    at the corners -- with footprints large enough (about the centre's distance from the image edge) to reach into it."""
    sc = make_scene(P, views, h, w, seed=seed)
    g = torch.Generator().manual_seed(seed + 1000)
    z = _U(g, 2.0, 8.0, n_off)
    side = torch.randint(0, 8, (n_off,), generator=g)
    ang = side.float() * (math.pi / 4) + _U(g, -0.3, 0.3, n_off)
    r = _U(g, 1.4, 3.0, n_off)                                   # in units of tanfov, along the dominant axis
    d = torch.stack([torch.cos(ang), torch.sin(ang)], -1)
    d = d / d.abs().amax(-1, keepdim=True)                       # onto the square |x| = 1 or |y| = 1
    uv = d * r[:, None] * TANFOV                                 # x/z, y/z
    means = torch.stack([uv[:, 0] * z, uv[:, 1] * z, z], -1)
    f_px = w / (2 * TANFOV)
    out_px = (r - 1.0) * (w / 2)                                 # distance of the centre from the image edge, in pixels
    sigma = out_px * _U(g, 0.6, 1.2, n_off) * z / f_px           # ~1 sigma of the (unclamped) footprint reaches the image
    scales = sigma[:, None] * torch.exp(_U(g, -0.3, 0.3, n_off, 3))
    opac = _U(g, 0.3, 1.0, n_off)
    return _with_extra(sc, means, scales, opac, g)


def near_plane_scene(P: int, n_near: int, n_cull: int, n_behind: int, views: int, h: int, w: int, seed: int = 0) -> Scene:
    """P ordinary splats plus n_near at 0.2004 <= z <= 1.2 (enormous footprints, rects clamped to the grid), n_cull at
    0.05 <= z <= 0.1996 (culled by the z > 0.2 near plane) and n_behind behind the camera.  No z lies within 2e-3
    relative of 0.2, so the oracle's near-plane fragility flag (1e-5 relative) stays unset."""
    sc = make_scene(P, views, h, w, seed=seed)
    g = torch.Generator().manual_seed(seed + 2000)
    near_z = torch.where(torch.rand(n_near, generator=g) < 0.3, _U(g, 0.2004, 0.3, n_near), _U(g, 0.3, 1.2, n_near))
    z = torch.cat([near_z, _U(g, 0.05, 0.1996, n_cull), _U(g, -3.0, -0.05, n_behind)])
    n = z.shape[0]
    uv = _U(g, -1.2, 1.2, n, 2) * TANFOV
    means = torch.stack([uv[:, 0] * z.abs(), uv[:, 1] * z.abs(), z], -1)
    sigma = torch.exp(_U(g, math.log(0.004), math.log(0.25), n))
    scales = sigma[:, None] * torch.exp(_U(g, -0.4, 0.4, n, 3))
    opac = _U(g, 0.05, 1.0, n)
    return _with_extra(sc, means, scales, opac, g)


def opaque_stack_scene(layers: int, grid: int, views: int, h: int, w: int, seed: int = 0) -> Scene:
    """`layers` sheets at depths 2, 3, ..., each a jittered grid x grid of Gaussians with opacity U(0.97, 1) whose
    footprints overlap their neighbours': alpha clamps at 0.99 near the centres and most pixels reach T < 1e-4 well before
    the end of their tile lists."""
    sc = make_scene(0, views, h, w, seed=seed)
    g = torch.Generator().manual_seed(seed + 3000)
    means, scales = [], []
    for k in range(layers):
        z = 2.0 + k + _U(g, -0.2, 0.2, grid * grid)
        ij = torch.stack(torch.meshgrid(torch.arange(grid), torch.arange(grid), indexing="ij"), -1).reshape(-1, 2).float()
        uv = ((ij + 0.5 + _U(g, -0.35, 0.35, grid * grid, 2)) / grid * 2.2 - 1.1) * TANFOV
        means.append(torch.stack([uv[:, 0] * z, uv[:, 1] * z, z], -1))
        spacing = 2.2 * TANFOV * z / grid                        # world distance between neighbouring centres
        scales.append((0.55 * spacing)[:, None] * torch.exp(_U(g, -0.25, 0.25, grid * grid, 3)))
    means, scales = torch.cat(means), torch.cat(scales)
    opac = _U(g, 0.97, 1.0, means.shape[0])
    return _with_extra(sc, means, scales, opac, g)


def _at_pixels(u, v, z, h: int, w: int):
    """World points (view 0, identity camera) whose centres project to pixel coordinates (u, v) at depth z -- the
    inverse of the rasterizer's ((ndc + 1) * W - 1) / 2."""
    x = ((2 * u + 1) / w - 1) * TANFOV * z
    y = ((2 * v + 1) / h - 1) * TANFOV * z
    return torch.stack([x, y, z], -1)


def edge_straddle_scene(P: int, n_edge: int, views: int, h: int, w: int, seed: int = 0) -> Scene:
    """P ordinary splats plus n_edge whose centres lie within 2 pixels of the last column or the last row (half of them
    each; some beyond the frame), with footprints of 0.5-3 pixels: they reach the pixels of a partial warp column (8
    wide) or row (4 high) of the backward compositor, and the last tile row and column of the frame."""
    sc = make_scene(P, views, h, w, seed=seed)
    g = torch.Generator().manual_seed(seed + 4000)
    z = _U(g, 2.0, 8.0, n_edge)
    right = torch.arange(n_edge) % 2 == 0
    along_u, along_v = _U(g, -1.0, w, n_edge), _U(g, -1.0, h, n_edge)
    u = torch.where(right, (w - 1) + _U(g, -2.0, 2.0, n_edge), along_u)
    v = torch.where(right, along_v, (h - 1) + _U(g, -2.0, 2.0, n_edge))
    means = _at_pixels(u, v, z, h, w)
    f_px = w / (2 * TANFOV)
    sigma = torch.exp(_U(g, math.log(0.5), math.log(3.0), n_edge)) * z / f_px
    scales = sigma[:, None] * torch.exp(_U(g, -0.3, 0.3, n_edge, 3))
    opac = _U(g, 0.2, 0.95, n_edge)
    return _with_extra(sc, means, scales, opac, g)


def long_list_scene(n: int, views: int, h: int, w: int, box=None, n_sparse: int = 0, sparse_box=None,
                    seed: int = 0) -> Scene:
    """n faint, nearly pixel-sized splats (opacity 0.01-0.03, sigma about 0.2 px before the 0.3 px^2 dilation) spread
    over the pixel box (u0, v0, u1, v1) of view 0 at depths 3-8 -- all of them in one 16 x 16 tile when the box is
    inside one: that tile's list is n long, each pixel is reached by about n * 3 / (box area) of them, and its
    transmittance stays far above 1e-4, so its last contributor sits near the end of the list.  Plus n_sparse
    ordinary-sized ones (0.5-2 px, opacity 0.1-0.8) in `sparse_box`, so that the tiles outside both boxes stay empty."""
    sc = make_scene(0, views, h, w, seed=seed)
    g = torch.Generator().manual_seed(seed + 5000)
    f_px = w / (2 * TANFOV)

    def cloud(k, bx, sig_lo, sig_hi, o_lo, o_hi):
        u0, v0, u1, v1 = bx
        z = _U(g, 3.0, 8.0, k)
        means = _at_pixels(_U(g, u0, u1, k), _U(g, v0, v1, k), z, h, w)
        sigma = torch.exp(_U(g, math.log(sig_lo), math.log(sig_hi), k)) * z / f_px
        return means, sigma[:, None] * torch.exp(_U(g, -0.2, 0.2, k, 3)), _U(g, o_lo, o_hi, k)

    m, s, o = cloud(n, box or (0.0, 0.0, w - 1.0, h - 1.0), 0.15, 0.3, 0.01, 0.03)
    if n_sparse:
        m2, s2, o2 = cloud(n_sparse, sparse_box, 0.5, 2.0, 0.1, 0.8)
        m, s, o = torch.cat([m, m2]), torch.cat([s, s2]), torch.cat([o, o2])
    return _with_extra(sc, m, s, o, g)


def stacked_views_cameras(sc: Scene, views_per_chunk: int = 8, step: float = 8.0) -> Scene:
    """sc with view k moved back along the optical axis by step * (k // views_per_chunk): each chunk of views sees the
    cloud at its own range of depths (the depth-stratum boundaries of one chunk do not fit the next)."""
    ext = sc.extrinsics.clone()
    k = torch.arange(ext.shape[0])
    ext[:, 2, 3] = -step * (k // views_per_chunk).float()
    kw = dict(sc.__dict__)
    kw["extrinsics"] = ext
    return Scene(**kw)


# ---------------------------------------------------------------------------------------------------------------------
# Designed tile lists: exactly n splats in chosen (view, tile) cells, for checking the rasterizer's tile lists
# ---------------------------------------------------------------------------------------------------------------------
DEPTH_PATTERNS = ("random", "equal", "ulp", "binades", "reversed")
PARKED = (0.0, 0.0, 0.1)   # world point in front of neither designed camera (z = 0.1 in view 0, -0.1 in view 1)


def designed_cameras(views: int):
    """View 0 = identity; view 1 = turned half a circle about the y axis (it looks along -z).  Each view's splats are
    behind the other's camera, so no splat reaches a tile of another view.  Both rotations are exact in fp32, so a
    splat's camera-space depth is its world z (or -z) bit for bit."""
    assert 1 <= views <= 2
    ext, intr, near, far, bg = make_cameras(views, 16, 16)
    ext = torch.eye(4).repeat(views, 1, 1)
    if views == 2:
        ext[1] = torch.diag(torch.tensor([-1.0, 1.0, -1.0, 1.0]))
    return ext, intr, near, far, bg


def designed_depths(pattern: str, n: int, g) -> torch.Tensor:
    """n camera-space depths (float32) of one tile's splats, by pattern:
    random    U(3, 8);
    equal     all 5.0 (ties settled by index; every depth digit of the keys is the same);
    ulp       384 consecutive float32 values from 5.0 on, repeated: >= 256 distinct depths, one top 16 bits;
    binades   log-uniform in (0.25, 1e3): every byte of the depth word varies;
    reversed  decreasing with the index, 8 down to 3."""
    if pattern == "random":
        return _U(g, 3.0, 8.0, n)
    if pattern == "equal":
        return torch.full((n,), 5.0)
    if pattern == "ulp":
        base = torch.tensor([5.0]).view(torch.int32)
        return (base + (torch.arange(n, dtype=torch.int32) % 384)).view(torch.float32)
    if pattern == "binades":
        return torch.exp(_U(g, math.log(0.25), math.log(1e3), n))
    if pattern == "reversed":
        return torch.linspace(8.0, 3.0, n)
    raise ValueError(pattern)


class Designed:
    """Splats placed into (view, tile) cells, in the order of the cells: means (n, 3), scales (n, 3), rotations (n, 4),
    cov6 (n, 6), opacities (n,), sh (n, d_sh, 3); view, tile and pixel centre (u, v) of each; lengths {(view, tile): n}."""

    def __init__(self, **kw):
        self.__dict__.update(kw)


def designed_tiles(h: int, w: int, cells, d_sh: int = 1, seed: int = 0) -> Designed:
    """cells: (view, tile_x, tile_y, n, pattern) -- n faint, nearly pixel-sized splats (sigma 0.15-0.3 px before the
    0.3 px^2 dilation: a 3-sigma radius of 3 px) centred at least 4 px inside the 16 x 16 tile, so that the tile's list
    is exactly n long and no other tile's list holds them (tests/test_sync_free_cpu.py checks this in fp64)."""
    g = torch.Generator().manual_seed(seed + 6000)
    f_px = w / (2 * TANFOV)
    gx = -(-w // 16)
    out = {k: [] for k in ("means", "scales", "rot", "opac", "view", "tile", "u", "v")}
    lengths = {}
    for view, tx, ty, n, pattern in cells:
        assert 16 * tx + 12 <= w and 16 * ty + 12 <= h, (tx, ty)
        key = (view, ty * gx + tx)
        assert key not in lengths, key
        lengths[key] = n
        z = designed_depths(pattern, n, g)
        u, v = _U(g, 16 * tx + 4, 16 * tx + 12, n), _U(g, 16 * ty + 4, 16 * ty + 12, n)
        cam = _at_pixels(u, v, z, h, w)
        if view == 1:
            cam = cam * torch.tensor([-1.0, 1.0, -1.0])          # world = R cam, R = diag(-1, 1, -1)
        sigma = torch.exp(_U(g, math.log(0.15), math.log(0.3), n)) * z / f_px
        q = torch.randn(n, 4, generator=g)
        for k, t in (("means", cam), ("scales", sigma[:, None] * torch.exp(_U(g, -0.2, 0.2, n, 3))),
                     ("rot", q / q.norm(dim=-1, keepdim=True)), ("opac", _U(g, 0.01, 0.03, n)),
                     ("view", torch.full((n,), view)), ("tile", torch.full((n,), key[1])), ("u", u), ("v", v)):
            out[k].append(t)
    c = {k: torch.cat(t) for k, t in out.items()}
    n = c["means"].shape[0]
    R = quat_to_rotmat(c["rot"])
    cov = R @ torch.diag_embed(c["scales"] ** 2) @ R.transpose(-1, -2)
    cov6 = torch.stack([cov[:, 0, 0], cov[:, 0, 1], cov[:, 0, 2], cov[:, 1, 1], cov[:, 1, 2], cov[:, 2, 2]], -1)
    mask = torch.full((d_sh,), 0.05)
    mask[0] = 1.0
    sh = (torch.randn(n, 3, d_sh, generator=g) * mask).transpose(1, 2).contiguous()
    return Designed(means=c["means"].contiguous(), scales=c["scales"].contiguous(), rotations=c["rot"].contiguous(),
                    cov6=cov6.contiguous(), opacities=c["opac"], sh=sh, view=c["view"], tile=c["tile"], u=c["u"],
                    v=c["v"], lengths=lengths, h=h, w=w)


def designed_tile_of(d: Designed, views: int):
    """fp64 restatement of the projection and the 3-sigma tile rect of every designed splat in every view, with a
    1 px margin: (tile each splat certainly covers alone, or -1 when it is culled; (n, views) int64)."""
    ext = designed_cameras(views)[0].double()
    tan = 0.5 / 0.86
    m, cov = d.means.double(), torch.zeros(d.means.shape[0], 3, 3, dtype=torch.float64)
    c6 = d.cov6.double()
    for k, (i, j) in enumerate(((0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2))):
        cov[:, i, j] = cov[:, j, i] = c6[:, k]
    gx = -(-d.w // 16)
    out = torch.full((m.shape[0], views), -2, dtype=torch.int64)
    for view in range(views):
        R, t = ext[view, :3, :3], ext[view, :3, 3]
        p = (m - t) @ R                                           # R^T (x - t)
        x, y, z = p.unbind(-1)
        culled = z <= 0.2
        zs = torch.where(culled, torch.ones_like(z), z)
        fx, fy = d.w / (2 * tan), d.h / (2 * tan)
        px = ((x / zs / tan + 1) * d.w - 1) / 2
        py = ((y / zs / tan + 1) * d.h - 1) / 2
        J = torch.zeros(m.shape[0], 2, 3, dtype=torch.float64)
        J[:, 0, 0], J[:, 0, 2] = fx / zs, -fx * x / zs ** 2
        J[:, 1, 1], J[:, 1, 2] = fy / zs, -fy * y / zs ** 2
        T = J @ R.T
        c2 = T @ cov @ T.transpose(-1, -2) + 0.3 * torch.eye(2, dtype=torch.float64)
        a, b, cc = c2[:, 0, 0], c2[:, 0, 1], c2[:, 1, 1]
        mid, det = 0.5 * (a + cc), a * cc - b * b
        rad = torch.ceil(3 * torch.sqrt(mid + torch.sqrt(torch.clamp(mid * mid - det, min=0.1))))
        lo_x, hi_x = torch.floor((px - rad - 1) / 16), torch.floor((px + rad + 1) / 16)
        lo_y, hi_y = torch.floor((py - rad - 1) / 16), torch.floor((py + rad + 1) / 16)
        inside = (lo_x == hi_x) & (lo_y == hi_y) & (lo_x >= 0) & (lo_y >= 0)
        tile = torch.where(inside, (lo_y * gx + lo_x).long(), torch.full_like(lo_x, -2).long())
        out[:, view] = torch.where(culled, torch.full_like(tile, -1), tile)
    return out


def _spread(lengths, views, gx, gy, pattern="random"):
    """cells for `lengths`, dealt to the views in turn and to the tiles of each view in row-major order"""
    cells, nxt = [], [0] * views
    for k, n in enumerate(lengths):
        v = k % views
        t = nxt[v]
        nxt[v] += 1
        cells.append((v, t % gx, t // gx, n, pattern if isinstance(pattern, str) else pattern[k]))
    assert max(nxt) <= gx * gy
    return cells


CLASS_EDGES = (1, 1023, 1024, 1025, 2047, 2048, 2049, 4095, 4096, 4097, 8191, 8192)
LONG_LISTS = ((0, 0, 0, 8193, "random"), (0, 1, 0, 9216, "equal"), (0, 2, 0, 9217, "ulp"), (0, 1, 1, 700, "random"),
              (1, 1, 1, 16384, "binades"), (1, 2, 1, 65537, "reversed"), (1, 3, 1, 9217, "random"))
# the cells of the shifting-lists sequence at their longest (each call keeps the first k splats of each)
SHIFT_POOL = ((0, 0, 0, 9300, "random"), (0, 1, 0, 4200, "ulp"), (0, 2, 1, 2100, "reversed"), (1, 0, 0, 8300, "equal"),
              (1, 3, 2, 1100, "binades"))
SHIFT_CALLS = ((1024, 1024, 2048, 8192, 1024), (1025, 2049, 2049, 8193, 1), (9300, 4200, 2100, 8300, 1100),
               (8192, 4096, 2048, 1024, 0), (8193, 4097, 1025, 1025, 1100), (0, 0, 0, 0, 0), (9216, 4095, 2047, 8191, 1023),
               (9217, 1, 2100, 8192, 1024), (1, 4200, 1, 8300, 1), (4096, 2048, 1024, 8193, 1025),
               (9299, 4199, 2099, 4000, 1099), (8193, 2049, 1025, 4097, 1))


def designed_case(name: str):
    """(h, w, views, cells) of the designed-list cases of tests/test_gpu_sync_free_regimes.py"""
    if name == "class_edges":
        return 64, 64, 2, _spread(CLASS_EDGES, 2, 4, 4)
    if name == "class_edges_8193":
        return 64, 64, 2, _spread(CLASS_EDGES + (8193,), 2, 4, 4)
    if name == "long_lists":
        return 48, 64, 2, list(LONG_LISTS)
    if name.startswith("pattern_"):
        p = name[len("pattern_"):]
        return 48, 48, 1, [(0, 0, 0, 8193, p), (0, 1, 0, 20000, p), (0, 2, 1, 3000, p)]
    if name == "index_digit3":
        return 32, 32, 1, [(0, 1, 1, 10096, "random")]
    if name == "shifting":
        return 48, 64, 2, list(SHIFT_POOL)
    if name == "scene_long":
        return 48, 48, 2, [(0, 0, 0, 9000, "random"), (1, 1, 1, 20000, "binades"), (0, 2, 2, 300, "equal")]
    if name == "scene_ordinary":
        return 48, 48, 2, _spread((100, 700, 1500, 3000, 40, 2200), 2, 3, 3)
    raise ValueError(name)


DESIGNED_CASES = ("class_edges", "class_edges_8193", "long_lists", "index_digit3", "shifting", "scene_long",
                  "scene_ordinary") + tuple("pattern_" + p for p in DEPTH_PATTERNS)
