"""Seeded scenes for the regimes the ordinary synthetic distribution (pf3plat_b200.synthetic.make_scene: centres inside
+-1.05 NDC, depths >= 1.5, opacities U(0.05, 1)) never reaches.  Each is small enough for the CPU oracle and is built from
a make_scene cloud, whose cameras it keeps (view 0 is the identity; the others are displaced in the image plane only, so
camera-space z equals world z in every view)."""
from __future__ import annotations

import math

import torch

from pf3plat_b200.synthetic import FX, Scene, make_scene, quat_to_rotmat

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
