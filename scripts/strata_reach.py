"""How much of the stratum sort lies behind saturation: CPU estimate on the C2 shape (DESIGN.md 5.2, 8).

For every (view, tile) of C2 (500k Gaussians, 8 views, 256x256) the CPU oracle gives the tile's depth-ordered list and
every pixel's n_contrib / final_T.  The compositor stops a tile at the first list position where every pixel is
saturated (T < 1e-4); positions past it are never read.  The list is cut into per-view depth octiles the way
k_depth_hist / k_strata_from_hist cut it (2048 log-spaced bins, weighted by each Gaussian's candidate-tile count), and
the script reports the share of (view, tile, stratum) triples, and of tile instances, that lie wholly behind the last
position the compositor reads -- with and without the one-stratum margin a learned table would keep.

ESTIMATE: the oracle bins with upstream's 3-sigma squares, not the tight per-tile test of the CUDA binning, so its lists
are longer than the device's and its octile weights differ.

    python scripts/strata_reach.py [--gaussians 500000 --views 8 --size 256]
"""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from pf3plat_b200.synthetic import make_scene  # noqa: E402
from tests.util import oracle_view  # noqa: E402

BIN_SUB = 8
STRATA_BINS = 2048
STRATA_BASE = 0x3E000000 >> 17  # bit pattern of 0.125f, in bin units


def depth_bin(d: np.ndarray) -> np.ndarray:
    b = (d.astype(np.float32).view(np.uint32) >> 17).astype(np.int64) - STRATA_BASE
    return np.clip(b, 0, STRATA_BINS - 1)


def view_boundaries(depths: np.ndarray, weight: np.ndarray) -> np.ndarray:
    """k_strata_from_hist: boundary q-1 = upper edge of the bin that completes the q/8 quantile of the weighted depths."""
    hist = np.bincount(depth_bin(depths[weight > 0]), weights=weight[weight > 0], minlength=STRATA_BINS).astype(np.uint64)
    bounds = np.full(BIN_SUB, np.inf, np.float32)
    total = int(hist.sum())
    if total == 0:
        return bounds
    cum = np.concatenate([[0], np.cumsum(hist)])  # cum[b] = mass below bin b
    for q in range(1, BIN_SUB):
        target = (total * q + BIN_SUB - 1) // BIN_SUB
        b = int(np.argmax(cum[1:] >= target))  # first bin whose upper edge reaches the target
        bounds[q - 1] = np.uint32((b + 1 + STRATA_BASE) << 17).view(np.float32)
    return bounds


def tile_reach(o, xy, co, ids, nc, tx, ty) -> int:
    """Last list position (0-based) any pixel of the tile reads.  A pixel's last contributor sits at n_contrib - 1; the
    next entry with alpha >= 1/255 there is the one that saturates it (T < 1e-4, not added).  A pixel without such an
    entry never saturates and reads the whole list."""
    ys = np.arange(ty * 16, min(ty * 16 + 16, o.H))
    xs = np.arange(tx * 16, min(tx * 16 + 16, o.W))
    px, py = np.meshgrid(xs, ys)
    px, py = px.ravel().astype(np.float32), py.ravel().astype(np.float32)
    first = nc[py.astype(int), px.astype(int)].astype(np.int64)
    lo = int(first.min())
    g = ids[lo:]
    dx, dy = xy[g, 0:1] - px[None], xy[g, 1:2] - py[None]
    c = co[g]
    power = -0.5 * (c[:, 0:1] * dx * dx + c[:, 2:3] * dy * dy) - c[:, 1:2] * dx * dy
    hit = (power <= 0) & (np.minimum(0.99, c[:, 3:4] * np.exp(np.minimum(power, 0))) >= 1 / 255)
    hit &= (np.arange(lo, len(ids))[:, None] >= first[None])
    if not hit.any(axis=0).all():
        return len(ids) - 1
    return lo + int(hit.argmax(axis=0).max())


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--gaussians", type=int, default=500_000)
    ap.add_argument("--views", type=int, default=8)
    ap.add_argument("--size", type=int, default=256)
    a = ap.parse_args()
    sc = make_scene(a.gaussians, a.views, a.size, a.size, seed=0)
    triples = nonempty = behind = behind_margin = 0
    inst = inst_behind = inst_behind_margin = 0
    need_hist = np.zeros(BIN_SUB + 1, np.int64)
    for v in range(a.views):
        o = oracle_view(sc, v)
        depths, touched = o.depths, o.tiles_touched
        bounds = view_boundaries(depths, touched.astype(np.float64))
        pl, rg = o.point_list, o.ranges
        nc, xy, co = o.n_contrib, o.xy, o.conic_opacity
        gx, gy = (o.W + 15) // 16, (o.H + 15) // 16
        for t in range(gx * gy):
            ty, tx = divmod(t, gx)
            s, e = int(rg[t, 0]), int(rg[t, 1])
            n = e - s
            ids = pl[s:e]
            strat = np.searchsorted(bounds[:BIN_SUB - 1], depths[ids], side="right")  # sum of (d >= b_q)
            cnt = np.bincount(strat, minlength=BIN_SUB)
            start = np.concatenate([[0], np.cumsum(cnt)])
            if n == 0:
                need = 0
            else:
                last = min(tile_reach(o, xy, co, ids, nc, tx, ty), n - 1)
                need = int(np.searchsorted(start[1:], last, side="right")) + 1
            need_hist[need] += 1
            for k in range(BIN_SUB):
                triples += 1
                if cnt[k] == 0:
                    continue
                nonempty += 1
                inst += int(cnt[k])
                if k >= need:
                    behind += 1
                    inst_behind += int(cnt[k])
                if k >= need + 1:
                    behind_margin += 1
                    inst_behind_margin += int(cnt[k])
        print(f"view {v}: {gx * gy} tiles, mean list {len(pl) / (gx * gy):.0f}", flush=True)
        o.close()
    print("ESTIMATE from the CPU oracle: 3-sigma square binning, not the tight per-tile lists of the CUDA path")
    print(f"(view, tile, stratum) triples: {triples}, non-empty {nonempty}")
    print(f"strata needed per tile (histogram 0..8): {need_hist.tolist()}")
    print(f"behind the last read position:       {behind / nonempty:.1%} of non-empty strata, "
          f"{inst_behind / inst:.1%} of instances")
    print(f"behind it with a one-stratum margin: {behind_margin / nonempty:.1%} of non-empty strata, "
          f"{inst_behind_margin / inst:.1%} of instances")


if __name__ == "__main__":
    main()
