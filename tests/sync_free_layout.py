"""The byte layout of a sync-free workspace (gs_capi.cu: sf_layout and saved_layout, DESIGN.md 5.18), restated per
region, and a reader that copies one forward's tile lists back from the workspace and checks them against a plain sort.

Layout: 256 bytes of status words | the saved planes rec0, rec1, rec2, meta, ranges, final_T, n_contrib, sched |
point_list[capacity] | scratch, which holds either the forward's binning buffers or the backward's accumulators.  Every
region starts 256-byte aligned.  `regions` is used by the CPU test that compares the total with
gs_sync_free_workspace_bytes, so the offsets the GPU checks read at are the ones that total is checked with."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

TILE = 16
BIN_SUB = 8
STATUS_WORDS = ("D", "max_list", "max_sub", "verdict", "exceeded", "required")   # SF_D .. SF_REQUIRED


def _align(x):
    return (x + 255) // 256 * 256


def regions(S, V, P, H, W, cap, det=False, cam=False) -> dict:
    """{name: (byte offset, bytes)} of every region of the workspace, plus "total" -> (0, workspace bytes).  The
    forward's binning buffers and the backward's accumulators share the scratch; "backward" spans the latter."""
    n, ntiles = V * P, -(-W // TILE) * -(-H // TILE)
    nvt, px, cap1 = V * ntiles, V * H * W, max(cap, 1)
    out, off = {}, 0

    def take(name, nbytes):
        nonlocal off
        out[name] = (off, nbytes)
        off += _align(nbytes)

    take("status", 256)
    for name, nbytes in (("rec0", n * 16), ("rec1", n * 16), ("rec2", n * 16), ("meta", n), ("ranges", nvt * 8),
                         ("final_T", px * 4), ("n_contrib", px * 4), ("sched", 8), ("point_list", cap1 * 4)):
        take(name, nbytes)
    scratch = off
    ctr = nvt * BIN_SUB * 8 * 4                 # BIN_SUB sub-counters per tile, one per 32-byte sector
    for name, nbytes in (("rects", n * 8), ("tile_counts", ctr), ("cursor", ctr), ("sub_offsets", nvt * BIN_SUB * 4),
                         ("tile_start", nvt * 4), ("tile_n", nvt * 4), ("bucket", cap1 * 8), ("tmp", cap1 * 8)):
        take(name, nbytes)
    warps = -(-P // 128) * 4                    # preprocess-backward warps of one scene
    acc = n * (10 * 3 * 8 + 4) if det else n * 10 * 4
    bwd = _align(acc) + max(warps * V * 32 * 4 if cam else 0, V * warps * 4 * 4 if det else 0)
    out["backward"] = (scratch, bwd)
    out["total"] = (0, max(off, scratch + bwd))
    return out


@dataclass
class TileLists:
    status: dict            # SF_* words by name
    ranges: np.ndarray      # [V * ntiles, 2] uint32
    lengths: np.ndarray     # [V * ntiles] int64
    index: np.ndarray       # point_list[:D] (uint32)
    tile: np.ndarray        # the (view, tile) of each entry
    depth_bits: np.ndarray  # rec2[v * P + i].y of each entry, as its float32 bits (uint32)
    ntiles: int

    def keys(self):
        return (self.depth_bits.astype(np.uint64) << np.uint64(32)) | self.index.astype(np.uint64)

    def tile_entries(self, v, t):
        """(index, depth bits) of the list of view v, tile t"""
        a, b = (int(x) for x in self.ranges[v * self.ntiles + t])
        return self.index[a:b], self.depth_bits[a:b]


def read_lists(ws) -> TileLists:
    """Status words, ranges, point_list[:D] and the listed splats' depths of the last forward on SyncFreeWorkspace `ws`
    (nothing but the status words and ranges when that forward exceeded the capacity)."""
    import torch
    S, V, P, H, W = ws.dims
    reg = regions(S, V, P, H, W, ws.instance_capacity, ws.deterministic, ws.camera_grad)
    buf = ws.buffer

    def words(name, count=None):
        off, nbytes = reg[name]
        return buf[off:off + (nbytes if count is None else count * 4)].view(torch.int32)

    status = dict(zip(STATUS_WORDS, (words("status", 6).cpu().numpy().view(np.uint32)).tolist()))
    ranges = words("ranges").cpu().numpy().view(np.uint32).reshape(-1, 2)
    ntiles = ranges.shape[0] // V
    lengths = ranges[:, 1].astype(np.int64) - ranges[:, 0].astype(np.int64)
    D = status["D"]
    if status["verdict"] or D == 0:
        empty = np.zeros(0, np.uint32)
        return TileLists(status, ranges, lengths, empty, empty.astype(np.int64), empty, ntiles)
    lst = words("point_list", D)
    tile = np.repeat(np.arange(V * ntiles), np.maximum(lengths, 0))
    assert tile.shape[0] == D, ("the ranges do not cover point_list[:D]", tile.shape[0], D)
    view = torch.from_numpy(tile // ntiles).to(buf.device)
    rec2_y = words("rec2").view(-1, 4)[:, 1]
    gi = view * P + (lst.long() & 0xffffffff).clamp_max(max(P - 1, 0))   # (a bad index fails the check below)
    depth = rec2_y[gi]
    return TileLists(status, ranges, lengths, lst.cpu().numpy().view(np.uint32), tile,
                     depth.cpu().numpy().view(np.uint32), ntiles)


def check_lists(ws, radii, lengths=None, D=None) -> TileLists:
    """Reads the last forward's lists from `ws` and checks them against a sort: the ranges are the exclusive scan of the
    per-tile lengths in (view, tile) order, ending at SF_D, the longest is SF_MAX_LIST; every listed index is below P and
    drawn (radii > 0) in its view; within a tile the keys (depth bits << 32 | index) increase strictly -- np.lexsort's
    order of (index, depth), the radix fallback's.  `lengths` ({(view, tile): n}, every other tile empty) and D, when
    given, are the designed ones.  An exceeded forward must have every range empty and its verdict set."""
    lists = read_lists(ws)
    st, r = lists.status, lists.ranges
    S, V, P, H, W = ws.dims
    if D is not None:
        assert st["D"] == D, (st["D"], D)
    if st["D"] > ws.instance_capacity:
        assert st["verdict"] == 1 and st["exceeded"] == 1, st
        assert not r.any(), "an exceeded forward left a non-empty range"
        return lists
    assert st["verdict"] == 0, st
    n = lists.lengths
    assert (n >= 0).all()
    starts = np.concatenate([[0], np.cumsum(n)[:-1]])
    assert np.array_equal(r[:, 0].astype(np.int64), starts), "ranges are not the exclusive scan of the lengths"
    assert int(n.sum()) == st["D"] and int(r[-1, 1]) == st["D"], (int(n.sum()), st["D"])
    assert int(n.max(initial=0)) == st["max_list"], (int(n.max(initial=0)), st["max_list"])
    if lengths is not None:
        want = np.zeros_like(n)
        for (v, t), k in lengths.items():
            want[v * lists.ntiles + t] = k
        bad = np.nonzero(want != n)[0]
        assert bad.size == 0, [(int(vt // lists.ntiles), int(vt % lists.ntiles), int(n[vt]), int(want[vt]))
                               for vt in bad[:8]]
    if st["D"] == 0:
        return lists
    idx = lists.index.astype(np.int64)
    assert (idx < P).all(), "an index at or above P"
    view = lists.tile // lists.ntiles
    rad = radii.detach().reshape(V, P).cpu().numpy()
    assert (rad[view, idx] > 0).all(), "a listed splat that is not drawn in its view"
    keys = lists.keys()
    same = lists.tile[1:] == lists.tile[:-1]
    order_ok = keys[1:] > keys[:-1]
    bad = np.nonzero(same & ~order_ok)[0]
    assert bad.size == 0, ("keys out of order", [(int(lists.tile[k]), k, hex(int(keys[k])), hex(int(keys[k + 1])))
                                                for k in bad[:8]])
    # the same order as a plain sort of each tile's (depth, index) pairs
    perm = np.lexsort((idx, lists.depth_bits, lists.tile))
    assert np.array_equal(perm, np.arange(idx.shape[0])), "the lists are not in lexsort order"
    return lists
