// gs_bin_policy.h -- how a forward bins its tile instances and what a context learns about a shape from each call: shape
// slots, bucket capacities, the depth-strata state machine (DESIGN.md 5.2).  Host-only C++ without CUDA, so that
// tests/test_bin_policy_cpu.py replays call sequences on the CPU; gs_forward (gs_capi.cu) carries the plans out.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include "../../include/gsplat_b200.h"

#define BIN_SMEM_CAP 8192  // longest tile list the shared-memory merge sort takes (256 threads x 32 keys)
#define BIN_SUB 8          // sub-counters per (view, tile), selected by Gaussian index & (BIN_SUB-1)
constexpr uint32_t BIN_STRATUM_CAP = 2048;  // longest sub-bucket k_stratum_sort handles (128 threads x 16 keys)
// Bigger bucket sets are filled by the view-major k_emit_buckets: appends from preprocess touch all views' buckets, far
// beyond L2 as partial-sector DRAM writes.  C2's (above the 50 MB L2) still fill faster from preprocess on an H100 (README.md).
constexpr size_t BIN_FUSED_EMIT_MAX_BYTES = (size_t)96 << 20;
// Lazy strata: k_composite_fwd sorts a stratum the stratum sort skipped in its record stage (2 x 256 x 48 bytes), as
// 8-byte keys.  A shape whose sub-buckets do not fit it sorts every stratum up front.
constexpr size_t BIN_LAZY_STAGE_BYTES = 2 * 256 * 48;
inline bool lazy_stratum_fits(uint32_t sub_cap) { return (size_t)sub_cap * 8 <= BIN_LAZY_STAGE_BYTES; }

enum { STRATA_UNKNOWN = 0, STRATA_TRIAL = 1, STRATA_ON = 2, STRATA_OFF = 3 };

// what earlier forwards of one shape taught (sub_cap 0: none yet, or lists too long: exact path)
struct SpecState {
    uint32_t sub_cap = 0;     // capacity of one of a tile's BIN_SUB sub-buckets
    uint32_t tile_limit = 0;  // list length the tile sort is launched for
    int strata_state = STRATA_UNKNOWN;
    // per_tile: the per-view trial overflowed (tiles that each see a narrow depth range, e.g. PF3plat's pixel-aligned
    // Gaussians on a smooth surface), so boundaries are learned per (view, tile) from the exact call's sorted lists and
    // refreshed by every stratum sort: two tables, tile_tab the one to read, swapped on success
    int per_tile = 0, tile_tab = 0;
    // the shape's "strata needed" table (one byte per (view, tile): how many of the tile's strata its last forward read)
    // holds what a committed lazy forward wrote; otherwise it must be reset to BIN_SUB (sort everything) before use
    bool need_learned = false;
};

// A context remembers a few shapes (views, tiles, Gaussians per scene, scenes), so a caller that alternates shapes --
// context and target views, training and validation batches -- keeps every one of them on the speculative path.
struct BinShape {
    int V, ntiles, P, S;
};
struct ShapeSlot {
    BinShape key{-1, -1, -1, -1};
    uint64_t last_use = 0;
    SpecState spec;
};

// index of this shape's slot; on a miss the least recently used slot, its state reset (the caller keeps the slot's
// boundary tables: the exact call re-fills them)
inline int pick_slot(ShapeSlot *slots, int count, uint64_t &use_counter, const BinShape &k) {
    int hit = -1, lru = 0;
    for (int i = 0; i < count; i++) {
        const BinShape &s = slots[i].key;
        if (s.V == k.V && s.ntiles == k.ntiles && s.P == k.P && s.S == k.S) hit = i;
        if (slots[i].last_use < slots[lru].last_use) lru = i;
    }
    if (hit < 0) {
        hit = lru;
        slots[hit].spec = SpecState{};
        slots[hit].key = k;
    }
    slots[hit].last_use = ++use_counter;
    return hit;
}

// How one forward bins: speculative (fixed-capacity sub-buckets, verified afterwards) or exact (count, scan, sync, emit).
struct BinPlan {
    bool speculate = false;
    bool strata = false;       // sub-bucket = depth stratum (else Gaussian index % BIN_SUB)
    int per_tile = 0;          // strata: boundaries per (view, tile) instead of per view
    uint32_t sub_cap = 0;      // capacity of one sub-bucket
    int read_tab = -1;         // boundary table the emission reads (index into the slot's tables; -1: none)
    int write_tab = -1;        // table the stratum sort writes the next call's boundaries into (-1: none)
    bool fused_emit = false;   // preprocess appends to the buckets itself (else k_emit_buckets)
    // per-view strata with the rank sort: the stratum sort sorts only the strata the tile's last forward needed, the
    // compositor sorts any further one it reaches and records what this call needed; reset_need: the table is stale
    bool lazy_strata = false, reset_need = false;
};

inline BinPlan plan_binning(const SpecState &s, const BinShape &sh, size_t n, bool have_table, uint32_t tuning) {
    BinPlan p;
    p.speculate = s.sub_cap > 0 && n > 0 && !(tuning & (GS_TUNE_FORCE_RADIX_BINNING | GS_TUNE_NO_SPECULATION));
    if (!p.speculate) return p;
    const size_t slots = (size_t)sh.V * sh.ntiles * BIN_SUB;
    p.strata = (s.strata_state == STRATA_TRIAL || s.strata_state == STRATA_ON) && !(tuning & GS_TUNE_NO_STRATA) && have_table;
    p.sub_cap = s.sub_cap;
    if (p.strata && s.strata_state == STRATA_TRIAL) {
        // capacities were learned unstratified: the trial runs on doubled ones -- if the kernels' 32-bit bucket
        // offsets still hold them (learn_capacities checked the undoubled value only)
        uint32_t trial = p.sub_cap * 2;
        if (trial > BIN_STRATUM_CAP) trial = BIN_STRATUM_CAP;
        if ((uint64_t)trial * slots > 0xffffffffull) p.strata = false;
        else p.sub_cap = trial;
    }
    if (p.strata && p.sub_cap > BIN_STRATUM_CAP) p.sub_cap = BIN_STRATUM_CAP;
    p.per_tile = p.strata ? s.per_tile : 0;
    if (p.strata) p.read_tab = p.per_tile ? s.tile_tab : 0;
    if (p.strata && p.per_tile) p.write_tab = s.tile_tab ^ 1;
    p.fused_emit = slots * p.sub_cap * 8 <= BIN_FUSED_EMIT_MAX_BYTES && !(tuning & GS_TUNE_SEPARATE_EMIT);
    // per-tile boundaries are refreshed by the stratum sort from every position of the list, the merge sort and the
    // warp-specialised compositor have no lazy counterpart
    p.lazy_strata = p.strata && !p.per_tile && lazy_stratum_fits(p.sub_cap) &&
                    !(tuning & (GS_TUNE_ALL_STRATA | GS_TUNE_STRATA_MERGE_SORT | GS_TUNE_FWD_WS));
    p.reset_need = p.lazy_strata && !s.need_learned;
    return p;
}

// 64-quantised; the current capacity is kept while it fits and is at most 1.5x the need, so that a cloud that moves a
// little every step asks the memory pool for the same block sizes call after call (DESIGN.md 4)
inline uint32_t sticky_capacity(uint32_t need, uint32_t current) {
    need = (need + 63u) & ~63u;
    return (current >= need && (uint64_t)current * 2 <= (uint64_t)need * 3) ? current : need;
}

// capacities for the next forward of this shape: 30 % headroom over the largest sub-counter, 10 % over the longest list
inline void learn_capacities(SpecState &s, const BinShape &sh, uint32_t max_tile, uint32_t max_sub) {
    const uint32_t sub_cap = sticky_capacity(max_sub + max_sub * 3 / 10 + 16, s.sub_cap);
    const uint32_t limit = sticky_capacity(max_tile + max_tile / 10 + 32, s.tile_limit);
    if (limit > BIN_SMEM_CAP || (uint64_t)sub_cap * BIN_SUB * sh.V * sh.ntiles > 0xffffffffull) {
        s.sub_cap = 0;  // lists too long for the shared-memory sort (or offsets beyond 32 bits): exact path
        return;
    }
    s.sub_cap = sub_cap;
    s.tile_limit = limit;
}

// After a speculative call, from its verdict words ([0] tile instances, [1] longest tile list, [2] largest
// sub-counter, [3] overflow).  Returns false when the results are invalid and the call is redone on the exact path.
// *release_sort: the trial's generous buckets (sort_bytes of them) are not needed again.
inline bool learn_speculative(SpecState &s, const BinShape &sh, const BinPlan &p, const uint32_t *words, size_t sort_bytes,
                              uint32_t tuning, bool *release_sort) {
    *release_sort = false;
    s.need_learned = p.lazy_strata && words[3] == 0;  // an overflowed call's compositor read clamped lists
    if (words[3] != 0) {
        s.sub_cap = 0;
        if (p.strata) {
            if (s.strata_state == STRATA_TRIAL && !p.per_tile && !(tuning & GS_TUNE_NO_TILE_STRATA)) {
                s.per_tile = 1;   // the per-view boundaries crowd some tile into one stratum: the redo learns per-tile ones
                s.strata_state = STRATA_UNKNOWN;
            } else {
                s.strata_state = s.strata_state == STRATA_TRIAL ? STRATA_OFF : STRATA_UNKNOWN;
            }
        }
        return false;
    }
    if (!p.strata) {
        learn_capacities(s, sh, words[1], words[2]);
        return true;
    }
    uint32_t next = sticky_capacity(words[2] + words[2] * 3 / 10 + 16, s.strata_state == STRATA_ON ? p.sub_cap : 0u);
    if (next > BIN_STRATUM_CAP && words[2] + words[2] / 10 <= BIN_STRATUM_CAP) next = BIN_STRATUM_CAP;  // 10 % headroom still fits
    if (next > BIN_STRATUM_CAP) {   // a stratum beyond the small sort's capacity: whole-tile sorts from now on
        s.strata_state = STRATA_OFF;
        s.sub_cap = 0;
        return true;
    }
    const size_t slots = (size_t)sh.V * sh.ntiles * BIN_SUB;
    *release_sort = s.strata_state == STRATA_TRIAL && sort_bytes > 2 * (slots * (size_t)next * 8) + ((size_t)8 << 20);
    s.strata_state = STRATA_ON;
    s.sub_cap = next;
    if (p.per_tile) s.tile_tab ^= 1;  // the sort wrote the next call's boundaries into the other table
    return true;
}

// After an exact call's scan: learns capacities and returns which depth-stratum boundaries the call should learn
// (only after a shared-memory sort; OFF is sticky).  Once they are enqueued, start_trial makes the next call the trial.
enum { LEARN_NONE = 0, LEARN_PER_VIEW = 1, LEARN_PER_TILE = 2 };

inline int learn_exact(SpecState &s, const BinShape &sh, size_t n, uint32_t max_tile, uint32_t max_sub, bool smem_sort,
                       uint32_t tuning) {
    s.need_learned = false;
    learn_capacities(s, sh, max_tile, max_sub);
    if (!(smem_sort && s.sub_cap > 0 && s.strata_state != STRATA_OFF && !(tuning & GS_TUNE_NO_STRATA) && n > 0))
        return LEARN_NONE;
    return s.per_tile ? LEARN_PER_TILE : LEARN_PER_VIEW;
}

inline void start_trial(SpecState &s) {
    s.strata_state = STRATA_TRIAL;
    s.tile_tab = 0;   // per-tile boundaries are learned into the first table
}
