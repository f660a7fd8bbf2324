// gs_composite_fwd.cu -- stage 3 of the forward: per-pixel front-to-back alpha compositing.
//
// Semantics: SURVEY.md Appendix A "Composite forward" (upstream renderCUDA): walk the tile's list in
// (depth, index) order; skip power > 0; alpha = min(0.99, o*G); skip alpha < 1/255; stop (without adding)
// when T*(1-alpha) < 1e-4; C += c*alpha*T; out = C + T*bg; keep final T and the last contributor's position.
//
// Design (DESIGN.md section 5.3).  One CTA per (view, 16x16 tile), 8 warps, each warp owning an 8x4 pixel
// block.  Batches of 256 splat records are gathered into a double-buffered shared-memory stage with 16-byte
// cp.async copies (LDGSTS), the next batch in flight while the current one is composited; every warp
// CULLS the batch against its own 8x4 block 32 Gaussians at a time -- lane k tests whether Gaussian k's
// alpha>=1/255 ellipse reaches the block (gs_box_reaches, exact), one ballot yields the survivors -- and only
// survivors are evaluated by the 32 pixel lanes (shared-memory broadcast reads).  With PF3plat-sized splats (sigma 0.1-3 px) this removes ~10x of the
// (pixel, Gaussian) pair evaluations that the reference design spends on alpha < 1/255 rejections, without
// changing a single pixel: a culled Gaussian fails the alpha test at every pixel of the block.
//
// Tried and dropped: fusing the per-tile merge sort (k_tile_sort, latency-bound) into this kernel's
// prologue so that one CTA's sort latency hides behind other CTAs' compositing.  Fused was slower than
// separate on C2 and C4 (the sort's 63-125 registers cut the compositor's occupancy, and
// CTAs of a wave run their phases in lock-step, so little overlap materialises).  Also tried: a two-stage software
// pipeline over groups of views (k_tile_sort of group g+1 on a side stream under the compositing of group g):
// slower than serial on C2 -- the co-resident sort CTAs take registers/shared memory from the
// compositor without filling its idle issue slots.
#include <type_traits>

#include "gs_common.cuh"

namespace {

constexpr int CF_THREADS = 256;
constexpr int CF_BATCH = 256;

// Shared-memory staging: two buffers of one batch each (48-byte records rec0 | rec1 | rec2 of gs_common.cuh).
// While the warps composite batch b out of one buffer, the cp.async (LDGSTS) gathers of batch b+1 land in the other.
struct CfStage {
    float4 rec[CF_BATCH][3];
};
static_assert(2 * sizeof(CfStage) == BIN_LAZY_STAGE_BYTES, "the lazy stratum sort's keys live in the stage");

// Lazy strata, off the compositing path (own frames, so the main loop keeps its registers).
// The tile's next non-empty stratum -- the one whose entries start at list position `sorted` -- is sorted by the whole
// CTA into its final place: its keys into the stage, every key ranked against all of them (keys are unique: depth bits,
// index), its index stored at its rank.  Returns the stratum's length (0: the list is complete).
__device__ __noinline__ uint32_t lazy_sort_next(const LazyStrata lz, uint32_t vt, uint32_t sorted, uint64_t *keys,
                                                uint32_t *list /* the tile's list */) {
    __shared__ uint32_t s_k, s_n;
    if (threadIdx.x == 0) {
        uint32_t below = 0, kk = BIN_SUB, nn = 0;
        for (uint32_t k = 0; k < BIN_SUB; k++) {
            const uint32_t cnt = min(lz.cursor[((size_t)vt * BIN_SUB + k) * BIN_PAD], lz.sub_cap);
            if (below >= sorted && cnt > 0) {  // (the sorted prefix always ends on a stratum boundary)
                kk = k;
                nn = cnt;
                break;
            }
            below += cnt;
        }
        s_k = kk;
        s_n = nn;
    }
    __syncthreads();
    const uint32_t k = s_k, n = s_n;
    if (n == 0) return 0;
    const uint64_t *src = lz.bucket + ((size_t)vt * BIN_SUB + k) * lz.sub_cap;
    for (uint32_t i = threadIdx.x; i < n; i += CF_THREADS) keys[i] = src[i];
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < n; i += CF_THREADS) {
        const uint64_t key = keys[i];
        uint32_t rank = 0;
        for (uint32_t j = 0; j < n; j++) rank += keys[j] < key ? 1u : 0u;
        list[sorted + rank] = (uint32_t)key;
    }
    __syncthreads();  // the entries are visible to the whole CTA, and the stage is free again
    return n;
}

// Lazy strata, when the CTA retires (thread 0): the list's sorted length goes to ranges[vt].y (every later reader of the
// list sees the entries sorted here), and need[vt] = 1 + the stratum of list position `reach` (1-based; 0: none), which
// lies at or a chunk behind the entry that saturated the tile's last pixel, or BIN_SUB when a pixel is not saturated.
__device__ __noinline__ void lazy_record(const LazyStrata lz, uint32_t vt, uint32_t reach, bool all_done, uint2 *range,
                                         uint32_t sorted) {
    uint32_t need = BIN_SUB;
    if (all_done) {
        uint32_t below = 0;
        need = 1;
        for (uint32_t k = 0; k + 1 < BIN_SUB; k++) {
            below += min(lz.cursor[((size_t)vt * BIN_SUB + k) * BIN_PAD], lz.sub_cap);
            need += reach > 0 && below < reach ? 1u : 0u;  // the entry at 0-based position reach - 1 lies past stratum k
        }
    }
    lz.need[vt] = (uint8_t)need;
    range->y = range->x + sorted;
}

// DEPTH: 0 no depth channel; 1 the channel composites rec2.y (GS_DEPTH_Z); 2 it composites rec2.w, the f(z) preprocess
// stored for the other depth modes.  Values 0 and 1 are the kernels of before, instruction for instruction.
// ALPHA: also store the accumulated opacity 1 - T next to final_T (GsAlpha); false is the kernel of before.
// LAZY: lazy strata (`lazy`): past the end of the sorted prefix the CTA sorts the next stratum and composites it as a list
// of its own; false is the kernel of before.
template <int DEPTH, int MINB, bool ALPHA = false, bool LAZY = false>
__global__ void __launch_bounds__(CF_THREADS, MINB)
k_composite_fwd(const DevCfg c, const float4 *__restrict__ rec0, const float4 *__restrict__ rec1,
                const float4 *__restrict__ rec2, const uint32_t *__restrict__ point_list,
                uint2 *__restrict__ ranges, float *__restrict__ color, float *__restrict__ depth,
                float *__restrict__ final_T, uint32_t *__restrict__ n_contrib, float *__restrict__ alpha_out,
                const LazyStrata lazy) {
    __shared__ CfStage stage[2];

    const int v = blockIdx.y;
    const int tile = blockIdx.x;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int bx = (tile % c.gx) * GS_TILE + (warp & 1) * 8;   // this warp's 8x4 pixel block
    const int by = (tile / c.gx) * GS_TILE + (warp >> 1) * 4;
    const int px = bx + (lane & 7), py = by + (lane >> 3);
    const bool inside = px < c.W && py < c.H;
    const float pxf = (float)px, pyf = (float)py;
    const float bx0 = (float)bx, bx1 = (float)(bx + 7), by0 = (float)by, by1 = (float)(by + 3);

    const uint32_t vt = (uint32_t)v * (uint32_t)c.ntiles + (uint32_t)tile;
    const uint2 range = ranges[vt];
    // the list composited below: `total` entries from point_list[lbase] on (LAZY: then each stratum sorted here)
    uint32_t lbase = range.x, total = range.y - range.x;
    const size_t rbase = (size_t)v * c.P;
    const uint32_t stage_addr = smem_u32(&stage[0].rec[0][0]);

    // gather the records of batch b (this thread: list entry b * CF_BATCH + tid, whose index is `id`) into its buffer
    auto gather = [&](uint32_t b, uint32_t id) {
        if (b * CF_BATCH + tid < total) {
            const size_t r = rbase + id;
            float4 *dst = &stage[b & 1].rec[tid][0];
            cp_async16(dst, rec0 + r);
            cp_async16(dst + 1, rec1 + r);
            cp_async16(dst + 2, rec2 + r);
        }
        cp_async_commit();  // one group per batch, empty or not, so that wait_group<1> always means "batch b landed"
    };
    // (LAZY: a coherent load -- entries the CTA sorted itself must not come through the non-coherent path)
    auto load_id = [&](uint32_t b) -> uint32_t {
        const uint32_t e = b * CF_BATCH + tid;
        return e < total ? (LAZY ? __ldca(point_list + lbase + e) : point_list[lbase + e]) : 0u;
    };

    float T = 1.0f, C0 = 0.f, C1 = 0.f, C2 = 0.f, Dz = 0.f;
    uint32_t last = 0;
    bool done = !inside;
    bool warp_done = false;
    // LAZY: per warp, the 1-based list position of the last entry of the 32-entry chunk in which its last pixel saturated
    // (0: not yet).  Recorded where the warp leaves the list: anything inside the survivor loop costs it the uniform
    // datapath.
    __shared__ uint32_t s_wreach[LAZY ? CF_THREADS / 32 : 1];
    if (LAZY && lane == 0) s_wreach[warp] = 0;

    // composites the list set up in (lbase, total).  LAZY: inlined twice -- the tile's sorted prefix first, in the code
    // of the plain kernel (its survivor loop keeps the uniform datapath, which a single copy inside the stratum loop
    // below loses: 6 % on C2), then every stratum sorted here
    auto composite_list = [&]() {
    const uint32_t nbatches = (total + CF_BATCH - 1) / CF_BATCH;
    gather(0, load_id(0));
    uint32_t id_next = load_id(1);  // index for the batch after the one in flight: its latency hides behind a whole batch
    for (uint32_t b = 0; b < nbatches; b++) {
        // everybody is past batch b-1 (so its buffer may be overwritten); stop when every pixel of the tile is done
        if (__syncthreads_and(done)) break;
        gather(b + 1, id_next);
        id_next = load_id(b + 2);
        cp_async_wait<1>();  // this thread's part of batch b has landed ...
        __syncthreads();     // ... and so has everybody else's
        if (warp_done) continue;
        const uint32_t nb = min((uint32_t)CF_BATCH, total - b * CF_BATCH);
        const uint32_t pos0 = b * CF_BATCH + 1;  // 1-based list position of this batch's first entry
        const uint32_t rec_addr = stage_addr + (b & 1u) * (uint32_t)sizeof(CfStage);
        for (uint32_t chunk = 0; chunk < nb; chunk += 32) {
            const uint32_t j = chunk + lane;
            bool hit = false;
            if (j < nb) {
                // exact: does the alpha >= 1/255 ellipse reach this warp's 8x4 block?
                const uint32_t a = rec_addr + j * 48u;
                const float4 g0 = lds128(a);
                hit = gs_box_reaches(g0.x, g0.y, g0.z, g0.w, lds32(a + 16u), lds32(a + 40u), bx0, bx1, by0, by1);
            }
            uint32_t mask = __ballot_sync(0xffffffffu, hit);
            const uint32_t chunk_addr = rec_addr + chunk * 48u;
            while (mask) {
                const uint32_t bit = (uint32_t)__ffs(mask) - 1u;
                mask &= mask - 1u;
                const uint32_t a = chunk_addr + bit * 48u;
                const float4 q0 = lds128(a), q1 = lds128(a + 16u);
                const float dx = q0.x - pxf, dy = q0.y - pyf;
                const float p2 = gs_power2(q0.z, q0.w, q1.x, dx, dy);
                const float alpha = fminf(GS_ALPHA_MAX, q1.y * gs_ex2(p2));
                // one divergent region: everything above is evaluated by all lanes unconditionally
                if (!done && p2 <= 0.0f && alpha >= GS_ALPHA_MIN) {
                    const float test_T = T * (1.0f - alpha);
                    if (test_T < GS_T_MIN) {
                        done = true;
                    } else {
                        const float2 q2 = lds64(a + 32u);
                        const float w = alpha * T;
                        C0 = fmaf(q1.z, w, C0);
                        C1 = fmaf(q1.w, w, C1);
                        C2 = fmaf(q2.x, w, C2);
                        if (DEPTH) Dz = fmaf(DEPTH == 2 ? lds32(a + 44u) : q2.y, w, Dz);
                        T = test_T;
                        last = pos0 + chunk + bit;
                    }
                }
            }
            if (__all_sync(0xffffffffu, done)) {
                warp_done = true;
                if (LAZY && lane == 0) s_wreach[warp] = pos0 + chunk + 31u + (lbase - range.x);
                break;
            }
        }
    }
    cp_async_wait<0>();  // nothing of ours may still be in flight into shared memory when the CTA retires (or sorts)
    };
    composite_list();
    if (LAZY) {
        uint32_t sorted = total;
        for (;;) {
            const bool all_done = __syncthreads_and(done);
            const uint32_t more = all_done ? 0u
                                           : lazy_sort_next(lazy, vt, sorted, reinterpret_cast<uint64_t *>(&stage[0]),
                                                            const_cast<uint32_t *>(point_list) + range.x);
            if (more == 0) {
                if (tid == 0) {
                    uint32_t reach = 0;
                    for (int w = 0; w < CF_THREADS / 32; w++) reach = max(reach, s_wreach[w]);
                    lazy_record(lazy, vt, min(reach, sorted), all_done, ranges + vt, sorted);
                }
                break;
            }
            const uint32_t prev = last;  // positions in the stratum's list count from its first entry
            last = 0;
            lbase = range.x + sorted;
            total = more;
            composite_list();
            last = last ? last + sorted : prev;
            sorted += more;
        }
    }

    if (inside) {
        const size_t hw = (size_t)c.H * c.W;
        const size_t pix = (size_t)py * c.W + px;
        const float *bg = c.bg ? c.bg + (size_t)v * 3 : nullptr;
        float *out = color + (size_t)v * 3 * hw + pix;
        out[0] = C0 + T * (bg ? bg[0] : 0.f);
        out[hw] = C1 + T * (bg ? bg[1] : 0.f);
        out[2 * hw] = C2 + T * (bg ? bg[2] : 0.f);
        if (DEPTH) depth[(size_t)v * hw + pix] = Dz;
        final_T[(size_t)v * hw + pix] = T;
        if (ALPHA) alpha_out[(size_t)v * hw + pix] = 1.0f - T;
        n_contrib[(size_t)v * hw + pix] = last;
    }
}


// ---------------------------------------------------------------------------------------------------------
// Round-2 variant (GS_TUNE_FWD_WS): persistent, warp-specialised producer / consumers over an mbarrier ring
// ---------------------------------------------------------------------------------------------------------
// What v1's profile showed (ncu, C2): the biggest stall reason is the CTA barrier -- the
// eight warps of a tile have very different amounts of work per batch (0 to 60 survivors), and two __syncthreads per
// batch keep them in lock step -- and part of the elapsed time is the tail of the 2048-CTA grid (a few waves of CTAs
// of very different length).  v2:
//  * one PRODUCER warp per CTA streams the tile's list: it loads the indices, issues the 16-byte cp.async gathers of the
//    three record planes into a ring of CP_STAGES stages of CP_BATCH entries and lets the copies themselves arrive on
//    the stage's "full" mbarrier (cp.async.mbarrier.arrive.noinc) -- it never waits for data;
//  * eight CONSUMER warps (one 8x4 block each, culling and compositing exactly as in v1) wait on "full", work, and
//    arrive on the stage's "empty" mbarrier; a fast warp runs up to CP_STAGES - 1 stages ahead of a slow one and no
//    CTA-wide barrier is left inside a tile;
//  * consumers whose pixels are all saturated report it; once all eight have, the producer publishes the batch number
//    it stops at and completes that stage empty-handed, so everybody leaves the tile with the ring in a consistent state;
//  * the grid is PERSISTENT (SMs x resident CTAs), tiles are handed out by an atomic counter: no tail of short waves.
// Pixels, skip decisions and arithmetic order are those of v1: the images are bit-identical (tested).
// It removes the barrier stalls at the cost of a few more instructions, and runs in about the time of v1 (DESIGN.md 5.3).
// The barrier-synchronised kernel above stays the default (no faster alternative, simpler, and the sanitizer can check it).
constexpr int CP_CONSUMERS = 8;
constexpr int CP_THREADS = 32 * (CP_CONSUMERS + 1);
constexpr int CP_STAGES = 4;
constexpr int CP_BATCH = 128;

struct CpSmem {
    float4 rec[CP_STAGES][CP_BATCH][3];
    uint64_t full[CP_STAGES], empty[CP_STAGES];
    uint32_t tile;   // work item of the current round
    uint32_t done;   // consumer warps whose pixels are all saturated (this tile)
    uint32_t stop;   // batch number at which the producer stopped early (0xffffffff: it did not)
};

__device__ __forceinline__ uint32_t ld_volatile_shared(const uint32_t *p) {
    uint32_t v;
    asm volatile("ld.volatile.shared.u32 %0, [%1];" : "=r"(v) : "r"(smem_u32(p)));
    return v;
}

template <int DEPTH, int MINB, bool ALPHA = false>   // DEPTH, ALPHA as k_composite_fwd
__global__ void __launch_bounds__(CP_THREADS, MINB)
k_composite_fwd_ws(const DevCfg c, const float4 *__restrict__ rec0, const float4 *__restrict__ rec1,
                   const float4 *__restrict__ rec2, const uint32_t *__restrict__ point_list,
                   const uint2 *__restrict__ ranges, float *__restrict__ color, float *__restrict__ depth,
                   float *__restrict__ final_T, uint32_t *__restrict__ n_contrib, uint32_t *__restrict__ sched,
                const uint32_t total_tiles, float *__restrict__ alpha_out) {  // (lists sorted whole: no lazy strata)
    __shared__ __align__(16) CpSmem sm;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid == 0) {
#pragma unroll
        for (int s = 0; s < CP_STAGES; s++) {
            mbar_init(&sm.full[s], 32);            // the 32 producer lanes (through their copies)
            mbar_init(&sm.empty[s], CP_CONSUMERS);  // one arrival per consumer warp
        }
        mbar_fence_init();
    }
    uint32_t use = 0;  // stages used so far: the same sequence on both sides, continuing across tiles
    const uint32_t stage_addr = smem_u32(&sm.rec[0][0][0]);
    constexpr uint32_t STAGE_BYTES = (uint32_t)sizeof(float4) * CP_BATCH * 3;

    for (;;) {
        __syncthreads();  // the previous tile is finished everywhere (first round: the barriers are initialised)
        if (tid == 0) {
            sm.tile = atomicAdd(sched, 1u);
            sm.done = 0;
            sm.stop = 0xffffffffu;
        }
        __syncthreads();
        const uint32_t item = sm.tile;
        if (item >= total_tiles) break;
        const int v = (int)(item / (uint32_t)c.ntiles), tile = (int)(item - (uint32_t)v * (uint32_t)c.ntiles);
        const uint2 range = ranges[(size_t)v * c.ntiles + tile];
        const uint32_t total = range.y - range.x;
        const uint32_t nbatches = (total + CP_BATCH - 1) / CP_BATCH;
        const size_t rbase = (size_t)v * c.P;

        if (warp == CP_CONSUMERS) {
            // ================= producer =================
            constexpr int PER_LANE = CP_BATCH / 32;
            uint32_t ids[PER_LANE];
            auto load_ids = [&](uint32_t b) {
#pragma unroll
                for (int k = 0; k < PER_LANE; k++) {
                    const uint32_t e = b * CP_BATCH + k * 32 + lane;
                    ids[k] = e < total ? point_list[range.x + e] : 0xffffffffu;
                }
            };
            if (nbatches) load_ids(0);
            for (uint32_t b = 0; b < nbatches; b++) {
                const uint32_t s = use % CP_STAGES, ph = (use / CP_STAGES) & 1u;
                use++;
                mbar_wait(&sm.empty[s], ph ^ 1u);  // every consumer has released the stage's previous use
                if (ld_volatile_shared(&sm.done) == CP_CONSUMERS) {
                    // every pixel of the tile is saturated: complete this stage empty-handed and stop
                    if (lane == 0) sm.stop = b;
                    __syncwarp();
                    mbar_arrive(&sm.full[s]);   // release: the store above is visible to whoever sees the phase complete
                    break;
                }
#pragma unroll
                for (int k = 0; k < PER_LANE; k++) {
                    if (ids[k] != 0xffffffffu) {
                        const size_t r = rbase + ids[k];
                        float4 *dst = &sm.rec[s][k * 32 + lane][0];
                        cp_async16(dst, rec0 + r);
                        cp_async16(dst + 1, rec1 + r);
                        cp_async16(dst + 2, rec2 + r);
                    }
                }
                cp_async_mbar_arrive(&sm.full[s]);
                if (b + 1 < nbatches) load_ids(b + 1);  // its latency hides behind the consumers' work on the ring
            }
            continue;
        }

        // ================= consumers =================
        const int bx = (tile % c.gx) * GS_TILE + (warp & 1) * 8;   // this warp's 8x4 pixel block
        const int by = (tile / c.gx) * GS_TILE + (warp >> 1) * 4;
        const int px = bx + (lane & 7), py = by + (lane >> 3);
        const bool inside = px < c.W && py < c.H;
        const float pxf = (float)px, pyf = (float)py;
        const float bx0 = (float)bx, bx1 = (float)(bx + 7), by0 = (float)by, by1 = (float)(by + 3);
        float T = 1.0f, C0 = 0.f, C1 = 0.f, C2 = 0.f, Dz = 0.f;
        uint32_t last = 0;
        bool done = !inside;
        bool warp_done = false;
        for (uint32_t b = 0; b < nbatches; b++) {
            const uint32_t s = use % CP_STAGES, ph = (use / CP_STAGES) & 1u;
            use++;
            mbar_wait(&sm.full[s], ph);
            const bool stopped = ld_volatile_shared(&sm.stop) == b;
            if (!stopped && !warp_done) {
                const uint32_t nb = min((uint32_t)CP_BATCH, total - b * CP_BATCH);
                const uint32_t pos0 = b * CP_BATCH + 1;  // 1-based list position of this batch's first entry
                const uint32_t rec_addr = stage_addr + s * STAGE_BYTES;
                for (uint32_t chunk = 0; chunk < nb; chunk += 32) {
                    const uint32_t j = chunk + lane;
                    bool hit = false;
                    if (j < nb) {
                        // exact: does the alpha >= 1/255 ellipse reach this warp's 8x4 block?
                        const uint32_t a = rec_addr + j * 48u;
                        const float4 g0 = lds128(a);
                        hit = gs_box_reaches(g0.x, g0.y, g0.z, g0.w, lds32(a + 16u), lds32(a + 40u), bx0, bx1, by0, by1);
                    }
                    uint32_t mask = __ballot_sync(0xffffffffu, hit);
                    const uint32_t chunk_addr = rec_addr + chunk * 48u;
                    while (mask) {
                        const uint32_t bit = (uint32_t)__ffs(mask) - 1u;
                        mask &= mask - 1u;
                        const uint32_t a = chunk_addr + bit * 48u;
                        const float4 q0 = lds128(a), q1 = lds128(a + 16u);
                        const float dx = q0.x - pxf, dy = q0.y - pyf;
                        const float p2 = gs_power2(q0.z, q0.w, q1.x, dx, dy);
                        const float alpha = fminf(GS_ALPHA_MAX, q1.y * gs_ex2(p2));
                        // one divergent region: everything above is evaluated by all lanes unconditionally
                        if (!done && p2 <= 0.0f && alpha >= GS_ALPHA_MIN) {
                            const float test_T = T * (1.0f - alpha);
                            if (test_T < GS_T_MIN) {
                                done = true;
                            } else {
                                const float2 q2 = lds64(a + 32u);
                                const float w = alpha * T;
                                C0 = fmaf(q1.z, w, C0);
                                C1 = fmaf(q1.w, w, C1);
                                C2 = fmaf(q2.x, w, C2);
                                if (DEPTH) Dz = fmaf(DEPTH == 2 ? lds32(a + 44u) : q2.y, w, Dz);
                                T = test_T;
                                last = pos0 + chunk + bit;
                            }
                        }
                    }
                    if (__all_sync(0xffffffffu, done)) {
                        warp_done = true;
                        if (lane == 0) atomicAdd(&sm.done, 1u);
                        break;
                    }
                }
            }
            __syncwarp();                              // every lane has finished reading the stage
            if (lane == 0) mbar_arrive(&sm.empty[s]);  // (also for the stage the producer completed empty-handed)
            if (stopped) break;
        }
        if (inside) {
            const size_t hw = (size_t)c.H * c.W;
            const size_t pix = (size_t)py * c.W + px;
            const float *bg = c.bg ? c.bg + (size_t)v * 3 : nullptr;
            float *out = color + (size_t)v * 3 * hw + pix;
            out[0] = C0 + T * (bg ? bg[0] : 0.f);
            out[hw] = C1 + T * (bg ? bg[1] : 0.f);
            out[2 * hw] = C2 + T * (bg ? bg[2] : 0.f);
            if (DEPTH) depth[(size_t)v * hw + pix] = Dz;
            final_T[(size_t)v * hw + pix] = T;
            if (ALPHA) alpha_out[(size_t)v * hw + pix] = 1.0f - T;
            n_contrib[(size_t)v * hw + pix] = last;
        }
    }
}

}  // namespace

int launch_composite_fwd(const DevCfg &c, const GsSaved &s, float *color, float *depth, cudaStream_t st, int variant,
                         float *alpha, const LazyStrata &lazy) {
    if (c.V == 0 || c.ntiles == 0) return GS_OK;
    if (variant == 2) {
        if (lazy.cursor) return gs_set_error(GS_ERR_INVALID, "lazy strata with the warp-specialised compositor");
        // warp-specialised variant: persistent grid of SMs x resident CTAs; tiles handed out through s.sched
        constexpr int MINB_WS = 5;
        static int ctas_per_device[64] = {};   // per device: SM count x occupancy of the kernel
        int dev = 0;
        GS_CUDA_OK(cudaGetDevice(&dev));
        const int depth_kind = !(c.flags & GS_FLAG_DEPTH) ? 0 : (s.depth_mode == GS_DEPTH_Z ? 1 : 2);
        if (dev >= 0 && dev < 64 && ctas_per_device[dev] == 0) {
            int sms = 0, per_sm = 0;
            GS_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
            GS_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_composite_fwd_ws<0, MINB_WS>, CP_THREADS, 0));
            ctas_per_device[dev] = sms * (per_sm > 0 ? per_sm : 1);
        }
        const uint32_t total = (uint32_t)c.ntiles * (uint32_t)c.V;
        const uint32_t resident = (dev >= 0 && dev < 64) ? (uint32_t)ctas_per_device[dev] : 132u * MINB_WS;
        const uint32_t nctas = total < resident ? total : resident;
        GS_CUDA_OK(cudaMemsetAsync(s.sched, 0, 8, st));
        auto launch_ws = [&](auto kern) {
            kern<<<nctas, CP_THREADS, 0, st>>>(c, s.rec0, s.rec1, s.rec2, s.point_list, s.ranges, color, depth, s.final_T,
                                               s.n_contrib, s.sched, total, alpha);
        };
        if (alpha) {
            if (depth_kind == 2) launch_ws(k_composite_fwd_ws<2, MINB_WS, true>);
            else if (depth_kind == 1) launch_ws(k_composite_fwd_ws<1, MINB_WS, true>);
            else launch_ws(k_composite_fwd_ws<0, MINB_WS, true>);
        } else if (depth_kind == 2) launch_ws(k_composite_fwd_ws<2, MINB_WS>);
        else if (depth_kind == 1) launch_ws(k_composite_fwd_ws<1, MINB_WS>);
        else launch_ws(k_composite_fwd_ws<0, MINB_WS>);
        GS_CUDA_OK(cudaGetLastError());
        return GS_OK;
    }
    dim3 grid(c.ntiles, c.V);
    // 6 resident CTAs per SM (39 registers).  Bounding the registers to 32 for 8 CTAs/SM (28 B of spills) was slower on
    // C2 -- issue-bound, like the backward.
    constexpr int MINB = 6;
    auto launch = [&](auto kern) {
        kern<<<grid, CF_THREADS, 0, st>>>(c, s.rec0, s.rec1, s.rec2, s.point_list, s.ranges, color, depth, s.final_T, s.n_contrib,
                                          alpha, lazy);
    };
    auto by_depth = [&](auto alpha_tag, auto lazy_tag) {
        constexpr bool A = decltype(alpha_tag)::value, L = decltype(lazy_tag)::value;
        if (!(c.flags & GS_FLAG_DEPTH)) launch(k_composite_fwd<0, MINB, A, L>);
        else if (s.depth_mode == GS_DEPTH_Z) launch(k_composite_fwd<1, MINB, A, L>);
        else launch(k_composite_fwd<2, MINB, A, L>);
    };
    using T_ = std::true_type;
    using F_ = std::false_type;
    if (alpha) lazy.cursor ? by_depth(T_{}, T_{}) : by_depth(T_{}, F_{});
    else lazy.cursor ? by_depth(F_{}, T_{}) : by_depth(F_{}, F_{});
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}
