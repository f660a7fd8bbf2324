// gs_binning.cu -- stage 2 of the forward: per-tile lists of Gaussians in (depth, index) order.
//
// Semantics: SURVEY.md Appendix A "Binning" (upstream K2-K5): every (view, tile) list holds the Gaussians whose
// footprint touches the tile, ordered by fp32 depth bits, ties by Gaussian index.  Upstream gets that order from
// ONE device-wide radix sort of 64-bit (tile | depth) keys over all D tile instances: ~6 passes of 12-byte pairs.
//
// Design (DESIGN.md section 5.2), all views of the call at once.
//  FAST PATH (every tile list fits one CTA's shared memory, <= BIN_SMEM_CAP entries):
//    1. preprocess already counted the instances per (view, tile) with global reductions (RED.ADD).  Same-sector
//       atomics serialise in L2, so every tile has
//       BIN_SUB sub-counters, chosen by the Gaussian's index, each alone in its 32-byte sector;
//    2. k_tile_scan: one CTA turns the counters into sub-bucket offsets, the total D and the longest list;
//    3. k_emit_buckets: every Gaussian appends (depth_bits << 32 | index) to its sub-bucket of each tile it
//       touches (atomic cursor per sub-bucket; the arrival order is arbitrary).  A tile's sub-buckets are
//       contiguous, so together they are the tile's bucket;
//    4. k_tile_sort: one CTA per (view, tile) loads its bucket into registers/shared memory, merge-sorts the
//       64-bit keys -- a total order, so the arbitrary arrival order does not matter -- and writes the index list
//       and the tile's [start, end) range.
//    HBM traffic: 8 B written + 8 B read + 4 B written per instance, one pass each (vs ~6 x 24 B upstream).
//  FALLBACK (some list longer than BIN_SMEM_CAP, or forced through GsConfig.tuning): two-level device-wide radix
//    sort -- Gaussians by depth (64-bit keys, bits [32,64)), instances emitted in that order and sorted stably
//    by (view, tile) only.
// The block-level merge sort, the device scan and the device radix sorts are CUB primitives (library code, like
// cuBLAS for a plain GEMM); the count / scan / emit / range kernels are ours.
#include <cub/cub.cuh>
#include <thrust/iterator/transform_iterator.h>

#include "gs_common.cuh"
#include "gs_tile_sort.cuh"

namespace {

inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

// ---------------------------------------------------------------------------------------------------------
// fast path
// ---------------------------------------------------------------------------------------------------------
constexpr int SCAN_THREADS = 1024;

// counters[nvt * BIN_SUB] (padded: one per 32-byte sector) -> exclusive sub-bucket offsets[nvt * BIN_SUB],
// per-tile totals tile_n[nvt], tile starts tile_start[nvt]; info[0] = total, info[1] = longest tile list,
// info[2] = largest sub-counter
__global__ void __launch_bounds__(SCAN_THREADS)
k_tile_scan(int nvt, const uint32_t *__restrict__ counters, uint32_t *__restrict__ offsets,
            uint32_t *__restrict__ tile_start, uint32_t *__restrict__ tile_n, uint32_t *__restrict__ info) {
    using BlockScan = cub::BlockScan<uint32_t, SCAN_THREADS>;
    using BlockReduce = cub::BlockReduce<uint32_t, SCAN_THREADS>;
    __shared__ union {
        typename BlockScan::TempStorage scan;
        typename BlockReduce::TempStorage reduce;
    } tmp;
    const int per = (nvt + SCAN_THREADS - 1) / SCAN_THREADS;  // tiles per thread
    const int b = threadIdx.x * per, e = min(nvt, b + per);
    uint32_t sum = 0, mx = 0, mxs = 0;
    unsigned long long sum64 = 0;  // the offsets are 32-bit; the TOTAL is also taken in 64 bits so that a wrap is seen
    for (int t = b; t < e; t++) {
        uint32_t tn = 0;
#pragma unroll
        for (int k = 0; k < BIN_SUB; k++) {
            const uint32_t cnt = counters[((size_t)t * BIN_SUB + k) * BIN_PAD];
            tn += cnt;
            mxs = max(mxs, cnt);
        }
        sum += tn;
        sum64 += tn;
        mx = max(mx, tn);
    }
    uint32_t excl, total;
    BlockScan(tmp.scan).ExclusiveSum(sum, excl, total);
    __syncthreads();
    {
        using Reduce64 = cub::BlockReduce<unsigned long long, SCAN_THREADS>;
        __shared__ typename Reduce64::TempStorage tmp64;
        const unsigned long long total64 = Reduce64(tmp64).Sum(sum64);
        if (threadIdx.x == 0 && total64 > 0xffffffffull) total = 0xffffffffu;  // saturate: the host rejects D > 2^31-1
    }
    const uint32_t bmax = BlockReduce(tmp.reduce).Reduce(mx, cub::Max());
    __syncthreads();
    const uint32_t bmaxs = BlockReduce(tmp.reduce).Reduce(mxs, cub::Max());
    for (int t = b; t < e; t++) {
        tile_start[t] = excl;
        uint32_t tn = 0;
#pragma unroll
        for (int k = 0; k < BIN_SUB; k++) {
            offsets[(size_t)t * BIN_SUB + k] = excl + tn;
            tn += counters[((size_t)t * BIN_SUB + k) * BIN_PAD];
        }
        tile_n[t] = tn;
        excl += tn;
    }
    if (threadIdx.x == 0) {
        info[0] = total;
        info[1] = bmax;
        info[2] = bmaxs;
    }
}

// GATED (sync-free path): nothing is emitted when status[SF_VERDICT] is set, and every exact-capacity store index is
// checked against `capacity` before the store.
template <bool GATED = false>
__global__ void k_emit_buckets(const DevCfg c, const float4 *__restrict__ rec0, const float4 *__restrict__ rec1,
                               const float4 *__restrict__ rec2, const ushort4 *__restrict__ rects,
                               const uint32_t *__restrict__ offsets, const uint32_t sub_cap,
                               const float *__restrict__ strata, const int strata_per_tile,
                               uint32_t *__restrict__ cursor, uint64_t *__restrict__ bucket,
                               const uint32_t *__restrict__ status = nullptr, uint32_t capacity = 0) {
    const size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= (size_t)c.V * c.P) return;
    if (GATED && status[SF_VERDICT]) return;
    const ushort4 r = rects[g];
    if (r.z <= r.x || r.w <= r.y) return;
    const uint32_t v = (uint32_t)(g / c.P);
    const uint32_t i = (uint32_t)(g - (size_t)v * c.P);
    const float4 q0 = rec0[g], q1 = rec1[g], q2 = rec2[g];
    const uint64_t key = ((uint64_t)__float_as_uint(q2.y) << 32) | i;
    const uint32_t tbase = v * (uint32_t)c.ntiles;
    uint32_t sub = i & (BIN_SUB - 1);
    if (strata && !strata_per_tile) {  // sub-bucket = depth stratum of this view (same rule as k_preprocess)
        sub = 0;
#pragma unroll
        for (int q = 0; q < BIN_SUB - 1; q++) sub += q2.y >= strata[(size_t)v * BIN_SUB + q] ? 1u : 0u;
    }
    // The cursor atomics return values and the stores depend on them: handle the candidate tiles four at a time so
    // that several round trips to L2 are in flight per thread (the kernel is latency-bound).
    constexpr int BATCH = 4;
    const int w = r.z - r.x, nt = w * (r.w - r.y);
    int cx = r.x, cy = r.y;  // row-major walk of the rectangle (no integer division per candidate)
    for (int t0 = 0; t0 < nt; t0 += BATCH) {
        size_t slot[BATCH];
        uint32_t pos[BATCH];
        bool ok[BATCH];
#pragma unroll
        for (int k = 0; k < BATCH; k++) {
            ok[k] = cy < (int)r.w && gs_tile_reached(q0, q1, q2, cx, cy);  // same predicate as the count in k_preprocess
            const uint32_t tile = tbase + (uint32_t)(cy * c.gx + cx);
            const uint32_t subk = (strata_per_tile && ok[k]) ? gs_tile_stratum(strata, tile, q2.y) : sub;
            slot[k] = (size_t)tile * BIN_SUB + subk;
            if (++cx == (int)r.z) {
                cx = r.x;
                cy++;
            }
        }
#pragma unroll
        for (int k = 0; k < BATCH; k++)
            if (ok[k]) pos[k] = atomicAdd(&cursor[slot[k] * BIN_PAD], 1u);
#pragma unroll
        for (int k = 0; k < BATCH; k++) {
            if (!ok[k]) continue;
            if (GATED) {
                const size_t at = (size_t)offsets[slot[k]] + pos[k];
                if (at < capacity) bucket[at] = key;
            } else if (offsets) bucket[(size_t)offsets[slot[k]] + pos[k]] = key;              // exact-capacity buckets
            else if (pos[k] < sub_cap) bucket[slot[k] * (size_t)sub_cap + pos[k]] = key;     // fixed-capacity buckets
        }
    }
}

template <int THREADS, int MAX_ITEMS>
__global__ void __launch_bounds__(THREADS)
k_tile_sort(const uint32_t *__restrict__ tile_n, const uint32_t *__restrict__ tile_start,
            const uint64_t *__restrict__ bucket, uint32_t *__restrict__ point_list, uint2 *__restrict__ ranges) {
    extern __shared__ __align__(16) unsigned char ts_smem[];
    const uint32_t vt = blockIdx.x;
    const uint32_t n = tile_n[vt], off = tile_start[vt];
    if (threadIdx.x == 0) ranges[vt] = make_uint2(off, off + n);
    if (n == 0) return;
    const uint64_t *src = bucket + off;
    sort_bucket_dispatch<THREADS, MAX_ITEMS>([src](uint32_t i) { return src[i]; }, point_list + off, n, ts_smem);
}

template <int THREADS, int MAX_ITEMS>
int launch_tile_sort(int nvt, const uint32_t *counts, const uint32_t *offsets, const uint64_t *bucket,
                     uint32_t *point_list, uint2 *ranges, cudaStream_t st) {
    const size_t smem = tile_sort_smem_bytes<THREADS, MAX_ITEMS>();
    GS_CUDA_OK(cudaFuncSetAttribute(k_tile_sort<THREADS, MAX_ITEMS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_tile_sort<THREADS, MAX_ITEMS><<<nvt, THREADS, smem, st>>>(counts, offsets, bucket, point_list, ranges);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}

// Capacity ladder of the per-tile sort: the smallest (threads x keys-per-thread) configuration that holds the
// longest list of the call.  More threads with fewer keys each shorten the serial part of every merge round.
template <int THREADS>
int dispatch_tile_sort(uint32_t max_count, int nvt, const uint32_t *tile_n, const uint32_t *tile_start,
                       const uint64_t *bucket, uint32_t *point_list, uint2 *ranges, cudaStream_t st) {
    constexpr int CAP_ITEMS = BIN_SMEM_CAP / THREADS;
    if (max_count <= THREADS * (CAP_ITEMS / 8)) return launch_tile_sort<THREADS, CAP_ITEMS / 8>(nvt, tile_n, tile_start, bucket, point_list, ranges, st);
    if (max_count <= THREADS * (CAP_ITEMS / 4)) return launch_tile_sort<THREADS, CAP_ITEMS / 4>(nvt, tile_n, tile_start, bucket, point_list, ranges, st);
    if (max_count <= THREADS * (CAP_ITEMS / 2)) return launch_tile_sort<THREADS, CAP_ITEMS / 2>(nvt, tile_n, tile_start, bucket, point_list, ranges, st);
    return launch_tile_sort<THREADS, CAP_ITEMS>(nvt, tile_n, tile_start, bucket, point_list, ranges, st);
}

// ---------------------------------------------------------------------------------------------------------
// speculative-capacity path: preprocess has already appended the keys to fixed-capacity sub-buckets
// (bucket[(vt * BIN_SUB + sub) * sub_cap + pos]); the cursors hold the counts.  k_spec_check turns the cursors
// into the verdict (info: [0] total instances, [1] longest tile list, [2] largest sub-counter, [3] overflow flag);
// k_tile_sort_spec gathers a tile's sub-buckets, sorts, and writes list + range.
// ---------------------------------------------------------------------------------------------------------
// One CTA: the verdict on a speculative forward, from the cursors alone (runs right after preprocess so that the
// host can read it while the tile sort and the compositor are already enqueued behind it).
__global__ void __launch_bounds__(SCAN_THREADS)
k_spec_check(int nvt, uint32_t sub_cap, uint32_t tile_limit, const uint32_t *__restrict__ cursor,
             uint32_t *__restrict__ info) {
    using BlockReduce = cub::BlockReduce<uint32_t, SCAN_THREADS>;
    __shared__ typename BlockReduce::TempStorage tmp;
    uint32_t sum = 0, mx = 0, mxs = 0, over = 0;
    for (int t = threadIdx.x; t < nvt; t += SCAN_THREADS) {
        uint32_t tn = 0;
#pragma unroll
        for (int k = 0; k < BIN_SUB; k++) {
            const uint32_t cnt = cursor[((size_t)t * BIN_SUB + k) * BIN_PAD];
            mxs = max(mxs, cnt);
            over |= cnt > sub_cap ? 1u : 0u;
            tn += cnt;
        }
        over |= tn > tile_limit ? 1u : 0u;
        over |= sum + tn < sum ? 1u : 0u;  // a 32-bit wrap of the running total counts as an overflow (redone exactly)
        sum += tn;
        mx = max(mx, tn);
    }
    const uint32_t total = BlockReduce(tmp).Sum(sum);
    __syncthreads();
    using Reduce64 = cub::BlockReduce<unsigned long long, SCAN_THREADS>;
    __shared__ typename Reduce64::TempStorage tmp64;
    if (Reduce64(tmp64).Sum((unsigned long long)sum) > 0xffffffffull) over |= 1u;  // (thread 0 holds the block sum)
    __syncthreads();
    const uint32_t bmax = BlockReduce(tmp).Reduce(mx, cub::Max());
    __syncthreads();
    const uint32_t bmaxs = BlockReduce(tmp).Reduce(mxs, cub::Max());
    __syncthreads();
    const uint32_t bover = BlockReduce(tmp).Reduce(over, cub::Max());
    if (threadIdx.x == 0) {
        info[0] = total;
        info[1] = bmax;
        info[2] = bmaxs;
        info[3] = bover;
    }
}

template <int THREADS, int MAX_ITEMS>
__global__ void __launch_bounds__(THREADS)
k_tile_sort_spec(uint32_t sub_cap, const uint32_t *__restrict__ cursor, const uint64_t *__restrict__ bucket,
                 uint32_t *__restrict__ point_list, uint2 *__restrict__ ranges) {
    extern __shared__ __align__(16) unsigned char ts_smem[];
    __shared__ uint32_t s_start[BIN_SUB + 1];
    const uint32_t vt = blockIdx.x;
    if (threadIdx.x == 0) {
        uint32_t n = 0;
        for (int k = 0; k < BIN_SUB; k++) {
            s_start[k] = n;
            n += min(cursor[((size_t)vt * BIN_SUB + k) * BIN_PAD], sub_cap);  // clamped: an overflowed call is redone
        }
        n = min(n, (uint32_t)(THREADS * MAX_ITEMS));
        s_start[BIN_SUB] = n;
        const uint32_t off = vt * BIN_SUB * sub_cap;
        ranges[vt] = make_uint2(off, off + n);
    }
    __syncthreads();
    const uint32_t n = s_start[BIN_SUB];
    if (n == 0) return;
    uint32_t st[BIN_SUB + 1];
#pragma unroll
    for (int k = 0; k <= BIN_SUB; k++) st[k] = s_start[k];
    const uint64_t *base = bucket + (size_t)vt * BIN_SUB * sub_cap;
    auto load = [&](uint32_t i) {
        uint32_t k = 0, first = 0;  // sub-bucket holding logical entry i and that sub-bucket's first logical entry
#pragma unroll
        for (int j = 1; j < BIN_SUB; j++)
            if (i >= st[j]) {
                k = (uint32_t)j;
                first = st[j];
            }
        return base[(size_t)k * sub_cap + (i - first)];
    };
    sort_bucket_dispatch<THREADS, MAX_ITEMS>(load, point_list + (size_t)vt * BIN_SUB * sub_cap, n, ts_smem);
}

template <int THREADS, int MAX_ITEMS>
int launch_tile_sort_spec(int nvt, uint32_t sub_cap, const uint32_t *cursor, const uint64_t *bucket, uint32_t *point_list,
                          uint2 *ranges, cudaStream_t st) {
    const size_t smem = tile_sort_smem_bytes<THREADS, MAX_ITEMS>();
    GS_CUDA_OK(cudaFuncSetAttribute(k_tile_sort_spec<THREADS, MAX_ITEMS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_tile_sort_spec<THREADS, MAX_ITEMS><<<nvt, THREADS, smem, st>>>(sub_cap, cursor, bucket, point_list, ranges);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}

// ---------------------------------------------------------------------------------------------------------
// fallback path (device-wide radix sorts)
// ---------------------------------------------------------------------------------------------------------
// number of tiles of the candidate rectangle the Gaussian really reaches (the predicate of the fast path)
__device__ __forceinline__ uint32_t reached_tiles(ushort4 r, float4 q0, float4 q1, float4 q2) {
    uint32_t n = 0;
    for (int y = r.y; y < r.w; y++)
        for (int x = r.x; x < r.z; x++) n += gs_tile_reached(q0, q1, q2, x, y) ? 1u : 0u;
    return n;
}

__global__ void k_depth_keys(size_t n, const float4 *__restrict__ rec0, const float4 *__restrict__ rec1,
                             const float4 *__restrict__ rec2, const ushort4 *__restrict__ rects,
                             uint64_t *__restrict__ keys, uint32_t *__restrict__ cnt) {
    const size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= n) return;
    const ushort4 r = rects[g];
    uint32_t nt = 0, d = 0xffffffffu;  // Gaussians without tiles sort to the end (their records were never written)
    if (r.z > r.x && r.w > r.y) {
        const float4 q2 = rec2[g];
        nt = reached_tiles(r, rec0[g], rec1[g], q2);
        if (nt) d = __float_as_uint(q2.y);
    }
    cnt[g] = nt;
    keys[g] = ((uint64_t)d << 32) | (uint64_t)g;
}

struct TilesInOrder {  // tile count gathered through the depth order (input functor of the scan)
    const uint32_t *cnt;
    __host__ __device__ __forceinline__ uint32_t operator()(const uint64_t &key) const { return cnt[(uint32_t)key]; }
};

__global__ void k_emit_ordered(const DevCfg c, const uint64_t *__restrict__ order, const float4 *__restrict__ rec0,
                               const float4 *__restrict__ rec1, const float4 *__restrict__ rec2,
                               const ushort4 *__restrict__ rects, const uint32_t *__restrict__ cnt,
                               const uint32_t *__restrict__ offsets, uint32_t *__restrict__ keys,
                               uint32_t *__restrict__ vals) {
    const size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= (size_t)c.V * c.P) return;
    const uint32_t g = (uint32_t)order[j];
    if (cnt[g] == 0) return;
    const ushort4 r = rects[g];
    const float4 q0 = rec0[g], q1 = rec1[g], q2 = rec2[g];
    uint32_t off = j == 0 ? 0u : offsets[j - 1];
    const uint32_t v = g / (uint32_t)c.P;
    const uint32_t i = g - v * (uint32_t)c.P;
    const uint32_t tbase = v * (uint32_t)c.ntiles;
    for (int y = r.y; y < r.w; y++)
        for (int x = r.x; x < r.z; x++) {
            if (!gs_tile_reached(q0, q1, q2, x, y)) continue;
            keys[off] = tbase + (uint32_t)(y * c.gx + x);
            vals[off] = i;
            off++;
        }
}

__global__ void k_ranges(int64_t D, const uint32_t *__restrict__ keys, uint2 *__restrict__ ranges) {
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= D) return;
    const uint32_t t = keys[idx];
    if (idx == 0 || t != keys[idx - 1]) ranges[t].x = (uint32_t)idx;
    if (idx == D - 1 || t != keys[idx + 1]) ranges[t].y = (uint32_t)(idx + 1);
}

int tile_bits(const DevCfg &c) {
    int tb = 1;
    while ((1ll << tb) < (long long)c.V * c.ntiles) tb++;
    return tb;
}

size_t cub_temp_bytes(const DevCfg &c, int64_t n, int64_t D) {
    size_t t1 = 0, t2 = 0, t3 = 0;
    cub::DeviceRadixSort::SortKeys(nullptr, t1, (const uint64_t *)nullptr, (uint64_t *)nullptr, (int)n, 32, 64);
    auto it = thrust::make_transform_iterator((const uint64_t *)nullptr, TilesInOrder{nullptr});
    cub::DeviceScan::InclusiveSum(nullptr, t2, it, (uint32_t *)nullptr, (int)n);
    cub::DeviceRadixSort::SortPairs(nullptr, t3, (const uint32_t *)nullptr, (uint32_t *)nullptr,
                                    (const uint32_t *)nullptr, (uint32_t *)nullptr, (int)D, 0, tile_bits(c));
    size_t t = t1 > t2 ? t1 : t2;
    return align256(t > t3 ? t : t3);
}

}  // namespace

size_t bin_counter_bytes(const DevCfg &c) { return (size_t)c.V * c.ntiles * BIN_SUB * BIN_PAD * sizeof(uint32_t); }

int bin_tile_scan(const DevCfg &c, const uint32_t *counters, uint32_t *offsets, uint32_t *tile_start, uint32_t *tile_n,
                  uint32_t *info, cudaStream_t st) {
    k_tile_scan<<<1, SCAN_THREADS, 0, st>>>(c.V * c.ntiles, counters, offsets, tile_start, tile_n, info);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}

bool bin_fits_fast_path(uint32_t max_count) { return max_count <= (uint32_t)BIN_SMEM_CAP; }

size_t bin_scratch_bytes(const DevCfg &c, int64_t D, bool fast) {
    const size_t n = (size_t)c.V * c.P;
    if (fast) return align256((size_t)(D > 0 ? D : 1) * 8);
    // depth_keys[n] | order[n] | cnt[n] | offsets[n] | keys_in[D] | keys_out[D] | vals_in[D] | cub temp
    return 2 * align256(n * 8) + 2 * align256(n * 4) + 3 * align256((size_t)D * 4) + cub_temp_bytes(c, (int64_t)n, D);
}

int bin_emit_fast(const DevCfg &c, int64_t D, const float4 *rec0, const float4 *rec1, const float4 *rec2,
                  const ushort4 *rects, const uint32_t *offsets, uint32_t sub_cap, const float *strata, int strata_per_tile,
                  uint32_t *cursor, void *scratch, cudaStream_t st) {
    if (D <= 0) return GS_OK;
    GS_CUDA_OK(cudaMemsetAsync(cursor, 0, bin_counter_bytes(c), st));
    const size_t n = (size_t)c.V * c.P;
    k_emit_buckets<false><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(c, rec0, rec1, rec2, rects, offsets, sub_cap, strata,
                                                                 strata_per_tile, cursor, static_cast<uint64_t *>(scratch));
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}

int bin_sort_fast(const DevCfg &c, uint32_t max_count, const uint32_t *tile_start, const uint32_t *tile_n,
                  const void *scratch, uint32_t *point_list, uint2 *ranges, cudaStream_t st) {
    const int nvt = c.V * c.ntiles;
    const uint64_t *bucket = static_cast<const uint64_t *>(scratch);
    // The merge sort is latency-bound: every round is a binary search plus a serial merge of ITEMS keys per thread.
    // Fewer keys per thread (more threads per tile) shorten the serial part, so long lists get 1024 threads.
    if (max_count > 2048) return dispatch_tile_sort<1024>(max_count, nvt, tile_n, tile_start, bucket, point_list, ranges, st);
    if (max_count > 1024) return dispatch_tile_sort<512>(max_count, nvt, tile_n, tile_start, bucket, point_list, ranges, st);
    return dispatch_tile_sort<256>(max_count, nvt, tile_n, tile_start, bucket, point_list, ranges, st);
}

// The launch configuration that sorts lists of up to tile_limit entries (lists longer than that make k_spec_check
// raise the overflow flag, so the clamp inside the kernel never decides a result that is kept).
static uint32_t spec_sort_capacity(uint32_t tile_limit) {
    return tile_limit <= 1024 ? 1024u : tile_limit <= 2048 ? 2048u : tile_limit <= 4096 ? 4096u : 8192u;
}

int bin_spec_check(const DevCfg &c, uint32_t sub_cap, uint32_t tile_limit, const uint32_t *cursor, uint32_t *info,
                   cudaStream_t st) {
    const uint32_t cap = spec_sort_capacity(tile_limit);
    k_spec_check<<<1, SCAN_THREADS, 0, st>>>(c.V * c.ntiles, sub_cap, cap, cursor, info);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}

// ---------------------------------------------------------------------------------------------------------
// Depth strata.  With sub-bucket = index % BIN_SUB a tile's list has to be sorted as a whole: one 1024-thread CTA,
// ten merge rounds of CTA-wide barriers.  If instead the sub-bucket is chosen by DEPTH -- stratum q
// holds the depths in [b_q, b_q+1) -- the tile's sorted list is the concatenation of its sorted sub-buckets, and each
// is sorted on its own by a 128-thread CTA (seven rounds, four-warp barriers, eight times as many independent CTAs to
// interleave), which is faster.  The boundaries are per-view octiles of the depths of the previous exact-path call
// (k_depth_hist / k_strata_from_hist); how well they balance only affects speed and capacity, never the result.
// (16 strata instead of 8 were no faster, and made the verdict kernel and preprocess slower.)
// ---------------------------------------------------------------------------------------------------------
constexpr int STRATA_BINS = 2048;                       // 64 bins per octave of depth from 0.125 up
constexpr uint32_t STRATA_BASE = 0x3E000000u >> 17;     // bit pattern of 0.125f, in bin units

__device__ __forceinline__ int depth_bin(float d) {
    const int b = (int)(__float_as_uint(d) >> 17) - (int)STRATA_BASE;  // monotone in d for positive floats
    return min(max(b, 0), STRATA_BINS - 1);
}

// hist[v][bin] += number of candidate tiles of every binned Gaussian of view v (rect area: a proxy of its instances)
__global__ void __launch_bounds__(256)
k_depth_hist(const DevCfg c, const ushort4 *__restrict__ rects, const float4 *__restrict__ rec2, uint32_t *__restrict__ hist) {
    __shared__ uint32_t h[STRATA_BINS];
    const int v = blockIdx.y;
    for (int k = threadIdx.x; k < STRATA_BINS; k += blockDim.x) h[k] = 0u;
    __syncthreads();
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < c.P; i += gridDim.x * blockDim.x) {
        const size_t o = (size_t)v * c.P + i;
        const ushort4 r = rects[o];
        const uint32_t area = (uint32_t)(r.z - r.x) * (uint32_t)(r.w - r.y);
        if (area) atomicAdd(&h[depth_bin(rec2[o].y)], area);
    }
    __syncthreads();
    for (int k = threadIdx.x; k < STRATA_BINS; k += blockDim.x)
        if (h[k]) atomicAdd(&hist[(size_t)v * STRATA_BINS + k], h[k]);
}

// strata[v][q] = lower edge of the first bin above the (q+1)/BIN_SUB quantile, q < BIN_SUB - 1; last entry +inf.
__global__ void __launch_bounds__(1024)
k_strata_from_hist(const uint32_t *__restrict__ hist, float *__restrict__ strata) {
    using Scan = cub::BlockScan<uint32_t, 1024>;
    __shared__ typename Scan::TempStorage tmp;
    const int v = blockIdx.x, t = threadIdx.x;
    static_assert(STRATA_BINS == 2048, "two bins per thread");
    const uint32_t a = hist[(size_t)v * STRATA_BINS + 2 * t], b = hist[(size_t)v * STRATA_BINS + 2 * t + 1];
    uint32_t excl, total;
    Scan(tmp).ExclusiveSum(a + b, excl, total);
    if (t < BIN_SUB) strata[(size_t)v * BIN_SUB + t] = __int_as_float(0x7f800000);  // +inf: nothing reaches that stratum
    __syncthreads();
    if (total == 0) return;
    const uint32_t cum[3] = {excl, excl + a, excl + a + b};  // mass below bin 2t, below bin 2t+1, below bin 2t+2
#pragma unroll
    for (int q = 1; q < BIN_SUB; q++) {
        const uint64_t target = ((uint64_t)total * q + BIN_SUB - 1) / BIN_SUB;  // mass that should lie below boundary q
#pragma unroll
        for (int k = 0; k < 2; k++)
            if (cum[k] < target && cum[k + 1] >= target)  // bin 2t+k completes the quantile: the boundary is its upper edge
                strata[(size_t)v * BIN_SUB + q - 1] = __uint_as_float((uint32_t)(2 * t + k + 1 + STRATA_BASE) << 17);
    }
}

// One sub-bucket (= depth stratum) of one tile per CTA; it lands behind the tile's earlier strata.  CTA (vt, 0)
// also writes the tile's range and adds the tile to the call's verdict (what k_spec_check computes for the whole-tile
// path): acc = [0] total instances, [1] longest tile list, [2] largest sub-counter, [3] overflow flag, [4] tiles
// accounted for; the last tile to arrive publishes [0..3] to `info` (mapped pinned memory the host is waiting on).
template <int THREADS, int MAX_ITEMS>
__global__ void __launch_bounds__(THREADS)
k_stratum_sort(uint32_t nvt, uint32_t sub_cap, const uint32_t *__restrict__ cursor, const uint64_t *__restrict__ bucket,
               uint32_t *__restrict__ point_list, uint2 *__restrict__ ranges, uint32_t *__restrict__ acc,
               uint32_t *__restrict__ info) {
    extern __shared__ __align__(16) unsigned char ts_smem[];
    const uint32_t vt = blockIdx.x / BIN_SUB, k = blockIdx.x % BIN_SUB;
    uint32_t off = 0, n = 0, total = 0, raw_total = 0, raw_max = 0;
#pragma unroll
    for (int j = 0; j < BIN_SUB; j++) {
        const uint32_t raw = cursor[((size_t)vt * BIN_SUB + j) * BIN_PAD];
        const uint32_t cnt = min(raw, sub_cap);  // clamped: an overflowed call is redone
        if (j < (int)k) off += cnt;
        if (j == (int)k) n = cnt;
        total += cnt;
        raw_total += raw;
        raw_max = max(raw_max, raw);
    }
    const uint32_t base = vt * BIN_SUB * sub_cap;
    if (k == 0 && threadIdx.x == 0) {
        ranges[vt] = make_uint2(base, base + total);
        if (atomicAdd(&acc[0], raw_total) + raw_total < raw_total) atomicOr(&acc[3], 1u);  // 32-bit wrap: redo exactly
        atomicMax(&acc[1], raw_total);
        atomicMax(&acc[2], raw_max);
        if (raw_max > sub_cap) atomicOr(&acc[3], 1u);
        __threadfence();
        if (atomicAdd(&acc[4], 1u) == nvt - 1) {  // every tile has been accounted for
            __threadfence();
            info[0] = atomicAdd(&acc[0], 0u);
            info[1] = atomicAdd(&acc[1], 0u);
            info[2] = atomicAdd(&acc[2], 0u);
            info[3] = atomicAdd(&acc[3], 0u);  // the host reads them after an event recorded behind this kernel
        }
    }
    if (n == 0) return;
    n = min(n, (uint32_t)(THREADS * MAX_ITEMS));
    const uint64_t *src = bucket + ((size_t)vt * BIN_SUB + k) * sub_cap;
    auto load = [src](uint32_t i) { return src[i]; };
    uint32_t *dst = point_list + base + off;
    // cheapest instantiation that holds the stratum (the kernel itself is instantiated for the call's capacity)
    if (MAX_ITEMS > 8 && n > THREADS * 8) sort_bucket_merge<THREADS, (MAX_ITEMS > 8 ? 16 : 1)>(load, dst, n, ts_smem);
    else if (MAX_ITEMS > 4 && n > THREADS * 4) sort_bucket_merge<THREADS, (MAX_ITEMS > 4 ? 8 : 1)>(load, dst, n, ts_smem);
    else if (n > THREADS * 2) sort_bucket_merge<THREADS, 4>(load, dst, n, ts_smem);
    else if (n > THREADS) sort_bucket_merge<THREADS, 2>(load, dst, n, ts_smem);
    else sort_bucket_merge<THREADS, 1>(load, dst, n, ts_smem);
}

// ---------------------------------------------------------------------------------------------------------
// Hand-written stratum sort (round 2): ONE WARP per stratum, no CTA barrier, no library primitive.
// cub::BlockMergeSort spends seven merge rounds of binary searches, two CTA barriers each, on a stratum of a few
// hundred keys.  A stratum is small and its depths are spread over a narrow, roughly
// uniform range, so one distribution pass nearly sorts it:
//   1. warp min / max of the depth bits (REDUX);
//   2. 64 depth buckets, bucket = floor((bits - min) * 64 / (range + 1)) -- monotone in the key, so sorted buckets
//      concatenate to the sorted stratum.  Counting is ATOMIC-FREE: six ballots of the bucket number's bits give every
//      lane L the masks of the round's keys that fall into buckets L and L + 32 (whose counts it keeps in registers);
//   3. a warp scan turns counts into bucket offsets; a second sweep of the same ballots scatters the keys to their
//      bucket in shared memory (position = bucket cursor + rank among the round's equal-bucket lanes);
//   4. every key is RANKED inside its bucket (~6 keys: one pass over the bucket's members per key, lanes = keys, so the
//      work is balanced whatever the bucket sizes) on the full 64-bit (depth, index) key -- index ties included -- and
//      its index is stored straight to its final position.
// Depth ties en masse (all depths of the stratum equal) switch the buckets to the index bits; any other crowding only
// lengthens step 4 (quadratic in the bucket, always correct).  A first version (32 buckets, per-lane insertion sort)
// was held back by the slowest lane's bucket set.
// ---------------------------------------------------------------------------------------------------------
constexpr int RS_WARPS = 4;          // strata per CTA (independent warps)

__global__ void __launch_bounds__(RS_WARPS * 32)
k_stratum_rank_sort(uint32_t nvt, uint32_t sub_cap, uint32_t cap_pad, const uint32_t *__restrict__ cursor,
                    const uint64_t *__restrict__ bucket, uint32_t *__restrict__ point_list, uint2 *__restrict__ ranges,
                    uint32_t *__restrict__ acc, uint32_t *__restrict__ info, const float4 *__restrict__ rec2, uint32_t P,
                    uint32_t ntiles, float *__restrict__ next, const uint8_t *__restrict__ need) {
    extern __shared__ __align__(16) unsigned char rs_smem[];
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t sidx = blockIdx.x * RS_WARPS + warp;   // (view, tile, stratum)
    if (sidx >= nvt * BIN_SUB) return;
    const uint32_t vt = sidx / BIN_SUB, k = sidx % BIN_SUB;
    // lazy strata: the strata the tile's previous forward read; the compositor sorts the rest if it gets there (a margin
    // of one more stratum, for a moving cloud, was slower on C2 and on the moving cloud alike: DESIGN.md 5.2).  Stratum 0
    // is always sorted: its warp also accounts for the tile in the verdict.
    const uint32_t sorted = need ? min(max((uint32_t)need[vt], 1u), (uint32_t)BIN_SUB) : (uint32_t)BIN_SUB;
    if (k >= sorted) return;
    // the tile's eight cursors: clamped counts, this stratum's offset inside the tile's list, the verdict's sums
    const uint32_t raw = lane < BIN_SUB ? cursor[((size_t)vt * BIN_SUB + lane) * BIN_PAD] : 0u;
    const uint32_t cnt = min(raw, sub_cap);  // clamped: an overflowed call is redone
    const uint32_t total = __reduce_add_sync(0xffffffffu, cnt);
    const uint32_t below = __reduce_add_sync(0xffffffffu, lane < k ? cnt : 0u);
    const uint32_t n = __shfl_sync(0xffffffffu, cnt, k);
    const uint32_t base = vt * BIN_SUB * sub_cap;
    if (k == 0) {
        const uint32_t raw_total = __reduce_add_sync(0xffffffffu, raw), raw_max = __reduce_max_sync(0xffffffffu, raw);
        const uint32_t prefix = __reduce_add_sync(0xffffffffu, lane < sorted ? cnt : 0u);  // the sorted strata, in order
        if (lane == 0) {
            ranges[vt] = make_uint2(base, base + prefix);
            if (atomicAdd(&acc[0], raw_total) + raw_total < raw_total) atomicOr(&acc[3], 1u);  // 32-bit wrap: redo exactly
            atomicMax(&acc[1], raw_total);
            atomicMax(&acc[2], raw_max);
            if (raw_max > sub_cap) atomicOr(&acc[3], 1u);
            __threadfence();
            if (atomicAdd(&acc[4], 1u) == nvt - 1) {  // every tile has been accounted for
                __threadfence();
                info[0] = atomicAdd(&acc[0], 0u);
                info[1] = atomicAdd(&acc[1], 0u);
                info[2] = atomicAdd(&acc[2], 0u);
                info[3] = atomicAdd(&acc[3], 0u);  // the host reads them after an event recorded behind this kernel
            }
        }
    }
    // Per-tile mode: this call's sorted lists define the boundaries of the NEXT call (row vt of `next`): entry q is the
    // depth of the list element at position total (q+1) / BIN_SUB, written by the warp whose stratum holds that position
    // (below); entries nobody owns (empty tile, the unused eighth) are +inf.
    if (next && k == 0 && lane < BIN_SUB && (total == 0 || lane == BIN_SUB - 1))
        next[(size_t)vt * BIN_SUB + lane] = __int_as_float(0x7f800000);
    if (n == 0) return;
    const uint64_t *__restrict__ src = bucket + (size_t)sidx * sub_cap;
    uint64_t *srt = reinterpret_cast<uint64_t *>(rs_smem) + (size_t)warp * cap_pad;
    uint32_t *dst = point_list + base + below;

    // 1. range of the depth bits (positive floats order like their bit patterns)
    uint32_t lo = 0xffffffffu, hi = 0u;
    for (uint32_t i = lane; i < n; i += 32) {
        const uint32_t d = (uint32_t)(src[i] >> 32);
        lo = min(lo, d);
        hi = max(hi, d);
    }
    lo = __reduce_min_sync(0xffffffffu, lo);
    hi = __reduce_max_sync(0xffffffffu, hi);
    const bool by_index = lo == hi;  // every depth equal: spread the keys by their index instead
    if (by_index) {
        lo = 0xffffffffu, hi = 0u;
        for (uint32_t i = lane; i < n; i += 32) {
            const uint32_t d = (uint32_t)src[i];
            lo = min(lo, d);
            hi = max(hi, d);
        }
        lo = __reduce_min_sync(0xffffffffu, lo);
        hi = __reduce_max_sync(0xffffffffu, hi);
    }
    const float scale = 64.0f / ((float)(hi - lo) + 1.0f);
    auto bucket_of = [&](uint64_t key) -> uint32_t {  // monotone in the key: int -> float -> int conversions all are
        const uint32_t x = by_index ? (uint32_t)key : (uint32_t)(key >> 32);
        return min(63u, (uint32_t)(__uint2float_rz(x - lo) * scale));
    };
    // masks of the round's lanes whose key falls into bucket `lane` (lo) and `lane + 32` (hi), from the ballots of the
    // bucket number's six bits
    const uint32_t x0 = (lane & 1u) ? 0u : ~0u, x1 = (lane & 2u) ? 0u : ~0u, x2 = (lane & 4u) ? 0u : ~0u,
                   x3 = (lane & 8u) ? 0u : ~0u, x4 = (lane & 16u) ? 0u : ~0u;
    auto masks = [&](uint32_t b, bool valid, uint32_t &m_lo, uint32_t &m_hi) {
        uint32_t m = __ballot_sync(0xffffffffu, valid);
        m &= __ballot_sync(0xffffffffu, b & 1u) ^ x0;
        m &= __ballot_sync(0xffffffffu, b & 2u) ^ x1;
        m &= __ballot_sync(0xffffffffu, b & 4u) ^ x2;
        m &= __ballot_sync(0xffffffffu, b & 8u) ^ x3;
        m &= __ballot_sync(0xffffffffu, b & 16u) ^ x4;
        const uint32_t top = __ballot_sync(0xffffffffu, b & 32u);
        m_lo = m & ~top;
        m_hi = m & top;
    };
    // 2. count
    uint32_t c_lo = 0, c_hi = 0;
    for (uint32_t r0 = 0; r0 < n; r0 += 32) {
        const uint32_t i = r0 + lane;
        const bool valid = i < n;
        const uint32_t b = valid ? bucket_of(src[i]) : 0u;
        uint32_t m_lo, m_hi;
        masks(b, valid, m_lo, m_hi);
        c_lo += __popc(m_lo);
        c_hi += __popc(m_hi);
    }
    // 3. offsets (buckets 0..31 first, then 32..63), scatter
    uint32_t i_lo = c_lo, i_hi = c_hi;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t t_lo = __shfl_up_sync(0xffffffffu, i_lo, d), t_hi = __shfl_up_sync(0xffffffffu, i_hi, d);
        if ((int)lane >= d) {
            i_lo += t_lo;
            i_hi += t_hi;
        }
    }
    const uint32_t s_lo = i_lo - c_lo, s_hi = __shfl_sync(0xffffffffu, i_lo, 31) + i_hi - c_hi;  // bucket starts
    uint32_t run_lo = s_lo, run_hi = s_hi;
    const uint32_t lt = (1u << lane) - 1u;
    for (uint32_t r0 = 0; r0 < n; r0 += 32) {
        const uint32_t i = r0 + lane;
        const bool valid = i < n;
        const uint64_t key = valid ? src[i] : 0ull;
        const uint32_t b = valid ? bucket_of(key) : 0u;
        uint32_t m_lo, m_hi;
        masks(b, valid, m_lo, m_hi);
        const uint32_t owner = b & 31u;
        const uint32_t same_lo = __shfl_sync(0xffffffffu, m_lo, owner), same_hi = __shfl_sync(0xffffffffu, m_hi, owner);
        const uint32_t at_lo = __shfl_sync(0xffffffffu, run_lo, owner), at_hi = __shfl_sync(0xffffffffu, run_hi, owner);
        const uint32_t same = (b & 32u) ? same_hi : same_lo, at = (b & 32u) ? at_hi : at_lo;
        if (valid) srt[at + __popc(same & lt)] = key;
        run_lo += __popc(m_lo);
        run_hi += __popc(m_hi);
    }
    __syncwarp();
    // 4. rank every key inside its bucket; its index goes straight to its final position
    for (uint32_t r0 = 0; r0 < n; r0 += 32) {
        const uint32_t i = r0 + lane;
        const bool valid = i < n;
        const uint64_t key = valid ? src[i] : 0ull;
        const uint32_t b = valid ? bucket_of(key) : 0u;
        const uint32_t owner = b & 31u;
        const uint32_t st_lo = __shfl_sync(0xffffffffu, s_lo, owner), st_hi = __shfl_sync(0xffffffffu, s_hi, owner);
        const uint32_t n_lo = __shfl_sync(0xffffffffu, c_lo, owner), n_hi = __shfl_sync(0xffffffffu, c_hi, owner);
        const uint32_t bs = (b & 32u) ? st_hi : st_lo, bn = valid ? ((b & 32u) ? n_hi : n_lo) : 0u;
        uint32_t rank = 0;
        for (uint32_t q = 0; q < bn; q++) rank += srt[bs + q] < key ? 1u : 0u;  // keys are distinct: (depth, index)
        if (valid) dst[bs + rank] = (uint32_t)key;
    }
    if (next) {
        __syncwarp();  // the list segment written above is visible to every lane of this warp
        if (lane < BIN_SUB - 1) {
            const uint32_t pos = (uint32_t)(((uint64_t)total * (lane + 1)) / BIN_SUB);
            if (pos >= below && pos < below + n)
                next[(size_t)vt * BIN_SUB + lane] = rec2[(size_t)(vt / ntiles) * P + dst[pos - below]].y;
        }
    }
}

// per-tile boundaries from the sorted lists of an exact-path call: thread (tile, q) reads the depth of the entry at the
// (q+1)-th octile of the tile's list
__global__ void k_tile_octiles(const DevCfg c, const uint32_t *__restrict__ point_list, const uint2 *__restrict__ ranges,
                               const float4 *__restrict__ rec2, float *__restrict__ table) {
    const size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t nvt = (size_t)c.V * c.ntiles;
    if (g >= nvt * BIN_SUB) return;
    const size_t vt = g / BIN_SUB;
    const uint32_t q = (uint32_t)(g % BIN_SUB);
    const uint2 r = ranges[vt];
    const uint32_t n = r.y - r.x;
    float b = __int_as_float(0x7f800000);
    if (n > 0 && q < BIN_SUB - 1) {
        const uint32_t pos = r.x + (uint32_t)(((uint64_t)n * (q + 1)) / BIN_SUB);
        b = rec2[(vt / c.ntiles) * (size_t)c.P + point_list[pos]].y;
    }
    table[g] = b;
}

int bin_learn_tile_strata(const DevCfg &c, const uint32_t *point_list, const uint2 *ranges, const float4 *rec2, float *table,
                          cudaStream_t st) {
    const size_t n = (size_t)c.V * c.ntiles * BIN_SUB;
    if (n == 0) return GS_OK;
    k_tile_octiles<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(c, point_list, ranges, rec2, table);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}

template <int THREADS, int MAX_ITEMS>
int launch_stratum_sort(int nvt, uint32_t sub_cap, const uint32_t *cursor, const uint64_t *bucket, uint32_t *point_list,
                        uint2 *ranges, uint32_t *acc, uint32_t *info, cudaStream_t st) {
    const size_t smem = tile_sort_smem_bytes<THREADS, MAX_ITEMS>();
    GS_CUDA_OK(cudaFuncSetAttribute(k_stratum_sort<THREADS, MAX_ITEMS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_stratum_sort<THREADS, MAX_ITEMS><<<nvt * BIN_SUB, THREADS, smem, st>>>((uint32_t)nvt, sub_cap, cursor, bucket, point_list, ranges,
                                                                             acc, info);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}

int bin_sort_strata(const DevCfg &c, uint32_t sub_cap, const uint32_t *cursor, const void *bucket, uint32_t *point_list,
                    uint2 *ranges, uint32_t *acc, uint32_t *info, cudaStream_t st, bool merge_sort, const float4 *rec2,
                    float *next_tile_strata, const uint8_t *need) {
    if (!merge_sort || next_tile_strata) {   // (the merge-sort kernel does not refresh per-tile boundaries)
        // hand-written warp-per-stratum distribution sort (default)
        if (sub_cap > BIN_STRATUM_CAP) return gs_set_error(GS_ERR_INVALID, "stratum capacity beyond the sort's");
        const uint32_t nvt = (uint32_t)c.V * (uint32_t)c.ntiles;
        const uint32_t cap_pad = (sub_cap + 31u) & ~31u;
        const size_t smem = (size_t)RS_WARPS * cap_pad * 8;
        if (smem > ((size_t)48 << 10))  // (per device and cheap: no process-wide cache, a process may drive several GPUs)
            GS_CUDA_OK(cudaFuncSetAttribute(k_stratum_rank_sort, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        const uint32_t ctas = (nvt * BIN_SUB + RS_WARPS - 1) / RS_WARPS;
        k_stratum_rank_sort<<<ctas, RS_WARPS * 32, smem, st>>>(nvt, sub_cap, cap_pad, cursor, static_cast<const uint64_t *>(bucket),
                                                               point_list, ranges, acc, info, rec2, (uint32_t)c.P, (uint32_t)c.ntiles,
                                                               next_tile_strata, need);
        GS_CUDA_OK(cudaGetLastError());
        return GS_OK;
    }
    // 128 threads: faster than 64 or 256 on C2's sub-buckets of a few hundred keys.
    // The kernel is instantiated for the call's capacity: the 4- and 8-keys-per-thread versions need fewer registers
    // and less shared memory than the 16-key one, i.e. more resident CTAs for this latency-bound sort.
    constexpr int THREADS = 128;
    static_assert(THREADS * 16 == BIN_STRATUM_CAP, "capacity of a stratum");
    if (sub_cap > BIN_STRATUM_CAP) return gs_set_error(GS_ERR_INVALID, "stratum capacity beyond the sort's");
    const int nvt = c.V * c.ntiles;
    const uint64_t *b = static_cast<const uint64_t *>(bucket);
    if (sub_cap <= THREADS * 4) return launch_stratum_sort<THREADS, 4>(nvt, sub_cap, cursor, b, point_list, ranges, acc, info, st);
    if (sub_cap <= THREADS * 8) return launch_stratum_sort<THREADS, 8>(nvt, sub_cap, cursor, b, point_list, ranges, acc, info, st);
    return launch_stratum_sort<THREADS, 16>(nvt, sub_cap, cursor, b, point_list, ranges, acc, info, st);
}

size_t bin_strata_bytes(const DevCfg &c) {
    const size_t per_view = (size_t)c.V * BIN_SUB * 4 + (size_t)c.V * STRATA_BINS * 4;
    const size_t per_tile = 2 * (size_t)c.V * c.ntiles * BIN_SUB * 4;  // two tables: this call's and the next one's
    return align256(per_view > per_tile ? per_view : per_tile) + (size_t)c.V * c.ntiles;
}

uint8_t *bin_need_table(const DevCfg &c, void *strata_buf) {
    return static_cast<uint8_t *>(strata_buf) + bin_strata_bytes(c) - (size_t)c.V * c.ntiles;
}

int bin_learn_strata(const DevCfg &c, const ushort4 *rects, const float4 *rec2, void *strata_buf, cudaStream_t st) {
    float *strata = static_cast<float *>(strata_buf);
    uint32_t *hist = reinterpret_cast<uint32_t *>(strata + (size_t)c.V * BIN_SUB);
    GS_CUDA_OK(cudaMemsetAsync(hist, 0, (size_t)c.V * STRATA_BINS * 4, st));
    const int bx = max(1, min(64, (c.P + 255) / 256));
    k_depth_hist<<<dim3(bx, c.V), 256, 0, st>>>(c, rects, rec2, hist);
    GS_CUDA_OK(cudaGetLastError());
    k_strata_from_hist<<<c.V, 1024, 0, st>>>(hist, strata);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}

int bin_sort_spec(const DevCfg &c, uint32_t sub_cap, uint32_t tile_limit, const uint32_t *cursor, const void *bucket,
                  uint32_t *point_list, uint2 *ranges, cudaStream_t st) {
    const int nvt = c.V * c.ntiles;
    const uint64_t *b = static_cast<const uint64_t *>(bucket);
    switch (spec_sort_capacity(tile_limit)) {
        case 1024: return launch_tile_sort_spec<256, 4>(nvt, sub_cap, cursor, b, point_list, ranges, st);
        case 2048: return launch_tile_sort_spec<512, 4>(nvt, sub_cap, cursor, b, point_list, ranges, st);
        case 4096: return launch_tile_sort_spec<1024, 4>(nvt, sub_cap, cursor, b, point_list, ranges, st);
        default: return launch_tile_sort_spec<1024, 8>(nvt, sub_cap, cursor, b, point_list, ranges, st);
    }
}

int bin_sort_fallback(const DevCfg &c, int64_t D, const float4 *rec0, const float4 *rec1, const float4 *rec2,
                      const ushort4 *rects, void *scratch, size_t scratch_bytes, uint32_t *point_list, uint2 *ranges,
                      cudaStream_t st) {
    GS_CUDA_OK(cudaMemsetAsync(ranges, 0, sizeof(uint2) * (size_t)c.V * c.ntiles, st));
    if (D == 0) return GS_OK;
    const size_t n = (size_t)c.V * c.P;
    unsigned char *p = static_cast<unsigned char *>(scratch);
    auto take = [&](size_t bytes) {
        unsigned char *q = p;
        p += align256(bytes);
        return q;
    };
    uint64_t *depth_keys = reinterpret_cast<uint64_t *>(take(n * 8));
    uint64_t *order = reinterpret_cast<uint64_t *>(take(n * 8));
    uint32_t *cnt = reinterpret_cast<uint32_t *>(take(n * 4));
    uint32_t *offsets = reinterpret_cast<uint32_t *>(take(n * 4));
    uint32_t *keys_in = reinterpret_cast<uint32_t *>(take((size_t)D * 4));
    uint32_t *keys_out = reinterpret_cast<uint32_t *>(take((size_t)D * 4));
    uint32_t *vals_in = reinterpret_cast<uint32_t *>(take((size_t)D * 4));
    size_t temp_bytes = scratch_bytes - (size_t)(p - static_cast<unsigned char *>(scratch));
    const unsigned blocks = (unsigned)((n + 255) / 256);

    k_depth_keys<<<blocks, 256, 0, st>>>(n, rec0, rec1, rec2, rects, depth_keys, cnt);
    GS_CUDA_OK(cudaGetLastError());
    GS_CUDA_OK(cub::DeviceRadixSort::SortKeys(p, temp_bytes, depth_keys, order, (int)n, 32, 64, st));
    auto it = thrust::make_transform_iterator((const uint64_t *)order, TilesInOrder{cnt});
    GS_CUDA_OK(cub::DeviceScan::InclusiveSum(p, temp_bytes, it, offsets, (int)n, st));
    k_emit_ordered<<<blocks, 256, 0, st>>>(c, order, rec0, rec1, rec2, rects, cnt, offsets, keys_in, vals_in);
    GS_CUDA_OK(cudaGetLastError());
    GS_CUDA_OK(cub::DeviceRadixSort::SortPairs(p, temp_bytes, keys_in, keys_out, vals_in, point_list, (int)D, 0,
                                               tile_bits(c), st));
    k_ranges<<<(unsigned)((D + 255) / 256), 256, 0, st>>>(D, keys_out, ranges);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}

// ---------------------------------------------------------------------------------------------------------
// Sync-free binning (DESIGN.md 5.18).  The exact path's count (k_preprocess), k_tile_scan, k_emit_buckets and tile
// merge sort, with the decisions the host takes there from the read-back words taken on the device instead:
//   k_capacity_gate  D > capacity: every tile range empty, every tile count zero, the verdict set (emission and the
//                    sorts then have nothing to do, and the caller's planes become NaN);
//   size classes     each class of the merge sort is launched over every (view, tile) CTA; a CTA sorts its tile only
//                    if its list falls in the class, so a short list never pays for an 8192-key sort;
//   k_tile_sort_long lists longer than BIN_SMEM_CAP, which the exact path hands to the CUB radix fallback: one CTA per
//                    long (view, tile), an LSD radix sort of the tile's bucket in global memory.
// No kernel reads or writes past the workspace for any D: stores into the buckets and lists are at offsets below D,
// and nothing is stored unless D <= capacity.
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_capacity_gate(uint32_t nvt, uint32_t capacity, uint32_t *__restrict__ status, const uint32_t *__restrict__ tile_start,
                uint32_t *__restrict__ tile_n, uint2 *__restrict__ ranges) {
    const uint32_t D = status[SF_D];
    const bool over = D > capacity;
    for (uint32_t vt = blockIdx.x * blockDim.x + threadIdx.x; vt < nvt; vt += gridDim.x * blockDim.x) {
        const uint32_t start = over ? 0u : tile_start[vt];
        const uint32_t n = over ? 0u : tile_n[vt];
        if (over) tile_n[vt] = 0u;
        ranges[vt] = make_uint2(start, start + n);
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        status[SF_VERDICT] = over ? 1u : 0u;
        if (over) status[SF_EXCEEDED] = 1u;
        status[SF_REQUIRED] = max(status[SF_REQUIRED], D);
    }
}

// One size class of the tile merge sort: lists of (lo, THREADS * MAX_ITEMS] entries.  Ranges come from the gate.
template <int THREADS, int MAX_ITEMS>
__global__ void __launch_bounds__(THREADS)
k_tile_sort_class(uint32_t lo, const uint32_t *__restrict__ tile_n, const uint32_t *__restrict__ tile_start,
                  const uint64_t *__restrict__ bucket, uint32_t *__restrict__ point_list) {
    extern __shared__ __align__(16) unsigned char ts_smem[];
    const uint32_t vt = blockIdx.x;
    const uint32_t n = tile_n[vt];
    if (n <= lo || n > (uint32_t)(THREADS * MAX_ITEMS)) return;
    const uint32_t off = tile_start[vt];
    const uint64_t *src = bucket + off;
    sort_bucket_dispatch<THREADS, MAX_ITEMS>([src](uint32_t i) { return src[i]; }, point_list + off, n, ts_smem);
}

template <int THREADS, int MAX_ITEMS>
int launch_tile_sort_class(uint32_t lo, int nvt, const uint32_t *tile_n, const uint32_t *tile_start, const uint64_t *bucket,
                           uint32_t *point_list, cudaStream_t st) {
    const size_t smem = tile_sort_smem_bytes<THREADS, MAX_ITEMS>();
    GS_CUDA_OK(cudaFuncSetAttribute(k_tile_sort_class<THREADS, MAX_ITEMS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_tile_sort_class<THREADS, MAX_ITEMS><<<nvt, THREADS, smem, st>>>(lo, tile_n, tile_start, bucket, point_list);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}

// Lists longer than BIN_SMEM_CAP: a stable LSD radix sort of the 64-bit (depth bits, index) keys, 8-bit digits, between
// the tile's bucket and its stretch of `tmp`, in chunks of one key per thread.  A key's place in its chunk is its warp's
// count of the digit before it (match_any) plus the counts of the earlier warps; a pass whose digit is the same for
// every key would be the identity and is skipped.  The keys are a total order, so the list is the radix fallback's.
constexpr int LS_THREADS = 1024, LS_WARPS = LS_THREADS / 32, LS_RADIX = 256;

__global__ void __launch_bounds__(LS_THREADS)
k_tile_sort_long(const uint32_t *__restrict__ tile_n, const uint32_t *__restrict__ tile_start, uint64_t *__restrict__ bucket,
                 uint64_t *__restrict__ tmp, uint32_t *__restrict__ point_list) {
    __shared__ uint32_t warp_at[LS_WARPS][LS_RADIX];   // per chunk: warp w's count of digit d, then its first position
    __shared__ uint32_t hist[LS_RADIX], next[LS_RADIX];
    __shared__ int s_skip;
    const uint32_t vt = blockIdx.x;
    const uint32_t n = tile_n[vt];
    if (n <= (uint32_t)BIN_SMEM_CAP) return;
    const uint32_t off = tile_start[vt];
    const uint32_t tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const uint32_t lt = (1u << lane) - 1u;
    uint64_t *src = bucket + off, *dst = tmp + off;
    for (int shift = 0; shift < 64; shift += 8) {
        for (int d = tid; d < LS_RADIX; d += LS_THREADS) hist[d] = 0u;
        if (tid == 0) s_skip = 0;
        __syncthreads();
        for (uint32_t i = tid; i < n; i += LS_THREADS) atomicAdd(&hist[(uint32_t)(src[i] >> shift) & 255u], 1u);
        __syncthreads();
        if (tid < LS_RADIX && hist[tid] == n) s_skip = 1;
        if (warp == 0) {   // exclusive scan of the histogram: eight digits per lane
            uint32_t v[8], sum = 0;
#pragma unroll
            for (int k = 0; k < 8; k++) {
                v[k] = hist[lane * 8 + k];
                sum += v[k];
            }
            uint32_t incl = sum;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint32_t t = __shfl_up_sync(0xffffffffu, incl, d);
                if ((int)lane >= d) incl += t;
            }
            uint32_t run = incl - sum;
#pragma unroll
            for (int k = 0; k < 8; k++) {
                next[lane * 8 + k] = run;
                run += v[k];
            }
        }
        __syncthreads();
        const int skip = s_skip;
        __syncthreads();   // every thread has read it before thread 0 resets it for the next pass
        if (skip) continue;
        for (uint32_t c0 = 0; c0 < n; c0 += LS_THREADS) {
            const uint32_t i = c0 + tid;
            const bool valid = i < n;
            const uint64_t key = valid ? src[i] : 0ull;
            const uint32_t d = valid ? ((uint32_t)(key >> shift) & 255u) : 0xffffffffu;
            const uint32_t peers = __match_any_sync(0xffffffffu, d);
            for (int k = tid; k < LS_WARPS * LS_RADIX; k += LS_THREADS) (&warp_at[0][0])[k] = 0u;
            __syncthreads();
            if (valid && (peers & lt) == 0) warp_at[warp][d] = __popc(peers);
            __syncthreads();
            if (tid < LS_RADIX) {
                uint32_t run = next[tid];
                for (int w = 0; w < LS_WARPS; w++) {
                    const uint32_t cnt = warp_at[w][tid];
                    warp_at[w][tid] = run;
                    run += cnt;
                }
                next[tid] = run;
            }
            __syncthreads();
            if (valid) dst[warp_at[warp][d] + __popc(peers & lt)] = key;
            __syncthreads();
        }
        uint64_t *t = src;
        src = dst;
        dst = t;
    }
    __syncthreads();
    for (uint32_t i = tid; i < n; i += LS_THREADS) point_list[off + i] = (uint32_t)src[i];
}

// NaN into the arrays of `a` when the verdict is set
__global__ void __launch_bounds__(256) k_sf_poison(const uint32_t *__restrict__ status, const SfPoison a) {
    if (!status[SF_VERDICT]) return;
    const float nan = __int_as_float(0x7fffffff);
    for (int k = 0; k < a.count; k++)
        for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.n[k]; i += (size_t)gridDim.x * blockDim.x)
            a.ptr[k][i] = nan;
}

int bin_sync_free(const DevCfg &c, const SyncFreeBins &b, const float4 *rec0, const float4 *rec1, const float4 *rec2,
                  cudaStream_t st) {
    const int nvt = c.V * c.ntiles;
    const size_t n = (size_t)c.V * c.P;
    int rc = bin_tile_scan(c, b.tile_counts, b.sub_offsets, b.tile_start, b.tile_n, b.status, st);
    if (rc != GS_OK) return rc;
    const unsigned gate_ctas = (unsigned)min((nvt + 255) / 256, 1024);
    k_capacity_gate<<<gate_ctas, 256, 0, st>>>((uint32_t)nvt, b.capacity, b.status, b.tile_start, b.tile_n, b.ranges);
    GS_CUDA_OK(cudaGetLastError());
    if (n > 0) {
        GS_CUDA_OK(cudaMemsetAsync(b.cursor, 0, bin_counter_bytes(c), st));
        k_emit_buckets<true><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(c, rec0, rec1, rec2, b.rects, b.sub_offsets, 0,
                                                                          nullptr, 0, b.cursor, b.bucket, b.status,
                                                                          b.capacity);
        GS_CUDA_OK(cudaGetLastError());
    }
    // the size classes of bin_sort_fast's ladder: (0, 1024], (1024, 2048], (2048, 4096], (4096, 8192]
    if ((rc = launch_tile_sort_class<256, 4>(0, nvt, b.tile_n, b.tile_start, b.bucket, b.point_list, st)) != GS_OK) return rc;
    if ((rc = launch_tile_sort_class<512, 4>(1024, nvt, b.tile_n, b.tile_start, b.bucket, b.point_list, st)) != GS_OK) return rc;
    if ((rc = launch_tile_sort_class<1024, 4>(2048, nvt, b.tile_n, b.tile_start, b.bucket, b.point_list, st)) != GS_OK) return rc;
    if ((rc = launch_tile_sort_class<1024, 8>(4096, nvt, b.tile_n, b.tile_start, b.bucket, b.point_list, st)) != GS_OK) return rc;
    k_tile_sort_long<<<nvt, LS_THREADS, 0, st>>>(b.tile_n, b.tile_start, b.bucket, b.tmp, b.point_list);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}

int sf_poison_if_exceeded(const uint32_t *status, const SfPoison &arrays, cudaStream_t st) {
    if (arrays.count == 0) return GS_OK;
    size_t most = 0;
    for (int k = 0; k < arrays.count; k++) most = arrays.n[k] > most ? arrays.n[k] : most;
    const unsigned ctas = (unsigned)(most < (size_t)256 * 512 ? (most + 255) / 256 : 512);
    k_sf_poison<<<ctas, 256, 0, st>>>(status, arrays);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}
