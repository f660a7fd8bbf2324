// gs_capi.cu -- the C ABI declared in include/gsplat_b200.h: argument validation, workspace management,
// stage sequencing.  No torch, no exceptions across the boundary.
#include <cstdio>
#include <cstring>
#include <new>

#include "gs_common.cuh"

// ---------------------------------------------------------------------------------------------------------
// errors
// ---------------------------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";

int gs_set_error(int code, const char *msg) {
    snprintf(g_err, sizeof(g_err), "%s", msg);
    return code;
}
int gs_set_cuda_error(cudaError_t e, const char *what, const char *file, int line) {
    snprintf(g_err, sizeof(g_err), "CUDA error %d (%s) in %s at %s:%d", (int)e, cudaGetErrorString(e), what, file, line);
    return e == cudaErrorMemoryAllocation ? GS_ERR_OOM : GS_ERR_CUDA;
}

extern "C" const char *gs_last_error(void) { return g_err; }
extern "C" int gs_abi_version(void) { return GS_ABI_VERSION; }
extern "C" uint32_t gs_supported_flags(void) {
    return GS_FLAG_DEPTH | GS_FLAG_PREFILTERED | GS_FLAG_DETERMINISTIC | GS_FLAG_ANTIALIAS;
}

// ---------------------------------------------------------------------------------------------------------
// context: grow-only scratch, pinned read-back word, optional stage timers
// ---------------------------------------------------------------------------------------------------------
// Grow-only scratch.  With a pool and a stream, growth is stream-ordered (cudaFreeAsync + cudaMallocFromPoolAsync on the
// context's own stream and pool): no device-wide synchronisation when a bigger batch arrives mid-training.  Without
// (pool == nullptr: the host-staging buffer, which a second stream writes into) it is cudaFree + cudaMalloc.
struct GrowBuf {
    void *p = nullptr;
    size_t bytes = 0;
    bool pooled = false;
    int reserve(size_t need, double headroom, cudaMemPool_t pool = nullptr, cudaStream_t st = nullptr) {
        if (need <= bytes) return GS_OK;
        if (p) {
            if (pooled) GS_CUDA_OK(cudaFreeAsync(p, st));  // everything that used it was enqueued on st before this point
            else GS_CUDA_OK(cudaFree(p));                  // implicit device sync
        }
        p = nullptr;
        bytes = 0;
        size_t want = (size_t)((double)need * headroom) + 256;
        if (pool) GS_CUDA_OK(cudaMallocFromPoolAsync(&p, want, pool, st));
        else GS_CUDA_OK(cudaMalloc(&p, want));
        pooled = pool != nullptr;
        bytes = want;
        return GS_OK;
    }
    void release() {  // after a device synchronisation
        if (p) cudaFree(p);
        p = nullptr;
        bytes = 0;
    }
};

struct GsContext {
    // Private stream-ordered pool: saved state (records, lists, image planes) and scratch -- never the device's default
    // pool.  Blocks freed by gs_saved_free stay cached for the next calls (pool_follow: a periodic, bounded trim);
    // gs_context_trim() / gs_context_destroy() hand everything back.
    cudaMemPool_t pool = nullptr;
    int calls_since_peak_reset = 0;   // pool_follow: forwards since the pool's used-bytes high-water mark was last reset
    GrowBuf per_gaussian;  // rects | tile counts / offsets / cursors ; backward: accumulators
    GrowBuf sort;          // buckets (fast path) or radix-sort buffers (fallback)
    GrowBuf host_stage;    // device mirror of host buffers (gs_render_host)
    uint32_t *d_word = nullptr;  // device alias of h_word (mapped pinned memory)
    uint32_t *h_word = nullptr;  // pinned, written by the device: [0] tile instances, [1] longest tile list, [2] largest sub-counter, [3] overflow
    // the shapes earlier forwards taught (gs_bin_policy.h), each with its boundary tables: [V][BIN_SUB] (or two tables
    // of [V*tiles][BIN_SUB]) stratum boundaries + histogram scratch
    static constexpr int SHAPE_SLOTS = 4;
    ShapeSlot slots[SHAPE_SLOTS];
    GrowBuf strata_tabs[SHAPE_SLOTS];
    uint64_t use_counter = 0;
    cudaEvent_t ev_pre = nullptr;   // "preprocess done" (speculative path: lets the radii copy start early)
    cudaEvent_t ev_info = nullptr;  // "binning verdict copied to the host"
    // gs_render_host's split pipeline: k_sh_colour pulls the SH block out of the caller's pinned buffer on aux_stream while
    // geometry, binning and the tile sort run on the launch stream; the compositor waits for ev_colour
    cudaStream_t aux_stream = nullptr;
    cudaEvent_t ev_alloc = nullptr, ev_colour = nullptr;
    // gs_render_host: radii are final once the forward's mid-way sync has passed, so their copy to the host
    // overlaps binning + compositing on a side stream
    cudaStream_t copy_stream = nullptr;
    static constexpr int FEED_MAX = 8;
    cudaEvent_t feed_ev[FEED_MAX] = {};   // gs_render_host: piece k of the SH block has landed (HostFeed)
    GsStats stats{};
    bool profiling = false;
    cudaEvent_t ev[GS_NUM_STAGES + 1][2]{};
    bool ev_valid[GS_NUM_STAGES] = {};
    float stage_ms[GS_NUM_STAGES] = {};
};

namespace {

inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

struct StageTimer {
    GsContext *ctx;
    int stage;
    cudaStream_t st;
    StageTimer(GsContext *c, int s, cudaStream_t stream) : ctx(c), stage(s), st(stream) {
        if (ctx->profiling) cudaEventRecord(ctx->ev[stage][0], st);
    }
    ~StageTimer() {
        if (ctx->profiling) {
            cudaEventRecord(ctx->ev[stage][1], st);
            ctx->ev_valid[stage] = true;
        }
    }
};

int validate(const GsConfig *cfg, const GsInputs *in) {
    if (!cfg || !in) return gs_set_error(GS_ERR_INVALID, "null config/inputs");
    if (cfg->P < 0 || cfg->S < 1 || cfg->V < 1 || cfg->V % cfg->S != 0)
        return gs_set_error(GS_ERR_INVALID, "need P >= 0, S >= 1, V >= 1 and V % S == 0");
    if (cfg->image_height < 1 || cfg->image_width < 1) return gs_set_error(GS_ERR_INVALID, "empty image");
    if ((in->shs == nullptr) == (in->colors_precomp == nullptr) && cfg->P > 0)
        return gs_set_error(GS_ERR_INVALID, "Please provide excatly one of either SHs or precomputed colors!");
    const bool sr = in->scales != nullptr || in->rotations != nullptr;
    if (cfg->P > 0 && ((sr && in->cov3D_precomp) || (!sr && !in->cov3D_precomp) ||
                       (sr && (!in->scales || !in->rotations))))
        return gs_set_error(GS_ERR_INVALID,
                            "Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!");
    if (in->shs && cfg->M < 1) return gs_set_error(GS_ERR_INVALID, "shs given but M < 1");
    if (cfg->P > 0 && (!in->means3D || !in->opacities)) return gs_set_error(GS_ERR_INVALID, "means3D/opacities missing");
    if (!cfg->viewmatrix || !cfg->projmatrix || !cfg->campos)
        return gs_set_error(GS_ERR_INVALID, "viewmatrix/projmatrix/campos missing");
    if ((int64_t)cfg->P * cfg->V > 0x7fffffffll) return gs_set_error(GS_ERR_OVERFLOW, "P*V exceeds 2^31-1");
    if ((cfg->image_width + GS_TILE - 1) / GS_TILE > 65535 || (cfg->image_height + GS_TILE - 1) / GS_TILE > 65535)
        return gs_set_error(GS_ERR_INVALID, "image too large");
    return GS_OK;
}

// The forward's depth mode (GsConfig::depth_mode): known, on a depth channel, with the near / far its f(z) reads.
int validate_depth_mode(const GsConfig *cfg) {
    const int m = cfg->depth_mode;
    if (m < GS_DEPTH_Z || m > GS_DEPTH_LOG) return gs_set_error(GS_ERR_INVALID, "unknown depth_mode");
    if (m != GS_DEPTH_Z && !(cfg->flags & GS_FLAG_DEPTH))
        return gs_set_error(GS_ERR_INVALID, "a depth_mode other than GS_DEPTH_Z needs GS_FLAG_DEPTH");
    if ((m == GS_DEPTH_RELATIVE_DISPARITY || m == GS_DEPTH_LOG) && !cfg->depth_near_far)
        return gs_set_error(GS_ERR_INVALID, "depth_mode GS_DEPTH_RELATIVE_DISPARITY / GS_DEPTH_LOG needs depth_near_far");
    return GS_OK;
}

// GS_FLAG_ANTIALIAS has no kernel behind two tuning knobs (the forward refuses both: its backward could not run)
int validate_antialias(uint32_t flags, uint32_t tuning, uint32_t knobs) {
    if (!(flags & GS_FLAG_ANTIALIAS)) return GS_OK;
    if (tuning & knobs & GS_TUNE_PRE_OCC6)
        return gs_set_error(GS_ERR_INVALID, "GS_TUNE_PRE_OCC6 has no anti-aliased kernel (GS_FLAG_ANTIALIAS)");
    if (tuning & knobs & GS_TUNE_PBWD_2PHASE)
        return gs_set_error(GS_ERR_INVALID, "GS_TUNE_PBWD_2PHASE has no anti-aliased kernel (GS_FLAG_ANTIALIAS)");
    return GS_OK;
}
constexpr uint32_t AA_FWD_KNOBS = GS_TUNE_PRE_OCC6 | GS_TUNE_PBWD_2PHASE, AA_BWD_KNOBS = GS_TUNE_PBWD_2PHASE;

DevCfg make_dev_cfg(const GsConfig *cfg) {
    DevCfg c{};
    c.P = cfg->P; c.S = cfg->S; c.V = cfg->V; c.VPS = cfg->V / cfg->S; c.M = cfg->M;
    const int maxdeg = cfg->sh_eval_max_degree > 0 ? cfg->sh_eval_max_degree : 3;
    int deg = cfg->sh_degree < maxdeg ? cfg->sh_degree : maxdeg;
    if (deg > 4) deg = 4;                                    // the evaluator implements bands 0..4
    while (deg > 0 && (deg + 1) * (deg + 1) > cfg->M) deg--;  // never read past the coefficients supplied
    if (deg < 0) deg = 0;
    c.deg = deg;
    c.H = cfg->image_height; c.W = cfg->image_width;
    c.gx = (c.W + GS_TILE - 1) / GS_TILE; c.gy = (c.H + GS_TILE - 1) / GS_TILE; c.ntiles = c.gx * c.gy;
    c.flags = cfg->flags;
    c.tanfovx = cfg->tanfovx; c.tanfovy = cfg->tanfovy; c.scale_modifier = cfg->scale_modifier;
    c.near_cull_z = cfg->near_cull_z > 0.f ? cfg->near_cull_z : 0.2f;
    c.dilation = cfg->dilation > 0.f ? cfg->dilation : 0.3f;
    c.guard_band = cfg->guard_band > 0.f ? cfg->guard_band : 1.3f;
    c.view = cfg->viewmatrix; c.proj = cfg->projmatrix; c.campos = cfg->campos; c.bg = cfg->bg;
    c.tanfov = cfg->tanfov; c.view_scale = cfg->view_scale;
    return c;
}

DevInputs make_dev_inputs(const GsInputs *in) {
    DevInputs d{};
    d.means3D = in->means3D; d.opacities = in->opacities; d.shs = in->shs; d.colors_precomp = in->colors_precomp;
    d.scales = in->scales; d.rotations = in->rotations; d.cov3D = in->cov3D_precomp;
    return d;
}

// carve the saved-state block (everything but the tile-instance list, which gets its own exactly-sized
// allocation once its length has been read back)
size_t saved_layout(GsSaved *s, const DevCfg &c, unsigned char *base) {
    size_t off = 0;
    const size_t n = (size_t)c.V * c.P, px = (size_t)c.V * c.H * c.W;
    auto take = [&](size_t bytes) {
        unsigned char *p = base ? base + off : nullptr;
        off += align256(bytes);
        return p;
    };
    s->rec0 = reinterpret_cast<float4 *>(take(n * 16));
    s->rec1 = reinterpret_cast<float4 *>(take(n * 16));
    s->rec2 = reinterpret_cast<float4 *>(take(n * 16));
    s->meta = reinterpret_cast<uint8_t *>(take(n));
    s->ranges = reinterpret_cast<uint2 *>(take((size_t)c.V * c.ntiles * 8));
    s->final_T = reinterpret_cast<float *>(take(px * 4));
    s->n_contrib = reinterpret_cast<uint32_t *>(take(px * 4));
    s->sched = reinterpret_cast<uint32_t *>(take(8));
    return off;
}

}  // namespace

extern "C" int gs_context_create(GsContext **out) {
    if (!out) return gs_set_error(GS_ERR_INVALID, "null out");
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return gs_set_error(GS_ERR_NO_DEVICE, "no CUDA device");
    GsContext *ctx = new (std::nothrow) GsContext();
    if (!ctx) return gs_set_error(GS_ERR_OOM, "host allocation failed");
    cudaMemPoolProps props{};
    props.allocType = cudaMemAllocationTypePinned;
    props.handleTypes = cudaMemHandleTypeNone;
    props.location.type = cudaMemLocationTypeDevice;
    props.location.id = dev;
    cudaError_t e = cudaMemPoolCreate(&ctx->pool, &props);
    if (e != cudaSuccess) {
        delete ctx;
        return gs_set_cuda_error(e, "cudaMemPoolCreate", __FILE__, __LINE__);
    }
    uint64_t never = UINT64_MAX;   // freed blocks stay cached in the pool: see pool_follow
    cudaMemPoolSetAttribute(ctx->pool, cudaMemPoolAttrReleaseThreshold, &never);
    e = cudaHostAlloc(reinterpret_cast<void **>(&ctx->h_word), 64, cudaHostAllocMapped);
    if (e == cudaSuccess) e = cudaHostGetDevicePointer(reinterpret_cast<void **>(&ctx->d_word), ctx->h_word, 0);
    if (e != cudaSuccess) {
        cudaMemPoolDestroy(ctx->pool);
        delete ctx;
        return gs_set_cuda_error(e, "cudaHostAlloc", __FILE__, __LINE__);
    }
    *out = ctx;
    return GS_OK;
}

extern "C" void gs_context_destroy(GsContext *ctx) {
    if (!ctx) return;
    cudaDeviceSynchronize();
    ctx->per_gaussian.release();
    ctx->sort.release();
    ctx->host_stage.release();
    for (auto &b : ctx->strata_tabs) b.release();
    if (ctx->copy_stream) cudaStreamDestroy(ctx->copy_stream);
    if (ctx->aux_stream) cudaStreamDestroy(ctx->aux_stream);
    if (ctx->ev_alloc) cudaEventDestroy(ctx->ev_alloc);
    if (ctx->ev_colour) cudaEventDestroy(ctx->ev_colour);
    for (cudaEvent_t ev : ctx->feed_ev)
        if (ev) cudaEventDestroy(ev);
    if (ctx->ev_pre) cudaEventDestroy(ctx->ev_pre);
    if (ctx->ev_info) cudaEventDestroy(ctx->ev_info);
    if (ctx->h_word) cudaFreeHost(ctx->h_word);
    if (ctx->pool) cudaMemPoolDestroy(ctx->pool);  // outstanding GsSaved blocks are returned when they are freed
    if (ctx->profiling)
        for (auto &e : ctx->ev) {
            if (e[0]) cudaEventDestroy(e[0]);
            if (e[1]) cudaEventDestroy(e[1]);
        }
    delete ctx;
}

extern "C" int gs_context_trim(GsContext *ctx) {
    if (!ctx) return gs_set_error(GS_ERR_INVALID, "null context");
    GS_CUDA_OK(cudaMemPoolTrimTo(ctx->pool, 0));
    return GS_OK;
}

namespace {
// Memory policy of the context's private pool (DESIGN.md 4): freed blocks stay cached; every 256 calls the pool is
// trimmed when it holds more than twice the high-water mark of what those calls had handed out at any one time.
void pool_follow(GsContext *ctx) {
    if (++ctx->calls_since_peak_reset < 256) return;
    ctx->calls_since_peak_reset = 0;
    uint64_t used_high = 0, reserved = 0, zero = 0;
    cudaMemPoolGetAttribute(ctx->pool, cudaMemPoolAttrUsedMemHigh, &used_high);
    cudaMemPoolGetAttribute(ctx->pool, cudaMemPoolAttrReservedMemCurrent, &reserved);
    if (reserved > 2 * used_high + ((uint64_t)64 << 20)) cudaMemPoolTrimTo(ctx->pool, used_high + (used_high >> 2));
    cudaMemPoolSetAttribute(ctx->pool, cudaMemPoolAttrUsedMemHigh, &zero);
}
}  // namespace

extern "C" int gs_set_profiling(GsContext *ctx, int enabled) {
    if (!ctx) return gs_set_error(GS_ERR_INVALID, "null context");
    if (enabled && !ctx->ev[0][0]) {
        for (int s = 0; s < GS_NUM_STAGES; s++) {
            GS_CUDA_OK(cudaEventCreate(&ctx->ev[s][0]));
            GS_CUDA_OK(cudaEventCreate(&ctx->ev[s][1]));
        }
    }
    ctx->profiling = enabled != 0;
    return GS_OK;
}

extern "C" int gs_get_stage_ms(GsContext *ctx, float *ms) {
    if (!ctx || !ms) return gs_set_error(GS_ERR_INVALID, "null argument");
    for (int s = 0; s < GS_NUM_STAGES; s++) {
        ms[s] = 0.f;
        if (ctx->ev_valid[s]) {
            GS_CUDA_OK(cudaEventSynchronize(ctx->ev[s][1]));
            GS_CUDA_OK(cudaEventElapsedTime(&ms[s], ctx->ev[s][0], ctx->ev[s][1]));
        }
    }
    return GS_OK;
}

extern "C" int gs_get_stats(const GsContext *ctx, GsStats *out) {
    if (!ctx || !out) return gs_set_error(GS_ERR_INVALID, "null argument");
    *out = ctx->stats;
    out->scratch_bytes = (int64_t)(ctx->per_gaussian.bytes + ctx->sort.bytes + ctx->host_stage.bytes);
    uint64_t reserved = 0, used = 0;
    if (ctx->pool) {
        cudaMemPoolGetAttribute(ctx->pool, cudaMemPoolAttrReservedMemCurrent, &reserved);
        cudaMemPoolGetAttribute(ctx->pool, cudaMemPoolAttrUsedMemCurrent, &used);
    }
    out->pool_reserved_bytes = (int64_t)reserved;
    out->pool_used_bytes = (int64_t)used;
    return GS_OK;
}

extern "C" void gs_saved_free(GsContext *ctx, GsSaved *saved, void *stream) {
    (void)ctx;
    if (!saved) return;
    if (saved->ws_base) {   // gs_forward_sync_free: the planes belong to the caller's workspace
        delete saved;
        return;
    }
    if (saved->point_list) cudaFreeAsync(saved->point_list, static_cast<cudaStream_t>(stream));
    if (saved->base) cudaFreeAsync(saved->base, static_cast<cudaStream_t>(stream));
    delete saved;
}

namespace {
// gs_render_host's per-call feed of the forward (null for device-resident inputs)
struct HostFeed {
    bool sh_zero_copy;   // in->shs is the device alias of the caller's pinned buffer (preprocess pulls it over PCIe)
    // the SH block arrives in `chunks` pieces on the copy stream, piece k (Gaussians [begin[k], begin[k+1])) complete
    // once ctx->feed_ev[k] has fired: preprocess runs piece by piece behind them (DESIGN.md 5.6)
    int chunks, begin[GsContext::FEED_MAX + 1];
    void *radii_dst;     // host buffer the radii ([V*P] int32) are copied to on the copy stream as soon as they are final
};

#define FWD_OK(call) do { const int rc_ = (call); if (rc_ != GS_OK) return rc_; } while (0)
#define FWD_CUDA(call, what) \
    do { const cudaError_t e_ = (call); if (e_ != cudaSuccess) return gs_set_cuda_error(e_, what, __FILE__, __LINE__); } while (0)

// One forward call: what its speculative attempt and its exact path share, and what they leave for the commit.
struct FwdCall {
    GsContext *ctx;
    DevCfg c;
    DevInputs di;
    const GsOutputs *out;
    float *alpha;                         // gs_forward_ex / gs_render_host_ex: accumulated opacity [V*H*W], else null
    cudaStream_t st;
    const HostFeed *feed;
    void *radii_dst; size_t radii_bytes;  // gs_render_host: host destination of the radii
    uint32_t tuning;
    DepthMode dm;                         // what the depth channel composites (launch_preprocess: rec2.w = f(z))
    int pre_variant, composite_variant;   // launch_preprocess / launch_composite_fwd variants
    bool split_colour, merge_sort;        // k_sh_colour on the aux stream; GS_TUNE_STRATA_MERGE_SORT
    // scratch: rects[n] | counters | cursors | verdict words | sub-bucket offsets | tile_start | tile_n
    ushort4 *rects;
    uint32_t *tile_counts, *cursor, *verdict_acc, *sub_offsets, *tile_start, *tile_n;
    size_t ctr_bytes;
    GsSaved *s;
    bool colour_pending;   // k_sh_colour is (or may still be) writing into s->rec1 / s->rec2 on the aux stream
    LazyStrata lazy;       // speculative call with lazy strata: what the compositor needs to sort the skipped strata
    int64_t D;
    size_t list_bytes;
    int start_colour();
    int speculate(SpecState &spec, const BinShape &shape, const BinPlan &plan, GrowBuf &tabs, bool *committed);
    int exact(SpecState &spec, const BinShape &shape, GrowBuf &tabs);
    size_t scratch_layout(unsigned char *base) {
        size_t off = 0;
        const size_t n = (size_t)c.V * c.P, nvt = (size_t)c.V * c.ntiles;
        auto take = [&](size_t bytes) {
            unsigned char *p = base ? base + off : nullptr;
            off += align256(bytes);
            return reinterpret_cast<uint32_t *>(p);
        };
        ctr_bytes = align256(bin_counter_bytes(c));
        rects = reinterpret_cast<ushort4 *>(take(n * 8));
        tile_counts = take(ctr_bytes);
        cursor = take(ctr_bytes);
        verdict_acc = take(256);  // directly behind the cursors: one memset clears both
        sub_offsets = take(nvt * BIN_SUB * 4);
        tile_start = take(nvt * 4);
        tile_n = take(nvt * 4);
        return off;
    }

    int fail(int code) {
        if (colour_pending) cudaStreamWaitEvent(st, ctx->ev_colour, 0);   // the free below is ordered on `st`
        gs_saved_free(ctx, s, st);
        return code;
    }
    // the tile-instance list lives in its own stream-ordered allocation (s->point_list stays null when it fails)
    cudaError_t alloc_list(size_t bytes) {
        void *p = nullptr;
        const cudaError_t e = cudaMallocFromPoolAsync(&p, bytes, ctx->pool, st);
        if (e == cudaSuccess) s->point_list = static_cast<uint32_t *>(p);
        list_bytes = bytes;
        return e;
    }
    template <class F> int timed(int stage, F launch) {
        StageTimer t(ctx, stage, st);
        return launch();
    }
    // the compositor needs the colour words: from here on `st` itself is ordered behind the colour kernel
    int composite() {
        if (colour_pending) {
            colour_pending = false;
            FWD_CUDA(cudaStreamWaitEvent(st, ctx->ev_colour, 0), "cudaStreamWaitEvent(colour)");
        }
        return timed(GS_STAGE_COMPOSITE, [&] { return launch_composite_fwd(c, *s, out->color, out->depth, st, composite_variant, alpha, lazy); });
    }
};

// gs_render_host's split pipeline: k_sh_colour writes the colour words of s->rec1 / s->rec2 on the aux stream, behind
// everything enqueued on `st` so far (the caller's uploads of means and cameras, the allocation of the records)
int FwdCall::start_colour() {
    const char *setup = "split colour pipeline setup";
    if (!ctx->aux_stream) FWD_CUDA(cudaStreamCreateWithFlags(&ctx->aux_stream, cudaStreamNonBlocking), setup);
    if (!ctx->ev_alloc) FWD_CUDA(cudaEventCreateWithFlags(&ctx->ev_alloc, cudaEventDisableTiming), setup);
    if (!ctx->ev_colour) FWD_CUDA(cudaEventCreateWithFlags(&ctx->ev_colour, cudaEventDisableTiming), setup);
    FWD_CUDA(cudaEventRecord(ctx->ev_alloc, st), setup);
    FWD_CUDA(cudaStreamWaitEvent(ctx->aux_stream, ctx->ev_alloc, 0), setup);
    {
        StageTimer t(ctx, GS_STAGE_SH_COLOUR, ctx->aux_stream);
        FWD_OK(launch_sh_colour(c, di, s->rec1, s->rec2, nullptr, ctx->aux_stream));
    }
    const cudaError_t e = cudaEventRecord(ctx->ev_colour, ctx->aux_stream);
    if (e != cudaSuccess) cudaStreamSynchronize(ctx->aux_stream);   // the caller frees the records
    FWD_CUDA(e, "cudaEventRecord(colour)");
    colour_pending = true;
    return GS_OK;
}

// Speculative attempt (DESIGN.md 5.2): the host reads the verdict only after the tile sort and the compositor have been
// enqueued.  *committed = false after an overflow: the results are discarded and the call is redone on the exact path.
int FwdCall::speculate(SpecState &spec, const BinShape &shape, const BinPlan &plan, GrowBuf &tabs, bool *committed) {
    const size_t slots = (size_t)c.V * c.ntiles * BIN_SUB;
    const float *strata_tab = plan.read_tab < 0 ? nullptr : static_cast<float *>(tabs.p) + (size_t)plan.read_tab * slots;
    float *strata_next = plan.write_tab < 0 ? nullptr : static_cast<float *>(tabs.p) + (size_t)plan.write_tab * slots;
    FWD_OK(ctx->sort.reserve(slots * plan.sub_cap * 8, 1.0, ctx->pool, st));
    FWD_CUDA(alloc_list(slots * plan.sub_cap * 4), "cudaMallocAsync(point_list)");
    FWD_CUDA(cudaMemsetAsync(cursor, 0, ctr_bytes + 256, st), "cudaMemsetAsync(cursors)");
    const PreEmit emit{plan.fused_emit ? cursor : nullptr, static_cast<uint64_t *>(ctx->sort.p), plan.sub_cap,
                       strata_tab, plan.per_tile};
    {
        StageTimer t(ctx, GS_STAGE_PREPROCESS, st);
        const int pieces = feed ? feed->chunks : 0;
        for (int k = 0; k < (pieces ? pieces : 1); k++) {
            if (pieces) FWD_CUDA(cudaStreamWaitEvent(st, ctx->feed_ev[k], 0), "cudaStreamWaitEvent(feed)");
            FWD_OK(launch_preprocess(c, di, s->rec0, s->rec1, s->rec2, s->meta, out->radii, rects, emit, st,
                                     pieces ? feed->begin[k] : 0, pieces ? feed->begin[k + 1] : -1, pre_variant, dm));
        }
    }
    if (!plan.fused_emit)
        FWD_OK(timed(GS_STAGE_BIN_EMIT, [&] {
            return bin_emit_fast(c, 1, s->rec0, s->rec1, s->rec2, rects, nullptr, plan.sub_cap, strata_tab,
                                 plan.per_tile, cursor, ctx->sort.p, st);
        }));
    // gs_render_host: the radii leave as soon as they are final; on the stratified path only after the sort, whose verdict
    // store into host memory would otherwise queue behind the 16 MB of radii on the PCIe link
    auto start_radii_copy = [&]() -> int {
        if (!radii_dst) return GS_OK;
        const char *what = "early radii copy";
        if (!ctx->ev_pre) FWD_CUDA(cudaEventCreateWithFlags(&ctx->ev_pre, cudaEventDisableTiming), what);
        FWD_CUDA(cudaEventRecord(ctx->ev_pre, st), what);
        FWD_CUDA(cudaStreamWaitEvent(ctx->copy_stream, ctx->ev_pre, 0), what);
        FWD_CUDA(cudaMemcpyAsync(radii_dst, out->radii, radii_bytes, cudaMemcpyDeviceToHost, ctx->copy_stream), what);
        return GS_OK;
    };
    if (!plan.strata) FWD_OK(start_radii_copy());
    // the verdict goes straight into mapped pinned memory, marked by ev_info: from k_spec_check on the whole-tile path,
    // from the stratum sort's last CTA on the stratified path
    if (!ctx->ev_info) FWD_CUDA(cudaEventCreateWithFlags(&ctx->ev_info, cudaEventDisableTiming), "cudaEventCreate");
    if (!plan.strata) {
        FWD_OK(timed(GS_STAGE_BIN_SCAN, [&] { return bin_spec_check(c, plan.sub_cap, spec.tile_limit, cursor, ctx->d_word, st); }));
        FWD_CUDA(cudaEventRecord(ctx->ev_info, st), "read back binning info");
    }
    {
        StageTimer t(ctx, GS_STAGE_BIN_SORT, st);
        if (plan.strata) {
            // lazy strata: one table per shape is enough -- this call's sort reads it before its compositor rewrites it
            uint8_t *need = plan.lazy_strata ? bin_need_table(c, tabs.p) : nullptr;
            if (plan.reset_need)
                FWD_CUDA(cudaMemsetAsync(need, BIN_SUB, (size_t)c.V * c.ntiles, st), "cudaMemsetAsync(need)");
            if (need) lazy = LazyStrata{cursor, static_cast<const uint64_t *>(ctx->sort.p), plan.sub_cap, need};
            FWD_OK(bin_sort_strata(c, plan.sub_cap, cursor, ctx->sort.p, s->point_list, s->ranges, verdict_acc,
                                   ctx->d_word, st, merge_sort, s->rec2, strata_next, need));
            FWD_CUDA(cudaEventRecord(ctx->ev_info, st), "read back binning info");
            FWD_OK(start_radii_copy());
        } else {
            FWD_OK(bin_sort_spec(c, plan.sub_cap, spec.tile_limit, cursor, ctx->sort.p, s->point_list, s->ranges, st));
        }
    }
    FWD_OK(composite());
    FWD_CUDA(cudaEventSynchronize(ctx->ev_info), "cudaEventSynchronize");  // the one host sync of the forward (verification only)
    bool release_sort;
    *committed = learn_speculative(spec, shape, plan, ctx->h_word, ctx->sort.bytes, tuning, &release_sort);
    if (release_sort) {   // stream-ordered
        ctx->sort.pooled ? cudaFreeAsync(ctx->sort.p, st) : cudaFree(ctx->sort.p);
        ctx->sort = GrowBuf{};
    }
    if (*committed) {
        D = (int64_t)ctx->h_word[0];
        // k_preprocess, [k_sh_colour,] [k_emit_buckets,] [k_spec_check,] tile sort, k_composite_fwd
        ctx->stats.kernel_launches = (plan.strata ? 3 : 4) + (plan.fused_emit ? 0 : 1) + (split_colour ? 1 : 0);
        ctx->stats.max_tile_list = (int32_t)ctx->h_word[1];
        ctx->stats.speculative = plan.strata ? 2 : 1;
        return GS_OK;
    }
    ctx->stats.overflow_redos++;
    if (radii_dst) cudaStreamSynchronize(ctx->copy_stream);
    cudaFreeAsync(s->point_list, st);
    s->point_list = nullptr;
    for (bool &valid : ctx->ev_valid) valid = false;
    return GS_OK;
}

// Exact path: count, scan, the one host sync, emit, sort; then boundaries for the coming speculative calls.
int FwdCall::exact(SpecState &spec, const BinShape &shape, GrowBuf &tabs) {
    ctx->stats.speculative = 0;
    {
        StageTimer t(ctx, GS_STAGE_PREPROCESS, st);
        FWD_CUDA(cudaMemsetAsync(tile_counts, 0, bin_counter_bytes(c), st), "cudaMemsetAsync(tile_counts)");
        const PreEmit emit{tile_counts, nullptr, 0, nullptr, 0};  // sub-bucket = index % BIN_SUB
        for (int k = 0; feed && k < feed->chunks; k++)  // gs_render_host: every piece of the SH block must have landed
            FWD_CUDA(cudaStreamWaitEvent(st, ctx->feed_ev[k], 0), "cudaStreamWaitEvent(feed)");
        FWD_OK(launch_preprocess(c, di, s->rec0, s->rec1, s->rec2, s->meta, out->radii, rects, emit, st, 0, -1, pre_variant, dm));
        ctx->stats.kernel_launches += (c.P > 0);
    }
    uint32_t max_count;   // longest tile list
    bool fast;            // shared-memory sort
    int learn;            // boundaries to learn
    {
        StageTimer t(ctx, GS_STAGE_BIN_SCAN, st);
        // the scan kernel stores its three result words straight into pinned host memory (no copy-engine hop)
        FWD_OK(bin_tile_scan(c, tile_counts, sub_offsets, tile_start, tile_n, ctx->d_word, st));
        FWD_CUDA(cudaStreamSynchronize(st), "read back num_rendered");
        D = (int64_t)ctx->h_word[0];
        max_count = ctx->h_word[1];
        fast = bin_fits_fast_path(max_count) && !(tuning & GS_TUNE_FORCE_RADIX_BINNING);
        learn = learn_exact(spec, shape, (size_t)c.V * c.P, max_count, ctx->h_word[2], fast, tuning);
        if (radii_dst)  // preprocess has completed: radii can leave now
            FWD_CUDA(cudaMemcpyAsync(radii_dst, out->radii, radii_bytes, cudaMemcpyDeviceToHost, ctx->copy_stream),
                     "cudaMemcpyAsync(radii)");
        if (D > 0x7fffffffll) return gs_set_error(GS_ERR_OVERFLOW, "more than 2^31-1 tile instances");
        FWD_CUDA(alloc_list((size_t)(D > 0 ? D : 1) * 4), "cudaMallocAsync(point_list)");
    }
    FWD_OK(ctx->sort.reserve(bin_scratch_bytes(c, D, fast), 1.25, ctx->pool, st));
    FWD_OK(timed(GS_STAGE_BIN_EMIT, [&] {
        return fast ? bin_emit_fast(c, D, s->rec0, s->rec1, s->rec2, rects, sub_offsets, 0, nullptr, 0,
                                    cursor, ctx->sort.p, st)
                    : bin_sort_fallback(c, D, s->rec0, s->rec1, s->rec2, rects, ctx->sort.p, ctx->sort.bytes,
                                        s->point_list, s->ranges, st);
    }));
    if (fast)
        FWD_OK(timed(GS_STAGE_BIN_SORT, [&] {
            return bin_sort_fast(c, max_count, tile_start, tile_n, ctx->sort.p, s->point_list, s->ranges, st);
        }));
    ctx->stats.kernel_launches += 1 + (D > 0 ? 1 : 0) + 1;  // scan, emit, tile sort (fallback: 3 + CUB's)
    ctx->stats.max_tile_list = (int32_t)max_count;
    FWD_OK(composite());
    ctx->stats.kernel_launches += 1;
    if (learn != LEARN_NONE) {
        FWD_OK(tabs.reserve(bin_strata_bytes(c), 1.0, ctx->pool, st));
        FWD_OK(learn == LEARN_PER_TILE ? bin_learn_tile_strata(c, s->point_list, s->ranges, s->rec2, static_cast<float *>(tabs.p), st)
                                       : bin_learn_strata(c, rects, s->rec2, tabs.p, st));
        start_trial(spec);
        ctx->stats.kernel_launches += learn == LEARN_PER_TILE ? 1 : 2;  // k_tile_octiles | k_depth_hist, k_strata_from_hist
    }
    return GS_OK;
}
#undef FWD_OK
#undef FWD_CUDA

int forward(GsContext *ctx, const GsConfig *cfg, const GsInputs *in, const GsOutputs *out, GsSaved **saved_out,
            cudaStream_t st, const HostFeed *feed, float *alpha) {
    if (saved_out) *saved_out = nullptr;
    if (!ctx || !out) return gs_set_error(GS_ERR_INVALID, "null context/outputs");
    int rc = validate(cfg, in);
    if (rc != GS_OK) return rc;
    if (!out->color || (cfg->P > 0 && !out->radii)) return gs_set_error(GS_ERR_INVALID, "color/radii outputs missing");
    if ((cfg->flags & GS_FLAG_DEPTH) && !out->depth) return gs_set_error(GS_ERR_INVALID, "GS_FLAG_DEPTH needs out->depth");
    if ((rc = validate_depth_mode(cfg)) != GS_OK) return rc;
    if ((rc = validate_antialias(cfg->flags, cfg->tuning, AA_FWD_KNOBS)) != GS_OK) return rc;
    FwdCall f{};
    f.ctx = ctx; f.c = make_dev_cfg(cfg); f.di = make_dev_inputs(in); f.out = out; f.alpha = alpha; f.st = st; f.feed = feed;
    const DevCfg &c = f.c;
    const size_t n = (size_t)c.V * c.P;
    const BinShape shape{c.V, c.ntiles, c.P, c.S};
    const int slot = pick_slot(ctx->slots, GsContext::SHAPE_SLOTS, ctx->use_counter, shape);
    SpecState &spec = ctx->slots[slot].spec;
    GrowBuf &tabs = ctx->strata_tabs[slot];
    const BinPlan plan = plan_binning(spec, shape, n, tabs.p != nullptr, cfg->tuning);

    // kernel variants (gs_render_host with a pinned SH block: geometry-only preprocess, colours in k_sh_colour)
    f.tuning = cfg->tuning;
    f.dm = DepthMode{cfg->depth_mode, cfg->depth_near_far};
    const bool zero_copy = feed && feed->sh_zero_copy;
    f.split_colour = zero_copy && !(f.tuning & GS_TUNE_NO_SPLIT_COLOUR) && n > 0 && sh_colour_supported(c, f.di);
    f.pre_variant = ((f.tuning & GS_TUNE_PRE_OCC6) ? 1 : 0) | (((f.tuning & GS_TUNE_PRE_SH_RAW16) || zero_copy) ? 2 : 0) |
                    (f.split_colour ? 4 : 0);
    f.composite_variant = (f.tuning & GS_TUNE_FWD_WS) ? 2 : 0;
    f.merge_sort = (f.tuning & GS_TUNE_STRATA_MERGE_SORT) != 0;
    f.radii_dst = feed && ctx->copy_stream ? feed->radii_dst : nullptr;
    f.radii_bytes = n * 4;
    for (bool &valid : ctx->ev_valid) valid = false;
    ctx->stats.kernel_launches = 0;

    rc = ctx->per_gaussian.reserve(f.scratch_layout(nullptr), 1.0, ctx->pool, st);
    if (rc != GS_OK) return rc;
    f.scratch_layout(static_cast<unsigned char *>(ctx->per_gaussian.p));
    // ---- saved state: geometry / image planes now, the tile-instance list once its length is known ----
    GsSaved *s = f.s = new (std::nothrow) GsSaved();   // value-initialised: all zero
    if (!s) return gs_set_error(GS_ERR_OOM, "host allocation failed");
    s->bytes = saved_layout(s, c, nullptr);
    const cudaError_t e = cudaMallocFromPoolAsync(&s->base, s->bytes, ctx->pool, st);
    if (e != cudaSuccess) {
        delete s;
        return gs_set_cuda_error(e, "cudaMallocAsync(saved)", __FILE__, __LINE__);
    }
    saved_layout(s, c, static_cast<unsigned char *>(s->base));
    s->depth_mode = cfg->depth_mode;   // (the compositor reads it)
    if (f.split_colour && (rc = f.start_colour()) != GS_OK) return f.fail(rc);

    bool committed = false;
    if (plan.speculate && (rc = f.speculate(spec, shape, plan, tabs, &committed)) != GS_OK) return f.fail(rc);
    if (!committed && (rc = f.exact(spec, shape, tabs)) != GS_OK) return f.fail(rc);

    s->D = f.D;
    s->P = c.P; s->S = c.S; s->V = c.V; s->H = c.H; s->W = c.W;
    s->flags = c.flags;
    s->has_sh = in->shs != nullptr;
    s->has_scales = in->scales != nullptr;
    ctx->stats.num_rendered = f.D;
    ctx->stats.num_visible = -1;
    ctx->stats.saved_bytes = (int64_t)(s->bytes + f.list_bytes);
    pool_follow(ctx);
    if (saved_out) *saved_out = s;
    else gs_saved_free(ctx, s, st);
    return GS_OK;
}
}  // namespace

extern "C" int gs_forward(GsContext *ctx, const GsConfig *cfg, const GsInputs *in, const GsOutputs *out,
                          GsSaved **saved_out, void *stream) {
    return forward(ctx, cfg, in, out, saved_out, static_cast<cudaStream_t>(stream), nullptr, nullptr);
}

extern "C" int gs_forward_ex(GsContext *ctx, const GsConfig *cfg, const GsInputs *in, const GsOutputs *out,
                             const GsAlpha *alpha, GsSaved **saved_out, void *stream) {
    if (saved_out) *saved_out = nullptr;
    if (!alpha) return gs_set_error(GS_ERR_INVALID, "null alpha request");
    if (!alpha->alpha) return gs_set_error(GS_ERR_INVALID, "gs_forward_ex needs alpha->alpha (gs_forward renders without it)");
    return forward(ctx, cfg, in, out, saved_out, static_cast<cudaStream_t>(stream), nullptr, alpha->alpha);
}

namespace {
// What gs_backward_sync_free hands the backward: the workspace's accumulator region (validated to be large enough for
// this call) and its status words.
struct SfBwd {
    unsigned char *scratch;
    const uint32_t *status;
};

int backward(GsContext *ctx, const GsConfig *cfg, const GsInputs *in, const GsSaved *saved, const GsOutGrads *gout,
             const float *dL_dalpha, const GsInGrads *gin, void *stream, const GsCameraGrads *cam = nullptr,
             float *dL_dtanfov = nullptr, const SfBwd *sf = nullptr) {
    if (!ctx || !saved || !gout || !gin) return gs_set_error(GS_ERR_INVALID, "null argument");
    int rc = validate(cfg, in);
    if (rc != GS_OK) return rc;
    if (!gout->dL_dcolor) return gs_set_error(GS_ERR_INVALID, "dL_dcolor missing");
    if ((rc = validate_antialias(cfg->flags, cfg->tuning, AA_BWD_KNOBS)) != GS_OK) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    DevCfg c = make_dev_cfg(cfg);
    if (saved->P != c.P || saved->V != c.V || saved->S != c.S || saved->H != c.H || saved->W != c.W)
        return gs_set_error(GS_ERR_INVALID, "saved state does not match the configuration");
    if (!sf && saved->ws_base)
        return gs_set_error(GS_ERR_INVALID, "the saved state of gs_forward_sync_free needs gs_backward_sync_free");
    c.flags = saved->flags;   // (GS_FLAG_ANTIALIAS included: the backward differentiates what its forward drew)
    if ((rc = validate_antialias(c.flags, cfg->tuning, AA_BWD_KNOBS)) != GS_OK) return rc;
    if (cam && gin->dL_dviewmatrix_z)
        return gs_set_error(GS_ERR_INVALID, "dL_dviewmatrix_z and GsCameraGrads in one call: the camera gradient already "
                                            "contains the depth channel's z column");
    if (cam && (cfg->tuning & GS_TUNE_PBWD_2PHASE))
        return gs_set_error(GS_ERR_INVALID, "GS_TUNE_PBWD_2PHASE has no camera-gradient kernel (GsCameraGrads)");
    if (gin->dL_dviewmatrix_z && !(c.flags & GS_FLAG_DEPTH))
        return gs_set_error(GS_ERR_INVALID, "dL_dviewmatrix_z needs a forward with GS_FLAG_DEPTH");
    // the forward's depth mode, with this call's near / far
    const DepthMode dm{saved->depth_mode, cfg->depth_near_far};
    if ((dm.mode == GS_DEPTH_RELATIVE_DISPARITY || dm.mode == GS_DEPTH_LOG) && !dm.near_far)
        return gs_set_error(GS_ERR_INVALID, "the forward's depth_mode needs depth_near_far in the backward too");
    const bool det = (cfg->flags & GS_FLAG_DETERMINISTIC) != 0;
    if (det) {
        if (cfg->tuning & GS_TUNE_BWD_V1)
            return gs_set_error(GS_ERR_INVALID, "GS_FLAG_DETERMINISTIC: the round-1 backward kernel (GS_TUNE_BWD_V1) has no deterministic mode");
        // every 8x4 pixel block of a view adds at most one term to an accumulator: the limbs' headroom bounds their number
        if ((int64_t)((c.H + 3) / 4) * ((c.W + 7) / 8) >= GS_DET_MAX_TERMS)
            return gs_set_error(GS_ERR_INVALID, "GS_FLAG_DETERMINISTIC: the frame has 2^21 or more 8x4 pixel blocks "
                                                "(ceil(H/4) * ceil(W/8) must stay below 2097152)");
    }
    const DevInputs di = make_dev_inputs(in);
    // the view-matrix gradient is written: zero it, then the kernels accumulate into it (nothing when there is no
    // incoming depth gradient: it stays zero and the default kernels run)
    GsInGrads g = *gin;
    if (g.dL_dviewmatrix_z) {
        GS_CUDA_OK(cudaMemsetAsync(g.dL_dviewmatrix_z, 0, (size_t)c.V * 4 * sizeof(float), st));
        if (!gout->dL_ddepth) g.dL_dviewmatrix_z = nullptr;
    }
    const size_t n = (size_t)c.V * c.P;
    if (n == 0) {
        // no pair contributes: the camera gradient is zero
        if (cam && cam->dL_dviewmatrix) GS_CUDA_OK(cudaMemsetAsync(cam->dL_dviewmatrix, 0, (size_t)c.V * 16 * 4, st));
        if (cam && cam->dL_dprojmatrix) GS_CUDA_OK(cudaMemsetAsync(cam->dL_dprojmatrix, 0, (size_t)c.V * 16 * 4, st));
        if (cam && cam->dL_dcampos) GS_CUDA_OK(cudaMemsetAsync(cam->dL_dcampos, 0, (size_t)c.V * 3 * 4, st));
        if (cam && dL_dtanfov) GS_CUDA_OK(cudaMemsetAsync(dL_dtanfov, 0, (size_t)c.V * 2 * 4, st));
        return GS_OK;
    }

    // Accumulators: n x GS_ACC_STRIDE floats; deterministic mode: n x GS_ACC_STRIDE x 3 int64 limbs + n poison masks
    // (zeroed together), then the per-warp partials of the view-matrix gradient; with the camera gradient, its per-warp
    // partials, in both modes
    const size_t acc_bytes = det ? n * (GS_ACC_STRIDE * GS_DET_LIMBS * 8 + 4) : n * GS_ACC_STRIDE * 4;
    const size_t vz_off = align256(acc_bytes);
    const size_t vz_bytes = cam ? camera_grad_scratch_bytes(c) : det ? det_view_z_bytes(c) : 0;
    unsigned char *scratch = sf ? sf->scratch : nullptr;   // (the workspace was checked against this call's needs)
    if (!sf) {
        rc = ctx->per_gaussian.reserve(vz_bytes ? vz_off + vz_bytes : acc_bytes, 1.0, ctx->pool, st);
        if (rc != GS_OK) return rc;
        scratch = static_cast<unsigned char *>(ctx->per_gaussian.p);
    }
    float *acc = reinterpret_cast<float *>(scratch);
    DetAcc da{};
    if (cam) da.view_z = reinterpret_cast<float *>(scratch + vz_off);
    if (det) {
        unsigned char *base = scratch;
        da.acc = reinterpret_cast<unsigned long long *>(base);
        da.poison = reinterpret_cast<uint32_t *>(base + n * GS_ACC_STRIDE * GS_DET_LIMBS * 8);
        da.view_z = reinterpret_cast<float *>(base + vz_off);
        acc = nullptr;
    }
    {
        StageTimer t(ctx, GS_STAGE_COMPOSITE_BWD, st);
        GS_CUDA_OK(cudaMemsetAsync(scratch, 0, acc_bytes, st));
        rc = launch_composite_bwd(c, *saved, gout->dL_dcolor, gout->dL_ddepth, acc, st, (cfg->tuning & GS_TUNE_BWD_V1) ? 1 : ((cfg->tuning & GS_TUNE_BWD_OCC4) ? 2 : 0), da,
                                  dL_dalpha);
        if (rc != GS_OK) return rc;
    }
    {
        StageTimer t(ctx, GS_STAGE_PREPROCESS_BWD, st);
        rc = launch_preprocess_bwd(c, di, *saved, acc, g, st, (cfg->tuning & GS_TUNE_PBWD_2PHASE) ? 1 : 0, da, dm, cam,
                                   dL_dtanfov);
        if (rc != GS_OK) return rc;
    }
    ctx->stats.kernel_launches += 2;  // k_composite_bwd, k_preprocess_bwd
    if (det && g.dL_dviewmatrix_z) ctx->stats.kernel_launches += 1;  // k_view_z_finalize
    if (cam) ctx->stats.kernel_launches += 1;                        // k_camera_finalize
    if (sf) {
        // the backward of a forward that exceeded its workspace: NaN into every gradient it writes
        const size_t sp = (size_t)c.S * c.P, vp = (size_t)c.V * c.P, V = (size_t)c.V;
        SfPoison grads{};
        grads.add(gin->dL_dmeans3D, sp * 3);
        grads.add(gin->dL_dmeans2D, vp * 3);
        grads.add(gin->dL_dshs, sp * c.M * 3);
        grads.add(gin->dL_dcolors, vp * 3);
        grads.add(gin->dL_dopacities, sp);
        grads.add(gin->dL_dscales, sp * 3);
        grads.add(gin->dL_drotations, sp * 4);
        grads.add(gin->dL_dcov3D, sp * 6);
        grads.add(gin->dL_dviewmatrix_z, V * 4);
        if (cam) {
            grads.add(cam->dL_dviewmatrix, V * 16);
            grads.add(cam->dL_dprojmatrix, V * 16);
            grads.add(cam->dL_dcampos, V * 3);
            grads.add(dL_dtanfov, V * 2);
        }
        if ((rc = sf_poison_if_exceeded(sf->status, grads, st)) != GS_OK) return rc;
        ctx->stats.kernel_launches += 1;   // k_sf_poison
    }
    return GS_OK;
}
}  // namespace

extern "C" int gs_backward(GsContext *ctx, const GsConfig *cfg, const GsInputs *in, const GsSaved *saved,
                           const GsOutGrads *gout, const GsInGrads *gin, void *stream) {
    return backward(ctx, cfg, in, saved, gout, nullptr, gin, stream);
}

extern "C" int gs_backward_ex(GsContext *ctx, const GsConfig *cfg, const GsInputs *in, const GsSaved *saved,
                              const GsOutGrads *gout, const GsAlpha *alpha, const GsInGrads *gin, void *stream) {
    if (!alpha) return gs_set_error(GS_ERR_INVALID, "null alpha request");
    return backward(ctx, cfg, in, saved, gout, alpha->dL_dalpha, gin, stream);
}

extern "C" int gs_backward_cam(GsContext *ctx, const GsConfig *cfg, const GsInputs *in, const GsSaved *saved,
                               const GsOutGrads *gout, const GsAlpha *alpha, const GsInGrads *gin, const GsCameraGrads *cam,
                               void *stream) {
    if (!cam) return gs_set_error(GS_ERR_INVALID, "null camera-gradient request");
    return backward(ctx, cfg, in, saved, gout, alpha ? alpha->dL_dalpha : nullptr, gin, stream, cam);
}

extern "C" int gs_backward_cam_tanfov(GsContext *ctx, const GsConfig *cfg, const GsInputs *in, const GsSaved *saved,
                                      const GsOutGrads *gout, const GsAlpha *alpha, const GsInGrads *gin,
                                      const GsCameraGrads *cam, float *dL_dtanfov, void *stream) {
    if (!cam) return gs_set_error(GS_ERR_INVALID, "null camera-gradient request");
    return backward(ctx, cfg, in, saved, gout, alpha ? alpha->dL_dalpha : nullptr, gin, stream, cam, dL_dtanfov);
}

// ---------------------------------------------------------------------------------------------------------
// sync-free forward and backward (DESIGN.md 5.18): every buffer in the caller's workspace, every size decision on
// the device
// ---------------------------------------------------------------------------------------------------------
namespace {
// Workspace layout: status words | saved planes | point_list[capacity] | scratch.  The scratch holds the forward's
// binning buffers or, once the forward's kernels have run, the backward's accumulators.
struct SfLayout {
    GsSaved saved;       // plane pointers; saved.point_list = the workspace's list
    size_t saved_bytes;  // planes + list
    SyncFreeBins bins;
    unsigned char *scratch;
    size_t bytes;
};

size_t sf_backward_bytes(const DevCfg &c, uint32_t needs) {
    const size_t n = (size_t)c.V * c.P;
    const bool det = (needs & GS_SYNC_FREE_DETERMINISTIC) != 0;
    const size_t acc = det ? n * (GS_ACC_STRIDE * GS_DET_LIMBS * 8 + 4) : n * GS_ACC_STRIDE * 4;
    const size_t cam = (needs & GS_SYNC_FREE_CAMERA_GRAD) ? camera_grad_scratch_bytes(c) : 0;
    const size_t vz = det ? det_view_z_bytes(c) : 0;
    return align256(acc) + (cam > vz ? cam : vz);
}

size_t sf_layout(SfLayout *L, const DevCfg &c, size_t capacity, uint32_t needs, unsigned char *base) {
    size_t off = 0;
    const size_t n = (size_t)c.V * c.P, nvt = (size_t)c.V * c.ntiles, cap = capacity > 0 ? capacity : 1;
    auto take = [&](size_t bytes) {
        unsigned char *p = base ? base + off : nullptr;
        off += align256(bytes);
        return p;
    };
    *L = SfLayout{};
    L->bins.capacity = (uint32_t)capacity;
    L->bins.status = reinterpret_cast<uint32_t *>(take(256));
    const size_t planes = saved_layout(&L->saved, c, base ? base + off : nullptr);
    off += planes;
    L->saved.point_list = reinterpret_cast<uint32_t *>(take(cap * 4));
    L->bins.point_list = L->saved.point_list;
    L->bins.ranges = L->saved.ranges;
    L->saved_bytes = planes + align256(cap * 4);
    L->scratch = base ? base + off : nullptr;
    const size_t scratch_off = off;
    const size_t ctr = bin_counter_bytes(c);
    L->bins.rects = reinterpret_cast<ushort4 *>(take(n * 8));
    L->bins.tile_counts = reinterpret_cast<uint32_t *>(take(ctr));
    L->bins.cursor = reinterpret_cast<uint32_t *>(take(ctr));
    L->bins.sub_offsets = reinterpret_cast<uint32_t *>(take(nvt * BIN_SUB * 4));
    L->bins.tile_start = reinterpret_cast<uint32_t *>(take(nvt * 4));
    L->bins.tile_n = reinterpret_cast<uint32_t *>(take(nvt * 4));
    L->bins.bucket = reinterpret_cast<uint64_t *>(take(cap * 8));
    L->bins.tmp = reinterpret_cast<uint64_t *>(take(cap * 8));
    const size_t bwd_end = scratch_off + sf_backward_bytes(c, needs);
    L->bytes = off > bwd_end ? off : bwd_end;
    return L->bytes;
}

// the dimensions a workspace is sized by (the pointers of cfg are not read)
int validate_dims(const GsConfig *cfg) {
    if (!cfg) return gs_set_error(GS_ERR_INVALID, "null config");
    if (cfg->P < 0 || cfg->S < 1 || cfg->V < 1 || cfg->V % cfg->S != 0)
        return gs_set_error(GS_ERR_INVALID, "need P >= 0, S >= 1, V >= 1 and V % S == 0");
    if (cfg->image_height < 1 || cfg->image_width < 1) return gs_set_error(GS_ERR_INVALID, "empty image");
    if ((int64_t)cfg->P * cfg->V > 0x7fffffffll) return gs_set_error(GS_ERR_OVERFLOW, "P*V exceeds 2^31-1");
    if ((cfg->image_width + GS_TILE - 1) / GS_TILE > 65535 || (cfg->image_height + GS_TILE - 1) / GS_TILE > 65535)
        return gs_set_error(GS_ERR_INVALID, "image too large");
    return GS_OK;
}

// the workspace against this call: aligned, a capacity the 32-bit lists can index, large enough for cfg and `needs`
int sf_check(const DevCfg &c, const GsSyncFreeWorkspace *ws, uint32_t needs, SfLayout *L) {
    if (!ws || !ws->base) return gs_set_error(GS_ERR_INVALID, "null sync-free workspace");
    if (reinterpret_cast<uintptr_t>(ws->base) & 255u) return gs_set_error(GS_ERR_INVALID, "sync-free workspace not 256-byte aligned");
    if (ws->instance_capacity < 0 || ws->instance_capacity > 0x7fffffffll)
        return gs_set_error(GS_ERR_INVALID, "instance_capacity must be in [0, 2^31-1]");
    if (ws->bytes < 0 || sf_layout(L, c, (size_t)ws->instance_capacity, needs, nullptr) > (size_t)ws->bytes)
        return gs_set_error(GS_ERR_INVALID, "sync-free workspace smaller than gs_sync_free_workspace_bytes for this "
                                            "configuration, capacity and backward (GS_SYNC_FREE_*)");
    sf_layout(L, c, (size_t)ws->instance_capacity, needs, static_cast<unsigned char *>(ws->base));
    return GS_OK;
}
}  // namespace

extern "C" int gs_sync_free_workspace_bytes(const GsConfig *cfg, int64_t instance_capacity, uint32_t needs, int64_t *bytes) {
    if (!bytes) return gs_set_error(GS_ERR_INVALID, "null bytes");
    *bytes = -1;
    int rc = validate_dims(cfg);
    if (rc != GS_OK) return rc;
    if (instance_capacity < 0 || instance_capacity > 0x7fffffffll)
        return gs_set_error(GS_ERR_INVALID, "instance_capacity must be in [0, 2^31-1]");
    if (needs & ~(uint32_t)(GS_SYNC_FREE_DETERMINISTIC | GS_SYNC_FREE_CAMERA_GRAD))
        return gs_set_error(GS_ERR_INVALID, "unknown GS_SYNC_FREE_* bit");
    SfLayout L;
    *bytes = (int64_t)sf_layout(&L, make_dev_cfg(cfg), (size_t)instance_capacity, needs, nullptr);
    return GS_OK;
}

extern "C" int gs_forward_sync_free(GsContext *ctx, const GsConfig *cfg, const GsInputs *in, const GsOutputs *out,
                                    const GsAlpha *alpha, const GsSyncFreeWorkspace *ws, GsSaved **saved_out,
                                    void *stream) {
    if (saved_out) *saved_out = nullptr;
    if (!ctx || !out) return gs_set_error(GS_ERR_INVALID, "null context/outputs");
    int rc = validate(cfg, in);
    if (rc != GS_OK) return rc;
    if (!out->color || (cfg->P > 0 && !out->radii)) return gs_set_error(GS_ERR_INVALID, "color/radii outputs missing");
    if ((cfg->flags & GS_FLAG_DEPTH) && !out->depth) return gs_set_error(GS_ERR_INVALID, "GS_FLAG_DEPTH needs out->depth");
    if (alpha && !alpha->alpha) return gs_set_error(GS_ERR_INVALID, "alpha given without alpha->alpha");
    if ((rc = validate_depth_mode(cfg)) != GS_OK) return rc;
    if ((rc = validate_antialias(cfg->flags, cfg->tuning, AA_FWD_KNOBS)) != GS_OK) return rc;
    const DevCfg c = make_dev_cfg(cfg);
    SfLayout L;
    if ((rc = sf_check(c, ws, 0, &L)) != GS_OK) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    GsSaved *s = new (std::nothrow) GsSaved(L.saved);
    if (!s) return gs_set_error(GS_ERR_OOM, "host allocation failed");
    s->base = nullptr;
    s->ws_base = ws->base;
    s->bytes = L.saved_bytes;
    s->D = -1;   // on the device only (status word SF_D)
    s->P = c.P; s->S = c.S; s->V = c.V; s->H = c.H; s->W = c.W;
    s->flags = c.flags;
    s->has_sh = in->shs != nullptr;
    s->has_scales = in->scales != nullptr;
    s->depth_mode = cfg->depth_mode;
    float *alpha_plane = alpha ? alpha->alpha : nullptr;
    const int pre_variant = ((cfg->tuning & GS_TUNE_PRE_OCC6) ? 1 : 0) | ((cfg->tuning & GS_TUNE_PRE_SH_RAW16) ? 2 : 0);
    const int composite_variant = (cfg->tuning & GS_TUNE_FWD_WS) ? 2 : 0;
    const size_t px = (size_t)c.V * c.H * c.W;
    auto run = [&]() -> int {
        GS_CUDA_OK(cudaMemsetAsync(L.bins.tile_counts, 0, bin_counter_bytes(c), st));
        const PreEmit emit{L.bins.tile_counts, nullptr, 0, nullptr, 0};  // sub-bucket = index % BIN_SUB
        int r = launch_preprocess(c, make_dev_inputs(in), s->rec0, s->rec1, s->rec2, s->meta, out->radii, L.bins.rects,
                                  emit, st, 0, -1, pre_variant, DepthMode{cfg->depth_mode, cfg->depth_near_far});
        if (r != GS_OK) return r;
        if ((r = bin_sync_free(c, L.bins, s->rec0, s->rec1, s->rec2, st)) != GS_OK) return r;
        if ((r = launch_composite_fwd(c, *s, out->color, out->depth, st, composite_variant, alpha_plane)) != GS_OK) return r;
        SfPoison planes{};
        planes.add(out->color, px * 3);
        if (c.flags & GS_FLAG_DEPTH) planes.add(out->depth, px);
        planes.add(alpha_plane, px);
        return sf_poison_if_exceeded(L.bins.status, planes, st);
    };
    if ((rc = run()) != GS_OK) {
        delete s;
        return rc;
    }
    for (bool &valid : ctx->ev_valid) valid = false;
    // k_preprocess, k_tile_scan, k_capacity_gate, [k_emit_buckets,] 4 size classes + k_tile_sort_long, k_composite_fwd,
    // k_sf_poison
    ctx->stats.kernel_launches = (c.P > 0 ? 1 : 0) + 2 + (c.P > 0 ? 1 : 0) + 5 + 1 + 1;
    ctx->stats.num_rendered = -1;
    ctx->stats.num_visible = -1;
    ctx->stats.max_tile_list = -1;
    ctx->stats.speculative = 0;
    ctx->stats.saved_bytes = (int64_t)s->bytes;
    if (saved_out) *saved_out = s;
    else delete s;
    return GS_OK;
}

extern "C" int gs_backward_sync_free(GsContext *ctx, const GsConfig *cfg, const GsInputs *in, const GsSaved *saved,
                                     const GsOutGrads *gout, const GsAlpha *alpha, const GsInGrads *gin,
                                     const GsCameraGrads *cam, float *dL_dtanfov, const GsSyncFreeWorkspace *ws,
                                     void *stream) {
    if (!ctx || !saved || !gout || !gin) return gs_set_error(GS_ERR_INVALID, "null argument");
    int rc = validate(cfg, in);
    if (rc != GS_OK) return rc;
    if (!ws || !saved->ws_base || saved->ws_base != ws->base)
        return gs_set_error(GS_ERR_INVALID, "gs_backward_sync_free needs the saved state of gs_forward_sync_free on the same workspace");
    if (dL_dtanfov && !cam) return gs_set_error(GS_ERR_INVALID, "dL_dtanfov needs the camera gradient (cam)");
    const uint32_t needs = ((cfg->flags & GS_FLAG_DETERMINISTIC) ? GS_SYNC_FREE_DETERMINISTIC : 0u) |
                           (cam ? GS_SYNC_FREE_CAMERA_GRAD : 0u);
    SfLayout L;
    if ((rc = sf_check(make_dev_cfg(cfg), ws, needs, &L)) != GS_OK) return rc;
    const SfBwd sf{L.scratch, L.bins.status};
    return backward(ctx, cfg, in, saved, gout, alpha ? alpha->dL_dalpha : nullptr, gin, stream, cam, dL_dtanfov, &sf);
}

extern "C" int gs_mark_visible(GsContext *ctx, const GsConfig *cfg, const float *means3D, uint8_t *present,
                               void *stream) {
    if (!ctx || !cfg || !means3D || !present) return gs_set_error(GS_ERR_INVALID, "null argument");
    if (cfg->S < 1 || cfg->V < 1 || cfg->V % cfg->S != 0 || !cfg->viewmatrix)
        return gs_set_error(GS_ERR_INVALID, "bad configuration");
    DevCfg c = make_dev_cfg(cfg);
    return launch_mark_visible(c, means3D, present, static_cast<cudaStream_t>(stream));
}

// ---------------------------------------------------------------------------------------------------------
// end-to-end entry with host buffers
// ---------------------------------------------------------------------------------------------------------
namespace {
// alpha_host: gs_render_host_ex's host buffer for the accumulated opacity, else null
int render_host(GsContext *ctx, const GsConfig *cfg, const GsInputs *in, const GsOutputs *out, float *alpha_host,
                void *stream) {
    if (!ctx || !out) return gs_set_error(GS_ERR_INVALID, "null context/outputs");
    int rc = validate(cfg, in);
    if (rc != GS_OK) return rc;
    if ((rc = validate_depth_mode(cfg)) != GS_OK) return rc;
    if ((rc = validate_antialias(cfg->flags, cfg->tuning, AA_FWD_KNOBS)) != GS_OK) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t SP = (size_t)cfg->S * cfg->P, VP = (size_t)cfg->V * cfg->P, V = (size_t)cfg->V;
    const size_t px = V * cfg->image_height * cfg->image_width;
    struct Item { const void *h; size_t bytes; const void **d; };
    GsConfig dc = *cfg;
    GsInputs din{};
    GsOutputs dout{};
    // device-side address of a PINNED host buffer (unified addressing), or null
    auto device_alias = [](const void *host) -> void * {
        cudaPointerAttributes at{};
        if (host && cudaPointerGetAttributes(&at, host) == cudaSuccess && at.type == cudaMemoryTypeHost && at.devicePointer)
            return at.devicePointer;
        cudaGetLastError();  // (an unregistered pointer is not an error for us)
        return nullptr;
    };
    // ZERO-COPY FEED of the SH block (default when the caller's buffer is pinned and M > 16).  The block is most of the
    // bytes (C2: 150 of 170 MB) and the evaluator reads 192 of every 300-byte row.  Instead of the copy engine moving whole
    // rows into a device buffer that a kernel then reads, the kernel that evaluates the colours pulls the 16-byte pieces it
    // wants straight out of the host buffer while staging them into shared memory -- k_sh_colour on a second stream, with
    // geometry, binning and the sort running meanwhile (gs_forward, split_colour), or the fused k_preprocess
    // (GS_TUNE_NO_SPLIT_COLOUR): no device copy of the block, no piece events, and the link carries 13 % fewer bytes
    // (64-byte granularity: scripts/probes/pcie_pull_probe.cu).
    void *sh_alias = nullptr;
    if (in->shs && cfg->M > 16 && !(cfg->tuning & GS_TUNE_NO_ZERO_COPY) &&
        (reinterpret_cast<uintptr_t>(in->shs) & 15u) == 0 && (cfg->S == 1 || ((size_t)cfg->P * cfg->M * 12) % 16 == 0))
        sh_alias = device_alias(in->shs);
    Item items[] = {
        {cfg->viewmatrix, V * 64, (const void **)&dc.viewmatrix},
        {cfg->projmatrix, V * 64, (const void **)&dc.projmatrix},
        {cfg->campos, V * 12, (const void **)&dc.campos},
        {cfg->bg, cfg->bg ? V * 12 : 0, (const void **)&dc.bg},
        {cfg->tanfov, cfg->tanfov ? V * 8 : 0, (const void **)&dc.tanfov},
        {cfg->view_scale, cfg->view_scale ? V * 4 : 0, (const void **)&dc.view_scale},
        {cfg->depth_near_far, cfg->depth_near_far ? V * 8 : 0, (const void **)&dc.depth_near_far},
        {in->means3D, SP * 12, (const void **)&din.means3D},
        {in->opacities, SP * 4, (const void **)&din.opacities},
        {in->shs, (in->shs && !sh_alias) ? SP * cfg->M * 12 : 0, (const void **)&din.shs},
        {in->colors_precomp, in->colors_precomp ? VP * 12 : 0, (const void **)&din.colors_precomp},
        {in->scales, in->scales ? SP * 12 : 0, (const void **)&din.scales},
        {in->rotations, in->rotations ? SP * 16 : 0, (const void **)&din.rotations},
        {in->cov3D_precomp, in->cov3D_precomp ? SP * 24 : 0, (const void **)&din.cov3D_precomp},
    };
    size_t total = 0;
    for (const Item &it : items) total += align256(it.bytes);
    const size_t out_off = total;
    total += align256(px * 12) + align256(VP * 4) + align256(px * 4) + (alpha_host ? align256(px * 4) : 0);
    rc = ctx->host_stage.reserve(total, 1.0);
    if (rc != GS_OK) return rc;
    unsigned char *base = static_cast<unsigned char *>(ctx->host_stage.p);
    // (A strided copy of only the SH bands the evaluator reads -- 192 of each 300-byte row -- was
    // SLOWER end to end than the plain contiguous copy: cudaMemcpy2DAsync with 192-byte rows runs far below PCIe
    // rate.  Rows are copied whole.)
    if (!ctx->copy_stream) GS_CUDA_OK(cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking));
    // The SH block is most of the bytes (C2: 150 of 170 MB).  A single scene's block goes over in pieces on the copy
    // stream, each marked with an event, and gs_forward runs preprocess piece by piece behind them.
    const size_t sh_row = (size_t)cfg->M * 12;
    HostFeed feed{};
    int pieces = 0;
    if (in->shs && !sh_alias && cfg->S == 1 && (size_t)cfg->P * sh_row >= ((size_t)16 << 20)) {
        // more pieces overlap more of preprocess with the transfer (scripts/ab_e2e.py compares piece counts)
        const int req = (int)((cfg->tuning >> GS_TUNE_FEED_PIECES_SHIFT) & 0xFu);
        pieces = req == 0 ? 6 : (req == 1 ? 0 : (req > GsContext::FEED_MAX ? GsContext::FEED_MAX : req));
    }
    // All copies of a pieced call go to the copy stream, everything else first and the SH pieces last (two streams
    // feeding the same copy engine slowed each other down with the small arrays left on the launch stream).
    size_t off = 0, sh_off = 0;
    for (const Item &it : items) {
        *it.d = nullptr;
        if (it.bytes) {
            *it.d = base + off;
            if (pieces && it.h == in->shs) sh_off = off;
            else GS_CUDA_OK(cudaMemcpyAsync(base + off, it.h, it.bytes, cudaMemcpyHostToDevice, pieces ? ctx->copy_stream : st));
        }
        off += align256(it.bytes);
    }
    // (Zero-copy feed: starting k_sh_colour as soon as cameras + means have landed, with the other 14 MB following on the
    // copy stream and gating only the geometry kernel, was dropped: the pull and the copy engine share the
    // link badly.  Everything is copied before the pull starts.
    // Also dropped: the per-Gaussian arrays in four pieces with the geometry preprocess behind them, so that the sort runs
    // underneath the pull instead of after it -- the starved sort slows the pull.)
    if (sh_alias) din.shs = static_cast<const float *>(sh_alias);
    if (pieces) {
        const int step = ((cfg->P + pieces - 1) / pieces + 511) / 512 * 512;  // whole CTAs, 16-byte aligned rows
        int k = 0;
        for (int g = 0; g < cfg->P; g += step, k++) {
            const int g1 = g + step < cfg->P ? g + step : cfg->P;
            if (!ctx->feed_ev[k]) GS_CUDA_OK(cudaEventCreateWithFlags(&ctx->feed_ev[k], cudaEventDisableTiming));
            GS_CUDA_OK(cudaMemcpyAsync(base + sh_off + (size_t)g * sh_row, reinterpret_cast<const char *>(in->shs) + (size_t)g * sh_row,
                                       (size_t)(g1 - g) * sh_row, cudaMemcpyHostToDevice, ctx->copy_stream));
            GS_CUDA_OK(cudaEventRecord(ctx->feed_ev[k], ctx->copy_stream));
            feed.begin[k] = g;
            feed.begin[k + 1] = g1;
        }
        pieces = k;
    }
    feed.chunks = pieces;
    feed.sh_zero_copy = sh_alias != nullptr;
    feed.radii_dst = (out->radii && VP) ? out->radii : nullptr;
    dout.color = reinterpret_cast<float *>(base + out_off);
    dout.radii = reinterpret_cast<int32_t *>(base + out_off + align256(px * 12));
    dout.depth = (cfg->flags & GS_FLAG_DEPTH) ? reinterpret_cast<float *>(base + out_off + align256(px * 12) + align256(VP * 4))
                                              : nullptr;
    float *dalpha = alpha_host ? reinterpret_cast<float *>(base + out_off + align256(px * 12) + align256(VP * 4) + align256(px * 4))
                               : nullptr;
    // Experiment (GS_TUNE_DIRECT_OUTPUT): let the compositor write the images STRAIGHT into the caller's buffers when those
    // are pinned (device-accessible under unified addressing), instead of a device-to-host copy of the whole image queued
    // behind it (C2: 6.3 MB at the very end of the call).  In-process on C2 (scripts/ab_e2e.py) direct output was
    // slower -- 32-byte posted writes over PCIe cost the compositor more than the copy engine's
    // one burst afterwards.  The copy stays the default.
    const bool direct = (cfg->tuning & GS_TUNE_DIRECT_OUTPUT) != 0;
    void *color_alias = direct ? device_alias(out->color) : nullptr;
    void *depth_alias = direct && dout.depth ? device_alias(out->depth) : nullptr;
    if (color_alias) dout.color = static_cast<float *>(color_alias);
    if (depth_alias) dout.depth = static_cast<float *>(depth_alias);
    void *alpha_alias = direct && alpha_host ? device_alias(alpha_host) : nullptr;
    if (alpha_alias) dalpha = static_cast<float *>(alpha_alias);
    rc = forward(ctx, &dc, &din, &dout, nullptr, st, &feed, dalpha);
    if (rc != GS_OK) {
        // nothing of ours may still be reading the caller's buffers (the colour kernel pulls out of them) once we return
        if (ctx->aux_stream) cudaStreamSynchronize(ctx->aux_stream);
        cudaStreamSynchronize(ctx->copy_stream);
        cudaStreamSynchronize(st);
        return rc;
    }
    if (out->color && !color_alias) GS_CUDA_OK(cudaMemcpyAsync(out->color, dout.color, px * 12, cudaMemcpyDeviceToHost, st));
    if (out->depth && dout.depth && !depth_alias)
        GS_CUDA_OK(cudaMemcpyAsync(out->depth, dout.depth, px * 4, cudaMemcpyDeviceToHost, st));
    if (alpha_host && !alpha_alias) GS_CUDA_OK(cudaMemcpyAsync(alpha_host, dalpha, px * 4, cudaMemcpyDeviceToHost, st));
    GS_CUDA_OK(cudaStreamSynchronize(st));
    GS_CUDA_OK(cudaStreamSynchronize(ctx->copy_stream));  // radii (started after the forward's mid-way sync)
    return GS_OK;
}
}  // namespace

extern "C" int gs_render_host(GsContext *ctx, const GsConfig *cfg, const GsInputs *in, const GsOutputs *out,
                              void *stream) {
    return render_host(ctx, cfg, in, out, nullptr, stream);
}

extern "C" int gs_render_host_ex(GsContext *ctx, const GsConfig *cfg, const GsInputs *in, const GsOutputs *out,
                                 const GsAlpha *alpha, void *stream) {
    if (!alpha) return gs_set_error(GS_ERR_INVALID, "null alpha request");
    if (!alpha->alpha) return gs_set_error(GS_ERR_INVALID, "gs_render_host_ex needs alpha->alpha (gs_render_host renders without it)");
    return render_host(ctx, cfg, in, out, alpha->alpha, stream);
}
