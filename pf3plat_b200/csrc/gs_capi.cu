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

enum { STRATA_UNKNOWN = 0, STRATA_TRIAL = 1, STRATA_ON = 2, STRATA_OFF = 3 };

// speculative bucket capacities learned from the previous forward of the same shape (0 = none yet)
struct SpecState {
    int V = 0, ntiles = 0;
    uint32_t sub_cap = 0;     // capacity of one of a tile's BIN_SUB sub-buckets
    uint32_t tile_limit = 0;  // list length the tile sort is launched for
    // Depth strata (gs_binning.cu).  UNKNOWN: no boundaries for this shape yet.  TRIAL: boundaries learned by the
    // last exact-path call, capacities still those of index % BIN_SUB sub-buckets -> the next speculative call
    // tries strata with doubled capacities.  ON: strata with capacities learned from stratified counts.
    // OFF: the trial overflowed (a tile whose depths crowd into one stratum): this shape stays on whole-tile sorts.
    int strata_state = STRATA_UNKNOWN;
    // Which boundaries `strata` holds: one row per view (octiles of the view's depths), or -- for shapes whose
    // per-view trial overflowed: tiles that each see a narrow depth range, e.g. PF3plat's pixel-aligned Gaussians on
    // a smooth surface -- one row per (view, tile), learned from the exact call's sorted lists and refreshed by the
    // stratum sort of every call (two tables, swapped on success).
    int strata_per_tile = 0, want_per_tile = 0, tile_tab = 0;
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
    // What earlier forwards of a SHAPE (views, tiles, Gaussians per scene, scenes) taught: speculative bucket capacities,
    // the strata state machine and its boundary tables.  A context remembers SHAPE_SLOTS shapes (least recently used one
    // evicted), so a caller that alternates shapes -- context and target views of a training step, training and validation
    // batches -- keeps every one of them on the speculative path; `spec` / `strata` point at the slot of the running call.
    static constexpr int SHAPE_SLOTS = 4;
    struct ShapeSlot {
        int key_V = -1, key_ntiles = -1, key_P = -1, key_S = -1;
        uint64_t last_use = 0;
        SpecState spec;
        GrowBuf strata;   // [V][BIN_SUB] (or two tables of [V*tiles][BIN_SUB]) stratum boundaries + histogram scratch
    } slots[SHAPE_SLOTS];
    uint64_t use_counter = 0;
    SpecState *spec = &slots[0].spec;
    GrowBuf *strata = &slots[0].strata;
    cudaEvent_t ev_pre = nullptr;   // "preprocess done" (speculative path: lets the radii copy start early)
    cudaEvent_t ev_info = nullptr;  // "binning verdict copied to the host"
    // gs_render_host's split pipeline: k_sh_colour pulls the SH block out of the caller's pinned buffer on aux_stream while
    // geometry, binning and the tile sort run on the launch stream; the compositor waits for ev_colour
    cudaStream_t aux_stream = nullptr;
    cudaEvent_t ev_alloc = nullptr, ev_colour = nullptr;
    // gs_render_host: radii are final once the forward's mid-way sync has passed, so their copy to the host
    // overlaps binning + compositing on a side stream
    cudaStream_t copy_stream = nullptr;
    void *host_radii_dst = nullptr;
    size_t host_radii_bytes = 0;
    // gs_render_host: the SH block arrives in feed_chunks pieces on the copy stream; piece k (Gaussians
    // [feed_begin[k], feed_begin[k+1])) is complete once feed_ev[k] has fired, and preprocess runs piece by piece
    // behind them, so all but the last piece of preprocess hides under the host-to-device transfer
    static constexpr int FEED_MAX = 8;
    int feed_chunks = 0;
    bool sh_zero_copy = false;         // gs_render_host: in->shs is the device alias of the caller's pinned buffer (preprocess pulls it over PCIe)
    int feed_begin[FEED_MAX + 1] = {};
    cudaEvent_t feed_ev[FEED_MAX] = {};
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

DevCfg make_dev_cfg(const GsConfig *cfg) {
    DevCfg c{};
    c.P = cfg->P; c.S = cfg->S; c.V = cfg->V; c.VPS = cfg->V / cfg->S; c.M = cfg->M;
    const int maxdeg = cfg->sh_eval_max_degree > 0 ? cfg->sh_eval_max_degree : 3;
    int deg = cfg->sh_degree < maxdeg ? cfg->sh_degree : maxdeg;
    if (deg > 3) deg = 3;                                    // the evaluator implements bands 0..3
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

// Capacities for the next forward of this shape: 30 % headroom over what this one needed.
// Capacities are quantised and sticky: a capacity that still fits and is not more than 1.5x what is needed is kept, so
// that a cloud that moves a little every step (training) asks the memory pool for the SAME block sizes call after call
// (with capacities re-derived every call, the varying sizes of a jittered cloud defeat the pool's reuse and the
// mapping of new blocks costs more than the kernels).
inline uint32_t sticky_capacity(uint32_t need, uint32_t current) {
    need = (need + 63u) & ~63u;
    return (current >= need && (uint64_t)current * 2 <= (uint64_t)need * 3) ? current : need;
}

void learn_capacities(GsContext *ctx, const DevCfg &c, uint32_t max_tile, uint32_t max_sub) {
    const bool same_shape = ctx->spec->V == c.V && ctx->spec->ntiles == c.ntiles;
    const uint32_t sub_cap = sticky_capacity(max_sub + max_sub * 3 / 10 + 16, same_shape ? ctx->spec->sub_cap : 0u);
    const uint32_t limit = sticky_capacity(max_tile + max_tile / 10 + 32, same_shape ? ctx->spec->tile_limit : 0u);
    if (limit > BIN_SMEM_CAP || (uint64_t)sub_cap * BIN_SUB * c.V * c.ntiles > 0xffffffffull) {
        ctx->spec->sub_cap = 0;  // lists too long for the shared-memory sort (or offsets beyond 32 bits): exact path
        return;
    }
    if (ctx->spec->V != c.V || ctx->spec->ntiles != c.ntiles) {
        ctx->spec->strata_state = STRATA_UNKNOWN;
        ctx->spec->strata_per_tile = ctx->spec->want_per_tile = 0;
    }
    ctx->spec->V = c.V;
    ctx->spec->ntiles = c.ntiles;
    ctx->spec->sub_cap = sub_cap;
    ctx->spec->tile_limit = limit;
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
    for (auto &sl : ctx->slots) sl.strata.release();
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
// Memory policy of the context's private pool.  Freed blocks stay in the pool (release threshold = never, set at creation):
// every automatic scheme tried released memory that the very next calls mapped again, and both directions are expensive
// (mapping is paid per MB, and releasing at a synchronisation stalls that call and the next):
//   * threshold = scratch + 1.25 x saved state, updated every call: a shape that is still settling (exact call, strata
//     trial, re-learned capacities, the backward's accumulator growing the scratch) changes its block sizes from call to call
//     -- forward + backward at the C4 size stalled for several steps, with hiccups well after that;
//   * the same once settled: the usual training loop (`out = render(...)`, rebinding `out`) keeps the previous step's saved
//     state alive until the new forward has returned -- room for one meant mapping a second every step;
//   * room for two: the reference's decoder makes a call per view plus one per view for depth, and autograd holds all their
//     saved states until the backward (12 at PF3plat's 2 x 3 views): mapping again every step; following the pool's
//     high-water mark fixed that but left hiccups whenever a capacity changed.
// So, like the caching allocator of the host framework, the pool only gives memory back when asked (gs_context_trim /
// rasterizer.trim_memory, gs_context_destroy) -- or here, every 256 calls, when it holds more than twice the high-water
// mark of what those 256 calls had handed out at any one time (a one-off large batch does not pin its memory for ever).
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
    if (saved->point_list) cudaFreeAsync(saved->point_list, static_cast<cudaStream_t>(stream));
    if (saved->base) cudaFreeAsync(saved->base, static_cast<cudaStream_t>(stream));
    delete saved;
}

extern "C" int gs_forward(GsContext *ctx, const GsConfig *cfg, const GsInputs *in, const GsOutputs *out,
                          GsSaved **saved_out, void *stream) {
    if (saved_out) *saved_out = nullptr;
    if (!ctx || !out) return gs_set_error(GS_ERR_INVALID, "null context/outputs");
    int rc = validate(cfg, in);
    if (rc != GS_OK) return rc;
    if (!out->color || (cfg->P > 0 && !out->radii)) return gs_set_error(GS_ERR_INVALID, "color/radii outputs missing");
    if ((cfg->flags & GS_FLAG_DEPTH) && !out->depth) return gs_set_error(GS_ERR_INVALID, "GS_FLAG_DEPTH needs out->depth");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const DevCfg c = make_dev_cfg(cfg);
    const DevInputs di = make_dev_inputs(in);
    const size_t n = (size_t)c.V * c.P;
    {   // this shape's slot: what its earlier calls taught (GsContext::ShapeSlot); least recently used slot on a miss
        GsContext::ShapeSlot *hit = nullptr, *lru = &ctx->slots[0];
        for (auto &sl : ctx->slots) {
            if (sl.key_V == c.V && sl.key_ntiles == c.ntiles && sl.key_P == c.P && sl.key_S == c.S) hit = &sl;
            if (sl.last_use < lru->last_use) lru = &sl;
        }
        if (!hit) {
            hit = lru;
            hit->spec = SpecState{};   // (the slot's boundary buffer is kept and re-filled by the exact call)
            hit->key_V = c.V; hit->key_ntiles = c.ntiles; hit->key_P = c.P; hit->key_S = c.S;
        }
        hit->last_use = ++ctx->use_counter;
        ctx->spec = &hit->spec;
        ctx->strata = &hit->strata;
    }
    // gs_render_host with a pinned SH block: geometry-only preprocess here, colours by k_sh_colour on a second stream
    const bool split_colour = ctx->sh_zero_copy && !(cfg->tuning & GS_TUNE_NO_SPLIT_COLOUR) && n > 0 && sh_colour_supported(c, di);
    const int pre_low = ((cfg->tuning & GS_TUNE_PRE_OCC6) ? 1 : 0) | (((cfg->tuning & GS_TUNE_PRE_SH_RAW16) || ctx->sh_zero_copy) ? 2 : 0) |
                        (split_colour ? 4 : 0);
    for (bool &v : ctx->ev_valid) v = false;
    ctx->stats.kernel_launches = 0;

    // ---- per-call scratch: rects[n] | counters | cursors | verdict words | sub-bucket offsets | tile_start | tile_n ----
    const size_t nvt = (size_t)c.V * c.ntiles;
    const size_t ctr_bytes = align256(bin_counter_bytes(c));
    const size_t pg_bytes = align256(n * 8) + 2 * ctr_bytes + 256 + align256(nvt * BIN_SUB * 4) + 2 * align256(nvt * 4);
    rc = ctx->per_gaussian.reserve(pg_bytes, 1.0, ctx->pool, st);
    if (rc != GS_OK) return rc;
    unsigned char *pg = static_cast<unsigned char *>(ctx->per_gaussian.p);
    ushort4 *rects = reinterpret_cast<ushort4 *>(pg);
    pg += align256(n * 8);
    uint32_t *tile_counts = reinterpret_cast<uint32_t *>(pg);
    pg += ctr_bytes;
    uint32_t *cursor = reinterpret_cast<uint32_t *>(pg);
    pg += ctr_bytes;
    uint32_t *verdict_acc = reinterpret_cast<uint32_t *>(pg);  // directly behind the cursors: one memset clears both
    pg += 256;
    uint32_t *sub_offsets = reinterpret_cast<uint32_t *>(pg);
    pg += align256(nvt * BIN_SUB * 4);
    uint32_t *tile_start = reinterpret_cast<uint32_t *>(pg);
    pg += align256(nvt * 4);
    uint32_t *tile_n = reinterpret_cast<uint32_t *>(pg);

    // ---- saved state: geometry / image planes now, the tile-instance list once its length is known ----
    GsSaved *s = new (std::nothrow) GsSaved();
    if (!s) return gs_set_error(GS_ERR_OOM, "host allocation failed");
    memset(s, 0, sizeof(*s));
    {
        const size_t bytes = saved_layout(s, c, nullptr);
        unsigned char *block = nullptr;
        cudaError_t e = cudaMallocFromPoolAsync(reinterpret_cast<void **>(&block), bytes, ctx->pool, st);
        if (e != cudaSuccess) {
            delete s;
            return gs_set_cuda_error(e, "cudaMallocAsync(saved)", __FILE__, __LINE__);
        }
        saved_layout(s, c, block);
        s->base = block;
        s->bytes = bytes;
    }
    bool colour_pending = false;   // k_sh_colour is (or may still be) writing into s->rec1 / s->rec2 on the aux stream
    auto fail = [&](int code) {
        if (colour_pending) cudaStreamWaitEvent(st, ctx->ev_colour, 0);   // the free below is ordered on `st`
        gs_saved_free(ctx, s, stream);
        return code;
    };
    if (split_colour) {
        cudaError_t e = cudaSuccess;
        if (!ctx->aux_stream) e = cudaStreamCreateWithFlags(&ctx->aux_stream, cudaStreamNonBlocking);
        if (e == cudaSuccess && !ctx->ev_alloc) e = cudaEventCreateWithFlags(&ctx->ev_alloc, cudaEventDisableTiming);
        if (e == cudaSuccess && !ctx->ev_colour) e = cudaEventCreateWithFlags(&ctx->ev_colour, cudaEventDisableTiming);
        // everything enqueued on `st` so far -- the caller's uploads of means and cameras, the allocation of the records --
        // precedes the colour kernel
        if (e == cudaSuccess) e = cudaEventRecord(ctx->ev_alloc, st);
        if (e == cudaSuccess) e = cudaStreamWaitEvent(ctx->aux_stream, ctx->ev_alloc, 0);
        if (e != cudaSuccess) return fail(gs_set_cuda_error(e, "split colour pipeline setup", __FILE__, __LINE__));
        {
            StageTimer t(ctx, GS_STAGE_SH_COLOUR, ctx->aux_stream);
            rc = launch_sh_colour(c, di, s->rec1, s->rec2, nullptr, ctx->aux_stream);
        }
        if (rc != GS_OK) return fail(rc);
        colour_pending = true;
        e = cudaEventRecord(ctx->ev_colour, ctx->aux_stream);
        if (e != cudaSuccess) {
            cudaStreamSynchronize(ctx->aux_stream);
            colour_pending = false;
            return fail(gs_set_cuda_error(e, "cudaEventRecord(colour)", __FILE__, __LINE__));
        }
    }
    // the compositor needs the colour words: called right before each of its launches
    auto join_colour = [&]() -> cudaError_t {
        if (!colour_pending) return cudaSuccess;
        colour_pending = false;   // from here on `st` itself is ordered behind the colour kernel
        return cudaStreamWaitEvent(st, ctx->ev_colour, 0);
    };

    // ---- speculative-capacity forward: no count/scan passes and no mid-pipeline bubble ----
    // The tile instances go straight into fixed-capacity sub-buckets sized from the previous forward of this shape;
    // a one-CTA kernel right after preprocess checks that nothing overflowed, and the host reads its verdict only
    // after the tile sort and the compositor have been enqueued behind it.  On overflow the results are discarded
    // and the call is redone below on the exact path (which re-learns the capacities).
    const bool speculate = ctx->spec->sub_cap > 0 && ctx->spec->V == c.V && ctx->spec->ntiles == c.ntiles && n > 0 &&
                           !(cfg->tuning & (GS_TUNE_FORCE_RADIX_BINNING | GS_TUNE_NO_SPECULATION));
    if (speculate) {
        bool strata = (ctx->spec->strata_state == STRATA_TRIAL || ctx->spec->strata_state == STRATA_ON) &&
                      !(cfg->tuning & GS_TUNE_NO_STRATA) && ctx->strata->p != nullptr;
        uint32_t sub_cap = ctx->spec->sub_cap;
        if (strata && ctx->spec->strata_state == STRATA_TRIAL) {
            // capacities were learned unstratified: the trial runs on doubled ones -- if the kernels' 32-bit bucket
            // offsets still hold them (learn_capacities checked the undoubled value only)
            // A cloud whose tiles each see a narrow depth range (PF3plat's pixel-aligned Gaussians on a smooth surface)
            // puts a tile's whole list into one or two of the per-view strata: the trial must be able to hold a whole
            // list per stratum, memory permitting (the capacities learned from it are what later calls allocate).
            // (Sizing the trial for a WHOLE tile list per stratum -- so that clouds whose tiles each see a narrow depth
            // range, like PF3plat's pixel-aligned Gaussians, stay stratified -- was dropped: such a shape
            // then sorts one or two 1 600-key strata per tile with a single warp each, slower than the whole-tile merge
            // sort + verdict kernel it falls back to.  Per-TILE boundaries are the fix.)
            uint32_t trial = sub_cap * 2;
            if (trial > BIN_STRATUM_CAP) trial = BIN_STRATUM_CAP;
            if ((uint64_t)trial * BIN_SUB * nvt > 0xffffffffull) strata = false;
            else sub_cap = trial;
        }
        if (strata && sub_cap > BIN_STRATUM_CAP) sub_cap = BIN_STRATUM_CAP;
        const int per_tile = strata ? ctx->spec->strata_per_tile : 0;
        const size_t tab_floats = nvt * BIN_SUB;  // one per-tile table
        float *tab0 = static_cast<float *>(ctx->strata->p);
        const float *strata_tab = !strata ? nullptr : (per_tile ? tab0 + (size_t)ctx->spec->tile_tab * tab_floats : tab0);
        float *strata_next = (strata && per_tile) ? tab0 + (size_t)(ctx->spec->tile_tab ^ 1) * tab_floats : nullptr;
        const size_t slots = nvt * BIN_SUB;
        rc = ctx->sort.reserve(slots * sub_cap * 8, 1.0, ctx->pool, st);
        if (rc != GS_OK) return fail(rc);
        cudaError_t e = cudaMallocFromPoolAsync(reinterpret_cast<void **>(&s->point_list), slots * sub_cap * 4, ctx->pool, st);
        if (e != cudaSuccess) {
            s->point_list = nullptr;
            return fail(gs_set_cuda_error(e, "cudaMallocAsync(point_list)", __FILE__, __LINE__));
        }
        e = cudaMemsetAsync(cursor, 0, ctr_bytes + 256, st);
        if (e != cudaSuccess) return fail(gs_set_cuda_error(e, "cudaMemsetAsync(cursors)", __FILE__, __LINE__));
        // Appending from inside preprocess touches the buckets of ALL views at once; far beyond L2 size those 8-byte
        // appends turn into partial-sector DRAM writes, so big bucket sets (C4) are filled by the view-major
        // k_emit_buckets instead.  The bound sits above the 50 MB L2 of an H100 because C2's buckets, which exceed it,
        // are still filled faster by the fused appends on an H100 (README.md; `bench.py --tuning 4` forces k_emit_buckets).
        const bool fused_emit = slots * sub_cap * 8 <= ((size_t)96 << 20) && !(cfg->tuning & GS_TUNE_SEPARATE_EMIT);
        {
            StageTimer t(ctx, GS_STAGE_PREPROCESS, st);
            const PreEmit emit{fused_emit ? cursor : nullptr, static_cast<uint64_t *>(ctx->sort.p), sub_cap, strata_tab, per_tile};
            if (ctx->feed_chunks > 0) {
                for (int k = 0; k < ctx->feed_chunks && rc == GS_OK; k++) {
                    e = cudaStreamWaitEvent(st, ctx->feed_ev[k], 0);
                    if (e != cudaSuccess) return fail(gs_set_cuda_error(e, "cudaStreamWaitEvent(feed)", __FILE__, __LINE__));
                    rc = launch_preprocess(c, di, s->rec0, s->rec1, s->rec2, s->meta, out->radii, rects, emit, st,
                                           ctx->feed_begin[k], ctx->feed_begin[k + 1], pre_low);
                }
            } else {
                rc = launch_preprocess(c, di, s->rec0, s->rec1, s->rec2, s->meta, out->radii, rects, emit, st, 0, -1, pre_low);
            }
            if (rc != GS_OK) return fail(rc);
        }
        if (!fused_emit) {
            StageTimer t(ctx, GS_STAGE_BIN_EMIT, st);
            rc = bin_emit_fast(c, 1, s->rec0, s->rec1, s->rec2, rects, nullptr, sub_cap, strata_tab, per_tile, cursor, ctx->sort.p, st);
            if (rc != GS_OK) return fail(rc);
        }
        // gs_render_host: the radii leave for the host on the copy stream as soon as they are final -- after preprocess
        // on the whole-tile path; after the sort on the stratified path, whose last CTA stores the verdict into host
        // memory (a store that would otherwise sit behind the 16 MB of radii on the PCIe link)
        auto start_radii_copy = [&]() -> cudaError_t {
            if (!(ctx->host_radii_dst && ctx->copy_stream)) return cudaSuccess;
            cudaError_t ee = cudaSuccess;
            if (!ctx->ev_pre) ee = cudaEventCreateWithFlags(&ctx->ev_pre, cudaEventDisableTiming);
            if (ee == cudaSuccess) ee = cudaEventRecord(ctx->ev_pre, st);
            if (ee == cudaSuccess) ee = cudaStreamWaitEvent(ctx->copy_stream, ctx->ev_pre, 0);
            if (ee == cudaSuccess)
                ee = cudaMemcpyAsync(ctx->host_radii_dst, out->radii, ctx->host_radii_bytes, cudaMemcpyDeviceToHost,
                                     ctx->copy_stream);
            return ee;
        };
        if (!strata && (e = start_radii_copy()) != cudaSuccess)
            return fail(gs_set_cuda_error(e, "early radii copy", __FILE__, __LINE__));
        // The verdict (overflow flag, counts) follows from the cursors alone.  Whole-tile path: one tiny kernel right
        // after preprocess; stratified path: the sort's CTAs add it up themselves and the last one publishes it.  Either
        // way it is stored straight into mapped pinned memory (an in-stream D2H copy would queue behind the 16 MB
        // radii copy of gs_render_host in the copy engine) and marked with an event, and the remaining kernels are
        // enqueued BEFORE the host waits on that event: the caller gets control back (to enqueue its next call) while
        // the GPU is still busy.
        if (!ctx->ev_info) {
            e = cudaEventCreateWithFlags(&ctx->ev_info, cudaEventDisableTiming);
            if (e != cudaSuccess) return fail(gs_set_cuda_error(e, "cudaEventCreate", __FILE__, __LINE__));
        }
        if (!strata) {
            StageTimer t(ctx, GS_STAGE_BIN_SCAN, st);
            rc = bin_spec_check(c, sub_cap, ctx->spec->tile_limit, cursor, ctx->d_word, st);
            if (rc != GS_OK) return fail(rc);
            e = cudaEventRecord(ctx->ev_info, st);
            if (e != cudaSuccess) return fail(gs_set_cuda_error(e, "read back binning info", __FILE__, __LINE__));
        }
        {
            StageTimer t(ctx, GS_STAGE_BIN_SORT, st);
            if (strata) {
                rc = bin_sort_strata(c, sub_cap, cursor, ctx->sort.p, s->point_list, s->ranges, verdict_acc, ctx->d_word, st,
                                     (cfg->tuning & GS_TUNE_STRATA_MERGE_SORT) != 0, s->rec2, strata_next);
                if (rc == GS_OK && (e = cudaEventRecord(ctx->ev_info, st)) != cudaSuccess)
                    return fail(gs_set_cuda_error(e, "read back binning info", __FILE__, __LINE__));
                if (rc == GS_OK && (e = start_radii_copy()) != cudaSuccess)
                    return fail(gs_set_cuda_error(e, "early radii copy", __FILE__, __LINE__));
            } else {
                rc = bin_sort_spec(c, sub_cap, ctx->spec->tile_limit, cursor, ctx->sort.p, s->point_list, s->ranges, st);
            }
            if (rc != GS_OK) return fail(rc);
        }
        if ((e = join_colour()) != cudaSuccess) return fail(gs_set_cuda_error(e, "cudaStreamWaitEvent(colour)", __FILE__, __LINE__));
        {
            StageTimer t(ctx, GS_STAGE_COMPOSITE, st);
            rc = launch_composite_fwd(c, *s, out->color, out->depth, st, (cfg->tuning & GS_TUNE_FWD_WS) ? 2 : 0);
            if (rc != GS_OK) return fail(rc);
        }
        e = cudaEventSynchronize(ctx->ev_info);  // the one host sync of the forward (verification only)
        if (e != cudaSuccess) return fail(gs_set_cuda_error(e, "cudaEventSynchronize", __FILE__, __LINE__));
        if (ctx->h_word[3] == 0) {
            const int64_t D = (int64_t)ctx->h_word[0];
            if (strata) {
                // capacities for the next call from the stratified counts just measured; a stratum beyond the small
                // sort's capacity sends this shape back to whole-tile sorts (via one exact-path call)
                uint32_t next = sticky_capacity(ctx->h_word[2] + ctx->h_word[2] * 3 / 10 + 16,
                                                ctx->spec->strata_state == STRATA_ON ? sub_cap : 0u);
                if (next > BIN_STRATUM_CAP && ctx->h_word[2] + ctx->h_word[2] / 10 <= BIN_STRATUM_CAP) next = BIN_STRATUM_CAP;  // 10 % headroom still fits
                if (next > BIN_STRATUM_CAP) {
                    ctx->spec->strata_state = STRATA_OFF;
                    ctx->spec->sub_cap = 0;
                } else {
                    if (ctx->spec->strata_state == STRATA_TRIAL && ctx->sort.bytes > 2 * (slots * (size_t)next * 8) + ((size_t)8 << 20)) {
                        // the trial's generous buckets are not needed again: give the block back (stream-ordered)
                        if (ctx->sort.pooled) cudaFreeAsync(ctx->sort.p, st);
                        else cudaFree(ctx->sort.p);
                        ctx->sort.p = nullptr;
                        ctx->sort.bytes = 0;
                    }
                    ctx->spec->strata_state = STRATA_ON;
                    ctx->spec->sub_cap = next;
                    if (per_tile) ctx->spec->tile_tab ^= 1;  // the sort wrote the next call's boundaries into the other table
                }
            } else {
                learn_capacities(ctx, c, ctx->h_word[1], ctx->h_word[2]);
            }
            s->D = D;
            s->P = c.P; s->S = c.S; s->V = c.V; s->H = c.H; s->W = c.W;
            s->flags = c.flags;
            s->has_sh = in->shs != nullptr;
            s->has_scales = in->scales != nullptr;
            ctx->stats.kernel_launches = (strata ? 3 : 4) + (fused_emit ? 0 : 1) + (split_colour ? 1 : 0);  // k_preprocess, [k_sh_colour,] [k_emit_buckets], [k_spec_check,] tile sort, k_composite_fwd
            ctx->stats.max_tile_list = (int32_t)ctx->h_word[1];
            ctx->stats.num_rendered = D;
            ctx->stats.num_visible = -1;
            ctx->stats.saved_bytes = (int64_t)(s->bytes + slots * sub_cap * 4);
            pool_follow(ctx);
            ctx->stats.speculative = strata ? 2 : 1;
            if (saved_out) *saved_out = s;
            else gs_saved_free(ctx, s, stream);
            return GS_OK;
        }
        // overflow: some sub-bucket or tile list outgrew its capacity.  Results are invalid; redo exactly.
        ctx->stats.overflow_redos++;
        ctx->spec->sub_cap = 0;
        if (strata) {
            if (ctx->spec->strata_state == STRATA_TRIAL && !per_tile && !(cfg->tuning & GS_TUNE_NO_TILE_STRATA)) {
                // the per-view boundaries crowd some tile into one stratum: the exact redo below learns per-tile ones
                ctx->spec->want_per_tile = 1;
                ctx->spec->strata_state = STRATA_UNKNOWN;
            } else {
                ctx->spec->strata_state = ctx->spec->strata_state == STRATA_TRIAL ? STRATA_OFF : STRATA_UNKNOWN;
            }
        }
        if (ctx->host_radii_dst && ctx->copy_stream) cudaStreamSynchronize(ctx->copy_stream);
        cudaFreeAsync(s->point_list, st);
        s->point_list = nullptr;
        for (bool &v : ctx->ev_valid) v = false;
    }
    ctx->stats.speculative = 0;

    {
        StageTimer t(ctx, GS_STAGE_PREPROCESS, st);
        cudaError_t e = cudaMemsetAsync(tile_counts, 0, bin_counter_bytes(c), st);
        if (e != cudaSuccess) return fail(gs_set_cuda_error(e, "cudaMemsetAsync(tile_counts)", __FILE__, __LINE__));
        const PreEmit emit{tile_counts, nullptr, 0, nullptr, 0};  // exact path: sub-bucket = index % BIN_SUB
        for (int k = 0; k < ctx->feed_chunks; k++) {  // gs_render_host: every piece of the SH block must have landed
            e = cudaStreamWaitEvent(st, ctx->feed_ev[k], 0);
            if (e != cudaSuccess) return fail(gs_set_cuda_error(e, "cudaStreamWaitEvent(feed)", __FILE__, __LINE__));
        }
        rc = launch_preprocess(c, di, s->rec0, s->rec1, s->rec2, s->meta, out->radii, rects, emit, st, 0, -1, pre_low);
        if (rc != GS_OK) return fail(rc);
        ctx->stats.kernel_launches += (c.P > 0);
    }

    int64_t D = 0;
    uint32_t max_count = 0;
    {
        StageTimer t(ctx, GS_STAGE_BIN_SCAN, st);
        // the scan kernel stores its three result words straight into pinned host memory (no copy-engine hop)
        rc = bin_tile_scan(c, tile_counts, sub_offsets, tile_start, tile_n, ctx->d_word, st);
        if (rc != GS_OK) return fail(rc);
        cudaError_t e = cudaStreamSynchronize(st);  // the one host sync of the (exact) forward
        if (e != cudaSuccess) return fail(gs_set_cuda_error(e, "read back num_rendered", __FILE__, __LINE__));
        D = (int64_t)ctx->h_word[0];
        max_count = ctx->h_word[1];
        learn_capacities(ctx, c, max_count, ctx->h_word[2]);
        if (ctx->host_radii_dst && ctx->copy_stream) {  // preprocess has completed: radii can leave now
            e = cudaMemcpyAsync(ctx->host_radii_dst, out->radii, ctx->host_radii_bytes, cudaMemcpyDeviceToHost,
                                ctx->copy_stream);
            if (e != cudaSuccess) return fail(gs_set_cuda_error(e, "cudaMemcpyAsync(radii)", __FILE__, __LINE__));
        }
        if (D > 0x7fffffffll) return fail(gs_set_error(GS_ERR_OVERFLOW, "more than 2^31-1 tile instances"));
        // the list lives in its own stream-ordered allocation (sized exactly)
        e = cudaMallocFromPoolAsync(reinterpret_cast<void **>(&s->point_list), (size_t)(D > 0 ? D : 1) * 4, ctx->pool, st);
        if (e != cudaSuccess) {
            s->point_list = nullptr;
            return fail(gs_set_cuda_error(e, "cudaMallocAsync(point_list)", __FILE__, __LINE__));
        }
        s->D = D;
    }
    const bool fast = bin_fits_fast_path(max_count) && !(cfg->tuning & GS_TUNE_FORCE_RADIX_BINNING);
    rc = ctx->sort.reserve(bin_scratch_bytes(c, D, fast), 1.25, ctx->pool, st);
    if (rc != GS_OK) return fail(rc);
    {
        StageTimer t(ctx, GS_STAGE_BIN_EMIT, st);
        if (fast)
            rc = bin_emit_fast(c, D, s->rec0, s->rec1, s->rec2, rects, sub_offsets, 0, nullptr, 0, cursor, ctx->sort.p, st);
        else
            rc = bin_sort_fallback(c, D, s->rec0, s->rec1, s->rec2, rects, ctx->sort.p, ctx->sort.bytes, s->point_list,
                                   s->ranges, st);
        if (rc != GS_OK) return fail(rc);
    }
    if (fast) {
        StageTimer t(ctx, GS_STAGE_BIN_SORT, st);
        rc = bin_sort_fast(c, max_count, tile_start, tile_n, ctx->sort.p, s->point_list, s->ranges, st);
        if (rc != GS_OK) return fail(rc);
    }
    ctx->stats.kernel_launches += 1 + (D > 0 ? 1 : 0) + 1;  // scan, emit, tile sort (fallback: 3 + CUB's)
    ctx->stats.max_tile_list = (int32_t)max_count;

    {
        cudaError_t e = join_colour();
        if (e != cudaSuccess) return fail(gs_set_cuda_error(e, "cudaStreamWaitEvent(colour)", __FILE__, __LINE__));
    }
    {
        StageTimer t(ctx, GS_STAGE_COMPOSITE, st);
        rc = launch_composite_fwd(c, *s, out->color, out->depth, st, (cfg->tuning & GS_TUNE_FWD_WS) ? 2 : 0);
        if (rc != GS_OK) return fail(rc);
        ctx->stats.kernel_launches += 1;
    }

    // Depth-stratum boundaries for the coming speculative calls, from this call's depths (off this call's critical
    // path: queued behind the compositor).  STRATA_OFF is sticky for the shape.
    if (fast && ctx->spec->sub_cap > 0 && ctx->spec->strata_state != STRATA_OFF && !(cfg->tuning & GS_TUNE_NO_STRATA) && n > 0) {
        rc = ctx->strata->reserve(bin_strata_bytes(c), 1.0, ctx->pool, st);
        if (rc != GS_OK) return fail(rc);
        if (ctx->spec->want_per_tile) {
            ctx->spec->tile_tab = 0;
            rc = bin_learn_tile_strata(c, s->point_list, s->ranges, s->rec2, static_cast<float *>(ctx->strata->p), st);
        } else {
            rc = bin_learn_strata(c, rects, s->rec2, ctx->strata->p, st);
        }
        if (rc != GS_OK) return fail(rc);
        ctx->spec->strata_state = STRATA_TRIAL;
        ctx->spec->strata_per_tile = ctx->spec->want_per_tile;
        ctx->stats.kernel_launches += ctx->spec->want_per_tile ? 1 : 2;  // k_tile_octiles | k_depth_hist, k_strata_from_hist
    }

    s->P = c.P; s->S = c.S; s->V = c.V; s->H = c.H; s->W = c.W;
    s->flags = c.flags;
    s->has_sh = in->shs != nullptr;
    s->has_scales = in->scales != nullptr;
    ctx->stats.num_rendered = D;
    ctx->stats.num_visible = -1;
    ctx->stats.saved_bytes = (int64_t)(s->bytes + (size_t)(D > 0 ? D : 1) * 4);
    pool_follow(ctx);
    if (saved_out) {
        *saved_out = s;
    } else {
        gs_saved_free(ctx, s, stream);
    }
    return GS_OK;
}

extern "C" int gs_backward(GsContext *ctx, const GsConfig *cfg, const GsInputs *in, const GsSaved *saved,
                           const GsOutGrads *gout, const GsInGrads *gin, void *stream) {
    if (!ctx || !saved || !gout || !gin) return gs_set_error(GS_ERR_INVALID, "null argument");
    int rc = validate(cfg, in);
    if (rc != GS_OK) return rc;
    if (!gout->dL_dcolor) return gs_set_error(GS_ERR_INVALID, "dL_dcolor missing");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    DevCfg c = make_dev_cfg(cfg);
    if (saved->P != c.P || saved->V != c.V || saved->S != c.S || saved->H != c.H || saved->W != c.W)
        return gs_set_error(GS_ERR_INVALID, "saved state does not match the configuration");
    c.flags = saved->flags;
    if (gin->dL_dviewmatrix_z && !(c.flags & GS_FLAG_DEPTH))
        return gs_set_error(GS_ERR_INVALID, "dL_dviewmatrix_z needs a forward with GS_FLAG_DEPTH");
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
    if (n == 0) return GS_OK;

    // Accumulators: n x GS_ACC_STRIDE floats; deterministic mode: n x GS_ACC_STRIDE x 3 int64 limbs + n poison masks
    // (zeroed together), then the per-warp partials of the view-matrix gradient
    const size_t acc_bytes = det ? n * (GS_ACC_STRIDE * GS_DET_LIMBS * 8 + 4) : n * GS_ACC_STRIDE * 4;
    const size_t vz_off = align256(acc_bytes);
    rc = ctx->per_gaussian.reserve(det ? vz_off + det_view_z_bytes(c) : acc_bytes, 1.0, ctx->pool, st);
    if (rc != GS_OK) return rc;
    float *acc = static_cast<float *>(ctx->per_gaussian.p);
    DetAcc da{};
    if (det) {
        unsigned char *base = static_cast<unsigned char *>(ctx->per_gaussian.p);
        da.acc = reinterpret_cast<unsigned long long *>(base);
        da.poison = reinterpret_cast<uint32_t *>(base + n * GS_ACC_STRIDE * GS_DET_LIMBS * 8);
        da.view_z = reinterpret_cast<float *>(base + vz_off);
        acc = nullptr;
    }
    {
        StageTimer t(ctx, GS_STAGE_COMPOSITE_BWD, st);
        GS_CUDA_OK(cudaMemsetAsync(ctx->per_gaussian.p, 0, acc_bytes, st));
        rc = launch_composite_bwd(c, *saved, gout->dL_dcolor, gout->dL_ddepth, acc, st, (cfg->tuning & GS_TUNE_BWD_V1) ? 1 : ((cfg->tuning & GS_TUNE_BWD_OCC4) ? 2 : 0), da);
        if (rc != GS_OK) return rc;
    }
    {
        StageTimer t(ctx, GS_STAGE_PREPROCESS_BWD, st);
        rc = launch_preprocess_bwd(c, di, *saved, acc, g, st, (cfg->tuning & GS_TUNE_PBWD_2PHASE) ? 1 : 0, da);
        if (rc != GS_OK) return rc;
    }
    ctx->stats.kernel_launches += 2;  // k_composite_bwd, k_preprocess_bwd
    if (det && g.dL_dviewmatrix_z) ctx->stats.kernel_launches += 1;  // k_view_z_finalize
    return GS_OK;
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
extern "C" int gs_render_host(GsContext *ctx, const GsConfig *cfg, const GsInputs *in, const GsOutputs *out,
                              void *stream) {
    if (!ctx || !out) return gs_set_error(GS_ERR_INVALID, "null context/outputs");
    int rc = validate(cfg, in);
    if (rc != GS_OK) return rc;
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
    total += align256(px * 12) + align256(VP * 4) + align256(px * 4);
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
            ctx->feed_begin[k] = g;
            ctx->feed_begin[k + 1] = g1;
        }
        pieces = k;
    }
    ctx->feed_chunks = pieces;
    ctx->host_radii_dst = (out->radii && VP) ? out->radii : nullptr;
    ctx->host_radii_bytes = VP * 4;
    dout.color = reinterpret_cast<float *>(base + out_off);
    dout.radii = reinterpret_cast<int32_t *>(base + out_off + align256(px * 12));
    dout.depth = (cfg->flags & GS_FLAG_DEPTH) ? reinterpret_cast<float *>(base + out_off + align256(px * 12) + align256(VP * 4))
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
    ctx->sh_zero_copy = sh_alias != nullptr;
    rc = gs_forward(ctx, &dc, &din, &dout, nullptr, stream);
    ctx->sh_zero_copy = false;
    ctx->host_radii_dst = nullptr;
    ctx->feed_chunks = 0;
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
    GS_CUDA_OK(cudaStreamSynchronize(st));
    GS_CUDA_OK(cudaStreamSynchronize(ctx->copy_stream));  // radii (started after the forward's mid-way sync)
    return GS_OK;
}
