// gs_common.cuh -- shared device/host declarations of the sm_90a (H100) splatting kernels.
//
// Data layout in HBM (DESIGN.md section 4).  Per (view, Gaussian) "splat record", three float4 SoA planes of
// V*P entries each, written by preprocess and gathered by the compositors with 16-byte loads:
//   rec0 = (x_pix, y_pix, -0.5*log2e*conic_a, -log2e*conic_b)
//   rec1 = (-0.5*log2e*conic_c, opacity, r, g)   opacity: o * rho under GS_FLAG_ANTIALIAS (gs_aa_rho)
//   rec2 = (b, z_cam, reach2, fz)     reach2 = -(log2(255*opacity) + margin): a pixel can receive the Gaussian
//                                     only where log2 G >= reach2 (see gs_box_reaches); fz = f(z) of a depth mode
//                                     other than GS_DEPTH_Z (the value its depth channel composites), else 0
// The conic is stored pre-scaled so that the compositors get log2(G) = power*log2(e) with five FP ops and feed
// it straight to ex2.approx (gs_power2 / gs_ex2 below; forward and backward share them bit for bit).
// plus meta[V*P] (uint8: bits 0-2 = SH clamp flags, bit 3 = visible).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/gsplat_b200.h"
#include "gs_bin_policy.h"
#include "gs_det.cuh"

#define GS_TILE 16
#define GS_TILE_PX (GS_TILE * GS_TILE)

#define GS_META_VISIBLE 8u

struct DevCfg {
    int P, S, V, VPS, M, deg, H, W, gx, gy, ntiles;
    uint32_t flags;
    float tanfovx, tanfovy, scale_modifier, near_cull_z, dilation, guard_band;
    const float *view, *proj, *campos, *bg, *tanfov, *view_scale;
};

struct DevInputs {
    const float *means3D, *opacities, *shs, *colors_precomp, *scales, *rotations, *cov3D;
};

// Depth mode of the depth channel (GsConfig::depth_mode).  Passed to the kernels as a trailing parameter of its own
// (DevCfg's layout, and with it every other kernel's parameter offsets, stays as it was).
struct DepthMode {
    int mode;                    // GS_DEPTH_*
    const float *near_far;       // device [V,2] unscaled (near, far), or NULL when the mode reads neither
};

// State a forward keeps for its backward; one stream-ordered allocation carved into planes.
struct GsSaved {
    void *base;
    size_t bytes;
    float4 *rec0, *rec1, *rec2;   // [V*P]
    uint8_t *meta;                // [V*P]
    uint32_t *point_list;         // [D] Gaussian index within its scene, per tile in (depth, index) order
    uint2 *ranges;                // [V*ntiles] [start,end) into point_list
    float *final_T;               // [V*H*W]
    uint32_t *n_contrib;          // [V*H*W] 1-based list position of the last contributor
    uint32_t *sched;              // [2] work counter of the persistent compositor (zeroed by its launcher)
    int64_t D;
    int P, S, V, H, W;
    uint32_t flags;
    int has_sh, has_scales;
    int depth_mode;               // GS_DEPTH_* of the forward (its backward chains the same f'(z))
    const void *ws_base;          // gs_forward_sync_free: the caller's workspace the planes live in (gs_saved_free frees
                                  // only the handle); NULL: the context's pool
};

#define GS_CUDA_OK(call)                                                             \
    do {                                                                             \
        cudaError_t e_ = (call);                                                     \
        if (e_ != cudaSuccess) return gs_set_cuda_error(e_, #call, __FILE__, __LINE__); \
    } while (0)

int gs_set_cuda_error(cudaError_t e, const char *what, const char *file, int line);
int gs_set_error(int code, const char *msg);

// ---- kernel launchers (one translation unit per stage) ----
// How preprocess hands its tile instances to the binning stage.
struct PreEmit {
    uint32_t *counters;   // padded sub-counters [V*tiles*BIN_SUB*BIN_PAD], zeroed: counts (exact path) or cursors
                          // (speculative path, fused emission); NULL = preprocess neither counts nor emits
    uint64_t *bucket;     // fused speculative emission only: fixed-capacity sub-buckets [V*tiles*BIN_SUB][sub_cap]
    uint32_t sub_cap;     // capacity of one sub-bucket (speculative path)
    const float *strata;  // NULL: sub-bucket = index % BIN_SUB.  Else ascending depth boundaries (BIN_SUB - 1 used of
                          // every BIN_SUB): sub-bucket = depth stratum, so that a tile's sorted list is the
                          // concatenation of its independently sorted sub-buckets (gs_binning.cu)
    int strata_per_tile;  // 0: one row of boundaries per view [V][BIN_SUB]; 1: one row per (view, tile) [V*tiles][BIN_SUB]
};

int launch_preprocess(const DevCfg &c, const DevInputs &in, float4 *rec0, float4 *rec1, float4 *rec2, uint8_t *meta,
                      int32_t *radii, ushort4 *rects, const PreEmit &emit, cudaStream_t st, int g_begin = 0,
                      int g_end = -1 /* = P */,
                      int variant = 0 /* bit 0: 80 registers, 6 CTAs/SM (GS_TUNE_PRE_OCC6); bit 1: M > 16 rows staged as 16-byte pieces at their own stride (zero-copy feed, GS_TUNE_PRE_SH_RAW16); bit 2: geometry only, colour words left to k_sh_colour */,
                      const DepthMode &dm = DepthMode{} /* mode != GS_DEPTH_Z: rec2.w = f(z) (the FZ kernels) */);
// the colour words (rec1.zw, rec2.x) of every (view, Gaussian) from the SH block -- gs_render_host's split pipeline
bool sh_colour_supported(const DevCfg &c, const DevInputs &in);
int launch_sh_colour(const DevCfg &c, const DevInputs &in, float4 *rec1, float4 *rec2, uint8_t *clamp_out /* [V*P] or NULL */, cudaStream_t st);
int launch_mark_visible(const DevCfg &c, const float *means3D, uint8_t *present, cudaStream_t st);

// binning (gs_binning.cu)
#define BIN_PAD 8          // uint32 stride between counters: one counter per 32-byte L2 sector
size_t bin_counter_bytes(const DevCfg &c);
int bin_tile_scan(const DevCfg &c, const uint32_t *counters, uint32_t *offsets, uint32_t *tile_start, uint32_t *tile_n,
                  uint32_t *info, cudaStream_t st);
bool bin_fits_fast_path(uint32_t max_count);
size_t bin_scratch_bytes(const DevCfg &c, int64_t D, bool fast);
// offsets != NULL: exact-capacity buckets at offsets[slot]; offsets == NULL: fixed-capacity buckets at slot * sub_cap
int bin_emit_fast(const DevCfg &c, int64_t D, const float4 *rec0, const float4 *rec1, const float4 *rec2,
                  const ushort4 *rects, const uint32_t *offsets, uint32_t sub_cap, const float *strata, int strata_per_tile,
                  uint32_t *cursor, void *scratch, cudaStream_t st);
int bin_sort_fast(const DevCfg &c, uint32_t max_count, const uint32_t *tile_start, const uint32_t *tile_n,
                  const void *scratch, uint32_t *point_list, uint2 *ranges, cudaStream_t st);
int bin_spec_check(const DevCfg &c, uint32_t sub_cap, uint32_t tile_limit, const uint32_t *cursor, uint32_t *info,
                   cudaStream_t st);
int bin_sort_strata(const DevCfg &c, uint32_t sub_cap, const uint32_t *cursor, const void *bucket, uint32_t *point_list,
                    uint2 *ranges, uint32_t *acc /* 8 zeroed words */, uint32_t *info, cudaStream_t st,
                    bool merge_sort = false /* the round-1 cub::BlockMergeSort kernel (GS_TUNE_STRATA_MERGE_SORT) */,
                    const float4 *rec2 = nullptr, float *next_tile_strata = nullptr /* per-tile mode: boundaries of the next call */,
                    const uint8_t *need = nullptr /* lazy strata: sort strata k <= need[vt] only (NULL: all) */);
// per-(view, tile) stratum boundaries from the sorted lists of an exact-path call
int bin_learn_tile_strata(const DevCfg &c, const uint32_t *point_list, const uint2 *ranges, const float4 *rec2, float *table,
                          cudaStream_t st);
// depth strata: per-view octiles of the depths of the binned Gaussians (weighted by their tile count), for the NEXT call
size_t bin_strata_bytes(const DevCfg &c);          // strata table [V][BIN_SUB] floats + histogram scratch + need table
uint8_t *bin_need_table(const DevCfg &c, void *strata_buf);  // lazy strata: [V * ntiles] strata each tile's last forward read
int bin_learn_strata(const DevCfg &c, const ushort4 *rects, const float4 *rec2, void *strata_buf, cudaStream_t st);
int bin_sort_spec(const DevCfg &c, uint32_t sub_cap, uint32_t tile_limit, const uint32_t *cursor, const void *bucket,
                  uint32_t *point_list, uint2 *ranges, cudaStream_t st);
int bin_sort_fallback(const DevCfg &c, int64_t D, const float4 *rec0, const float4 *rec1, const float4 *rec2,
                      const ushort4 *rects, void *scratch, size_t scratch_bytes, uint32_t *point_list, uint2 *ranges,
                      cudaStream_t st);

// Sync-free binning (gs_forward_sync_free, DESIGN.md 5.18): the exact path's count / scan / emit / per-tile sort with
// every size decision on the device, inside a caller-owned workspace of fixed instance capacity.  Status words at the
// workspace's start (uint32): the scan's three result words, this call's verdict, and two words the caller clears.
enum {
    SF_D = 0,          // tile instances of the last forward (saturated at 2^32-1)
    SF_MAX_LIST = 1,   // longest (view, tile) list of the last forward
    SF_MAX_SUB = 2,    // largest sub-counter of the last forward
    SF_VERDICT = 3,    // 1: the last forward's D exceeded the capacity (its planes and its backward's gradients are NaN)
    SF_EXCEEDED = 4,   // 1: some forward since the last clear exceeded the capacity (sticky)
    SF_REQUIRED = 5,   // largest D any forward since the last clear required (sticky)
};
struct SyncFreeBins {
    uint32_t capacity;                        // instances point_list / bucket / tmp hold
    uint32_t *status;                         // SF_* words
    ushort4 *rects;                           // [V*P] candidate tile rectangles (preprocess)
    uint32_t *tile_counts;                    // padded sub-counters, counted by preprocess
    uint32_t *cursor;                         // padded sub-cursors of the emission
    uint32_t *sub_offsets, *tile_start, *tile_n;
    uint64_t *bucket, *tmp;                   // [capacity] keys; tmp: the long-list sort's second buffer
    uint32_t *point_list;                     // [capacity]
    uint2 *ranges;                            // [V*ntiles]
};
int bin_sync_free(const DevCfg &c, const SyncFreeBins &b, const float4 *rec0, const float4 *rec1, const float4 *rec2,
                  cudaStream_t st);
// NaN into every listed array when status[SF_VERDICT] is set (one launch; nothing is written otherwise)
struct SfPoison {
    static constexpr int MAX = 16;
    float *ptr[MAX];
    size_t n[MAX];
    int count;
    void add(float *p, size_t k) {
        if (p && k && count < MAX) { ptr[count] = p; n[count] = k; count++; }
    }
};
int sf_poison_if_exceeded(const uint32_t *status, const SfPoison &arrays, cudaStream_t st);

// Deterministic backward (GS_FLAG_DETERMINISTIC, DESIGN.md 5.11): the composite backward adds its terms into exact
// fixed-point accumulators (gs_det.cuh) instead of the float ones, and the view-matrix gradient is summed in a fixed
// order from per-warp partials.  All NULL on the default path.
struct DetAcc {
    unsigned long long *acc;  // [V*P][GS_ACC_STRIDE][GS_DET_LIMBS], zeroed
    uint32_t *poison;         // [V*P], zeroed: bit k = component k received a non-finite or out-of-range term
    float *view_z;            // [V][warps of one scene's preprocess-backward grid][4] (needs no zeroing)
};

// GS_FLAG_DEPTH: the depth channel composites rec2.y (s.depth_mode == GS_DEPTH_Z) or rec2.w (any other mode); the backward
// compositors take the same word for the depth term of dL/dalpha
// alpha (GsAlpha): the forward also writes 1 - T_final per pixel ([V*H*W]); the backward takes dL/dalpha into the
// background term of every dL/dalpha_i.  NULL: the kernels of before.
// Lazy strata (DESIGN.md 5.2): ranges[vt] covers the sorted strata only; a tile whose pixels are not all saturated at its
// end sorts the next stratum from its sub-bucket into place, extends ranges[vt].y, and records in need[vt] how many
// strata it read.  cursor == NULL: the lists are sorted whole.
struct LazyStrata {
    const uint32_t *cursor;   // the sub-buckets' counts (BIN_PAD stride; clamped to sub_cap)
    const uint64_t *bucket;   // (depth bits << 32 | index) keys, sub-bucket (vt * BIN_SUB + k) at its * sub_cap
    uint32_t sub_cap;
    uint8_t *need;            // [V * ntiles]
};
int launch_composite_fwd(const DevCfg &c, const GsSaved &s, float *color, float *depth, cudaStream_t st,
                         int variant = 0 /* 2: the persistent warp-specialised kernel (GS_TUNE_FWD_WS) */,
                         float *alpha = nullptr, const LazyStrata &lazy = LazyStrata{});
int launch_composite_bwd(const DevCfg &c, const GsSaved &s, const float *dL_dcolor, const float *dL_ddepth,
                         float *grad_acc /* [V*P*GS_ACC_STRIDE], zeroed */, cudaStream_t st,
                         int variant = 0 /* 1: the round-1 kernel (GS_TUNE_BWD_V1) */,
                         const DetAcc &det = DetAcc{} /* det.acc != NULL: fixed-point accumulators instead of grad_acc */,
                         const float *dL_dalpha = nullptr);
// s.depth_mode != GS_DEPTH_Z: the depth gradient is chained through f'(z) (dm.near_far: the backward call's array)
int launch_preprocess_bwd(const DevCfg &c, const DevInputs &in, const GsSaved &s, const float *grad_acc,
                          const GsInGrads &g, cudaStream_t st, int variant = 0 /* 1: the two-phase kernel (GS_TUNE_PBWD_2PHASE) */,
                          const DetAcc &det = DetAcc{}, const DepthMode &dm = DepthMode{},
                          const GsCameraGrads *cam = nullptr /* non-NULL: also the camera gradient */,
                          float *dL_dtanfov = nullptr /* with cam: also dL/dtanfov [V,2] */);
// bytes of DetAcc::view_z for a configuration
size_t det_view_z_bytes(const DevCfg &c);
// bytes of DetAcc::view_z the camera gradient needs, in both modes: per-warp slots of 32 floats per view
size_t camera_grad_scratch_bytes(const DevCfg &c);

// per (view,Gaussian) accumulator written by the composite backward:
//   0-2 dL/drgb, 3-4 dL/dmean2D (NDC-scaled), 5-7 dL/dconic (a, b stored once, c), 8 dL/dopacity, 9 dL/dz
#define GS_ACC_STRIDE 10

// ---------------------------------------------------------------------------------------------------------
// device helpers
// ---------------------------------------------------------------------------------------------------------
#ifdef __CUDACC__

// Column-major flat (transposed) 4x4 times point; the explicit fma chain matches oracle/gs_oracle.c so the
// camera-space depth (the sort key) is bit-identical on both sides.
__device__ __forceinline__ float3 xform4x3(const float *__restrict__ m, float3 p) {
    float3 o;
    o.x = fmaf(m[0], p.x, fmaf(m[4], p.y, fmaf(m[8], p.z, m[12])));
    o.y = fmaf(m[1], p.x, fmaf(m[5], p.y, fmaf(m[9], p.z, m[13])));
    o.z = fmaf(m[2], p.x, fmaf(m[6], p.y, fmaf(m[10], p.z, m[14])));
    return o;
}
__device__ __forceinline__ float4 xform4x4(const float *__restrict__ m, float3 p) {
    float4 o;
    o.x = fmaf(m[0], p.x, fmaf(m[4], p.y, fmaf(m[8], p.z, m[12])));
    o.y = fmaf(m[1], p.x, fmaf(m[5], p.y, fmaf(m[9], p.z, m[13])));
    o.z = fmaf(m[2], p.x, fmaf(m[6], p.y, fmaf(m[10], p.z, m[14])));
    o.w = fmaf(m[3], p.x, fmaf(m[7], p.y, fmaf(m[11], p.z, m[15])));
    return o;
}
__device__ __forceinline__ float ndc2pix(float v, int S) { return ((v + 1.0f) * (float)S - 1.0f) * 0.5f; }

// Camera block of one view, staged in shared memory by every kernel that needs it.
struct ViewCam {
    float view[16];
    float proj[16];
    float campos[3];
    float tanfovx, tanfovy, scale;
    float bg[3];
};

#define GS_CAM_CHUNK 8  // cameras staged per barrier by the per-Gaussian kernels

// Stages cameras [v0, v0+count) into cams[0..count): called by all threads of the block, followed by
// __syncthreads() at the call site.  One barrier pair per GS_CAM_CHUNK views instead of per view.
__device__ __forceinline__ void load_view_cams(const DevCfg &c, int v0, int count, ViewCam *cams) {
    const int nthreads = blockDim.x * blockDim.y;
    for (int t = threadIdx.x + threadIdx.y * blockDim.x; t < count * 41; t += nthreads) {
        const int k = t / 41, f = t - k * 41, v = v0 + k;
        ViewCam *cam = cams + k;
        if (f < 16) cam->view[f] = c.view[v * 16 + f];
        else if (f < 32) cam->proj[f - 16] = c.proj[v * 16 + (f - 16)];
        else if (f < 35) cam->campos[f - 32] = c.campos[v * 3 + (f - 32)];
        else if (f < 38) cam->bg[f - 35] = c.bg ? c.bg[v * 3 + (f - 35)] : 0.0f;
        else if (f == 38) cam->tanfovx = c.tanfov ? c.tanfov[v * 2 + 0] : c.tanfovx;
        else if (f == 39) cam->tanfovy = c.tanfov ? c.tanfov[v * 2 + 1] : c.tanfovy;
        else cam->scale = c.view_scale ? c.view_scale[v] : 1.0f;
    }
}

// Projection Jacobian rows m0,m1 of M = J * Rview and the clamp masks (oracle build_jac).
struct ProjJac {
    float m0[3], m1[3];
    float tx, ty, tz, fx, fy;
    bool xin, yin;
};

__device__ __forceinline__ void build_jac(const ViewCam &cam, const DevCfg &c, float3 mean, ProjJac &o) {
    float3 t = xform4x3(cam.view, mean);
    const float limx = c.guard_band * cam.tanfovx, limy = c.guard_band * cam.tanfovy;
    const float txtz = t.x / t.z, tytz = t.y / t.z;
    o.xin = !(txtz < -limx || txtz > limx);
    o.yin = !(tytz < -limy || tytz > limy);
    t.x = fminf(limx, fmaxf(-limx, txtz)) * t.z;
    t.y = fminf(limy, fmaxf(-limy, tytz)) * t.z;
    o.fx = (float)c.W / (2.0f * cam.tanfovx);
    o.fy = (float)c.H / (2.0f * cam.tanfovy);
    const float J00 = o.fx / t.z, J02 = -(o.fx * t.x) / (t.z * t.z);
    const float J11 = o.fy / t.z, J12 = -(o.fy * t.y) / (t.z * t.z);
#pragma unroll
    for (int j = 0; j < 3; j++) {
        o.m0[j] = J00 * cam.view[j * 4 + 0] + J02 * cam.view[j * 4 + 2];
        o.m1[j] = J11 * cam.view[j * 4 + 1] + J12 * cam.view[j * 4 + 2];
    }
    o.tx = t.x; o.ty = t.y; o.tz = t.z;
}

__device__ __forceinline__ void sym6_mul(const float *c6, const float *v, float *o) {
    o[0] = c6[0] * v[0] + c6[1] * v[1] + c6[2] * v[2];
    o[1] = c6[1] * v[0] + c6[3] * v[1] + c6[4] * v[2];
    o[2] = c6[2] * v[0] + c6[4] * v[1] + c6[5] * v[2];
}

__device__ __forceinline__ void quat_to_R(const float *q, float R[3][3]) {
    const float r = q[0], x = q[1], y = q[2], z = q[3];
    R[0][0] = 1.f - 2.f * (y * y + z * z); R[0][1] = 2.f * (x * y - r * z); R[0][2] = 2.f * (x * z + r * y);
    R[1][0] = 2.f * (x * y + r * z); R[1][1] = 1.f - 2.f * (x * x + z * z); R[1][2] = 2.f * (y * z - r * x);
    R[2][0] = 2.f * (x * z - r * y); R[2][1] = 2.f * (y * z + r * x); R[2][2] = 1.f - 2.f * (x * x + y * y);
}

// Sigma = R diag((mod*s)^2) R^T
__device__ __forceinline__ void cov3d_from_scale_rot(const float *s, float mod, const float *q, float *c6) {
    float R[3][3];
    quat_to_R(q, R);
    const float v0 = mod * s[0] * mod * s[0], v1 = mod * s[1] * mod * s[1], v2 = mod * s[2] * mod * s[2];
    c6[0] = R[0][0] * v0 * R[0][0] + R[0][1] * v1 * R[0][1] + R[0][2] * v2 * R[0][2];
    c6[1] = R[0][0] * v0 * R[1][0] + R[0][1] * v1 * R[1][1] + R[0][2] * v2 * R[1][2];
    c6[2] = R[0][0] * v0 * R[2][0] + R[0][1] * v1 * R[2][1] + R[0][2] * v2 * R[2][2];
    c6[3] = R[1][0] * v0 * R[1][0] + R[1][1] * v1 * R[1][1] + R[1][2] * v2 * R[1][2];
    c6[4] = R[1][0] * v0 * R[2][0] + R[1][1] * v1 * R[2][1] + R[1][2] * v2 * R[2][2];
    c6[5] = R[2][0] * v0 * R[2][0] + R[2][1] * v1 * R[2][1] + R[2][2] * v2 * R[2][2];
}

// sub-bucket of depth d under one row of ascending per-(view, tile) boundaries (two 16-byte loads)
__device__ __forceinline__ uint32_t gs_tile_stratum(const float *__restrict__ table, uint32_t tile, float d) {
    const float4 *tb = reinterpret_cast<const float4 *>(table) + (size_t)tile * (BIN_SUB / 4);
    const float4 b0 = __ldg(tb), b1 = __ldg(tb + 1);
    return (uint32_t)(d >= b0.x) + (uint32_t)(d >= b0.y) + (uint32_t)(d >= b0.z) + (uint32_t)(d >= b0.w) + (uint32_t)(d >= b1.x) +
           (uint32_t)(d >= b1.y) + (uint32_t)(d >= b1.z);
}

#define GS_LOG2E 1.4426950408889634f
#define GS_ALPHA_MIN (1.0f / 255.0f)
#define GS_ALPHA_MAX 0.99f
#define GS_T_MIN 0.0001f

// log2 of the Gaussian falloff at offset (dx,dy) from the centre, from the pre-scaled conic in rec0/rec1.
// Explicit round-to-nearest intrinsics: no re-association or contraction, so the forward and backward
// compositors take identical skip decisions.
__device__ __forceinline__ float gs_power2(float hA, float nB, float hC, float dx, float dy) {
    const float t1 = __fmaf_rn(hA, dx, __fmul_rn(nB, dy));
    const float t2 = __fmul_rn(hC, dy);
    return __fmaf_rn(dx, t1, __fmul_rn(dy, t2));
}
// Can the Gaussian reach (alpha >= 1/255) ANY point of the axis-aligned box [x0,x1] x [y0,y1] (pixel coordinates)?
// Exact for the continuous box, hence conservative for the pixel centres inside it: the maximum of the concave
// quadratic log2 G over the box is 0 if the centre is inside, else it lies on one of the two edges facing the
// centre, where it is a clamped 1-D maximisation.  Used for tile binning (16x16 boxes) and for the compositors'
// per-warp culling (8x4 boxes); reach2 carries the rounding margin.
__device__ __forceinline__ bool gs_box_reaches(float cx, float cy, float hA, float nB, float hC, float reach2,
                                               float x0, float x1, float y0, float y1) {
    const float bx0 = x0 - cx, bx1 = x1 - cx, by0 = y0 - cy, by1 = y1 - cy;
    const float xe = fminf(fmaxf(0.0f, bx0), bx1), ye = fminf(fmaxf(0.0f, by0), by1);  // box point nearest the centre
    // edge x = xe: best y solves d/dy = nB*xe + 2*hC*y = 0 ; edge y = ye: best x solves nB*ye + 2*hA*x = 0
    const float yb = fminf(fmaxf(__fdividef(-nB * xe, 2.0f * hC), by0), by1);
    const float xb = fminf(fmaxf(__fdividef(-nB * ye, 2.0f * hA), bx0), bx1);
    const float p1 = gs_power2(hA, nB, hC, xe, yb), p2 = gs_power2(hA, nB, hC, xb, ye);
    return fmaxf(p1, p2) >= reach2;
}

// The binning predicate shared by k_preprocess (counting) and k_emit_buckets (emission): does the Gaussian with
// records (r0, r1, r2) reach tile (tx, ty)?  Both kernels evaluate it on the same stored values.
__device__ __forceinline__ bool gs_tile_reached(float4 r0, float4 r1, float4 r2, int tx, int ty) {
    const float x0 = (float)(tx * GS_TILE), y0 = (float)(ty * GS_TILE);
    return gs_box_reaches(r0.x, r0.y, r0.z, r0.w, r1.x, r2.z, x0, x0 + (float)(GS_TILE - 1), y0, y0 + (float)(GS_TILE - 1));
}

__device__ __forceinline__ float gs_ex2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

__device__ __forceinline__ float gs_rcp(float x) {
    float y;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// Depth modes other than GS_DEPTH_Z (render_depth_cuda, cuda_splatting.py:245-251, with depth_to_relative_disparity of
// conversions.py:17-27 in its own expression order): the fake colour f at the UNSCALED depth z, and the factor
// f'(z) * dz/dz_s that carries dL/df onto the view-scaled depth z_s = s z the kernels work with.  IEEE division (the
// default '/'); the mode is a uniform runtime branch.
#define GS_DEPTH_EPS 1e-10f
__device__ __forceinline__ float gs_depth_f(int mode, float z, float near_, float far_) {
    if (mode == GS_DEPTH_DISPARITY) return 1.0f / z;
    if (mode == GS_DEPTH_RELATIVE_DISPARITY) {
        const float d = 1.0f / (z + GS_DEPTH_EPS), dn = 1.0f / (near_ + GS_DEPTH_EPS), df = 1.0f / (far_ + GS_DEPTH_EPS);
        return 1.0f - (d - df) / (dn - df + GS_DEPTH_EPS);
    }
    return logf(fmaxf(fminf(z, near_), far_));   // GS_DEPTH_LOG, the clamp as written
}
__device__ __forceinline__ float gs_depth_chain(int mode, float zs, float s, float near_, float far_) {
    const float z = zs / s;
    if (mode == GS_DEPTH_DISPARITY) return -1.0f / (z * z) / s;
    if (mode == GS_DEPTH_RELATIVE_DISPARITY) {
        const float dn = 1.0f / (near_ + GS_DEPTH_EPS), df = 1.0f / (far_ + GS_DEPTH_EPS), ze = z + GS_DEPTH_EPS;
        return 1.0f / (ze * ze * (dn - df + GS_DEPTH_EPS)) / s;
    }
    // GS_DEPTH_LOG: d/dz log(max(min(z, near), far)) = 1/z where z passes both clamps (never, for near < far)
    return (z < near_ && z > far_) ? 1.0f / z / s : 0.0f;
}

// Anti-aliasing (GS_FLAG_ANTIALIAS, DESIGN.md 5.1): the screen-space filter's opacity compensation.  (a0, b, c0) is the
// projected 2-D covariance before the dilation h, det1 = (a0 + h)(c0 + h) - b^2 the determinant after it; the splat is
// drawn with the dilated covariance at opacity o * rho, rho = sqrt(max(GS_AA_RATIO_MIN, (a0 c0 - b^2) / det1)), so
// that its footprint keeps the weight of the undilated one.  Preprocess and its backward evaluate the same expressions.
#define GS_AA_RATIO_MIN 0.000025f
__device__ __forceinline__ float gs_aa_ratio(float a0, float b, float c0, float det1) { return (a0 * c0 - b * b) / det1; }
__device__ __forceinline__ float gs_aa_rho(float ratio) { return sqrtf(fmaxf(GS_AA_RATIO_MIN, ratio)); }

#define GS_SH_C0 0.28209479177387814f
#define GS_SH_C1 0.4886025119029199f
#define GS_SH_C2_0 1.0925484305920792f
#define GS_SH_C2_1 (-1.0925484305920792f)
#define GS_SH_C2_2 0.31539156525252005f
#define GS_SH_C2_3 (-1.0925484305920792f)
#define GS_SH_C2_4 0.5462742152960396f
#define GS_SH_C3_0 (-0.5900435899266435f)
#define GS_SH_C3_1 2.890611442640554f
#define GS_SH_C3_2 (-0.4570457994644658f)
#define GS_SH_C3_3 0.3731763325901154f
#define GS_SH_C3_4 (-0.4570457994644658f)
#define GS_SH_C3_5 1.445305721320277f
#define GS_SH_C3_6 (-0.5900435899266435f)
// band 4 (opt-in, GsConfig::sh_eval_max_degree = 4): the same real, orthonormal, Condon-Shortley-signed basis continued,
// on the unit view direction.  Coefficients 16..24 multiply
//   xy(xx-yy), yz(3xx-yy), xy(7zz-1), yz(7zz-3), zz(35zz-30)+3, xz(7zz-3), (xx-yy)(7zz-1), xz(xx-3yy),
//   xx(xx-3yy)-yy(3xx-yy)
// (the "-1" / "-3" forms hold on the unit sphere only; kernels and oracles use these forms alike)
#define GS_SH_C4_0 2.5033429417967046f
#define GS_SH_C4_1 (-1.7701307697799304f)
#define GS_SH_C4_2 0.9461746957575601f
#define GS_SH_C4_3 (-0.6690465435572892f)
#define GS_SH_C4_4 0.10578554691520431f
#define GS_SH_C4_5 (-0.6690465435572892f)
#define GS_SH_C4_6 0.47308734787878004f
#define GS_SH_C4_7 (-1.7701307697799304f)
#define GS_SH_C4_8 0.6258357354491761f

// ---- mbarrier + 1-D bulk TMA (cp.async.bulk) primitives ----
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// the mbarrier receives one arrival from this thread once all cp.async copies it has issued so far have landed
// (the barrier's expected count must already include that arrival: .noinc)
__device__ __forceinline__ void cp_async_mbar_arrive(uint64_t *bar) {
    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t phase) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(phase)
        : "memory");
}
// global -> shared bulk copy (TMA engine, SASS UBLKCP); bytes % 16 == 0, both addresses 16-byte aligned
__device__ __forceinline__ void tma_load_1d(void *smem_dst, const void *gsrc, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// shared -> global bulk store
__device__ __forceinline__ void tma_store_1d(void *gdst, const void *smem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(smem_src)),
                 "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void tma_store_commit_wait() {
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// shared-memory accesses with a precomputed 32-bit shared address (keeps the address arithmetic of the
// compositors' inner loops to one IMAD; the compiler otherwise rebuilds the shared-window base every iteration)
__device__ __forceinline__ float4 lds128(uint32_t addr) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
    return v;
}
__device__ __forceinline__ float lds32(uint32_t addr) {
    float v;
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ float2 lds64(uint32_t addr) {
    float2 v;
    asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr));
    return v;
}

// 16-byte cp.async (LDGSTS): the compositors gather the next batch of splat records into shared memory with it
// while they work on the current one
__device__ __forceinline__ void cp_async16(void *smem_dst, const void *gsrc) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
// 4-byte cp.async: gathers of rows that are only 4-byte aligned (the 12*M-byte SH rows)
__device__ __forceinline__ void cp_async4(void *smem_dst, const void *gsrc) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
#endif  // __CUDACC__
