/*
 * gsplat_b200.h -- C ABI of the H100-native (sm_90a) differentiable Gaussian-splatting rasterizer.
 *
 * This is the drop-in boundary for the hot path of cvlab-kaist/PF3plat: the
 * `diff_gaussian_rasterization` extension it imports at
 *   PF3plat's src/model/decoder/cuda_splatting.py:5-8
 * and calls at :99-124 (perspective), :192-217 (orthographic) and, through
 * render_depth_cuda, :255-268.  The reference has no C ABI of its own (its
 * boundary is a pybind/torch extension, absent from the tree:
 * PF3plat's requirements.txt:2); every entry point below names the piece
 * of that Python surface it stands behind.  INTEGRATION.md shows the
 * reference-side binding (the ctypes stub `diff_gaussian_rasterization/`
 * shipped in this repo).
 *
 * Conventions
 *  - plain C, no torch types; all device pointers are fp32/int32 arrays in the
 *    CUDA device current on the calling thread; `stream` is a cudaStream_t
 *    passed as void*.
 *  - every function returns 0 on success or a negative GS_ERR_* code; no
 *    exceptions cross the ABI; gs_last_error() gives a text for the calling
 *    thread's last failure.
 *  - 4x4 matrices are the TRANSPOSED (row-vector) matrices exactly as the
 *    reference passes them (cuda_splatting.py:85-87), i.e. column-major flats.
 *  - one call renders V views of S scenes (V % S == 0, view v shows scene
 *    v / (V/S)); the reference's per-view call is S = V = 1.
 */
#ifndef GSPLAT_B200_H
#define GSPLAT_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GS_ABI_VERSION 5   /* 5: GsConfig::depth_mode, depth_near_far appended; 4: sh_eval_max_degree = 4 evaluates band 4 */

#if defined(__GNUC__)
#define GS_API __attribute__((visibility("default")))
#else
#define GS_API
#endif

enum {
    GS_OK = 0,
    GS_ERR_INVALID = -1,   /* bad argument combination (mirrors the ValueErrors of GaussianRasterizer.forward) */
    GS_ERR_CUDA = -2,      /* a CUDA runtime call failed */
    GS_ERR_OOM = -3,       /* device allocation failed */
    GS_ERR_OVERFLOW = -4,  /* more than 2^31-1 tile instances */
    GS_ERR_NO_DEVICE = -5
};

enum {
    GS_FLAG_DEPTH = 1u,        /* also composite a depth channel (render_depth_cuda, cuda_splatting.py:226-269, fused): camera-space z, or f(z) of GsConfig::depth_mode */
    GS_FLAG_PREFILTERED = 2u,  /* GaussianRasterizationSettings.prefiltered */
    /* gs_backward: bit-reproducible gradients.  The composite backward adds its per-(view, Gaussian) terms as exact
     * fixed-point integers (2^-80 resolution, terms up to 2^45 in magnitude; NaN, Inf or larger terms make that gradient
     * component NaN) instead of float atomics, and the view-matrix gradient is summed in a fixed order.  Needs
     * 244 B instead of 40 B of context scratch per (view, Gaussian); frames with ceil(H/4) * ceil(W/8) >= 2^21 and
     * GS_TUNE_BWD_V1 are rejected (GS_ERR_INVALID).  The forward ignores it: it is deterministic already. */
    GS_FLAG_DETERMINISTIC = 4u,
    /* Anti-aliasing: the screen-space filter with opacity compensation (Mip-Splatting's 2-D filter, upstream's
     * `antialiasing` setting).  Per (view, Gaussian), with (a0, b, c0) the projected 2-D covariance before the dilation
     * h = GsConfig::dilation, the splat is drawn with the dilated covariance (a0 + h, b, c0 + h), as always, but at opacity
     * o * rho, rho = sqrt(max(2.5e-5, (a0 c0 - b^2) / ((a0 + h)(c0 + h) - b^2))): a sub-pixel splat keeps the weight of
     * its own footprint instead of covering the dilated one at full opacity.  Tile binning uses o * rho.  The backward
     * differentiates rho into opacities, covariances or scales / rotations and means (not the cameras); it follows its
     * forward's setting, whatever its own flags say.  GS_TUNE_PRE_OCC6 and GS_TUNE_PBWD_2PHASE have no anti-aliased
     * kernels: with this flag they are GS_ERR_INVALID.  Libraries that predate it ignore the bit: see
     * gs_supported_flags(). */
    GS_FLAG_ANTIALIAS = 8u
};

enum {
    GS_TUNE_FORCE_RADIX_BINNING = 1u, /* use the device-wide radix-sort binning even when every tile list fits shared memory */
    GS_TUNE_NO_SPECULATION = 2u,      /* always size the tile buckets exactly (count + scan + emit passes, mid-call sync) */
    GS_TUNE_SEPARATE_EMIT = 4u,       /* speculative path: fill the buckets with k_emit_buckets even when they fit L2 */
    GS_TUNE_NO_STRATA = 8u,           /* speculative path: never bin by depth stratum (whole-tile sorts only) */
    GS_TUNE_BWD_V1 = 16u,             /* backward compositor: the round-1 kernel (per-pixel 10-component gradients + transpose-reduce) instead of the pair-matrix kernel (A/B) */
    GS_TUNE_FWD_WS = 32u,             /* forward compositor: the persistent warp-specialised kernel (producer warp + 8 consumer warps over an mbarrier ring) instead of the barrier-synchronised one-CTA-per-tile kernel (A/B: a tie on C2, DESIGN.md 5.3) */
    GS_TUNE_STRATA_MERGE_SORT = 64u,  /* stratified binning: sort the strata with the round-1 cub::BlockMergeSort kernel instead of the hand-written warp-per-stratum distribution sort (A/B) */
    GS_TUNE_BWD_OCC4 = 128u,          /* backward compositor: batches of 128 entries and 64 registers (4 CTAs/SM) instead of 256 / 80 (3 CTAs/SM) (A/B) */
    GS_TUNE_PRE_OCC6 = 4096u,         /* preprocess: registers bounded to 80 (6 CTAs/SM) instead of unbounded (96, 5 CTAs/SM) (A/B) */
    GS_TUNE_PBWD_2PHASE = 8192u,      /* preprocess backward: the two-phase kernel (geometry, then one pass per colour channel: 80 registers) instead of the single-pass one (128 registers) (A/B: slower) */
    GS_TUNE_NO_TILE_STRATA = 16384u,  /* stratified binning: never fall back to per-(view, tile) boundaries when the per-view trial overflows (the shape then stays on whole-tile sorts) */
    GS_TUNE_DIRECT_OUTPUT = 32768u,   /* gs_render_host: the compositor writes the images directly into pinned caller buffers instead of a device-to-host copy afterwards (A/B: 1 % slower) */
    GS_TUNE_PRE_SH_RAW16 = 65536u,    /* preprocess, M > 16, device-resident SH: stage 16-byte pieces at the rows' own stride (what the zero-copy feed of gs_render_host uses) instead of gathering the 16 evaluated coefficients with 4-byte copies into compacted rows (A/B: 0.246 vs 0.220 ms on C2) */
    GS_TUNE_NO_ZERO_COPY = 131072u,   /* gs_render_host: always upload the SH block with the copy engine (in pieces) even when the caller's buffer is pinned and preprocess could pull it over PCIe itself (A/B) */
    GS_TUNE_NO_SPLIT_COLOUR = 262144u, /* gs_render_host, zero-copy feed: one fused preprocess pulling the SH block instead of geometry + tile sort on the launch stream with k_sh_colour pulling the block on a second stream (A/B) */
    GS_TUNE_ALL_STRATA = 524288u,     /* per-view stratified binning: the stratum sort sorts every stratum of every tile instead of those the tile's previous forward reached (+1); the reference of the lazily sorted lists (A/B) */
    GS_TUNE_FEED_PIECES_SHIFT = 8     /* gs_render_host: bits 8..11 = pieces the SH block is copied in (0 default, 1 = one plain copy) */
};

/* What the depth channel (GS_FLAG_DEPTH) composites: PF3plat's DepthRenderingMode (cuda_splatting.py:223-251), whose
 * fake colour f(z) render_depth_cuda builds from the UNSCALED camera-space depth z of each mean and the unscaled near
 * and far of the view.  The kernels see z_s = view_scale * z and evaluate f at z = z_s / view_scale. */
enum {
    GS_DEPTH_Z = 0,                  /* "depth": z_s itself (the caller multiplies by 1 / view_scale); default */
    GS_DEPTH_DISPARITY = 1,          /* "disparity": 1 / z */
    GS_DEPTH_RELATIVE_DISPARITY = 2, /* "relative_disparity": 1 - (1/(z+e) - 1/(far+e)) / (1/(near+e) - 1/(far+e) + e), e = 1e-10 */
    GS_DEPTH_LOG = 3                 /* "log": log(max(min(z, near), far)) -- the reference's clamp as written: log(far) for near < far */
};

/* GaussianRasterizationSettings (cuda_splatting.py:99-112), batched over views. */
typedef struct GsConfig {
    int32_t P;            /* Gaussians per scene */
    int32_t S;            /* scenes */
    int32_t V;            /* views in this call */
    int32_t M;            /* SH coefficients per channel = shs.shape[1]; 0 with colors_precomp */
    int32_t sh_degree;    /* settings.sh_degree */
    int32_t image_height; /* settings.image_height */
    int32_t image_width;  /* settings.image_width */
    uint32_t flags;       /* GS_FLAG_* */
    float tanfovx;        /* settings.tanfovx / tanfovy: used for every view when `tanfov` is NULL */
    float tanfovy;
    float scale_modifier; /* settings.scale_modifier */
    /* constants of the upstream algorithm; 0 selects the default (SURVEY.md Appendix C.1) */
    float near_cull_z;    /* default 0.2 */
    float dilation;       /* default 0.3 */
    float guard_band;     /* default 1.3 */
    /* Highest SH degree evaluated: default 3 (<=0 selects it), 4 opts in to band 4 (values above 4 evaluate 4).  The
     * degree evaluated is min(sh_degree, sh_eval_max_degree, the largest degree M covers).  Degree 4 rejects
     * GS_TUNE_PRE_OCC6 and GS_TUNE_PBWD_2PHASE (GS_ERR_INVALID).  ABI versions < 4 evaluated at most degree 3
     * whatever this field said. */
    int32_t sh_eval_max_degree;
    uint32_t tuning;      /* GS_TUNE_* implementation knobs (testing); 0 = default */
    const float *viewmatrix; /* device [V,16]  settings.viewmatrix */
    const float *projmatrix; /* device [V,16]  settings.projmatrix */
    const float *campos;     /* device [V,3]   settings.campos */
    const float *bg;         /* device [V,3]   settings.bg */
    const float *tanfov;     /* device [V,2] or NULL */
    const float *view_scale; /* device [V] or NULL: per-view factor s applied as mean*s, cov*s^2, scales*s
                                (the 1/near rescale of cuda_splatting.py:64-71 without materialising copies) */
    /* GS_DEPTH_*: what the depth channel composites.  A mode other than GS_DEPTH_Z needs GS_FLAG_DEPTH; an unknown mode,
     * or GS_DEPTH_RELATIVE_DISPARITY / GS_DEPTH_LOG without depth_near_far, is GS_ERR_INVALID.  A backward uses the mode
     * of its forward (the field is ignored there, depth_near_far is read again).  dL_dviewmatrix_z works in every mode. */
    int32_t depth_mode;
    const float *depth_near_far; /* device [V,2]: unscaled (near, far) per view, or NULL (GS_DEPTH_Z, GS_DEPTH_DISPARITY) */
} GsConfig;

/* Arguments of GaussianRasterizer.forward (cuda_splatting.py:117-124).  Exactly one of shs/colors_precomp and
 * exactly one of (scales,rotations)/cov3D_precomp must be non-NULL, as the reference op requires. */
typedef struct GsInputs {
    const float *means3D;        /* device [S,P,3] */
    const float *opacities;      /* device [S,P] */
    const float *shs;            /* device [S,P,M,3] or NULL */
    const float *colors_precomp; /* device [V,P,3] or NULL (per VIEW: PF3plat passes view-dependent fake colours) */
    const float *scales;         /* device [S,P,3] or NULL */
    const float *rotations;      /* device [S,P,4] (w,x,y,z) or NULL */
    const float *cov3D_precomp;  /* device [S,P,6] (xx,xy,xz,yy,yz,zz) or NULL */
} GsInputs;

/* Return values of GaussianRasterizer.forward: (color, radii); depth is the opt-in extra. */
typedef struct GsOutputs {
    float *color;   /* device [V,3,H,W] */
    int32_t *radii; /* device [V,P] */
    float *depth;   /* device [V,H,W], required iff GS_FLAG_DEPTH */
} GsOutputs;

/* Incoming gradients of backward. */
typedef struct GsOutGrads {
    const float *dL_dcolor; /* device [V,3,H,W] */
    const float *dL_ddepth; /* device [V,H,W] or NULL */
} GsOutGrads;

/* Gradients returned by the reference autograd Function (SURVEY.md section 8 a3).  Any pointer may be NULL.
 * Per-scene gradients are SUMMED over the views of the scene inside the kernel (V/S == 1 in the drop-in). */
typedef struct GsInGrads {
    float *dL_dmeans3D;    /* device [S,P,3] */
    float *dL_dmeans2D;    /* device [V,P,3] screen-space (NDC-scaled) gradient, z = 0 */
    float *dL_dshs;        /* device [S,P,M,3] */
    float *dL_dcolors;     /* device [V,P,3] */
    float *dL_dopacities;  /* device [S,P] */
    float *dL_dscales;     /* device [S,P,3] */
    float *dL_drotations;  /* device [S,P,4] */
    float *dL_dcov3D;      /* device [S,P,6] */
    /* device [V,4]: dL/d(viewmatrix flat entries 2, 6, 10, 14), the z column of the transposed view matrix, through the
     * fused depth channel only (z = that column . (view_scale * mean, 1)), as render_depth_cuda's fake colour carries it
     * (cuda_splatting.py:239-242); in a depth mode other than GS_DEPTH_Z, through f(z) of that mode (GS_DEPTH_LOG with
     * near < far: zeros).  Colour, projection and culling give the cameras no gradient.  NULL = not wanted;
     * needs GS_FLAG_DEPTH.  Written, not accumulated; zeros when dL_ddepth is NULL. */
    float *dL_dviewmatrix_z;
} GsInGrads;

/* Accumulated opacity, the opt-in third image of the colour pass: alpha = 1 - T_final per pixel, with the T_final the
 * colour composites the background with (same 1/255 threshold, 0.99 clamp and early stop), exactly 0 where nothing
 * contributes.  Its gradient reaches means, 2-D means, covariances or scales / rotations and opacities; SH, colours and
 * cameras get nothing from it.  Taken by the _ex entry points below (GsOutputs and GsOutGrads keep their layout). */
typedef struct GsAlpha {
    float *alpha;            /* gs_forward_ex: device [V,H,W]; gs_render_host_ex: host [V,H,W].  Required there; ignored
                                by gs_backward_ex */
    const float *dL_dalpha;  /* gs_backward_ex: device [V,H,W], or NULL (the gradients of gs_backward, bit for bit);
                                ignored by the forward entries */
} GsAlpha;

/* Counters of the last forward on a context (host-visible after the call returns). */
typedef struct GsStats {
    int64_t num_rendered;  /* tile instances after culling (the "D" of SURVEY.md section 8(d)) */
    int64_t num_visible;   /* Gaussians with radius > 0, summed over views */
    int64_t saved_bytes;   /* bytes held by the GsSaved handle */
    int64_t scratch_bytes; /* bytes of grow-only scratch held by the context */
    int32_t kernel_launches; /* OUR kernels launched by the last forward (+ backward, if it followed); CUB's scan/sort launches are not counted */
    int32_t max_tile_list;   /* longest (view, tile) list of the last forward */
    int32_t speculative;     /* last forward: 0 exact capacities; 1 speculative capacities (no count/scan/emit passes); 2 the same, binned by depth stratum */
    int32_t overflow_redos;  /* cumulative over the context's life: speculative forwards whose capacities overflowed and that were redone exactly */
    int64_t pool_reserved_bytes; /* the context's private memory pool right now: physical memory it holds ... */
    int64_t pool_used_bytes;     /* ... and how much of it is handed out (saved states alive + scratch) */
} GsStats;

typedef struct GsContext GsContext; /* per (device, caller) workspace; not thread-safe, one call at a time */
typedef struct GsSaved GsSaved;     /* state a forward keeps for its backward (what upstream hands autograd as 3 byte tensors) */

GS_API int gs_abi_version(void);
GS_API const char *gs_last_error(void);
/* The GS_FLAG_* bits this library honours (unknown bits of GsConfig::flags are ignored, not refused): a host checks it
 * before it relies on a flag that a library of the same ABI version may predate, such as GS_FLAG_ANTIALIAS. */
GS_API uint32_t gs_supported_flags(void);

/* Workspace lifetime (upstream allocates scratch through torch callbacks on every call; here it is a grow-only cache). */
GS_API int gs_context_create(GsContext **out);
GS_API void gs_context_destroy(GsContext *ctx);
/* Saved state and scratch come from a PRIVATE stream-ordered memory pool of the context (not the device's default
 * pool, and outside the caller's allocator).  Freed blocks stay cached for the next calls (every 256 forwards the pool is
 * trimmed if it holds more than twice what those calls needed at any one time); this hands everything that is not in use
 * back to the driver (call it where the host framework empties its own caches). */
GS_API int gs_context_trim(GsContext *ctx);

/*
 * Forward = _RasterizeGaussians.forward -> _C.rasterize_gaussians (SURVEY.md section 3.4): preprocess,
 * bin/sort, composite.  If `saved` is non-NULL a handle for gs_backward is returned (free it with
 * gs_saved_free); pass NULL for inference.  Performs ONE host synchronisation per call (upstream: one per view): on
 * the first call of a shape it sizes the tile-instance list mid-way; later calls reuse the learned bucket capacities
 * and only verify at the end that nothing overflowed (redoing the call exactly if it did).
 */
GS_API int gs_forward(GsContext *ctx, const GsConfig *cfg, const GsInputs *in, const GsOutputs *out, GsSaved **saved,
               void *stream);

/* Backward = _RasterizeGaussians.backward -> _C.rasterize_gaussians_backward. */
GS_API int gs_backward(GsContext *ctx, const GsConfig *cfg, const GsInputs *in, const GsSaved *saved,
                const GsOutGrads *gout, const GsInGrads *gin, void *stream);

/* gs_forward that also writes the accumulated opacity to alpha->alpha (GsAlpha).  Colour, depth and radii are the
 * bytes gs_forward writes, and the saved state is the same: either backward entry takes it. */
GS_API int gs_forward_ex(GsContext *ctx, const GsConfig *cfg, const GsInputs *in, const GsOutputs *out,
                         const GsAlpha *alpha, GsSaved **saved, void *stream);

/* gs_backward with an incoming gradient of the accumulated opacity (alpha->dL_dalpha, may be NULL).  Works on the
 * saved state of either forward entry: the opacity is 1 - the T_final every forward saves. */
GS_API int gs_backward_ex(GsContext *ctx, const GsConfig *cfg, const GsInputs *in, const GsSaved *saved,
                          const GsOutGrads *gout, const GsAlpha *alpha, const GsInGrads *gin, void *stream);

/* Camera gradient, opt-in (gs_backward_cam): dL/d of the three camera inputs of GsConfig, per view and in their own
 * layouts -- the exact partial derivatives of what the kernels compute, everything else held fixed.  They take in every
 * output of the forward: colour (from SH or colors_precomp), the depth channel in every depth_mode (through f'(z);
 * GS_DEPTH_LOG's clamp gives zero), the accumulated opacity and the anti-aliasing factor.  A guard-band-clamped t.x / t.y
 * has no gradient, an invisible or culled (view, Gaussian) pair contributes nothing, and the 0.99 alpha clamp passes the
 * gradient straight through, as for the means.  The values are in the view-scaled scene (GsConfig.view_scale), so they
 * are gradients of the matrices as passed.  tanfov gets its gradient from gs_backward_cam_tanfov; near, far and bg get
 * none.  Each pointer is device memory or NULL (not wanted); the arrays are written, not accumulated.  Deterministic:
 * per-warp partials summed in a fixed order, in both modes. */
typedef struct GsCameraGrads {
    float *dL_dviewmatrix;  /* device [V,16]: the flat transposed world-to-camera matrix (GsConfig.viewmatrix) */
    float *dL_dprojmatrix;  /* device [V,16]: the flat transposed full projection (GsConfig.projmatrix) */
    float *dL_dcampos;      /* device [V,3] (GsConfig.campos) */
} GsCameraGrads;

/* gs_backward_ex that also writes the camera gradient (cam, not NULL).  alpha may be NULL (no incoming dL/dalpha).  It
 * contains the depth channel's z column, so gin->dL_dviewmatrix_z must be NULL (else GS_ERR_INVALID).  GS_TUNE_PBWD_2PHASE
 * has no camera-gradient kernel: GS_ERR_INVALID. */
GS_API int gs_backward_cam(GsContext *ctx, const GsConfig *cfg, const GsInputs *in, const GsSaved *saved,
                           const GsOutGrads *gout, const GsAlpha *alpha, const GsInGrads *gin, const GsCameraGrads *cam,
                           void *stream);

/* gs_backward_cam that also writes dL/dtanfov (device [V,2], x then y per view; NULL = not wanted): the partial derivative
 * of what the kernels compute with respect to the tangent of the half field of view (GsConfig.tanfov, or tanfovx/tanfovy
 * for every view) as passed, projmatrix held fixed -- its 1/tanfov entries are a separate input, with their own gradient
 * in cam.  tanfov enters through the focal lengths of the projection Jacobian, fx = W / (2 tanfovx), and through the
 * guard-band clamp of the Jacobian's evaluation point, t.x = clamp(t.x / t.z, +-guard_band tanfovx) t.z (y likewise).
 * It reaches every output that reads the 2-D covariance: colour, the depth channel, the accumulated opacity and the
 * anti-aliasing factor.  Culling, radii and tile binning are discrete and give none.  The camera outputs in cam are the
 * bytes gs_backward_cam writes, with or without dL_dtanfov.  Same refusals as gs_backward_cam. */
GS_API int gs_backward_cam_tanfov(GsContext *ctx, const GsConfig *cfg, const GsInputs *in, const GsSaved *saved,
                                  const GsOutGrads *gout, const GsAlpha *alpha, const GsInGrads *gin,
                                  const GsCameraGrads *cam, float *dL_dtanfov, void *stream);

GS_API void gs_saved_free(GsContext *ctx, GsSaved *saved, void *stream);

/*
 * Sync-free forward and backward (opt-in, DESIGN.md 5.18): the host never waits for the device, nothing is allocated or
 * freed and nothing is read back during a call, so a training step around them can be captured in a CUDA graph.  Every
 * buffer lives in one caller-owned workspace of gs_sync_free_workspace_bytes(cfg, instance_capacity, needs) bytes
 * (256-byte aligned) that holds at most `instance_capacity` tile instances (the D of GsStats::num_rendered).  The
 * binning is the exact path's (count, scan, emit, per-tile sort) with every size decision taken on the device.
 * When a call's D is at most the capacity, colour, depth, alpha and radii are the bytes gs_forward / gs_forward_ex
 * write, and the gradients those of gs_backward_cam_tanfov (bit for bit under GS_FLAG_DETERMINISTIC).  When it is
 * larger, nothing is binned: colour, depth and alpha are NaN, the radii are still right, and the backward of that
 * forward writes NaN into every gradient it produces -- an undersized workspace costs a skipped optimizer step, never a
 * silently wrong one.  The first 32 bytes of the workspace are uint32 status words: [0] D of the last forward,
 * [1] its longest tile list, [3] 1 if it exceeded the capacity, [4] 1 if any forward exceeded it since the caller last
 * zeroed the words, [5] the largest D any forward required since then (words [4] and [5] are only ever raised).
 * The context's learned shapes, its pool and its pinned read-back word are not touched; GsStats reports
 * num_rendered = num_visible = max_tile_list = -1 for a sync-free forward.  The GsSaved of a sync-free forward points
 * into the workspace: gs_saved_free releases only the handle, and the next forward on the same workspace overwrites
 * what the backward reads.
 */
enum {
    GS_SYNC_FREE_DETERMINISTIC = 1u,  /* room for the GS_FLAG_DETERMINISTIC backward's fixed-point accumulators */
    GS_SYNC_FREE_CAMERA_GRAD = 2u     /* room for the camera gradient's per-warp partials (cam != NULL) */
};

typedef struct GsSyncFreeWorkspace {
    void *base;                 /* device memory, 256-byte aligned */
    int64_t bytes;              /* size of base */
    int64_t instance_capacity;  /* 0 .. 2^31-1 tile instances */
} GsSyncFreeWorkspace;

/* Bytes of a workspace for cfg's P, S, V and frame (the pointers of cfg are not read), `instance_capacity` and the
 * GS_SYNC_FREE_* bits of `needs`.  GS_ERR_INVALID for a bad configuration or capacity. */
GS_API int gs_sync_free_workspace_bytes(const GsConfig *cfg, int64_t instance_capacity, uint32_t needs, int64_t *bytes);
/* gs_forward_ex without a host wait; alpha may be NULL (no alpha plane).  GS_ERR_INVALID, before anything is launched,
 * when ws is too small for cfg or misaligned. */
GS_API int gs_forward_sync_free(GsContext *ctx, const GsConfig *cfg, const GsInputs *in, const GsOutputs *out,
                                const GsAlpha *alpha, const GsSyncFreeWorkspace *ws, GsSaved **saved, void *stream);
/* gs_backward_cam_tanfov without a host wait, for the GsSaved of gs_forward_sync_free on the same ws.  alpha, cam and
 * dL_dtanfov may be NULL.  ws needs GS_SYNC_FREE_DETERMINISTIC room under GS_FLAG_DETERMINISTIC and
 * GS_SYNC_FREE_CAMERA_GRAD room with cam (GS_ERR_INVALID otherwise, before anything is launched). */
GS_API int gs_backward_sync_free(GsContext *ctx, const GsConfig *cfg, const GsInputs *in, const GsSaved *saved,
                                 const GsOutGrads *gout, const GsAlpha *alpha, const GsInGrads *gin,
                                 const GsCameraGrads *cam, float *dL_dtanfov, const GsSyncFreeWorkspace *ws,
                                 void *stream);

/* GaussianRasterizer.markVisible (unused by PF3plat; kept for surface completeness): present[V,P] = in frustum. */
GS_API int gs_mark_visible(GsContext *ctx, const GsConfig *cfg, const float *means3D, uint8_t *present, void *stream);

GS_API int gs_get_stats(const GsContext *ctx, GsStats *out);

/*
 * End-to-end entry with HOST buffers (what a non-torch plugin host calls): copies inputs to the device,
 * renders, copies color/radii[/depth] back, and synchronises.  All pointers in cfg/in/out are HOST pointers
 * here (pinned memory makes the copies asynchronous).  Forward only.
 * An SH block (`in->shs`, M > 16) that sits in PINNED memory (cudaHostAlloc / cudaHostRegister, 16-byte aligned) is not
 * copied: a kernel pulls the coefficients it evaluates straight out of the caller's buffer over PCIe while geometry,
 * binning and the tile sort run (DESIGN.md 5.6).  The buffer must stay valid and unmodified until the call returns (it
 * does: the call synchronises).  Pageable or unaligned blocks are uploaded by the copy engine; results are identical.
 */
GS_API int gs_render_host(GsContext *ctx, const GsConfig *cfg, const GsInputs *in, const GsOutputs *out, void *stream);
/* gs_render_host that also returns the accumulated opacity in the HOST buffer alpha->alpha, from every feed (written
 * directly by the compositor under GS_TUNE_DIRECT_OUTPUT when that buffer is pinned). */
GS_API int gs_render_host_ex(GsContext *ctx, const GsConfig *cfg, const GsInputs *in, const GsOutputs *out,
                             const GsAlpha *alpha, void *stream);

/*
 * PSNR per image = compute_psnr of PF3plat's src/evaluation/metrics.py:11-19 (clip to [0,1], mean squared error
 * over the n = c*h*w values of each image, -10 log10).  Device pointers: ground_truth, predicted [batch, n];
 * scratch [gs_psnr_scratch_floats(batch, n)] floats; out [batch].  Deterministic (no atomics).
 */
GS_API int64_t gs_psnr_scratch_floats(int32_t batch, int64_t n);
GS_API int gs_psnr(const float *ground_truth, const float *predicted, int32_t batch, int64_t n, float *scratch, float *out,
            void *stream);

/*
 * Camera glue of render_cuda for all views of a call (PF3plat's src/model/decoder/cuda_splatting.py:64-87 with
 * get_fov, PF3plat's src/geometry/projection.py:233-247, and get_projection_matrix, cuda_splatting.py:17-44).
 * Device pointers.  In: extrinsics [B,16] camera-to-world (row-major), intrinsics [B,9] normalised, near/far [B];
 * scale_invariant != 0 applies the 1/near rescale.  Out, in the layout GsConfig takes: viewmatrix, projmatrix [B,16]
 * (transposed), campos [B,3], tanfov [B,2], view_scale [B].  No host synchronisation.
 */
GS_API int gs_view_batch(int32_t B, int32_t scale_invariant, const float *extrinsics, const float *intrinsics,
                  const float *near_, const float *far_, float *viewmatrix, float *projmatrix, float *campos, float *tanfov,
                  float *view_scale, void *stream);

/*
 * SSIM per image = compute_ssim of PF3plat's src/evaluation/metrics.py:38-54, i.e. skimage's
 * structural_similarity(win_size=11, gaussian_weights=True, channel_axis=0, data_range=1.0) -- on the device instead
 * of a per-image round trip through the CPU.  Device pointers: ground_truth, predicted [batch, channels, height,
 * width]; scratch [gs_ssim_scratch_floats(...)] floats, 8-byte aligned; out [batch].  Images smaller than 11 x 11
 * are an error, as in skimage.  Deterministic (no atomics).
 */
GS_API int64_t gs_ssim_scratch_floats(int32_t batch, int32_t channels, int32_t height, int32_t width);
GS_API int gs_ssim(const float *ground_truth, const float *predicted, int32_t batch, int32_t channels, int32_t height,
            int32_t width, float *scratch, float *out, void *stream);

/*
 * Fused Gaussian adapter (SURVEY.md section 8(f).2): the per-Gaussian arithmetic of GaussianAdapter.forward,
 * PF3plat's src/model/encoder/common/gaussian_adapter.py:48-98, for V cameras x R Gaussians each.  The
 * per-camera quantities are computed by the caller with ordinary (differentiable) tensor code:
 *   kinv       = intrinsics.inverse()                                   (geometry/projection.py:88-90)
 *   multiplier = get_scale_multiplier(intrinsics, pixel_size)           (gaussian_adapter.py:100-111)
 *   sh_rotation= block-diagonal Wigner-D of c2w[:3,:3] per degree       (misc/sh_rotation.py:10-36), NULL = identity
 * Harmonics are written in the rasterizer's [d_sh][xyz] order (the reference's (xyz, d_sh) tensor is the transposed
 * VIEW of it), so the relayout copy of decoder/cuda_splatting.py:75 disappears.  Opacities pass through untouched
 * and are not an argument.
 */
typedef struct GsAdapterConfig {
    int32_t V;          /* cameras (leading batch dims of extrinsics, flattened) */
    int32_t R;          /* Gaussians per camera */
    int32_t d_sh;       /* SH coefficients per channel, (sh_degree + 1)^2 <= 25 */
    uint32_t flags;     /* GS_ADAPTER_* */
    float scale_min;    /* GaussianAdapterCfg.gaussian_scale_min */
    float scale_max;    /* GaussianAdapterCfg.gaussian_scale_max */
    float eps;          /* forward(..., eps=1e-8) */
    float reserved2_;
    const float *c2w;         /* device [V,16] extrinsics, row-major */
    const float *kinv;        /* device [V,9] */
    const float *multiplier;  /* device [V] */
    const float *sh_rotation; /* device [V,d_sh,d_sh] or NULL; gs_sh_rotation_blocks on c2w (row_stride 4) writes it */
    const float *sh_mask;     /* device [d_sh] (gaussian_adapter.py:39-46) */
} GsAdapterConfig;

enum {
    /* gs_adapter_backward: bit-reproducible per-camera gradients (dL/dc2w, dL/dKinv, dL/dmultiplier).  Each CTA writes
     * its partial sums to GsAdapterInGrads.scratch and a second kernel adds them in CTA order (no float atomics). */
    GS_ADAPTER_DETERMINISTIC = 1u
};

typedef struct GsAdapterInputs {
    const float *coordinates;   /* device [V,R,2] */
    const float *depths;        /* device [V,R] */
    const float *raw_gaussians; /* device [V,R,7+3*d_sh]: scales 3 | quaternion xyzw 4 | sh (xyz, d_sh) */
} GsAdapterInputs;

typedef struct GsAdapterOutputs { /* the fields of the reference's Gaussians dataclass (gaussian_adapter.py:13-20) */
    float *means;       /* device [V,R,3] */
    float *covariances; /* device [V,R,3,3] */
    float *harmonics;   /* device [V,R,d_sh,3] */
    float *scales;      /* device [V,R,3] */
    float *rotations;   /* device [V,R,4] */
} GsAdapterOutputs;

typedef struct GsAdapterOutGrads { /* incoming gradients, same shapes as GsAdapterOutputs; NULL = zero */
    const float *means, *covariances, *harmonics, *scales, *rotations;
} GsAdapterOutGrads;

typedef struct GsAdapterInGrads { /* any pointer may be NULL */
    float *coordinates;   /* device [V,R,2] */
    float *depths;        /* device [V,R] */
    float *raw_gaussians; /* device [V,R,7+3*d_sh] */
    float *c2w;           /* device [V,16]: through the means only (rotation is detached elsewhere, gaussian_adapter.py:81) */
    float *kinv;          /* device [V,9] */
    float *multiplier;    /* device [V] */
    void *scratch;        /* device, gs_adapter_scratch_bytes(cfg) bytes, 16-byte aligned: required with
                             GS_ADAPTER_DETERMINISTIC when c2w, kinv or multiplier is wanted; ignored otherwise */
} GsAdapterInGrads;

GS_API int gs_adapter_forward(const GsAdapterConfig *cfg, const GsAdapterInputs *in, const GsAdapterOutputs *out, void *stream);
GS_API int gs_adapter_backward(const GsAdapterConfig *cfg, const GsAdapterInputs *in, const GsAdapterOutGrads *gout,
                        const GsAdapterInGrads *gin, void *stream);
GS_API int64_t gs_adapter_scratch_bytes(const GsAdapterConfig *cfg); /* -1 for an invalid config */

/*
 * Photometric training loss = PF3plat's LossMultiSSIM + LossMse (src/loss/loss_multissim.py:45-86, loss_mse.py:35),
 * forward and backward.  Per image: ssim = the mean over (c, h, w) of the single-scale SSIM map with the zero-padded
 * 11 x 11 Gaussian window (sigma 1.5) and population covariance, no clipping; mse = the mean of (pred - gt)^2.  Any
 * height and width >= 1 is legal (the window may be larger than the image).
 * Device pointers.  predicted / ground_truth: `batch` images, image i at i * stride floats, each (c,h,w) block
 * contiguous; scratch: gs_photometric_scratch_bytes(cfg) bytes, 8-byte aligned (the backward needs none and ignores
 * it); out_ssim [batch]; out_mse [batch], required iff with_mse.  The incoming gradients dL_dssim / dL_dmse [batch]
 * are device arrays (NULL = zero; dL_dmse is read only if with_mse); the gradients dL_dpredicted / dL_dground_truth are
 * written contiguous [batch, c, h, w] (NULL = not wanted).  Deterministic (no atomics), no host synchronisation.
 */
typedef struct GsLossConfig {
    int32_t batch, channels, height, width;
    int64_t pred_stride, gt_stride; /* floats between consecutive images (ignored when batch == 1) */
    int32_t with_mse, reserved_;    /* with_mse: 0 or 1 */
} GsLossConfig;

GS_API int64_t gs_photometric_scratch_bytes(const GsLossConfig *cfg); /* -1 for an invalid config */
GS_API int gs_photometric_forward(const GsLossConfig *cfg, const float *predicted, const float *ground_truth, void *scratch,
                                  float *out_ssim, float *out_mse, void *stream);
GS_API int gs_photometric_backward(const GsLossConfig *cfg, const float *predicted, const float *ground_truth,
                                   const float *dL_dssim, const float *dL_dmse, float *dL_dpredicted,
                                   float *dL_dground_truth, void *scratch, void *stream);

/*
 * Pose (correspondence) loss = PF3plat's Losspose (src/loss/loss_pose.py:29-129), per segment s = (scene, pair (a, c)),
 * segments scene-major and pairs in the reference's order [(a, c) for a in range(views) for c in range(a + 1, views)]:
 *   L3[s] = conf[s] sum_n (w_n / max(sum |w|, 1e-12)) |R_s xyz_a(p) + t_s - xyz_c(q)|
 *   L2[s] = sum_n huber_0.01(|project_s(p, d_a(p)) - xy(q)|) / 0.01
 * with p = id_a[n], q = id_c[n] flat pixel indices of views a and c of the segment's scene (DESIGN.md 5.12).  The
 * caller forms weight_3d mean(L3) + weight_2d mean(L2).  Device pointers: T [S,16] row-major (c2w[c] or
 * c2w[c] @ inverse(c2w[a])), kinv_a [S,9] (K_a^-1), k_c [S,9], conf [S], seg [S,3] (scene, a, c), offsets [S+1] into
 * the matches (CSR), id_a / id_c int64 [matches], w [matches], depth [batch*views, h, w], xyz [batch, views, 3, h, w].
 * Gradients are written (not accumulated): dL_dT [S,16], dL_ddepth and dL_dxyz shaped as their inputs, dL_dw
 * [matches], dL_dconf [S]; any may be NULL.  The incoming dL_dL3 / dL_dL2 [S] are device arrays (NULL = zero).  An index
 * outside [0, h w) is never read: its segment's L3, L2 and gradient terms are NaN.  Non-finite depth at an unmatched
 * source pixel makes dL_ddepth there and dL_dT of its pairs NaN, as the reference's dense projection does.  Scratch:
 * gs_pose_loss_scratch_bytes(cfg), 256-byte aligned, needed only for dL_ddepth / dL_dxyz.  Deterministic (no float
 * atomics), no host synchronisation.
 */
typedef struct GsPoseLossConfig {
    int32_t batch, views, height, width;
    int32_t segments, reserved_; /* segments = batch * views (views - 1) / 2 */
    int64_t matches;             /* total over all segments = offsets[S] */
} GsPoseLossConfig;

typedef struct GsPoseLossInputs {
    const float *T, *kinv_a, *k_c, *conf;
    const int32_t *seg;
    const int64_t *offsets, *id_a, *id_c;
    const float *w, *depth, *xyz;
} GsPoseLossInputs;

typedef struct GsPoseLossGrads {
    float *dL_dT, *dL_ddepth, *dL_dxyz, *dL_dw, *dL_dconf;
} GsPoseLossGrads;

GS_API int64_t gs_pose_loss_scratch_bytes(const GsPoseLossConfig *cfg); /* -1 for an invalid config */
GS_API int gs_pose_loss_forward(const GsPoseLossConfig *cfg, const GsPoseLossInputs *in, float *out_L3, float *out_L2,
                                void *stream);
GS_API int gs_pose_loss_backward(const GsPoseLossConfig *cfg, const GsPoseLossInputs *in, const float *dL_dL3,
                                 const float *dL_dL2, const GsPoseLossGrads *grads, void *scratch, void *stream);

/*
 * Plane-sweep cost volume = the parameter-free warp and correlation of PF3plat's DepthPredictorMultiView.forward
 * (src/model/encoder/costvolume/depth_predictor_multiview.py:309-343, the tensor before the torch.cat), DESIGN.md 5.13:
 *   cost[vb, d, p] = mean over the v-1 source views s of sum_c feat01[vb, c, p] warped_s[vb, c, d, p] / sqrt(C)
 * in the reference's (v b) order (vb = vi * batch + bi), with prepare_feat_proj_data_lists' relative poses (v = 2 takes
 * its special branch), the target view's intrinsics un-normalised row-wise, depth candidates
 * 1 / (1/far + linspace(0, 1, D) (1/near - 1/far)), pixel-index coordinates, z clamped to >= 1e-3 and grid_sample's
 * bilinear sampling (align_corners=True, zero padding per tap, every in-bounds tap multiplied in).
 * Device pointers: features [batch, views, C, h, w] at the element strides feat_stride; intrinsics [batch, views, r, r]
 * normalised, r = intrinsics_rows (3, or 4 read through [:3, :3]); extrinsics [batch, views, 4, 4]; near, far
 * [batch, views]; all contiguous except features.  out_cost [views * batch, D, h, w].  The backward takes dL_dcost of
 * that shape (contiguous) and writes dL_dfeatures contiguous [batch, views, C, h, w]; the cameras get no gradient (the
 * reference builds the grid under no_grad).  Scratch: gs_costvolume_scratch_bytes(cfg, backward) bytes, 256-byte
 * aligned, for the channel-last packing of the features, the camera block and, in the backward, the per-pixel gradient
 * rows and the source accumulators.  The forward and the backward's feat01 role are deterministic; the source role
 * adds float atomics unless flags has GS_COSTVOLUME_DETERMINISTIC, which makes it bit-reproducible (exact fixed-point
 * accumulation, a non-finite or out-of-range term makes its element NaN) and needs (views-1) D h w < 2^21.
 * No host synchronisation.
 */
enum { GS_COSTVOLUME_DETERMINISTIC = 1u };

typedef struct GsCostVolumeConfig {
    int32_t batch, views, channels, height, width; /* views >= 2, height, width >= 2 */
    int32_t depth_candidates;                      /* D >= 1 */
    int32_t intrinsics_rows;                       /* 3 or 4 */
    uint32_t flags;                                /* GS_COSTVOLUME_* */
    int64_t feat_stride[5];                        /* element strides of features [batch, views, C, h, w] */
} GsCostVolumeConfig;

typedef struct GsCostVolumeInputs {
    const float *features, *intrinsics, *extrinsics, *near_, *far_;
} GsCostVolumeInputs;

typedef struct GsCostVolumeGrads {
    const float *dL_dcost; /* in:  [views * batch, D, h, w] */
    float *dL_dfeatures;   /* out: [batch, views, C, h, w] */
} GsCostVolumeGrads;

GS_API int64_t gs_costvolume_scratch_bytes(const GsCostVolumeConfig *cfg, int32_t backward); /* -1: invalid config */
GS_API int gs_costvolume_forward(const GsCostVolumeConfig *cfg, const GsCostVolumeInputs *in, float *out_cost,
                                 void *scratch, void *stream);
GS_API int gs_costvolume_backward(const GsCostVolumeConfig *cfg, const GsCostVolumeInputs *in,
                                  const GsCostVolumeGrads *grads, void *scratch, void *stream);

/*
 * The encoder's pose path between PnP and the networks that read the poses (DESIGN.md 5.14).  No host synchronisation.
 *
 * gs_pose_sync = PF3plat's camera_synchronization (src/flow_util.py:623-743) at its default arguments: N = 2 chains
 * (camera_chaining); otherwise the float32 L of the confidence-weighted pairs, squared ten times in fp64, column block
 * 0 divided by its mass, the rotation projected onto SO(3) (one-sided Jacobi), rounded to float32.  If the smallest
 * mass over the whole batch is exactly 0, every scene is chained.  A scene whose L (as built, or its column block after
 * the squarings) holds a non-finite value gets NaN in all its outputs and a NaN mass, which turns the batch fallback off.
 * Device pointers: Ps [pairs, batch, 4, 4] in the order of pair_i / pair_j, confidence [pairs, batch] (may be NULL when
 * views == 2), out [batch, views, 4, 4]; all contiguous float32.  Pairs (i, j) need 0 <= i, j < views, i != j, no
 * repeat in either order, every view in some pair and (k, k+1) for every k < views - 1 (the chain).
 * Scratch: gs_pose_sync_scratch_bytes(cfg) bytes, 256-byte aligned.  Bit-reproducible (no atomics).
 */
enum { GS_POSES_MAX_VIEWS = 16, GS_POSES_MAX_PAIRS = 120 };

typedef struct GsPoseSyncConfig {
    int32_t batch, views, pairs, reserved_;   /* 2 <= views <= 16, 1 <= pairs <= views (views - 1) / 2 */
    int8_t pair_i[GS_POSES_MAX_PAIRS], pair_j[GS_POSES_MAX_PAIRS];
} GsPoseSyncConfig;

GS_API int64_t gs_pose_sync_scratch_bytes(const GsPoseSyncConfig *cfg); /* -1 for an invalid config */
GS_API int gs_pose_sync(const GsPoseSyncConfig *cfg, const float *Ps, const float *confidence, float *out, void *scratch,
                        void *stream);

/*
 * gs_refine_poses = encoder_costvolume.py:465-473 and the .inverse() of its result: x = pose_enc (view 0) or
 * pose_enc + delta * gamma (views >= 1), R = r6d2mat(x[:6]) (F.normalize's max(|v|, 1e-12), rows b1, b2, b1 x b2),
 * abspose = [R | x[6:9]; 0 0 0 1] and abspose_inv its general 4x4 inverse, fp64 inside.  A singular abspose gives a
 * non-finite inverse.  Device pointers, contiguous float32: pose_enc, delta [batch, views, 9], gamma [1]; abspose,
 * abspose_inv [batch, views, 4, 4].  The backward takes either cotangent (NULL = zero) and writes all three gradients;
 * dL_dgamma is a fixed-order fp64 reduction in one CTA, so the backward is bit-reproducible.
 */
typedef struct GsRefinePosesConfig {
    int32_t batch, views; /* views >= 1 */
} GsRefinePosesConfig;

typedef struct GsRefinePosesInputs {
    const float *pose_enc, *delta, *gamma;
} GsRefinePosesInputs;

typedef struct GsRefinePosesGrads {
    const float *dL_dabspose, *dL_dabspose_inv;       /* in:  [batch, views, 4, 4], either may be NULL */
    float *dL_dpose_enc, *dL_ddelta, *dL_dgamma;      /* out: [batch, views, 9], [batch, views, 9], [1] */
} GsRefinePosesGrads;

GS_API int gs_refine_poses_forward(const GsRefinePosesConfig *cfg, const GsRefinePosesInputs *in, float *abspose,
                                   float *abspose_inv, void *stream);
GS_API int gs_refine_poses_backward(const GsRefinePosesConfig *cfg, const GsRefinePosesInputs *in,
                                    const GsRefinePosesGrads *grads, void *stream);

/*
 * gs_plucker_rays = plucker_embedding(h, w, *get_world_rays(grid, abspose.inverse(), K)) (encoder_costvolume.py:387-392,
 * :211-221): pixel centres ((x + 1/2) / w, (y + 1/2) / h), d = normalise(K^-1 [x, y, 1]) rotated by c2w with w = 0,
 * origin o = c2w[:3, 3], out [(batch views), 6, h, w] = (d, o x d), fp64 inside.  abspose [batch, views, 4, 4] and
 * intrinsics [batch, views, 3, 3] contiguous float32; out contiguous.
 */
typedef struct GsPluckerConfig {
    int32_t batch, views, height, width;
} GsPluckerConfig;

GS_API int gs_plucker_rays(const GsPluckerConfig *cfg, const float *abspose, const float *intrinsics, float *out,
                           void *stream);

/*
 * The encoder's depth glue between UniDepth and the networks and losses that read its output (DESIGN.md 5.15).  No host
 * synchronisation, no atomics: every backward is a fixed-order gather and bit-reproducible.
 *
 * gs_depth_update = encoder_costvolume.py:265, :285-287 with get_scaleshift (:167-172) and the unprojections :304-307,
 * :506-528: d0 = clamp(depth, near, far); s = the scale-shift head's channel 1 bilinearly upsampled (align_corners =
 * False, PyTorch's source index) from the (grid_height, grid_width) feature grid to (height, width), clamped to
 * [-5, 5]; depths = clamp(d0 + s, near, far), all in fp64 and rounded once; xyz = K^-1 [(x + 1/2) / w, (y + 1/2) / h,
 * 1] depths (K^-1 in fp64).
 * clamp propagates NaN.  Device pointers, contiguous float32: depth, depths [(batch views), 1, h, w]; scale_shift
 * [batch, views, grid_height grid_width, 2] (channel 0 the scale, unused); intrinsics [batch, views, 3, 3]; near_,
 * far_ [batch, views]; xyz [batch, views, 3, h, w].  The backward takes dL/ddepths and dL/dxyz (either may be NULL),
 * masks them by both clamps (the gradient passes where lo <= x <= hi, a NaN passes nothing) and gathers them per
 * feature-grid cell, one warp per cell, into dL/dscale_shift (channel 0 written as 0).
 */
typedef struct GsDepthUpdateConfig {
    int32_t batch, views, height, width, grid_height, grid_width;
} GsDepthUpdateConfig;

typedef struct GsDepthUpdateInputs {
    const float *depth, *scale_shift, *intrinsics, *near_, *far_;
} GsDepthUpdateInputs;

typedef struct GsDepthUpdateGrads {
    const float *dL_ddepths, *dL_dxyz; /* in:  [(batch views), 1, h, w], [batch, views, 3, h, w]; either may be NULL */
    float *dL_dscale_shift;            /* out: [batch, views, grid_height grid_width, 2] */
} GsDepthUpdateGrads;

GS_API int gs_depth_update_forward(const GsDepthUpdateConfig *cfg, const GsDepthUpdateInputs *in, float *depths,
                                   float *xyz, void *stream);
GS_API int gs_depth_update_backward(const GsDepthUpdateConfig *cfg, const GsDepthUpdateInputs *in,
                                    const GsDepthUpdateGrads *grads, void *stream);

/*
 * gs_mono_cue = encoder_costvolume.py:292-298, the one-hot mono cue (forward only): depths [(batch views), 1, h, w]
 * downsampled bilinearly by exactly 4 (h, w multiples of 4: taps 4i+1, 4i+2 at weight 1/2, in PyTorch's order), then
 * the index of the first smallest |d - h_k| over GS_MONO_CUE_BINS hypotheses (a NaN difference counts as smallest, as
 * in torch.argmin), written as a one-hot into out [(views batch), GS_MONO_CUE_BINS, h/4, w/4].  Every scene uses
 * near_[0] and far_[0], read on the device: h_k = fl32(a + fl32(lin[k] fl32(B))), a = fl32(1 / far_[0]),
 * B = (double)fl32(1 / near_[0]) - (double)a.  lin is a device array of GS_MONO_CUE_BINS floats holding the values
 * of torch.linspace(0, 1, 128) on the CPU.
 */
enum { GS_MONO_CUE_BINS = 128 };

typedef struct GsMonoCueConfig {
    int32_t batch, views, height, width; /* height, width: the full-resolution frame, multiples of 4 */
} GsMonoCueConfig;

GS_API int gs_mono_cue(const GsMonoCueConfig *cfg, const float *depths, const float *near_, const float *far_,
                       const float *lin, float *out, void *stream);

/*
 * gs_pdf_peak = depth_predictor_multiview.py:379-384: max over D of softmax over D of logits [items, D, h, w],
 * i.e. 1 / sum_k exp(x_k - x_max), nearest-upsampled by the integer `upscale` into out [items, 1, h s, w s].  The
 * forward also writes the per-pixel peak [items, h, w] and argmax [items, h, w] (ties to the lowest index) for the
 * backward, which takes dL/dout, sums each pixel's s^2 cotangents in a fixed order into G and writes
 * dL/dlogits_k = G p* (delta_{k, k*} - p_k), with p_k recomputed from the logits.
 */
typedef struct GsPdfPeakConfig {
    int32_t items, depth_candidates, height, width, upscale;
} GsPdfPeakConfig;

GS_API int gs_pdf_peak_forward(const GsPdfPeakConfig *cfg, const float *logits, float *out, float *peak,
                               int32_t *argmax, void *stream);
GS_API int gs_pdf_peak_backward(const GsPdfPeakConfig *cfg, const float *logits, const float *peak,
                                const int32_t *argmax, const float *dL_dout, float *dL_dlogits, void *stream);

/*
 * The Gaussian head between the depth predictor's two output convolutions and the decoder (DESIGN.md 5.16), for
 * gaussians_per_pixel = num_surfaces = 1:
 *   depth_predictor_multiview.py:397-415   the (v b) c h w -> b v (h w) c rearrange of to_gaussians' output, the split
 *                                          of to_disparity's output and the sigmoid of its channel 1
 *   encoder_costvolume.py:509-518          pixel centres ((i + 1/2) / w, (j + 1/2) / h) moved by
 *                                          (sigmoid(raw[0:2]) - 1/2) (1/w, 1/h), in float32 as the reference rounds it
 *   encoder_costvolume.py:529-540          the adapter on raw[2:] with views 0 and V - 1 of depths, c2w and intrinsics
 *                                          (gaussian_adapter.py:60-92; K^-1 and get_scale_multiplier in fp64 per camera)
 *   encoder_costvolume.py:174-187, :534    opacities = 0.5 (1 - (1 - q) + q), q = sigmoid(density), / gpp = 1
 *   encoder_costvolume.py:556-573          every output in b (v r srf spp) order: slot 0's pixels row-major, then
 *                                          slot 1's (the context's view V - 1), G = 2 h w Gaussians per scene
 * One launch forward, two backward; no host synchronisation, no float atomics (bit-reproducible).
 */
typedef struct GsGaussianHeadConfig {
    int32_t batch;      /* b; 2 batch <= 65535 cameras */
    int32_t views;      /* V >= 2: the context views of depths, c2w and intrinsics (encoder_costvolume.py:530-533) */
    int32_t height;     /* h of the depth predictor's full-resolution output */
    int32_t width;      /* w */
    int32_t d_sh;       /* (sh_degree + 1)^2 <= 25 (gaussian_adapter.py:113-115) */
    uint32_t flags;     /* 0 */
    float scale_min;    /* GaussianAdapterCfg.gaussian_scale_min (gaussian_adapter.py:63) */
    float scale_max;    /* GaussianAdapterCfg.gaussian_scale_max (gaussian_adapter.py:64) */
    float eps;          /* GaussianAdapter.forward's eps, 1e-8 (gaussian_adapter.py:57, :73) */
    int32_t reserved_;
} GsGaussianHeadConfig;

typedef struct GsGaussianHeadInputs { /* device, contiguous float32 */
    const float *raw_gaussians;  /* [(2 batch), 9 + 3 d_sh, h, w]: to_gaussians' output (depth_predictor_multiview.py:397),
                                    (v b) order; channels: offset xy 2 | scales 3 | quaternion xyzw 4 | sh (xyz, d_sh) */
    const float *density_logits; /* [(2 batch), 2, h, w]: to_disparity's output (:403); channel 1 the raw density */
    const float *depths;         /* [(batch views), 1, h, w]: depths_final (encoder_costvolume.py:528) */
    const float *c2w;            /* [batch, views, 4, 4]: refine_sync_abspose.inverse() (:530) */
    const float *intrinsics;     /* [batch, views, 3, 3] normalised (:531) */
    const float *sh_rotation;    /* [batch, 2, d_sh, d_sh] block-diagonal Wigner-D of slot 0 / 1's c2w[:3, :3] after the
                                    rotation guard (misc/sh_rotation.py:21-34), or NULL = identity; gs_sh_rotation_blocks
                                    on c2w's views 0 and V - 1 (outer batch, inner 2, outer_stride 16 V, inner_stride
                                    16 (V - 1), row_stride 4) writes it */
    const float *sh_mask;        /* [d_sh] (gaussian_adapter.py:39-46) */
} GsGaussianHeadInputs;

typedef struct GsGaussianHeadOutputs { /* the four fields of model/types.py's Gaussians (encoder_costvolume.py:556-573) */
    float *means;       /* [batch, 2 h w, 3] */
    float *covariances; /* [batch, 2 h w, 3, 3] */
    float *harmonics;   /* [batch, 2 h w, d_sh, 3]: the reference's (3, d_sh) is the transposed view */
    float *opacities;   /* [batch, 2 h w] */
} GsGaussianHeadOutputs;

typedef struct GsGaussianHeadOutGrads { /* incoming gradients, shaped as GsGaussianHeadOutputs; NULL = zero */
    const float *means, *covariances, *harmonics, *opacities;
} GsGaussianHeadOutGrads;

typedef struct GsGaussianHeadInGrads { /* written, not accumulated; any may be NULL */
    float *raw_gaussians;  /* [(2 batch), 9 + 3 d_sh, h, w] */
    float *density_logits; /* [(2 batch), 2, h, w]: channel 0 (delta_disps, unused by :404) gets 0 */
    float *depths;         /* [(batch views), 1, h, w]: views 1 .. V - 2 get 0 */
    float *c2w;            /* [batch, views, 4, 4]: through the means only (gaussian_adapter.py:81 detaches the rotation
                              elsewhere); row 3 and views 1 .. V - 2 get 0 */
    void *scratch;         /* gs_gaussian_head_scratch_bytes(cfg) bytes, 16-byte aligned: required with c2w */
} GsGaussianHeadInGrads;

GS_API int64_t gs_gaussian_head_scratch_bytes(const GsGaussianHeadConfig *cfg); /* -1 for an invalid config */
GS_API int gs_gaussian_head_forward(const GsGaussianHeadConfig *cfg, const GsGaussianHeadInputs *in,
                                    const GsGaussianHeadOutputs *out, void *stream);
GS_API int gs_gaussian_head_backward(const GsGaussianHeadConfig *cfg, const GsGaussianHeadInputs *in,
                                     const GsGaussianHeadOutGrads *gout, const GsGaussianHeadInGrads *gin,
                                     void *stream);

/*
 * SH rotation (DESIGN.md 5.17): the block-diagonal Wigner-D matrices that GsAdapterConfig::sh_rotation and
 * GsGaussianHeadInputs::sh_rotation take, as misc/sh_rotation.py:10-36 builds them, for N = outer inner cameras:
 *   guard   sh_rotation.py:21-22: unless every determinant satisfies |det - 1| <= 1e-8 + 1e-5 (torch.allclose to 1;
 *           det in fp64 from the fp32 entries; NaN and +-Inf fail), every camera of the call uses the identity
 *   blocks  per degree l < sqrt(d_sh), D_l(R) with Y_l(R x) = D_l(R) Y_l(x), by pf3plat_b200/sh_rotation.py's
 *           least-squares fit over 64 fixed unit vectors in fp64, rounded to float32 once
 * rotations: device float32; matrix (i, s), 0 <= i < outer, 0 <= s < inner, starts at
 * rotations + i outer_stride + s inner_stride, its rows row_stride floats apart and its columns adjacent, so
 * contiguous [N, 3, 3] (row_stride 3) and the top-left blocks of a strided [outer, inner, 4, 4] view such as
 * c2w[:, ::V-1] (row_stride 4) are read in place.  out: device [N, d_sh, d_sh] contiguous, camera i inner + s; every
 * element is written.  workspace: gs_sh_rotation_workspace_bytes(cfg) bytes of device memory, 4-byte aligned, holding
 * the guard's flag between the two launches (one stream at a time).  Two launches, no atomics, no host
 * synchronisation; a camera's matrix depends only on its rotation and the guard.  GS_ERR_INVALID, with nothing
 * launched, for d_sh not in {1, 4, 9, 16, 25}, outer or inner < 1, N >= 2^31, row_stride not 3 or 4, or a NULL
 * pointer.
 */
typedef struct GsShRotationConfig {
    int32_t outer, inner;         /* N = outer inner matrices */
    int64_t outer_stride;         /* floats between matrix (i, s) and (i + 1, s) */
    int64_t inner_stride;         /* floats between matrix (i, s) and (i, s + 1) */
    int32_t row_stride;           /* 3 or 4 */
    int32_t d_sh;                 /* 1, 4, 9, 16 or 25 */
} GsShRotationConfig;

GS_API int64_t gs_sh_rotation_workspace_bytes(const GsShRotationConfig *cfg); /* -1 for an invalid config */
GS_API int gs_sh_rotation_blocks(const GsShRotationConfig *cfg, const float *rotations, float *out, void *workspace,
                                 void *stream);

/*
 * LPIPS-VGG = the `lpips` package's LPIPS(net="vgg", version="0.1"), spatial=False, as PF3plat's LossLpips
 * (src/loss/loss_lpips.py:55-59) and compute_lpips (src/evaluation/metrics.py:27-33) call it; forward and input
 * gradients (the weights are constants).  The weights are an input:
 *   gs_lpips_weights_create packs, on `stream`, the 13 conv weights [Cout, Cin, 3, 3] and biases [Cout] of VGG16
 *   features[0:30] (conv1_1 .. conv5_3), the 5 lin weights [C] (relu1_2 .. relu5_3) and the scaling layer's shift[3] and
 *   scale[3] (all device pointers on the current device) into private device memory; the sources may be freed once the
 *   stream has run the packing.  gs_lpips_weights_destroy synchronises with the device before it frees.
 * Inputs in0 / in1: `batch` images [3, height, width], image i at i * stride floats.  height, width >= 16.
 * workspace: gs_lpips_workspace_bytes(cfg) bytes, 256-byte aligned; with grads != 0 the forward keeps every activation
 * there for gs_lpips_backward, which must get the same config and workspace.  out [batch] (the package's (N,1,1,1)).
 * dL_dout [batch] is a device array; dL_din0 / dL_din1 are written contiguous [batch, 3, height, width], NULL = not
 * wanted (each needs its bit in grads).  Deterministic (no atomics), no host synchronisation.
 * precision GS_LPIPS_BF16 (opt-in) runs BF16 activations and inter-layer gradients with BF16 wgmma convolutions (fp32
 * accumulation), as torch.autocast(dtype=torch.bfloat16) would; inputs, out and dL_din stay fp32.  It needs
 * gs_lpips_weights_pack_bf16 on the handle first (GS_ERR_INVALID otherwise), which adds BF16 copies of the conv weights
 * (about 59 MB) from the same fp32 conv_weight[13] (only [1..12] are read); a handle packed already is left as it is.
 */
typedef struct GsLpipsWeights GsLpipsWeights;

enum { GS_LPIPS_TF32 = 0, GS_LPIPS_BF16 = 1 };

typedef struct GsLpipsConfig {
    int32_t batch, height, width;
    int32_t normalize;              /* 0 or 1: inputs are mapped x -> 2x - 1 first (the package's normalize=True) */
    int64_t in0_stride, in1_stride; /* floats between consecutive images (ignored when batch == 1) */
    int32_t grads;                  /* bit 0: dL/din0 will be wanted, bit 1: dL/din1; 0 = forward only */
    union {
        int32_t precision; /* GS_LPIPS_TF32 (0, the default) or GS_LPIPS_BF16; the workspace size depends on it */
        int32_t reserved_; /* the field's name before it held the precision */
    };
} GsLpipsConfig;

GS_API int gs_lpips_weights_create(const float *const *conv_weight /* [13] */, const float *const *conv_bias /* [13] */,
                                   const float *const *lin /* [5] */, const float *shift, const float *scale, void *stream,
                                   GsLpipsWeights **out);
GS_API int gs_lpips_weights_pack_bf16(GsLpipsWeights *weights, const float *const *conv_weight /* [13] */, void *stream);
GS_API void gs_lpips_weights_destroy(GsLpipsWeights *weights);
GS_API int64_t gs_lpips_workspace_bytes(const GsLpipsConfig *cfg); /* -1 for an invalid config */
GS_API int gs_lpips_forward(const GsLpipsWeights *weights, const GsLpipsConfig *cfg, const float *in0, const float *in1,
                            void *workspace, float *out, void *stream);
GS_API int gs_lpips_backward(const GsLpipsWeights *weights, const GsLpipsConfig *cfg, const float *dL_dout,
                             void *workspace, float *dL_din0, float *dL_din1, void *stream);

/* Per-stage device timings (ms) of the last forward/backward when profiling is enabled; CUDA events on `stream`. */
enum { GS_STAGE_PREPROCESS = 0,      /* k_preprocess (incl. tile counting) */
       GS_STAGE_BIN_SCAN = 1,        /* k_tile_scan + the forward's one host read-back */
       GS_STAGE_BIN_EMIT = 2,        /* k_emit_buckets (or the radix fallback's whole chain) */
       GS_STAGE_BIN_SORT = 3,        /* k_tile_sort */
       GS_STAGE_COMPOSITE = 4,       /* k_composite_fwd */
       GS_STAGE_COMPOSITE_BWD = 5,   /* accumulator memset + k_composite_bwd */
       GS_STAGE_PREPROCESS_BWD = 6,  /* k_preprocess_bwd */
       GS_STAGE_SH_COLOUR = 7,       /* k_sh_colour on its own stream (gs_render_host's split pipeline; overlaps stages 0-3) */
       GS_NUM_STAGES = 8 };
GS_API int gs_set_profiling(GsContext *ctx, int enabled);
GS_API int gs_get_stage_ms(GsContext *ctx, float *ms /* [GS_NUM_STAGES] */);

#ifdef __cplusplus
}
#endif
#endif /* GSPLAT_B200_H */
