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

#define GS_ABI_VERSION 1

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
    GS_FLAG_DEPTH = 1u,        /* also composite camera-space z as a 4th channel (render_depth_cuda mode "depth", cuda_splatting.py:226-269, fused) */
    GS_FLAG_PREFILTERED = 2u   /* GaussianRasterizationSettings.prefiltered */
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
    GS_TUNE_FEED_PIECES_SHIFT = 8     /* gs_render_host: bits 8..11 = pieces the SH block is copied in (0 default, 1 = one plain copy) */
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
    int32_t sh_eval_max_degree; /* default 3 (<=0 selects it) */
    uint32_t tuning;      /* GS_TUNE_* implementation knobs (testing); 0 = default */
    const float *viewmatrix; /* device [V,16]  settings.viewmatrix */
    const float *projmatrix; /* device [V,16]  settings.projmatrix */
    const float *campos;     /* device [V,3]   settings.campos */
    const float *bg;         /* device [V,3]   settings.bg */
    const float *tanfov;     /* device [V,2] or NULL */
    const float *view_scale; /* device [V] or NULL: per-view factor s applied as mean*s, cov*s^2, scales*s
                                (the 1/near rescale of cuda_splatting.py:64-71 without materialising copies) */
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
} GsInGrads;

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

GS_API void gs_saved_free(GsContext *ctx, GsSaved *saved, void *stream);

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
    int32_t reserved_;
    float scale_min;    /* GaussianAdapterCfg.gaussian_scale_min */
    float scale_max;    /* GaussianAdapterCfg.gaussian_scale_max */
    float eps;          /* forward(..., eps=1e-8) */
    float reserved2_;
    const float *c2w;         /* device [V,16] extrinsics, row-major */
    const float *kinv;        /* device [V,9] */
    const float *multiplier;  /* device [V] */
    const float *sh_rotation; /* device [V,d_sh,d_sh] or NULL */
    const float *sh_mask;     /* device [d_sh] (gaussian_adapter.py:39-46) */
} GsAdapterConfig;

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
} GsAdapterInGrads;

GS_API int gs_adapter_forward(const GsAdapterConfig *cfg, const GsAdapterInputs *in, const GsAdapterOutputs *out, void *stream);
GS_API int gs_adapter_backward(const GsAdapterConfig *cfg, const GsAdapterInputs *in, const GsAdapterOutGrads *gout,
                        const GsAdapterInGrads *gin, void *stream);

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
 */
typedef struct GsLpipsWeights GsLpipsWeights;

typedef struct GsLpipsConfig {
    int32_t batch, height, width;
    int32_t normalize;              /* 0 or 1: inputs are mapped x -> 2x - 1 first (the package's normalize=True) */
    int64_t in0_stride, in1_stride; /* floats between consecutive images (ignored when batch == 1) */
    int32_t grads;                  /* bit 0: dL/din0 will be wanted, bit 1: dL/din1; 0 = forward only */
    int32_t reserved_;
} GsLpipsConfig;

GS_API int gs_lpips_weights_create(const float *const *conv_weight /* [13] */, const float *const *conv_bias /* [13] */,
                                   const float *const *lin /* [5] */, const float *shift, const float *scale, void *stream,
                                   GsLpipsWeights **out);
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
