// gs_losses.cu -- PF3plat's photometric training loss on the device: the single-scale SSIM of
// src/loss/loss_multissim.py:45-86 and the squared error of src/loss/loss_mse.py:35, forward and backward.
//
// Semantics (per image and channel plane; x = predicted, y = ground truth; w = g g^T with g the 11-tap Gaussian,
// sigma 1.5, normalised; "*" is a zero-padded filter with a full H x W output, as F.conv2d(padding=5) computes it):
//   ux = w*x, uy = w*y, vx = w*(x^2) - ux^2, vy = w*(y^2) - uy^2, vxy = w*(xy) - ux uy   (population covariance)
//   S  = (2 ux uy + C1)(2 vxy + C2) / ((ux^2 + uy^2 + C1)(vx + vy + C2)),  C1 = 0.01^2, C2 = 0.03^2, no clipping.
// Per image the forward returns mean(S) and mean((x - y)^2) over (c, h, w).  Unlike gs_ssim (skimage's metric) there
// is no crop, no sample-covariance factor, and any H, W >= 1 is legal: the window may be larger than the image.
//
// Forward: one CTA per (32 x 32 tile, channel, image).  The tile plus a 5-px halo of both images is staged in shared
// memory (zero outside the image), the separable filter produces the five moment maps, and the per-tile fp64 sums of
// S and of the squared error are reduced per image by k_photometric_finalize in a fixed order (no atomics).
//
// Backward (closed form; g = dL/dS per map pixel = dL/dssim[img] / (c h w)):
//   A1 = 2 ux uy + C1, A2 = 2 vxy + C2, B1 = ux^2 + uy^2 + C1, B2 = vx + vy + C2
//   alpha = -g S / B2,  beta = 2 g A1 / (B1 B2),  gamma_x = g S (2 uy / A1 - 2 ux / B1) - 2 ux alpha - uy beta
//   dL/dx = w*gamma_x + 2x (w*alpha) + y (w*beta)     (and x <-> y for dL/dy)
// alpha, beta and gamma exist only on the image (zero outside it before the back-filter).  The kernel RECOMPUTES the
// moments on the tile plus a 10-px halo instead of reading maps the forward saved: the forward stays a pure reduction
// (2 reads per pixel, nothing written), and the backward reads 2 images instead of 4 saved maps, so the recompute
// costs arithmetic only (DESIGN.md 5.9).  Each gradient pixel is written exactly once (gather form, no atomics).
#include "gs_common.cuh"

namespace {

constexpr int PL_T = 32, PL_R = 5, PL_TAPS = 2 * PL_R + 1, PL_THREADS = 256;
constexpr int PL_IN = PL_T + 2 * PL_R;        // forward: tile + 5-px halo (42)
constexpr int PL_BIN = PL_T + 4 * PL_R;       // backward: tile + 10-px halo of the inputs (52)
constexpr int PL_MAP = PL_T + 2 * PL_R;       // backward: the alpha/beta/gamma grid, tile + 5-px halo (42)
constexpr float PL_C1 = 0.01f * 0.01f, PL_C2 = 0.03f * 0.03f;

struct PlWeights {
    float w[PL_TAPS];
};

// g of create_window (loss_multissim.py:46-55): exp(-(k-5)^2 / (2 sigma^2)), normalised; computed once per process
const PlWeights &window_weights() {
    static const PlWeights wt = [] {
        PlWeights r;
        double w[PL_TAPS], sum = 0.0;
        for (int k = 0; k < PL_TAPS; k++) {
            const double x = (double)(k - PL_R);
            w[k] = exp(-x * x / (2.0 * 1.5 * 1.5));
            sum += w[k];
        }
        for (int k = 0; k < PL_TAPS; k++) r.w[k] = (float)(w[k] / sum);
        return r;
    }();
    return wt;
}

__device__ __forceinline__ double block_sum(double v, double *red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
    if (threadIdx.x == 0) {
#pragma unroll
        for (int k = 0; k < PL_THREADS / 32; k++) t += red[k];
    }
    return t;  // valid in thread 0
}

__global__ void __launch_bounds__(PL_THREADS)
k_photometric_fwd(const float *__restrict__ pred, const float *__restrict__ gt, int64_t pred_stride, int64_t gt_stride,
                  int H, int W, int tiles_x, const PlWeights wt, double *__restrict__ partial) {
    __shared__ float sx[PL_IN][PL_IN + 1], sy[PL_IN][PL_IN + 1];
    __shared__ float hq[5][PL_IN][PL_T + 1];  // horizontally filtered x, y, xx, yy, xy
    __shared__ double red[2][PL_THREADS / 32];
    const int tile = blockIdx.x, ch = blockIdx.y, img = blockIdx.z, C = gridDim.y, tid = threadIdx.x;
    const int ox = (tile % tiles_x) * PL_T, oy = (tile / tiles_x) * PL_T;
    const size_t plane = (size_t)ch * H * W;
    const float *a = pred + (size_t)img * pred_stride + plane, *b = gt + (size_t)img * gt_stride + plane;
    for (int e = tid; e < PL_IN * PL_IN; e += PL_THREADS) {
        const int r = e / PL_IN, c = e - r * PL_IN;
        const int iy = oy - PL_R + r, ix = ox - PL_R + c;
        const bool in = iy >= 0 && iy < H && ix >= 0 && ix < W;  // zero padding
        sx[r][c] = in ? a[(size_t)iy * W + ix] : 0.f;
        sy[r][c] = in ? b[(size_t)iy * W + ix] : 0.f;
    }
    __syncthreads();
    for (int e = tid; e < PL_IN * PL_T; e += PL_THREADS) {
        const int r = e / PL_T, c = e - r * PL_T;
        float mx = 0.f, my = 0.f, mxx = 0.f, myy = 0.f, mxy = 0.f;
#pragma unroll
        for (int k = 0; k < PL_TAPS; k++) {
            const float x = sx[r][c + k], y = sy[r][c + k], w = wt.w[k];
            mx = fmaf(w, x, mx);
            my = fmaf(w, y, my);
            mxx = fmaf(w, x * x, mxx);
            myy = fmaf(w, y * y, myy);
            mxy = fmaf(w, x * y, mxy);
        }
        hq[0][r][c] = mx; hq[1][r][c] = my; hq[2][r][c] = mxx; hq[3][r][c] = myy; hq[4][r][c] = mxy;
    }
    __syncthreads();
    double acc_s = 0.0;
    float acc_e = 0.f;
    for (int e = tid; e < PL_T * PL_T; e += PL_THREADS) {
        const int r = e / PL_T, c = e - r * PL_T;
        if (oy + r >= H || ox + c >= W) continue;
        float ux = 0.f, uy = 0.f, uxx = 0.f, uyy = 0.f, uxy = 0.f;
#pragma unroll
        for (int k = 0; k < PL_TAPS; k++) {
            const float w = wt.w[k];
            ux = fmaf(w, hq[0][r + k][c], ux);
            uy = fmaf(w, hq[1][r + k][c], uy);
            uxx = fmaf(w, hq[2][r + k][c], uxx);
            uyy = fmaf(w, hq[3][r + k][c], uyy);
            uxy = fmaf(w, hq[4][r + k][c], uxy);
        }
        const float vx = uxx - ux * ux, vy = uyy - uy * uy, vxy = uxy - ux * uy;
        const float A1 = 2.f * ux * uy + PL_C1, A2 = 2.f * vxy + PL_C2;
        const float B1 = ux * ux + uy * uy + PL_C1, B2 = vx + vy + PL_C2;
        acc_s += (double)((A1 * A2) / (B1 * B2));
        const float d = sx[r + PL_R][c + PL_R] - sy[r + PL_R][c + PL_R];
        acc_e = fmaf(d, d, acc_e);
    }
    const double ts = block_sum(acc_s, red[0]);
    const double te = block_sum((double)acc_e, red[1]);
    if (tid == 0) {
        const size_t per_image = (size_t)C * gridDim.x, slot = (size_t)img * per_image + (size_t)ch * gridDim.x + tile;
        partial[slot] = ts;
        partial[(size_t)gridDim.z * per_image + slot] = te;
    }
}

// one warp per image: fixed summation order, so the result is bit-reproducible
__global__ void k_photometric_finalize(const double *__restrict__ partial, int batch, int per_image, double inv_n,
                                       float *__restrict__ out_ssim, float *__restrict__ out_mse) {
    const int img = blockIdx.x;
    double s = 0.0, e = 0.0;
    const double *ps = partial + (size_t)img * per_image, *pe = partial + ((size_t)batch + img) * per_image;
    for (int k = threadIdx.x; k < per_image; k += 32) {
        s += ps[k];
        e += pe[k];
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        s += __shfl_xor_sync(0xffffffffu, s, o);
        e += __shfl_xor_sync(0xffffffffu, e, o);
    }
    if (threadIdx.x == 0) {
        out_ssim[img] = (float)(s * inv_n);
        if (out_mse) out_mse[img] = (float)(e * inv_n);
    }
}

// dynamic shared memory of k_photometric_bwd (floats)
constexpr int PLB_SX = PL_BIN * (PL_BIN + 1);           // x, then y: tile + 10-px halo
constexpr int PLB_HQ = 5 * PL_BIN * (PL_MAP + 1);        // five horizontally filtered moments; later the back-filter
constexpr int PLB_HB = 4 * PL_MAP * (PL_T + 1);          // horizontally back-filtered gamma_x, gamma_y, alpha, beta
constexpr int PLB_MAPS = 4 * PL_MAP * (PL_MAP + 1);      // gamma_x, gamma_y, alpha, beta on the tile + 5-px halo
static_assert(PLB_HB <= PLB_HQ, "the back-filter reuses the moment buffer");
constexpr size_t PLB_SMEM = sizeof(float) * (2 * PLB_SX + PLB_HQ + PLB_MAPS);

__global__ void __launch_bounds__(PL_THREADS)
k_photometric_bwd(const float *__restrict__ pred, const float *__restrict__ gt, int64_t pred_stride, int64_t gt_stride,
                  int H, int W, int tiles_x, const PlWeights wt, double inv_n, const float *__restrict__ dL_dssim,
                  const float *__restrict__ dL_dmse, float *__restrict__ dpred, float *__restrict__ dgt) {
    extern __shared__ float smem[];
    float(*sx)[PL_BIN + 1] = reinterpret_cast<float(*)[PL_BIN + 1]>(smem);
    float(*sy)[PL_BIN + 1] = reinterpret_cast<float(*)[PL_BIN + 1]>(smem + PLB_SX);
    float(*hq)[PL_BIN][PL_MAP + 1] = reinterpret_cast<float(*)[PL_BIN][PL_MAP + 1]>(smem + 2 * PLB_SX);
    float(*hb)[PL_MAP][PL_T + 1] = reinterpret_cast<float(*)[PL_MAP][PL_T + 1]>(smem + 2 * PLB_SX);
    float(*maps)[PL_MAP][PL_MAP + 1] = reinterpret_cast<float(*)[PL_MAP][PL_MAP + 1]>(smem + 2 * PLB_SX + PLB_HQ);
    const int tile = blockIdx.x, ch = blockIdx.y, img = blockIdx.z, C = gridDim.y, tid = threadIdx.x;
    const int ox = (tile % tiles_x) * PL_T, oy = (tile / tiles_x) * PL_T;
    const size_t plane = (size_t)ch * H * W;
    const float *a = pred + (size_t)img * pred_stride + plane, *b = gt + (size_t)img * gt_stride + plane;
    const float g = (float)((double)dL_dssim[img] * inv_n);
    const float gm = dL_dmse ? (float)(2.0 * (double)dL_dmse[img] * inv_n) : 0.f;

    for (int e = tid; e < PL_BIN * PL_BIN; e += PL_THREADS) {
        const int r = e / PL_BIN, c = e - r * PL_BIN;
        const int iy = oy - 2 * PL_R + r, ix = ox - 2 * PL_R + c;
        const bool in = iy >= 0 && iy < H && ix >= 0 && ix < W;  // inputs are zero outside the image
        sx[r][c] = in ? a[(size_t)iy * W + ix] : 0.f;
        sy[r][c] = in ? b[(size_t)iy * W + ix] : 0.f;
    }
    __syncthreads();
    for (int e = tid; e < PL_BIN * PL_MAP; e += PL_THREADS) {
        const int r = e / PL_MAP, c = e - r * PL_MAP;
        float mx = 0.f, my = 0.f, mxx = 0.f, myy = 0.f, mxy = 0.f;
#pragma unroll
        for (int k = 0; k < PL_TAPS; k++) {
            const float x = sx[r][c + k], y = sy[r][c + k], w = wt.w[k];
            mx = fmaf(w, x, mx);
            my = fmaf(w, y, my);
            mxx = fmaf(w, x * x, mxx);
            myy = fmaf(w, y * y, myy);
            mxy = fmaf(w, x * y, mxy);
        }
        hq[0][r][c] = mx; hq[1][r][c] = my; hq[2][r][c] = mxx; hq[3][r][c] = myy; hq[4][r][c] = mxy;
    }
    __syncthreads();
    for (int e = tid; e < PL_MAP * PL_MAP; e += PL_THREADS) {
        const int r = e / PL_MAP, c = e - r * PL_MAP;
        const int py = oy - PL_R + r, px = ox - PL_R + c;
        float gx = 0.f, gy = 0.f, al = 0.f, be = 0.f;
        if (py >= 0 && py < H && px >= 0 && px < W) {  // the map exists only on the image
            float ux = 0.f, uy = 0.f, uxx = 0.f, uyy = 0.f, uxy = 0.f;
#pragma unroll
            for (int k = 0; k < PL_TAPS; k++) {
                const float w = wt.w[k];
                ux = fmaf(w, hq[0][r + k][c], ux);
                uy = fmaf(w, hq[1][r + k][c], uy);
                uxx = fmaf(w, hq[2][r + k][c], uxx);
                uyy = fmaf(w, hq[3][r + k][c], uyy);
                uxy = fmaf(w, hq[4][r + k][c], uxy);
            }
            const float vx = uxx - ux * ux, vy = uyy - uy * uy, vxy = uxy - ux * uy;
            const float A1 = 2.f * ux * uy + PL_C1, A2 = 2.f * vxy + PL_C2;
            const float B1 = ux * ux + uy * uy + PL_C1, B2 = vx + vy + PL_C2;
            const float d = 1.f / (B1 * B2);
            const float gS = g * (A1 * A2) * d;
            // S * 2uy / A1 written as 2uy A2 / (B1 B2): A1 may vanish for inputs outside [0, 1]
            const float t1 = 2.f * g * A2 * d, gSB1 = 2.f * gS / B1;
            al = -gS / B2;
            be = 2.f * g * A1 * d;
            gx = t1 * uy - gSB1 * ux - 2.f * ux * al - uy * be;
            gy = t1 * ux - gSB1 * uy - 2.f * uy * al - ux * be;
        }
        maps[0][r][c] = gx; maps[1][r][c] = gy; maps[2][r][c] = al; maps[3][r][c] = be;
    }
    __syncthreads();  // hq is dead from here: hb reuses it
    for (int e = tid; e < PL_MAP * PL_T; e += PL_THREADS) {
        const int r = e / PL_T, c = e - r * PL_T;
        float q0 = 0.f, q1 = 0.f, q2 = 0.f, q3 = 0.f;
#pragma unroll
        for (int k = 0; k < PL_TAPS; k++) {  // the window is symmetric: the adjoint filter is the same correlation
            const float w = wt.w[k];
            q0 = fmaf(w, maps[0][r][c + k], q0);
            q1 = fmaf(w, maps[1][r][c + k], q1);
            q2 = fmaf(w, maps[2][r][c + k], q2);
            q3 = fmaf(w, maps[3][r][c + k], q3);
        }
        hb[0][r][c] = q0; hb[1][r][c] = q1; hb[2][r][c] = q2; hb[3][r][c] = q3;
    }
    __syncthreads();
    float *gp = dpred ? dpred + ((size_t)img * C + ch) * H * W : nullptr;
    float *gg = dgt ? dgt + ((size_t)img * C + ch) * H * W : nullptr;
    for (int e = tid; e < PL_T * PL_T; e += PL_THREADS) {
        const int r = e / PL_T, c = e - r * PL_T;
        const int py = oy + r, px = ox + c;
        if (py >= H || px >= W) continue;
        float wgx = 0.f, wgy = 0.f, wal = 0.f, wbe = 0.f;
#pragma unroll
        for (int k = 0; k < PL_TAPS; k++) {
            const float w = wt.w[k];
            wgx = fmaf(w, hb[0][r + k][c], wgx);
            wgy = fmaf(w, hb[1][r + k][c], wgy);
            wal = fmaf(w, hb[2][r + k][c], wal);
            wbe = fmaf(w, hb[3][r + k][c], wbe);
        }
        const float x = sx[r + 2 * PL_R][c + 2 * PL_R], y = sy[r + 2 * PL_R][c + 2 * PL_R];
        const float m = gm * (x - y);
        const size_t o = (size_t)py * W + px;
        if (gp) gp[o] = wgx + 2.f * x * wal + y * wbe + m;
        if (gg) gg[o] = wgy + 2.f * y * wal + x * wbe - m;
    }
}

// the squared-error term alone (no SSIM gradient asked for): element-wise
__global__ void __launch_bounds__(PL_THREADS)
k_mse_bwd(const float *__restrict__ pred, const float *__restrict__ gt, int64_t pred_stride, int64_t gt_stride,
          int64_t n, double inv_n, const float *__restrict__ dL_dmse, float *__restrict__ dpred, float *__restrict__ dgt) {
    const int img = blockIdx.y;
    const float gm = dL_dmse ? (float)(2.0 * (double)dL_dmse[img] * inv_n) : 0.f;
    const float *a = pred + (size_t)img * pred_stride, *b = gt + (size_t)img * gt_stride;
    for (int64_t i = (int64_t)blockIdx.x * PL_THREADS + threadIdx.x; i < n; i += (int64_t)gridDim.x * PL_THREADS) {
        const float m = gm * (a[i] - b[i]);
        if (dpred) dpred[(size_t)img * n + i] = m;
        if (dgt) dgt[(size_t)img * n + i] = -m;
    }
}

int check_config(const GsLossConfig *cfg, const char *who) {
    if (!cfg) return gs_set_error(GS_ERR_INVALID, "photometric loss: null config");
    if (cfg->batch < 0 || cfg->batch > 65535 || cfg->channels < 1 || cfg->channels > 65535 || cfg->height < 1 ||
        cfg->width < 1 || (cfg->with_mse != 0 && cfg->with_mse != 1))
        return gs_set_error(GS_ERR_INVALID, who);
    const int64_t n = (int64_t)cfg->channels * cfg->height * cfg->width;
    if (cfg->batch > 1 && (cfg->pred_stride < n || cfg->gt_stride < n))
        return gs_set_error(GS_ERR_INVALID, "photometric loss: image strides must be at least channels * height * width");
    return GS_OK;
}

int64_t tiles_of(const GsLossConfig *cfg) {
    return (int64_t)((cfg->width + PL_T - 1) / PL_T) * ((cfg->height + PL_T - 1) / PL_T);
}

}  // namespace

extern "C" GS_API int64_t gs_photometric_scratch_bytes(const GsLossConfig *cfg) {
    if (!cfg || check_config(cfg, "bad GsLossConfig") != GS_OK) return -1;
    return 2 * (int64_t)sizeof(double) * cfg->batch * cfg->channels * tiles_of(cfg);
}

extern "C" GS_API int gs_photometric_forward(const GsLossConfig *cfg, const float *predicted, const float *ground_truth,
                                             void *scratch, float *out_ssim, float *out_mse, void *stream) {
    if (int rc = check_config(cfg, "bad GsLossConfig for gs_photometric_forward")) return rc;
    if (!predicted || !ground_truth || !scratch || !out_ssim || (cfg->with_mse && !out_mse))
        return gs_set_error(GS_ERR_INVALID, "gs_photometric_forward: null pointer argument");
    if (reinterpret_cast<uintptr_t>(scratch) & 7u)
        return gs_set_error(GS_ERR_INVALID, "gs_photometric_forward: scratch must be 8-byte aligned");
    if (cfg->batch == 0) return GS_OK;
    const int tiles_x = (cfg->width + PL_T - 1) / PL_T;
    const int64_t tiles = tiles_of(cfg);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    double *partial = static_cast<double *>(scratch);
    k_photometric_fwd<<<dim3((unsigned)tiles, cfg->channels, cfg->batch), PL_THREADS, 0, st>>>(
        predicted, ground_truth, cfg->pred_stride, cfg->gt_stride, cfg->height, cfg->width, tiles_x, window_weights(), partial);
    GS_CUDA_OK(cudaGetLastError());
    const double inv_n = 1.0 / ((double)cfg->channels * cfg->height * cfg->width);
    k_photometric_finalize<<<cfg->batch, 32, 0, st>>>(partial, cfg->batch, (int)(cfg->channels * tiles), inv_n, out_ssim,
                                                      cfg->with_mse ? out_mse : nullptr);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}

extern "C" GS_API int gs_photometric_backward(const GsLossConfig *cfg, const float *predicted, const float *ground_truth,
                                              const float *dL_dssim, const float *dL_dmse, float *dL_dpredicted,
                                              float *dL_dground_truth, void *scratch, void *stream) {
    (void)scratch;  // the backward recomputes what it needs on chip
    if (int rc = check_config(cfg, "bad GsLossConfig for gs_photometric_backward")) return rc;
    if (!predicted || !ground_truth)
        return gs_set_error(GS_ERR_INVALID, "gs_photometric_backward: null image pointer");
    if (!cfg->with_mse) dL_dmse = nullptr;
    if (cfg->batch == 0 || (!dL_dpredicted && !dL_dground_truth)) return GS_OK;
    const int64_t n = (int64_t)cfg->channels * cfg->height * cfg->width;
    const double inv_n = 1.0 / (double)n;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (!dL_dssim && !dL_dmse) {  // no incoming gradient: the gradients are zero
        if (dL_dpredicted) GS_CUDA_OK(cudaMemsetAsync(dL_dpredicted, 0, sizeof(float) * n * cfg->batch, st));
        if (dL_dground_truth) GS_CUDA_OK(cudaMemsetAsync(dL_dground_truth, 0, sizeof(float) * n * cfg->batch, st));
        return GS_OK;
    }
    if (!dL_dssim) {
        int64_t blocks = (n + PL_THREADS - 1) / PL_THREADS;
        if (blocks > 1024) blocks = 1024;
        k_mse_bwd<<<dim3((unsigned)blocks, cfg->batch), PL_THREADS, 0, st>>>(
            predicted, ground_truth, cfg->pred_stride, cfg->gt_stride, n, inv_n, dL_dmse, dL_dpredicted, dL_dground_truth);
        GS_CUDA_OK(cudaGetLastError());
        return GS_OK;
    }
    // 93 KB per CTA (two CTAs per SM): the 10-px halo of a 32 x 32 tile does not fit the 48 KB default
    GS_CUDA_OK(cudaFuncSetAttribute(k_photometric_bwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)PLB_SMEM));
    const int tiles_x = (cfg->width + PL_T - 1) / PL_T;
    k_photometric_bwd<<<dim3((unsigned)tiles_of(cfg), cfg->channels, cfg->batch), PL_THREADS, PLB_SMEM, st>>>(
        predicted, ground_truth, cfg->pred_stride, cfg->gt_stride, cfg->height, cfg->width, tiles_x, window_weights(), inv_n,
        dL_dssim, dL_dmse, dL_dpredicted, dL_dground_truth);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}
