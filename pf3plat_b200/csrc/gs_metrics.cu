// gs_metrics.cu -- PSNR and SSIM of rendered views against ground truth (SURVEY.md section 8(f).4).
//
// Semantics: compute_psnr of PF3plat's src/evaluation/metrics.py:11-19 -- clip both images to [0,1], mean
// squared error over (c,h,w) per image, -10 log10(mse).  One streaming pass with 16-byte loads, per-CTA partial
// sums, a deterministic fp64 finalisation (no atomics, so the result is bit-reproducible).
#include "gs_common.cuh"

namespace {

constexpr int PS_THREADS = 256;
constexpr int MAX_GRID_YZ = 65535;  // gridDim.y and gridDim.z limit: the batch is launched in chunks of at most this

// torch.clip propagates NaN, so a NaN pixel makes the image's PSNR NaN; fminf/fmaxf alone would clip it to 0
__device__ __forceinline__ float clip01(float x) { return x != x ? x : fminf(fmaxf(x, 0.0f), 1.0f); }

__global__ void __launch_bounds__(PS_THREADS)
k_sq_err_partial(const float *__restrict__ gt, const float *__restrict__ pred, int64_t n, float *__restrict__ partial) {
    const int img = blockIdx.y;
    const float *a = gt + (size_t)img * n, *b = pred + (size_t)img * n;
    float acc = 0.f;
    const bool vec = ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b)) & 15u) == 0;
    const int64_t n4 = vec ? n / 4 : 0;
    for (int64_t i = (int64_t)blockIdx.x * PS_THREADS + threadIdx.x; i < n4; i += (int64_t)gridDim.x * PS_THREADS) {
        const float4 x = reinterpret_cast<const float4 *>(a)[i], y = reinterpret_cast<const float4 *>(b)[i];
        const float d0 = clip01(x.x) - clip01(y.x), d1 = clip01(x.y) - clip01(y.y);
        const float d2 = clip01(x.z) - clip01(y.z), d3 = clip01(x.w) - clip01(y.w);
        acc += d0 * d0 + d1 * d1 + d2 * d2 + d3 * d3;
    }
    for (int64_t i = n4 * 4 + (int64_t)blockIdx.x * PS_THREADS + threadIdx.x; i < n; i += (int64_t)gridDim.x * PS_THREADS) {
        const float d = clip01(a[i]) - clip01(b[i]);
        acc += d * d;
    }
    __shared__ float s[PS_THREADS / 32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
#pragma unroll
        for (int w = 0; w < PS_THREADS / 32; w++) t += s[w];
        partial[(size_t)img * gridDim.x + blockIdx.x] = t;
    }
}

__global__ void k_psnr_finalize(const float *__restrict__ partial, int nblocks, int64_t n, float *__restrict__ out) {
    const int img = blockIdx.x;
    double t = 0.0;
    for (int k = threadIdx.x; k < nblocks; k += 32) t += (double)partial[(size_t)img * nblocks + k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if (threadIdx.x == 0) out[img] = (float)(-10.0 * log10(t / (double)n));
}


// ---------------------------------------------------------------------------------------------------------
// SSIM = compute_ssim of PF3plat's src/evaluation/metrics.py:38-54: per image,
//   skimage.metrics.structural_similarity(gt, hat, win_size=11, gaussian_weights=True, channel_axis=0, data_range=1.0)
// (scikit-image is a third-party dependency, unpinned in PF3plat's requirements.txt and absent here; its
// published algorithm, Wang et al. 2004 as implemented there): per channel, Gaussian-weighted local moments with
// sigma = 1.5 truncated at 3.5 sigma (11 taps, scipy.ndimage.gaussian_filter), SAMPLE covariance (x 121/120, the
// use_sample_covariance=True default the reference leaves on), C1 = 0.01^2, C2 = 0.03^2, the SSIM map cropped by
// 5 pixels on every side, mean over the crop (fp64) and over channels.  Because the crop equals the filter radius,
// no retained pixel's window touches the border: the filter's boundary mode never matters.
//
// One CTA per 32x32 tile of the cropped map and channel: the 42x42 input patch of both images is staged in shared
// memory once, the separable filter runs on the five moment images out of shared memory, and the per-tile sums are
// reduced deterministically (fp64, no atomics) by k_ssim_finalize.
//
// The moments are taken of x - x0 and y - y0, with (x0, y0) the tile's first map pixel: variance and covariance do
// not change under a shift, and w*x = w*(x - x0) + x0.  Unshifted, w*(x^2) - (w*x)^2 cancels in fp32 to a spurious
// variance of ~1e-7 x^2, which against C2 = 9e-4 moved S by ~1e-4 on flat bright regions (scipy's filter, which the
// reference uses, accumulates in fp64 and has no such error).  The last stage rounds every operation on its own
// (__f*_rn, no contraction), so that identical images give A1 = B1 and A2 = B2 and hence exactly 1.
// ---------------------------------------------------------------------------------------------------------
constexpr int SS_TILE = 32, SS_R = 5, SS_TAPS = 2 * SS_R + 1, SS_IN = SS_TILE + 2 * SS_R, SS_THREADS = 256;

struct SsimWeights {
    float w[SS_TAPS];
};

__global__ void __launch_bounds__(SS_THREADS)
k_ssim_partial(const float *__restrict__ gt, const float *__restrict__ pred, int H, int W, int tiles_x, int tiles_y,
               const SsimWeights wt, double *__restrict__ partial) {
    __shared__ float sx[SS_IN][SS_IN + 1], sy[SS_IN][SS_IN + 1];
    __shared__ float hq[5][SS_IN][SS_TILE + 1];  // horizontally filtered x, y, xx, yy, xy
    __shared__ double red[SS_THREADS / 32];
    const int tile = blockIdx.x, ch = blockIdx.y, img = blockIdx.z, tid = threadIdx.x;
    const int ox = (tile % tiles_x) * SS_TILE, oy = (tile / tiles_x) * SS_TILE;  // origin in the cropped map == in the image
    const size_t plane = ((size_t)img * gridDim.y + ch) * (size_t)H * W;
    const float *a = gt + plane, *b = pred + plane;
    // the shift: the image pixel of map pixel (oy, ox), inside the image (oy < H - 10, ox < W - 10)
    const size_t centre = (size_t)(oy + SS_R) * W + (ox + SS_R);
    const float x0 = a[centre], y0 = b[centre];
    for (int e = tid; e < SS_IN * SS_IN; e += SS_THREADS) {
        const int r = e / SS_IN, c = e - r * SS_IN;
        const int iy = oy + r, ix = ox + c;
        const bool in = iy < H && ix < W;  // outside the image: read only by map pixels the crop drops
        sx[r][c] = in ? a[(size_t)iy * W + ix] - x0 : 0.f;
        sy[r][c] = in ? b[(size_t)iy * W + ix] - y0 : 0.f;
    }
    __syncthreads();
    for (int e = tid; e < SS_IN * SS_TILE; e += SS_THREADS) {
        const int r = e / SS_TILE, c = e - r * SS_TILE;
        float mx = 0.f, my = 0.f, mxx = 0.f, myy = 0.f, mxy = 0.f;
#pragma unroll
        for (int k = 0; k < SS_TAPS; k++) {
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
    const int CH = H - 2 * SS_R, CW = W - 2 * SS_R;  // cropped map
    const float cov_norm = (float)(SS_TAPS * SS_TAPS) / (float)(SS_TAPS * SS_TAPS - 1);
    const float C1 = 0.01f * 0.01f, C2 = 0.03f * 0.03f;
    double acc = 0.0;
    for (int e = tid; e < SS_TILE * SS_TILE; e += SS_THREADS) {
        const int r = e / SS_TILE, c = e - r * SS_TILE;
        if (oy + r >= CH || ox + c >= CW) continue;
        float ux = 0.f, uy = 0.f, uxx = 0.f, uyy = 0.f, uxy = 0.f;
#pragma unroll
        for (int k = 0; k < SS_TAPS; k++) {
            const float w = wt.w[k];
            ux = fmaf(w, hq[0][r + k][c], ux);
            uy = fmaf(w, hq[1][r + k][c], uy);
            uxx = fmaf(w, hq[2][r + k][c], uxx);
            uyy = fmaf(w, hq[3][r + k][c], uyy);
            uxy = fmaf(w, hq[4][r + k][c], uxy);
        }
        // shifted moments: ux, uy are w*(x - x0), w*(y - y0)
        const float vx = __fmul_rn(cov_norm, __fsub_rn(uxx, __fmul_rn(ux, ux)));
        const float vy = __fmul_rn(cov_norm, __fsub_rn(uyy, __fmul_rn(uy, uy)));
        const float vxy = __fmul_rn(cov_norm, __fsub_rn(uxy, __fmul_rn(ux, uy)));
        const float mx = __fadd_rn(ux, x0), my = __fadd_rn(uy, y0);
        const float A1 = __fadd_rn(__fmul_rn(__fmul_rn(2.f, mx), my), C1);
        const float B1 = __fadd_rn(__fadd_rn(__fmul_rn(mx, mx), __fmul_rn(my, my)), C1);
        const float A2 = __fadd_rn(__fmul_rn(2.f, vxy), C2), B2 = __fadd_rn(__fadd_rn(vx, vy), C2);
        acc += (double)__fdiv_rn(__fmul_rn(A1, A2), __fmul_rn(B1, B2));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((tid & 31) == 0) red[tid >> 5] = acc;
    __syncthreads();
    if (tid == 0) {
        double t = 0.0;
#pragma unroll
        for (int w = 0; w < SS_THREADS / 32; w++) t += red[w];
        partial[((size_t)img * gridDim.y + ch) * gridDim.x + tile] = t;
    }
}

__global__ void k_ssim_finalize(const double *__restrict__ partial, int per_image, double count, float *__restrict__ out) {
    const int img = blockIdx.x;
    double t = 0.0;
    for (int k = threadIdx.x; k < per_image; k += 32) t += partial[(size_t)img * per_image + k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if (threadIdx.x == 0) out[img] = (float)(t / count);
}

}  // namespace

// scratch: at least gs_psnr_scratch_floats(batch, n) floats
extern "C" GS_API int64_t gs_psnr_scratch_floats(int32_t batch, int64_t n) {
    int64_t blocks = (n / 4 + PS_THREADS - 1) / PS_THREADS;
    if (blocks < 1) blocks = 1;
    if (blocks > 64) blocks = 64;
    return (int64_t)batch * blocks;
}

extern "C" GS_API int gs_psnr(const float *ground_truth, const float *predicted, int32_t batch, int64_t n, float *scratch,
                              float *out, void *stream) {
    if (!ground_truth || !predicted || !scratch || !out || batch < 0 || n < 1) return gs_set_error(GS_ERR_INVALID, "bad gs_psnr arguments");
    if (batch == 0) return GS_OK;
    const int blocks = (int)(gs_psnr_scratch_floats(batch, n) / batch);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    for (int64_t b0 = 0; b0 < batch; b0 += MAX_GRID_YZ) {
        const int nb = (int)(batch - b0 < MAX_GRID_YZ ? batch - b0 : MAX_GRID_YZ);
        k_sq_err_partial<<<dim3(blocks, nb), PS_THREADS, 0, st>>>(ground_truth + (size_t)b0 * n, predicted + (size_t)b0 * n, n,
                                                                 scratch + (size_t)b0 * blocks);
        GS_CUDA_OK(cudaGetLastError());
    }
    k_psnr_finalize<<<batch, 32, 0, st>>>(scratch, blocks, n, out);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}

// scratch: at least gs_ssim_scratch_floats(...) floats (holds fp64 per-tile sums; must be 8-byte aligned)
extern "C" GS_API int64_t gs_ssim_scratch_floats(int32_t batch, int32_t channels, int32_t height, int32_t width) {
    if (batch < 0 || channels < 1 || height < SS_TAPS || width < SS_TAPS) return 0;
    const int64_t tiles = (int64_t)((width - 2 * SS_R + SS_TILE - 1) / SS_TILE) * ((height - 2 * SS_R + SS_TILE - 1) / SS_TILE);
    return 2 * (int64_t)batch * channels * tiles;
}

extern "C" GS_API int gs_ssim(const float *ground_truth, const float *predicted, int32_t batch, int32_t channels,
                              int32_t height, int32_t width, float *scratch, float *out, void *stream) {
    if (!ground_truth || !predicted || !scratch || !out || batch < 0 || channels < 1 || channels > MAX_GRID_YZ)
        return gs_set_error(GS_ERR_INVALID, "bad gs_ssim arguments");
    if (height < SS_TAPS || width < SS_TAPS)  // skimage: "win_size exceeds image extent"
        return gs_set_error(GS_ERR_INVALID, "gs_ssim: images must be at least 11 x 11 (win_size exceeds image extent)");
    if (reinterpret_cast<uintptr_t>(scratch) & 7u) return gs_set_error(GS_ERR_INVALID, "gs_ssim: scratch must be 8-byte aligned");
    if (batch == 0) return GS_OK;
    SsimWeights wt;
    {
        // scipy.ndimage's _gaussian_kernel1d(sigma = 1.5, radius = int(3.5 * 1.5 + 0.5) = 5), normalised in fp64
        double w[SS_TAPS], sum = 0.0;
        for (int k = 0; k < SS_TAPS; k++) {
            const double x = (double)(k - SS_R);
            w[k] = exp(-0.5 / (1.5 * 1.5) * x * x);
            sum += w[k];
        }
        for (int k = 0; k < SS_TAPS; k++) wt.w[k] = (float)(w[k] / sum);
    }
    const int tiles_x = (width - 2 * SS_R + SS_TILE - 1) / SS_TILE, tiles_y = (height - 2 * SS_R + SS_TILE - 1) / SS_TILE;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    double *partial = reinterpret_cast<double *>(scratch);
    const size_t image = (size_t)channels * height * width, per_image = (size_t)channels * tiles_x * tiles_y;
    for (int64_t b0 = 0; b0 < batch; b0 += MAX_GRID_YZ) {
        const int nb = (int)(batch - b0 < MAX_GRID_YZ ? batch - b0 : MAX_GRID_YZ);
        k_ssim_partial<<<dim3(tiles_x * tiles_y, channels, nb), SS_THREADS, 0, st>>>(
            ground_truth + b0 * image, predicted + b0 * image, height, width, tiles_x, tiles_y, wt, partial + b0 * per_image);
        GS_CUDA_OK(cudaGetLastError());
    }
    const double count = (double)channels * (double)(height - 2 * SS_R) * (double)(width - 2 * SS_R);
    k_ssim_finalize<<<batch, 32, 0, st>>>(partial, channels * tiles_x * tiles_y, count, out);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}
