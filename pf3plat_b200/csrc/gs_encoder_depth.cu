// gs_encoder_depth.cu -- the encoder's depth glue between UniDepth and the networks that read it, DESIGN.md 5.15:
//   gs_depth_update   encoder_costvolume.py:265, :285-287 (get_scaleshift :167-172) and the unprojections :304-307,
//                     :506-528: the clamped, shifted depth and its unprojection, forward and backward
//   gs_mono_cue       :292-298, the one-hot mono cue over 128 disparity hypotheses (forward only)
//   gs_pdf_peak       depth_predictor_multiview.py:379-384, max over D of softmax over D, nearest-upsampled
// As stock PyTorch this stretch is a few dozen launches, two .item()s, a blocking host-to-device copy and two
// synchronising matrix inverses.  Here each op is one launch per direction, nothing is read back by the host, and no
// backward uses atomics: each is a gather in a fixed order, so it is bit-reproducible without a flag.
#include "gs_common.cuh"
#include "gs_inverse.cuh"

namespace {

constexpr int DU_THREADS = 256;
constexpr int DU_BWD_WARPS = 8;
constexpr int MONO_THREADS = 256;
constexpr int PDF_THREADS = 256;
constexpr double SHIFT_LIMIT = 5.0;  // get_scaleshift's shift.clamp(min=-5, max=5)

// torch.clamp(x, lo, hi) with tensor bounds: maximum, then minimum, a NaN anywhere propagates
__device__ __forceinline__ double clamp_t(double x, double lo, double hi) {
    const double t = isnan(x) ? x : (isnan(lo) ? lo : fmax(x, lo));
    return isnan(t) ? t : (isnan(hi) ? hi : fmin(t, hi));
}

// clamp's backward mask: the gradient passes where lo <= x <= hi (equality included); a NaN passes nothing
__device__ __forceinline__ bool clamp_pass(double x, double lo, double hi) { return x >= lo && x <= hi; }

// PyTorch's bilinear source index (align_corners = False, no explicit scale): scale = in / out,
// src = max(scale (dst + 1/2) - 1/2, 0), i0 = (int)src, i1 = i0 + (i0 < in - 1), l1 = src - i0, l0 = 1 - l1.
// Evaluated in fp64: in float32 the rounding of src alone moves l1 by up to ~2e-6 on a 40-cell grid, which shifts
// the depth by that much times the difference between neighbouring cells.
struct Tap {
    int i0, i1;
    double l0, l1;
};

__device__ __forceinline__ Tap bilinear_tap(int dst, int in, double scale) {
    double src = scale * (dst + 0.5) - 0.5;
    src = src < 0.0 ? 0.0 : src;
    Tap t;
    t.i0 = (int)src;
    t.i1 = t.i0 + (t.i0 < in - 1 ? 1 : 0);
    t.l1 = src - t.i0;
    t.l0 = 1.0 - t.l1;
    return t;
}

struct DuParams {
    int views, H, W, gh, gw;
    double sy, sx;  // grid / frame per axis
};

// the raw (unclamped) upsampled shift at (y, x) of item n: channel 1 of scale_shift [n, gh gw, 2], evaluated as
// h0 (w0 a + w1 b) + h1 (w0 c + w1 d) in fp64
__device__ __forceinline__ double shift_at(const DuParams &p, const float *__restrict__ ss, int n, const Tap &ty,
                                           const Tap &tx) {
    const float *s = ss + (size_t)n * p.gh * p.gw * 2 + 1;
    const double a = s[(ty.i0 * p.gw + tx.i0) * 2], b = s[(ty.i0 * p.gw + tx.i1) * 2];
    const double c = s[(ty.i1 * p.gw + tx.i0) * 2], d = s[(ty.i1 * p.gw + tx.i1) * 2];
    return ty.l0 * (tx.l0 * a + tx.l1 * b) + ty.l1 * (tx.l0 * c + tx.l1 * d);
}

__device__ __forceinline__ double clamp_shift(double s) {
    return isnan(s) ? s : fmin(fmax(s, -SHIFT_LIMIT), SHIFT_LIMIT);
}

__device__ __forceinline__ float pixel_u(int x, int w) { return __fdiv_rn(__fadd_rn((float)x, 0.5f), (float)w); }

// One thread per full-resolution pixel; a CTA's prologue inverts its item's K in fp64 into shared memory.
__global__ void __launch_bounds__(DU_THREADS)
k_depth_update_fwd(DuParams p, const float *__restrict__ depth, const float *__restrict__ ss,
                   const float *__restrict__ K, const float *__restrict__ near_, const float *__restrict__ far_,
                   float *__restrict__ depths, float *__restrict__ xyz) {
    __shared__ double kinv[9];
    const int n = blockIdx.y;
    if (threadIdx.x == 0) {
        double k[9];
        for (int i = 0; i < 9; i++) k[i] = K[(size_t)n * 9 + i];
        inverse3(k, kinv);
    }
    __syncthreads();
    const int hw = p.H * p.W, px = blockIdx.x * DU_THREADS + threadIdx.x;
    if (px >= hw) return;
    const int y = px / p.W, x = px % p.W;
    const double lo = near_[n], hi = far_[n];
    const double d0 = clamp_t(depth[(size_t)n * hw + px], lo, hi);
    const double sraw = shift_at(p, ss, n, bilinear_tap(y, p.gh, p.sy), bilinear_tap(x, p.gw, p.sx));
    const float out = (float)clamp_t(d0 + clamp_shift(sraw), lo, hi);  // rounded once; a clamped value is lo or hi
    depths[(size_t)n * hw + px] = out;
    const double u = pixel_u(x, p.W), v = pixel_u(y, p.H);
    float *o = xyz + (size_t)n * 3 * hw + px;
    for (int i = 0; i < 3; i++) o[(size_t)i * hw] = (float)((kinv[i * 3] * u + kinv[i * 3 + 1] * v + kinv[i * 3 + 2]) * out);
}

// the destination range [lo, hi] that may tap source cell i (i0 in {i - 1, i}), with a margin; each candidate is
// then checked exactly with bilinear_tap
__device__ __forceinline__ void dst_range(int i, int out, double s, int &lo, int &hi) {
    lo = max(0, (int)floor((i - 0.5) / s - 0.5) - 2);
    hi = min(out - 1, (int)ceil((i + 1.5) / s - 0.5) + 2);
}

// One warp per feature-grid cell: the lanes walk the cell's candidate pixels in a fixed order, recompute each
// pixel's masked cotangent g = (dL/ddepths + dL/dxyz . K^-1 [u, v, 1]) and add (l_y l_x) g for each of the
// pixel's four taps that lands on the cell (the forward's own weights); a fixed shuffle tree sums the lanes.
__global__ void __launch_bounds__(DU_BWD_WARPS * 32)
k_depth_update_bwd(DuParams p, int cells, const float *__restrict__ depth, const float *__restrict__ ss,
                   const float *__restrict__ K, const float *__restrict__ near_, const float *__restrict__ far_,
                   const float *__restrict__ g_depths, const float *__restrict__ g_xyz, float *__restrict__ d_ss) {
    const int warp = blockIdx.x * DU_BWD_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (warp >= cells) return;
    const int gcells = p.gh * p.gw, n = warp / gcells, cell = warp % gcells, cy = cell / p.gw, cx = cell % p.gw;
    double kinv[9];
    if (g_xyz) {
        double k[9];
        for (int i = 0; i < 9; i++) k[i] = K[(size_t)n * 9 + i];
        inverse3(k, kinv);
    }
    int y0, y1, x0, x1;
    dst_range(cy, p.H, p.sy, y0, y1);
    dst_range(cx, p.W, p.sx, x0, x1);
    const int ny = y1 - y0 + 1, nx = x1 - x0 + 1, hw = p.H * p.W;
    const double lo = near_[n], hi = far_[n];
    double acc = 0.0;
    for (int t = lane; t < ny * nx; t += 32) {
        const int y = y0 + t / nx, x = x0 + t % nx;
        const Tap ty = bilinear_tap(y, p.gh, p.sy), tx = bilinear_tap(x, p.gw, p.sx);
        const bool hy0 = ty.i0 == cy, hy1 = ty.i1 == cy, hx0 = tx.i0 == cx, hx1 = tx.i1 == cx;
        if (!((hy0 || hy1) && (hx0 || hx1))) continue;
        const int px = y * p.W + x;
        const double d0 = clamp_t(depth[(size_t)n * hw + px], lo, hi);
        const double sraw = shift_at(p, ss, n, ty, tx);
        if (!clamp_pass(sraw, -SHIFT_LIMIT, SHIFT_LIMIT) || !clamp_pass(d0 + clamp_shift(sraw), lo, hi)) continue;
        double g = g_depths ? (double)g_depths[(size_t)n * hw + px] : 0.0;
        if (g_xyz) {
            const double u = pixel_u(x, p.W), v = pixel_u(y, p.H);
            const float *gx = g_xyz + (size_t)n * 3 * hw + px;
            for (int i = 0; i < 3; i++)
                g += (double)gx[(size_t)i * hw] * (kinv[i * 3] * u + kinv[i * 3 + 1] * v + kinv[i * 3 + 2]);
        }
        if (hy0 && hx0) acc += ty.l0 * tx.l0 * g;
        if (hy0 && hx1) acc += ty.l0 * tx.l1 * g;
        if (hy1 && hx0) acc += ty.l1 * tx.l0 * g;
        if (hy1 && hx1) acc += ty.l1 * tx.l1 * g;
    }
    for (int off = 16; off > 0; off >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, off);
    if (lane == 0) {
        float *o = d_ss + (size_t)warp * 2;
        o[0] = 0.0f;
        o[1] = (float)acc;
    }
}

// One thread per downsampled pixel of one (v b) output item.  The CTA builds the 128 hypotheses from near_[0],
// far_[0] and the linspace table in shared memory, exactly as the reference's float32 ops round them.
__global__ void __launch_bounds__(MONO_THREADS)
k_mono_cue(int batch, int views, int H, int W, const float *__restrict__ depths, const float *__restrict__ near_,
           const float *__restrict__ far_, const float *__restrict__ lin, float *__restrict__ out) {
    __shared__ float hyp[GS_MONO_CUE_BINS];
    if (threadIdx.x < GS_MONO_CUE_BINS) {
        const float a = __fdiv_rn(1.0f, far_[0]), inv_near = __fdiv_rn(1.0f, near_[0]);
        const float B = (float)((double)inv_near - (double)a);  // the .item() difference in double, cast by the mul
        hyp[threadIdx.x] = __fadd_rn(a, __fmul_rn(lin[threadIdx.x], B));
    }
    __syncthreads();
    const int m = blockIdx.y, vi = m / batch, bi = m % batch, n = bi * views + vi;
    const int h4 = H >> 2, w4 = W >> 2, hw4 = h4 * w4, px = blockIdx.x * MONO_THREADS + threadIdx.x;
    if (px >= hw4) return;
    const int i = px / w4, j = px % w4;
    const float *src = depths + (size_t)n * H * W + (size_t)(4 * i + 1) * W + 4 * j + 1;
    const float a = src[0], b = src[1], c = src[W], d = src[W + 1];
    // h0 (w0 a + w1 b) + h1 (w0 c + w1 d) with every weight 1/2: each product is exact
    const float dn = __fadd_rn(__fmul_rn(0.5f, __fadd_rn(__fmul_rn(0.5f, a), __fmul_rn(0.5f, b))),
                               __fmul_rn(0.5f, __fadd_rn(__fmul_rn(0.5f, c), __fmul_rn(0.5f, d))));
    float best = fabsf(__fsub_rn(dn, hyp[0]));
    int bin = 0;
    for (int k = 1; k < GS_MONO_CUE_BINS && !isnan(best); k++) {
        const float e = fabsf(__fsub_rn(dn, hyp[k]));
        if (e < best || isnan(e)) {
            best = e;
            bin = k;
        }
    }
    float *o = out + (size_t)m * GS_MONO_CUE_BINS * hw4 + px;
    for (int k = 0; k < GS_MONO_CUE_BINS; k++) o[(size_t)k * hw4] = k == bin ? 1.0f : 0.0f;
}

// nearest upsampling's source index (scale_factor s): min(floor(dst * fl32(1 / s)), in - 1)
__device__ __forceinline__ int nearest_src(int dst, int in, float inv_s) {
    return min((int)floorf(__fmul_rn((float)dst, inv_s)), in - 1);
}

// One thread per low-resolution pixel: max (NaN wins, ties to the lowest index), then 1 / sum exp(x_k - x_max).
__global__ void __launch_bounds__(PDF_THREADS)
k_pdf_peak_fwd(int D, int H, int W, int s, float inv_s, const float *__restrict__ logits, float *__restrict__ out,
               float *__restrict__ peak, int32_t *__restrict__ argmax) {
    const int n = blockIdx.y, hw = H * W, px = blockIdx.x * PDF_THREADS + threadIdx.x;
    if (px >= hw) return;
    const float *x = logits + (size_t)n * D * hw + px;
    float m = x[0];
    int km = 0;
    for (int k = 1; k < D; k++) {
        const float v = x[(size_t)k * hw];
        if (!isnan(m) && (v > m || isnan(v))) {
            m = v;
            km = k;
        }
    }
    float sum = 0.0f;
    for (int k = 0; k < D; k++) sum += expf(x[(size_t)k * hw] - m);
    const float p = 1.0f / sum;
    peak[(size_t)n * hw + px] = p;
    argmax[(size_t)n * hw + px] = km;
    const int y = px / W, xx = px % W, Ho = H * s, Wo = W * s;
    float *o = out + (size_t)n * Ho * Wo;
    for (int oy = max(0, y * s - 1); oy <= min(Ho - 1, y * s + s); oy++) {
        if (nearest_src(oy, H, inv_s) != y) continue;
        for (int ox = max(0, xx * s - 1); ox <= min(Wo - 1, xx * s + s); ox++)
            if (nearest_src(ox, W, inv_s) == xx) o[(size_t)oy * Wo + ox] = p;
    }
}

// One thread per low-resolution pixel: G = the pixel's upsampled cotangents summed row by row, then
// dL/dx_k = G p* (delta_{k, k*} - p_k) with p_k = exp(x_k - x_{k*}) p*.
__global__ void __launch_bounds__(PDF_THREADS)
k_pdf_peak_bwd(int D, int H, int W, int s, float inv_s, const float *__restrict__ logits,
               const float *__restrict__ peak, const int32_t *__restrict__ argmax, const float *__restrict__ g_out,
               float *__restrict__ g_logits) {
    const int n = blockIdx.y, hw = H * W, px = blockIdx.x * PDF_THREADS + threadIdx.x;
    if (px >= hw) return;
    const int y = px / W, xx = px % W, Ho = H * s, Wo = W * s;
    const float *go = g_out + (size_t)n * Ho * Wo;
    float G = 0.0f;
    for (int oy = max(0, y * s - 1); oy <= min(Ho - 1, y * s + s); oy++) {
        if (nearest_src(oy, H, inv_s) != y) continue;
        for (int ox = max(0, xx * s - 1); ox <= min(Wo - 1, xx * s + s); ox++)
            if (nearest_src(ox, W, inv_s) == xx) G += go[(size_t)oy * Wo + ox];
    }
    const float p = peak[(size_t)n * hw + px];
    const int km = argmax[(size_t)n * hw + px];
    const float *x = logits + (size_t)n * D * hw + px;
    const float m = x[(size_t)km * hw], Gp = G * p;
    float *o = g_logits + (size_t)n * D * hw + px;
    for (int k = 0; k < D; k++) {
        const float pk = expf(x[(size_t)k * hw] - m) * p;
        o[(size_t)k * hw] = Gp * ((k == km ? 1.0f : 0.0f) - pk);
    }
}

int du_params(const GsDepthUpdateConfig *c, const GsDepthUpdateInputs *in, DuParams *p) {
    if (!c || c->batch < 1 || c->views < 1 || c->height < 1 || c->width < 1 || c->grid_height < 1 ||
        c->grid_width < 1 || (int64_t)c->batch * c->views > 65535 || (int64_t)c->height * c->width > (1 << 28) ||
        (int64_t)c->grid_height * c->grid_width > (1 << 24) ||
        (int64_t)c->batch * c->views * c->grid_height * c->grid_width > (1ll << 31) - 1 - 32 * DU_BWD_WARPS)
        return gs_set_error(GS_ERR_INVALID, "depth update: need batch, views, height, width, grid >= 1, batch views "
                                            "<= 65535, height width <= 2^28, batch views grid cells < 2^31");
    if (!in || !in->depth || !in->scale_shift || !in->intrinsics || !in->near_ || !in->far_)
        return gs_set_error(GS_ERR_INVALID, "depth update: null input pointer");
    p->views = c->views;
    p->H = c->height;
    p->W = c->width;
    p->gh = c->grid_height;
    p->gw = c->grid_width;
    p->sy = (double)c->grid_height / c->height;
    p->sx = (double)c->grid_width / c->width;
    return GS_OK;
}

int pdf_check(const GsPdfPeakConfig *c) {
    if (!c || c->items < 1 || c->items > 65535 || c->depth_candidates < 1 || c->height < 1 || c->width < 1 ||
        c->upscale < 1 || (int64_t)c->height * c->width * c->upscale * c->upscale > (1 << 28))
        return gs_set_error(GS_ERR_INVALID, "pdf peak: need 1 <= items <= 65535, depth_candidates, height, width, "
                                            "upscale >= 1, (height upscale) (width upscale) <= 2^28");
    return GS_OK;
}

}  // namespace

extern "C" GS_API int gs_depth_update_forward(const GsDepthUpdateConfig *cfg, const GsDepthUpdateInputs *in,
                                              float *depths, float *xyz, void *stream) {
    DuParams p;
    if (int rc = du_params(cfg, in, &p)) return rc;
    if (!depths || !xyz) return gs_set_error(GS_ERR_INVALID, "gs_depth_update_forward: null output pointer");
    const int hw = cfg->height * cfg->width;
    const dim3 grid((hw + DU_THREADS - 1) / DU_THREADS, cfg->batch * cfg->views);
    k_depth_update_fwd<<<grid, DU_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
        p, in->depth, in->scale_shift, in->intrinsics, in->near_, in->far_, depths, xyz);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}

extern "C" GS_API int gs_depth_update_backward(const GsDepthUpdateConfig *cfg, const GsDepthUpdateInputs *in,
                                               const GsDepthUpdateGrads *grads, void *stream) {
    DuParams p;
    if (int rc = du_params(cfg, in, &p)) return rc;
    if (!grads || !grads->dL_dscale_shift)
        return gs_set_error(GS_ERR_INVALID, "gs_depth_update_backward: null gradient pointer");
    const int cells = cfg->batch * cfg->views * cfg->grid_height * cfg->grid_width;
    k_depth_update_bwd<<<(cells + DU_BWD_WARPS - 1) / DU_BWD_WARPS, DU_BWD_WARPS * 32, 0,
                         static_cast<cudaStream_t>(stream)>>>(p, cells, in->depth, in->scale_shift, in->intrinsics,
                                                              in->near_, in->far_, grads->dL_ddepths, grads->dL_dxyz,
                                                              grads->dL_dscale_shift);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}

extern "C" GS_API int gs_mono_cue(const GsMonoCueConfig *cfg, const float *depths, const float *near_,
                                  const float *far_, const float *lin, float *out, void *stream) {
    if (!cfg || cfg->batch < 1 || cfg->views < 1 || (int64_t)cfg->batch * cfg->views > 65535 || cfg->height < 4 ||
        cfg->width < 4 || cfg->height % 4 || cfg->width % 4 || (int64_t)cfg->height * cfg->width > (1 << 28))
        return gs_set_error(GS_ERR_INVALID, "gs_mono_cue: need batch, views >= 1, batch views <= 65535, height and "
                                            "width positive multiples of 4, height width <= 2^28");
    if (!depths || !near_ || !far_ || !lin || !out) return gs_set_error(GS_ERR_INVALID, "gs_mono_cue: null pointer");
    const int hw4 = (cfg->height / 4) * (cfg->width / 4);
    const dim3 grid((hw4 + MONO_THREADS - 1) / MONO_THREADS, cfg->batch * cfg->views);
    k_mono_cue<<<grid, MONO_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(cfg->batch, cfg->views, cfg->height,
                                                                            cfg->width, depths, near_, far_, lin, out);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}

extern "C" GS_API int gs_pdf_peak_forward(const GsPdfPeakConfig *cfg, const float *logits, float *out, float *peak,
                                          int32_t *argmax, void *stream) {
    if (int rc = pdf_check(cfg)) return rc;
    if (!logits || !out || !peak || !argmax) return gs_set_error(GS_ERR_INVALID, "gs_pdf_peak_forward: null pointer");
    const int hw = cfg->height * cfg->width;
    const dim3 grid((hw + PDF_THREADS - 1) / PDF_THREADS, cfg->items);
    k_pdf_peak_fwd<<<grid, PDF_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
        cfg->depth_candidates, cfg->height, cfg->width, cfg->upscale, (float)(1.0 / cfg->upscale), logits, out, peak,
        argmax);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}

extern "C" GS_API int gs_pdf_peak_backward(const GsPdfPeakConfig *cfg, const float *logits, const float *peak,
                                           const int32_t *argmax, const float *dL_dout, float *dL_dlogits,
                                           void *stream) {
    if (int rc = pdf_check(cfg)) return rc;
    if (!logits || !peak || !argmax || !dL_dout || !dL_dlogits)
        return gs_set_error(GS_ERR_INVALID, "gs_pdf_peak_backward: null pointer");
    const int hw = cfg->height * cfg->width;
    const dim3 grid((hw + PDF_THREADS - 1) / PDF_THREADS, cfg->items);
    k_pdf_peak_bwd<<<grid, PDF_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
        cfg->depth_candidates, cfg->height, cfg->width, cfg->upscale, (float)(1.0 / cfg->upscale), logits, peak,
        argmax, dL_dout, dL_dlogits);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}
