// gs_costvolume.cu -- the plane-sweep correlation of PF3plat's depth predictor on the device:
// DepthPredictorMultiView.forward, src/model/encoder/costvolume/depth_predictor_multiview.py:309-343, up to the
// torch.cat, forward and backward, without the warped feature volume.
//
// Semantics (DESIGN.md 5.13).  Views are in the reference's (v b) order, vb = vi b + bi.  For target vb and source slot
// s = 1 .. v-1 the source is vb_s = ((vi + s) mod v) b + bi (prepare_feat_proj_data_lists, :91-141), with the pose
//   v > 2:  P = E[bi, (vi + s) mod v]^-1 E[bi, vi]
//   v = 2:  P0 = E[bi, 1]^-1 E[bi, 0];  P = P0 (vi = 0) or P0^-1 (vi = 1)
// and the TARGET view's intrinsics, un-normalised row-wise (row 0 x w, row 1 x h).  A target pixel (x, y) (pixel
// indices, coords_grid) at candidate depth z_d = 1 / (1/far + t_d (1/near - 1/far)), t_d = linspace(0, 1, D)[d], lands at
//   q = z_d H [x, y, 1] + e,  H = K R K^-1,  e = K t  (R, t of P),  (ix, iy) = q_xy / max(q_z, 1e-3)
// (warp_with_pose_depth_candidates, :28-88; a point behind the source camera is divided by 1e-3, not culled).  The
// sample is grid_sample's bilinear, align_corners=True, zero padding per tap: every in-bounds tap is multiplied in,
// weight 0 or not.  Then
//   cost[vb, d, p] = mean_s ( sum_c f01[vb, c, p] warped_s[c, d, p] / sqrt(C) ).
//
// Layout: features are packed once per call into channel-last rows F[(vb) h w][Cp] (Cp = C rounded up to 4, the pad
// zero), so a tap is one contiguous row.  Camera math (inverses, H, e, z_d) is fp64, in k_cv_cameras; the per-sample
// projection is fp64 too (a few DFMA and two divisions per sample, next to a 4 Cp-float gather).
//
// Per-pixel kernels: one warp per target pixel.  Lane l holds float4 chunks l and l + 32 of f01[p] (256 channels) in
// registers; wider features run in passes of 256 channels.  For every depth and source the warp gathers the in-bounds
// taps, forms warped[c] per channel as grid_sample does and reduces f01 . warped.
//   k_cv_forward:  writes cost[vb, d, p] only.
//   k_cv_backward: the f01 role, sum_{d,s} g'[d,p] warped_s[c,d,p] with g' = dL/dcost / sqrt(C) / (v-1), is kept in
//     registers and stored once per pixel (G1 rows: no atomics).  The source role scatters w_tap g'[d,p] f01[p] into
//     the taps' rows: default, one red.global.add.v4.f32 per lane and float4; GS_COSTVOLUME_DETERMINISTIC, the exact
//     fixed-point limbs of gs_det.cuh (DESIGN.md 5.11) with a per-element poison bit for non-finite terms.
//   k_cv_finalize: dL/dfeatures[b, v, c, h, w] = G1 + the source accumulator, transposed back.
#include "gs_common.cuh"

namespace {

constexpr int CV_THREADS = 256, CV_WARPS = CV_THREADS / 32;
constexpr int CV_NCH = 2;                       // float4 chunks per lane per pass
constexpr int CV_PASS_CHUNKS = 32 * CV_NCH;     // 64 float4 = 256 channels per pass
constexpr double CV_ZMIN = 1e-3;

struct CvCam {
    double H[9], e[3];
};

__device__ void inv_gauss_jordan(const double *a, int n, double *out) {  // n <= 4, partial pivoting
    double m[4][8];
    for (int i = 0; i < n; i++)
        for (int j = 0; j < n; j++) {
            m[i][j] = a[i * n + j];
            m[i][n + j] = i == j ? 1.0 : 0.0;
        }
    for (int c = 0; c < n; c++) {
        int piv = c;
        for (int r = c + 1; r < n; r++)
            if (fabs(m[r][c]) > fabs(m[piv][c])) piv = r;
        if (piv != c)
            for (int j = 0; j < 2 * n; j++) {
                const double t = m[c][j];
                m[c][j] = m[piv][j];
                m[piv][j] = t;
            }
        const double inv = 1.0 / m[c][c];
        for (int j = 0; j < 2 * n; j++) m[c][j] *= inv;
        for (int r = 0; r < n; r++) {
            if (r == c) continue;
            const double f = m[r][c];
            for (int j = 0; j < 2 * n; j++) m[r][j] -= f * m[c][j];
        }
    }
    for (int i = 0; i < n; i++)
        for (int j = 0; j < n; j++) out[i * n + j] = m[i][n + j];
}

__device__ void matmul4(const double *a, const double *b, double *o) {
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++) {
            double s = 0.0;
            for (int k = 0; k < 4; k++) s += a[i * 4 + k] * b[k * 4 + j];
            o[i * 4 + j] = s;
        }
}

// one thread per (target vb, source slot): H and e; the slot-0 thread of each vb also writes its D candidate depths
__global__ void k_cv_cameras(GsCostVolumeConfig c, const float *__restrict__ intr, const float *__restrict__ ext,
                             const float *__restrict__ near_, const float *__restrict__ far_, CvCam *__restrict__ cams,
                             double *__restrict__ depth) {
    const int b = c.batch, v = c.views, ns = v - 1;
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= v * b * ns) return;
    const int vb = t / ns, s = t - vb * ns + 1, vi = vb / b, bi = vb - vi * b;
    double E0[16], E1[16], inv1[16], P[16];
    const int v0 = v == 2 ? 0 : vi, v1 = v == 2 ? 1 : (vi + s) % v;
    for (int k = 0; k < 16; k++) {
        E0[k] = ext[((size_t)bi * v + v0) * 16 + k];
        E1[k] = ext[((size_t)bi * v + v1) * 16 + k];
    }
    inv_gauss_jordan(E1, 4, inv1);
    matmul4(inv1, E0, P);
    if (v == 2 && vi == 1) {
        double Pi[16];
        inv_gauss_jordan(P, 4, Pi);
        for (int k = 0; k < 16; k++) P[k] = Pi[k];
    }
    const int rows = c.intrinsics_rows;
    double K[9], Ki[9];
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
            const double scale = i == 0 ? (double)c.width : i == 1 ? (double)c.height : 1.0;
            K[i * 3 + j] = (double)intr[((size_t)bi * v + vi) * rows * rows + i * rows + j] * scale;
        }
    inv_gauss_jordan(K, 3, Ki);
    double KR[9];
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) KR[i * 3 + j] = K[i * 3] * P[j] + K[i * 3 + 1] * P[4 + j] + K[i * 3 + 2] * P[8 + j];
    CvCam o;
    for (int i = 0; i < 3; i++) {
        for (int j = 0; j < 3; j++) o.H[i * 3 + j] = KR[i * 3] * Ki[j] + KR[i * 3 + 1] * Ki[3 + j] + KR[i * 3 + 2] * Ki[6 + j];
        o.e[i] = K[i * 3] * P[3] + K[i * 3 + 1] * P[7] + K[i * 3 + 2] * P[11];
    }
    cams[t] = o;
    if (s == 1) {
        const double lo = 1.0 / (double)far_[(size_t)bi * v + vi], hi = 1.0 / (double)near_[(size_t)bi * v + vi];
        const int D = c.depth_candidates;
        for (int d = 0; d < D; d++) {
            const double td = D > 1 ? (double)d / (double)(D - 1) : 0.0;
            depth[(size_t)vb * D + d] = 1.0 / (lo + td * (hi - lo));
        }
    }
}

// Packs features [b, v, C, h, w] (any strides) into F[(vb) h w][Cp]; 32 x 32 tiles of (pixel, channel) through shared
// memory, so both sides are read and written along their contiguous axis.
__global__ void __launch_bounds__(CV_THREADS) k_cv_pack(GsCostVolumeConfig c, int Cp, const float *__restrict__ feat,
                                                        float *__restrict__ F) {
    __shared__ float tile[32][33];
    const int hw = c.height * c.width, vb = blockIdx.z, vi = vb / c.batch, bi = vb - vi * c.batch;
    const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    const int64_t *st = c.feat_stride;
    const float *src = feat + bi * st[0] + vi * st[1];
    for (int r = threadIdx.y; r < 32; r += blockDim.y) {  // r: channel, threadIdx.x: pixel
        const int ch = c0 + r, p = p0 + threadIdx.x;
        float val = 0.f;
        if (ch < c.channels && p < hw) {
            const int y = p / c.width, x = p - y * c.width;
            val = src[ch * st[2] + y * st[3] + x * st[4]];
        }
        tile[r][threadIdx.x] = val;
    }
    __syncthreads();
    for (int r = threadIdx.y; r < 32; r += blockDim.y) {  // r: pixel, threadIdx.x: channel
        const int p = p0 + r, ch = c0 + threadIdx.x;
        if (p < hw && ch < Cp) F[((size_t)vb * hw + p) * Cp + ch] = tile[threadIdx.x][r];
    }
}

// The four taps of one sample: row offsets into F (in float4 units of the pass) and weights; row -1 = out of bounds.
struct Taps {
    int64_t row[4];
    float w[4];
};

__device__ __forceinline__ void sample_taps(const CvCam &cam, double x, double y, double z, int h, int w, int64_t src_base,
                                            Taps &t) {
    const double hx = cam.H[0] * x + cam.H[1] * y + cam.H[2];
    const double hy = cam.H[3] * x + cam.H[4] * y + cam.H[5];
    const double hz = cam.H[6] * x + cam.H[7] * y + cam.H[8];
    const double qx = z * hx + cam.e[0], qy = z * hy + cam.e[1], qz0 = z * hz + cam.e[2];
    const double qz = qz0 < CV_ZMIN ? CV_ZMIN : qz0;  // clamp(min=1e-3); a NaN stays NaN
    const double ix = qx / qz, iy = qy / qz;
    const double x0 = floor(ix), y0 = floor(iy);
    const double ax = ix - x0, ay = iy - y0;
    t.w[0] = (float)((1.0 - ax) * (1.0 - ay));
    t.w[1] = (float)(ax * (1.0 - ay));
    t.w[2] = (float)((1.0 - ax) * ay);
    t.w[3] = (float)(ax * ay);
    // bounds in floating point first (NaN and huge coordinates are out), then the integer index
    const bool xin0 = x0 >= 0.0 && x0 <= (double)(w - 1), xin1 = x0 + 1.0 >= 0.0 && x0 + 1.0 <= (double)(w - 1);
    const bool yin0 = y0 >= 0.0 && y0 <= (double)(h - 1), yin1 = y0 + 1.0 >= 0.0 && y0 + 1.0 <= (double)(h - 1);
    const int64_t xi = xin0 || xin1 ? (int64_t)x0 : 0, yi = yin0 || yin1 ? (int64_t)y0 : 0;
    const int64_t r00 = src_base + yi * w + xi;
    t.row[0] = xin0 && yin0 ? r00 : -1;
    t.row[1] = xin1 && yin0 ? r00 + 1 : -1;
    t.row[2] = xin0 && yin1 ? r00 + w : -1;
    t.row[3] = xin1 && yin1 ? r00 + w + 1 : -1;
}

__device__ __forceinline__ float4 fma4(float s, float4 a, float4 acc) {
    return make_float4(fmaf(s, a.x, acc.x), fmaf(s, a.y, acc.y), fmaf(s, a.z, acc.z), fmaf(s, a.w, acc.w));
}

// warped[c] of one sample, tap by tap in grid_sample's order (nw, ne, sw, se), in-bounds taps only
__device__ __forceinline__ float4 gather(const float4 *__restrict__ F4, int64_t Cp4, int j, const Taps &t) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int k = 0; k < 4; k++)
        if (t.row[k] >= 0) acc = fma4(t.w[k], __ldg(F4 + t.row[k] * Cp4 + j), acc);
    return acc;
}

__device__ __forceinline__ float dot4(float4 a, float4 b) { return a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w; }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__global__ void __launch_bounds__(CV_THREADS) k_cv_forward(GsCostVolumeConfig c, int Cp, const float *__restrict__ F,
                                                           const CvCam *__restrict__ cams,
                                                           const double *__restrict__ depth, float *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int64_t hw = (int64_t)c.height * c.width;
    const int64_t pg = (int64_t)blockIdx.x * CV_WARPS + (threadIdx.x >> 5);
    if (pg >= hw * c.batch * c.views) return;
    const int vb = (int)(pg / hw), vi = vb / c.batch, bi = vb - vi * c.batch;
    const int64_t pix = pg - (int64_t)vb * hw;
    const int py = (int)(pix / c.width), px = (int)(pix - (int64_t)py * c.width);
    const int v = c.views, ns = v - 1, D = c.depth_candidates;
    const int64_t Cp4 = Cp / 4;
    const float4 *F4 = reinterpret_cast<const float4 *>(F);
    const float scale = (float)(1.0 / sqrt((double)c.channels) / (double)ns);
    for (int j0 = 0; j0 < Cp4; j0 += CV_PASS_CHUNKS) {
        float4 f01[CV_NCH];
#pragma unroll
        for (int k = 0; k < CV_NCH; k++) {
            const int j = j0 + lane + 32 * k;
            f01[k] = j < Cp4 ? F4[pg * Cp4 + j] : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        for (int d = 0; d < D; d++) {
            const double z = depth[(size_t)vb * D + d];
            float acc = 0.f;
            for (int s = 1; s <= ns; s++) {
                const CvCam cam = cams[(size_t)vb * ns + (s - 1)];
                const int vs = (vi + s) % v;
                Taps t;
                sample_taps(cam, (double)px, (double)py, z, c.height, c.width, ((int64_t)vs * c.batch + bi) * hw, t);
#pragma unroll
                for (int k = 0; k < CV_NCH; k++) {
                    const int j = j0 + lane + 32 * k;
                    if (j < Cp4) acc += dot4(f01[k], gather(F4, Cp4, j, t));
                }
            }
            acc = warp_sum(acc);
            if (lane == 0) {
                float *o = out + ((int64_t)vb * D + d) * hw + pix;
                *o = j0 == 0 ? acc * scale : *o + acc * scale;
            }
        }
    }
}

__device__ __forceinline__ void red_add_v4(float4 *addr, float4 v) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
                 : "memory");
}

// the exact fixed-point add of one float4 term into element rows e .. e+3 (channels 4j .. 4j+3)
__device__ __forceinline__ void det_add4(unsigned long long *__restrict__ limbs, uint32_t *__restrict__ poison, int PW,
                                         int64_t row, int64_t Cp, int j, float4 v) {
    const float vals[4] = {v.x, v.y, v.z, v.w};
    uint32_t bad = 0;
#pragma unroll
    for (int q = 0; q < 4; q++) {
        if (vals[q] == 0.f) continue;
        long long limb[GS_DET_LIMBS];
        if (!gs_det_encode(vals[q], limb)) {
            bad |= 1u << ((4 * j + q) & 31);
            continue;
        }
        unsigned long long *dst = limbs + (row * Cp + 4 * j + q) * GS_DET_LIMBS;
#pragma unroll
        for (int k = 0; k < GS_DET_LIMBS; k++)
            if (limb[k]) atomicAdd(dst + k, (unsigned long long)limb[k]);
    }
    if (bad) atomicOr(poison + row * PW + (4 * j) / 32, bad);
}

template <bool DET>
__global__ void __launch_bounds__(CV_THREADS)
k_cv_backward(GsCostVolumeConfig c, int Cp, const float *__restrict__ F, const CvCam *__restrict__ cams,
              const double *__restrict__ depth, const float *__restrict__ dcost, float *__restrict__ G1,
              float *__restrict__ acc, unsigned long long *__restrict__ limbs, uint32_t *__restrict__ poison) {
    const int lane = threadIdx.x & 31;
    const int64_t hw = (int64_t)c.height * c.width;
    const int64_t pg = (int64_t)blockIdx.x * CV_WARPS + (threadIdx.x >> 5);
    if (pg >= hw * c.batch * c.views) return;
    const int vb = (int)(pg / hw), vi = vb / c.batch, bi = vb - vi * c.batch;
    const int64_t pix = pg - (int64_t)vb * hw;
    const int py = (int)(pix / c.width), px = (int)(pix - (int64_t)py * c.width);
    const int v = c.views, ns = v - 1, D = c.depth_candidates;
    const int64_t Cp4 = Cp / 4;
    const int PW = (Cp + 31) / 32;
    const float4 *F4 = reinterpret_cast<const float4 *>(F);
    const float scale = (float)(1.0 / sqrt((double)c.channels) / (double)ns);
    for (int j0 = 0; j0 < Cp4; j0 += CV_PASS_CHUNKS) {
        float4 f01[CV_NCH], g01[CV_NCH];
#pragma unroll
        for (int k = 0; k < CV_NCH; k++) {
            const int j = j0 + lane + 32 * k;
            f01[k] = j < Cp4 ? F4[pg * Cp4 + j] : make_float4(0.f, 0.f, 0.f, 0.f);
            g01[k] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
        for (int d = 0; d < D; d++) {
            const double z = depth[(size_t)vb * D + d];
            const float gd = dcost[((int64_t)vb * D + d) * hw + pix] * scale;
            for (int s = 1; s <= ns; s++) {
                const CvCam cam = cams[(size_t)vb * ns + (s - 1)];
                const int vs = (vi + s) % v;
                Taps t;
                sample_taps(cam, (double)px, (double)py, z, c.height, c.width, ((int64_t)vs * c.batch + bi) * hw, t);
#pragma unroll
                for (int k = 0; k < CV_NCH; k++) {
                    const int j = j0 + lane + 32 * k;
                    if (j >= Cp4) continue;
                    g01[k] = fma4(gd, gather(F4, Cp4, j, t), g01[k]);
                    const float4 gs = make_float4(gd * f01[k].x, gd * f01[k].y, gd * f01[k].z, gd * f01[k].w);
#pragma unroll
                    for (int q = 0; q < 4; q++) {
                        if (t.row[q] < 0) continue;
                        const float wq = t.w[q];
                        const float4 term = make_float4(wq * gs.x, wq * gs.y, wq * gs.z, wq * gs.w);
                        if (term.x == 0.f && term.y == 0.f && term.z == 0.f && term.w == 0.f) continue;
                        if constexpr (DET) det_add4(limbs, poison, PW, t.row[q], Cp, j, term);
                        else red_add_v4(reinterpret_cast<float4 *>(acc) + t.row[q] * Cp4 + j, term);
                    }
                }
            }
        }
#pragma unroll
        for (int k = 0; k < CV_NCH; k++) {
            const int j = j0 + lane + 32 * k;
            if (j < Cp4) reinterpret_cast<float4 *>(G1)[pg * Cp4 + j] = g01[k];
        }
    }
}

// dL/dfeatures[b, v, c, h, w] = G1 + source accumulator (decoded in deterministic mode), transposed from the packed rows
template <bool DET>
__global__ void __launch_bounds__(CV_THREADS)
k_cv_finalize(GsCostVolumeConfig c, int Cp, const float *__restrict__ G1, const float *__restrict__ acc,
              const unsigned long long *__restrict__ limbs, const uint32_t *__restrict__ poison,
              float *__restrict__ out) {
    __shared__ float tile[32][33];
    const int hw = c.height * c.width, vb = blockIdx.z, vi = vb / c.batch, bi = vb - vi * c.batch;
    const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32, PW = (Cp + 31) / 32;
    for (int r = threadIdx.y; r < 32; r += blockDim.y) {  // r: pixel, threadIdx.x: channel
        const int p = p0 + r, ch = c0 + threadIdx.x;
        float val = 0.f;
        if (p < hw && ch < c.channels) {
            const int64_t e = ((int64_t)vb * hw + p) * Cp + ch;
            float src;
            if constexpr (DET) {
                const long long *l = reinterpret_cast<const long long *>(limbs) + e * GS_DET_LIMBS;
                src = gs_det_decode(l, (poison[((int64_t)vb * hw + p) * PW + ch / 32] >> (ch & 31)) & 1u);
            } else {
                src = acc[e];
            }
            val = G1[e] + src;
        }
        tile[threadIdx.x][r] = val;
    }
    __syncthreads();
    float *dst = out + ((int64_t)bi * c.views + vi) * c.channels * (int64_t)hw;
    for (int r = threadIdx.y; r < 32; r += blockDim.y) {  // r: channel, threadIdx.x: pixel
        const int ch = c0 + r, p = p0 + threadIdx.x;
        if (ch < c.channels && p < hw) dst[(int64_t)ch * hw + p] = tile[r][threadIdx.x];
    }
}

int padded_channels(const GsCostVolumeConfig *c) { return (c->channels + 3) & ~3; }

int check_config(const GsCostVolumeConfig *c, const char *who) {
    if (!c) return gs_set_error(GS_ERR_INVALID, "cost volume: null config");
    const int64_t nv = (int64_t)c->batch * c->views, hw = (int64_t)c->height * c->width;
    const bool det = (c->flags & GS_COSTVOLUME_DETERMINISTIC) != 0;
    if (c->batch < 1 || c->views < 2 || c->channels < 1 || c->height < 2 || c->width < 2 || c->depth_candidates < 1 ||
        (c->intrinsics_rows != 3 && c->intrinsics_rows != 4) || (c->flags & ~(uint32_t)GS_COSTVOLUME_DETERMINISTIC) ||
        nv > 65535 || hw > INT32_MAX || nv * hw > INT32_MAX || (int64_t)c->channels + 3 > 65535 * 32 ||
        nv * hw * c->depth_candidates > INT32_MAX ||
        (det && (int64_t)(c->views - 1) * c->depth_candidates * hw >= GS_DET_MAX_TERMS))
        return gs_set_error(GS_ERR_INVALID, who);
    return GS_OK;
}

int check_inputs(const GsCostVolumeInputs *in, const char *who) {
    if (!in || !in->features || !in->intrinsics || !in->extrinsics || !in->near_ || !in->far_)
        return gs_set_error(GS_ERR_INVALID, who);
    return GS_OK;
}

size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

struct Scratch {
    float *F, *G1, *acc;
    CvCam *cams;
    double *depth;
    unsigned long long *limbs;
    uint32_t *poison;
};

int64_t scratch_layout(const GsCostVolumeConfig *c, bool backward, char *base, Scratch *sc) {
    const int64_t rows = (int64_t)c->batch * c->views * c->height * c->width, Cp = padded_channels(c);
    const bool det = (c->flags & GS_COSTVOLUME_DETERMINISTIC) != 0;
    size_t off = 0;
    auto take = [&](size_t bytes) { char *p = base ? base + off : nullptr; off += align256(bytes); return p; };
    Scratch s{};
    s.F = (float *)take(sizeof(float) * rows * Cp);
    s.cams = (CvCam *)take(sizeof(CvCam) * c->batch * c->views * (c->views - 1));
    s.depth = (double *)take(sizeof(double) * c->batch * c->views * c->depth_candidates);
    if (backward) {
        s.G1 = (float *)take(sizeof(float) * rows * Cp);
        if (det) {
            s.limbs = (unsigned long long *)take(sizeof(unsigned long long) * GS_DET_LIMBS * rows * Cp);
            s.poison = (uint32_t *)take(sizeof(uint32_t) * rows * ((Cp + 31) / 32));
        } else {
            s.acc = (float *)take(sizeof(float) * rows * Cp);
        }
    }
    if (sc) *sc = s;
    return (int64_t)off;
}

// packing and camera math, shared by both directions
int prologue(const GsCostVolumeConfig *c, const GsCostVolumeInputs *in, const Scratch &s, cudaStream_t st) {
    const int Cp = padded_channels(c), nv = c->batch * c->views, hw = c->height * c->width;
    k_cv_pack<<<dim3((hw + 31) / 32, (Cp + 31) / 32, nv), dim3(32, 8), 0, st>>>(*c, Cp, in->features, s.F);
    GS_CUDA_OK(cudaGetLastError());
    const int ncam = nv * (c->views - 1);
    k_cv_cameras<<<(ncam + 127) / 128, 128, 0, st>>>(*c, in->intrinsics, in->extrinsics, in->near_, in->far_, s.cams,
                                                     s.depth);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}

unsigned pixel_blocks(const GsCostVolumeConfig *c) {
    const int64_t npix = (int64_t)c->batch * c->views * c->height * c->width;
    return (unsigned)((npix + CV_WARPS - 1) / CV_WARPS);
}

int check_scratch(void *scratch, const char *who) {
    if (!scratch) return gs_set_error(GS_ERR_INVALID, who);
    if (reinterpret_cast<uintptr_t>(scratch) & 255u) return gs_set_error(GS_ERR_INVALID, who);
    return GS_OK;
}

}  // namespace

extern "C" GS_API int64_t gs_costvolume_scratch_bytes(const GsCostVolumeConfig *cfg, int32_t backward) {
    if (check_config(cfg, "bad GsCostVolumeConfig")) return -1;
    return scratch_layout(cfg, backward != 0, nullptr, nullptr);
}

extern "C" GS_API int gs_costvolume_forward(const GsCostVolumeConfig *cfg, const GsCostVolumeInputs *in, float *out_cost,
                                            void *scratch, void *stream) {
    if (int rc = check_config(cfg, "bad GsCostVolumeConfig for gs_costvolume_forward")) return rc;
    if (check_inputs(in, "gs_costvolume_forward: null input pointer")) return GS_ERR_INVALID;
    if (!out_cost) return gs_set_error(GS_ERR_INVALID, "gs_costvolume_forward: null output pointer");
    if (check_scratch(scratch, "gs_costvolume_forward: scratch must be non-null and 256-byte aligned")) return GS_ERR_INVALID;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    Scratch s;
    scratch_layout(cfg, false, static_cast<char *>(scratch), &s);
    if (int rc = prologue(cfg, in, s, st)) return rc;
    k_cv_forward<<<pixel_blocks(cfg), CV_THREADS, 0, st>>>(*cfg, padded_channels(cfg), s.F, s.cams, s.depth, out_cost);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}

extern "C" GS_API int gs_costvolume_backward(const GsCostVolumeConfig *cfg, const GsCostVolumeInputs *in,
                                             const GsCostVolumeGrads *grads, void *scratch, void *stream) {
    if (int rc = check_config(cfg, "bad GsCostVolumeConfig for gs_costvolume_backward")) return rc;
    if (check_inputs(in, "gs_costvolume_backward: null input pointer")) return GS_ERR_INVALID;
    if (!grads || !grads->dL_dcost || !grads->dL_dfeatures)
        return gs_set_error(GS_ERR_INVALID, "gs_costvolume_backward: null gradient pointer");
    if (check_scratch(scratch, "gs_costvolume_backward: scratch must be non-null and 256-byte aligned")) return GS_ERR_INVALID;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const bool det = (cfg->flags & GS_COSTVOLUME_DETERMINISTIC) != 0;
    const int Cp = padded_channels(cfg), nv = cfg->batch * cfg->views, hw = cfg->height * cfg->width;
    const int64_t rows = (int64_t)nv * hw;
    Scratch s;
    scratch_layout(cfg, true, static_cast<char *>(scratch), &s);
    if (det) {
        GS_CUDA_OK(cudaMemsetAsync(s.limbs, 0, sizeof(unsigned long long) * GS_DET_LIMBS * rows * Cp, st));
        GS_CUDA_OK(cudaMemsetAsync(s.poison, 0, sizeof(uint32_t) * rows * ((Cp + 31) / 32), st));
    } else {
        GS_CUDA_OK(cudaMemsetAsync(s.acc, 0, sizeof(float) * rows * Cp, st));
    }
    if (int rc = prologue(cfg, in, s, st)) return rc;
    const dim3 tiles((hw + 31) / 32, (cfg->channels + 31) / 32, nv), tile_threads(32, 8);
    if (det) {
        k_cv_backward<true><<<pixel_blocks(cfg), CV_THREADS, 0, st>>>(*cfg, Cp, s.F, s.cams, s.depth, grads->dL_dcost,
                                                                      s.G1, nullptr, s.limbs, s.poison);
        GS_CUDA_OK(cudaGetLastError());
        k_cv_finalize<true><<<tiles, tile_threads, 0, st>>>(*cfg, Cp, s.G1, nullptr, s.limbs, s.poison,
                                                            grads->dL_dfeatures);
    } else {
        k_cv_backward<false><<<pixel_blocks(cfg), CV_THREADS, 0, st>>>(*cfg, Cp, s.F, s.cams, s.depth, grads->dL_dcost,
                                                                       s.G1, s.acc, nullptr, nullptr);
        GS_CUDA_OK(cudaGetLastError());
        k_cv_finalize<false><<<tiles, tile_threads, 0, st>>>(*cfg, Cp, s.G1, s.acc, nullptr, nullptr,
                                                             grads->dL_dfeatures);
    }
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}
