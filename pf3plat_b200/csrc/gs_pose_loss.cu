// gs_pose_loss.cu -- PF3plat's correspondence (pose) loss on the device: Losspose.forward of src/loss/loss_pose.py,
// forward and backward.
//
// Semantics (per segment s = (scene i, pair (a, c)), pairs [(a, c) for a < c] in the reference's order, :47):
//   T_s = c2w[1][i, c] (a == 0) or c2w[1][i, c] @ inverse(c2w[1][i, a]) (get_relative_Rt, :141-156); built by the caller.
//   For match n, p = id_a[n], q = id_c[n]:
//     x(p) = ((p mod w) + 0.5) / w, y(p) = ((p div w) + 0.5) / h           (sample_image_grid, projection.py:117-137)
//     r = K_a^-1 [x, y, 1],  X = d_a(p) r,  Q = T_s [X, 1],  P = Q_xyz / (Q_w + 1e-6),  u = K_c P,
//     pi = u_xy / (u_z + 1e-6)                              (batch_project_to_other_img and from_homogeneous, flow_util.py:187-225)
//     h2 = huber_0.01(|pi - (x(q), y(q))|) / 0.01                                                    (loss_pose.py:92)
//     e3 = |R_s xyz_a(p) + t_s - xyz_c(q)|                                             (transform_points_Rt, :110, :116)
//   L3_s = conf_s sum_n (w_n / max(sum |w|, 1e-12)) e3_n    (F.normalize(p=1), :81, :119, :123)
//   L2_s = sum_n h2_n                                       (:96)
// The caller forms weight_3d mean_s L3_s + weight_2d mean_s L2_s (:128-129).
//
// Forward: k_pose_loss_fwd, one CTA per segment, threads striding over its matches; only matched pixels are projected
// (the reference projects all h w pixels of every pair and gathers).  Per-thread fp64 sums, reduced in a fixed order.
//
// Backward: k_pose_loss_bwd_match (one CTA per segment) recomputes sum |w| and sum w e3, then per match the exact
// derivatives of the chain above, mirroring PyTorch's rules (the norm's gradient at 0 is 0; Huber is linear at exactly
// delta; clamp_min passes at equality).  dL/dT [S,16] and dL/dconf [S] are reduced in a fixed order, dL/dw is per match.
// The depth / xyz terms of match n go to two entries, keyed (scene, view, pixel): (i, a, p) with dL/dxyz_a and dL/dd,
// and (i, c, q) with dL/dxyz_c.  A stable radix sort of the keys (entry index breaks ties, so the order is the
// entries') and k_pose_loss_dense, which walks each pixel's run in sorted order, give a deterministic scatter with no
// atomics: every element of dL/ddepth and dL/dxyz is written once.
//
// The reference's dense projection makes one gradient non-finite that a gathered one would not: the zero gradient
// that reaches an unmatched pixel is multiplied through the pixel's projection (0 x NaN = NaN), so a non-finite depth
// at a pixel no match reads poisons dL/dd there and dL/dT_s of every pair it is a source of.  k_pose_loss_dense
// evaluates that projection at every source pixel and writes NaN wherever the reference's zero-gradient backward
// would turn non-finite (pose_loss_poisoned).  A match index outside [0, h w) is never dereferenced: its segment's
// L3, L2 and every gradient term it writes become NaN.
#include "gs_common.cuh"

#include <cub/cub.cuh>

namespace {

constexpr int PO_THREADS = 256, PO_WARPS = PO_THREADS / 32;
constexpr float PO_DELTA = 0.01f, PO_EPS_H = 1e-6f, PO_EPS_N = 1e-12f;
constexpr int PO_NRED = 18;  // dL/dT (16), dL/dconf, bad-segment flag

struct Seg {
    float T[16], ki[9], kc[9], conf;
    int scene, a, c;
};

__device__ __forceinline__ void load_seg(Seg &g, int s, const float *__restrict__ T, const float *__restrict__ kinv,
                                         const float *__restrict__ kc, const float *__restrict__ conf,
                                         const int32_t *__restrict__ seg) {
#pragma unroll
    for (int k = 0; k < 16; k++) g.T[k] = T[(size_t)s * 16 + k];
#pragma unroll
    for (int k = 0; k < 9; k++) {
        g.ki[k] = kinv[(size_t)s * 9 + k];
        g.kc[k] = kc[(size_t)s * 9 + k];
    }
    g.conf = conf ? conf[s] : 0.f;
    g.scene = seg[3 * s];
    g.a = seg[3 * s + 1];
    g.c = seg[3 * s + 2];
}

// the pixel-centre coordinates sample_image_grid builds, in float32
__device__ __forceinline__ void grid_xy(int64_t p, int h, int w, float &x, float &y) {
    x = ((float)(p % w) + 0.5f) / (float)w;
    y = ((float)(p / w) + 0.5f) / (float)h;
}

// The projection of pixel (x, y) at depth d into the other view; the intermediates the backward needs.
struct Proj {
    float r[3], X[3], den1, P[3], u[3], den2, pi[2];
};

__device__ __forceinline__ void project(const Seg &g, float x, float y, float d, Proj &o) {
#pragma unroll
    for (int i = 0; i < 3; i++) {
        o.r[i] = g.ki[3 * i] * x + g.ki[3 * i + 1] * y + g.ki[3 * i + 2];
        o.X[i] = o.r[i] * d;
    }
    float Q[4];
#pragma unroll
    for (int i = 0; i < 4; i++) Q[i] = g.T[4 * i] * o.X[0] + g.T[4 * i + 1] * o.X[1] + g.T[4 * i + 2] * o.X[2] + g.T[4 * i + 3];
    o.den1 = Q[3] + PO_EPS_H;
#pragma unroll
    for (int i = 0; i < 3; i++) o.P[i] = Q[i] / o.den1;
#pragma unroll
    for (int i = 0; i < 3; i++) o.u[i] = g.kc[3 * i] * o.P[0] + g.kc[3 * i + 1] * o.P[1] + g.kc[3 * i + 2] * o.P[2];
    o.den2 = o.u[2] + PO_EPS_H;
    o.pi[0] = o.u[0] / o.den2;
    o.pi[1] = o.u[1] / o.den2;
}

// Whether the reference's backward of this projection, fed a gradient of exactly zero, yields a non-finite value: the
// divisions' backward multiplies it by 1/den and by (num/den)/den, the matmuls' by T, K_c, [X, 1] and r.
__device__ __forceinline__ bool pose_loss_poisoned(const Seg &g, const Proj &o) {
    bool ok = o.den1 != 0.f && o.den2 != 0.f && isfinite(o.den1) && isfinite(o.den2);
#pragma unroll
    for (int i = 0; i < 3; i++) ok = ok && isfinite(o.r[i]) && isfinite(o.X[i]) && isfinite(o.P[i] / o.den1);
    ok = ok && isfinite(o.pi[0] / o.den2) && isfinite(o.pi[1] / o.den2);
#pragma unroll
    for (int k = 0; k < 16; k++) ok = ok && isfinite(g.T[k]);
#pragma unroll
    for (int k = 0; k < 9; k++) ok = ok && isfinite(g.kc[k]);
    return !ok;
}

__device__ __forceinline__ float huber_over_delta(float e) {  // F.huber_loss(e, 0, delta=0.01) / 0.01
    const float hb = e < PO_DELTA ? 0.5f * e * e : PO_DELTA * (e - 0.5f * PO_DELTA);
    return hb / PO_DELTA;
}

// the residual vector R xyz_a + t - xyz_c (transform_points_Rt with inverse=False)
__device__ __forceinline__ void residual3(const Seg &g, const float xa[3], const float xc[3], float v[3]) {
#pragma unroll
    for (int k = 0; k < 3; k++) v[k] = g.T[4 * k] * xa[0] + g.T[4 * k + 1] * xa[1] + g.T[4 * k + 2] * xa[2] + g.T[4 * k + 3] - xc[k];
}

struct Match {
    float xa[3], xc[3], d, wq[2];  // xyz_a(p), xyz_c(q), d_a(p), (x(q), y(q))
    float x, y;                    // (x(p), y(p))
};

__device__ __forceinline__ void load_match(const Seg &g, int64_t p, int64_t q, int v, int h, int w,
                                           const float *__restrict__ depth, const float *__restrict__ xyz, Match &m) {
    const int64_t hw = (int64_t)h * w;
    const size_t ia = (size_t)g.scene * v + g.a, ic = (size_t)g.scene * v + g.c;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        m.xa[k] = xyz[(ia * 3 + k) * hw + p];
        m.xc[k] = xyz[(ic * 3 + k) * hw + q];
    }
    m.d = depth[ia * hw + p];
    grid_xy(p, h, w, m.x, m.y);
    grid_xy(q, h, w, m.wq[0], m.wq[1]);
}

// warp butterfly, then one slot per warp; thread k < n sums slot k over the warps in order.  Fixed order.
template <int N>
__device__ __forceinline__ void block_sums(double (&v)[N], double (*red)[PO_WARPS]) {
#pragma unroll
    for (int k = 0; k < N; k++) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
    }
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int k = 0; k < N; k++) red[k][threadIdx.x >> 5] = v[k];
    }
    __syncthreads();
    if (threadIdx.x < N) {
        double t = 0.0;
#pragma unroll
        for (int wp = 0; wp < PO_WARPS; wp++) t += red[threadIdx.x][wp];
        red[threadIdx.x][0] = t;
    }
    __syncthreads();
}

__device__ __forceinline__ bool index_ok(int64_t p, int64_t hw) { return p >= 0 && p < hw; }

// the normaliser max(sum |w|, 1e-12) as clamp_min computes it: a NaN sum stays NaN (fmax would return the bound)
__device__ __forceinline__ double clamp_norm(double s) { return s < (double)PO_EPS_N ? (double)PO_EPS_N : s; }

// per segment: sum_n w_n e3_n, sum_n |w_n|, sum_n h2_n, and whether an index is out of range
__device__ __forceinline__ void segment_sums(const Seg &g, int64_t beg, int64_t end, const int64_t *__restrict__ id_a,
                                             const int64_t *__restrict__ id_c, const float *__restrict__ wts, int v, int h,
                                             int w, const float *__restrict__ depth, const float *__restrict__ xyz,
                                             bool with_2d, double (*red)[PO_WARPS]) {
    const int64_t hw = (int64_t)h * w;
    double acc[4] = {0.0, 0.0, 0.0, 0.0};
    for (int64_t n = beg + threadIdx.x; n < end; n += PO_THREADS) {
        const int64_t p = id_a[n], q = id_c[n];
        if (!index_ok(p, hw) || !index_ok(q, hw)) {
            acc[3] = 1.0;
            continue;
        }
        Match m;
        load_match(g, p, q, v, h, w, depth, xyz, m);
        float r3[3];
        residual3(g, m.xa, m.xc, r3);
        const float e3 = sqrtf(r3[0] * r3[0] + r3[1] * r3[1] + r3[2] * r3[2]);
        const float wn = wts[n];
        acc[0] += (double)wn * (double)e3;
        acc[1] += (double)fabsf(wn);
        if (with_2d) {
            Proj o;
            project(g, m.x, m.y, m.d, o);
            const float dx = o.pi[0] - m.wq[0], dy = o.pi[1] - m.wq[1];
            acc[2] += (double)huber_over_delta(sqrtf(dx * dx + dy * dy));
        }
    }
    block_sums<4>(acc, red);
}

__global__ void __launch_bounds__(PO_THREADS)
k_pose_loss_fwd(int v, int h, int w, const float *__restrict__ T, const float *__restrict__ kinv,
                const float *__restrict__ kc, const float *__restrict__ conf, const int32_t *__restrict__ seg,
                const int64_t *__restrict__ offsets, const int64_t *__restrict__ id_a, const int64_t *__restrict__ id_c,
                const float *__restrict__ wts, const float *__restrict__ depth, const float *__restrict__ xyz,
                float *__restrict__ L3, float *__restrict__ L2) {
    __shared__ double red[PO_NRED][PO_WARPS];
    const int s = blockIdx.x;
    Seg g;
    load_seg(g, s, T, kinv, kc, conf, seg);
    segment_sums(g, offsets[s], offsets[s + 1], id_a, id_c, wts, v, h, w, depth, xyz, true, red);
    if (threadIdx.x == 0) {
        const bool bad = red[3][0] != 0.0;
        const double D = clamp_norm(red[1][0]);
        L3[s] = bad ? __int_as_float(0x7fffffff) : (float)((double)g.conf * (red[0][0] / D));
        L2[s] = bad ? __int_as_float(0x7fffffff) : (float)red[2][0];
    }
}

__global__ void __launch_bounds__(PO_THREADS)
k_pose_loss_bwd_match(int v, int h, int w, const float *__restrict__ T, const float *__restrict__ kinv,
                      const float *__restrict__ kc, const float *__restrict__ conf, const int32_t *__restrict__ seg,
                      const int64_t *__restrict__ offsets, const int64_t *__restrict__ id_a,
                      const int64_t *__restrict__ id_c, const float *__restrict__ wts, const float *__restrict__ depth,
                      const float *__restrict__ xyz, const float *__restrict__ dL_dL3, const float *__restrict__ dL_dL2,
                      float *__restrict__ dT, float *__restrict__ dconf, float *__restrict__ dw,
                      uint64_t *__restrict__ keys, int32_t *__restrict__ vals, float4 *__restrict__ contrib,
                      uint64_t key_end) {
    __shared__ double red[PO_NRED][PO_WARPS];
    const int s = blockIdx.x;
    const int64_t hw = (int64_t)h * w, beg = offsets[s], end = offsets[s + 1];
    Seg g;
    load_seg(g, s, T, kinv, kc, conf, seg);
    // pass 1: the segment's normaliser and weighted sum (the 2-D sum is not needed)
    segment_sums(g, beg, end, id_a, id_c, wts, v, h, w, depth, xyz, false, red);
    const double S_we = red[0][0], S_abs = red[1][0];
    const bool bad = red[3][0] != 0.0;
    __syncthreads();  // red is reused below
    const float nanf_ = __int_as_float(0x7fffffff);
    const float g3 = dL_dL3 ? dL_dL3[s] : 0.f, g2 = dL_dL2 ? dL_dL2[s] : 0.f;
    const float D = (float)clamp_norm(S_abs);
    const float c3 = g3 * g.conf;                                    // dL/d(sum_n wn_n e3_n)
    const float dD = S_abs >= (double)PO_EPS_N ? (float)(-(double)c3 * S_we / ((double)D * D)) : 0.f;  // via |w|
    double acc[PO_NRED];
#pragma unroll
    for (int k = 0; k < PO_NRED; k++) acc[k] = 0.0;
    for (int64_t n = beg + threadIdx.x; n < end; n += PO_THREADS) {
        const int64_t p = id_a[n], q = id_c[n];
        const bool pok = index_ok(p, hw), qok = index_ok(q, hw);
        const float wn = wts[n];
        float ga[4] = {0.f, 0.f, 0.f, 0.f}, gc[3] = {0.f, 0.f, 0.f};
        if (pok && qok) {
            Match m;
            load_match(g, p, q, v, h, w, depth, xyz, m);
            float dTl[16];
            // 3-D term: e3 = |vv|, dL/de3 = c3 wn / D; the norm's gradient is 0 where it vanishes
            float vv[3];
            residual3(g, m.xa, m.xc, vv);
            const float e3 = sqrtf(vv[0] * vv[0] + vv[1] * vv[1] + vv[2] * vv[2]);
            const float ge3 = c3 * (wn / D);
            const float s3 = e3 == 0.f ? 0.f : ge3 / e3;
            float dv[3];
#pragma unroll
            for (int k = 0; k < 3; k++) {
                dv[k] = vv[k] * s3;
                dTl[4 * k] = dv[k] * m.xa[0];
                dTl[4 * k + 1] = dv[k] * m.xa[1];
                dTl[4 * k + 2] = dv[k] * m.xa[2];
                dTl[4 * k + 3] = dv[k];
                gc[k] = -dv[k];
            }
            dTl[12] = dTl[13] = dTl[14] = dTl[15] = 0.f;
#pragma unroll
            for (int j = 0; j < 3; j++) ga[j] = g.T[j] * dv[0] + g.T[4 + j] * dv[1] + g.T[8 + j] * dv[2];
            if (dw) dw[n] = bad ? nanf_ : c3 * (e3 / D) + (wn > 0.f ? dD : wn < 0.f ? -dD : 0.f * dD);
            // 2-D term
            Proj o;
            project(g, m.x, m.y, m.d, o);
            const float ex = o.pi[0] - m.wq[0], ey = o.pi[1] - m.wq[1];
            const float e2 = sqrtf(ex * ex + ey * ey);
            // huber_loss backward (x > delta -> delta, else x; NaN stays NaN), then the / 0.01
            const float ge2 = (g2 / PO_DELTA) * (e2 > PO_DELTA ? PO_DELTA : e2);
            const float s2 = e2 == 0.f ? 0.f : ge2 / e2;
            const float dpi0 = ex * s2, dpi1 = ey * s2;
            const float du[3] = {dpi0 / o.den2, dpi1 / o.den2,
                                 -(dpi0 * (o.pi[0] / o.den2) + dpi1 * (o.pi[1] / o.den2))};
            float dP[3], dQ[4];
#pragma unroll
            for (int j = 0; j < 3; j++) dP[j] = du[0] * g.kc[j] + du[1] * g.kc[3 + j] + du[2] * g.kc[6 + j];
#pragma unroll
            for (int j = 0; j < 3; j++) dQ[j] = dP[j] / o.den1;
            dQ[3] = -(dP[0] * (o.P[0] / o.den1) + dP[1] * (o.P[1] / o.den1) + dP[2] * (o.P[2] / o.den1));
            float dd = 0.f;
#pragma unroll
            for (int j = 0; j < 3; j++) {
                const float dX = dQ[0] * g.T[j] + dQ[1] * g.T[4 + j] + dQ[2] * g.T[8 + j] + dQ[3] * g.T[12 + j];
                dd += dX * o.r[j];
            }
            ga[3] = dd;
#pragma unroll
            for (int i = 0; i < 4; i++) {
                dTl[4 * i] += dQ[i] * o.X[0];
                dTl[4 * i + 1] += dQ[i] * o.X[1];
                dTl[4 * i + 2] += dQ[i] * o.X[2];
                dTl[4 * i + 3] += dQ[i];
            }
#pragma unroll
            for (int k = 0; k < 16; k++) acc[k] += (double)dTl[k];
            acc[16] += (double)wn * (double)e3;
        } else {
            acc[17] = 1.0;
            if (dw) dw[n] = nanf_;
        }
        if (keys) {
            const size_t e = 2 * (size_t)n;
            keys[e] = pok && qok ? ((uint64_t)g.scene * v + g.a) * hw + p : key_end;
            keys[e + 1] = pok && qok ? ((uint64_t)g.scene * v + g.c) * hw + q : key_end;
            vals[e] = (int32_t)e;
            vals[e + 1] = (int32_t)(e + 1);
            contrib[e] = bad ? make_float4(nanf_, nanf_, nanf_, nanf_) : make_float4(ga[0], ga[1], ga[2], ga[3]);
            contrib[e + 1] = bad ? make_float4(nanf_, nanf_, nanf_, 0.f) : make_float4(gc[0], gc[1], gc[2], 0.f);
        }
    }
    block_sums<PO_NRED>(acc, red);
    if (threadIdx.x < 16 && dT) dT[(size_t)s * 16 + threadIdx.x] = bad ? nanf_ : (float)red[threadIdx.x][0];
    if (threadIdx.x == 16 && dconf) dconf[s] = bad ? nanf_ : (float)((double)g3 * (red[16][0] / (double)D));
}

// first[key] = position of the key's first entry in sorted order (the sentinel key_end has no slot)
__global__ void k_pose_loss_run_heads(const uint64_t *__restrict__ skeys, int64_t n, uint64_t key_end,
                                      int32_t *__restrict__ first) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t k = skeys[i];
    if (k != key_end && (i == 0 || skeys[i - 1] != k)) first[k] = (int32_t)i;
}

// one thread per (scene, view, pixel): sum the pixel's entries in sorted order, then the dense projection's poison
__global__ void __launch_bounds__(PO_THREADS)
k_pose_loss_dense(int v, int h, int w, int pairs, int64_t total, const float *__restrict__ T,
                  const float *__restrict__ kinv, const float *__restrict__ kc, const int32_t *__restrict__ seg,
                  const float *__restrict__ depth, const uint64_t *__restrict__ skeys, const int32_t *__restrict__ svals,
                  const float4 *__restrict__ contrib, const int32_t *__restrict__ first, int64_t nkeys,
                  float *__restrict__ ddepth, float *__restrict__ dxyz, float *__restrict__ dT) {
    const int64_t e = (int64_t)blockIdx.x * PO_THREADS + threadIdx.x;
    if (e >= total) return;
    const int64_t hw = (int64_t)h * w, sv = e / hw, p = e - sv * hw;
    const int scene = (int)(sv / v), view = (int)(sv - (int64_t)scene * v);
    float gx = 0.f, gy = 0.f, gz = 0.f, gd = 0.f;
    if (first) {
        int64_t i = first[e];
        if (i >= 0) {
            for (; i < nkeys && skeys[i] == (uint64_t)e; i++) {
                const float4 t = contrib[svals[i]];
                gx += t.x;
                gy += t.y;
                gz += t.z;
                gd += t.w;
            }
        }
    }
    if (view < v - 1 && (ddepth || dT)) {  // a source view: the pairs (view, c > view)
        float x, y;
        grid_xy(p, h, w, x, y);
        const float d = depth[e];
        const int base = scene * pairs + view * v - view * (view + 1) / 2;
        for (int c = view + 1; c < v; c++) {
            const int s = base + (c - view - 1);
            Seg g;
            load_seg(g, s, T, kinv, kc, nullptr, seg);
            Proj o;
            project(g, x, y, d, o);
            if (pose_loss_poisoned(g, o)) {
                gd = __int_as_float(0x7fffffff);
                if (dT) {
#pragma unroll
                    for (int k = 0; k < 16; k++) dT[(size_t)s * 16 + k] = __int_as_float(0x7fffffff);
                }
            }
        }
    }
    if (ddepth) ddepth[e] = gd;
    if (dxyz) {
        float *o = dxyz + sv * 3 * hw + p;
        o[0] = gx;
        o[hw] = gy;
        o[2 * hw] = gz;
    }
}

int end_bit_of(uint64_t key_end) {
    int b = 1;
    while (b < 64 && (key_end >> b) != 0) b++;
    return b;
}

int check_config(const GsPoseLossConfig *cfg, const char *who) {
    if (!cfg) return gs_set_error(GS_ERR_INVALID, "pose loss: null config");
    const int64_t pairs = (int64_t)cfg->views * (cfg->views - 1) / 2;
    if (cfg->batch < 0 || cfg->views < 2 || cfg->height < 1 || cfg->width < 1 || cfg->matches < 0 ||
        cfg->segments != cfg->batch * pairs || (int64_t)cfg->height * cfg->width > INT32_MAX ||
        2 * cfg->matches > INT32_MAX || (int64_t)cfg->batch * cfg->views * cfg->height * cfg->width > INT32_MAX)
        return gs_set_error(GS_ERR_INVALID, who);
    return GS_OK;
}

struct Scratch {
    uint64_t *keys, *skeys;
    int32_t *vals, *svals, *first;
    float4 *contrib;
    void *cub;
    size_t cub_bytes;
};

size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

int64_t scratch_layout(const GsPoseLossConfig *cfg, char *base, Scratch *sc) {
    const int64_t n = 2 * cfg->matches, pix = (int64_t)cfg->batch * cfg->views * cfg->height * cfg->width;
    const uint64_t key_end = (uint64_t)pix;
    size_t cub_bytes = 0;
    if (cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, (const uint64_t *)nullptr, (uint64_t *)nullptr,
                                        (const int32_t *)nullptr, (int32_t *)nullptr, (int)n, 0,
                                        end_bit_of(key_end)) != cudaSuccess)
        return -1;
    size_t off = 0;
    auto take = [&](size_t bytes) { char *p = base ? base + off : nullptr; off += align256(bytes); return p; };
    Scratch s;
    s.keys = (uint64_t *)take(sizeof(uint64_t) * n);
    s.skeys = (uint64_t *)take(sizeof(uint64_t) * n);
    s.vals = (int32_t *)take(sizeof(int32_t) * n);
    s.svals = (int32_t *)take(sizeof(int32_t) * n);
    s.contrib = (float4 *)take(sizeof(float4) * n);
    s.first = (int32_t *)take(sizeof(int32_t) * pix);
    s.cub_bytes = cub_bytes;
    s.cub = take(cub_bytes);
    if (sc) *sc = s;
    return (int64_t)off;
}

int check_inputs(const GsPoseLossConfig *cfg, const GsPoseLossInputs *in, const char *who) {
    if (!in || !in->T || !in->kinv_a || !in->k_c || !in->conf || !in->seg || !in->offsets || !in->depth || !in->xyz ||
        (cfg->matches > 0 && (!in->id_a || !in->id_c || !in->w)))
        return gs_set_error(GS_ERR_INVALID, who);
    return GS_OK;
}

}  // namespace

extern "C" GS_API int64_t gs_pose_loss_scratch_bytes(const GsPoseLossConfig *cfg) {
    if (check_config(cfg, "bad GsPoseLossConfig") != GS_OK) return -1;
    return scratch_layout(cfg, nullptr, nullptr);
}

extern "C" GS_API int gs_pose_loss_forward(const GsPoseLossConfig *cfg, const GsPoseLossInputs *in, float *out_L3,
                                           float *out_L2, void *stream) {
    if (int rc = check_config(cfg, "bad GsPoseLossConfig for gs_pose_loss_forward")) return rc;
    if (check_inputs(cfg, in, "gs_pose_loss_forward: null input pointer")) return GS_ERR_INVALID;
    if (!out_L3 || !out_L2) return gs_set_error(GS_ERR_INVALID, "gs_pose_loss_forward: null output pointer");
    if (cfg->segments == 0) return GS_OK;
    k_pose_loss_fwd<<<cfg->segments, PO_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
        cfg->views, cfg->height, cfg->width, in->T, in->kinv_a, in->k_c, in->conf, in->seg, in->offsets, in->id_a,
        in->id_c, in->w, in->depth, in->xyz, out_L3, out_L2);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}

extern "C" GS_API int gs_pose_loss_backward(const GsPoseLossConfig *cfg, const GsPoseLossInputs *in,
                                            const float *dL_dL3, const float *dL_dL2, const GsPoseLossGrads *grads,
                                            void *scratch, void *stream) {
    if (int rc = check_config(cfg, "bad GsPoseLossConfig for gs_pose_loss_backward")) return rc;
    if (check_inputs(cfg, in, "gs_pose_loss_backward: null input pointer")) return GS_ERR_INVALID;
    if (!grads) return gs_set_error(GS_ERR_INVALID, "gs_pose_loss_backward: null gradient struct");
    const bool scatter = grads->dL_ddepth || grads->dL_dxyz;
    const bool any = scatter || grads->dL_dT || grads->dL_dw || grads->dL_dconf;
    if (cfg->segments == 0 || !any) return GS_OK;
    if (scatter && !scratch) return gs_set_error(GS_ERR_INVALID, "gs_pose_loss_backward: null scratch");
    if (reinterpret_cast<uintptr_t>(scratch) & 255u)
        return gs_set_error(GS_ERR_INVALID, "gs_pose_loss_backward: scratch must be 256-byte aligned");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int64_t n = 2 * cfg->matches, pix = (int64_t)cfg->batch * cfg->views * cfg->height * cfg->width;
    const uint64_t key_end = (uint64_t)pix;
    Scratch sc{};
    if (scatter && scratch_layout(cfg, static_cast<char *>(scratch), &sc) < 0)
        return gs_set_error(GS_ERR_CUDA, "gs_pose_loss_backward: sort sizing failed");
    k_pose_loss_bwd_match<<<cfg->segments, PO_THREADS, 0, st>>>(
        cfg->views, cfg->height, cfg->width, in->T, in->kinv_a, in->k_c, in->conf, in->seg, in->offsets, in->id_a,
        in->id_c, in->w, in->depth, in->xyz, dL_dL3, dL_dL2, grads->dL_dT, grads->dL_dconf, grads->dL_dw,
        scatter ? sc.keys : nullptr, sc.vals, sc.contrib, key_end);
    GS_CUDA_OK(cudaGetLastError());
    if (scatter && n > 0) {
        size_t bytes = sc.cub_bytes;
        GS_CUDA_OK(cub::DeviceRadixSort::SortPairs(sc.cub, bytes, sc.keys, sc.skeys, sc.vals, sc.svals, (int)n, 0,
                                                   end_bit_of(key_end), st));
        GS_CUDA_OK(cudaMemsetAsync(sc.first, 0xff, sizeof(int32_t) * pix, st));
        k_pose_loss_run_heads<<<(unsigned)((n + PO_THREADS - 1) / PO_THREADS), PO_THREADS, 0, st>>>(sc.skeys, n, key_end,
                                                                                                 sc.first);
        GS_CUDA_OK(cudaGetLastError());
    }
    if (scatter || grads->dL_dT) {
        const int pairs = cfg->views * (cfg->views - 1) / 2;
        k_pose_loss_dense<<<(unsigned)((pix + PO_THREADS - 1) / PO_THREADS), PO_THREADS, 0, st>>>(
            cfg->views, cfg->height, cfg->width, pairs, pix, in->T, in->kinv_a, in->k_c, in->seg, in->depth, sc.skeys,
            sc.svals, sc.contrib, scatter && n > 0 ? sc.first : nullptr, n, grads->dL_ddepth, grads->dL_dxyz,
            grads->dL_dT);
        GS_CUDA_OK(cudaGetLastError());
    }
    return GS_OK;
}
