// gs_adapter_math.cuh -- the per-Gaussian arithmetic of PF3plat's GaussianAdapter.forward
// (src/model/encoder/common/gaussian_adapter.py:60-92), shared by the fused adapter (gs_adapter.cu) and the Gaussian
// head (gs_gaussian_head.cu): the per-camera header a CTA keeps in shared memory, the geometry of one Gaussian
// (direction, scales, quaternion), the covariance factor, and the block-diagonal SH rotation of one Gaussian's
// coefficients, forward and backward.  Everything is float32.
#pragma once

namespace {

constexpr int AD_THREADS = 128;
constexpr int AD_MAX_DSH = 25;
constexpr float AD_QUAT_EPS = 1e-8f;  // quaternion_to_matrix's own eps (PF3plat's src/model/encoder/common/gaussians.py:10)

// one camera: K^-1, the c2w rotation C and translation t, the scale multiplier, the SH mask, and room for a CTA's
// per-warp partial sums
struct AdHdr {
    float kinv[9], rot[9], t[3], mult;
    float mask[AD_MAX_DSH];
    float red[AD_THREADS / 32][24];
    uint64_t bar;
};
constexpr int AD_HDR_BYTES = (sizeof(AdHdr) + 127) / 128 * 128;

// The geometry part of one Gaussian (everything but the harmonics); kept by the backward for its chain rule.
struct AdGeom {
    float dc[3], inv_n;   // camera-space unit direction, 1 / |Kinv (x,y,1)|
    float dw[3];          // world-space direction
    float sg[3], s0[3], s[3];
    float q[4], nq, A;    // normalised quaternion (i,j,k,r), |raw quaternion|, two_s
    float Rq[9];
};

__device__ __forceinline__ void adapter_geometry(const AdHdr &h, float x, float y, float z, const float *sraw, const float *qraw,
                                                 float smin, float smax, float eps, AdGeom &g) {
    float u[3];
#pragma unroll
    for (int i = 0; i < 3; i++) u[i] = h.kinv[i * 3] * x + h.kinv[i * 3 + 1] * y + h.kinv[i * 3 + 2];
    g.inv_n = 1.0f / sqrtf(u[0] * u[0] + u[1] * u[1] + u[2] * u[2]);
#pragma unroll
    for (int i = 0; i < 3; i++) g.dc[i] = u[i] * g.inv_n;
#pragma unroll
    for (int i = 0; i < 3; i++) g.dw[i] = h.rot[i * 3] * g.dc[0] + h.rot[i * 3 + 1] * g.dc[1] + h.rot[i * 3 + 2] * g.dc[2];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        g.sg[k] = 1.0f / (1.0f + expf(-sraw[k]));
        g.s0[k] = smin + (smax - smin) * g.sg[k];
        g.s[k] = g.s0[k] * z * h.mult;
    }
    g.nq = sqrtf(qraw[0] * qraw[0] + qraw[1] * qraw[1] + qraw[2] * qraw[2] + qraw[3] * qraw[3]);
    const float inv = 1.0f / (g.nq + eps);
#pragma unroll
    for (int k = 0; k < 4; k++) g.q[k] = qraw[k] * inv;
    const float i = g.q[0], j = g.q[1], k = g.q[2], r = g.q[3];
    g.A = 2.0f / (i * i + j * j + k * k + r * r + AD_QUAT_EPS);
    const float A = g.A;
    g.Rq[0] = 1.0f - A * (j * j + k * k); g.Rq[1] = A * (i * j - k * r);        g.Rq[2] = A * (i * k + j * r);
    g.Rq[3] = A * (i * j + k * r);        g.Rq[4] = 1.0f - A * (i * i + k * k); g.Rq[5] = A * (j * k - i * r);
    g.Rq[6] = A * (i * k - j * r);        g.Rq[7] = A * (j * k + i * r);        g.Rq[8] = 1.0f - A * (i * i + j * j);
}

// N = C Rq diag(s): the world-space covariance is N N^T
__device__ __forceinline__ void adapter_factor(const AdHdr &h, const AdGeom &g, float *N) {
    float M[9];
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int k = 0; k < 3; k++) M[i * 3 + k] = g.Rq[i * 3 + k] * g.s[k];
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int k = 0; k < 3; k++)
            N[i * 3 + k] = h.rot[i * 3] * M[k] + h.rot[i * 3 + 1] * M[3 + k] + h.rot[i * 3 + 2] * M[6 + k];
}

__device__ __forceinline__ int isqrt_small(int n) {
    int r = 0;
    while ((r + 1) * (r + 1) <= n) r++;
    return r;
}

}  // namespace

// The SH rotation of one Gaussian's coefficients, gaussian_adapter.py:76-77 and :92, forward and backward.  These are
// macros, not device functions: NVVM simplifies a callee before inlining it, so moving these loops into a function
// changes the instruction schedule of the adapter kernels that have always run them inline; as macros, the adapter's
// kernels compile to the same SASS as before and the Gaussian head runs the same text.
//
// GS_SH_ROTATE_FWD: out[d][c] = sum_j D[d][j] sh[c][j] mask[j], D the camera's block-diagonal Wigner-D [d_sh][d_sh]
// (row-major), sh the raw coefficients in (xyz, d_sh) order, out in the rasterizer's (d_sh, xyz) order.
#define GS_SH_ROTATE_FWD(D, d_sh, mask, sh, out)                                    \
    do {                                                                            \
        const int degs_ = isqrt_small(d_sh);                                        \
        for (int l = 0; l < degs_; l++) {                                           \
            const int b = l * l, w = 2 * l + 1;                                     \
            for (int i = 0; i < w; i++) {                                           \
                float acc0 = 0.f, acc1 = 0.f, acc2 = 0.f;                           \
                for (int j = 0; j < w; j++) {                                       \
                    const float d = D[(b + i) * d_sh + b + j] * mask[b + j];        \
                    acc0 = fmaf(d, sh[b + j], acc0);                                \
                    acc1 = fmaf(d, sh[d_sh + b + j], acc1);                         \
                    acc2 = fmaf(d, sh[2 * d_sh + b + j], acc2);                     \
                }                                                                   \
                out[(b + i) * 3] = acc0;                                            \
                out[(b + i) * 3 + 1] = acc1;                                        \
                out[(b + i) * 3 + 2] = acc2;                                        \
            }                                                                       \
        }                                                                           \
    } while (0)

// the same with D the identity (the reference's rotation guard failed, or no rotation was supplied)
#define GS_SH_MASK_FWD(d_sh, mask, sh, out)                                         \
    do {                                                                            \
        for (int d = 0; d < d_sh; d++) {                                            \
            const float m = mask[d];                                                \
            out[d * 3] = sh[d] * m;                                                 \
            out[d * 3 + 1] = sh[d_sh + d] * m;                                      \
            out[d * 3 + 2] = sh[2 * d_sh + d] * m;                                  \
        }                                                                           \
    } while (0)

// GS_SH_ROTATE_BWD: dsh[c][j] = mask[j] sum_i D[i][j] gh[i][c], gh the cotangent in (d_sh, xyz) order.  dsh is a float
// pointer or anything whose operator[] yields a float lvalue (the Gaussian head writes channel planes).
#define GS_SH_ROTATE_BWD(D, d_sh, mask, gh, dsh)                                    \
    do {                                                                            \
        const int degs_ = isqrt_small(d_sh);                                        \
        for (int l = 0; l < degs_; l++) {                                           \
            const int b = l * l, w = 2 * l + 1;                                     \
            for (int j = 0; j < w; j++) {                                           \
                float acc0 = 0.f, acc1 = 0.f, acc2 = 0.f;                           \
                for (int i = 0; i < w; i++) {                                       \
                    const float d = D[(b + i) * d_sh + b + j];                      \
                    acc0 = fmaf(d, gh[(b + i) * 3], acc0);                          \
                    acc1 = fmaf(d, gh[(b + i) * 3 + 1], acc1);                      \
                    acc2 = fmaf(d, gh[(b + i) * 3 + 2], acc2);                      \
                }                                                                   \
                const float m = mask[b + j];                                        \
                dsh[b + j] = acc0 * m;                                              \
                dsh[d_sh + b + j] = acc1 * m;                                       \
                dsh[2 * d_sh + b + j] = acc2 * m;                                   \
            }                                                                       \
        }                                                                           \
    } while (0)

#define GS_SH_MASK_BWD(d_sh, mask, gh, dsh)                                         \
    do {                                                                            \
        for (int d = 0; d < d_sh; d++) {                                            \
            const float m = mask[d];                                                \
            dsh[d] = gh[d * 3] * m;                                                 \
            dsh[d_sh + d] = gh[d * 3 + 1] * m;                                      \
            dsh[2 * d_sh + d] = gh[d * 3 + 2] * m;                                  \
        }                                                                           \
    } while (0)
