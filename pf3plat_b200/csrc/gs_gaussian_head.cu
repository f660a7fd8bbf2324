// gs_gaussian_head.cu -- the Gaussian head between the depth predictor's two output convolutions and the decoder,
// DESIGN.md 5.16: depth_predictor_multiview.py:397-415 (the rearrange of to_gaussians' output, the sigmoid of
// to_disparity's density channel), encoder_costvolume.py:509-540 (the pixel grid and its learned offset, the opacity
// map, the [:, (0, -1)] selections, the adapter) and :556-573 (the b (v r srf spp) rearrange of every output), for
// gaussians_per_pixel = num_surfaces = 1, in one launch forward and two backward.
//
// Per pixel p = (i, j) of slot s in {0, 1} (context view 0 or V - 1) of scene b, with raw = to_gaussians' channels there:
//   x = fl(fl((i + 1/2) / w) + fl(fl(sigmoid(raw[0]) - 1/2) fl(1/w))), y likewise with j, h and raw[1]   [:509-518]
//   means, covariances, harmonics = the adapter at (x, y) with depth z, raw[2:] (gs_adapter_math.cuh)   [:529-540]
//   opacities = 0.5 (fl(1 - fl(1 - q)) + q), q = sigmoid(density_logits[1])                            [:174-187]
// written at Gaussian index s h w + p of scene b.  K^-1 and the scale multiplier 0.1 sum(K[:2,:2]^-1 (1/w, 1/h)) are
// computed per camera in fp64 from the float32 K.  The SH rotation blocks come from the caller (tensor code, no host
// synchronisation), NULL = identity.
//
// Forward: one thread per (slot, scene, pixel), 128 per CTA, one camera per blockIdx.y.  The 9 + 3 d_sh channel planes
// are read coalesced into per-thread rows in shared memory (odd stride: no bank conflicts); means, covariance and
// harmonics rows are assembled in shared memory and leave by bulk TMA stores (coalesced loops where a block is not
// 16-byte aligned) straight into the b-major outputs.  Backward: the cotangent rows come in the same way, dL/draw and
// dL/dlogits leave as coalesced planes, dL/ddepths per pixel; the 12 per-camera dL/dc2w sums (through the means: the
// rotation is detached in covariance and harmonics) are written per CTA and added in CTA order by k_head_finalize,
// which also zeroes the depth gradient of the middle views.  No float atomics: bit-reproducible.
#include "gs_common.cuh"
#include "gs_adapter_math.cuh"
#include "gs_inverse.cuh"

namespace {

constexpr int HD_CAM_SUMS = 12;  // per-camera sums of the backward: dC 9 (row-major) | dt 3
constexpr int HD_FIN_THREADS = 256;

struct HeadArgs {
    int b, V, H, W, hw, d_sh, C, CS;  // C = 9 + 3 d_sh channels, CS = C | 1: the shared-memory row stride
    float smin, smax, eps, inv_w, inv_h;
    const float *raw, *logits, *depths, *c2w, *K, *sh_rot, *sh_mask;
};
struct HeadOut {
    float *means, *cov, *harm, *opac;
};
struct HeadOutGrads {
    const float *means, *cov, *harm, *opac;
};
struct HeadInGrads {
    float *raw, *logits, *depths, *c2w, *cam_partial;
};

// one channel of one item, indexed by channel offset: the backward's dL/draw planes seen as a row
struct Plane {
    float *p;
    size_t stride;
    __device__ __forceinline__ float &operator[](int k) const { return p[(size_t)k * stride]; }
};

// the camera of slot s of scene bi: view 0 or V - 1
__device__ __forceinline__ size_t head_view(const HeadArgs &a, int bi, int s) {
    return (size_t)bi * a.V + (s ? a.V - 1 : 0);
}

__device__ __forceinline__ void load_head_camera(const HeadArgs &a, size_t ci, AdHdr *h) {
    const int tid = threadIdx.x;
    if (tid < 9) {
        h->rot[tid] = a.c2w[ci * 16 + (tid / 3) * 4 + tid % 3];
    } else if (tid < 12) {
        h->t[tid - 9] = a.c2w[ci * 16 + (tid - 9) * 4 + 3];
    } else if (tid == 32) {
        double k[9], ki[9];
        for (int i = 0; i < 9; i++) k[i] = a.K[ci * 9 + i];
        inverse3(k, ki);
        for (int i = 0; i < 9; i++) h->kinv[i] = (float)ki[i];
        // get_scale_multiplier (gaussian_adapter.py:100-111): 0.1 sum_ij (K[:2,:2]^-1)_ij pixel_size_j
        const double det = k[0] * k[4] - k[1] * k[3];
        h->mult = (float)(0.1 * ((k[4] - k[3]) * (double)a.inv_w + (k[0] - k[1]) * (double)a.inv_h) / det);
    }
    if (tid >= 64 && tid < 64 + a.d_sh) h->mask[tid - 64] = a.sh_mask[tid - 64];
}

// encoder_costvolume.py:509-518: the pixel centre plus the learned offset, in the reference's float32 rounding
__device__ __forceinline__ float pixel_coord(int i, int len, float inv_len, float sg) {
    const float c = __fdiv_rn((float)i + 0.5f, (float)len);
    return __fadd_rn(c, __fmul_rn(__fsub_rn(sg, 0.5f), inv_len));
}

__device__ __forceinline__ float sigmoidf(float x) { return 1.0f / (1.0f + expf(-x)); }

// a CTA's contiguous block of `count` floats from shared memory to global: one bulk TMA store by thread 0 when both
// ends are 16-byte aligned, a coalesced loop otherwise.  Call after fence_proxy_async_smem + __syncthreads; thread 0
// then waits with tma_store_commit_wait.
__device__ __forceinline__ void store_block(float *dst, const float *src, uint32_t count) {
    const uint32_t bytes = count * 4u;
    if (((reinterpret_cast<uintptr_t>(dst) & 15u) == 0) && ((bytes & 15u) == 0)) {
        if (threadIdx.x == 0 && bytes) tma_store_1d(dst, src, bytes);
    } else {
        for (uint32_t k = threadIdx.x; k < count; k += AD_THREADS) dst[k] = src[k];
    }
}

__global__ void __launch_bounds__(AD_THREADS) k_head_fwd(const HeadArgs a, const HeadOut o) {
    extern __shared__ __align__(128) unsigned char hd_smem[];
    AdHdr *h = reinterpret_cast<AdHdr *>(hd_smem);
    const int HS = 3 * a.d_sh;
    float *harm_s = reinterpret_cast<float *>(hd_smem + AD_HDR_BYTES);  // [AD_THREADS][3 d_sh]
    float *means_s = harm_s + (size_t)AD_THREADS * HS;                  // [AD_THREADS][3]
    float *cov_s = means_s + AD_THREADS * 3;                            // [AD_THREADS][9]
    float *raw_s = cov_s + AD_THREADS * 9;                              // [AD_THREADS][CS]

    const int cam = blockIdx.y, bi = cam >> 1, s = cam & 1, px0 = blockIdx.x * AD_THREADS, tid = threadIdx.x;
    const int n = min(AD_THREADS, a.hw - px0), px = px0 + tid;
    const bool active = tid < n;
    const size_t ci = head_view(a, bi, s), item = (size_t)s * a.b + bi;  // the camera; the (v b) item of the convs
    load_head_camera(a, ci, h);
    float z = 0.f, lg = 0.f;
    float *row = raw_s + (size_t)tid * a.CS;
    if (active) {
        const float *src = a.raw + item * a.C * a.hw + px;
        for (int c = 0; c < a.C; c++) row[c] = src[(size_t)c * a.hw];
        z = a.depths[ci * a.hw + px];
        lg = a.logits[(item * 2 + 1) * a.hw + px];
    }
    __syncthreads();
    const size_t first = (size_t)bi * 2 * a.hw + (size_t)s * a.hw + px0;  // the CTA's first Gaussian, b-major
    if (active) {
        const int py = px / a.W, pxx = px - py * a.W;
        const float x = pixel_coord(pxx, a.W, a.inv_w, sigmoidf(row[0]));
        const float y = pixel_coord(py, a.H, a.inv_h, sigmoidf(row[1]));
        AdGeom g;
        adapter_geometry(*h, x, y, z, row + 2, row + 5, a.smin, a.smax, a.eps, g);
        float N[9];
        adapter_factor(*h, g, N);
#pragma unroll
        for (int i = 0; i < 3; i++) means_s[tid * 3 + i] = h->t[i] + g.dw[i] * z;
#pragma unroll
        for (int i = 0; i < 3; i++)
#pragma unroll
            for (int j = 0; j < 3; j++)
                cov_s[tid * 9 + i * 3 + j] = N[i * 3] * N[j * 3] + N[i * 3 + 1] * N[j * 3 + 1] + N[i * 3 + 2] * N[j * 3 + 2];
        float *out = harm_s + (size_t)tid * HS;
        const float *sh = row + 9;
        const float *mask = h->mask;
        if (a.sh_rot) {
            const float *D = a.sh_rot + (size_t)cam * a.d_sh * a.d_sh;  // same address across the CTA: L1 broadcast
            GS_SH_ROTATE_FWD(D, a.d_sh, mask, sh, out);
        } else {
            GS_SH_MASK_FWD(a.d_sh, mask, sh, out);
        }
        const float q = sigmoidf(lg);
        o.opac[first + tid] = 0.5f * __fadd_rn(__fsub_rn(1.0f, __fsub_rn(1.0f, q)), q);
    }
    fence_proxy_async_smem();
    __syncthreads();
    store_block(o.means + first * 3, means_s, (uint32_t)n * 3);
    store_block(o.cov + first * 9, cov_s, (uint32_t)n * 9);
    store_block(o.harm + first * HS, harm_s, (uint32_t)n * HS);
    if (tid == 0) tma_store_commit_wait();
}

__global__ void __launch_bounds__(AD_THREADS)
k_head_bwd(const HeadArgs a, const HeadOutGrads go, const HeadInGrads gi_) {
    extern __shared__ __align__(128) unsigned char hd_smem[];
    AdHdr *h = reinterpret_cast<AdHdr *>(hd_smem);
    const int HS = 3 * a.d_sh;
    float *gh_s = reinterpret_cast<float *>(hd_smem + AD_HDR_BYTES);  // [AD_THREADS][3 d_sh] incoming dL/dharmonics
    float *gm_s = gh_s + (size_t)AD_THREADS * HS;                      // [AD_THREADS][3]
    float *gc_s = gm_s + AD_THREADS * 3;                               // [AD_THREADS][9]

    const int cam = blockIdx.y, bi = cam >> 1, s = cam & 1, px0 = blockIdx.x * AD_THREADS, tid = threadIdx.x;
    const int lane = tid & 31, warp = tid >> 5;
    const int n = min(AD_THREADS, a.hw - px0), px = px0 + tid;
    const bool active = tid < n;
    const size_t ci = head_view(a, bi, s), item = (size_t)s * a.b + bi;
    const size_t first = (size_t)bi * 2 * a.hw + (size_t)s * a.hw + px0;

    bool bulk_in = false;
    if (go.harm) {
        const float *src = go.harm + first * HS;
        const uint32_t in_bytes = (uint32_t)n * HS * 4u;
        bulk_in = ((reinterpret_cast<uintptr_t>(src) & 15u) == 0) && ((in_bytes & 15u) == 0);
        if (bulk_in) {
            if (tid == 0) {
                mbar_init(&h->bar, 1);
                mbar_fence_init();
                mbar_expect_tx(&h->bar, in_bytes);
                tma_load_1d(gh_s, src, in_bytes, &h->bar);
            }
        } else {
            for (uint32_t k = tid; k < (uint32_t)n * HS; k += AD_THREADS) gh_s[k] = src[k];
        }
    }
    if (go.means)
        for (int k = tid; k < n * 3; k += AD_THREADS) gm_s[k] = go.means[first * 3 + k];
    if (go.cov)
        for (int k = tid; k < n * 9; k += AD_THREADS) gc_s[k] = go.cov[first * 9 + k];
    load_head_camera(a, ci, h);
    float r[9], z = 0.f, lg = 0.f, gop = 0.f;
#pragma unroll
    for (int c = 0; c < 9; c++) r[c] = 0.f;
    r[8] = 1.f;
    const float *src = a.raw + item * a.C * a.hw + px;
    if (active) {
#pragma unroll
        for (int c = 0; c < 9; c++) r[c] = src[(size_t)c * a.hw];
        z = a.depths[ci * a.hw + px];
        lg = a.logits[(item * 2 + 1) * a.hw + px];
        if (go.opac) gop = go.opac[first + tid];
    }
    __syncthreads();
    if (bulk_in) mbar_wait(&h->bar, 0);

    float cam_s[HD_CAM_SUMS];  // dC 9 | dt 3
#pragma unroll
    for (int k = 0; k < HD_CAM_SUMS; k++) cam_s[k] = 0.f;

    if (active) {
        const int py = px / a.W, pxx = px - py * a.W;
        const float sx = sigmoidf(r[0]), sy = sigmoidf(r[1]);
        const float x = pixel_coord(pxx, a.W, a.inv_w, sx), y = pixel_coord(py, a.H, a.inv_h, sy);
        AdGeom g;
        adapter_geometry(*h, x, y, z, r + 2, r + 5, a.smin, a.smax, a.eps, g);
        float dz = 0.f;
        // ---- means = t + dw z ----
        float gm[3] = {0, 0, 0};
        if (go.means) {
#pragma unroll
            for (int i = 0; i < 3; i++) gm[i] = gm_s[tid * 3 + i];
        }
        float ddc[3] = {0, 0, 0};
#pragma unroll
        for (int i = 0; i < 3; i++) {
            cam_s[9 + i] = gm[i];
            const float ddw = gm[i] * z;
            dz = fmaf(gm[i], g.dw[i], dz);
#pragma unroll
            for (int j = 0; j < 3; j++) {
                cam_s[i * 3 + j] = ddw * g.dc[j];
                ddc[j] = fmaf(h->rot[i * 3 + j], ddw, ddc[j]);
            }
        }
        const float dot = ddc[0] * g.dc[0] + ddc[1] * g.dc[1] + ddc[2] * g.dc[2];
        float du[3];
#pragma unroll
        for (int i = 0; i < 3; i++) du[i] = (ddc[i] - g.dc[i] * dot) * g.inv_n;
        const float gx = h->kinv[0] * du[0] + h->kinv[3] * du[1] + h->kinv[6] * du[2];
        const float gy = h->kinv[1] * du[0] + h->kinv[4] * du[1] + h->kinv[7] * du[2];
        // ---- covariance = N N^T, N = C Rq diag(s) ----
        float ds[3] = {0, 0, 0}, dRq[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
        if (go.cov) {
            float N[9], G[9], dN[9];
            adapter_factor(*h, g, N);
#pragma unroll
            for (int k = 0; k < 9; k++) G[k] = gc_s[tid * 9 + k];
#pragma unroll
            for (int i = 0; i < 3; i++)
#pragma unroll
                for (int k = 0; k < 3; k++)
                    dN[i * 3 + k] = (G[i * 3] + G[i]) * N[k] + (G[i * 3 + 1] + G[3 + i]) * N[3 + k] +
                                    (G[i * 3 + 2] + G[6 + i]) * N[6 + k];
#pragma unroll
            for (int i = 0; i < 3; i++)
#pragma unroll
                for (int k = 0; k < 3; k++) {
                    const float dM = h->rot[i] * dN[k] + h->rot[3 + i] * dN[3 + k] + h->rot[6 + i] * dN[6 + k];  // C^T dN
                    ds[k] = fmaf(dM, g.Rq[i * 3 + k], ds[k]);
                    dRq[i * 3 + k] = dM * g.s[k];
                }
        }
        float drow[9];
        drow[0] = gx * a.inv_w * sx * (1.0f - sx);
        drow[1] = gy * a.inv_h * sy * (1.0f - sy);
#pragma unroll
        for (int k = 0; k < 3; k++) {
            dz = fmaf(ds[k], g.s0[k] * h->mult, dz);
            drow[2 + k] = ds[k] * z * h->mult * (a.smax - a.smin) * g.sg[k] * (1.0f - g.sg[k]);
        }
        // ---- quaternion ----
        {
            const float i = g.q[0], j = g.q[1], k = g.q[2], rr = g.q[3], A = g.A;
            const float *d = dRq;
            const float dA = -(j * j + k * k) * d[0] + (i * j - k * rr) * d[1] + (i * k + j * rr) * d[2] +
                             (i * j + k * rr) * d[3] - (i * i + k * k) * d[4] + (j * k - i * rr) * d[5] +
                             (i * k - j * rr) * d[6] + (j * k + i * rr) * d[7] - (i * i + j * j) * d[8];
            float dq[4];
            dq[0] = A * (j * d[1] + k * d[2] + j * d[3] - 2.f * i * d[4] - rr * d[5] + k * d[6] + rr * d[7] - 2.f * i * d[8]);
            dq[1] = A * (-2.f * j * d[0] + i * d[1] + rr * d[2] + i * d[3] + k * d[5] - rr * d[6] + k * d[7] - 2.f * j * d[8]);
            dq[2] = A * (-2.f * k * d[0] - rr * d[1] + i * d[2] + rr * d[3] - 2.f * k * d[4] + j * d[5] + i * d[6] + j * d[7]);
            dq[3] = A * (-k * d[1] + j * d[2] + k * d[3] - i * d[5] - j * d[6] + i * d[7]);
            const float back = -A * A * dA;  // dA/dq_m = -A^2 q_m
#pragma unroll
            for (int m = 0; m < 4; m++) dq[m] = fmaf(back, g.q[m], dq[m]);
            const float *qraw = r + 5;
            const float inv = 1.0f / (g.nq + a.eps);
            const float dotq = dq[0] * qraw[0] + dq[1] * qraw[1] + dq[2] * qraw[2] + dq[3] * qraw[3];
            // d|q|/dq = q / |q| is 0/0 at a zero (or fully underflowed) raw quaternion: 0 there, as torch's norm
            const float radial = g.nq == 0.f ? 0.f : dotq * inv * inv / g.nq;
#pragma unroll
            for (int m = 0; m < 4; m++) drow[5 + m] = dq[m] * inv - qraw[m] * radial;
        }
        if (gi_.depths) gi_.depths[ci * a.hw + px] = dz;
        if (gi_.logits) {
            const float q = sigmoidf(lg);
            gi_.logits[item * 2 * a.hw + px] = 0.0f;
            gi_.logits[(item * 2 + 1) * a.hw + px] = gop * (1.0f - q) * q;
        }
        if (gi_.raw) {
            float *dst = gi_.raw + item * a.C * a.hw + px;
#pragma unroll
            for (int c = 0; c < 9; c++) dst[(size_t)c * a.hw] = drow[c];
            // ---- harmonics: d raw[9 + c d_sh + j] = mask[j] sum_i D[i][j] g[i][c] ----
            const Plane dsh{dst + (size_t)9 * a.hw, (size_t)a.hw};
            const float *mask = h->mask;
            if (!go.harm) {
                for (int k = 0; k < HS; k++) dsh[k] = 0.f;
            } else {
                const float *gh = gh_s + (size_t)tid * HS;
                if (a.sh_rot) {
                    const float *D = a.sh_rot + (size_t)cam * a.d_sh * a.d_sh;
                    GS_SH_ROTATE_BWD(D, a.d_sh, mask, gh, dsh);
                } else {
                    GS_SH_MASK_BWD(a.d_sh, mask, gh, dsh);
                }
            }
        }
    }
    if (!gi_.c2w) return;
    // ---- per-camera sums: warp shuffle tree, warps in order, one partial per CTA ----
#pragma unroll
    for (int k = 0; k < HD_CAM_SUMS; k++) {
        float v = cam_s[k];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
        if (lane == 0) h->red[warp][k] = v;
    }
    __syncthreads();
    if (tid < HD_CAM_SUMS) {
        float v = 0.f;
#pragma unroll
        for (int w = 0; w < AD_THREADS / 32; w++) v += h->red[w][tid];
        gi_.cam_partial[((size_t)cam * gridDim.x + blockIdx.x) * HD_CAM_SUMS + tid] = v;
    }
}

// dL/dc2w [b, V, 16]: for views 0 and V - 1 the sum, in CTA order, of their camera's partials (row 3 gets 0); middle
// views 0.  Then the depth gradient of the middle views, which the head does not read: 0.
__global__ void __launch_bounds__(HD_FIN_THREADS)
k_head_finalize(int b, int V, int hw, int ctas, const float *__restrict__ part, float *__restrict__ d_c2w,
                float *__restrict__ d_depths) {
    const int64_t t = (int64_t)blockIdx.x * HD_FIN_THREADS + threadIdx.x;
    const int64_t nc = d_c2w ? (int64_t)b * V * 16 : 0;
    if (t < nc) {
        const int e = (int)(t & 15), view = (int)((t >> 4) % V), bi = (int)((t >> 4) / V);
        const int row = e >> 2, col = e & 3, slot = view == 0 ? 0 : (view == V - 1 ? 1 : -1);
        float v = 0.f;
        if (slot >= 0 && row < 3) {
            const int src = col < 3 ? row * 3 + col : 9 + row;
            const float *p = part + (size_t)(bi * 2 + slot) * ctas * HD_CAM_SUMS + src;
            for (int k = 0; k < ctas; k++) v += p[(size_t)k * HD_CAM_SUMS];
        }
        d_c2w[t] = v;
        return;
    }
    if (!d_depths || V < 3) return;
    const int64_t idx = t - nc, per_scene = (int64_t)(V - 2) * hw;
    if (idx >= (int64_t)b * per_scene) return;
    const int64_t bi = idx / per_scene, rem = idx - bi * per_scene;
    d_depths[(bi * V + 1) * hw + rem] = 0.f;  // views 1 .. V - 2 are contiguous
}

constexpr int head_row_stride(int d_sh) { return (9 + 3 * d_sh) | 1; }
constexpr size_t head_fwd_smem(int d_sh) {
    return AD_HDR_BYTES + (size_t)AD_THREADS * (3 * d_sh + 3 + 9 + head_row_stride(d_sh)) * 4;
}
constexpr size_t head_bwd_smem(int d_sh) { return AD_HDR_BYTES + (size_t)AD_THREADS * (3 * d_sh + 3 + 9) * 4; }

int head_check(const GsGaussianHeadConfig *c) {
    if (!c) return gs_set_error(GS_ERR_INVALID, "gaussian head: null config");
    const int d = c->d_sh;
    if (d != 1 && d != 4 && d != 9 && d != 16 && d != 25)
        return gs_set_error(GS_ERR_INVALID, "gaussian head: d_sh must be (sh_degree + 1)^2 with sh_degree <= 4");
    if (c->batch < 1 || c->views < 2 || c->height < 1 || c->width < 1 || c->batch > 32767 ||
        (int64_t)c->height * c->width > (1 << 28) ||
        (int64_t)c->batch * 2 * c->height * c->width * (9 + 3 * d) > (1ll << 40))
        return gs_set_error(GS_ERR_INVALID, "gaussian head: need batch in [1, 32767], views >= 2, height, width >= 1, "
                                            "height width <= 2^28");
    if (c->flags) return gs_set_error(GS_ERR_INVALID, "gaussian head: unknown flags");
    return GS_OK;
}

int head_args(const GsGaussianHeadConfig *c, const GsGaussianHeadInputs *in, HeadArgs &a) {
    if (int rc = head_check(c)) return rc;
    if (!in || !in->raw_gaussians || !in->density_logits || !in->depths || !in->c2w || !in->intrinsics || !in->sh_mask)
        return gs_set_error(GS_ERR_INVALID, "gaussian head: null input pointer");
    a.b = c->batch; a.V = c->views; a.H = c->height; a.W = c->width; a.hw = c->height * c->width;
    a.d_sh = c->d_sh; a.C = 9 + 3 * c->d_sh; a.CS = head_row_stride(c->d_sh);
    a.smin = c->scale_min; a.smax = c->scale_max; a.eps = c->eps;
    a.inv_w = 1.0f / (float)c->width; a.inv_h = 1.0f / (float)c->height;  // pixel_size = 1 / tensor((w, h)), float32
    a.raw = in->raw_gaussians; a.logits = in->density_logits; a.depths = in->depths; a.c2w = in->c2w;
    a.K = in->intrinsics; a.sh_rot = in->sh_rotation; a.sh_mask = in->sh_mask;
    return GS_OK;
}

}  // namespace

extern "C" GS_API int64_t gs_gaussian_head_scratch_bytes(const GsGaussianHeadConfig *cfg) {
    if (!cfg || head_check(cfg) != GS_OK) return -1;
    const int64_t ctas = ((int64_t)cfg->height * cfg->width + AD_THREADS - 1) / AD_THREADS;
    return (int64_t)cfg->batch * 2 * ctas * HD_CAM_SUMS * 4;
}

extern "C" GS_API int gs_gaussian_head_forward(const GsGaussianHeadConfig *cfg, const GsGaussianHeadInputs *in,
                                               const GsGaussianHeadOutputs *out, void *stream) {
    HeadArgs a;
    if (int rc = head_args(cfg, in, a)) return rc;
    if (!out || !out->means || !out->covariances || !out->harmonics || !out->opacities)
        return gs_set_error(GS_ERR_INVALID, "gs_gaussian_head_forward: null output pointer");
    const HeadOut o{out->means, out->covariances, out->harmonics, out->opacities};
    const size_t smem = head_fwd_smem(a.d_sh);
    GS_CUDA_OK(cudaFuncSetAttribute(k_head_fwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const dim3 grid((a.hw + AD_THREADS - 1) / AD_THREADS, 2 * a.b);
    k_head_fwd<<<grid, AD_THREADS, smem, static_cast<cudaStream_t>(stream)>>>(a, o);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}

extern "C" GS_API int gs_gaussian_head_backward(const GsGaussianHeadConfig *cfg, const GsGaussianHeadInputs *in,
                                                const GsGaussianHeadOutGrads *gout, const GsGaussianHeadInGrads *gin,
                                                void *stream) {
    HeadArgs a;
    if (int rc = head_args(cfg, in, a)) return rc;
    if (!gout || !gin) return gs_set_error(GS_ERR_INVALID, "gs_gaussian_head_backward: null gradients");
    if (gin->c2w && !gin->scratch)
        return gs_set_error(GS_ERR_INVALID, "gs_gaussian_head_backward: dL/dc2w needs scratch "
                                            "(gs_gaussian_head_scratch_bytes)");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const HeadOutGrads go{gout->means, gout->covariances, gout->harmonics, gout->opacities};
    const HeadInGrads gi{gin->raw_gaussians, gin->density_logits, gin->depths, gin->c2w,
                         static_cast<float *>(gin->scratch)};
    const size_t smem = head_bwd_smem(a.d_sh);
    const dim3 grid((a.hw + AD_THREADS - 1) / AD_THREADS, 2 * a.b);
    GS_CUDA_OK(cudaFuncSetAttribute(k_head_bwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_head_bwd<<<grid, AD_THREADS, smem, st>>>(a, go, gi);
    GS_CUDA_OK(cudaGetLastError());
    const int64_t work = (gi.c2w ? (int64_t)a.b * a.V * 16 : 0) + (gi.depths ? (int64_t)a.b * (a.V - 2) * a.hw : 0);
    if (work > 0) {
        k_head_finalize<<<(unsigned)((work + HD_FIN_THREADS - 1) / HD_FIN_THREADS), HD_FIN_THREADS, 0, st>>>(
            a.b, a.V, a.hw, (int)grid.x, gi.cam_partial, gi.c2w, gi.depths);
        GS_CUDA_OK(cudaGetLastError());
    }
    return GS_OK;
}
