// gs_adapter.cu -- fused Gaussian adapter (SURVEY.md section 8(f).2): the per-Gaussian arithmetic of
// PF3plat's src/model/encoder/common/gaussian_adapter.py:48-98 (GaussianAdapter.forward) in ONE kernel per
// direction, writing the harmonics directly in the (d_sh, xyz) layout the rasterizer reads (the relayout +
// .contiguous() copy of PF3plat's src/model/decoder/cuda_splatting.py:75 disappears).
//
// Per Gaussian g of camera v (reference line in brackets):
//   scales    = (smin + (smax - smin) * sigmoid(raw[0:3])) * depth * multiplier[v]                  [:62-70]
//   rotations = raw[3:7] / (|raw[3:7]| + eps)                                                       [:73]
//   sh        = raw[7:].view(3, d_sh) * sh_mask                                                     [:76-77]
//   cov       = C (Rq S S^T Rq^T) C^T, Rq = quaternion_to_matrix(rotations) (xyzw), C = c2w[:3,:3]  [:80-82]
//   means     = c2w[:3,3] + C normalize(Kinv (x, y, 1)) * depth                                     [:86-87]
//   harmonics = D_v sh  (block-diagonal Wigner-D of C, computed by the caller; NULL = identity)     [:92]
// C is detached in cov and harmonics (:81), not in means.  The tiny per-camera quantities (Kinv, multiplier, D)
// stay with the caller, which keeps them differentiable with ordinary tensor ops; the backward kernel returns the
// per-camera sums dL/dKinv, dL/dc2w, dL/dmultiplier.
//
// Design: one thread per Gaussian, 128 per CTA, one camera per blockIdx.y.  The CTA's contiguous block of raw
// rows (128 x 328 B) arrives by one bulk TMA copy; the harmonics block (128 x 300 B) is assembled in shared memory and
// leaves by one bulk TMA store, so both big streams are fully coalesced; the backward mirrors it (gradient of the
// harmonics in by TMA, gradient of the raw rows out by TMA).  HBM-bound: 328 + 12 B in, 300 + 76 B out per Gaussian.
#include "gs_common.cuh"
#include "gs_adapter_math.cuh"

namespace {

struct AdapterArgs {
    int V, R, d_sh, C;  // C = 7 + 3 * d_sh
    float smin, smax, eps;
    const float *c2w, *kinv, *mult, *sh_rot, *sh_mask;
    const float *coords, *depths, *raw;
};
struct AdapterOut {
    float *means, *cov, *harm, *scales, *rot;
};
struct AdapterOutGrads {
    const float *means, *cov, *harm, *scales, *rot;
};
struct AdapterInGrads {
    float *coords, *depths, *raw, *c2w, *kinv, *mult;
    float *cam_partial;  // deterministic mode: [V][CTAs per camera][AD_CAM_SUMS] per-CTA sums (see k_adapter_bwd)
};

constexpr int AD_CAM_SUMS = 22;  // per-camera sums of the backward: dKinv 9 | dC 9 | dt 3 | dmultiplier 1

__device__ __forceinline__ void load_camera(const AdapterArgs &a, int v, AdHdr *h) {
    const int tid = threadIdx.x;
    if (tid < 9) {
        h->kinv[tid] = a.kinv[(size_t)v * 9 + tid];
        h->rot[tid] = a.c2w[(size_t)v * 16 + (tid / 3) * 4 + tid % 3];
    } else if (tid < 12) {
        h->t[tid - 9] = a.c2w[(size_t)v * 16 + (tid - 9) * 4 + 3];
    } else if (tid == 12) {
        h->mult = a.mult[v];
    }
    if (tid >= 32 && tid < 32 + a.d_sh) h->mask[tid - 32] = a.sh_mask[tid - 32];
}

__global__ void __launch_bounds__(AD_THREADS) k_adapter_fwd(const AdapterArgs a, const AdapterOut o) {
    extern __shared__ __align__(128) unsigned char ad_smem[];
    AdHdr *h = reinterpret_cast<AdHdr *>(ad_smem);
    float *raw_s = reinterpret_cast<float *>(ad_smem + AD_HDR_BYTES);  // [AD_THREADS][C]
    float *harm_s = raw_s + (size_t)AD_THREADS * a.C;                   // [AD_THREADS][3 * d_sh]

    const int v = blockIdx.y, g0 = blockIdx.x * AD_THREADS, tid = threadIdx.x;
    const int n = min(AD_THREADS, a.R - g0);
    const size_t first = (size_t)v * a.R + g0;
    const bool active = tid < n;
    const int HS = 3 * a.d_sh;

    const float *src = a.raw + first * a.C;
    const uint32_t in_bytes = (uint32_t)n * a.C * 4u;
    const bool bulk_in = ((reinterpret_cast<uintptr_t>(src) & 15u) == 0) && ((in_bytes & 15u) == 0);
    if (bulk_in) {
        if (tid == 0) {
            mbar_init(&h->bar, 1);
            mbar_fence_init();
            mbar_expect_tx(&h->bar, in_bytes);
            tma_load_1d(raw_s, src, in_bytes, &h->bar);
        }
    } else {
        for (uint32_t k = tid; k < (uint32_t)n * a.C; k += AD_THREADS) raw_s[k] = src[k];
    }
    load_camera(a, v, h);
    float x = 0.f, y = 0.f, z = 0.f;
    if (active) {
        x = a.coords[(first + tid) * 2];
        y = a.coords[(first + tid) * 2 + 1];
        z = a.depths[first + tid];
    }
    __syncthreads();
    if (bulk_in) mbar_wait(&h->bar, 0);

    if (active) {
        const float *row = raw_s + (size_t)tid * a.C;
        AdGeom g;
        adapter_geometry(*h, x, y, z, row, row + 3, a.smin, a.smax, a.eps, g);
        float N[9];
        adapter_factor(*h, g, N);
        const size_t gi = first + tid;
#pragma unroll
        for (int i = 0; i < 3; i++) {
            o.means[gi * 3 + i] = h->t[i] + g.dw[i] * z;
            o.scales[gi * 3 + i] = g.s[i];
        }
#pragma unroll
        for (int k = 0; k < 4; k++) o.rot[gi * 4 + k] = g.q[k];
#pragma unroll
        for (int i = 0; i < 3; i++)
#pragma unroll
            for (int j = 0; j < 3; j++)
                o.cov[gi * 9 + i * 3 + j] = N[i * 3] * N[j * 3] + N[i * 3 + 1] * N[j * 3 + 1] + N[i * 3 + 2] * N[j * 3 + 2];
        // harmonics: out[d][c] = sum_j D[d][j] * raw[c][j] * mask[j], D block-diagonal by degree
        float *out = harm_s + (size_t)tid * HS;
        const float *sh = row + 7;
        if (a.sh_rot) {
            const float *D = a.sh_rot + (size_t)v * a.d_sh * a.d_sh;  // same address across the CTA: L1 broadcast
            GS_SH_ROTATE_FWD(D, a.d_sh, h->mask, sh, out);
        } else {
            GS_SH_MASK_FWD(a.d_sh, h->mask, sh, out);
        }
    }
    float *dst = o.harm + first * HS;
    const uint32_t out_bytes = (uint32_t)n * HS * 4u;
    const bool bulk_out = ((reinterpret_cast<uintptr_t>(dst) & 15u) == 0) && ((out_bytes & 15u) == 0);
    if (bulk_out) {
        fence_proxy_async_smem();
        __syncthreads();
        if (tid == 0) {
            tma_store_1d(dst, harm_s, out_bytes);
            tma_store_commit_wait();
        }
    } else {
        __syncthreads();
        for (uint32_t k = tid; k < (uint32_t)n * HS; k += AD_THREADS) dst[k] = harm_s[k];
    }
}

// DET (GS_ADAPTER_DETERMINISTIC): the CTA's 22 per-camera sums are stored to gi_.cam_partial instead of being added to the
// outputs with float atomics; k_adapter_cam_finalize adds them up in CTA order.
template <bool DET>
__global__ void __launch_bounds__(AD_THREADS)
k_adapter_bwd(const AdapterArgs a, const AdapterOutGrads go, const AdapterInGrads gi_) {
    extern __shared__ __align__(128) unsigned char ad_smem[];
    AdHdr *h = reinterpret_cast<AdHdr *>(ad_smem);
    float *draw_s = reinterpret_cast<float *>(ad_smem + AD_HDR_BYTES);  // [AD_THREADS][C]   gradient of the raw rows
    float *gh_s = draw_s + (size_t)AD_THREADS * a.C;                    // [AD_THREADS][3 * d_sh] incoming dL/dharmonics

    const int v = blockIdx.y, g0 = blockIdx.x * AD_THREADS, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int n = min(AD_THREADS, a.R - g0);
    const size_t first = (size_t)v * a.R + g0;
    const bool active = tid < n;
    const int HS = 3 * a.d_sh;

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
    load_camera(a, v, h);
    float x = 0.f, y = 0.f, z = 0.f, sraw[3] = {0, 0, 0}, qraw[4] = {0, 0, 0, 1};
    const size_t gi = first + tid;
    if (active) {
        x = a.coords[gi * 2];
        y = a.coords[gi * 2 + 1];
        z = a.depths[gi];
        const float *row = a.raw + gi * a.C;
#pragma unroll
        for (int k = 0; k < 3; k++) sraw[k] = row[k];
#pragma unroll
        for (int k = 0; k < 4; k++) qraw[k] = row[3 + k];
    }
    __syncthreads();
    if (bulk_in) mbar_wait(&h->bar, 0);

    // per-camera sums: [0..8] dKinv, [9..17] dC (through the means only), [18..20] dt, [21] dmultiplier
    float cam[22];
#pragma unroll
    for (int k = 0; k < 22; k++) cam[k] = 0.f;

    if (active) {
        AdGeom g;
        adapter_geometry(*h, x, y, z, sraw, qraw, a.smin, a.smax, a.eps, g);
        float *drow = draw_s + (size_t)tid * a.C;
        float dz = 0.f;
        // ---- means = t + dw * z ----
        float gm[3] = {0, 0, 0};
        if (go.means) {
#pragma unroll
            for (int i = 0; i < 3; i++) gm[i] = go.means[gi * 3 + i];
        }
        float ddc[3] = {0, 0, 0};
#pragma unroll
        for (int i = 0; i < 3; i++) {
            cam[18 + i] = gm[i];
            const float ddw = gm[i] * z;
            dz = fmaf(gm[i], g.dw[i], dz);
#pragma unroll
            for (int j = 0; j < 3; j++) {
                cam[9 + i * 3 + j] = ddw * g.dc[j];
                ddc[j] = fmaf(h->rot[i * 3 + j], ddw, ddc[j]);
            }
        }
        const float dot = ddc[0] * g.dc[0] + ddc[1] * g.dc[1] + ddc[2] * g.dc[2];
        float du[3];
#pragma unroll
        for (int i = 0; i < 3; i++) {
            du[i] = (ddc[i] - g.dc[i] * dot) * g.inv_n;
            cam[i * 3] = du[i] * x;
            cam[i * 3 + 1] = du[i] * y;
            cam[i * 3 + 2] = du[i];
        }
        if (gi_.coords) {
            gi_.coords[gi * 2] = h->kinv[0] * du[0] + h->kinv[3] * du[1] + h->kinv[6] * du[2];
            gi_.coords[gi * 2 + 1] = h->kinv[1] * du[0] + h->kinv[4] * du[1] + h->kinv[7] * du[2];
        }
        // ---- covariance = N N^T, N = C Rq diag(s) ----
        float ds[3] = {0, 0, 0}, dRq[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
        if (go.cov) {
            float N[9], G[9], dN[9];
            adapter_factor(*h, g, N);
#pragma unroll
            for (int k = 0; k < 9; k++) G[k] = go.cov[gi * 9 + k];
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
        // ---- scales ----
        if (go.scales) {
#pragma unroll
            for (int k = 0; k < 3; k++) ds[k] += go.scales[gi * 3 + k];
        }
        float dmult = 0.f;
#pragma unroll
        for (int k = 0; k < 3; k++) {
            dz = fmaf(ds[k], g.s0[k] * h->mult, dz);
            dmult = fmaf(ds[k], g.s0[k] * z, dmult);
            drow[k] = ds[k] * z * h->mult * (a.smax - a.smin) * g.sg[k] * (1.0f - g.sg[k]);
        }
        cam[21] = dmult;
        // ---- quaternion ----
        {
            const float i = g.q[0], j = g.q[1], k = g.q[2], r = g.q[3], A = g.A;
            const float *d = dRq;
            const float dA = -(j * j + k * k) * d[0] + (i * j - k * r) * d[1] + (i * k + j * r) * d[2] + (i * j + k * r) * d[3] -
                             (i * i + k * k) * d[4] + (j * k - i * r) * d[5] + (i * k - j * r) * d[6] + (j * k + i * r) * d[7] -
                             (i * i + j * j) * d[8];
            float dq[4];
            dq[0] = A * (j * d[1] + k * d[2] + j * d[3] - 2.f * i * d[4] - r * d[5] + k * d[6] + r * d[7] - 2.f * i * d[8]);
            dq[1] = A * (-2.f * j * d[0] + i * d[1] + r * d[2] + i * d[3] + k * d[5] - r * d[6] + k * d[7] - 2.f * j * d[8]);
            dq[2] = A * (-2.f * k * d[0] - r * d[1] + i * d[2] + r * d[3] - 2.f * k * d[4] + j * d[5] + i * d[6] + j * d[7]);
            dq[3] = A * (-k * d[1] + j * d[2] + k * d[3] - i * d[5] - j * d[6] + i * d[7]);
            const float back = -A * A * dA;  // dA/dq_m = -A^2 q_m
#pragma unroll
            for (int m = 0; m < 4; m++) dq[m] = fmaf(back, g.q[m], dq[m]);
            if (go.rot) {
#pragma unroll
                for (int m = 0; m < 4; m++) dq[m] += go.rot[gi * 4 + m];
            }
            // q = qraw / (|qraw| + eps)
            const float inv = 1.0f / (g.nq + a.eps);
            const float dotq = dq[0] * qraw[0] + dq[1] * qraw[1] + dq[2] * qraw[2] + dq[3] * qraw[3];
            // d|q|/dq = q / |q| is 0/0 at a zero (or fully underflowed) raw quaternion: 0 there, as torch's norm
            const float radial = g.nq == 0.f ? 0.f : dotq * inv * inv / g.nq;
#pragma unroll
            for (int m = 0; m < 4; m++) drow[3 + m] = dq[m] * inv - qraw[m] * radial;
        }
        if (gi_.depths) gi_.depths[gi] = dz;
        // ---- harmonics: d raw[c][j] = mask[j] * sum_i D[i][j] g[i][c] ----
        float *dsh = drow + 7;
        if (!go.harm) {
            for (int k = 0; k < HS; k++) dsh[k] = 0.f;
        } else {
            const float *gh = gh_s + (size_t)tid * HS;
            if (a.sh_rot) {
                const float *D = a.sh_rot + (size_t)v * a.d_sh * a.d_sh;
                GS_SH_ROTATE_BWD(D, a.d_sh, h->mask, gh, dsh);
            } else {
                GS_SH_MASK_BWD(a.d_sh, h->mask, gh, dsh);
            }
        }
    }
    // ---- per-camera sums: warp reduce, then one atomic per value and CTA ----
#pragma unroll
    for (int k = 0; k < 22; k++) {
        float s = cam[k];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
        if (lane == 0) h->red[warp][k] = s;
    }
    float *dst = gi_.raw ? gi_.raw + first * a.C : nullptr;
    const uint32_t out_bytes = (uint32_t)n * a.C * 4u;
    const bool bulk_out = dst && ((reinterpret_cast<uintptr_t>(dst) & 15u) == 0) && ((out_bytes & 15u) == 0);
    if (bulk_out) fence_proxy_async_smem();
    __syncthreads();
    if (DET && tid < AD_CAM_SUMS) {
        float s = 0.f;
#pragma unroll
        for (int w = 0; w < AD_THREADS / 32; w++) s += h->red[w][tid];
        gi_.cam_partial[((size_t)v * gridDim.x + blockIdx.x) * AD_CAM_SUMS + tid] = s;
    } else if (tid < 22) {
        float s = 0.f;
#pragma unroll
        for (int w = 0; w < AD_THREADS / 32; w++) s += h->red[w][tid];
        if (tid < 9) {
            if (gi_.kinv) atomicAdd(&gi_.kinv[(size_t)v * 9 + tid], s);
        } else if (tid < 18) {
            const int e = tid - 9;
            if (gi_.c2w) atomicAdd(&gi_.c2w[(size_t)v * 16 + (e / 3) * 4 + e % 3], s);
        } else if (tid < 21) {
            if (gi_.c2w) atomicAdd(&gi_.c2w[(size_t)v * 16 + (tid - 18) * 4 + 3], s);
        } else {
            if (gi_.mult) atomicAdd(&gi_.mult[v], s);
        }
    }
    if (dst) {
        if (bulk_out) {
            if (tid == 32) {
                tma_store_1d(dst, draw_s, out_bytes);
                tma_store_commit_wait();
            }
        } else {
            for (uint32_t k = tid; k < (uint32_t)n * a.C; k += AD_THREADS) dst[k] = draw_s[k];
        }
    }
}

// Deterministic mode: every element of dL/dKinv [V,9], dL/dc2w [V,16] (zeros outside the top 3x4 block) and
// dL/dmultiplier [V] is the sum, in CTA order, of the CTAs' partials.
__global__ void k_adapter_cam_finalize(int V, int ctas, const float *__restrict__ part, float *__restrict__ kinv,
                                       float *__restrict__ c2w, float *__restrict__ mult) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= V * 26) return;
    const int v = t / 26, e = t - v * 26;  // e: 0-8 Kinv, 9-24 c2w (row-major), 25 multiplier
    float *dst;
    int src = -1;  // index of the partial, -1: a c2w entry the adapter gives no gradient
    if (e < 9) {
        dst = kinv ? kinv + (size_t)v * 9 + e : nullptr;
        src = e;
    } else if (e < 25) {
        const int r = (e - 9) >> 2, col = (e - 9) & 3;
        dst = c2w ? c2w + (size_t)v * 16 + (e - 9) : nullptr;
        if (r < 3) src = col < 3 ? 9 + r * 3 + col : 18 + r;
    } else {
        dst = mult ? mult + v : nullptr;
        src = 21;
    }
    if (!dst) return;
    float s = 0.f;
    if (src >= 0)
        for (int k = 0; k < ctas; k++) s += part[((size_t)v * ctas + k) * AD_CAM_SUMS + src];
    *dst = s;
}

constexpr size_t adapter_smem_bytes(int d_sh) { return AD_HDR_BYTES + (size_t)AD_THREADS * ((7 + 3 * d_sh) + 3 * d_sh) * 4; }

}  // namespace

static int adapter_args(const GsAdapterConfig *cfg, const GsAdapterInputs *in, AdapterArgs &a) {
    if (!cfg || !in) return gs_set_error(GS_ERR_INVALID, "null adapter config/inputs");
    if (cfg->V < 0 || cfg->R < 0) return gs_set_error(GS_ERR_INVALID, "negative adapter sizes");
    const int d = cfg->d_sh;
    if (d != 1 && d != 4 && d != 9 && d != 16 && d != 25)
        return gs_set_error(GS_ERR_INVALID, "d_sh must be (sh_degree + 1)^2 with sh_degree <= 4");
    if ((size_t)cfg->V * (size_t)cfg->R > 0) {
        if (!cfg->c2w || !cfg->kinv || !cfg->multiplier || !cfg->sh_mask)
            return gs_set_error(GS_ERR_INVALID, "adapter camera arrays missing");
        if (!in->coordinates || !in->depths || !in->raw_gaussians)
            return gs_set_error(GS_ERR_INVALID, "adapter inputs missing");
    }
    if (cfg->V > 65535) return gs_set_error(GS_ERR_INVALID, "more than 65535 cameras in one adapter call");
    a.V = cfg->V; a.R = cfg->R; a.d_sh = d; a.C = 7 + 3 * d;
    a.smin = cfg->scale_min; a.smax = cfg->scale_max; a.eps = cfg->eps;
    a.c2w = cfg->c2w; a.kinv = cfg->kinv; a.mult = cfg->multiplier; a.sh_rot = cfg->sh_rotation; a.sh_mask = cfg->sh_mask;
    a.coords = in->coordinates; a.depths = in->depths; a.raw = in->raw_gaussians;
    return GS_OK;
}

extern "C" GS_API int gs_adapter_forward(const GsAdapterConfig *cfg, const GsAdapterInputs *in, const GsAdapterOutputs *out,
                                         void *stream) {
    AdapterArgs a;
    int rc = adapter_args(cfg, in, a);
    if (rc != GS_OK) return rc;
    if (!out) return gs_set_error(GS_ERR_INVALID, "null adapter outputs");
    if ((size_t)a.V * a.R == 0) return GS_OK;
    if (!out->means || !out->covariances || !out->harmonics || !out->scales || !out->rotations)
        return gs_set_error(GS_ERR_INVALID, "adapter outputs missing");
    const AdapterOut o{out->means, out->covariances, out->harmonics, out->scales, out->rotations};
    const size_t smem = adapter_smem_bytes(a.d_sh);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    GS_CUDA_OK(cudaFuncSetAttribute(k_adapter_fwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid((a.R + AD_THREADS - 1) / AD_THREADS, a.V);
    k_adapter_fwd<<<grid, AD_THREADS, smem, st>>>(a, o);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}

extern "C" GS_API int gs_adapter_backward(const GsAdapterConfig *cfg, const GsAdapterInputs *in, const GsAdapterOutGrads *gout,
                                          const GsAdapterInGrads *gin, void *stream) {
    AdapterArgs a;
    int rc = adapter_args(cfg, in, a);
    if (rc != GS_OK) return rc;
    if (!gout || !gin) return gs_set_error(GS_ERR_INVALID, "null adapter gradients");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const bool cam_grads = gin->c2w || gin->kinv || gin->multiplier;
    const bool det = (cfg->flags & GS_ADAPTER_DETERMINISTIC) && cam_grads && (size_t)a.V * a.R > 0;
    if (det && !gin->scratch)
        return gs_set_error(GS_ERR_INVALID, "GS_ADAPTER_DETERMINISTIC needs gin->scratch (gs_adapter_scratch_bytes)");
    if (!det) {  // the kernel accumulates into them (deterministic mode: k_adapter_cam_finalize writes every element)
        if (gin->c2w && a.V) GS_CUDA_OK(cudaMemsetAsync(gin->c2w, 0, (size_t)a.V * 16 * 4, st));
        if (gin->kinv && a.V) GS_CUDA_OK(cudaMemsetAsync(gin->kinv, 0, (size_t)a.V * 9 * 4, st));
        if (gin->multiplier && a.V) GS_CUDA_OK(cudaMemsetAsync(gin->multiplier, 0, (size_t)a.V * 4, st));
    }
    if ((size_t)a.V * a.R == 0) return GS_OK;
    const AdapterOutGrads go{gout->means, gout->covariances, gout->harmonics, gout->scales, gout->rotations};
    const AdapterInGrads gi{gin->coordinates, gin->depths, gin->raw_gaussians, gin->c2w, gin->kinv, gin->multiplier,
                            static_cast<float *>(gin->scratch)};
    const size_t smem = adapter_smem_bytes(a.d_sh);
    dim3 grid((a.R + AD_THREADS - 1) / AD_THREADS, a.V);
    if (det) {
        GS_CUDA_OK(cudaFuncSetAttribute(k_adapter_bwd<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        k_adapter_bwd<true><<<grid, AD_THREADS, smem, st>>>(a, go, gi);
        GS_CUDA_OK(cudaGetLastError());
        k_adapter_cam_finalize<<<(a.V * 26 + 127) / 128, 128, 0, st>>>(a.V, (int)grid.x, gi.cam_partial, gi.kinv, gi.c2w,
                                                                       gi.mult);
    } else {
        GS_CUDA_OK(cudaFuncSetAttribute(k_adapter_bwd<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        k_adapter_bwd<false><<<grid, AD_THREADS, smem, st>>>(a, go, gi);
    }
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}

extern "C" GS_API int64_t gs_adapter_scratch_bytes(const GsAdapterConfig *cfg) {
    if (!cfg || cfg->V < 0 || cfg->R < 0 || cfg->V > 65535) return -1;
    const int d = cfg->d_sh;
    if (d != 1 && d != 4 && d != 9 && d != 16 && d != 25) return -1;
    return (int64_t)cfg->V * ((cfg->R + AD_THREADS - 1) / AD_THREADS) * AD_CAM_SUMS * 4;
}
