// gs_preprocess_bwd.cu -- stage 2 of the backward: per-(view, Gaussian) accumulators -> input gradients.
//
// Semantics: SURVEY.md Appendix A "Preprocess backward" (upstream computeCov2DCUDA + preprocessCUDA backward):
// conic -> cov2D (with 1/(det^2+1e-7)) -> cov3D(6) and mean through the clamped projection Jacobian; mean2D
// (NDC-scaled) -> mean through the perspective divide; colour -> SH coefficients and mean through the view
// direction, honouring the clamp flags; cov3D -> scales/rotations when those were the inputs.
//
// Design (DESIGN.md section 5.5): one thread per Gaussian looping over the views of its scene and
// summing in registers / shared memory, so scene-level gradients are written ONCE, coalesced, with no atomics
// and no zero-fill pass (every output element is written, zeros included).  The SH block is staged in by one
// bulk TMA load and its gradient block leaves by one bulk TMA store.
#include "gs_common.cuh"

namespace {

constexpr int PB_THREADS = 128;
// Resident CTAs per SM the register allocation is bounded for.  The kernel is latency-bound; unbounded it takes 150
// registers (3 CTAs/SM).  On C2, 4 CTAs (128 registers, 36 B of spills) were faster than 3, and 5 CTAs (96 registers,
// 304 B of spills inside the view loop) much slower.
constexpr int PB_MIN_CTAS = 4;

struct PbSmem {
    ViewCam cams[GS_CAM_CHUNK];
    uint64_t bar;
};
constexpr int PB_SMEM_HDR = (sizeof(PbSmem) + 127) / 128 * 128;

constexpr int PB_SH_EVAL = 16;  // coefficients per channel the evaluator can touch (bands 0..3)
constexpr int PB_SH_B4 = 27;    // band-4 accumulators per Gaussian (9 coefficients x 3 channels), degree-4 kernels only

// dL/dsh_k += basis_k(dir) * g  and  dL/ddir, for one colour channel.  sh: stride-3 view of this channel's
// coefficients in shared memory; gsh: stride-3 view of this channel's accumulators (REGISTERS: all indices are
// compile-time constants after inlining).
template <int GS = 3 /* stride of gsh */>
__device__ __forceinline__ void sh_backward_channel(int deg, const float *sh, float *gsh, float g, float x, float y,
                                                    float z, float &ddx, float &ddy, float &ddz) {
    gsh[0 * GS] += GS_SH_C0 * g;
    if (deg < 1) return;
    gsh[1 * GS] += -GS_SH_C1 * y * g;
    gsh[2 * GS] += GS_SH_C1 * z * g;
    gsh[3 * GS] += -GS_SH_C1 * x * g;
    float dx_ = -GS_SH_C1 * sh[3 * 3], dy_ = -GS_SH_C1 * sh[1 * 3], dz_ = GS_SH_C1 * sh[2 * 3];
    if (deg > 1) {
        const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
        gsh[4 * GS] += GS_SH_C2_0 * xy * g;
        gsh[5 * GS] += GS_SH_C2_1 * yz * g;
        gsh[6 * GS] += GS_SH_C2_2 * (2.0f * zz - xx - yy) * g;
        gsh[7 * GS] += GS_SH_C2_3 * xz * g;
        gsh[8 * GS] += GS_SH_C2_4 * (xx - yy) * g;
        dx_ += GS_SH_C2_0 * y * sh[4 * 3] + GS_SH_C2_2 * 2.0f * -x * sh[6 * 3] + GS_SH_C2_3 * z * sh[7 * 3] +
               GS_SH_C2_4 * 2.0f * x * sh[8 * 3];
        dy_ += GS_SH_C2_0 * x * sh[4 * 3] + GS_SH_C2_1 * z * sh[5 * 3] + GS_SH_C2_2 * 2.0f * -y * sh[6 * 3] +
               GS_SH_C2_4 * 2.0f * -y * sh[8 * 3];
        dz_ += GS_SH_C2_1 * y * sh[5 * 3] + GS_SH_C2_2 * 4.0f * z * sh[6 * 3] + GS_SH_C2_3 * x * sh[7 * 3];
        if (deg > 2) {
            gsh[9 * GS] += GS_SH_C3_0 * y * (3.0f * xx - yy) * g;
            gsh[10 * GS] += GS_SH_C3_1 * xy * z * g;
            gsh[11 * GS] += GS_SH_C3_2 * y * (4.0f * zz - xx - yy) * g;
            gsh[12 * GS] += GS_SH_C3_3 * z * (2.0f * zz - 3.0f * xx - 3.0f * yy) * g;
            gsh[13 * GS] += GS_SH_C3_4 * x * (4.0f * zz - xx - yy) * g;
            gsh[14 * GS] += GS_SH_C3_5 * z * (xx - yy) * g;
            gsh[15 * GS] += GS_SH_C3_6 * x * (xx - 3.0f * yy) * g;
            dx_ += GS_SH_C3_0 * sh[9 * 3] * 6.0f * xy + GS_SH_C3_1 * sh[10 * 3] * yz +
                   GS_SH_C3_2 * sh[11 * 3] * -2.0f * xy + GS_SH_C3_3 * sh[12 * 3] * -6.0f * xz +
                   GS_SH_C3_4 * sh[13 * 3] * (-3.0f * xx + 4.0f * zz - yy) + GS_SH_C3_5 * sh[14 * 3] * 2.0f * xz +
                   GS_SH_C3_6 * sh[15 * 3] * 3.0f * (xx - yy);
            dy_ += GS_SH_C3_0 * sh[9 * 3] * 3.0f * (xx - yy) + GS_SH_C3_1 * sh[10 * 3] * xz +
                   GS_SH_C3_2 * sh[11 * 3] * (-3.0f * yy + 4.0f * zz - xx) + GS_SH_C3_3 * sh[12 * 3] * -6.0f * yz +
                   GS_SH_C3_4 * sh[13 * 3] * -2.0f * xy + GS_SH_C3_5 * sh[14 * 3] * -2.0f * yz +
                   GS_SH_C3_6 * sh[15 * 3] * -6.0f * xy;
            dz_ += GS_SH_C3_1 * sh[10 * 3] * xy + GS_SH_C3_2 * sh[11 * 3] * 8.0f * yz +
                   GS_SH_C3_3 * sh[12 * 3] * 3.0f * (2.0f * zz - xx - yy) + GS_SH_C3_4 * sh[13 * 3] * 8.0f * xz +
                   GS_SH_C3_5 * sh[14 * 3] * (xx - yy);
        }
    }
    ddx += dx_ * g;
    ddy += dy_ * g;
    ddz += dz_ * g;
}

// Band 4 (degree-4 kernels only): dL/dsh_k += basis_k(dir) * g_ch for k = 16..24 and all three channels, and band 4's
// share of dL/ddir.  sh: this Gaussian's staged [M][3] row; g4: its [9][3] band-4 accumulators in SHARED memory (see
// k_preprocess_bwd).  Same polynomial forms as eval_sh (gs_preprocess.cu); their partial derivatives in x, y, z taken as
// independent variables (the "-1" / "-3" forms differ from homogeneous ones only along dir, which the normalisation
// projects out).
__device__ __forceinline__ void sh_backward_band4(const float *sh, float *g4, const float g[3], float x, float y, float z,
                                                  float &ddx, float &ddy, float &ddz) {
    const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
    const float xx_yy = xx - yy, xx3_yy = 3.0f * xx - yy, xx_3yy = xx - 3.0f * yy;
    const float zz7m1 = 7.0f * zz - 1.0f, zz7m3 = 7.0f * zz - 3.0f, zz21m3 = 21.0f * zz - 3.0f;
    // basis value and its partials (d/dx, d/dy, d/dz) per coefficient 16 + k
    const float B[9] = {GS_SH_C4_0 * xy * xx_yy, GS_SH_C4_1 * yz * xx3_yy, GS_SH_C4_2 * xy * zz7m1,
                        GS_SH_C4_3 * yz * zz7m3, GS_SH_C4_4 * (zz * (35.0f * zz - 30.0f) + 3.0f), GS_SH_C4_5 * xz * zz7m3,
                        GS_SH_C4_6 * xx_yy * zz7m1, GS_SH_C4_7 * xz * xx_3yy,
                        GS_SH_C4_8 * (xx * xx_3yy - yy * xx3_yy)};
    const float DX[9] = {GS_SH_C4_0 * y * xx3_yy, GS_SH_C4_1 * 6.0f * x * yz, GS_SH_C4_2 * y * zz7m1, 0.0f, 0.0f,
                         GS_SH_C4_5 * z * zz7m3, GS_SH_C4_6 * 2.0f * x * zz7m1, GS_SH_C4_7 * 3.0f * z * xx_yy,
                         GS_SH_C4_8 * 4.0f * x * xx_3yy};
    const float DY[9] = {GS_SH_C4_0 * x * xx_3yy, GS_SH_C4_1 * 3.0f * z * xx_yy, GS_SH_C4_2 * x * zz7m1,
                         GS_SH_C4_3 * z * zz7m3, 0.0f, 0.0f, GS_SH_C4_6 * -2.0f * y * zz7m1, GS_SH_C4_7 * -6.0f * x * yz,
                         GS_SH_C4_8 * -4.0f * y * xx3_yy};
    const float DZ[9] = {0.0f, GS_SH_C4_1 * y * xx3_yy, GS_SH_C4_2 * 14.0f * xy * z, GS_SH_C4_3 * y * zz21m3,
                         GS_SH_C4_4 * z * (140.0f * zz - 60.0f), GS_SH_C4_5 * x * zz21m3, GS_SH_C4_6 * 14.0f * z * xx_yy,
                         GS_SH_C4_7 * x * xx_3yy, 0.0f};
    float dx_ = 0.f, dy_ = 0.f, dz_ = 0.f;
#pragma unroll
    for (int k = 0; k < 9; k++) {
#pragma unroll
        for (int ch = 0; ch < 3; ch++) {
            g4[k * 3 + ch] += B[k] * g[ch];
            const float w = sh[(16 + k) * 3 + ch] * g[ch];
            dx_ += DX[k] * w;
            dy_ += DY[k] * w;
            dz_ += DZ[k] * w;
        }
    }
    ddx += dx_;
    ddy += dy_;
    ddz += dz_;
}

// Per-view gradients (the depth channel's z column, the camera gradient) are sums over the Gaussians of a scene.  Each
// warp adds up its lanes' terms with a butterfly over the 32 lanes.  Every lane of the warp must make the same sequence of
// calls for the same view (inactive lanes with zeros); the calls may sit at different points of the code (shfl.sync on
// sm_70 and later).
template <int N>
__device__ __forceinline__ void warp_sum(float (&x)[N]) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
#pragma unroll
        for (int k = 0; k < N; k++) x[k] += __shfl_xor_sync(0xffffffffu, x[k], off);
    }
}

// The warp's sum of x goes with plain stores to components [c0, c0 + N) of its own slot of slots[V][warps of the scene's
// grid][NC], which a finalize kernel adds up in a fixed order: deterministic, and free of same-address atomics.
// N, c0 and NC are multiples of 4.
template <int NC, int N>
__device__ __forceinline__ void view_partial(float *slots, int v, int c0, float (&x)[N]) {
    static_assert(N % 4 == 0 && NC % 4 == 0, "slots are written in float4s");
    warp_sum(x);
    if ((threadIdx.x & 31) == 0) {
        const size_t warps = (size_t)gridDim.x * (PB_THREADS / 32);
        const size_t w = (size_t)blockIdx.x * (PB_THREADS / 32) + (threadIdx.x >> 5);
        float4 *dst = reinterpret_cast<float4 *>(slots + ((size_t)v * warps + w) * NC + c0);
#pragma unroll
        for (int k = 0; k < N / 4; k++) dst[k] = make_float4(x[4 * k], x[4 * k + 1], x[4 * k + 2], x[4 * k + 3]);
    }
}

// dL/d(view matrix entries 2, 6, 10, 14) of one view += the warp's sum of (gz * m, gz): warp_sum's butterfly written out
// for four scalars (the array form allocates registers differently in the kernels that exist without the camera
// gradient), then one RED per component from lane 0.  Same calling rules as warp_sum.
__device__ __forceinline__ void red_view_z_grad(float *dst, float a, float b, float c, float d) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, off);
        b += __shfl_xor_sync(0xffffffffu, b, off);
        c += __shfl_xor_sync(0xffffffffu, c, off);
        d += __shfl_xor_sync(0xffffffffu, d, off);
    }
    if ((threadIdx.x & 31) == 0) {
        atomicAdd(dst + 0, a);
        atomicAdd(dst + 1, b);
        atomicAdd(dst + 2, c);
        atomicAdd(dst + 3, d);
    }
}

// Deterministic mode: the warp's sum goes to its own slot of det.view_z ([V][warps of the scene's grid][4]) with a
// plain store, as view_partial<4> would, and k_view_z_finalize adds the slots up in warp order.  This and
// red_view_z_grad are warp_sum / view_partial written out for four scalars: the three must stay in step.
template <bool DET>
__device__ __forceinline__ void view_z_grad(const GsInGrads &g, const DetAcc &det, int v, float a, float b, float c,
                                            float d) {
    if constexpr (DET) {
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            a += __shfl_xor_sync(0xffffffffu, a, off);
            b += __shfl_xor_sync(0xffffffffu, b, off);
            c += __shfl_xor_sync(0xffffffffu, c, off);
            d += __shfl_xor_sync(0xffffffffu, d, off);
        }
        if ((threadIdx.x & 31) == 0) {
            const size_t warps = (size_t)gridDim.x * (PB_THREADS / 32);
            const size_t w = (size_t)blockIdx.x * (PB_THREADS / 32) + (threadIdx.x >> 5);
            reinterpret_cast<float4 *>(det.view_z)[(size_t)v * warps + w] = make_float4(a, b, c, d);
        }
    } else {
        red_view_z_grad(g.dL_dviewmatrix_z + (size_t)v * 4, a, b, c, d);
    }
}

// Camera gradient (GsCameraGrads): 29 terms per (view, Gaussian) pair in the slots of det.view_z, [V][warps][GS_CAM_NC]:
//   0..11  dL/dviewmatrix[4k + r] at component 3k + r (k = 0..3, r = 0..2; the fourth column is never read)
//   12..23 dL/dprojmatrix[4k + c] at component 12 + 3k + i, c = (0, 1, 3)[i] (the third column feeds no output)
//   24..26 dL/dcampos, 27..28 dL/dtanfov (x, y), 29..31 zero (one component per lane of k_camera_finalize)
// Each of the three groups is reduced where it is computed, which keeps few of the terms live at once.
constexpr int GS_CAM_NC = 32;

// the three partials of a pair that adds nothing (same calls as a visible pair makes)
__device__ __forceinline__ void cam_partial_zero(float *slots, int v) {
    float z12[12] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    view_partial<GS_CAM_NC>(slots, v, 0, z12);
    float z12b[12] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    view_partial<GS_CAM_NC>(slots, v, 12, z12b);
    float z8[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    view_partial<GS_CAM_NC>(slots, v, 24, z8);
}

// VIEW_Z = 2 kernels: the depth channel carried f(z) of dm.mode, so the accumulated gz = sum alpha T dL/ddepth is dL/df,
// and f'(z) dz/dz_s (this factor) carries it onto the view-scaled depth z_s, recomputed exactly as preprocess computed it.
__device__ __forceinline__ float depth_chain(const ViewCam &cam, float3 mean, const DepthMode &dm, int v) {
    const float s = cam.scale;
    const float zs = xform4x3(cam.view, make_float3(mean.x * s, mean.y * s, mean.z * s)).z;
    const float nr = dm.near_far ? dm.near_far[v * 2] : 0.f, fr = dm.near_far ? dm.near_far[v * 2 + 1] : 0.f;
    return gs_depth_chain(dm.mode, zs, s, nr, fr);
}

// The decoded fixed-point accumulators of (view, Gaussian) o (deterministic mode), written to out; returns out.
__device__ __forceinline__ const float *load_det_acc(const DetAcc &det, size_t o, float out[GS_ACC_STRIDE]) {
    const uint32_t bad = det.poison[o];
    const long long *l = reinterpret_cast<const long long *>(det.acc) + o * GS_ACC_STRIDE * GS_DET_LIMBS;
#pragma unroll
    for (int k = 0; k < GS_ACC_STRIDE; k++) out[k] = gs_det_decode(l + k * GS_DET_LIMBS, (bad >> k) & 1u);
    return out;
}

// VIEW_Z: 1 also write g.dL_dviewmatrix_z, the depth channel's gradient w.r.t. the z column of each view matrix
// (z = view[2] m.x + view[6] m.y + view[10] m.z + view[14], m the view-scaled mean).  The default instantiations
// (VIEW_Z = 0) are the kernels without it, instruction for instruction.  2: the forward's depth mode was not GS_DEPTH_Z --
// the depth gradient is chained through f'(z) of dm.mode, and the view-matrix gradient is written if g asks for it.
// DET: the accumulators are the fixed-point ones of the deterministic backward (det.acc, det.poison) and the view-matrix
// gradient goes through det.view_z.
// B4: degree 4 (c.deg == 4, M >= 25).  The 48 accumulators of bands 0..3 stay in registers as in the default kernel; the
// 27 of band 4 live in a shared-memory row per thread next to the staged inputs (stride 27, odd: conflict-free), which
// keeps the register bound -- and so the 4 resident CTAs per SM -- of the default kernel.
// AA: the forward ran with GS_FLAG_ANTIALIAS and drew opacity o' = o rho (gs_aa_rho), so the accumulated dL/dopacity is
// dL/do'.  rho is recomputed from the rebuilt 2-D covariance: dL/do = sum_v rho_v dL/do'_v, and o dL/do' drho/d(a0, b, c0)
// joins dL/d(a, b, c) ahead of the cov2D -> cov3D and cov2D -> J -> mean chains (DESIGN.md 5.5).  The AA = false kernels
// are the ones without it, instruction for instruction.
// CAM: also the camera gradient (GsCameraGrads), into the slots of det.view_z (GS_CAM_NC components, in both modes), which
// k_camera_finalize turns into dL/dviewmatrix, dL/dprojmatrix, dL/dcampos and dL/dtanfov (DESIGN.md 5.5).  Never
// with VIEW_Z = 1: the full gradient contains the z column.  The CAM = false kernels are the ones without it.
template <bool HAS_SH, int MINB, int VIEW_Z = 0, bool DET = false, bool B4 = false, bool AA = false, bool CAM = false>
__global__ void __launch_bounds__(PB_THREADS, MINB)
k_preprocess_bwd(const DevCfg c, const DevInputs in, const uint8_t *__restrict__ meta, const float *__restrict__ acc,
                    const GsInGrads g, const DetAcc det, const DepthMode dm) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    PbSmem *sm = reinterpret_cast<PbSmem *>(smem_raw);
    float *sh_s = reinterpret_cast<float *>(smem_raw + PB_SMEM_HDR);
    // B4: this thread's band-4 accumulators, behind the staged block of PB_THREADS rows
    float *g4 = B4 ? sh_s + (size_t)PB_THREADS * c.M * 3 + (size_t)threadIdx.x * PB_SH_B4 : nullptr;
    if constexpr (B4) {
#pragma unroll
        for (int k = 0; k < PB_SH_B4; k++) g4[k] = 0.f;
    }

    const int scene = blockIdx.y;
    const int g0 = blockIdx.x * PB_THREADS;
    const int n = min(PB_THREADS, c.P - g0);
    const int tid = threadIdx.x;
    const int i = g0 + tid;
    const bool active = tid < n;
    const size_t sg = (size_t)scene * c.P + i;
    const uint32_t sh_floats = (uint32_t)n * c.M * 3u;

    bool bulk = false;
    if (HAS_SH) {
        const float *src = in.shs + ((size_t)scene * c.P + g0) * c.M * 3;
        const float *dst = g.dL_dshs ? g.dL_dshs + ((size_t)scene * c.P + g0) * c.M * 3 : nullptr;
        bulk = ((reinterpret_cast<uintptr_t>(src) & 15u) == 0) && (((sh_floats * 4u) & 15u) == 0) &&
               ((reinterpret_cast<uintptr_t>(dst) & 15u) == 0);
        if (bulk) {
            if (tid == 0) {
                mbar_init(&sm->bar, 1);
                mbar_fence_init();
                mbar_expect_tx(&sm->bar, sh_floats * 4u);
                tma_load_1d(sh_s, src, sh_floats * 4u, &sm->bar);
            }
        } else {
            for (uint32_t k = tid; k < sh_floats; k += PB_THREADS) sh_s[k] = src[k];
        }
    }
    float gsh[PB_SH_EVAL * 3];
#pragma unroll
    for (int k = 0; k < PB_SH_EVAL * 3; k++) gsh[k] = 0.f;

    float3 mean = make_float3(0, 0, 0);
    float c6[6] = {0, 0, 0, 0, 0, 0};
    float sc[3] = {0, 0, 0}, q[4] = {0, 0, 0, 0};
    float opac = 0.f;   // AA only: the scene-level opacity o
    if (active) {
        mean = make_float3(in.means3D[sg * 3 + 0], in.means3D[sg * 3 + 1], in.means3D[sg * 3 + 2]);
        if constexpr (AA) opac = in.opacities[sg];
        if (in.cov3D) {
#pragma unroll
            for (int k = 0; k < 6; k++) c6[k] = in.cov3D[sg * 6 + k];
        } else {
#pragma unroll
            for (int k = 0; k < 3; k++) sc[k] = in.scales[sg * 3 + k];
#pragma unroll
            for (int k = 0; k < 4; k++) q[k] = in.rotations[sg * 4 + k];
            cov3d_from_scale_rot(sc, c.scale_modifier, q, c6);
        }
    }
    if (HAS_SH) {
        __syncthreads();
        if (bulk) mbar_wait(&sm->bar, 0);
    }

    float gmean[3] = {0, 0, 0}, gcov[6] = {0, 0, 0, 0, 0, 0}, gopac = 0.f;

    for (int vi = 0; vi < c.VPS; vi++) {
        const int v = scene * c.VPS + vi;
        if (vi % GS_CAM_CHUNK == 0) {
            __syncthreads();
            load_view_cams(c, v, min(GS_CAM_CHUNK, c.VPS - vi), sm->cams);
            __syncthreads();
        }
        if (!active) {
            if (VIEW_Z == 1 || (VIEW_Z == 2 && g.dL_dviewmatrix_z)) view_z_grad<DET>(g, det, v, 0.f, 0.f, 0.f, 0.f);
            if constexpr (CAM) cam_partial_zero(det.view_z, v);
            continue;
        }
        const ViewCam &cam = sm->cams[vi % GS_CAM_CHUNK];
        const size_t o = (size_t)v * c.P + i;
        const uint32_t mb = meta[o];
        float m2d[2] = {0.f, 0.f}, gcol[3] = {0.f, 0.f, 0.f};
        if ((VIEW_Z == 1 || (VIEW_Z == 2 && g.dL_dviewmatrix_z)) && !(mb & GS_META_VISIBLE)) view_z_grad<DET>(g, det, v, 0.f, 0.f, 0.f, 0.f);
        if constexpr (CAM) {
            if (!(mb & GS_META_VISIBLE)) cam_partial_zero(det.view_z, v);
        }
        if (mb & GS_META_VISIBLE) {
            const float *a = acc + o * GS_ACC_STRIDE;
            float a_det[GS_ACC_STRIDE];
            if constexpr (DET) a = load_det_acc(det, o, a_det);
            gcol[0] = a[0]; gcol[1] = a[1]; gcol[2] = a[2];
            m2d[0] = a[3]; m2d[1] = a[4];
            const float gcx = a[5], gcy = a[6], gcz = a[7];
            if constexpr (!AA) gopac += a[8];
            const float gz = VIEW_Z == 2 ? a[9] * depth_chain(cam, mean, dm, v) : a[9];
            const float s = cam.scale, s2 = s * s;
            const float3 m = make_float3(mean.x * s, mean.y * s, mean.z * s);
            const float cv[6] = {c6[0] * s2, c6[1] * s2, c6[2] * s2, c6[3] * s2, c6[4] * s2, c6[5] * s2};
            float gm[3] = {0.f, 0.f, 0.f};  // dL/dm (view-scaled mean)
            // CAM: components 24..31 of the slot: dL/dcampos = -dL/dd (d = m - campos), then dL/dtanfov
            float gcp[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            // ---- conic -> cov2D -> cov3D, mean (through J) ----
            {
                ProjJac j;
                build_jac(cam, c, m, j);
                float s0[3], s1[3];
                sym6_mul(cv, j.m0, s0);
                sym6_mul(cv, j.m1, s1);
                const float aa = j.m0[0] * s0[0] + j.m0[1] * s0[1] + j.m0[2] * s0[2] + c.dilation;
                const float bb = j.m0[0] * s1[0] + j.m0[1] * s1[1] + j.m0[2] * s1[2];
                const float cc = j.m1[0] * s1[0] + j.m1[1] * s1[1] + j.m1[2] * s1[2] + c.dilation;
                const float denom = aa * cc - bb * bb;
                const float d2inv = 1.0f / (denom * denom + 0.0000001f);
                float dL_da = 0.f, dL_db = 0.f, dL_dc = 0.f;
                // AA: rho as preprocess computed it, and the factor k = o dL/do' h / (2 rho det1^2) of its derivatives
                float aa_k = 0.f, a0 = 0.f, c0 = 0.f;
                if constexpr (AA) {
                    a0 = j.m0[0] * s0[0] + j.m0[1] * s0[1] + j.m0[2] * s0[2];
                    c0 = j.m1[0] * s1[0] + j.m1[1] * s1[1] + j.m1[2] * s1[2];
                    const float ratio = gs_aa_ratio(a0, bb, c0, denom);
                    const float rho = gs_aa_rho(ratio);
                    gopac += rho * a[8];
                    // below the clamp rho is a constant
                    if (ratio > GS_AA_RATIO_MIN) aa_k = opac * a[8] * c.dilation / (2.0f * rho * denom * denom);
                }
                if (d2inv != 0.0f) {
                    dL_da = d2inv * (-cc * cc * gcx + 2.0f * bb * cc * gcy + (denom - aa * cc) * gcz);
                    dL_dc = d2inv * (-aa * aa * gcz + 2.0f * aa * bb * gcy + (denom - aa * cc) * gcx);
                    dL_db = d2inv * 2.0f * (bb * cc * gcx - (denom + 2.0f * bb * bb) * gcy + aa * bb * gcz);
                    if constexpr (AA) {
                        // ratio = det0 / det1: d/da0 = h (c0 cc + b^2) / det1^2, d/dc0 = h (a0 aa + b^2) / det1^2,
                        // d/db = -2 b h (aa + c0) / det1^2 (aa = a0 + h, cc = c0 + h)
                        dL_da += aa_k * (c0 * cc + bb * bb);
                        dL_dc += aa_k * (a0 * aa + bb * bb);
                        dL_db -= 2.0f * aa_k * bb * (aa + c0);
                    }
                    const float *m0 = j.m0, *m1 = j.m1;
                    gcov[0] += s2 * (m0[0] * m0[0] * dL_da + m0[0] * m1[0] * dL_db + m1[0] * m1[0] * dL_dc);
                    gcov[3] += s2 * (m0[1] * m0[1] * dL_da + m0[1] * m1[1] * dL_db + m1[1] * m1[1] * dL_dc);
                    gcov[5] += s2 * (m0[2] * m0[2] * dL_da + m0[2] * m1[2] * dL_db + m1[2] * m1[2] * dL_dc);
                    gcov[1] += s2 * (2.0f * m0[0] * m0[1] * dL_da + (m0[0] * m1[1] + m0[1] * m1[0]) * dL_db +
                                     2.0f * m1[0] * m1[1] * dL_dc);
                    gcov[2] += s2 * (2.0f * m0[0] * m0[2] * dL_da + (m0[0] * m1[2] + m0[2] * m1[0]) * dL_db +
                                     2.0f * m1[0] * m1[2] * dL_dc);
                    gcov[4] += s2 * (2.0f * m0[2] * m0[1] * dL_da + (m0[1] * m1[2] + m0[2] * m1[1]) * dL_db +
                                     2.0f * m1[1] * m1[2] * dL_dc);
                }
                float dJ00 = 0.f, dJ02 = 0.f, dJ11 = 0.f, dJ12 = 0.f;
                float gw0[3], gw1[3];   // CAM: dL/d(rows of T = J W), kept for the view matrix's W
#pragma unroll
                for (int k = 0; k < 3; k++) {
                    const float gm0 = 2.0f * dL_da * s0[k] + dL_db * s1[k];
                    const float gm1 = 2.0f * dL_dc * s1[k] + dL_db * s0[k];
                    if constexpr (CAM) { gw0[k] = gm0; gw1[k] = gm1; }
                    dJ00 += gm0 * cam.view[k * 4 + 0];
                    dJ02 += gm0 * cam.view[k * 4 + 2];
                    dJ11 += gm1 * cam.view[k * 4 + 1];
                    dJ12 += gm1 * cam.view[k * 4 + 2];
                }
                const float tz = 1.0f / j.tz, tz2 = tz * tz, tz3 = tz2 * tz;
                const float dtx = j.xin ? -j.fx * tz2 * dJ02 : 0.0f;
                const float dty = j.yin ? -j.fy * tz2 * dJ12 : 0.0f;
                const float dtz = -j.fx * tz2 * dJ00 - j.fy * tz2 * dJ11 + (2.0f * j.fx * j.tx) * tz3 * dJ02 +
                                  (2.0f * j.fy * j.ty) * tz3 * dJ12;
#pragma unroll
                for (int k = 0; k < 3; k++)
                    gm[k] += cam.view[k * 4 + 0] * dtx + cam.view[k * 4 + 1] * dty + cam.view[k * 4 + 2] * dtz;
                if constexpr (CAM) {
                    // t = W m + view[12..14]: dL/dview[4k + r] = dL/dt_r m_k, with the depth channel's gz on t.z; and
                    // T = J W: dL/dW[r][k] = sum_i J[i][r] dL/dT[i][k] (J01 = J10 = 0)
                    const float J00 = j.fx * tz, J11 = j.fy * tz, J02 = -j.fx * j.tx * tz2, J12 = -j.fy * j.ty * tz2;
                    const float dt[3] = {dtx, dty, dtz + gz}, mk[3] = {m.x, m.y, m.z};
                    float cv[12];
#pragma unroll
                    for (int k = 0; k < 3; k++) {
                        cv[3 * k + 0] = dt[0] * mk[k] + J00 * gw0[k];
                        cv[3 * k + 1] = dt[1] * mk[k] + J11 * gw1[k];
                        cv[3 * k + 2] = dt[2] * mk[k] + J02 * gw0[k] + J12 * gw1[k];
                    }
                    cv[9] = dt[0]; cv[10] = dt[1]; cv[11] = dt[2];
                    view_partial<GS_CAM_NC>(det.view_z, v, 0, cv);
                    // fx = W / (2 tanfovx) scales J00 and J02, so dL/dtanfovx = -(dL/dJ00 J00 + dL/dJ02 J02) / tanfovx;
                    // a clamped t.x = +-guard_band tanfovx t.z makes J02 independent of tanfovx and drops its term
                    // (y likewise)
                    gcp[3] = -(dJ00 * J00 + (j.xin ? dJ02 * J02 : 0.0f)) / cam.tanfovx;
                    gcp[4] = -(dJ11 * J11 + (j.yin ? dJ12 * J12 : 0.0f)) / cam.tanfovy;
                }
            }
            // ---- mean2D (NDC units) -> mean through the perspective divide ----
            {
                const float4 mh = xform4x4(cam.proj, m);
                const float mw = 1.0f / (mh.w + 0.0000001f);
                const float mul1 = mh.x * mw * mw, mul2 = mh.y * mw * mw;
                const float *pr = cam.proj;
                gm[0] += (pr[0] * mw - pr[3] * mul1) * m2d[0] + (pr[1] * mw - pr[3] * mul2) * m2d[1];
                gm[1] += (pr[4] * mw - pr[7] * mul1) * m2d[0] + (pr[5] * mw - pr[7] * mul2) * m2d[1];
                gm[2] += (pr[8] * mw - pr[11] * mul1) * m2d[0] + (pr[9] * mw - pr[11] * mul2) * m2d[1];
                if constexpr (CAM) {
                    // mh = Pf m + Pf[12..15]: dL/dPf[4k + c] = dL/dmh_c m_k for c = x, y, w (mh.z feeds no output)
                    const float dmh[3] = {m2d[0] * mw, m2d[1] * mw, -(mul1 * m2d[0] + mul2 * m2d[1])};
                    const float mk[3] = {m.x, m.y, m.z};
                    float cp[12];
#pragma unroll
                    for (int k = 0; k < 3; k++) {
#pragma unroll
                        for (int i2 = 0; i2 < 3; i2++) cp[3 * k + i2] = dmh[i2] * mk[k];
                    }
                    cp[9] = dmh[0]; cp[10] = dmh[1]; cp[11] = dmh[2];
                    view_partial<GS_CAM_NC>(det.view_z, v, 12, cp);
                }
            }
            // ---- fused depth channel: z = (view * m).z ----
            gm[0] += cam.view[2] * gz;
            gm[1] += cam.view[6] * gz;
            gm[2] += cam.view[10] * gz;
            if (VIEW_Z == 1 || (VIEW_Z == 2 && g.dL_dviewmatrix_z)) view_z_grad<DET>(g, det, v, gz * m.x, gz * m.y, gz * m.z, gz);
            // ---- colour -> SH coefficients and mean (view direction) ----
            if (HAS_SH) {
                const float d[3] = {m.x - cam.campos[0], m.y - cam.campos[1], m.z - cam.campos[2]};
                const float len2 = d[0] * d[0] + d[1] * d[1] + d[2] * d[2];
                const float inv = 1.0f / sqrtf(len2);
                const float x = d[0] * inv, y = d[1] * inv, z = d[2] * inv;
                float ddx = 0.f, ddy = 0.f, ddz = 0.f;
                const float *sh = sh_s + (size_t)tid * c.M * 3;
#pragma unroll
                for (int ch = 0; ch < 3; ch++) {
                    const float gch = (mb & (1u << ch)) ? 0.0f : gcol[ch];
                    sh_backward_channel(c.deg, sh + ch, gsh + ch, gch, x, y, z, ddx, ddy, ddz);
                }
                if constexpr (B4) {
                    const float g3[3] = {(mb & 1u) ? 0.0f : gcol[0], (mb & 2u) ? 0.0f : gcol[1], (mb & 4u) ? 0.0f : gcol[2]};
                    sh_backward_band4(sh, g4, g3, x, y, z, ddx, ddy, ddz);
                }
                const float dot = d[0] * ddx + d[1] * ddy + d[2] * ddz;
                const float inv3 = inv * inv * inv;
                if constexpr (CAM) {
                    gcp[0] = -(ddx * len2 - d[0] * dot) * inv3;
                    gcp[1] = -(ddy * len2 - d[1] * dot) * inv3;
                    gcp[2] = -(ddz * len2 - d[2] * dot) * inv3;
                }
                gm[0] += (ddx * len2 - d[0] * dot) * inv3;
                gm[1] += (ddy * len2 - d[1] * dot) * inv3;
                gm[2] += (ddz * len2 - d[2] * dot) * inv3;
            }
            if constexpr (CAM) view_partial<GS_CAM_NC>(det.view_z, v, 24, gcp);
#pragma unroll
            for (int k = 0; k < 3; k++) gmean[k] += s * gm[k];
        }
        if (g.dL_dmeans2D) {
            g.dL_dmeans2D[o * 3 + 0] = m2d[0];
            g.dL_dmeans2D[o * 3 + 1] = m2d[1];
            g.dL_dmeans2D[o * 3 + 2] = 0.0f;
        }
        if (g.dL_dcolors) {
            g.dL_dcolors[o * 3 + 0] = gcol[0];
            g.dL_dcolors[o * 3 + 1] = gcol[1];
            g.dL_dcolors[o * 3 + 2] = gcol[2];
        }
    }

    if (active) {
        if (g.dL_dmeans3D) {
#pragma unroll
            for (int k = 0; k < 3; k++) g.dL_dmeans3D[sg * 3 + k] = gmean[k];
        }
        if (g.dL_dopacities) g.dL_dopacities[sg] = gopac;
        if (in.cov3D) {
            if (g.dL_dcov3D) {
#pragma unroll
                for (int k = 0; k < 6; k++) g.dL_dcov3D[sg * 6 + k] = gcov[k];
            }
        } else {
            // Sigma = R diag(v) R^T, v_k = (mod*s_k)^2 : dL/dv_k = (R^T G R)_kk ; dL/dR = 2 G R diag(v)
            float R[3][3];
            quat_to_R(q, R);
            const float G[3][3] = {{gcov[0], 0.5f * gcov[1], 0.5f * gcov[2]},
                                   {0.5f * gcov[1], gcov[3], 0.5f * gcov[4]},
                                   {0.5f * gcov[2], 0.5f * gcov[4], gcov[5]}};
            const float mod = c.scale_modifier;
            float dR[3][3];
#pragma unroll
            for (int k = 0; k < 3; k++) {
                const float sv = mod * sc[k];
                float GRk[3];
#pragma unroll
                for (int a = 0; a < 3; a++) GRk[a] = G[a][0] * R[0][k] + G[a][1] * R[1][k] + G[a][2] * R[2][k];
                const float dv = R[0][k] * GRk[0] + R[1][k] * GRk[1] + R[2][k] * GRk[2];
                if (g.dL_dscales) g.dL_dscales[sg * 3 + k] = dv * 2.0f * sv * mod;
#pragma unroll
                for (int a = 0; a < 3; a++) dR[a][k] = 2.0f * GRk[a] * sv * sv;
            }
            if (g.dL_drotations) {
                const float r = q[0], x = q[1], y = q[2], z = q[3];
                float *gq = g.dL_drotations + sg * 4;
                gq[0] = 2.0f * (-z * dR[0][1] + y * dR[0][2] + z * dR[1][0] - x * dR[1][2] - y * dR[2][0] + x * dR[2][1]);
                gq[1] = 2.0f * (y * dR[0][1] + z * dR[0][2] + y * dR[1][0] - 2.0f * x * dR[1][1] - r * dR[1][2] +
                                z * dR[2][0] + r * dR[2][1] - 2.0f * x * dR[2][2]);
                gq[2] = 2.0f * (-2.0f * y * dR[0][0] + x * dR[0][1] + r * dR[0][2] + x * dR[1][0] + z * dR[1][2] -
                                r * dR[2][0] + z * dR[2][1] - 2.0f * y * dR[2][2]);
                gq[3] = 2.0f * (-2.0f * z * dR[0][0] - r * dR[0][1] + x * dR[0][2] + r * dR[1][0] - 2.0f * z * dR[1][1] +
                                y * dR[1][2] + x * dR[2][0] + y * dR[2][1]);
            }
        }
    }

    if (HAS_SH && g.dL_dshs) {
        // the staged input block is dead now: overwrite it with the gradient block (zeros beyond the evaluated
        // bands) and send it out with one bulk store
        float *dst = g.dL_dshs + ((size_t)scene * c.P + g0) * c.M * 3;
        __syncthreads();  // every thread has finished reading sh_s
        if (active) {
            float *row = sh_s + (size_t)tid * c.M * 3;
            const int used = min(c.M, PB_SH_EVAL) * 3;
#pragma unroll
            for (int k = 0; k < PB_SH_EVAL * 3; k++)
                if (k < used) row[k] = gsh[k];
            if constexpr (B4) {   // M >= 25: band 4 follows from the shared accumulators, zeros beyond it
#pragma unroll
                for (int k = 0; k < PB_SH_B4; k++) row[PB_SH_EVAL * 3 + k] = g4[k];
                for (int k = PB_SH_EVAL * 3 + PB_SH_B4; k < c.M * 3; k++) row[k] = 0.f;
            } else {
                for (int k = used; k < c.M * 3; k++) row[k] = 0.f;
            }
        }
        if (bulk) {
            fence_proxy_async_smem();  // make the generic-proxy smem writes visible to the TMA engine
            __syncthreads();
            if (tid == 0) {
                tma_store_1d(dst, sh_s, sh_floats * 4u);
                tma_store_commit_wait();
            }
        } else {
            __syncthreads();
            for (uint32_t k = tid; k < sh_floats; k += PB_THREADS) dst[k] = sh_s[k];
        }
    }
}


// ---------------------------------------------------------------------------------------------------------
// Round-2 experiment (GS_TUNE_PBWD_2PHASE; measured SLOWER, kept for the A/B): two phases per thread instead of one
// ---------------------------------------------------------------------------------------------------------
// v1 carried the 48 SH-gradient accumulators through the whole geometry chain: 150 registers unbounded, 128 bounded,
// low occupancy (latency-bound).  The SH gradient is linear in (basis(dir_v) x dL/dcolour_v)
// and touches the rest of the backward only through dL/ddir, so the loop over the views is run four times with a small
// live state each time:
//   phase G   conic -> cov2D -> cov3D / mean, mean2D -> mean, depth -> mean            (no SH state at all)
//   phase S_c for each colour channel c: 16 accumulators; the channel's 16 staged INPUT coefficients are dead once its
//             loop over the views is done and are overwritten in place by its gradients
// Only the 16 coefficients per channel the evaluator can touch are staged (192 instead of 300 bytes per thread).  The
// gradient rows leave by ONE bulk TMA store when M <= 16, else by coalesced stores that append the zero bands.
// Result on C2: 80 registers instead of 128 and higher occupancy -- but about 1.5x the warp-instructions (the per-view
// camera / direction / basis work is redone per phase), and slower.  The single-pass kernel stays the default.
constexpr int PB2_MIN_CTAS = 6;

template <bool HAS_SH, int VIEW_Z = 0, bool DET = false>   // VIEW_Z as k_preprocess_bwd
__global__ void __launch_bounds__(PB_THREADS, PB2_MIN_CTAS)
k_preprocess_bwd_2phase(const DevCfg c, const DevInputs in, const uint8_t *__restrict__ meta, const float *__restrict__ acc,
                 const GsInGrads g, const DetAcc det, const DepthMode dm) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    PbSmem *sm = reinterpret_cast<PbSmem *>(smem_raw);
    float *sh_s = reinterpret_cast<float *>(smem_raw + PB_SMEM_HDR);

    const int scene = blockIdx.y;
    const int g0 = blockIdx.x * PB_THREADS;
    const int n = min(PB_THREADS, c.P - g0);
    const int tid = threadIdx.x;
    const int i = g0 + tid;
    const bool active = tid < n;
    const size_t sg = (size_t)scene * c.P + i;
    const int MS = c.M < PB_SH_EVAL ? c.M : PB_SH_EVAL;   // coefficients staged per Gaussian
    const int RS = c.M == MS ? MS * 3 : MS * 3 + 1;       // floats per staged row: compacted rows get an odd stride (no
                                                          // 16-way bank conflicts between the threads of a warp)
    const uint32_t stage_floats = (uint32_t)n * MS * 3u;

    bool bulk = false;
    if (HAS_SH) {
        const float *src = in.shs + ((size_t)scene * c.P + g0) * c.M * 3;
        const float *dst = g.dL_dshs ? g.dL_dshs + ((size_t)scene * c.P + g0) * c.M * 3 : nullptr;
        bulk = c.M == MS && ((reinterpret_cast<uintptr_t>(src) & 15u) == 0) && (((stage_floats * 4u) & 15u) == 0) &&
               ((reinterpret_cast<uintptr_t>(dst) & 15u) == 0);
        if (bulk) {
            if (tid == 0) {
                mbar_init(&sm->bar, 1);
                mbar_fence_init();
                mbar_expect_tx(&sm->bar, stage_floats * 4u);
                tma_load_1d(sh_s, src, stage_floats * 4u, &sm->bar);
            }
        } else {
            const uint32_t row_f = (uint32_t)c.M * 3u, take = (uint32_t)MS * 3u;
            for (uint32_t e = tid; e < stage_floats; e += PB_THREADS) {   // asynchronous 4-byte gathers (LDGSTS)
                const uint32_t row = e / take, col = e - row * take;
                cp_async4(sh_s + row * RS + col, src + (size_t)row * row_f + col);
            }
            cp_async_commit();
        }
    }

    float3 mean = make_float3(0, 0, 0);
    float c6[6] = {0, 0, 0, 0, 0, 0};
    float sc[3] = {0, 0, 0}, q[4] = {0, 0, 0, 0};
    if (active) {
        mean = make_float3(in.means3D[sg * 3 + 0], in.means3D[sg * 3 + 1], in.means3D[sg * 3 + 2]);
        if (in.cov3D) {
#pragma unroll
            for (int k = 0; k < 6; k++) c6[k] = in.cov3D[sg * 6 + k];
        } else {
#pragma unroll
            for (int k = 0; k < 3; k++) sc[k] = in.scales[sg * 3 + k];
#pragma unroll
            for (int k = 0; k < 4; k++) q[k] = in.rotations[sg * 4 + k];
            cov3d_from_scale_rot(sc, c.scale_modifier, q, c6);
        }
    }
    if (HAS_SH) {
        cp_async_wait<0>();
        __syncthreads();
        if (bulk) mbar_wait(&sm->bar, 0);
    }

    float gmean[3] = {0, 0, 0};

    // ================= phase G: geometry =================
    {
        float gcov[6] = {0, 0, 0, 0, 0, 0}, gopac = 0.f;
        for (int vi = 0; vi < c.VPS; vi++) {
            const int v = scene * c.VPS + vi;
            if (vi % GS_CAM_CHUNK == 0) {
                __syncthreads();
                load_view_cams(c, v, min(GS_CAM_CHUNK, c.VPS - vi), sm->cams);
                __syncthreads();
            }
            if (!active) {
                if (VIEW_Z == 1 || (VIEW_Z == 2 && g.dL_dviewmatrix_z)) view_z_grad<DET>(g, det, v, 0.f, 0.f, 0.f, 0.f);
                continue;
            }
            const ViewCam &cam = sm->cams[vi % GS_CAM_CHUNK];
            const size_t o = (size_t)v * c.P + i;
            const uint32_t mb = meta[o];
            float m2d[2] = {0.f, 0.f}, gcol[3] = {0.f, 0.f, 0.f};
            if ((VIEW_Z == 1 || (VIEW_Z == 2 && g.dL_dviewmatrix_z)) && !(mb & GS_META_VISIBLE)) view_z_grad<DET>(g, det, v, 0.f, 0.f, 0.f, 0.f);
            if (mb & GS_META_VISIBLE) {
                const float *a = acc + o * GS_ACC_STRIDE;
                float a_det[GS_ACC_STRIDE];
                if constexpr (DET) a = load_det_acc(det, o, a_det);
                gcol[0] = a[0]; gcol[1] = a[1]; gcol[2] = a[2];
                m2d[0] = a[3]; m2d[1] = a[4];
                const float gcx = a[5], gcy = a[6], gcz = a[7];
                gopac += a[8];
                const float gz = VIEW_Z == 2 ? a[9] * depth_chain(cam, mean, dm, v) : a[9];
                const float s = cam.scale, s2 = s * s;
                const float3 m = make_float3(mean.x * s, mean.y * s, mean.z * s);
                const float cv[6] = {c6[0] * s2, c6[1] * s2, c6[2] * s2, c6[3] * s2, c6[4] * s2, c6[5] * s2};
                float gm[3] = {0.f, 0.f, 0.f};  // dL/dm (view-scaled mean)
                // ---- conic -> cov2D -> cov3D, mean (through J) ----
                {
                    ProjJac j;
                    build_jac(cam, c, m, j);
                    float s0[3], s1[3];
                    sym6_mul(cv, j.m0, s0);
                    sym6_mul(cv, j.m1, s1);
                    const float aa = j.m0[0] * s0[0] + j.m0[1] * s0[1] + j.m0[2] * s0[2] + c.dilation;
                    const float bb = j.m0[0] * s1[0] + j.m0[1] * s1[1] + j.m0[2] * s1[2];
                    const float cc = j.m1[0] * s1[0] + j.m1[1] * s1[1] + j.m1[2] * s1[2] + c.dilation;
                    const float denom = aa * cc - bb * bb;
                    const float d2inv = 1.0f / (denom * denom + 0.0000001f);
                    float dL_da = 0.f, dL_db = 0.f, dL_dc = 0.f;
                    if (d2inv != 0.0f) {
                        dL_da = d2inv * (-cc * cc * gcx + 2.0f * bb * cc * gcy + (denom - aa * cc) * gcz);
                        dL_dc = d2inv * (-aa * aa * gcz + 2.0f * aa * bb * gcy + (denom - aa * cc) * gcx);
                        dL_db = d2inv * 2.0f * (bb * cc * gcx - (denom + 2.0f * bb * bb) * gcy + aa * bb * gcz);
                        const float *m0 = j.m0, *m1 = j.m1;
                        gcov[0] += s2 * (m0[0] * m0[0] * dL_da + m0[0] * m1[0] * dL_db + m1[0] * m1[0] * dL_dc);
                        gcov[3] += s2 * (m0[1] * m0[1] * dL_da + m0[1] * m1[1] * dL_db + m1[1] * m1[1] * dL_dc);
                        gcov[5] += s2 * (m0[2] * m0[2] * dL_da + m0[2] * m1[2] * dL_db + m1[2] * m1[2] * dL_dc);
                        gcov[1] += s2 * (2.0f * m0[0] * m0[1] * dL_da + (m0[0] * m1[1] + m0[1] * m1[0]) * dL_db +
                                         2.0f * m1[0] * m1[1] * dL_dc);
                        gcov[2] += s2 * (2.0f * m0[0] * m0[2] * dL_da + (m0[0] * m1[2] + m0[2] * m1[0]) * dL_db +
                                         2.0f * m1[0] * m1[2] * dL_dc);
                        gcov[4] += s2 * (2.0f * m0[2] * m0[1] * dL_da + (m0[1] * m1[2] + m0[2] * m1[1]) * dL_db +
                                         2.0f * m1[1] * m1[2] * dL_dc);
                    }
                    float dJ00 = 0.f, dJ02 = 0.f, dJ11 = 0.f, dJ12 = 0.f;
#pragma unroll
                    for (int k = 0; k < 3; k++) {
                        const float gm0 = 2.0f * dL_da * s0[k] + dL_db * s1[k];
                        const float gm1 = 2.0f * dL_dc * s1[k] + dL_db * s0[k];
                        dJ00 += gm0 * cam.view[k * 4 + 0];
                        dJ02 += gm0 * cam.view[k * 4 + 2];
                        dJ11 += gm1 * cam.view[k * 4 + 1];
                        dJ12 += gm1 * cam.view[k * 4 + 2];
                    }
                    const float tz = 1.0f / j.tz, tz2 = tz * tz, tz3 = tz2 * tz;
                    const float dtx = j.xin ? -j.fx * tz2 * dJ02 : 0.0f;
                    const float dty = j.yin ? -j.fy * tz2 * dJ12 : 0.0f;
                    const float dtz = -j.fx * tz2 * dJ00 - j.fy * tz2 * dJ11 + (2.0f * j.fx * j.tx) * tz3 * dJ02 +
                                      (2.0f * j.fy * j.ty) * tz3 * dJ12;
#pragma unroll
                    for (int k = 0; k < 3; k++)
                        gm[k] += cam.view[k * 4 + 0] * dtx + cam.view[k * 4 + 1] * dty + cam.view[k * 4 + 2] * dtz;
                }
                // ---- mean2D (NDC units) -> mean through the perspective divide ----
                {
                    const float4 mh = xform4x4(cam.proj, m);
                    const float mw = 1.0f / (mh.w + 0.0000001f);
                    const float mul1 = mh.x * mw * mw, mul2 = mh.y * mw * mw;
                    const float *pr = cam.proj;
                    gm[0] += (pr[0] * mw - pr[3] * mul1) * m2d[0] + (pr[1] * mw - pr[3] * mul2) * m2d[1];
                    gm[1] += (pr[4] * mw - pr[7] * mul1) * m2d[0] + (pr[5] * mw - pr[7] * mul2) * m2d[1];
                    gm[2] += (pr[8] * mw - pr[11] * mul1) * m2d[0] + (pr[9] * mw - pr[11] * mul2) * m2d[1];
                }
                // ---- fused depth channel: z = (view * m).z ----
                gm[0] += cam.view[2] * gz;
                gm[1] += cam.view[6] * gz;
                gm[2] += cam.view[10] * gz;
                if (VIEW_Z == 1 || (VIEW_Z == 2 && g.dL_dviewmatrix_z)) view_z_grad<DET>(g, det, v, gz * m.x, gz * m.y, gz * m.z, gz);
#pragma unroll
                for (int k = 0; k < 3; k++) gmean[k] += s * gm[k];
            }
            if (g.dL_dmeans2D) {
                g.dL_dmeans2D[o * 3 + 0] = m2d[0];
                g.dL_dmeans2D[o * 3 + 1] = m2d[1];
                g.dL_dmeans2D[o * 3 + 2] = 0.0f;
            }
            if (g.dL_dcolors) {
                g.dL_dcolors[o * 3 + 0] = gcol[0];
                g.dL_dcolors[o * 3 + 1] = gcol[1];
                g.dL_dcolors[o * 3 + 2] = gcol[2];
            }
        }
        if (active) {
            if (g.dL_dopacities) g.dL_dopacities[sg] = gopac;
            if (in.cov3D) {
                if (g.dL_dcov3D) {
#pragma unroll
                    for (int k = 0; k < 6; k++) g.dL_dcov3D[sg * 6 + k] = gcov[k];
                }
            } else {
                // Sigma = R diag(v) R^T, v_k = (mod*s_k)^2 : dL/dv_k = (R^T G R)_kk ; dL/dR = 2 G R diag(v)
                float R[3][3];
                quat_to_R(q, R);
                const float G[3][3] = {{gcov[0], 0.5f * gcov[1], 0.5f * gcov[2]},
                                       {0.5f * gcov[1], gcov[3], 0.5f * gcov[4]},
                                       {0.5f * gcov[2], 0.5f * gcov[4], gcov[5]}};
                const float mod = c.scale_modifier;
                float dR[3][3];
#pragma unroll
                for (int k = 0; k < 3; k++) {
                    const float sv = mod * sc[k];
                    float GRk[3];
#pragma unroll
                    for (int a = 0; a < 3; a++) GRk[a] = G[a][0] * R[0][k] + G[a][1] * R[1][k] + G[a][2] * R[2][k];
                    const float dv = R[0][k] * GRk[0] + R[1][k] * GRk[1] + R[2][k] * GRk[2];
                    if (g.dL_dscales) g.dL_dscales[sg * 3 + k] = dv * 2.0f * sv * mod;
#pragma unroll
                    for (int a = 0; a < 3; a++) dR[a][k] = 2.0f * GRk[a] * sv * sv;
                }
                if (g.dL_drotations) {
                    const float r = q[0], x = q[1], y = q[2], z = q[3];
                    float *gq = g.dL_drotations + sg * 4;
                    gq[0] = 2.0f * (-z * dR[0][1] + y * dR[0][2] + z * dR[1][0] - x * dR[1][2] - y * dR[2][0] + x * dR[2][1]);
                    gq[1] = 2.0f * (y * dR[0][1] + z * dR[0][2] + y * dR[1][0] - 2.0f * x * dR[1][1] - r * dR[1][2] +
                                    z * dR[2][0] + r * dR[2][1] - 2.0f * x * dR[2][2]);
                    gq[2] = 2.0f * (-2.0f * y * dR[0][0] + x * dR[0][1] + r * dR[0][2] + x * dR[1][0] + z * dR[1][2] -
                                    r * dR[2][0] + z * dR[2][1] - 2.0f * y * dR[2][2]);
                    gq[3] = 2.0f * (-2.0f * z * dR[0][0] - r * dR[0][1] + x * dR[0][2] + r * dR[1][0] - 2.0f * z * dR[1][1] +
                                    y * dR[1][2] + x * dR[2][0] + y * dR[2][1]);
                }
            }
        }
    }

    // ================= phases S_0..S_2: colour -> SH coefficients and mean (view direction), one channel at a time ====
    if (HAS_SH) {
        float *row = sh_s + (size_t)tid * RS;
#pragma unroll 1
        for (int ch = 0; ch < 3; ch++) {
            float gsh[PB_SH_EVAL];
#pragma unroll
            for (int k = 0; k < PB_SH_EVAL; k++) gsh[k] = 0.f;
            for (int vi = 0; vi < c.VPS; vi++) {
                const int v = scene * c.VPS + vi;
                if (c.VPS > GS_CAM_CHUNK && vi % GS_CAM_CHUNK == 0) {  // (a single chunk is still staged from phase G)
                    __syncthreads();
                    load_view_cams(c, v, min(GS_CAM_CHUNK, c.VPS - vi), sm->cams);
                    __syncthreads();
                }
                if (!active) continue;
                const ViewCam &cam = sm->cams[vi % GS_CAM_CHUNK];
                const size_t o = (size_t)v * c.P + i;
                const uint32_t mb = meta[o];
                if (!(mb & GS_META_VISIBLE) || (mb & (1u << ch))) continue;   // invisible, or this channel was clamped at 0
                float gch;
                if constexpr (DET)
                    gch = gs_det_decode(reinterpret_cast<const long long *>(det.acc) + (o * GS_ACC_STRIDE + ch) * GS_DET_LIMBS,
                                        (det.poison[o] >> ch) & 1u);
                else
                    gch = acc[o * GS_ACC_STRIDE + ch];
                const float s = cam.scale;
                const float d[3] = {mean.x * s - cam.campos[0], mean.y * s - cam.campos[1], mean.z * s - cam.campos[2]};
                const float len2 = d[0] * d[0] + d[1] * d[1] + d[2] * d[2];
                const float inv = 1.0f / sqrtf(len2);
                float ddx = 0.f, ddy = 0.f, ddz = 0.f;
                sh_backward_channel<1>(c.deg, row + ch, gsh, gch, d[0] * inv, d[1] * inv, d[2] * inv, ddx, ddy, ddz);
                const float dot = d[0] * ddx + d[1] * ddy + d[2] * ddz;
                const float inv3 = inv * inv * inv;
                gmean[0] += s * (ddx * len2 - d[0] * dot) * inv3;
                gmean[1] += s * (ddy * len2 - d[1] * dot) * inv3;
                gmean[2] += s * (ddz * len2 - d[2] * dot) * inv3;
            }
            // this channel's staged inputs are dead: its gradients take their place
            if (active) {
#pragma unroll
                for (int k = 0; k < PB_SH_EVAL; k++)
                    if (k < MS) row[k * 3 + ch] = gsh[k];
            }
        }
    }
    if (active && g.dL_dmeans3D) {
#pragma unroll
        for (int k = 0; k < 3; k++) g.dL_dmeans3D[sg * 3 + k] = gmean[k];
    }

    if (HAS_SH && g.dL_dshs) {
        float *dst = g.dL_dshs + ((size_t)scene * c.P + g0) * c.M * 3;
        if (bulk) {
            fence_proxy_async_smem();  // make the generic-proxy smem writes visible to the TMA engine
            __syncthreads();
            if (tid == 0) {
                tma_store_1d(dst, sh_s, stage_floats * 4u);
                tma_store_commit_wait();
            }
        } else {
            __syncthreads();
            // rows of M*3 floats: the staged MS*3 gradients, then zeros for the bands the evaluator never reads
            const uint32_t row_f = (uint32_t)c.M * 3u, take = (uint32_t)MS * 3u, total = (uint32_t)n * row_f;
            for (uint32_t e = tid; e < total; e += PB_THREADS) {
                const uint32_t r = e / row_f, col = e - r * row_f;
                dst[e] = col < take ? sh_s[r * RS + col] : 0.f;
            }
        }
    }
}

// AA: the anti-aliased kernels; CAM: the camera-gradient kernels (single pass only: the two-phase kernel has neither)
template <int VIEW_Z, bool DET, bool AA, bool CAM>
int launch_preprocess_bwd_t(const DevCfg &c, const DevInputs &in, const GsSaved &s, const float *grad_acc,
                            const GsInGrads &g, cudaStream_t st, int variant, const DetAcc &det, const DepthMode &dm) {
    dim3 grid((c.P + PB_THREADS - 1) / PB_THREADS, c.S);
    if (AA && variant == 1)
        return gs_set_error(GS_ERR_INVALID, "GS_TUNE_PBWD_2PHASE has no anti-aliased kernel (GS_FLAG_ANTIALIAS)");
    if (CAM && variant == 1)
        return gs_set_error(GS_ERR_INVALID, "GS_TUNE_PBWD_2PHASE has no camera-gradient kernel (GsCameraGrads)");
    if (in.shs && c.deg > 3) {   // degree 4: the single-pass kernel with band 4 compiled in
        if (variant == 1)
            return gs_set_error(GS_ERR_INVALID, "GS_TUNE_PBWD_2PHASE has no degree-4 kernel (sh_eval_max_degree = 4)");
        const size_t smem = PB_SMEM_HDR + (size_t)PB_THREADS * (c.M * 3 + PB_SH_B4) * 4;
        auto kern = k_preprocess_bwd<true, PB_MIN_CTAS, VIEW_Z, DET, true, AA, CAM>;
        GS_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kern<<<grid, PB_THREADS, smem, st>>>(c, in, s.meta, grad_acc, g, det, dm);
    } else if (AA || CAM || variant != 1) {  // single pass over the views (default)
        if (in.shs) {
            size_t smem = PB_SMEM_HDR + (size_t)PB_THREADS * c.M * 12;
            auto kern = k_preprocess_bwd<true, PB_MIN_CTAS, VIEW_Z, DET, false, AA, CAM>;
            GS_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            kern<<<grid, PB_THREADS, smem, st>>>(c, in, s.meta, grad_acc, g, det, dm);
        } else {
            k_preprocess_bwd<false, PB_MIN_CTAS, VIEW_Z, DET, false, AA, CAM><<<grid, PB_THREADS, PB_SMEM_HDR, st>>>(c, in, s.meta, grad_acc, g, det, dm);
        }
    } else if constexpr (!CAM) {
        if (in.shs) {
            size_t smem = PB_SMEM_HDR + (size_t)PB_THREADS * (c.M <= PB_SH_EVAL ? c.M * 3 : PB_SH_EVAL * 3 + 1) * 4;
            GS_CUDA_OK(cudaFuncSetAttribute(k_preprocess_bwd_2phase<true, VIEW_Z, DET>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            k_preprocess_bwd_2phase<true, VIEW_Z, DET><<<grid, PB_THREADS, smem, st>>>(c, in, s.meta, grad_acc, g, det, dm);
        } else {
            k_preprocess_bwd_2phase<false, VIEW_Z, DET><<<grid, PB_THREADS, PB_SMEM_HDR, st>>>(c, in, s.meta, grad_acc, g, det, dm);
        }
    }
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}

// dL/dviewmatrix_z[v][k] = sum over w, in order, of the per-warp partials view_z[v][w][k]
__global__ void k_view_z_finalize(int V, int warps, const float *__restrict__ view_z, float *__restrict__ out) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= V * 4) return;
    const int v = t >> 2, k = t & 3;
    const float *p = view_z + (size_t)v * warps * 4 + k;
    float sum = 0.f;
    for (int w = 0; w < warps; w++) sum += p[(size_t)w * 4];
    out[t] = sum;
}

// The camera gradient of view blockIdx.x from its per-warp slots [V][warps][GS_CAM_NC], written into GsCameraGrads in
// its own layouts (zeros where an entry feeds nothing; a NULL output is skipped).  Fixed order, so deterministic: lane x
// of row y adds component x of the slots w = y, y + 32, y + 64, ... in turn (each row reads whole 128-byte slots), then
// row 0 adds the 32 row sums in row order.  One CTA of 32 x 32 threads per view: a view's slots are spread over 32
// sequential chains instead of one (a scene of 500k Gaussians has 15 625 slots per view).  dL_dtanfov: [V,2] or NULL.
__global__ void __launch_bounds__(1024) k_camera_finalize(int warps, const float *__restrict__ slots, GsCameraGrads out,
                                                          float *__restrict__ dL_dtanfov) {
    __shared__ float part[32][33];
    const int v = blockIdx.x, k = threadIdx.x, r = threadIdx.y;
    const float *p = slots + (size_t)v * warps * GS_CAM_NC + k;
    float sum = 0.f;
    for (int w = r; w < warps; w += 32) sum += p[(size_t)w * GS_CAM_NC];
    part[r][k] = sum;
    __syncthreads();
    if (r == 0) {
        float t = 0.f;
        for (int i = 0; i < 32; i++) t += part[i][k];
        if (k < 12) {          // dL/dviewmatrix[4 (k / 3) + k % 3]
            if (out.dL_dviewmatrix) out.dL_dviewmatrix[v * 16 + 4 * (k / 3) + k % 3] = t;
        } else if (k < 24) {   // dL/dprojmatrix[4 i + (0, 1, 3)[j]], k - 12 = 3 i + j
            const int i = (k - 12) / 3, j = (k - 12) % 3;
            if (out.dL_dprojmatrix) out.dL_dprojmatrix[v * 16 + 4 * i + (j == 2 ? 3 : j)] = t;
        } else if (k < 27) {
            if (out.dL_dcampos) out.dL_dcampos[v * 3 + k - 24] = t;
        } else if (k < 29) {
            if (dL_dtanfov) dL_dtanfov[v * 2 + k - 27] = t;
        }
    } else if (r == 1 && k < 8) {   // the entries that feed nothing: the view matrix's 4th column, Pf's 3rd
        if (k < 4 && out.dL_dviewmatrix) out.dL_dviewmatrix[v * 16 + 4 * k + 3] = 0.f;
        if (k >= 4 && out.dL_dprojmatrix) out.dL_dprojmatrix[v * 16 + 4 * (k - 4) + 2] = 0.f;
    }
}

int view_z_warps(const DevCfg &c) { return (c.P + PB_THREADS - 1) / PB_THREADS * (PB_THREADS / 32); }

// the VIEW_Z kernels of one (DET, AA, CAM) triple: 2 after a forward whose depth channel carried f(z), else 1 when the
// view matrix's z column is wanted (never with CAM), else 0
template <bool DET, bool AA, bool CAM>
int launch_preprocess_bwd_vz(const DevCfg &c, const DevInputs &in, const GsSaved &s, const float *grad_acc,
                             const GsInGrads &g, cudaStream_t st, int variant, const DetAcc &det, const DepthMode &dm) {
    const bool fz = (s.flags & GS_FLAG_DEPTH) && s.depth_mode != GS_DEPTH_Z;
    if (fz) return launch_preprocess_bwd_t<2, DET, AA, CAM>(c, in, s, grad_acc, g, st, variant, det, dm);
    if constexpr (CAM) {
        return launch_preprocess_bwd_t<0, DET, AA, true>(c, in, s, grad_acc, g, st, variant, det, dm);
    } else {
        return g.dL_dviewmatrix_z ? launch_preprocess_bwd_t<1, DET, AA, false>(c, in, s, grad_acc, g, st, variant, det, dm)
                                  : launch_preprocess_bwd_t<0, DET, AA, false>(c, in, s, grad_acc, g, st, variant, det, dm);
    }
}

template <bool CAM>
int launch_preprocess_bwd_cam(const DevCfg &c, const DevInputs &in, const GsSaved &s, const float *grad_acc,
                              const GsInGrads &g, cudaStream_t st, int variant, const DetAcc &det, const DepthMode &dm) {
    // the forward's anti-aliasing setting, whatever this call's flags say
    const bool aa = (s.flags & GS_FLAG_ANTIALIAS) != 0;
    if (!det.acc)
        return aa ? launch_preprocess_bwd_vz<false, true, CAM>(c, in, s, grad_acc, g, st, variant, det, dm)
                  : launch_preprocess_bwd_vz<false, false, CAM>(c, in, s, grad_acc, g, st, variant, det, dm);
    return aa ? launch_preprocess_bwd_vz<true, true, CAM>(c, in, s, grad_acc, g, st, variant, det, dm)
              : launch_preprocess_bwd_vz<true, false, CAM>(c, in, s, grad_acc, g, st, variant, det, dm);
}

}  // namespace

size_t det_view_z_bytes(const DevCfg &c) { return (size_t)c.V * view_z_warps(c) * 4 * sizeof(float); }

size_t camera_grad_scratch_bytes(const DevCfg &c) { return (size_t)view_z_warps(c) * c.V * GS_CAM_NC * sizeof(float); }

// g.dL_dviewmatrix_z non-NULL selects the VIEW_Z kernels; the caller has zeroed it (the kernels accumulate into it, or in
// deterministic mode k_view_z_finalize writes it).  det.acc non-NULL selects the deterministic kernels.  cam non-NULL
// selects the camera-gradient kernels (never with dL_dviewmatrix_z): det.view_z then holds camera_grad_scratch_bytes of
// per-warp slots, in both modes, and dL_dtanfov (may be NULL) receives the tanfov gradient.
int launch_preprocess_bwd(const DevCfg &c, const DevInputs &in, const GsSaved &s, const float *grad_acc,
                          const GsInGrads &g, cudaStream_t st, int variant, const DetAcc &det, const DepthMode &dm,
                          const GsCameraGrads *cam, float *dL_dtanfov) {
    if (c.P == 0) return GS_OK;
    if (cam) {
        const int rc = launch_preprocess_bwd_cam<true>(c, in, s, grad_acc, g, st, variant, det, dm);
        if (rc != GS_OK) return rc;
        k_camera_finalize<<<c.V, dim3(32, 32), 0, st>>>(view_z_warps(c), det.view_z, *cam, dL_dtanfov);
        GS_CUDA_OK(cudaGetLastError());
        return GS_OK;
    }
    const int rc = launch_preprocess_bwd_cam<false>(c, in, s, grad_acc, g, st, variant, det, dm);
    if (rc != GS_OK || !det.acc || !g.dL_dviewmatrix_z) return rc;
    k_view_z_finalize<<<(c.V * 4 + 127) / 128, 128, 0, st>>>(c.V, view_z_warps(c), det.view_z, g.dL_dviewmatrix_z);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}
