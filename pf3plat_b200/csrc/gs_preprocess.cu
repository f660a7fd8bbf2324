// gs_preprocess.cu -- stage 1 of the forward: per (view, Gaussian) projection, culling, 2-D conic, SH colour.
//
// Semantics: SURVEY.md Appendix A "Preprocess" (the external extension's preprocessCUDA; call site
// PF3plat's src/model/decoder/cuda_splatting.py:117-124).  Design (DESIGN.md section 5.1):
//  * one thread per Gaussian, LOOPING over the views of its scene, so the scene-level inputs (mean, covariance
//    and the 300-byte SH block) are read from HBM once per call instead of once per view;
//  * the coefficients the evaluator reads (bands 0..3 by default: 16 of PF3plat's 25; all 25 at the opt-in degree 4,
//    the B4 instantiations) are staged into shared memory -- one 1-D bulk TMA copy (cp.async.bulk, SASS UBLKCP)
//    completing on an mbarrier when they form a contiguous aligned block, a 4-byte cp.async gather into odd-stride
//    rows otherwise -- fully coalesced, no register staging;
//  * k_sh_colour (below): the colour words alone, pulled out of PINNED HOST memory, for gs_render_host's split pipeline,
//    with k_preprocess running geometry-only (COLOUR = 0) next to it;
//  * outputs are three float4 SoA planes written with 16-byte stores;
//  * tile binning keeps, of upstream's 3-sigma square, only the tiles the alpha >= 1/255 ellipse really reaches
//    (exact box test), so tile lists only hold Gaussians that can contribute (identical pixels, -27 % instances).
#include "gs_common.cuh"

namespace {

constexpr int PRE_THREADS = 128;
constexpr int EMIT_BATCH = 4;  // cursor atomics in flight per thread

// Knock-out builds for scripts/preprocess_ablation.py (-DGS_PRE_ABLATE=<mask>; 0, the product build, removes nothing).
// Each bit drops one piece of k_preprocess's work on the speculative path; what the compiler could dead-code around it is
// kept alive by abl_sink.  The results of such a build are wrong by design: it exists to be timed.
#ifndef GS_PRE_ABLATE
#define GS_PRE_ABLATE 0
#endif
constexpr unsigned ABL = GS_PRE_ABLATE;
constexpr unsigned ABL_EMIT = 1;    // fused emission: no cursor atomics, no bucket stores (the tile tests stay)
constexpr unsigned ABL_TESTS = 2;   // the candidate tile tests (every candidate of the 3-sigma square passes)
constexpr unsigned ABL_SH = 4;      // SH staging and eval_sh: the colour is a constant
constexpr unsigned ABL_REC = 8;     // the rec0..rec2 stores
constexpr unsigned ABL_RRM = 16;    // the radii / rects / meta stores
constexpr unsigned ABL_BAR = 32;    // the barrier pair of the first camera chunk (its cameras ride on the SH barrier)

// a store that never happens but that the compiler cannot prove never happens
__device__ __forceinline__ void abl_sink(uint32_t v, int32_t *dst) {
    if (v == 0x9e3779b9u) *dst = (int32_t)v;
}

struct PreSmem {
    ViewCam cams[GS_CAM_CHUNK];
    float strata[GS_CAM_CHUNK][BIN_SUB];  // depth-stratum boundaries of the staged views (PreEmit::strata)
    uint64_t bar;
    float2 near_far[GS_CAM_CHUNK];        // unscaled (near, far) of the staged views (FZ kernels only; inside the padding)
};
constexpr int PRE_SMEM_HDR = (sizeof(PreSmem) + 127) / 128 * 128;

// SH colour of one Gaussian seen from direction `dir` (unit vector), bands 0..deg (Appendix A "SH -> RGB": upstream's
// left-to-right sum, +0.5, clamp at 0 with the clamp recorded per channel).  Every operation is an explicit
// round-to-nearest intrinsic -- no contraction or re-association left to the compiler -- because TWO kernels inline this
// function (k_preprocess and k_sh_colour, the split pipeline of gs_render_host) and must produce the same bits.
// B4: band 4 is compiled in (evaluated when deg == 4); the default instantiation is the degree-<=3 evaluator unchanged.
template <bool B4 = false>
__device__ __forceinline__ float3 eval_sh(int deg, const float *sh /* [M][3] for this Gaussian */, float3 dir,
                                          uint32_t &clamped) {
    const float x = dir.x, y = dir.y, z = dir.z;
    float v[3];
    // band by band (basis values of one band live at a time), every channel's sum in upstream's left-to-right order
#pragma unroll
    for (int c = 0; c < 3; c++) v[c] = __fmul_rn(GS_SH_C0, sh[c]);
    if (deg > 0) {   // (uniform branches: the degree is a launch constant)
        const float b1 = __fmul_rn(-GS_SH_C1, y), b2 = __fmul_rn(GS_SH_C1, z), b3 = __fmul_rn(-GS_SH_C1, x);
#pragma unroll
        for (int c = 0; c < 3; c++)
            v[c] = __fmaf_rn(b3, sh[3 * 3 + c], __fmaf_rn(b2, sh[2 * 3 + c], __fmaf_rn(b1, sh[1 * 3 + c], v[c])));
        if (deg > 1) {
            const float xx = __fmul_rn(x, x), yy = __fmul_rn(y, y), zz = __fmul_rn(z, z);
            const float xy = __fmul_rn(x, y), yz = __fmul_rn(y, z), xz = __fmul_rn(x, z);
            {
                const float b4 = __fmul_rn(GS_SH_C2_0, xy), b5 = __fmul_rn(GS_SH_C2_1, yz);
                const float b6 = __fmul_rn(GS_SH_C2_2, __fsub_rn(__fsub_rn(__fmul_rn(2.0f, zz), xx), yy));
                const float b7 = __fmul_rn(GS_SH_C2_3, xz), b8 = __fmul_rn(GS_SH_C2_4, __fsub_rn(xx, yy));
#pragma unroll
                for (int c = 0; c < 3; c++) {
                    float t = __fmaf_rn(b5, sh[5 * 3 + c], __fmaf_rn(b4, sh[4 * 3 + c], v[c]));
                    t = __fmaf_rn(b7, sh[7 * 3 + c], __fmaf_rn(b6, sh[6 * 3 + c], t));
                    v[c] = __fmaf_rn(b8, sh[8 * 3 + c], t);
                }
            }
            if (deg > 2) {
                const float zz4 = __fsub_rn(__fsub_rn(__fmul_rn(4.0f, zz), xx), yy);
                const float b9 = __fmul_rn(__fmul_rn(GS_SH_C3_0, y), __fsub_rn(__fmul_rn(3.0f, xx), yy));
                const float b10 = __fmul_rn(__fmul_rn(GS_SH_C3_1, xy), z);
                const float b11 = __fmul_rn(__fmul_rn(GS_SH_C3_2, y), zz4);
                const float b12 = __fmul_rn(__fmul_rn(GS_SH_C3_3, z), __fsub_rn(__fsub_rn(__fmul_rn(2.0f, zz), __fmul_rn(3.0f, xx)), __fmul_rn(3.0f, yy)));
                const float b13 = __fmul_rn(__fmul_rn(GS_SH_C3_4, x), zz4);
                const float b14 = __fmul_rn(__fmul_rn(GS_SH_C3_5, z), __fsub_rn(xx, yy));
                const float b15 = __fmul_rn(__fmul_rn(GS_SH_C3_6, x), __fsub_rn(xx, __fmul_rn(3.0f, yy)));
#pragma unroll
                for (int c = 0; c < 3; c++) {
                    float t = __fmaf_rn(b10, sh[10 * 3 + c], __fmaf_rn(b9, sh[9 * 3 + c], v[c]));
                    t = __fmaf_rn(b12, sh[12 * 3 + c], __fmaf_rn(b11, sh[11 * 3 + c], t));
                    t = __fmaf_rn(b14, sh[14 * 3 + c], __fmaf_rn(b13, sh[13 * 3 + c], t));
                    v[c] = __fmaf_rn(b15, sh[15 * 3 + c], t);
                }
                if (B4 && deg > 3) {
                    const float xx_yy = __fsub_rn(xx, yy), xx3_yy = __fsub_rn(__fmul_rn(3.0f, xx), yy);
                    const float xx_3yy = __fsub_rn(xx, __fmul_rn(3.0f, yy)), zz7 = __fmul_rn(7.0f, zz);
                    const float zz7m1 = __fsub_rn(zz7, 1.0f), zz7m3 = __fsub_rn(zz7, 3.0f);
                    const float b16 = __fmul_rn(__fmul_rn(GS_SH_C4_0, xy), xx_yy);
                    const float b17 = __fmul_rn(__fmul_rn(GS_SH_C4_1, yz), xx3_yy);
                    const float b18 = __fmul_rn(__fmul_rn(GS_SH_C4_2, xy), zz7m1);
                    const float b19 = __fmul_rn(__fmul_rn(GS_SH_C4_3, yz), zz7m3);
                    const float b20 = __fmul_rn(GS_SH_C4_4, __fadd_rn(__fmul_rn(zz, __fsub_rn(__fmul_rn(35.0f, zz), 30.0f)), 3.0f));
                    const float b21 = __fmul_rn(__fmul_rn(GS_SH_C4_5, xz), zz7m3);
                    const float b22 = __fmul_rn(__fmul_rn(GS_SH_C4_6, xx_yy), zz7m1);
                    const float b23 = __fmul_rn(__fmul_rn(GS_SH_C4_7, xz), xx_3yy);
                    const float b24 = __fmul_rn(GS_SH_C4_8, __fsub_rn(__fmul_rn(xx, xx_3yy), __fmul_rn(yy, xx3_yy)));
#pragma unroll
                    for (int c = 0; c < 3; c++) {
                        float t = __fmaf_rn(b17, sh[17 * 3 + c], __fmaf_rn(b16, sh[16 * 3 + c], v[c]));
                        t = __fmaf_rn(b19, sh[19 * 3 + c], __fmaf_rn(b18, sh[18 * 3 + c], t));
                        t = __fmaf_rn(b21, sh[21 * 3 + c], __fmaf_rn(b20, sh[20 * 3 + c], t));
                        t = __fmaf_rn(b23, sh[23 * 3 + c], __fmaf_rn(b22, sh[22 * 3 + c], t));
                        v[c] = __fmaf_rn(b24, sh[24 * 3 + c], t);
                    }
                }
            }
        }
    }
    float r[3];
#pragma unroll
    for (int c = 0; c < 3; c++) {
        const float w = __fadd_rn(v[c], 0.5f);
        if (w < 0.0f) clamped |= (1u << c);
        r[c] = fmaxf(w, 0.0f);
    }
    return make_float3(r[0], r[1], r[2]);
}

// unit vector from the camera to the (scaled) mean; pinned like eval_sh
__device__ __forceinline__ float3 sh_view_dir(float3 m, const float *campos) {
    const float dx = __fsub_rn(m.x, campos[0]), dy = __fsub_rn(m.y, campos[1]), dz = __fsub_rn(m.z, campos[2]);
    const float inv = __frcp_rn(__fsqrt_rn(__fmaf_rn(dz, dz, __fmaf_rn(dy, dy, __fmul_rn(dx, dx)))));
    return make_float3(__fmul_rn(dx, inv), __fmul_rn(dy, inv), __fmul_rn(dz, inv));
}

// FZ kernels: the unscaled (near, far) of views [v0, v0 + count) next to their cameras (all threads; the caller's barrier
// follows).  Modes that read neither may come without the array.
__device__ __forceinline__ void stage_near_far(const DepthMode &dm, int v0, int count, float2 *dst) {
    for (int t = threadIdx.x; t < count; t += blockDim.x)
        dst[t] = dm.near_far ? make_float2(dm.near_far[(v0 + t) * 2], dm.near_far[(v0 + t) * 2 + 1]) : make_float2(0.f, 0.f);
}

// Everything preprocess derives for one (view, Gaussian).
struct Splat {
    float4 r0, r1, r2;
    int32_t radius;
    uint32_t meta;
    ushort4 rect;
};

// Appendix A "Preprocess" for one Gaussian in one view.  COLOUR = 2: `sh` points at this Gaussian's [M][3] block in
// shared memory; 1: `rgb_in` is its precomputed colour; 0: geometry only (the colour words are written by k_sh_colour).
// AA: GS_FLAG_ANTIALIAS -- the splat's opacity is o * rho (gs_aa_rho) wherever the kernels read it: the record and the
// tight-binning threshold.  Conic, radius and tile rectangle stay those of the dilated covariance.
template <int COLOUR, bool B4 = false, bool AA = false>
__device__ __forceinline__ void project_splat(const DevCfg &c, const ViewCam &cam, float3 mean, const float *c6,
                                              float opac, const float *sh, const float *rgb_in, Splat &out) {
    out.radius = 0;
    out.meta = 0;
    out.rect = make_ushort4(0, 0, 0, 0);
    const float s = cam.scale, s2 = s * s;
    const float3 m = make_float3(mean.x * s, mean.y * s, mean.z * s);
    const float3 pv = xform4x3(cam.view, m);
    if (!(pv.z > c.near_cull_z)) return;  // in_frustum
    const float4 ph = xform4x4(cam.proj, m);
    const float pw = 1.0f / (ph.w + 0.0000001f);
    const float cv[6] = {c6[0] * s2, c6[1] * s2, c6[2] * s2, c6[3] * s2, c6[4] * s2, c6[5] * s2};
    ProjJac j;
    build_jac(cam, c, m, j);
    float s0[3], s1[3];
    sym6_mul(cv, j.m0, s0);
    sym6_mul(cv, j.m1, s1);
    const float a = j.m0[0] * s0[0] + j.m0[1] * s0[1] + j.m0[2] * s0[2] + c.dilation;
    const float b = j.m0[0] * s1[0] + j.m0[1] * s1[1] + j.m0[2] * s1[2];
    const float cc = j.m1[0] * s1[0] + j.m1[1] * s1[1] + j.m1[2] * s1[2] + c.dilation;
    const float det = a * cc - b * b;
    if (det == 0.0f) return;
    if constexpr (AA) {   // (the undilated diagonal: the sums above without + c.dilation)
        const float a0 = j.m0[0] * s0[0] + j.m0[1] * s0[1] + j.m0[2] * s0[2];
        const float c0 = j.m1[0] * s1[0] + j.m1[1] * s1[1] + j.m1[2] * s1[2];
        opac = opac * gs_aa_rho(gs_aa_ratio(a0, b, c0, det));
    }
    const float det_inv = 1.0f / det;
    const float A = cc * det_inv, B = -b * det_inv, C = a * det_inv;
    const float mid = 0.5f * (a + cc);
    const float sq = sqrtf(fmaxf(0.1f, mid * mid - det));
    const float rad = ceilf(3.0f * sqrtf(fmaxf(mid + sq, mid - sq)));
    const float px = ndc2pix(ph.x * pw, c.W), py = ndc2pix(ph.y * pw, c.H);
    // upstream's 3-sigma square in tiles (getRect)
    const int rminx = min(c.gx, max(0, (int)((px - rad) / (float)GS_TILE)));
    const int rminy = min(c.gy, max(0, (int)((py - rad) / (float)GS_TILE)));
    const int rmaxx = min(c.gx, max(0, (int)((px + rad + (float)(GS_TILE - 1)) / (float)GS_TILE)));
    const int rmaxy = min(c.gy, max(0, (int)((py + rad + (float)(GS_TILE - 1)) / (float)GS_TILE)));
    if ((rmaxx - rminx) * (rmaxy - rminy) == 0) return;
    out.radius = (int32_t)rad;
    out.meta = GS_META_VISIBLE;
    float3 rgb;
    if (COLOUR == 2 && (ABL & ABL_SH)) rgb = make_float3(0.5f, 0.5f, 0.5f);
    else if (COLOUR == 2) rgb = eval_sh<B4>(c.deg, sh, sh_view_dir(m, cam.campos), out.meta);
    else if (COLOUR == 1) rgb = make_float3(rgb_in[0], rgb_in[1], rgb_in[2]);
    else rgb = make_float3(0.f, 0.f, 0.f);   // COLOUR == 0: k_sh_colour fills the three colour words of the record
    // Tight binning.  A pixel can only receive this Gaussian if alpha = o*G >= 1/255, i.e. log2 G >= -log2(255 o).
    // The candidate tiles are upstream's 3-sigma square; k_preprocess / k_emit_buckets keep a candidate only if the
    // alpha >= 1/255 ellipse really reaches it (gs_box_reaches, exact).  Tiles dropped this way cannot change any
    // pixel.  The threshold carries a margin for the fp32 rounding of log2 G in the compositor (it grows with the
    // reach of the footprint).
    const float reach = rad + (float)GS_TILE;
    const float margin = 1e-3f + 4e-6f * reach * reach;              // in units of tau = 2 ln(255 o)
    const float tau = 2.0f * logf(255.0f * opac) + margin;
    const float hA = (-0.5f * GS_LOG2E) * A, nB = -GS_LOG2E * B, hC = (-0.5f * GS_LOG2E) * C;
    const float reach2 = -(0.5f * GS_LOG2E) * tau;                     // same threshold in log2-G units
    if (tau > 0.0f)  // else opacity < 1/255: visible (radius reported) but it can never contribute
        out.rect = make_ushort4((unsigned short)rminx, (unsigned short)rminy, (unsigned short)rmaxx, (unsigned short)rmaxy);
    out.r0 = make_float4(px, py, hA, nB);
    out.r1 = make_float4(hC, opac, rgb.x, rgb.y);
    out.r2 = make_float4(rgb.z, pv.z, reach2, 0.0f);
}

// MINB: resident CTAs per SM the register allocation is bounded for.  Unbounded the kernel takes 96 registers (5 CTAs/SM;
// latency-bound).  Bounded to 64 (8 CTAs/SM, 116 bytes of spills and more instructions) it was slower on C2.
// B4: degree-4 evaluation (25 coefficients staged per Gaussian); the B4 = false kernels are the degree-<=3 ones unchanged.
// FZ: a depth mode other than GS_DEPTH_Z -- rec2.w = f(z) of dm.mode (a uniform runtime branch), with the views' near and
// far staged next to their cameras.  The FZ = false kernels are the ones without it, instruction for instruction (dm unused).
// AA: GS_FLAG_ANTIALIAS (project_splat); the AA = false kernels are the ones without it, instruction for instruction.
template <int COLOUR, int MINB, bool B4 = false, bool FZ = false, bool AA = false>
__global__ void __launch_bounds__(PRE_THREADS, MINB)
k_preprocess(const DevCfg c, const DevInputs in, float4 *__restrict__ rec0, float4 *__restrict__ rec1,
             float4 *__restrict__ rec2, uint8_t *__restrict__ meta, int32_t *__restrict__ radii,
             ushort4 *__restrict__ rects, const PreEmit emit, const int g_begin, const int g_end, const int sh_raw16,
             const DepthMode dm) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    PreSmem *sm = reinterpret_cast<PreSmem *>(smem_raw);
    float *sh_s = reinterpret_cast<float *>(smem_raw + PRE_SMEM_HDR);

    const int scene = blockIdx.y;
    const int g0 = g_begin + blockIdx.x * PRE_THREADS;  // this launch covers Gaussians [g_begin, g_end) of every scene
    const int n = min(PRE_THREADS, g_end - g0);
    const int tid = threadIdx.x;
    const int i = g0 + tid;
    const bool active = tid < n;
    const size_t sg = (size_t)scene * c.P + i;  // scene-level index

    // ---- stage this CTA's SH block ----
    // Only the bands the evaluator can touch are wanted: MS = min(M, 16) coefficients per Gaussian (PF3plat hands over
    // M = 25 of which 16..24 are never read).
    //  * M <= 16: the block is contiguous and arrives by ONE 1-D bulk TMA copy (cp.async.bulk, SASS UBLKCP) completing on
    //    an mbarrier.
    //  * M > 16 (default): the wanted 192 bytes of every row are gathered with 4-byte cp.async into rows compacted to an
    //    ODD stride (49 floats): with 48, thread t's row starts at bank 16 t mod 32 and all 32 lanes of a warp hit two
    //    banks, and bank conflicts make preprocess far slower.  Rows are only 4-byte aligned (300 = 18 * 16 +
    //    12), so neither a bulk copy per row nor a 2-D tensor map is possible.
    //  * M > 16, sh_raw16 (gs_render_host's ZERO-COPY feed; GS_TUNE_PRE_SH_RAW16 for the A/B): rows keep their own stride of
    //    3 M floats in shared memory and only the 16-byte pieces that hold a wanted coefficient are copied (16-byte
    //    cp.async, SASS LDGSTS.128).  Built for a source in PINNED HOST memory, which is pulled over PCIe faster by
    //    16-byte loads than by 4-byte ones (scripts/probes/pcie_pull_probe.cu compares them with the copy engine).  On
    //    device-resident SH it loses to the compacting gather (38 instead of 25 KB of shared memory per CTA leave the L1 28 KB at five CTAs per SM).
    //  * B4 (degree 4): all 25 coefficients are wanted, so for PF3plat's M = 25 the block is contiguous again: one bulk TMA
    //    copy when it is 16-byte aligned, else a 4-byte cp.async gather; rows keep their own odd stride of 75 floats.
    //    (M > 25 compacts to 75 floats.)  The B4 constants are spelled inline: named constexpr locals, though folded
    //    away, renumber the front end's virtual registers and perturb the default kernels' register allocation.
    const int MS = c.M < (B4 ? 25 : 16) ? c.M : (B4 ? 25 : 16);
    const int RS = (c.M == MS || sh_raw16) ? c.M * 3 : (B4 ? 75 : 49);   // floats per staged row (3 M = 75 for PF3plat: 11 t mod 32, conflict-free)
    constexpr bool HAS_SH = COLOUR == 2;
    bool bulk = false;
    if (HAS_SH && !(ABL & ABL_SH)) {
        const float *src = in.shs + ((size_t)scene * c.P + g0) * c.M * 3;
        if (c.M == MS) {
            const uint32_t bytes = (uint32_t)n * c.M * 12u;
            bulk = ((reinterpret_cast<uintptr_t>(src) & 15u) == 0) && ((bytes & 15u) == 0);
            if (bulk) {
                if (tid == 0) {
                    mbar_init(&sm->bar, 1);
                    mbar_fence_init();
                    mbar_expect_tx(&sm->bar, bytes);
                    tma_load_1d(sh_s, src, bytes, &sm->bar);
                }
            } else if constexpr (B4) {  // unaligned slice or ragged tail: asynchronous coalesced 4-byte copies
                for (uint32_t k = tid; k < (uint32_t)n * c.M * 3u; k += PRE_THREADS) cp_async4(sh_s + k, src + k);
                cp_async_commit();
            } else {  // unaligned slice or ragged tail: plain coalesced copy
                for (uint32_t k = tid; k < (uint32_t)n * c.M * 3u; k += PRE_THREADS) sh_s[k] = src[k];
            }
        } else if (sh_raw16) {
            const uint32_t row_f = (uint32_t)c.M * 3u, want_f = (uint32_t)MS * 3u, nfl = (uint32_t)n * row_f, nq = nfl >> 2;
            const float4 *src4 = reinterpret_cast<const float4 *>(src);
            for (uint32_t q = tid; q < nq; q += PRE_THREADS) {
                const uint32_t f0 = q << 2, r = f0 / row_f, c0 = f0 - r * row_f;
                // floats [c0, c0 + 4) of row r (running over into the next row's first coefficients when c0 + 3 >= row_f)
                if (c0 < want_f || c0 + 3u >= row_f) cp_async16(sh_s + f0, src4 + q);
            }
            for (uint32_t f = (nq << 2) + tid; f < nfl; f += PRE_THREADS)   // ragged end of the block (n * row_f % 4 floats)
                if (f % row_f < want_f) cp_async4(sh_s + f, src + f);
            cp_async_commit();
        } else {
            // asynchronous 4-byte copies (cp.async, SASS LDGSTS): all 48 per thread are in flight together while the
            // scalar inputs load -- a plain load/store loop here serialises the latencies
            const uint32_t row_f = (uint32_t)c.M * 3u;
            for (uint32_t e = tid; e < (uint32_t)n * (B4 ? 75u : 48u); e += PRE_THREADS) {
                const uint32_t row = e / (B4 ? 75u : 48u), col = e - row * (B4 ? 75u : 48u);
                cp_async4(sh_s + row * (B4 ? 75u : 49u) + col, src + (size_t)row * row_f + col);
            }
            cp_async_commit();
        }
    }
    // ---- scene-level inputs (issued while the bulk copy is in flight) ----
    float3 mean = make_float3(0, 0, 0);
    float c6[6] = {0, 0, 0, 0, 0, 0};
    float opac = 0.f;
    if (active) {
        mean = make_float3(in.means3D[sg * 3 + 0], in.means3D[sg * 3 + 1], in.means3D[sg * 3 + 2]);
        opac = in.opacities[sg];
        if (in.cov3D) {
#pragma unroll
            for (int k = 0; k < 6; k++) c6[k] = in.cov3D[sg * 6 + k];
        } else {
            const float s[3] = {in.scales[sg * 3 + 0], in.scales[sg * 3 + 1], in.scales[sg * 3 + 2]};
            const float q[4] = {in.rotations[sg * 4 + 0], in.rotations[sg * 4 + 1], in.rotations[sg * 4 + 2],
                                in.rotations[sg * 4 + 3]};
            cov3d_from_scale_rot(s, c.scale_modifier, q, c6);
        }
    }
    // (knock-out build only) the first chunk's cameras are staged before the SH barrier instead of between a pair of their own
    constexpr bool EARLY_CAMS = (ABL & ABL_BAR) && HAS_SH;
    if (EARLY_CAMS) {
        const int nv = min(GS_CAM_CHUNK, c.VPS);
        load_view_cams(c, scene * c.VPS, nv, sm->cams);
        if (emit.strata && !emit.strata_per_tile)
            for (int t = tid; t < nv * BIN_SUB; t += PRE_THREADS)
                sm->strata[t / BIN_SUB][t % BIN_SUB] = emit.strata[(size_t)(scene * c.VPS) * BIN_SUB + t];
        if (FZ) stage_near_far(dm, scene * c.VPS, nv, sm->near_far);
    }
    if (HAS_SH) {
        cp_async_wait<0>();  // this thread's share of the strided copy (no-op on the other paths)
        __syncthreads();     // barrier init (bulk) or the copies (fallbacks) visible to everyone
        if (bulk) mbar_wait(&sm->bar, 0);
    }

    // appends whose cursor value is still on its way back from L2 (see the emission below)
    bool pend_ok[EMIT_BATCH];
    uint32_t pend_slot[EMIT_BATCH], pend_pos[EMIT_BATCH];
    uint64_t pend_key = 0;
#pragma unroll
    for (int k = 0; k < EMIT_BATCH; k++) {
        pend_ok[k] = false;
        pend_slot[k] = pend_pos[k] = 0;
    }
    auto flush_pending = [&]() {
#pragma unroll
        for (int k = 0; k < EMIT_BATCH; k++) {
            if (pend_ok[k] && pend_pos[k] < emit.sub_cap)
                emit.bucket[(size_t)pend_slot[k] * emit.sub_cap + pend_pos[k]] = pend_key;
            pend_ok[k] = false;
        }
    };

    for (int v0 = 0; v0 < c.VPS; v0 += GS_CAM_CHUNK) {
        const int nv = min(GS_CAM_CHUNK, c.VPS - v0);
        if (!(EARLY_CAMS && v0 == 0)) {
            __syncthreads();
            load_view_cams(c, scene * c.VPS + v0, nv, sm->cams);
            if (emit.strata && !emit.strata_per_tile)
                for (int t = tid; t < nv * BIN_SUB; t += PRE_THREADS)
                    sm->strata[t / BIN_SUB][t % BIN_SUB] = emit.strata[(size_t)(scene * c.VPS + v0) * BIN_SUB + t];
            if (FZ) stage_near_far(dm, scene * c.VPS + v0, nv, sm->near_far);
            __syncthreads();
        }
        if (!active) continue;
        for (int vi = 0; vi < nv; vi++) {
            const int v = scene * c.VPS + v0 + vi;
            const size_t o = (size_t)v * c.P + i;
            Splat sp;
            project_splat<COLOUR, B4, AA>(c, sm->cams[vi], mean, c6, opac, sh_s + (size_t)tid * RS,
                                  COLOUR == 1 ? in.colors_precomp + o * 3 : nullptr, sp);
            // the depth channel's value: f at the unscaled depth z = z_s / s
            if (FZ && sp.radius > 0)
                sp.r2.w = gs_depth_f(dm.mode, sp.r2.y / sm->cams[vi].scale, sm->near_far[vi].x, sm->near_far[vi].y);
            // fused speculative emission: nothing reads the rects afterwards (k_emit_buckets and the strata learning, their
            // readers, run on the other paths only)
            const bool fused = emit.counters && emit.bucket;
            // (the knock-out builds keep every store and emission of the exact path, where the capacities they run on are learned)
            const bool abl_spec = ABL && fused;
            if ((ABL & ABL_REC) && abl_spec && sp.radius > 0) {
                abl_sink(__float_as_uint(sp.r0.x) ^ __float_as_uint(sp.r0.y) ^ __float_as_uint(sp.r0.z) ^ __float_as_uint(sp.r0.w) ^
                             __float_as_uint(sp.r1.x) ^ __float_as_uint(sp.r1.y) ^ __float_as_uint(sp.r1.z) ^ __float_as_uint(sp.r1.w) ^
                             __float_as_uint(sp.r2.x) ^ __float_as_uint(sp.r2.y) ^ __float_as_uint(sp.r2.z),
                         radii + o);
            } else if (COLOUR != 0 && !((ABL & ABL_REC) && abl_spec)) {
                // Every pair's records are stored, zeros for a pair that is not visible (nothing reads those): a warp then
                // writes whole 32-byte sectors.  Skipping the invisible lanes left sectors half written, which L2 has to
                // complete with a DRAM read before it can write them back.
                const bool vis = sp.radius > 0;
                const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
                rec0[o] = vis ? sp.r0 : z;
                rec1[o] = vis ? sp.r1 : z;
                rec2[o] = vis ? sp.r2 : z;
            } else if (COLOUR == 0 && sp.radius > 0) {
                // the colour words (rec1.zw, rec2.x) belong to k_sh_colour, which may be running right now
                rec0[o] = sp.r0;
                *reinterpret_cast<float2 *>(&rec1[o]) = make_float2(sp.r1.x, sp.r1.y);
                reinterpret_cast<float *>(&rec2[o])[1] = sp.r2.y;
                reinterpret_cast<float2 *>(&rec2[o])[1] = make_float2(sp.r2.z, sp.r2.w);
            }
            if ((ABL & ABL_RRM) && abl_spec) {
                abl_sink((uint32_t)sp.radius ^ sp.meta ^ sp.rect.x ^ ((uint32_t)sp.rect.y << 8) ^ ((uint32_t)sp.rect.z << 16) ^
                             ((uint32_t)sp.rect.w << 24),
                         radii + o);
            } else {
                radii[o] = sp.radius;
                if (!fused) rects[o] = sp.rect;
            }
            // Hand this Gaussian to every (view, tile) list it joins.  Exact path: count it (RED.ADD, no return;
            // k_emit_buckets appends it later, once the offsets are known).  Speculative path: append it now to the
            // tile's fixed-capacity sub-bucket; an entry beyond the capacity is dropped and the overflow is detected
            // from the cursor by k_spec_check (the call is then redone on the exact path).  Sub-bucket
            // i % BIN_SUB, one counter per 32-byte sector -- see gs_binning.cu.  (With very many (view, tile) buckets the
            // fused appends of all views thrash L2; gs_forward then passes counters = NULL and emits per view instead.)
            if (emit.counters) {
                const int w = sp.rect.z - sp.rect.x, nt = w * (sp.rect.w - sp.rect.y);
                const uint32_t tbase = (uint32_t)v * (uint32_t)c.ntiles;
                uint32_t sub = (uint32_t)i & (BIN_SUB - 1);
                if (emit.strata && !emit.strata_per_tile) {
                    sub = 0;
#pragma unroll
                    for (int q = 0; q < BIN_SUB - 1; q++) sub += sp.r2.y >= sm->strata[vi][q] ? 1u : 0u;
                }
                if (emit.bucket) {
                    // The cursor atomics return the slot to write, an L2 round trip each (the largest stall when
                    // the store followed its atomic directly).  Candidates go EMIT_BATCH at a time,
                    // all their atomics in flight together, and the dependent stores are deferred until the next batch
                    // is about to be issued -- normally one whole view of arithmetic later.
                    // candidates in row-major order of the rectangle; (cx, cy) walks it without the integer division
                    // that t / w cost per candidate (the emission loop is a large share of this kernel's instructions)
                    int cx = sp.rect.x, cy = sp.rect.y;
                    uint32_t abl_acc = 0;
                    for (int t0 = 0; t0 < nt; t0 += EMIT_BATCH) {
                        bool ok[EMIT_BATCH];
                        uint32_t slot[EMIT_BATCH];
#pragma unroll
                        for (int k = 0; k < EMIT_BATCH; k++) {
                            ok[k] = cy < (int)sp.rect.w && ((ABL & ABL_TESTS) || gs_tile_reached(sp.r0, sp.r1, sp.r2, cx, cy));
                            const uint32_t tile = tbase + (uint32_t)(cy * c.gx + cx);
                            // per-tile boundaries (clouds whose tiles each see a narrow depth range): the candidate
                            // tile's own eight floats decide the stratum
                            const uint32_t subk = (emit.strata_per_tile && ok[k]) ? gs_tile_stratum(emit.strata, tile, sp.r2.y) : sub;
                            slot[k] = tile * BIN_SUB + subk;
                            if (++cx == (int)sp.rect.z) {
                                cx = sp.rect.x;
                                cy++;
                            }
                        }
                        if (ABL & ABL_EMIT) {
#pragma unroll
                            for (int k = 0; k < EMIT_BATCH; k++) abl_acc ^= ok[k] ? slot[k] : 0u;
                            continue;
                        }
                        flush_pending();
                        pend_key = ((uint64_t)__float_as_uint(sp.r2.y) << 32) | (uint32_t)i;
#pragma unroll
                        for (int k = 0; k < EMIT_BATCH; k++) {
                            pend_ok[k] = ok[k];
                            pend_slot[k] = slot[k];
                            if (ok[k]) pend_pos[k] = atomicAdd(&emit.counters[(size_t)slot[k] * BIN_PAD], 1u);
                        }
                    }
                    if (ABL & ABL_EMIT) abl_sink(abl_acc, radii + o);
                } else {
                    for (int ty = sp.rect.y; ty < (int)sp.rect.w; ty++)
                        for (int tx = sp.rect.x; tx < (int)sp.rect.z; tx++)
                            if (gs_tile_reached(sp.r0, sp.r1, sp.r2, tx, ty))
                                atomicAdd(&emit.counters[(size_t)((tbase + (uint32_t)(ty * c.gx + tx)) * BIN_SUB + sub) * BIN_PAD], 1u);
                }
            }
            if (!((ABL & ABL_RRM) && abl_spec)) meta[o] = (uint8_t)sp.meta;
        }
    }
    flush_pending();
}

// ---------------------------------------------------------------------------------------------------------
// k_sh_colour: the colour words of the splat records, computed apart from the geometry (gs_render_host's split pipeline)
// ---------------------------------------------------------------------------------------------------------
// With host buffers the SH block is 88 % of the bytes that cross PCIe, and geometry + binning + the tile sort need none
// of it.  gs_render_host therefore runs k_preprocess in geometry-only mode (COLOUR = 0) followed by the tile sort on the
// launch stream, while THIS kernel, on a second stream, pulls the SH rows straight out of the caller's pinned buffer
// (16-byte pieces at the rows' own stride, as k_preprocess's sh_raw16 mode) and writes rec1.zw / rec2.x; the compositor
// waits for both.  Link-bound by design: a persistent grid of three CTAs per SM keeps ~11 MB of host reads in flight (see
// launch_sh_colour for what that does to the geometry kernel on the same SMs, and why it is still the fastest).
// Same eval_sh / sh_view_dir as k_preprocess (pinned arithmetic): the split pipeline's images are bit-identical.
constexpr int SHC_THREADS = 128;
constexpr int SHC_VIEWS = 64;   // cameras staged at a time

template <bool B4 = false>   // B4: degree 4, all 25 coefficients of a row are pulled
__global__ void __launch_bounds__(SHC_THREADS, 3)
k_sh_colour(const DevCfg c, const float *__restrict__ means3D, const float *__restrict__ shs, float4 *__restrict__ rec1,
            float4 *__restrict__ rec2, uint8_t *__restrict__ clamp_out /* [V*P] or NULL */, const int blocks_per_scene) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float4 *cam_s = reinterpret_cast<float4 *>(smem_raw);                    // (campos xyz, scale) per staged view
    float *sh_s = reinterpret_cast<float *>(smem_raw + SHC_VIEWS * sizeof(float4));
    const int tid = threadIdx.x;
    constexpr int MSMAX = B4 ? 25 : 16;
    const uint32_t row_f = (uint32_t)c.M * 3u, want_f = (uint32_t)(c.M < MSMAX ? c.M : MSMAX) * 3u;
    const int total = blocks_per_scene * c.S;
    for (int blk = blockIdx.x; blk < total; blk += gridDim.x) {
        const int scene = blk / blocks_per_scene, g0 = (blk - scene * blocks_per_scene) * SHC_THREADS;
        const int n = min(SHC_THREADS, c.P - g0);
        const bool active = tid < n;
        const size_t sg = (size_t)scene * c.P + g0 + tid;
        __syncthreads();   // the previous block's rows and cameras have been read by everybody
        {
            const float *src = shs + ((size_t)scene * c.P + g0) * row_f;
            const uint32_t nfl = (uint32_t)n * row_f, nq = nfl >> 2;
            const float4 *src4 = reinterpret_cast<const float4 *>(src);
            for (uint32_t q = tid; q < nq; q += SHC_THREADS) {
                const uint32_t f0 = q << 2, r = f0 / row_f, c0 = f0 - r * row_f;
                if (c0 < want_f || c0 + 3u >= row_f) cp_async16(sh_s + f0, src4 + q);
            }
            for (uint32_t f = (nq << 2) + tid; f < nfl; f += SHC_THREADS)
                if (f % row_f < want_f) cp_async4(sh_s + f, src + f);
            cp_async_commit();
        }
        float3 mean = make_float3(0.f, 0.f, 0.f);
        if (active) mean = make_float3(means3D[sg * 3 + 0], means3D[sg * 3 + 1], means3D[sg * 3 + 2]);
        for (int v0 = 0; v0 < c.VPS; v0 += SHC_VIEWS) {
            const int nv = min(SHC_VIEWS, c.VPS - v0);
            if (v0) __syncthreads();
            for (int t = tid; t < nv; t += SHC_THREADS) {
                const int v = scene * c.VPS + v0 + t;
                cam_s[t] = make_float4(c.campos[v * 3 + 0], c.campos[v * 3 + 1], c.campos[v * 3 + 2], c.view_scale ? c.view_scale[v] : 1.0f);
            }
            if (v0 == 0) cp_async_wait<0>();
            __syncthreads();
            if (!active) continue;
            const float *sh = sh_s + (size_t)tid * row_f;
            for (int vi = 0; vi < nv; vi++) {
                const float4 cam = cam_s[vi];
                const size_t o = (size_t)(scene * c.VPS + v0 + vi) * c.P + g0 + tid;
                const float3 m = make_float3(mean.x * cam.w, mean.y * cam.w, mean.z * cam.w);
                const float cp[3] = {cam.x, cam.y, cam.z};
                uint32_t clamped = 0;
                const float3 rgb = eval_sh<B4>(c.deg, sh, sh_view_dir(m, cp), clamped);
                reinterpret_cast<float2 *>(&rec1[o])[1] = make_float2(rgb.x, rgb.y);
                reinterpret_cast<float *>(&rec2[o])[0] = rgb.z;
                if (clamp_out) clamp_out[o] = (uint8_t)clamped;
            }
        }
    }
}

__global__ void k_mark_visible(const DevCfg c, const float *__restrict__ means3D, uint8_t *__restrict__ present) {
    __shared__ ViewCam cam;
    const int v = blockIdx.y;
    load_view_cams(c, v, 1, &cam);
    __syncthreads();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= c.P) return;
    const size_t sg = (size_t)(v / c.VPS) * c.P + i;
    const float s = cam.scale;
    const float3 m = make_float3(means3D[sg * 3] * s, means3D[sg * 3 + 1] * s, means3D[sg * 3 + 2] * s);
    present[(size_t)v * c.P + i] = xform4x3(cam.view, m).z > c.near_cull_z;
}

}  // namespace

int launch_preprocess(const DevCfg &c, const DevInputs &in, float4 *rec0, float4 *rec1, float4 *rec2, uint8_t *meta,
                      int32_t *radii, ushort4 *rects, const PreEmit &emit, cudaStream_t st, int g_begin, int g_end,
                      int variant, const DepthMode &dm) {
    if (g_end < 0) g_end = c.P;
    if (g_end <= g_begin) return GS_OK;
    const bool more_ctas = (variant & 1) != 0;
    dim3 grid((g_end - g_begin + PRE_THREADS - 1) / PRE_THREADS, c.S);
    // M > 16, on request: 16-byte pieces at the rows' own stride -- if every CTA's block starts 16-byte aligned (CTAs cover
    // 128 rows = 1536 M bytes, so the first one decides -- per scene); else the compacting 4-byte gather
    int sh_raw16 = 0;
    if (in.shs && c.M > 16 && (variant & 2) && !(variant & 4)) {
        const uintptr_t first = reinterpret_cast<uintptr_t>(in.shs) + (size_t)g_begin * c.M * 12;
        sh_raw16 = (first & 15u) == 0 && (c.S == 1 || ((size_t)c.P * c.M * 12) % 16 == 0);
    }
    // degree 4 evaluates (and stages) 25 coefficients per Gaussian: the B4 kernel
    const bool b4 = in.shs && !(variant & 4) && c.deg > 3;
    if (b4 && more_ctas)
        return gs_set_error(GS_ERR_INVALID, "GS_TUNE_PRE_OCC6 has no degree-4 kernel (sh_eval_max_degree = 4)");
    const int max_rs = b4 ? 75 : 49;   // floats per compacted row
    const size_t smem = PRE_SMEM_HDR + ((in.shs && !(variant & 4)) ? (size_t)PRE_THREADS * ((c.M <= (b4 ? 25 : 16) || sh_raw16) ? c.M * 3 : max_rs) * 4 : 0);
    if (smem > (size_t)227 * 1024) return gs_set_error(GS_ERR_INVALID, "too many SH coefficients per Gaussian for the staging buffer");
    auto launch = [&](auto kern) -> int {
        GS_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kern<<<grid, PRE_THREADS, smem, st>>>(c, in, rec0, rec1, rec2, meta, radii, rects, emit, g_begin, g_end, sh_raw16, dm);
        return GS_OK;
    };
    // anti-aliasing: the AA kernels, at 5 CTAs per SM only
    const bool aa = (c.flags & GS_FLAG_ANTIALIAS) != 0;
    if (aa && more_ctas)
        return gs_set_error(GS_ERR_INVALID, "GS_TUNE_PRE_OCC6 has no anti-aliased kernel (GS_FLAG_ANTIALIAS)");
    int rc;
    if (aa) {
        const bool fz = dm.mode != GS_DEPTH_Z;
        if (variant & 4) rc = fz ? launch(k_preprocess<0, 5, false, true, true>) : launch(k_preprocess<0, 5, false, false, true>);
        else if (b4) rc = fz ? launch(k_preprocess<2, 5, true, true, true>) : launch(k_preprocess<2, 5, true, false, true>);
        else if (in.shs) rc = fz ? launch(k_preprocess<2, 5, false, true, true>) : launch(k_preprocess<2, 5, false, false, true>);
        else rc = fz ? launch(k_preprocess<1, 5, false, true, true>) : launch(k_preprocess<1, 5, false, false, true>);
    } else if (dm.mode != GS_DEPTH_Z) {   // rec2.w = f(z): the FZ kernels
        if (variant & 4) rc = more_ctas ? launch(k_preprocess<0, 6, false, true>) : launch(k_preprocess<0, 5, false, true>);
        else if (b4) rc = launch(k_preprocess<2, 5, true, true>);
        else if (in.shs) rc = more_ctas ? launch(k_preprocess<2, 6, false, true>) : launch(k_preprocess<2, 5, false, true>);
        else rc = more_ctas ? launch(k_preprocess<1, 6, false, true>) : launch(k_preprocess<1, 5, false, true>);
    } else if (variant & 4) rc = more_ctas ? launch(k_preprocess<0, 6>) : launch(k_preprocess<0, 5>);   // geometry only
    else if (b4) rc = launch(k_preprocess<2, 5, true>);
    else if (in.shs) rc = more_ctas ? launch(k_preprocess<2, 6>) : launch(k_preprocess<2, 5>);
    else rc = more_ctas ? launch(k_preprocess<1, 6>) : launch(k_preprocess<1, 5>);
    if (rc != GS_OK) return rc;
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}

bool sh_colour_supported(const DevCfg &c, const DevInputs &in) {
    return in.shs && c.M > 16 && (reinterpret_cast<uintptr_t>(in.shs) & 15u) == 0 &&
           (c.S == 1 || ((size_t)c.P * c.M * 12) % 16 == 0) &&
           SHC_VIEWS * sizeof(float4) + (size_t)SHC_THREADS * c.M * 12 <= (size_t)72 * 1024;
}

int launch_sh_colour(const DevCfg &c, const DevInputs &in, float4 *rec1, float4 *rec2, uint8_t *clamp_out, cudaStream_t st) {
    if (c.P == 0 || c.V == 0) return GS_OK;
    if (!sh_colour_supported(c, in)) return gs_set_error(GS_ERR_INVALID, "k_sh_colour: unsupported SH layout");
    static int sms_of_device[64] = {};
    int dev = 0;
    GS_CUDA_OK(cudaGetDevice(&dev));
    if (dev >= 0 && dev < 64 && sms_of_device[dev] == 0)
        GS_CUDA_OK(cudaDeviceGetAttribute(&sms_of_device[dev], cudaDevAttrMultiProcessorCount, dev));
    const int sms = (dev >= 0 && dev < 64 && sms_of_device[dev] > 0) ? sms_of_device[dev] : 132;
    const int bps = (c.P + SHC_THREADS - 1) / SHC_THREADS;
    const long long total = (long long)bps * c.S;
    // Three CTAs per SM, each issuing its block's pieces all at once: the link wants its reads deep.  An SM with host reads
    // in flight slows all its other memory instructions, so geometry ends with the pull and the sort runs after it.
    // Shallower pulls (fewer pieces per thread or fewer CTAs), per-row bulk copies, fewer SMs pulling, or holding the
    // reads back until geometry + sort are done all hid those kernels but slowed the pull by more than they take on
    // C2: the pull at full rate wins.
    const int per_sm = 3;
    const int grid = (int)(total < (long long)sms * per_sm ? total : (long long)sms * per_sm);
    const size_t smem = SHC_VIEWS * sizeof(float4) + (size_t)SHC_THREADS * c.M * 12;
    auto kern = c.deg > 3 ? k_sh_colour<true> : k_sh_colour<false>;
    GS_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<grid, SHC_THREADS, smem, st>>>(c, in.means3D, in.shs, rec1, rec2, clamp_out, bps);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}

int launch_mark_visible(const DevCfg &c, const float *means3D, uint8_t *present, cudaStream_t st) {
    if (c.P == 0) return GS_OK;
    dim3 grid((c.P + 255) / 256, c.V);
    k_mark_visible<<<grid, 256, 0, st>>>(c, means3D, present);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}
