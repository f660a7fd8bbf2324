// gs_composite_bwd.cu -- stage 1 of the backward: per-pixel reverse walk, gradients scattered to per-(view,
// Gaussian) accumulators.
//
// Semantics: SURVEY.md Appendix A "Composite backward" (upstream renderCUDA backward): starting at the last
// contributor, recompute alpha, T <- T/(1-alpha), and accumulate dL/d{colour, mean2D, conic, opacity}; the
// gradient passes straight through the 0.99 clamp; the conic's off-diagonal term is stored once.
//
// Design (DESIGN.md section 5.4).  Same CTA/warp/pixel mapping and the same ballot culling as the forward
// (so both walk identical survivor sets).  Upstream issues 9 global float atomics per (pixel, Gaussian) pair;
// here the 32 pixel lanes of a warp keep their 10 partial gradients for up to THREE Gaussians in registers
// (30 values), transpose them through a per-warp shared-memory buffer so that lane L ends up holding the
// warp total of value L, and ONE red.global.add.f32 instruction with 30 distinct addresses retires them:
// one atomic instruction per three Gaussians per warp instead of 288 atomics.  (The first version did the
// transpose-reduce with a 31-shuffle register butterfly: 124 instructions per group against 71 now.)
#include <type_traits>

#include "gs_common.cuh"

namespace {

constexpr int CB_THREADS = 256;
constexpr int CB_BATCH_MAX = 256;
constexpr int CB_GROUP = 3;  // Gaussians reduced together (3 * GS_ACC_STRIDE = 30 values <= 32 lanes)
constexpr int CB_RED_STRIDE = 36;  // floats per row of the transpose buffer: 16-byte aligned rows, conflict-free LDS.128

// Shared memory of one CTA (dynamic: 61 KB).
template <int CB_BATCH>
struct CbSmem {
    float4 rec[2][CB_BATCH][3];                       // rec0 | rec1 | rec2, read as warp-wide broadcasts (double-buffered)
    float red[CB_THREADS / 32][CB_GROUP * GS_ACC_STRIDE][CB_RED_STRIDE];  // per-warp transpose buffer of the reduction
    uint32_t id[2][CB_BATCH];                         // Gaussian index of every staged entry (target of the atomics)
    uint32_t max[CB_THREADS / 32];
};

// Per-pixel state of the reverse walk.
struct PixState {
    float T, T_final, last_alpha;
    float accum[3], last_color[3];
    float accum_d, last_d;
    float dLp[3], dLd, bg_dot;
    uint32_t last;  // number of list entries this pixel walked up to its last contributor
};

// Returns whether this pixel received the Gaussian (and hence wrote non-trivial partial gradients to g).
// DEPTH: as k_composite_fwd (2: the depth value is rec2.w)
template <int DEPTH>
__device__ __forceinline__ bool pixel_grad(PixState &ps, bool live, uint32_t rec_addr, float pxf, float pyf,
                                           float half_w, float half_h, float *g /* [GS_ACC_STRIDE] */) {
#pragma unroll
    for (int k = 0; k < GS_ACC_STRIDE; k++) g[k] = 0.f;
    const float4 q0 = lds128(rec_addr), q1 = lds128(rec_addr + 16u);
    const float dx = q0.x - pxf, dy = q0.y - pyf;
    const float p2 = gs_power2(q0.z, q0.w, q1.x, dx, dy);
    const float G = gs_ex2(p2);
    const float alpha = fminf(GS_ALPHA_MAX, q1.y * G);
    // one divergent region: the test above is evaluated by all lanes unconditionally
    if (!(live && p2 <= 0.0f && alpha >= GS_ALPHA_MIN)) return false;
    const float2 q2 = lds64(rec_addr + 32u);  // (b, z)
    // one approximate reciprocal (MUFU.RCP, <= 1 ulp) serves both divisions by (1 - alpha); the IEEE divisions
    // upstream uses cost ~10 instructions each and the 1e-3 gradient tolerance does not need them
    const float inv_1ma = gs_rcp(1.0f - alpha);
    ps.T *= inv_1ma;
    const float w = alpha * ps.T;
    const float keep = 1.0f - ps.last_alpha;
    const float col[3] = {q1.z, q1.w, q2.x};
    float dL_dalpha = 0.f;
#pragma unroll
    for (int ch = 0; ch < 3; ch++) {
        ps.accum[ch] = fmaf(ps.last_alpha, ps.last_color[ch], keep * ps.accum[ch]);
        ps.last_color[ch] = col[ch];
        dL_dalpha = fmaf(col[ch] - ps.accum[ch], ps.dLp[ch], dL_dalpha);
        g[ch] = w * ps.dLp[ch];
    }
    if (DEPTH) {
        const float dz = DEPTH == 2 ? lds32(rec_addr + 44u) : q2.y;
        ps.accum_d = fmaf(ps.last_alpha, ps.last_d, keep * ps.accum_d);
        ps.last_d = dz;
        dL_dalpha = fmaf(dz - ps.accum_d, ps.dLd, dL_dalpha);
        g[9] = w * ps.dLd;
    }
    ps.last_alpha = alpha;
    dL_dalpha = fmaf(dL_dalpha, ps.T, -(ps.T_final * inv_1ma) * ps.bg_dot);
    // With s = G dL/dalpha (the opacity gradient; dL/dG = o dL/dalpha passes straight through the 0.99 clamp) and
    // m = -0.5 o s, written in the pre-scaled conic (A = -2 ln2 hA, B = -ln2 nB, C = -2 ln2 hC):
    //   dL/dconic = m (dx^2, dx dy, dy^2)
    //   dL/dmean2D = m (-2 ln2) (W/2 (2 hA dx + nB dy), H/2 (2 hC dy + nB dx))
    const float sgrad = dL_dalpha * G;
    const float m = (-0.5f * q1.y) * sgrad;
    const float mdx = m * dx, mdy = m * dy;
    g[3] = (m * (-2.0f * 0.6931471805599453f * half_w)) * fmaf(q0.z + q0.z, dx, q0.w * dy);
    g[4] = (m * (-2.0f * 0.6931471805599453f * half_h)) * fmaf(q1.x + q1.x, dy, q0.w * dx);
    g[5] = mdx * dx;
    g[6] = mdx * dy;
    g[7] = mdy * dy;
    g[8] = sgrad;
    return true;
}

// ALPHA: dL/d(accumulated opacity) per pixel joins the background term (GsAlpha; false is the kernel of before)
template <int DEPTH, int CB_BATCH, int MINB, bool ALPHA = false>
__global__ void __launch_bounds__(CB_THREADS, MINB)
k_composite_bwd_v1(const DevCfg c, const float4 *__restrict__ rec0, const float4 *__restrict__ rec1,
                const float4 *__restrict__ rec2, const uint32_t *__restrict__ point_list,
                const uint2 *__restrict__ ranges, const float *__restrict__ final_T,
                const uint32_t *__restrict__ n_contrib, const float *__restrict__ dL_dcolor,
                const float *__restrict__ dL_ddepth, float *__restrict__ acc, const float *__restrict__ dL_dalpha) {
    // double-buffered staging, as in the forward: the cp.async gathers of the next batch land in one buffer while the
    // warps walk the other
    extern __shared__ __align__(16) unsigned char cb_smem[];
    CbSmem<CB_BATCH> &sm = *reinterpret_cast<CbSmem<CB_BATCH> *>(cb_smem);
    auto &s_rec = sm.rec;
    auto &s_id = sm.id;
    auto &s_max = sm.max;

    const int v = blockIdx.y;
    const int tile = blockIdx.x;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int bx = (tile % c.gx) * GS_TILE + (warp & 1) * 8;
    const int by = (tile / c.gx) * GS_TILE + (warp >> 1) * 4;
    const int px = bx + (lane & 7), py = by + (lane >> 3);
    const bool inside = px < c.W && py < c.H;
    const float pxf = (float)px, pyf = (float)py;
    const float bx0 = (float)bx, bx1 = (float)(bx + 7), by0 = (float)by, by1 = (float)(by + 3);
    const float half_w = 0.5f * (float)c.W, half_h = 0.5f * (float)c.H;
    const uint32_t stage_addr = smem_u32(&s_rec[0][0][0]);
    constexpr uint32_t STAGE_BYTES = (uint32_t)sizeof(float4) * CB_BATCH * 3;

    const uint2 range = ranges[(size_t)v * c.ntiles + tile];
    const size_t rbase = (size_t)v * c.P;
    const size_t hw = (size_t)c.H * c.W;
    const size_t pix = (size_t)py * c.W + px;

    PixState ps;
    ps.last = 0;
    ps.T_final = 1.f;
    ps.dLp[0] = ps.dLp[1] = ps.dLp[2] = 0.f;
    ps.dLd = 0.f;
    if (inside) {
        ps.last = n_contrib[(size_t)v * hw + pix];
        ps.T_final = final_T[(size_t)v * hw + pix];
        const float *dl = dL_dcolor + (size_t)v * 3 * hw + pix;
        ps.dLp[0] = dl[0];
        ps.dLp[1] = dl[hw];
        ps.dLp[2] = dl[2 * hw];
        if (DEPTH && dL_ddepth) ps.dLd = dL_ddepth[(size_t)v * hw + pix];
    }
    ps.T = ps.T_final;
    ps.last_alpha = 0.f;
    ps.accum_d = ps.last_d = 0.f;
#pragma unroll
    for (int ch = 0; ch < 3; ch++) ps.accum[ch] = ps.last_color[ch] = 0.f;
    const float *bg = c.bg ? c.bg + (size_t)v * 3 : nullptr;
    ps.bg_dot = bg ? bg[0] * ps.dLp[0] + bg[1] * ps.dLp[1] + bg[2] * ps.dLp[2] : 0.f;
    // alpha = 1 - T_final: its gradient is the background's with dL/dalpha in place of -bg . dL/dC
    if (ALPHA && inside) ps.bg_dot -= dL_dalpha[(size_t)v * hw + pix];

    // the walk starts at the deepest position any pixel of the tile reached
    const uint32_t warp_last = __reduce_max_sync(0xffffffffu, ps.last);
    if (lane == 0) s_max[warp] = warp_last;
    __syncthreads();
    uint32_t cta_last = 0;
#pragma unroll
    for (int w = 0; w < CB_THREADS / 32; w++) cta_last = max(cta_last, s_max[w]);

    // batch k covers list positions [lo_k, hi_k), hi_k = cta_last - k * CB_BATCH, walked from the back
    const uint32_t nbatches = (cta_last + CB_BATCH - 1) / CB_BATCH;
    auto batch_lo = [&](uint32_t k) { const uint32_t hi = cta_last - k * CB_BATCH; return hi > CB_BATCH ? hi - CB_BATCH : 0u; };
    auto load_id = [&](uint32_t k) -> uint32_t {
        if (k >= nbatches) return 0u;
        const uint32_t e = batch_lo(k) + tid;
        return e < cta_last - k * CB_BATCH ? point_list[range.x + e] : 0u;
    };
    auto gather = [&](uint32_t k, uint32_t id) {
        if (k < nbatches && batch_lo(k) + tid < cta_last - k * CB_BATCH) {
            const size_t r = rbase + id;
            float4 *dst = &s_rec[k & 1][tid][0];
            cp_async16(dst, rec0 + r);
            cp_async16(dst + 1, rec1 + r);
            cp_async16(dst + 2, rec2 + r);
            s_id[k & 1][tid] = id;
        }
        cp_async_commit();  // one group per batch, empty or not
    };
    gather(0, load_id(0));
    uint32_t id_next = load_id(1);
    for (uint32_t k = 0; k < nbatches; k++) {
        const uint32_t hi = cta_last - k * CB_BATCH, lo = batch_lo(k), nb = hi - lo;
        __syncthreads();  // batch k-1 fully consumed: its buffer may be overwritten
        gather(k + 1, id_next);
        id_next = load_id(k + 2);
        cp_async_wait<1>();  // this thread's part of batch k has landed ...
        __syncthreads();     // ... and so has everybody else's
        const uint32_t rec_addr = stage_addr + (k & 1u) * STAGE_BYTES;
        const uint32_t *sid = s_id[k & 1];
        if (lo >= warp_last) continue;  // nothing in this batch is below any of this warp's last contributors
        for (int chunk = (int)((nb - 1) & ~31u); chunk >= 0; chunk -= 32) {
            const uint32_t j = (uint32_t)chunk + lane;
            bool hit = false;
            if (j < nb && lo + j < warp_last) {
                const uint32_t a = rec_addr + j * 48u;
                const float4 g0 = lds128(a);
                hit = gs_box_reaches(g0.x, g0.y, g0.z, g0.w, lds32(a + 16u), lds32(a + 40u), bx0, bx1, by0, by1);
            }
            uint32_t mask = __ballot_sync(0xffffffffu, hit);
            while (mask) {
                float gv[CB_GROUP * GS_ACC_STRIDE];
                uint32_t gid[CB_GROUP];
                bool any_got = false;
#pragma unroll
                for (int slot = 0; slot < CB_GROUP; slot++) {
                    float *g = gv + slot * GS_ACC_STRIDE;
                    if (mask) {
                        const int b = 31 - __clz(mask);  // deepest first
                        mask &= ~(1u << b);
                        const uint32_t jj = (uint32_t)chunk + b;
                        gid[slot] = sid[jj];
                        any_got |= pixel_grad<DEPTH>(ps, lo + jj < ps.last, rec_addr + jj * 48u, pxf, pyf, half_w,
                                                     half_h, g);
                    } else {
                        gid[slot] = 0xffffffffu;
#pragma unroll
                        for (int k = 0; k < GS_ACC_STRIDE; k++) g[k] = 0.f;
                    }
                }
                if (!__any_sync(0xffffffffu, any_got)) continue;  // box hits that reached no pixel: nothing to add
                // Transpose-reduce through shared memory: every lane stores its 30 partial values down a column
                // (row = value, column = lane; conflict-free), then lane r < 30 adds up row r with eight 16-byte loads.
                // 30 STS + 8 LDS.128 + 31 FADD per group, against 31 SHFL + 62 FSEL + 31 FADD for a register butterfly.
                float *red = &sm.red[warp][0][0];
                __syncwarp();  // the previous group's row sums have been read
#pragma unroll
                for (int k = 0; k < CB_GROUP * GS_ACC_STRIDE; k++) red[k * CB_RED_STRIDE + lane] = gv[k];
                __syncwarp();
                float total = 0.f;
                if (lane < CB_GROUP * GS_ACC_STRIDE) {
                    const float4 *row = reinterpret_cast<const float4 *>(red + lane * CB_RED_STRIDE);
                    float4 t = row[0];
#pragma unroll
                    for (int q = 1; q < 8; q++) {
                        const float4 u = row[q];
                        t.x += u.x; t.y += u.y; t.z += u.z; t.w += u.w;
                    }
                    total = (t.x + t.y) + (t.z + t.w);
                }
                const int slot = lane / GS_ACC_STRIDE, comp = lane - slot * GS_ACC_STRIDE;
                uint32_t id = gid[0];
                if (slot == 1) id = gid[1];
                if (slot == 2) id = gid[2];
                if (lane < CB_GROUP * GS_ACC_STRIDE && id != 0xffffffffu && total != 0.0f)
                    atomicAdd(acc + (rbase + id) * GS_ACC_STRIDE + comp, total);
            }
        }
    }
    cp_async_wait<0>();  // nothing of ours may still be in flight into shared memory when the CTA retires
}


// ---------------------------------------------------------------------------------------------------------
// v2 (round 2): pair matrices + dense per-Gaussian reduction
// ---------------------------------------------------------------------------------------------------------
// Where v1 spent its instructions (ncu, C2): 118 warp-instructions per (warp, survivor) -- ~60 of them the 10-component
// gradient arithmetic executed by 32 lanes of which 7.8 hold a live pixel, 24 the transpose-reduce of 30 values per
// three survivors.  v2 splits the work by what it depends on:
//   walk   (lanes = the 32 pixels of the warp's 8x4 block; one survivor per iteration, as before): recover T, and
//          produce the only two per-(pixel, Gaussian) scalars the gradients are linear in,
//              W = alpha * T                      (every colour/depth gradient is  sum_pix W * dL/dC_pix)
//              S = dL/dalpha * G                  (opacity, conic and mean2D gradients are moments of S over the pixels)
//          with dL/dalpha in the premultiplied suffix form  T*(c . dL/dC) - Y/(1-alpha),  Y = T_final*(bg . dL/dC) +
//          sum_{j behind} W_j (c_j . dL/dC): one running scalar instead of upstream's four-component accum_rec
//          recurrence (algebraically identical: accum_rec_i = sum_{j>i} W_j c_j / T_{i+1}).  (W, S) go into row `slot`
//          of a per-warp [16 slots][32 pixels] matrix in shared memory.
//   reduce (every 16 slots; lanes = (slot, half of the block)): each lane adds up ITS Gaussian's row against the
//          per-pixel dL/dC and the pixel offsets -- 16 pixels x 15 instructions, all 32 lanes busy, no cross-lane
//          traffic but one xor-16 exchange -- and five RED.ADD.F32 instructions (32 addresses each) retire the ten sums
//          of the 16 Gaussians.
// Same survivors, same skip decisions (gs_power2 / gs_ex2 shared with the forward), same accumulator layout as v1.
constexpr int CB2_NS = 16;                 // slots (survivors) per reduction
constexpr int CB2_ROW = 2 * 32 + 2;        // floats per slot row: 32 x (W, S) + 2 pad (conflict-free LDS.64 down a column)

template <int CB_BATCH>
struct Cb2Smem {
    float4 rec[2][CB_BATCH][3];
    uint32_t id[2][CB_BATCH];
    float pairs[CB_THREADS / 32][CB2_NS][CB2_ROW];
    float4 slot_a[CB_THREADS / 32][CB2_NS];   // (x, y, hA, nB) of the slot's Gaussian
    float4 slot_b[CB_THREADS / 32][CB2_NS];   // (hC, opacity, Gaussian index as bits, -)
    float4 dl[CB_THREADS / 32][32];           // per pixel of the block: dL/dC (rgb), dL/ddepth
    uint32_t max[CB_THREADS / 32];
};

// DET (GS_FLAG_DETERMINISTIC): the ten sums of a (warp, Gaussian) -- already independent of scheduling, they depend only
// on the order of the tile list -- are added into exact fixed-point accumulators (gs_det.cuh) with 64-bit integer REDs
// instead of float REDs, so the totals do not depend on the order in which warps arrive.  A term with no encoding
// (non-finite, out of range) sets its component's bit in the poison mask.  DET = false is the default kernel,
// instruction for instruction (the two trailing parameters are unused).  DEPTH: as k_composite_fwd (2: the depth term of
// dL/dalpha takes rec2.w).  ALPHA: dL/d(accumulated opacity) per pixel joins the background term Y (GsAlpha; false is the
// kernel of before, instruction for instruction).
template <int DEPTH, int CB_BATCH, int MINB, bool DET = false, bool ALPHA = false>
__global__ void __launch_bounds__(CB_THREADS, MINB)
k_composite_bwd(const DevCfg c, const float4 *__restrict__ rec0, const float4 *__restrict__ rec1,
                const float4 *__restrict__ rec2, const uint32_t *__restrict__ point_list,
                const uint2 *__restrict__ ranges, const float *__restrict__ final_T,
                const uint32_t *__restrict__ n_contrib, const float *__restrict__ dL_dcolor,
                const float *__restrict__ dL_ddepth, float *__restrict__ acc,
                unsigned long long *__restrict__ det_acc, uint32_t *__restrict__ det_poison,
                const float *__restrict__ dL_dalpha) {
    extern __shared__ __align__(16) unsigned char cb_smem[];
    Cb2Smem<CB_BATCH> &sm = *reinterpret_cast<Cb2Smem<CB_BATCH> *>(cb_smem);
    auto &s_rec = sm.rec;
    auto &s_id = sm.id;

    const int v = blockIdx.y;
    const int tile = blockIdx.x;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int bx = (tile % c.gx) * GS_TILE + (warp & 1) * 8;
    const int by = (tile / c.gx) * GS_TILE + (warp >> 1) * 4;
    const int px = bx + (lane & 7), py = by + (lane >> 3);
    const bool inside = px < c.W && py < c.H;
    const float pxf = (float)px, pyf = (float)py;
    const float bx0 = (float)bx, bx1 = (float)(bx + 7), by0 = (float)by, by1 = (float)(by + 3);
    const uint32_t stage_addr = smem_u32(&s_rec[0][0][0]);
    constexpr uint32_t STAGE_BYTES = (uint32_t)sizeof(float4) * CB_BATCH * 3;

    const uint2 range = ranges[(size_t)v * c.ntiles + tile];
    const size_t rbase = (size_t)v * c.P;
    const size_t hw = (size_t)c.H * c.W;
    const size_t pix = (size_t)py * c.W + px;

    // per-pixel state of the reverse walk
    uint32_t last = 0;
    float T = 1.f, Y = 0.f;
    float4 dl = make_float4(0.f, 0.f, 0.f, 0.f);
    if (inside) {
        last = n_contrib[(size_t)v * hw + pix];
        T = final_T[(size_t)v * hw + pix];
        const float *dlp = dL_dcolor + (size_t)v * 3 * hw + pix;
        dl.x = dlp[0];
        dl.y = dlp[hw];
        dl.z = dlp[2 * hw];
        if (DEPTH && dL_ddepth) dl.w = dL_ddepth[(size_t)v * hw + pix];
        const float *bg = c.bg ? c.bg + (size_t)v * 3 : nullptr;
        if constexpr (ALPHA) {
            // alpha = 1 - T_final enters exactly as the background does, with dL/dalpha in place of -bg . dL/dC
            const float bg_dot = bg ? bg[0] * dl.x + bg[1] * dl.y + bg[2] * dl.z : 0.f;
            Y = T * (bg_dot - dL_dalpha[(size_t)v * hw + pix]);
        } else if (bg) Y = T * (bg[0] * dl.x + bg[1] * dl.y + bg[2] * dl.z);   // the background term of every dL/dalpha
    }
    sm.dl[warp][lane] = dl;

    const uint32_t warp_last = __reduce_max_sync(0xffffffffu, last);
    if (lane == 0) sm.max[warp] = warp_last;
    __syncthreads();
    uint32_t cta_last = 0;
#pragma unroll
    for (int w = 0; w < CB_THREADS / 32; w++) cta_last = max(cta_last, sm.max[w]);

    // ---- reduction of the filled slots: lane = (slot s, half h of the block's pixels) ----
    // Moments are taken in block-local pixel coordinates centred on the half's 8x2 pixels, (u, w) in {-3.5..3.5} x
    // {-0.5, 0.5}: the coordinates are immediates of the unrolled loop (FFMA with an immediate operand), and the shift
    // to the Gaussian's own offsets dx = X - u, dy = Yc - w happens once per slot:
    //   sum S dx^2 = X^2 M0 - 2 X Mu + Muu   etc.     |u| <= 3.5 keeps the cancellation below 1e-5 relative.
    float *pairs = &sm.pairs[warp][0][0];
    const int rs = lane & (CB2_NS - 1), rh = lane >> 4;
    const float half_w = 0.5f * (float)c.W, half_h = 0.5f * (float)c.H;
    auto reduce_slots = [&](int nslots) {
        __syncwarp();
        const float4 ga = sm.slot_a[warp][rs];   // (x, y, hA, nB)
        const float4 gb = sm.slot_b[warp][rs];   // (hC, opacity, index bits, -)
        const float *row = pairs + rs * CB2_ROW + 32 * rh;
        const float4 *dlh = &sm.dl[warp][16 * rh];
        float c0 = 0.f, c1 = 0.f, c2 = 0.f, cz = 0.f, M0 = 0.f, Mu = 0.f, Mw = 0.f, Muu = 0.f, Muw = 0.f, Mww = 0.f;
#pragma unroll
        for (int p = 0; p < 16; p++) {
            const float2 ws = *reinterpret_cast<const float2 *>(row + 2 * p);
            const float4 d = dlh[p];
            const float u = (float)(p & 7) - 3.5f, w = (float)(p >> 3) - 0.5f;
            c0 = fmaf(ws.x, d.x, c0);
            c1 = fmaf(ws.x, d.y, c1);
            c2 = fmaf(ws.x, d.z, c2);
            if (DEPTH) cz = fmaf(ws.x, d.w, cz);
            M0 += ws.y;
            Mu = fmaf(ws.y, u, Mu);
            Mw = fmaf(ws.y, w, Mw);
            Muu = fmaf(ws.y, u * u, Muu);
            Muw = fmaf(ws.y, u * w, Muw);
            Mww = fmaf(ws.y, w * w, Mww);
        }
        // offsets of the Gaussian from the centre of this half's pixels
        const float X = ga.x - (bx0 + 3.5f), Yc = ga.y - (by0 + 0.5f + (float)(2 * rh));
        const float m1 = fmaf(X, M0, -Mu);                                   // sum S dx
        const float m2 = fmaf(Yc, M0, -Mw);                                  // sum S dy
        const float m3 = fmaf(X, fmaf(X, M0, -2.0f * Mu), Muu);              // sum S dx^2
        const float m4 = fmaf(X, fmaf(Yc, M0, -Mw), fmaf(-Yc, Mu, Muw));     // sum S dx dy
        const float m5 = fmaf(Yc, fmaf(Yc, M0, -2.0f * Mw), Mww);            // sum S dy^2
        // dL/dmean2D (NDC-scaled), dL/dconic, dL/dopacity from the moments (see pixel_grad of v1 for the algebra)
        const float o = gb.y;
        float g3 = (o * 0.6931471805599453f * half_w) * fmaf(ga.z + ga.z, m1, ga.w * m2);
        float g4 = (o * 0.6931471805599453f * half_h) * fmaf(gb.x + gb.x, m2, ga.w * m1);
        const float mo = -0.5f * o;
        float g5 = mo * m3, g6 = mo * m4, g7 = mo * m5;
        // both halves of the block
        c0 += __shfl_xor_sync(0xffffffffu, c0, 16);
        c1 += __shfl_xor_sync(0xffffffffu, c1, 16);
        c2 += __shfl_xor_sync(0xffffffffu, c2, 16);
        g3 += __shfl_xor_sync(0xffffffffu, g3, 16);
        g4 += __shfl_xor_sync(0xffffffffu, g4, 16);
        g5 += __shfl_xor_sync(0xffffffffu, g5, 16);
        g6 += __shfl_xor_sync(0xffffffffu, g6, 16);
        g7 += __shfl_xor_sync(0xffffffffu, g7, 16);
        M0 += __shfl_xor_sync(0xffffffffu, M0, 16);
        if (DEPTH) cz += __shfl_xor_sync(0xffffffffu, cz, 16);
        if (rs < nslots) {
            // lanes of half 0 retire components 0-4, lanes of half 1 components 5-9: five RED instructions, 32 addresses each
            if constexpr (DET) {
                const size_t e = rbase + __float_as_uint(gb.z);
                unsigned long long *dst = det_acc + (e * GS_ACC_STRIDE + 5 * rh) * GS_DET_LIMBS;
                const float vals[5] = {rh ? g5 : c0, rh ? g6 : c1, rh ? g7 : c2, rh ? M0 : g3, rh ? cz : g4};
                uint32_t bad = 0;
#pragma unroll
                for (int q = 0; q < 5; q++) {
                    if (vals[q] == 0.f) continue;
                    long long limb[GS_DET_LIMBS];
                    if (!gs_det_encode(vals[q], limb)) {
                        bad |= 1u << (5 * rh + q);
                        continue;
                    }
#pragma unroll
                    for (int k = 0; k < GS_DET_LIMBS; k++)  // at most two of the three are non-zero
                        if (limb[k]) atomicAdd(dst + q * GS_DET_LIMBS + k, (unsigned long long)limb[k]);
                }
                if (bad) atomicOr(det_poison + e, bad);
            } else {
                float *dst = acc + (rbase + __float_as_uint(gb.z)) * GS_ACC_STRIDE + 5 * rh;
                const float v0 = rh ? g5 : c0, v1 = rh ? g6 : c1, v2 = rh ? g7 : c2, v3 = rh ? M0 : g3, v4 = rh ? cz : g4;
                if (v0 != 0.f) atomicAdd(dst + 0, v0);
                if (v1 != 0.f) atomicAdd(dst + 1, v1);
                if (v2 != 0.f) atomicAdd(dst + 2, v2);
                if (v3 != 0.f) atomicAdd(dst + 3, v3);
                if (v4 != 0.f) atomicAdd(dst + 4, v4);
            }
        }
        __syncwarp();  // the rows may be overwritten
    };

    const uint32_t nbatches = (cta_last + CB_BATCH - 1) / CB_BATCH;
    auto batch_lo = [&](uint32_t k) { const uint32_t hi = cta_last - k * CB_BATCH; return hi > CB_BATCH ? hi - CB_BATCH : 0u; };
    auto load_id = [&](uint32_t k) -> uint32_t {
        if (k >= nbatches) return 0u;
        const uint32_t e = batch_lo(k) + tid;
        return e < cta_last - k * CB_BATCH ? point_list[range.x + e] : 0u;
    };
    auto gather = [&](uint32_t k, uint32_t id) {
        if (k < nbatches && batch_lo(k) + tid < cta_last - k * CB_BATCH) {
            const size_t r = rbase + id;
            float4 *dst = &s_rec[k & 1][tid][0];
            cp_async16(dst, rec0 + r);
            cp_async16(dst + 1, rec1 + r);
            cp_async16(dst + 2, rec2 + r);
            s_id[k & 1][tid] = id;
        }
        cp_async_commit();  // one group per batch, empty or not
    };
    int fill = 0;
    gather(0, load_id(0));
    uint32_t id_next = load_id(1);
    for (uint32_t k = 0; k < nbatches; k++) {
        const uint32_t hi = cta_last - k * CB_BATCH, lo = batch_lo(k), nb = hi - lo;
        __syncthreads();  // batch k-1 fully consumed: its buffer may be overwritten
        gather(k + 1, id_next);
        id_next = load_id(k + 2);
        cp_async_wait<1>();  // this thread's part of batch k has landed ...
        __syncthreads();     // ... and so has everybody else's
        const uint32_t rec_addr = stage_addr + (k & 1u) * STAGE_BYTES;
        const uint32_t *sid = s_id[k & 1];
        if (lo >= warp_last) continue;  // nothing in this batch is below any of this warp's last contributors
        for (int chunk = (int)((nb - 1) & ~31u); chunk >= 0; chunk -= 32) {
            const uint32_t j = (uint32_t)chunk + lane;
            bool hit = false;
            if (j < nb && lo + j < warp_last) {
                const uint32_t a = rec_addr + j * 48u;
                const float4 g0 = lds128(a);
                hit = gs_box_reaches(g0.x, g0.y, g0.z, g0.w, lds32(a + 16u), lds32(a + 40u), bx0, bx1, by0, by1);
            }
            uint32_t mask = __ballot_sync(0xffffffffu, hit);
            // this pixel takes the entries at list positions < last, i.e. bits b < last - (lo + chunk) of this round
            const int rel_last = (int)min(32u, last - min(last, lo + (uint32_t)chunk));
            // (Prefetching the next survivor's records while the current one is worked on was tried and was slower -- the
            // extra live registers cost more than the shared-memory latency they hide.)
            while (mask) {
                const int b = 31 - __clz(mask);  // deepest first
                mask &= ~(1u << b);
                const uint32_t jj = (uint32_t)chunk + b;
                const uint32_t a = rec_addr + jj * 48u;
                const float4 q0 = lds128(a), q1 = lds128(a + 16u);
                const float dx = q0.x - pxf, dy = q0.y - pyf;
                const float p2 = gs_power2(q0.z, q0.w, q1.x, dx, dy);
                const float G = gs_ex2(p2);
                const float alpha = fminf(GS_ALPHA_MAX, q1.y * G);
                const bool live = b < rel_last && p2 <= 0.0f && alpha >= GS_ALPHA_MIN;
                float2 ws = make_float2(0.f, 0.f);
                if (live) {  // the one divergent region
                    const float2 q2 = lds64(a + 32u);  // (b, z)
                    // one approximate reciprocal (MUFU.RCP, <= 1 ulp) serves T/(1-alpha) and Y/(1-alpha)
                    const float inv = gs_rcp(1.0f - alpha);
                    T *= inv;
                    ws.x = alpha * T;
                    float cdot = fmaf(q2.x, dl.z, fmaf(q1.w, dl.y, q1.z * dl.x));
                    if (DEPTH) cdot = fmaf(DEPTH == 2 ? lds32(a + 44u) : q2.y, dl.w, cdot);
                    ws.y = fmaf(T, cdot, -(Y * inv)) * G;   // dL/dalpha * G (the gradient passes through the 0.99 clamp)
                    Y = fmaf(ws.x, cdot, Y);
                }
                if (!__any_sync(0xffffffffu, live)) continue;  // box hit that reached no pixel
                *reinterpret_cast<float2 *>(pairs + fill * CB2_ROW + 2 * lane) = ws;
                // every lane stores the same two words to the same address (no branch; one wins)
                sm.slot_a[warp][fill] = q0;
                sm.slot_b[warp][fill] = make_float4(q1.x, q1.y, __uint_as_float(sid[jj]), 0.f);
                if (++fill == CB2_NS) {
                    reduce_slots(CB2_NS);
                    fill = 0;
                }
            }
        }
    }
    if (fill) reduce_slots(fill);
    cp_async_wait<0>();  // nothing of ours may still be in flight into shared memory when the CTA retires
}

}  // namespace

int launch_composite_bwd(const DevCfg &c, const GsSaved &s, const float *dL_dcolor, const float *dL_ddepth,
                         float *grad_acc, cudaStream_t st, int variant, const DetAcc &det, const float *dL_dalpha) {
    if (c.V == 0 || c.ntiles == 0) return GS_OK;
    dim3 grid(c.ntiles, c.V);
    if (variant != 1) {
        // v2.  variant 0: batch of 256 entries, 68 KB of shared memory, 80 registers, 3 CTAs/SM;
        //      variant 2: batch of 128, 55 KB, registers bounded to 64 -> 4 CTAs/SM (the kernel is latency-bound at
        //      24 resident warps)
        auto launch = [&](auto kern, size_t smem) -> int {
            GS_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            kern<<<grid, CB_THREADS, smem, st>>>(c, s.rec0, s.rec1, s.rec2, s.point_list, s.ranges, s.final_T, s.n_contrib,
                                                 dL_dcolor, dL_ddepth, grad_acc, det.acc, det.poison, dL_dalpha);
            return GS_OK;
        };
        const bool dep = (c.flags & GS_FLAG_DEPTH) != 0;
        // A: an incoming alpha gradient (the ALPHA instantiations); without one, the kernels of before
        auto pick = [&](auto alpha_tag) -> int {
            constexpr bool A = decltype(alpha_tag)::value;
            if (dep && s.depth_mode != GS_DEPTH_Z) {   // the depth channel carried f(z) in rec2.w
                if (det.acc)
                    return variant == 2 ? launch(k_composite_bwd<2, 128, 4, true, A>, sizeof(Cb2Smem<128>)) : launch(k_composite_bwd<2, 256, 3, true, A>, sizeof(Cb2Smem<256>));
                return variant == 2 ? launch(k_composite_bwd<2, 128, 4, false, A>, sizeof(Cb2Smem<128>)) : launch(k_composite_bwd<2, 256, 3, false, A>, sizeof(Cb2Smem<256>));
            }
            if (det.acc) {
                if (variant == 2)
                    return dep ? launch(k_composite_bwd<1, 128, 4, true, A>, sizeof(Cb2Smem<128>)) : launch(k_composite_bwd<0, 128, 4, true, A>, sizeof(Cb2Smem<128>));
                return dep ? launch(k_composite_bwd<1, 256, 3, true, A>, sizeof(Cb2Smem<256>)) : launch(k_composite_bwd<0, 256, 3, true, A>, sizeof(Cb2Smem<256>));
            }
            if (variant == 2)
                return dep ? launch(k_composite_bwd<1, 128, 4, false, A>, sizeof(Cb2Smem<128>)) : launch(k_composite_bwd<0, 128, 4, false, A>, sizeof(Cb2Smem<128>));
            return dep ? launch(k_composite_bwd<1, 256, 3, false, A>, sizeof(Cb2Smem<256>)) : launch(k_composite_bwd<0, 256, 3, false, A>, sizeof(Cb2Smem<256>));
        };
        const int rc = dL_dalpha ? pick(std::true_type{}) : pick(std::false_type{});
        if (rc != GS_OK) return rc;
        GS_CUDA_OK(cudaGetLastError());
        return GS_OK;
    }
    if (det.acc) return gs_set_error(GS_ERR_INVALID, "the round-1 backward kernel has no deterministic mode");
    // Batch of 256 entries, registers unbounded (80 -> 3 CTAs/SM).  On C2 a batch of 128 with registers bounded
    // to 64 (4 CTAs/SM, 32 B of spills) and a batch of 128 at 3 CTAs/SM were both slower -- the kernel is issue-bound, more resident warps do not help it.
    constexpr int BATCH = CB_BATCH_MAX, MINB = 3;
    const size_t smem = sizeof(CbSmem<BATCH>);
    auto launch = [&](auto kern) -> int {
        GS_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kern<<<grid, CB_THREADS, smem, st>>>(c, s.rec0, s.rec1, s.rec2, s.point_list, s.ranges, s.final_T, s.n_contrib,
                                             dL_dcolor, dL_ddepth, grad_acc, dL_dalpha);
        return GS_OK;
    };
    const int rc = dL_dalpha ? (!(c.flags & GS_FLAG_DEPTH) ? launch(k_composite_bwd_v1<0, BATCH, MINB, true>)
                                : s.depth_mode == GS_DEPTH_Z ? launch(k_composite_bwd_v1<1, BATCH, MINB, true>)
                                                              : launch(k_composite_bwd_v1<2, BATCH, MINB, true>))
                   : !(c.flags & GS_FLAG_DEPTH) ? launch(k_composite_bwd_v1<0, BATCH, MINB>)
                   : s.depth_mode == GS_DEPTH_Z ? launch(k_composite_bwd_v1<1, BATCH, MINB>)
                                                 : launch(k_composite_bwd_v1<2, BATCH, MINB>);
    if (rc != GS_OK) return rc;
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}
