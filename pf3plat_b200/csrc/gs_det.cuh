// gs_det.cuh -- exact fixed-point accumulation for the deterministic backward (GS_FLAG_DETERMINISTIC, DESIGN.md 5.11).
//
// A float term t becomes the integer N = round(t * 2^GS_DET_E) (to nearest, ties to even), held as three signed limbs of
// GS_DET_LIMB_BITS bits: N = L0 + L1 2^42 + L2 2^84, every limb carrying the sign of t.  A float's 24-bit mantissa
// touches at most two limbs.  The limbs of many terms are added with 64-bit integer adds, whose result does not
// depend on their order; each limb has 63 - 42 = 21 bits of headroom, i.e. room for 2^21 - 1 terms.
//
//   range       |t| < 2^GS_DET_RANGE_LOG2 = 2^45 per term
//   resolution  2^-GS_DET_E = 2^-80 per term (a term below 2^-81 in magnitude contributes nothing)
//
// A term that is NaN, +-Inf or outside the range has no encoding: gs_det_encode returns false and the caller sets the
// component's bit in a poison mask instead (an idempotent OR), so that the decoded sum is NaN, as the float sum would
// have been non-finite.  gs_det_decode normalises the carries in integer arithmetic and rounds the exact sum ONCE to
// float (to nearest, ties to even).
//
// Everything here is __host__ __device__ so that a CPU test can compile and exercise it.
#pragma once
#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#define GS_DET_HD __host__ __device__ __forceinline__
#else
#define GS_DET_HD inline
#endif

#define GS_DET_E 80
#define GS_DET_LIMB_BITS 42
#define GS_DET_LIMBS 3
#define GS_DET_RANGE_LOG2 45
#define GS_DET_MAX_TERMS (1 << 21)  // exclusive bound on the terms one accumulator may receive

GS_DET_HD uint32_t gs_det_f2u(float v) {
#if defined(__CUDA_ARCH__)
    return __float_as_uint(v);
#else
    uint32_t b;
    memcpy(&b, &v, 4);
    return b;
#endif
}

GS_DET_HD float gs_det_u2f(uint32_t b) {
#if defined(__CUDA_ARCH__)
    return __uint_as_float(b);
#else
    float v;
    memcpy(&v, &b, 4);
    return v;
#endif
}

GS_DET_HD int gs_det_clz64(uint64_t x) {  // x != 0
#if defined(__CUDA_ARCH__)
    return __clzll((long long)x);
#else
    return __builtin_clzll(x);
#endif
}

// The limbs of one term.  Returns false (limbs all zero) when the term has no encoding: NaN, +-Inf, |t| >= 2^45.
GS_DET_HD bool gs_det_encode(float t, long long limb[GS_DET_LIMBS]) {
    limb[0] = limb[1] = limb[2] = 0;
    const uint32_t b = gs_det_f2u(t);
    const uint32_t ef = (b >> 23) & 0xffu;
    if (ef >= 127u + GS_DET_RANGE_LOG2) return false;
    uint64_t m = b & 0x7fffffu;
    int e = -149;  // t = m 2^e
    if (ef) {
        m |= 0x800000u;
        e = (int)ef - 150;
    }
    const int sh = e + GS_DET_E;  // N = m 2^sh
    const uint64_t mask = (1ull << GS_DET_LIMB_BITS) - 1;
    uint64_t mag[GS_DET_LIMBS] = {0, 0, 0};
    if (sh < 0) {
        // below the resolution: round to the nearest integer, ties to even (m < 2^24, so r >= 25 always rounds to 0)
        const int r = -sh;
        if (r <= 24) {
            uint64_t q = m >> r;
            const uint64_t rem = m & ((1ull << r) - 1), half = 1ull << (r - 1);
            if (rem > half || (rem == half && (q & 1u))) q++;
            mag[0] = q;
        }
    } else {
#pragma unroll
        for (int k = 0; k < GS_DET_LIMBS; k++) {
            const int s = sh - GS_DET_LIMB_BITS * k;
            if (s >= 0) mag[k] = s < GS_DET_LIMB_BITS ? (m << s) & mask : 0;
            else mag[k] = -s < 64 ? (m >> -s) & mask : 0;
        }
    }
    const bool neg = (b >> 31) != 0;
#pragma unroll
    for (int k = 0; k < GS_DET_LIMBS; k++) limb[k] = neg ? -(long long)mag[k] : (long long)mag[k];
    return true;
}

namespace gs_det_detail {
// carries of a limb into the next one: afterwards a0, a1 are in [0, 2^42)
GS_DET_HD void carry(long long &a0, long long &a1, long long &a2) {
    const long long one = 1ll << GS_DET_LIMB_BITS;
    long long c = a0 >> GS_DET_LIMB_BITS;  // arithmetic shift: floor division
    a0 -= c * one;
    a1 += c;
    c = a1 >> GS_DET_LIMB_BITS;
    a1 -= c * one;
    a2 += c;
}
// bits [lo, lo + 64) of X = u0 + u1 2^42 + u2 2^84 (non-negative, non-overlapping limbs)
GS_DET_HD uint64_t window(const uint64_t u[3], int lo) {
    uint64_t w = 0;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const int d = GS_DET_LIMB_BITS * k - lo;
        if (d >= 0) w |= d < 64 ? u[k] << d : 0;
        else w |= -d < 64 ? u[k] >> -d : 0;
    }
    return w;
}
// whether any bit of X below bit lo is set
GS_DET_HD bool sticky(const uint64_t u[3], int lo) {
    bool s = false;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const int nb = lo - GS_DET_LIMB_BITS * k;  // bits of limb k below lo
        if (nb <= 0) continue;
        s |= nb >= GS_DET_LIMB_BITS ? u[k] != 0 : (u[k] & ((1ull << nb) - 1)) != 0;
    }
    return s;
}
}  // namespace gs_det_detail

// The sum the limbs hold, times 2^-80, rounded once to float (nearest, ties to even); NaN when poisoned.
GS_DET_HD float gs_det_decode(const long long limb[GS_DET_LIMBS], bool poisoned) {
    if (poisoned) return gs_det_u2f(0x7fffffffu);
    long long a0 = limb[0], a1 = limb[1], a2 = limb[2];
    gs_det_detail::carry(a0, a1, a2);
    const bool neg = a2 < 0;
    if (neg) {  // magnitude: negate the normalised value and normalise again
        a0 = -a0;
        a1 = -a1;
        a2 = -a2;
        gs_det_detail::carry(a0, a1, a2);
    }
    const uint64_t u[3] = {(uint64_t)a0, (uint64_t)a1, (uint64_t)a2};
    int top;  // index of the leading bit
    if (u[2]) top = 2 * GS_DET_LIMB_BITS + 63 - gs_det_clz64(u[2]);
    else if (u[1]) top = GS_DET_LIMB_BITS + 63 - gs_det_clz64(u[1]);
    else if (u[0]) top = 63 - gs_det_clz64(u[0]);
    else return 0.0f;
    uint64_t m;
    int lo;  // value = m 2^(lo - 80)
    if (top < 24) {
        m = u[0];
        lo = 0;
    } else {
        // 24 significant bits, the rounding bit below them, and whether anything below that is set
        const int rb = top - 24;
        const uint64_t w = gs_det_detail::window(u, rb) & ((1ull << 25) - 1);
        m = w >> 1;
        if ((w & 1u) && (gs_det_detail::sticky(u, rb) || (m & 1u))) m++;
        lo = rb + 1;
    }
    // m <= 2^24 converts exactly; 2^(lo - 80) is a normal float for every reachable lo (-80 .. 124)
    const float scale = gs_det_u2f((uint32_t)(127 + lo - GS_DET_E) << 23);
    const float r = (float)m * scale;
    return neg ? -r : r;
}
