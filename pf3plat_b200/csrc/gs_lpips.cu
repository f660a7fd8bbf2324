// gs_lpips.cu -- LPIPS-VGG (the `lpips` package, version 0.1, net="vgg", lpips=True, spatial=False), forward and
// input gradients, for PF3plat's LossLpips (src/loss/loss_lpips.py:55-59) and compute_lpips
// (src/evaluation/metrics.py:27-33).  The weights are an input (gs_lpips_weights_create).
//
// Semantics per image pair (x0, x1):
//   x <- 2x - 1 if normalize;  x <- (x - shift) / scale                       (the package's ScalingLayer)
//   VGG16 features[0:30]: 13 conv3x3 (pad 1, bias) + ReLU, 2x2/2 max-pools (floor) before conv2_1, conv3_1, conv4_1,
//   conv5_1; taps f_l at relu1_2, relu2_2, relu3_3, relu4_3, relu5_3
//   n = f / (||f||_c + 1e-10) per pixel;  out = sum_l mean_{h,w} sum_c lin_l[c] (n0 - n1)^2
//
// Layout: activations are NHWC fp32 holding TF32-representable values (every epilogue that stores an operand of a
// later convolution rounds with cvt.rna); both images of every pair go through each layer in one launch (images
// 0..N-1 are in0, N..2N-1 are in1).  Kernels:
//   k_conv0_fwd / k_conv0_bwd  conv1_1 (Cin = 3, K = 27) on CUDA cores, with the scaling layer; its backward is dL/dx
//   k_conv3x3                 the 12 layers with Cin >= 64 as one implicit GEMM on tensor cores (mma.sync m16n8k8
//                             TF32): M = pixels of all images, N = Cout, K = 9 Cin.  The backward-data pass is the same
//                             kernel on weights rotated by 180 degrees with Cin/Cout swapped (packed once), its epilogue
//                             applying the ReLU mask of the layer below
//   k_pool / k_unpool_bwd     2x2 max-pool; its backward routes to the first maximum of each window, or to its last NaN
//                             (PyTorch's choice), adds the head's gradient of the tap and applies the tap's ReLU mask
//   k_head_fwd / k_head_bwd   one warp per pixel: channel norms, the lin-weighted squared difference, per-CTA fp64
//                             partial sums reduced in a fixed order by k_head_final; the backward's closed form below
// No atomics, no host synchronisation: results are bit-identical from run to run.
//
// BF16 path (GsLpipsConfig.precision = GS_LPIPS_BF16, opt-in): the same network with BF16 activations and BF16
// gradients between layers (round-to-nearest-even at every store), the mixed precision torch.autocast gives.  The kernels
// above are instantiated on the element type; the 12 convolutions with Cin >= 64 run k_conv3x3_wgmma instead: BF16 wgmma
// with fp32 accumulators, operands in 128-byte-swizzled shared memory, a cp.async producer warpgroup and two wgmma
// consumer warpgroups handing 4 stages back and forth through mbarriers.  conv1_1, the head and the pool keep fp32
// arithmetic; dL/din0 and dL/din1 are written in fp32.  Its weights are packed separately (gs_lpips_weights_pack_bf16).
//
// Non-finite inputs follow PyTorch's rules, so a NaN or Inf pixel gives the image a NaN distance and NaN gradients
// where autograd has them: ReLU and max-pool propagate NaN (max.NaN), ReLU's backward zeroes the gradient only where
// act <= 0 (a NaN activation passes it), and the max-pool backward routes to a NaN as described above.
//
// Head backward: with s = ||f||, n = f/(s+e), g = dL/dn:  dL/df = (g - n (n.g)(s+e)/s) / (s+e).  At s = 0 the second
// term's limit is 0 (|n (n.g)(s+e)/s| <= |g| s/(s+e)), so dL/df = g/e there (the derivative of f/(s+e) at f = 0);
// autograd's dL/df is NaN there (sqrt's backward at 0).  A tap pixel with s = 0 has every channel 0, so the ReLU mask
// drops that gradient before it reaches the layer below, on both sides.
#include "gs_common.cuh"

#include <cuda_bf16.h>

#include <algorithm>
#include <new>
#include <type_traits>
#include <utility>

namespace {

constexpr int LP_LAYERS = 13, LP_NTAPS = 5;
constexpr int LP_CIN[LP_LAYERS] = {3, 64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512};
constexpr int LP_COUT[LP_LAYERS] = {64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512, 512};
constexpr int LP_LEVEL[LP_LAYERS] = {0, 0, 1, 1, 2, 2, 2, 3, 3, 3, 4, 4, 4};  // resolution H >> level
constexpr int LP_TAP_OF[LP_LAYERS] = {-1, 0, -1, 1, -1, -1, 2, -1, -1, 3, -1, -1, 4};
constexpr int LP_TAP_C[LP_NTAPS] = {64, 128, 256, 512, 512};
constexpr bool lp_pooled_input(int l) { return l == 2 || l == 4 || l == 7 || l == 10; }
constexpr float LP_EPS = 1e-10f;
constexpr int LP_HEAD_BLOCKS = 32;  // CTAs per (tap, image) of the head's forward: fixed, so the sum order is too

__device__ __forceinline__ float tf32_round(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return __uint_as_float(r);
}

// max that returns NaN if either operand is NaN (PyTorch's relu and max_pool2d); otherwise the bits of fmaxf
__device__ __forceinline__ float max_nan(float a, float b) {
    float r;
    asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
}

// activation element types: float holding TF32 values (the default path) or bf16
using bf16 = __nv_bfloat16;
__device__ __forceinline__ float to_f(float x) { return x; }
__device__ __forceinline__ float to_f(bf16 x) { return __bfloat162float(x); }
// rounds a value that a later convolution reads as an operand: cvt.rna to TF32, or round-to-nearest-even to BF16
template <typename T> __device__ __forceinline__ T act_round(float x);
template <> __device__ __forceinline__ float act_round<float>(float x) { return tf32_round(x); }
template <> __device__ __forceinline__ bf16 act_round<bf16>(float x) { return __float2bfloat16_rn(x); }
template <typename T> __device__ __forceinline__ T act_zero() { return T(0.f); }
// 16 bytes of consecutive channels, the unit the pool kernels move
template <typename T> struct alignas(16) Act16 {
    static constexpr int E = 16 / sizeof(T);
    T e[E];
};
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
    const __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<const uint32_t *>(&v);
}

// ---------------------------------------------------------------------------------------------------------
// weight packing
// ---------------------------------------------------------------------------------------------------------
// forward [9 Cin][Cout] (k = (ky*3+kx)*Cin + ci) and backward-data [9 Cout][Cin] (the 180-degree rotation), TF32-rounded
__global__ void k_pack_conv(const float *__restrict__ w, int Cin, int Cout, float *__restrict__ fwd, float *__restrict__ rot) {
    const int64_t n = (int64_t)Cout * Cin * 9;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int tap = (int)(i % 9), ky = tap / 3, kx = tap % 3;
        const int ci = (int)((i / 9) % Cin), co = (int)(i / (9 * (int64_t)Cin));
        const float v = tf32_round(w[i]);
        fwd[((int64_t)tap * Cin + ci) * Cout + co] = v;
        rot[((int64_t)((2 - ky) * 3 + (2 - kx)) * Cout + co) * Cin + ci] = v;
    }
}

// BF16 (round-to-nearest-even from the fp32 weights), K-major for wgmma: forward [Cout][9 Cin] and backward-data
// [Cin][9 Cout] (the 180-degree rotation), k = tap * C + c in both
__global__ void k_pack_conv_bf16(const float *__restrict__ w, int Cin, int Cout, bf16 *__restrict__ fwd, bf16 *__restrict__ rot) {
    const int64_t n = (int64_t)Cout * Cin * 9;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int tap = (int)(i % 9), ky = tap / 3, kx = tap % 3;
        const int ci = (int)((i / 9) % Cin), co = (int)(i / (9 * (int64_t)Cin));
        const bf16 v = __float2bfloat16_rn(w[i]);
        fwd[((int64_t)co * 9 + tap) * Cin + ci] = v;
        rot[((int64_t)ci * 9 + (2 - ky) * 3 + (2 - kx)) * Cout + co] = v;
    }
}

// conv1_1: [27][64] with k = (ky*3+kx)*3 + c, full fp32 (CUDA cores)
__global__ void k_pack_conv0(const float *__restrict__ w, float *__restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 64 * 27) return;
    const int tap = i % 9, c = (i / 9) % 3, co = i / 27;
    out[(tap * 3 + c) * 64 + co] = w[i];
}

// ---------------------------------------------------------------------------------------------------------
// conv1_1 (Cin = 3) with the scaling layer
// ---------------------------------------------------------------------------------------------------------
constexpr int C0_THREADS = 256;

template <typename T>
__global__ void __launch_bounds__(C0_THREADS)
k_conv0_fwd(const float *__restrict__ in0, const float *__restrict__ in1, int64_t s0, int64_t s1, int N, int H, int W,
            int normalize, const float *__restrict__ w0, const float *__restrict__ b0, const float *__restrict__ shift,
            const float *__restrict__ scale, T *__restrict__ out) {
    __shared__ float sw[27 * 64], sb[64], ssh[3], ssc[3];
    for (int i = threadIdx.x; i < 27 * 64; i += C0_THREADS) sw[i] = w0[i];
    if (threadIdx.x < 64) sb[threadIdx.x] = b0[threadIdx.x];
    if (threadIdx.x < 3) { ssh[threadIdx.x] = shift[threadIdx.x]; ssc[threadIdx.x] = scale[threadIdx.x]; }
    __syncthreads();
    const int64_t HW = (int64_t)H * W, total = 2 * (int64_t)N * HW * 8;
    const int64_t t = (int64_t)blockIdx.x * C0_THREADS + threadIdx.x;
    if (t >= total) return;
    const int cg = (int)(t & 7);
    const int64_t pix = t >> 3;
    const int img = (int)(pix / HW), rem = (int)(pix - (int64_t)img * HW), y = rem / W, x = rem - y * W;
    const float *src = img < N ? in0 + (int64_t)img * s0 : in1 + (int64_t)(img - N) * s1;
    float acc[8];
#pragma unroll
    for (int o = 0; o < 8; o++) acc[o] = sb[cg * 8 + o];
#pragma unroll
    for (int tap = 0; tap < 9; tap++) {
        const int yy = y + tap / 3 - 1, xx = x + tap % 3 - 1;
        if (yy < 0 || yy >= H || xx < 0 || xx >= W) continue;  // zero padding of the scaled input
#pragma unroll
        for (int c = 0; c < 3; c++) {
            float v = src[c * HW + (int64_t)yy * W + xx];
            if (normalize) v = 2.f * v - 1.f;
            v = (v - ssh[c]) / ssc[c];
            const float *wr = sw + (tap * 3 + c) * 64 + cg * 8;
#pragma unroll
            for (int o = 0; o < 8; o++) acc[o] = fmaf(wr[o], v, acc[o]);
        }
    }
    if constexpr (std::is_same<T, float>::value) {
        float4 *dst = reinterpret_cast<float4 *>(out + pix * 64 + cg * 8);
#pragma unroll
        for (int o = 0; o < 8; o++) acc[o] = tf32_round(max_nan(acc[o], 0.f));
        dst[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
        dst[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
    } else {
#pragma unroll
        for (int o = 0; o < 8; o++) acc[o] = max_nan(acc[o], 0.f);
        *reinterpret_cast<uint4 *>(out + pix * 64 + cg * 8) = make_uint4(
            pack_bf16x2(acc[0], acc[1]), pack_bf16x2(acc[2], acc[3]), pack_bf16x2(acc[4], acc[5]), pack_bf16x2(acc[6], acc[7]));
    }
}

// dL/dx from g = dL/d(conv1_1 pre-activation) [nb][H][W][64]; images [0, nsplit) go to out0, the rest to out1
// (contiguous [., 3, H, W])
__device__ __forceinline__ void conv0_bwd_acc(float (&d)[3], const float4 *sw, int tap, int q, float4 gv) {
#pragma unroll
    for (int c = 0; c < 3; c++) {
        const float4 wv = sw[(tap * 3 + c) * 16 + q];
        d[c] = fmaf(wv.x, gv.x, fmaf(wv.y, gv.y, fmaf(wv.z, gv.z, fmaf(wv.w, gv.w, d[c]))));
    }
}

template <typename T>
__global__ void __launch_bounds__(C0_THREADS)
k_conv0_bwd(const T *__restrict__ g, int nb, int H, int W, const float *__restrict__ w0,
            const float *__restrict__ scale, float mul, float *__restrict__ out0, float *__restrict__ out1, int nsplit) {
    __shared__ float4 sw[27 * 16];
    for (int i = threadIdx.x; i < 27 * 16; i += C0_THREADS) sw[i] = reinterpret_cast<const float4 *>(w0)[i];
    __syncthreads();
    const int64_t HW = (int64_t)H * W;
    const int64_t pix = (int64_t)blockIdx.x * C0_THREADS + threadIdx.x;
    if (pix >= (int64_t)nb * HW) return;
    const int img = (int)(pix / HW), rem = (int)(pix - (int64_t)img * HW), y = rem / W, x = rem - y * W;
    float d[3] = {0.f, 0.f, 0.f};
#pragma unroll 1
    for (int tap = 0; tap < 9; tap++) {
        const int yy = y - tap / 3 + 1, xx = x - tap % 3 + 1;
        if (yy < 0 || yy >= H || xx < 0 || xx >= W) continue;
        if constexpr (std::is_same<T, float>::value) {
            const float4 *gp = reinterpret_cast<const float4 *>(g + ((int64_t)img * HW + (int64_t)yy * W + xx) * 64);
#pragma unroll 4
            for (int q = 0; q < 16; q++) conv0_bwd_acc(d, sw, tap, q, gp[q]);
        } else {  // 8 channels per 16-byte load, summed in the fp32 path's order
            const uint4 *gp = reinterpret_cast<const uint4 *>(g + ((int64_t)img * HW + (int64_t)yy * W + xx) * 64);
#pragma unroll 2
            for (int q = 0; q < 8; q++) {
                const uint4 raw = gp[q];
                const bf16 *h = reinterpret_cast<const bf16 *>(&raw);
                conv0_bwd_acc(d, sw, tap, 2 * q, make_float4(to_f(h[0]), to_f(h[1]), to_f(h[2]), to_f(h[3])));
                conv0_bwd_acc(d, sw, tap, 2 * q + 1, make_float4(to_f(h[4]), to_f(h[5]), to_f(h[6]), to_f(h[7])));
            }
        }
    }
    float *dst = img < nsplit ? out0 + (int64_t)img * 3 * HW : out1 + (int64_t)(img - nsplit) * 3 * HW;
#pragma unroll
    for (int c = 0; c < 3; c++) dst[c * HW + rem] = d[c] * mul / scale[c];
}

// ---------------------------------------------------------------------------------------------------------
// conv3x3, Cin >= 64: implicit GEMM on tensor cores
// ---------------------------------------------------------------------------------------------------------
constexpr int CV_BM = 128, CV_BN = 64, CV_BK = 32, CV_STAGES = 3, CV_THREADS = 128;
constexpr int CV_AS = CV_BK + 4;  // A row stride (floats): the fragment loads hit 32 distinct banks
constexpr int CV_BS = CV_BN + 8;  // B row stride
constexpr int CV_STAGE = CV_BM * CV_AS + CV_BK * CV_BS;
constexpr size_t CV_SMEM = sizeof(float) * CV_STAGES * CV_STAGE;

struct ConvArgs {
    const float *in;    // NHWC [img][H][W][Cin], TF32 values
    const float *wp;    // [9 Cin][Cout], TF32 values
    const float *bias;  // [Cout]: forward (bias + ReLU); NULL: backward-data
    const float *mask;  // backward: NHWC [img][H][W][Cout] activation of the layer below (gradient zeroed where <= 0, so
                        // a NaN activation passes it), or NULL
    float *out;         // NHWC [img][H][W][Cout]
    int64_t M;          // images * H * W
    int H, W, Cin, Cout;
};

__device__ __forceinline__ void cp_async16_zfill(void *dst, const void *src, bool valid) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(valid ? 16 : 0)
                 : "memory");
}

__device__ __forceinline__ void mma_tf32(float *c, const uint32_t *a, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// CTA tile 128 pixels x 64 output channels, K in steps of 32 (one tap, 32 input channels), 3-stage cp.async pipeline;
// 4 warps of 64 x 32.  Out-of-image taps are zero-filled by cp.async.
__global__ void __launch_bounds__(CV_THREADS, 2) k_conv3x3(const ConvArgs p) {
    extern __shared__ __align__(16) float smem[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t m0 = (int64_t)blockIdx.x * CV_BM;
    const int n0 = blockIdx.y * CV_BN;
    const int H = p.H, W = p.W, Cin = p.Cin, Cout = p.Cout;
    const int64_t HW = (int64_t)H * W;

    // A: this thread copies 16-byte chunk (tid & 7) of rows (tid >> 3) + 16 i
    const int ac = tid & 7;
    int ay[8], ax[8];
    int64_t abase[8];
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const int64_t m = m0 + (tid >> 3) + 16 * i;
        if (m < p.M) {
            const int64_t img = m / HW;
            const int rem = (int)(m - img * HW);
            ay[i] = rem / W;
            ax[i] = rem - ay[i] * W;
            abase[i] = m * Cin + ac * 4;
        } else {
            ay[i] = -1000000;  // never inside the image
            ax[i] = 0;
            abase[i] = 0;
        }
    }
    // B: 16-byte chunk (tid & 15) of rows (tid >> 4) + 8 i
    const int bc = tid & 15, br = tid >> 4;
    const int ksteps_per_tap = Cin / CV_BK, ksteps = 9 * ksteps_per_tap;

    auto load = [&](int kt, int slot) {
        float *As = smem + slot * CV_STAGE, *Bs = As + CV_BM * CV_AS;
        const int tap = kt / ksteps_per_tap, ci0 = (kt - tap * ksteps_per_tap) * CV_BK;
        const int dy = tap / 3 - 1, dx = tap % 3 - 1;
        const int64_t shift = ((int64_t)dy * W + dx) * Cin + ci0;
#pragma unroll
        for (int i = 0; i < 8; i++) {
            const int yy = ay[i] + dy, xx = ax[i] + dx;
            const bool ok = yy >= 0 && yy < H && xx >= 0 && xx < W;
            cp_async16_zfill(As + ((tid >> 3) + 16 * i) * CV_AS + ac * 4, ok ? p.in + abase[i] + shift : p.in, ok);
        }
        const float *wsrc = p.wp + ((int64_t)kt * CV_BK + br) * Cout + n0 + bc * 4;
#pragma unroll
        for (int i = 0; i < 4; i++) cp_async16(Bs + (br + 8 * i) * CV_BS + bc * 4, wsrc + (int64_t)8 * i * Cout);
    };

    float acc[4][4][4];
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++)
#pragma unroll
            for (int r = 0; r < 4; r++) acc[i][j][r] = 0.f;

#pragma unroll
    for (int s = 0; s < CV_STAGES - 1; s++) {
        if (s < ksteps) load(s, s);
        cp_async_commit();
    }
    const int g = lane >> 2, t = lane & 3, wm = (warp & 1) * 64, wn = (warp >> 1) * 32;
    for (int kt = 0; kt < ksteps; kt++) {
        cp_async_wait<CV_STAGES - 2>();
        __syncthreads();  // stage kt landed for every thread; every warp is done with stage kt - 1
        if (kt + CV_STAGES - 1 < ksteps) load(kt + CV_STAGES - 1, (kt + CV_STAGES - 1) % CV_STAGES);
        cp_async_commit();
        const float *As = smem + (kt % CV_STAGES) * CV_STAGE, *Bs = As + CV_BM * CV_AS;
#pragma unroll
        for (int kk = 0; kk < CV_BK; kk += 8) {
            uint32_t a[4][4], b[4][2];
#pragma unroll
            for (int i = 0; i < 4; i++) {
                const float *ar = As + (wm + i * 16 + g) * CV_AS + kk + t;
                a[i][0] = __float_as_uint(ar[0]);
                a[i][1] = __float_as_uint(ar[8 * CV_AS]);
                a[i][2] = __float_as_uint(ar[4]);
                a[i][3] = __float_as_uint(ar[8 * CV_AS + 4]);
            }
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const float *bp = Bs + (kk + t) * CV_BS + wn + j * 8 + g;
                b[j][0] = __float_as_uint(bp[0]);
                b[j][1] = __float_as_uint(bp[4 * CV_BS]);
            }
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int j = 0; j < 4; j++) mma_tf32(acc[i][j], a[i], b[j][0], b[j][1]);
        }
    }
    cp_async_wait<0>();

#pragma unroll
    for (int j = 0; j < 4; j++) {
        const int n = n0 + wn + j * 8 + 2 * t;
        const float2 bias = p.bias ? *reinterpret_cast<const float2 *>(p.bias + n) : make_float2(0.f, 0.f);
#pragma unroll
        for (int i = 0; i < 4; i++) {
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int64_t m = m0 + wm + i * 16 + g + 8 * h;
                if (m >= p.M) continue;
                float v0 = acc[i][j][2 * h], v1 = acc[i][j][2 * h + 1];
                if (p.bias) {
                    v0 = max_nan(v0 + bias.x, 0.f);
                    v1 = max_nan(v1 + bias.y, 0.f);
                } else if (p.mask) {  // ReLU's backward: zero where act <= 0, so a NaN activation passes the gradient
                    const float2 mk = *reinterpret_cast<const float2 *>(p.mask + m * Cout + n);
                    v0 = !(mk.x <= 0.f) ? v0 : 0.f;
                    v1 = !(mk.y <= 0.f) ? v1 : 0.f;
                }
                *reinterpret_cast<float2 *>(p.out + m * Cout + n) = make_float2(tf32_round(v0), tf32_round(v1));
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------
// conv3x3, Cin >= 64, BF16: implicit GEMM on wgmma
// ---------------------------------------------------------------------------------------------------------
// CTA tile 128 pixels x BN output channels (BN = 128, or 64 where the layer has 64), K in steps of 64 channels of one
// tap: one 128-byte row per pixel and per output channel, stored with the 128-byte swizzle wgmma reads.  Warpgroup 0
// stages the operands with cp.async (zero-fill for the padding and past the last pixel) and signals each stage's
// `full` mbarrier; warpgroups 1 and 2 each own 64 pixel rows, issue m64nBNk16 wgmmas on a landed stage and release it
// on its `empty` mbarrier once those have retired.
constexpr int WG_BM = 128, WG_BK = 64, WG_STAGES = 4, WG_THREADS = 384;
template <int BN> constexpr int wg_stage_bytes() { return (WG_BM + BN) * WG_BK * 2; }
template <int BN> constexpr size_t wg_smem() { return (size_t)WG_STAGES * wg_stage_bytes<BN>() + 2 * WG_STAGES * 8 + 1024; }

struct ConvArgsBf16 {
    const bf16 *in;     // NHWC [img][H][W][Cin]
    const bf16 *wp;     // [Cout][9 Cin]
    const float *bias;  // [Cout]: forward (bias + ReLU); NULL: backward-data
    const bf16 *mask;   // backward: NHWC [img][H][W][Cout] activation of the layer below, or NULL
    bf16 *out;          // NHWC [img][H][W][Cout]
    int64_t M;
    int H, W, Cin, Cout;
};

// shared-memory matrix descriptor: K-major, 128-byte swizzle, 8-row groups 1024 bytes apart
__device__ __forceinline__ uint64_t wg_desc(uint32_t saddr) {
    return (uint64_t)((saddr & 0x3FFFF) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}

template <int BN> __device__ __forceinline__ void wgmma_bf16(float (&d)[BN / 2], uint64_t da, uint64_t db);
template <> __device__ __forceinline__ void wgmma_bf16<64>(float (&d)[32], uint64_t da, uint64_t db) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, "
        "%13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, "
        "0, 0;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(1));
}
template <> __device__ __forceinline__ void wgmma_bf16<128>(float (&d)[64], uint64_t da, uint64_t db) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, "
        "%13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, "
        "%35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, "
        "%57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
          "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
          "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
          "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
          "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(1));
}

template <int BN>
__global__ void __launch_bounds__(WG_THREADS, 1) k_conv3x3_wgmma(const ConvArgsBf16 p) {
    constexpr int A_BYTES = WG_BM * WG_BK * 2, STAGE = wg_stage_bytes<BN>();
    extern __shared__ __align__(16) uint8_t wg_raw[];
    uint8_t *smem = wg_raw + ((1024 - (smem_u32(wg_raw) & 1023)) & 1023);  // the swizzle needs 1024-byte alignment
    uint64_t *full = reinterpret_cast<uint64_t *>(smem + WG_STAGES * STAGE), *empty = full + WG_STAGES;
    const int tid = threadIdx.x, wg = tid >> 7, t128 = tid & 127;
    const int ntiles = p.Cout / BN;
    const int64_t m0 = (int64_t)(blockIdx.x / ntiles) * WG_BM;  // the CTAs sharing a pixel tile run side by side
    const int n0 = (int)(blockIdx.x % ntiles) * BN;
    const int H = p.H, W = p.W, Cin = p.Cin, Cout = p.Cout;
    const int ksteps_per_tap = Cin / WG_BK, ksteps = 9 * ksteps_per_tap;
    if (tid == 0) {
        for (int s = 0; s < WG_STAGES; s++) {
            mbar_init(full + s, 128);  // one cp.async arrival per producer thread
            mbar_init(empty + s, 2);   // one arrival per consumer warpgroup
        }
    }
    __syncthreads();

    if (wg == 0) {
        // producer: 16-byte chunk c = t128 & 7 of rows (t128 >> 3) + 16 i; a row's chunk c lands at chunk c ^ (row & 7)
        const int c = t128 & 7, r0 = t128 >> 3, sw = ((c ^ (r0 & 7)) << 4);
        const int64_t HW = (int64_t)H * W;
        int ay[8], ax[8];
        int64_t abase[8];
#pragma unroll
        for (int i = 0; i < 8; i++) {
            const int64_t m = m0 + r0 + 16 * i;
            if (m < p.M) {
                const int64_t img = m / HW;
                const int rem = (int)(m - img * HW);
                ay[i] = rem / W;
                ax[i] = rem - ay[i] * W;
                abase[i] = m * Cin + c * 8;
            } else {
                ay[i] = -1000000;  // never inside the image
                ax[i] = 0;
                abase[i] = 0;
            }
        }
        const bf16 *wsrc = p.wp + (int64_t)(n0 + r0) * 9 * Cin + c * 8;
        for (int kt = 0; kt < ksteps; kt++) {
            const int s = kt % WG_STAGES;
            if (kt >= WG_STAGES) mbar_wait(empty + s, ((kt / WG_STAGES) & 1) ^ 1);
            uint8_t *As = smem + s * STAGE, *Bs = As + A_BYTES;
            const int tap = kt / ksteps_per_tap, ci0 = (kt - tap * ksteps_per_tap) * WG_BK;
            const int dy = tap / 3 - 1, dx = tap % 3 - 1;
            const int64_t shift = ((int64_t)dy * W + dx) * Cin + ci0;
#pragma unroll
            for (int i = 0; i < 8; i++) {
                const int yy = ay[i] + dy, xx = ax[i] + dx;
                const bool ok = yy >= 0 && yy < H && xx >= 0 && xx < W;
                cp_async16_zfill(As + (r0 + 16 * i) * 128 + sw, ok ? p.in + abase[i] + shift : p.in, ok);
            }
#pragma unroll
            for (int i = 0; i < BN / 16; i++)
                cp_async16(Bs + (r0 + 16 * i) * 128 + sw, wsrc + (int64_t)16 * i * 9 * Cin + (int64_t)kt * WG_BK);
            cp_async_mbar_arrive(full + s);
        }
        cp_async_wait<0>();
        return;
    }

    // consumers: warpgroup 1 + cw owns pixel rows 64 cw .. 64 cw + 63 of the tile
    const int cw = wg - 1;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; i++) acc[i] = 0.f;
    const uint32_t sbase = smem_u32(smem);
    for (int kt = 0; kt < ksteps; kt++) {
        const int s = kt % WG_STAGES;
        mbar_wait(full + s, (kt / WG_STAGES) & 1);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // cp.async's writes, visible to wgmma's reads
        asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
        const uint32_t a = sbase + s * STAGE + cw * 64 * 128, b = sbase + s * STAGE + A_BYTES;
#pragma unroll
        for (int kk = 0; kk < WG_BK / 16; kk++) wgmma_bf16<BN>(acc, wg_desc(a + 32 * kk), wg_desc(b + 32 * kk));
        asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
        asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory");  // the previous step's wgmmas have retired
        if (kt > 0 && t128 == 0) mbar_arrive(empty + (kt - 1) % WG_STAGES);
    }
    asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");

    // accumulator layout: row 16 w + g (+8), columns 8 j + 2 t (+1) of this warpgroup's 64 x BN block
    const int lane = t128 & 31, w4 = t128 >> 5, g = lane >> 2, t = lane & 3;
#pragma unroll
    for (int j = 0; j < BN / 8; j++) {
        const int n = n0 + j * 8 + 2 * t;
        const float2 bias = p.bias ? *reinterpret_cast<const float2 *>(p.bias + n) : make_float2(0.f, 0.f);
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int64_t m = m0 + cw * 64 + w4 * 16 + g + 8 * h;
            if (m >= p.M) continue;
            float v0 = acc[j * 4 + 2 * h], v1 = acc[j * 4 + 2 * h + 1];
            if (p.bias) {
                v0 = max_nan(v0 + bias.x, 0.f);
                v1 = max_nan(v1 + bias.y, 0.f);
            } else if (p.mask) {  // ReLU's backward: zero where act <= 0, so a NaN activation passes the gradient
                const __nv_bfloat162 mk = *reinterpret_cast<const __nv_bfloat162 *>(p.mask + m * Cout + n);
                v0 = !(to_f(mk.x) <= 0.f) ? v0 : 0.f;
                v1 = !(to_f(mk.y) <= 0.f) ? v1 : 0.f;
            }
            *reinterpret_cast<uint32_t *>(p.out + m * Cout + n) = pack_bf16x2(v0, v1);
        }
    }
}

// ---------------------------------------------------------------------------------------------------------
// max-pool and its backward
// ---------------------------------------------------------------------------------------------------------
constexpr int EW_THREADS = 256;

// NHWC [img][H][W][C] -> [img][H/2][W/2][C], floor.  The maximum of BF16 values is one of them: no rounding.
template <typename T>
__global__ void k_pool(const T *__restrict__ in, int nimg, int H, int W, int C, T *__restrict__ out) {
    using V = Act16<T>;
    const int Ho = H / 2, Wo = W / 2, C4 = C / V::E;
    const int64_t total = (int64_t)nimg * Ho * Wo * C4;
    const int64_t i = (int64_t)blockIdx.x * EW_THREADS + threadIdx.x;
    if (i >= total) return;
    const int c4 = (int)(i % C4);
    const int64_t po = i / C4;
    const int xo = (int)(po % Wo), yo = (int)((po / Wo) % Ho);
    const int64_t img = po / ((int64_t)Wo * Ho);
    const V *src = reinterpret_cast<const V *>(in) + ((img * H + 2 * yo) * W + 2 * xo) * C4 + c4;
    const V a = src[0], b = src[C4], c = src[(int64_t)W * C4], d = src[(int64_t)W * C4 + C4];
    V r;
#pragma unroll
    for (int e = 0; e < V::E; e++)
        r.e[e] = T(max_nan(max_nan(to_f(a.e[e]), to_f(b.e[e])), max_nan(to_f(c.e[e]), to_f(d.e[e]))));
    reinterpret_cast<V *>(out)[i] = r;
}

// index (0..3, row-major) of the element max_pool2d's backward routes a 2x2 window's gradient to: PyTorch's scan
// `val > maxval || isnan(val)`, i.e. the first maximum, or the last NaN if the window holds one
__device__ __forceinline__ int first_max(float a, float b, float c, float d) {
    int k = 0;
    float m = a;
    if (b > m || b != b) { m = b; k = 1; }
    if (c > m || c != c) { m = c; k = 2; }
    if (d > m || d != d) k = 3;
    return k;
}

// g [img][H][W][C] holds the head's (masked) gradient of the tap; adds the pooled gradient gp [img][H/2][W/2][C]
// routed by first_max, under the tap's ReLU mask (zero where act <= 0), in place
template <typename T>
__global__ void k_unpool_bwd(const T *__restrict__ act, const T *__restrict__ gp, int nimg, int H, int W, int C,
                             T *__restrict__ g) {
    using V = Act16<T>;
    const int Ho = H / 2, Wo = W / 2, C4 = C / V::E;
    const int64_t total = (int64_t)nimg * H * W * C4;
    const int64_t i = (int64_t)blockIdx.x * EW_THREADS + threadIdx.x;
    if (i >= total) return;
    const int c4 = (int)(i % C4);
    const int64_t pix = i / C4;
    const int x = (int)(pix % W), y = (int)((pix / W) % H);
    const int64_t img = pix / ((int64_t)W * H);
    if (y >= 2 * Ho || x >= 2 * Wo) return;  // a row or column the floor pool drops: the head's gradient alone
    const int yo = y >> 1, xo = x >> 1, me = (y & 1) * 2 + (x & 1);
    const V *a4 = reinterpret_cast<const V *>(act);
    const int64_t w0 = ((img * H + 2 * yo) * W + 2 * xo) * C4 + c4;
    const V a = a4[w0], b = a4[w0 + C4], c = a4[w0 + (int64_t)W * C4], d = a4[w0 + (int64_t)W * C4 + C4];
    const V up = reinterpret_cast<const V *>(gp)[((img * Ho + yo) * Wo + xo) * C4 + c4];
    const V self = a4[pix * C4 + c4];
    V v = reinterpret_cast<V *>(g)[i];
    if constexpr (std::is_same<T, float>::value) {
        if (first_max(a.e[0], b.e[0], c.e[0], d.e[0]) == me && !(self.e[0] <= 0.f)) v.e[0] = tf32_round(v.e[0] + up.e[0]);
        if (first_max(a.e[1], b.e[1], c.e[1], d.e[1]) == me && !(self.e[1] <= 0.f)) v.e[1] = tf32_round(v.e[1] + up.e[1]);
        if (first_max(a.e[2], b.e[2], c.e[2], d.e[2]) == me && !(self.e[2] <= 0.f)) v.e[2] = tf32_round(v.e[2] + up.e[2]);
        if (first_max(a.e[3], b.e[3], c.e[3], d.e[3]) == me && !(self.e[3] <= 0.f)) v.e[3] = tf32_round(v.e[3] + up.e[3]);
    } else {
#pragma unroll
        for (int e = 0; e < V::E; e++)
            if (first_max(to_f(a.e[e]), to_f(b.e[e]), to_f(c.e[e]), to_f(d.e[e])) == me && !(to_f(self.e[e]) <= 0.f))
                v.e[e] = act_round<T>(to_f(v.e[e]) + to_f(up.e[e]));
    }
    reinterpret_cast<V *>(g)[i] = v;
}

// ---------------------------------------------------------------------------------------------------------
// head
// ---------------------------------------------------------------------------------------------------------
constexpr int HD_THREADS = 256, HD_WARPS = HD_THREADS / 32;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// f: tap [2N][HW][C]; partial[img * LP_HEAD_BLOCKS + block] = sum over this CTA's pixels of sum_c lin (n0 - n1)^2
template <int CPL, typename T>
__global__ void __launch_bounds__(HD_THREADS)
k_head_fwd(const T *__restrict__ f, int N, int HW, const float *__restrict__ lin, double *__restrict__ partial) {
    constexpr int C = CPL * 32;
    __shared__ double red[HD_WARPS];
    const int img = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float w[CPL];
#pragma unroll
    for (int k = 0; k < CPL; k++) w[k] = lin[lane + 32 * k];
    double acc = 0.0;
    for (int px = blockIdx.x * HD_WARPS + warp; px < HW; px += LP_HEAD_BLOCKS * HD_WARPS) {
        const T *p0 = f + ((int64_t)img * HW + px) * C + lane, *p1 = f + ((int64_t)(img + N) * HW + px) * C + lane;
        float a[CPL], b[CPL], sa = 0.f, sb = 0.f;
#pragma unroll
        for (int k = 0; k < CPL; k++) {
            a[k] = to_f(p0[32 * k]);
            b[k] = to_f(p1[32 * k]);
            sa = fmaf(a[k], a[k], sa);
            sb = fmaf(b[k], b[k], sb);
        }
        const float na = sqrtf(warp_sum(sa)) + LP_EPS, nb = sqrtf(warp_sum(sb)) + LP_EPS;
        float d = 0.f;
#pragma unroll
        for (int k = 0; k < CPL; k++) {
            const float e = a[k] / na - b[k] / nb;
            d = fmaf(w[k] * e, e, d);
        }
        acc += (double)warp_sum(d);
    }
    if (lane == 0) red[warp] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
#pragma unroll
        for (int k = 0; k < HD_WARPS; k++) s += red[k];
        partial[(int64_t)img * LP_HEAD_BLOCKS + blockIdx.x] = s;
    }
}

struct TapSizes {
    int hw[LP_NTAPS];
};

// out[img] = sum_l (sum of tap l's partials) / HW_l, in a fixed order
__global__ void k_head_final(const double *__restrict__ partial, int N, const TapSizes ts, float *__restrict__ out) {
    const int img = blockIdx.x * blockDim.x + threadIdx.x;
    if (img >= N) return;
    double v = 0.0;
    for (int l = 0; l < LP_NTAPS; l++) {
        const double *p = partial + ((int64_t)l * N + img) * LP_HEAD_BLOCKS;
        double s = 0.0;
        for (int b = 0; b < LP_HEAD_BLOCKS; b++) s += p[b];
        v += s / (double)ts.hw[l];
    }
    out[img] = (float)v;
}

// g[img - i0][HW][C] = dL/df of image img (i0 <= img < i0 + nb, of 2N) under the tap's ReLU mask.  Image img's pair
// partner is img +- N; dL/dout[img mod N] / HW is the gradient of each pixel's distance.
template <int CPL, typename T>
__global__ void __launch_bounds__(HD_THREADS)
k_head_bwd(const T *__restrict__ f, int N, int i0, int HW, const float *__restrict__ lin,
           const float *__restrict__ dout, T *__restrict__ g) {
    constexpr int C = CPL * 32;
    const int lane = threadIdx.x & 31, px = blockIdx.x * HD_WARPS + (threadIdx.x >> 5);
    if (px >= HW) return;
    const int img = i0 + blockIdx.y, other = img < N ? img + N : img - N;
    const float scale = 2.f * dout[img < N ? img : img - N] / (float)HW;
    const T *p0 = f + ((int64_t)img * HW + px) * C + lane, *p1 = f + ((int64_t)other * HW + px) * C + lane;
    float a[CPL], b[CPL], sa = 0.f, sb = 0.f;
#pragma unroll
    for (int k = 0; k < CPL; k++) {
        a[k] = to_f(p0[32 * k]);
        b[k] = to_f(p1[32 * k]);
        sa = fmaf(a[k], a[k], sa);
        sb = fmaf(b[k], b[k], sb);
    }
    const float s = sqrtf(warp_sum(sa)), na = s + LP_EPS, nb = sqrtf(warp_sum(sb)) + LP_EPS;
    float gn[CPL], dot = 0.f;
#pragma unroll
    for (int k = 0; k < CPL; k++) {
        const float n = a[k] / na;
        gn[k] = scale * lin[lane + 32 * k] * (n - b[k] / nb);
        dot = fmaf(n, gn[k], dot);
    }
    dot = warp_sum(dot);
    const float proj = s == 0.f ? 0.f : dot * na / s;  // the limit at s = 0 (see the top of the file); a NaN s stays NaN
    T *dst = g + ((int64_t)(img - i0) * HW + px) * C + lane;
#pragma unroll
    for (int k = 0; k < CPL; k++) dst[32 * k] = !(a[k] <= 0.f) ? act_round<T>((gn[k] - (a[k] / na) * proj) / na) : act_zero<T>();
}

// ---------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------
int64_t align64(int64_t floats) { return (floats + 63) & ~(int64_t)63; }
int64_t align256(int64_t bytes) { return (bytes + 255) & ~(int64_t)255; }

// workspace carve-up (offsets in bytes; every region 256-byte aligned); activations and gradients are `esize`-byte
// elements (4: TF32 path, 2: BF16 path)
struct Plan {
    int N, nimg, nb;
    int h[5], w[5];
    bool full;              // every activation kept (gradients wanted); else two ping-pong buffers
    int64_t act[LP_LAYERS];  // full: per layer output; else -1
    int64_t pool[4];         // full: pooled inputs of layers 2, 4, 7, 10
    int64_t ping[2];         // !full
    int64_t grad[2];         // full: two gradient buffers of nb images
    int64_t partial;         // head partial sums (doubles)
    int64_t total;
};

Plan make_plan(const GsLpipsConfig &c) {
    Plan p{};
    p.N = c.batch;
    p.nimg = 2 * c.batch;
    p.nb = ((c.grads & 1) ? c.batch : 0) + ((c.grads & 2) ? c.batch : 0);
    p.full = c.grads != 0;
    for (int l = 0; l < 5; l++) { p.h[l] = c.height >> l; p.w[l] = c.width >> l; }
    const int64_t esize = c.precision == GS_LPIPS_BF16 ? 2 : 4;
    int64_t off = 0;
    auto take = [&](int64_t elems) { const int64_t o = off; off += align256(elems * esize); return o; };
    const int64_t big = (int64_t)p.nimg * p.h[0] * p.w[0] * 64;  // the largest activation (conv1_x)
    if (p.full) {
        int pi = 0;
        for (int l = 0; l < LP_LAYERS; l++) {
            const int v = LP_LEVEL[l];
            if (lp_pooled_input(l)) p.pool[pi++] = take((int64_t)p.nimg * p.h[v] * p.w[v] * LP_CIN[l]);
            p.act[l] = take((int64_t)p.nimg * p.h[v] * p.w[v] * LP_COUT[l]);
        }
        const int64_t gbig = (int64_t)p.nb * p.h[0] * p.w[0] * 64;
        p.grad[0] = take(gbig);
        p.grad[1] = take(gbig);
        p.ping[0] = p.ping[1] = -1;
    } else {
        for (int l = 0; l < LP_LAYERS; l++) p.act[l] = -1;
        p.ping[0] = take(big);
        p.ping[1] = take(big);
        p.grad[0] = p.grad[1] = -1;
    }
    p.partial = off;
    off += align256(8 * (int64_t)LP_NTAPS * p.N * LP_HEAD_BLOCKS);  // doubles
    p.total = off;
    return p;
}

int check_config(const GsLpipsConfig *c, const char *who) {
    if (!c) return gs_set_error(GS_ERR_INVALID, who);
    if (c->batch < 0 || c->batch > 32767 || c->height < 16 || c->width < 16 || c->height > 16384 || c->width > 16384 ||
        (c->normalize != 0 && c->normalize != 1) || c->grads < 0 || c->grads > 3 ||
        (c->precision != GS_LPIPS_TF32 && c->precision != GS_LPIPS_BF16))
        return gs_set_error(GS_ERR_INVALID, who);
    const int64_t n = 3 * (int64_t)c->height * c->width;
    if (c->batch > 1 && (c->in0_stride < n || c->in1_stride < n))
        return gs_set_error(GS_ERR_INVALID, "LPIPS: image strides must be at least 3 * height * width");
    if ((int64_t)2 * c->batch * c->height * c->width * 64 > ((int64_t)1 << 40))
        return gs_set_error(GS_ERR_INVALID, "LPIPS: batch * height * width is too large");
    return GS_OK;
}

unsigned blocks_for(int64_t n, int threads) { return (unsigned)((n + threads - 1) / threads); }

int launch_conv(const float *in, const float *wp, const float *bias, const float *mask, float *out, int nimg, int H, int W,
                int Cin, int Cout, cudaStream_t st) {
    // 81 KB per CTA (two CTAs per SM): above the 48 KB default
    GS_CUDA_OK(cudaFuncSetAttribute(k_conv3x3, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CV_SMEM));
    ConvArgs a;
    a.in = in; a.wp = wp; a.bias = bias; a.mask = mask; a.out = out;
    a.M = (int64_t)nimg * H * W;
    a.H = H; a.W = W; a.Cin = Cin; a.Cout = Cout;
    k_conv3x3<<<dim3(blocks_for(a.M, CV_BM), Cout / CV_BN), CV_THREADS, CV_SMEM, st>>>(a);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}

template <int BN>
int launch_conv_wgmma(const ConvArgsBf16 &a, cudaStream_t st) {
    GS_CUDA_OK(cudaFuncSetAttribute(k_conv3x3_wgmma<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)wg_smem<BN>()));
    const int64_t ctas = (int64_t)blocks_for(a.M, WG_BM) * (a.Cout / BN);
    if (ctas > 0x7fffffff) return gs_set_error(GS_ERR_INVALID, "LPIPS: batch * height * width is too large for BF16");
    k_conv3x3_wgmma<BN><<<(unsigned)ctas, WG_THREADS, wg_smem<BN>(), st>>>(a);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}

int launch_conv(const bf16 *in, const bf16 *wp, const float *bias, const bf16 *mask, bf16 *out, int nimg, int H, int W,
                int Cin, int Cout, cudaStream_t st) {
    ConvArgsBf16 a;
    a.in = in; a.wp = wp; a.bias = bias; a.mask = mask; a.out = out;
    a.M = (int64_t)nimg * H * W;
    a.H = H; a.W = W; a.Cin = Cin; a.Cout = Cout;
    return Cout % 128 == 0 ? launch_conv_wgmma<128>(a, st) : launch_conv_wgmma<64>(a, st);
}

template <typename T>
int launch_head_fwd(const T *f, int C, int N, int HW, const float *lin, double *partial, cudaStream_t st) {
    const dim3 grid(LP_HEAD_BLOCKS, N);
    switch (C) {
        case 64: k_head_fwd<2, T><<<grid, HD_THREADS, 0, st>>>(f, N, HW, lin, partial); break;
        case 128: k_head_fwd<4, T><<<grid, HD_THREADS, 0, st>>>(f, N, HW, lin, partial); break;
        case 256: k_head_fwd<8, T><<<grid, HD_THREADS, 0, st>>>(f, N, HW, lin, partial); break;
        default: k_head_fwd<16, T><<<grid, HD_THREADS, 0, st>>>(f, N, HW, lin, partial); break;
    }
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}

template <typename T>
int launch_head_bwd(const T *f, int C, int N, int i0, int nb, int HW, const float *lin, const float *dout, T *g,
                    cudaStream_t st) {
    const dim3 grid(blocks_for(HW, HD_WARPS), nb);
    switch (C) {
        case 64: k_head_bwd<2, T><<<grid, HD_THREADS, 0, st>>>(f, N, i0, HW, lin, dout, g); break;
        case 128: k_head_bwd<4, T><<<grid, HD_THREADS, 0, st>>>(f, N, i0, HW, lin, dout, g); break;
        case 256: k_head_bwd<8, T><<<grid, HD_THREADS, 0, st>>>(f, N, i0, HW, lin, dout, g); break;
        default: k_head_bwd<16, T><<<grid, HD_THREADS, 0, st>>>(f, N, i0, HW, lin, dout, g); break;
    }
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}

}  // namespace

struct GsLpipsWeights {
    void *base;
    const float *fwd[LP_LAYERS], *rot[LP_LAYERS], *bias[LP_LAYERS];  // fwd[0] = conv1_1's [27][64]; rot[0] unused
    const float *lin[LP_NTAPS], *shift, *scale;
    void *base16;  // gs_lpips_weights_pack_bf16, else NULL
    const bf16 *fwd16[LP_LAYERS], *rot16[LP_LAYERS];  // [Cout][9 Cin] and [Cin][9 Cout]; [0] unused (conv1_1 stays fp32)
};

namespace {

// the packed convolution weights a layer l >= 1 reads on each path
const float *conv_fwd(const GsLpipsWeights *w, int l, float *) { return w->fwd[l]; }
const float *conv_rot(const GsLpipsWeights *w, int l, float *) { return w->rot[l]; }
const bf16 *conv_fwd(const GsLpipsWeights *w, int l, bf16 *) { return w->fwd16[l]; }
const bf16 *conv_rot(const GsLpipsWeights *w, int l, bf16 *) { return w->rot16[l]; }

template <typename T>
int lpips_forward(const GsLpipsWeights *w, const GsLpipsConfig *cfg, const float *in0, const float *in1, void *workspace,
                  float *out, cudaStream_t st) {
    const Plan p = make_plan(*cfg);
    char *ws = static_cast<char *>(workspace);
    double *partial = reinterpret_cast<double *>(ws + p.partial);
    const int N = p.N, nimg = p.nimg;
    const int64_t in0_stride = cfg->batch > 1 ? cfg->in0_stride : 0, in1_stride = cfg->batch > 1 ? cfg->in1_stride : 0;

    int pp = 0;  // ping-pong buffer the next output goes to (activations not kept)
    auto next_buf = [&](int64_t kept) {
        if (p.full) return reinterpret_cast<T *>(ws + kept);
        T *r = reinterpret_cast<T *>(ws + p.ping[pp]);
        pp ^= 1;
        return r;
    };

    T *cur = next_buf(p.act[0]);
    k_conv0_fwd<T><<<blocks_for((int64_t)nimg * p.h[0] * p.w[0] * 8, C0_THREADS), C0_THREADS, 0, st>>>(
        in0, in1, in0_stride, in1_stride, N, p.h[0], p.w[0], cfg->normalize, w->fwd[0], w->bias[0], w->shift, w->scale, cur);
    GS_CUDA_OK(cudaGetLastError());
    int pi = 0;
    for (int l = 1; l < LP_LAYERS; l++) {
        const int v = LP_LEVEL[l];
        if (lp_pooled_input(l)) {
            T *pooled = next_buf(p.full ? p.pool[pi] : 0);
            pi++;
            k_pool<T><<<blocks_for((int64_t)nimg * p.h[v] * p.w[v] * (LP_CIN[l] / Act16<T>::E), EW_THREADS), EW_THREADS, 0, st>>>(
                cur, nimg, p.h[v - 1], p.w[v - 1], LP_CIN[l], pooled);
            GS_CUDA_OK(cudaGetLastError());
            cur = pooled;
        }
        T *o = next_buf(p.act[l]);
        if (int rc = launch_conv(cur, conv_fwd(w, l, cur), w->bias[l], nullptr, o, nimg, p.h[v], p.w[v], LP_CIN[l], LP_COUT[l], st))
            return rc;
        cur = o;
        const int t = LP_TAP_OF[l];
        if (t >= 0)
            if (int rc = launch_head_fwd(cur, LP_COUT[l], N, p.h[v] * p.w[v], w->lin[t], partial + (int64_t)t * N * LP_HEAD_BLOCKS, st))
                return rc;
    }
    TapSizes ts;
    for (int l = 0; l < LP_LAYERS; l++)
        if (LP_TAP_OF[l] >= 0) ts.hw[LP_TAP_OF[l]] = p.h[LP_LEVEL[l]] * p.w[LP_LEVEL[l]];
    k_head_final<<<blocks_for(N, 128), 128, 0, st>>>(partial, N, ts, out);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}

template <typename T>
int lpips_backward(const GsLpipsWeights *w, const GsLpipsConfig *cfg, const float *dL_dout, void *workspace,
                   float *dL_din0, float *dL_din1, cudaStream_t st) {
    const Plan p = make_plan(*cfg);
    char *ws = static_cast<char *>(workspace);
    const int N = p.N;
    const int i0 = dL_din0 ? 0 : N, nb = (dL_din0 && dL_din1) ? 2 * N : N;
    auto at = [&](int64_t off) { return reinterpret_cast<T *>(ws + off); };
    // activations of images [i0, i0 + nb)
    auto act = [&](int l) { const int v = LP_LEVEL[l]; return at(p.act[l]) + (int64_t)i0 * p.h[v] * p.w[v] * LP_COUT[l]; };
    T *cur = at(p.grad[0]), *oth = at(p.grad[1]);

    if (int rc = launch_head_bwd(at(p.act[12]), 512, N, i0, nb, p.h[4] * p.w[4], w->lin[4], dL_dout, cur, st)) return rc;
    for (int l = LP_LAYERS - 1; l >= 1; l--) {
        const int v = LP_LEVEL[l];
        // cur = dL/d(pre-activation of layer l) -> oth = dL/d(input of layer l)
        if (int rc = launch_conv(cur, conv_rot(w, l, cur), nullptr, lp_pooled_input(l) ? nullptr : act(l - 1), oth, nb, p.h[v],
                                 p.w[v], LP_COUT[l], LP_CIN[l], st))
            return rc;
        if (lp_pooled_input(l)) {
            const int u = v - 1, t = LP_TAP_OF[l - 1], C = LP_COUT[l - 1];
            if (int rc = launch_head_bwd(at(p.act[l - 1]), C, N, i0, nb, p.h[u] * p.w[u], w->lin[t], dL_dout, cur, st)) return rc;
            k_unpool_bwd<T><<<blocks_for((int64_t)nb * p.h[u] * p.w[u] * (C / Act16<T>::E), EW_THREADS), EW_THREADS, 0, st>>>(
                act(l - 1), oth, nb, p.h[u], p.w[u], C, cur);
            GS_CUDA_OK(cudaGetLastError());
        } else {
            std::swap(cur, oth);
        }
    }
    k_conv0_bwd<T><<<blocks_for((int64_t)nb * p.h[0] * p.w[0], C0_THREADS), C0_THREADS, 0, st>>>(
        cur, nb, p.h[0], p.w[0], w->fwd[0], w->scale, cfg->normalize ? 2.f : 1.f, dL_din0 ? dL_din0 : dL_din1, dL_din1,
        dL_din0 ? N : nb);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}

int check_bf16_weights(const GsLpipsWeights *w, const GsLpipsConfig *cfg, const char *who) {
    if (cfg->precision == GS_LPIPS_BF16 && !w->base16) return gs_set_error(GS_ERR_INVALID, who);
    return GS_OK;
}

}  // namespace

extern "C" GS_API int gs_lpips_weights_create(const float *const *conv_weight, const float *const *conv_bias,
                                              const float *const *lin, const float *shift, const float *scale,
                                              void *stream, GsLpipsWeights **out) {
    if (!out) return gs_set_error(GS_ERR_INVALID, "gs_lpips_weights_create: null output handle");
    *out = nullptr;
    if (!conv_weight || !conv_bias || !lin || !shift || !scale)
        return gs_set_error(GS_ERR_INVALID, "gs_lpips_weights_create: null pointer argument");
    for (int l = 0; l < LP_LAYERS; l++)
        if (!conv_weight[l] || !conv_bias[l]) return gs_set_error(GS_ERR_INVALID, "gs_lpips_weights_create: null conv weight or bias");
    for (int t = 0; t < LP_NTAPS; t++)
        if (!lin[t]) return gs_set_error(GS_ERR_INVALID, "gs_lpips_weights_create: null lin weight");
    int64_t off[LP_LAYERS][3], lin_off[LP_NTAPS], o = 0;
    for (int l = 0; l < LP_LAYERS; l++) {
        const int64_t n = (int64_t)9 * LP_CIN[l] * LP_COUT[l];
        off[l][0] = o; o += align64(n);
        off[l][1] = o; o += l ? align64(n) : 0;
        off[l][2] = o; o += align64(LP_COUT[l]);
    }
    for (int t = 0; t < LP_NTAPS; t++) { lin_off[t] = o; o += align64(LP_TAP_C[t]); }
    const int64_t shift_off = o, scale_off = o + 64;
    o += 128;
    GsLpipsWeights *w = new (std::nothrow) GsLpipsWeights();
    if (!w) return gs_set_error(GS_ERR_OOM, "gs_lpips_weights_create: host allocation failed");
    if (cudaMalloc(&w->base, sizeof(float) * o) != cudaSuccess) {
        delete w;
        cudaGetLastError();
        return gs_set_error(GS_ERR_OOM, "gs_lpips_weights_create: device allocation failed");
    }
    float *b = static_cast<float *>(w->base);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int rc = GS_OK;
    auto fail = [&](cudaError_t e, const char *what) {
        if (e != cudaSuccess && rc == GS_OK) rc = gs_set_cuda_error(e, what, __FILE__, __LINE__);
    };
    for (int l = 0; l < LP_LAYERS; l++) {
        w->fwd[l] = b + off[l][0];
        w->rot[l] = l ? b + off[l][1] : nullptr;
        w->bias[l] = b + off[l][2];
        if (l == 0) {
            k_pack_conv0<<<blocks_for(64 * 27, 256), 256, 0, st>>>(conv_weight[0], b + off[0][0]);
        } else {
            const int64_t n = (int64_t)9 * LP_CIN[l] * LP_COUT[l];
            k_pack_conv<<<(unsigned)std::min<int64_t>(blocks_for(n, 256), 4096), 256, 0, st>>>(
                conv_weight[l], LP_CIN[l], LP_COUT[l], b + off[l][0], b + off[l][1]);
        }
        fail(cudaGetLastError(), "k_pack_conv");
        fail(cudaMemcpyAsync(b + off[l][2], conv_bias[l], sizeof(float) * LP_COUT[l], cudaMemcpyDeviceToDevice, st), "bias copy");
    }
    for (int t = 0; t < LP_NTAPS; t++) {
        w->lin[t] = b + lin_off[t];
        fail(cudaMemcpyAsync(b + lin_off[t], lin[t], sizeof(float) * LP_TAP_C[t], cudaMemcpyDeviceToDevice, st), "lin copy");
    }
    w->shift = b + shift_off;
    w->scale = b + scale_off;
    fail(cudaMemcpyAsync(b + shift_off, shift, 3 * sizeof(float), cudaMemcpyDeviceToDevice, st), "shift copy");
    fail(cudaMemcpyAsync(b + scale_off, scale, 3 * sizeof(float), cudaMemcpyDeviceToDevice, st), "scale copy");
    if (rc != GS_OK) {
        cudaFree(w->base);
        delete w;
        return rc;
    }
    *out = w;
    return GS_OK;
}

extern "C" GS_API int gs_lpips_weights_pack_bf16(GsLpipsWeights *w, const float *const *conv_weight, void *stream) {
    if (!w || !conv_weight) return gs_set_error(GS_ERR_INVALID, "gs_lpips_weights_pack_bf16: null pointer argument");
    for (int l = 1; l < LP_LAYERS; l++)
        if (!conv_weight[l]) return gs_set_error(GS_ERR_INVALID, "gs_lpips_weights_pack_bf16: null conv weight");
    if (w->base16) return GS_OK;  // packed already: the handle's weights do not change
    int64_t off[LP_LAYERS], o = 0;  // in bf16 elements, every region 256-byte aligned
    for (int l = 1; l < LP_LAYERS; l++) {
        off[l] = o;
        o += 2 * (align64((int64_t)9 * LP_CIN[l] * LP_COUT[l]) * 2);
    }
    void *base = nullptr;
    if (cudaMalloc(&base, sizeof(bf16) * o) != cudaSuccess) {
        cudaGetLastError();
        return gs_set_error(GS_ERR_OOM, "gs_lpips_weights_pack_bf16: device allocation failed");
    }
    bf16 *b = static_cast<bf16 *>(base);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    for (int l = 1; l < LP_LAYERS; l++) {
        const int64_t n = (int64_t)9 * LP_CIN[l] * LP_COUT[l];
        k_pack_conv_bf16<<<(unsigned)std::min<int64_t>(blocks_for(n, 256), 4096), 256, 0, st>>>(
            conv_weight[l], LP_CIN[l], LP_COUT[l], b + off[l], b + off[l] + align64(n) * 2);
        if (cudaError_t e = cudaGetLastError(); e != cudaSuccess) {
            cudaFree(base);
            return gs_set_cuda_error(e, "k_pack_conv_bf16", __FILE__, __LINE__);
        }
    }
    w->base16 = base;
    w->fwd16[0] = w->rot16[0] = nullptr;
    for (int l = 1; l < LP_LAYERS; l++) {
        w->fwd16[l] = b + off[l];
        w->rot16[l] = b + off[l] + align64((int64_t)9 * LP_CIN[l] * LP_COUT[l]) * 2;
    }
    return GS_OK;
}

extern "C" GS_API void gs_lpips_weights_destroy(GsLpipsWeights *w) {
    if (!w) return;
    cudaFree(w->base);  // synchronises with the device: no kernel still reads the weights
    if (w->base16) cudaFree(w->base16);
    delete w;
}

extern "C" GS_API int64_t gs_lpips_workspace_bytes(const GsLpipsConfig *cfg) {
    if (check_config(cfg, "bad GsLpipsConfig") != GS_OK) return -1;
    return make_plan(*cfg).total;
}

extern "C" GS_API int gs_lpips_forward(const GsLpipsWeights *w, const GsLpipsConfig *cfg, const float *in0,
                                       const float *in1, void *workspace, float *out, void *stream) {
    if (int rc = check_config(cfg, "bad GsLpipsConfig for gs_lpips_forward")) return rc;
    if (!w || !in0 || !in1 || !workspace || !out)
        return gs_set_error(GS_ERR_INVALID, "gs_lpips_forward: null pointer argument");
    if (reinterpret_cast<uintptr_t>(workspace) & 255u)
        return gs_set_error(GS_ERR_INVALID, "gs_lpips_forward: the workspace must be 256-byte aligned");
    if (int rc = check_bf16_weights(w, cfg, "gs_lpips_forward: precision GS_LPIPS_BF16 needs gs_lpips_weights_pack_bf16 on the weights"))
        return rc;
    if (cfg->batch == 0) return GS_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    return cfg->precision == GS_LPIPS_BF16 ? lpips_forward<bf16>(w, cfg, in0, in1, workspace, out, st)
                                           : lpips_forward<float>(w, cfg, in0, in1, workspace, out, st);
}

extern "C" GS_API int gs_lpips_backward(const GsLpipsWeights *w, const GsLpipsConfig *cfg, const float *dL_dout,
                                        void *workspace, float *dL_din0, float *dL_din1, void *stream) {
    if (int rc = check_config(cfg, "bad GsLpipsConfig for gs_lpips_backward")) return rc;
    if (!w || !dL_dout || !workspace) return gs_set_error(GS_ERR_INVALID, "gs_lpips_backward: null pointer argument");
    if (reinterpret_cast<uintptr_t>(workspace) & 255u)
        return gs_set_error(GS_ERR_INVALID, "gs_lpips_backward: the workspace must be 256-byte aligned");
    if ((dL_din0 && !(cfg->grads & 1)) || (dL_din1 && !(cfg->grads & 2)))
        return gs_set_error(GS_ERR_INVALID, "gs_lpips_backward: a gradient the forward's config did not provide for (grads)");
    if (int rc = check_bf16_weights(w, cfg, "gs_lpips_backward: precision GS_LPIPS_BF16 needs gs_lpips_weights_pack_bf16 on the weights"))
        return rc;
    if (cfg->batch == 0 || (!dL_din0 && !dL_din1)) return GS_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    return cfg->precision == GS_LPIPS_BF16 ? lpips_backward<bf16>(w, cfg, dL_dout, workspace, dL_din0, dL_din1, st)
                                           : lpips_backward<float>(w, cfg, dL_dout, workspace, dL_din0, dL_din1, st);
}
