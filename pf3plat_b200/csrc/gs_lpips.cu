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
// Non-finite inputs follow PyTorch's rules, so a NaN or Inf pixel gives the image a NaN distance and NaN gradients
// where autograd has them: ReLU and max-pool propagate NaN (max.NaN), ReLU's backward zeroes the gradient only where
// act <= 0 (a NaN activation passes it), and the max-pool backward routes to a NaN as described above.
//
// Head backward: with s = ||f||, n = f/(s+e), g = dL/dn:  dL/df = (g - n (n.g)(s+e)/s) / (s+e).  At s = 0 the second
// term's limit is 0 (|n (n.g)(s+e)/s| <= |g| s/(s+e)), so dL/df = g/e there (the derivative of f/(s+e) at f = 0);
// autograd's dL/df is NaN there (sqrt's backward at 0).  A tap pixel with s = 0 has every channel 0, so the ReLU mask
// drops that gradient before it reaches the layer below, on both sides.
#include "gs_common.cuh"

#include <algorithm>
#include <new>
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

__global__ void __launch_bounds__(C0_THREADS)
k_conv0_fwd(const float *__restrict__ in0, const float *__restrict__ in1, int64_t s0, int64_t s1, int N, int H, int W,
            int normalize, const float *__restrict__ w0, const float *__restrict__ b0, const float *__restrict__ shift,
            const float *__restrict__ scale, float *__restrict__ out) {
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
    float4 *dst = reinterpret_cast<float4 *>(out + pix * 64 + cg * 8);
#pragma unroll
    for (int o = 0; o < 8; o++) acc[o] = tf32_round(max_nan(acc[o], 0.f));
    dst[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
    dst[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
}

// dL/dx from g = dL/d(conv1_1 pre-activation) [nb][H][W][64]; images [0, nsplit) go to out0, the rest to out1
// (contiguous [., 3, H, W])
__global__ void __launch_bounds__(C0_THREADS)
k_conv0_bwd(const float *__restrict__ g, int nb, int H, int W, const float *__restrict__ w0,
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
        const float4 *gp = reinterpret_cast<const float4 *>(g + ((int64_t)img * HW + (int64_t)yy * W + xx) * 64);
#pragma unroll 4
        for (int q = 0; q < 16; q++) {
            const float4 gv = gp[q];
#pragma unroll
            for (int c = 0; c < 3; c++) {
                const float4 wv = sw[(tap * 3 + c) * 16 + q];
                d[c] = fmaf(wv.x, gv.x, fmaf(wv.y, gv.y, fmaf(wv.z, gv.z, fmaf(wv.w, gv.w, d[c]))));
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
// max-pool and its backward
// ---------------------------------------------------------------------------------------------------------
constexpr int EW_THREADS = 256;

// NHWC [img][H][W][C] -> [img][H/2][W/2][C], floor
__global__ void k_pool(const float *__restrict__ in, int nimg, int H, int W, int C, float *__restrict__ out) {
    const int Ho = H / 2, Wo = W / 2, C4 = C / 4;
    const int64_t total = (int64_t)nimg * Ho * Wo * C4;
    const int64_t i = (int64_t)blockIdx.x * EW_THREADS + threadIdx.x;
    if (i >= total) return;
    const int c4 = (int)(i % C4);
    const int64_t po = i / C4;
    const int xo = (int)(po % Wo), yo = (int)((po / Wo) % Ho);
    const int64_t img = po / ((int64_t)Wo * Ho);
    const float4 *src = reinterpret_cast<const float4 *>(in) + ((img * H + 2 * yo) * W + 2 * xo) * C4 + c4;
    const float4 a = src[0], b = src[C4], c = src[(int64_t)W * C4], d = src[(int64_t)W * C4 + C4];
    reinterpret_cast<float4 *>(out)[i] =
        make_float4(max_nan(max_nan(a.x, b.x), max_nan(c.x, d.x)), max_nan(max_nan(a.y, b.y), max_nan(c.y, d.y)),
                    max_nan(max_nan(a.z, b.z), max_nan(c.z, d.z)), max_nan(max_nan(a.w, b.w), max_nan(c.w, d.w)));
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
__global__ void k_unpool_bwd(const float *__restrict__ act, const float *__restrict__ gp, int nimg, int H, int W, int C,
                             float *__restrict__ g) {
    const int Ho = H / 2, Wo = W / 2, C4 = C / 4;
    const int64_t total = (int64_t)nimg * H * W * C4;
    const int64_t i = (int64_t)blockIdx.x * EW_THREADS + threadIdx.x;
    if (i >= total) return;
    const int c4 = (int)(i % C4);
    const int64_t pix = i / C4;
    const int x = (int)(pix % W), y = (int)((pix / W) % H);
    const int64_t img = pix / ((int64_t)W * H);
    if (y >= 2 * Ho || x >= 2 * Wo) return;  // a row or column the floor pool drops: the head's gradient alone
    const int yo = y >> 1, xo = x >> 1, me = (y & 1) * 2 + (x & 1);
    const float4 *a4 = reinterpret_cast<const float4 *>(act);
    const int64_t w0 = ((img * H + 2 * yo) * W + 2 * xo) * C4 + c4;
    const float4 a = a4[w0], b = a4[w0 + C4], c = a4[w0 + (int64_t)W * C4], d = a4[w0 + (int64_t)W * C4 + C4];
    const float4 up = reinterpret_cast<const float4 *>(gp)[((img * Ho + yo) * Wo + xo) * C4 + c4];
    const float4 self = a4[pix * C4 + c4];
    float4 v = reinterpret_cast<float4 *>(g)[i];
    if (first_max(a.x, b.x, c.x, d.x) == me && !(self.x <= 0.f)) v.x = tf32_round(v.x + up.x);
    if (first_max(a.y, b.y, c.y, d.y) == me && !(self.y <= 0.f)) v.y = tf32_round(v.y + up.y);
    if (first_max(a.z, b.z, c.z, d.z) == me && !(self.z <= 0.f)) v.z = tf32_round(v.z + up.z);
    if (first_max(a.w, b.w, c.w, d.w) == me && !(self.w <= 0.f)) v.w = tf32_round(v.w + up.w);
    reinterpret_cast<float4 *>(g)[i] = v;
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
template <int CPL>
__global__ void __launch_bounds__(HD_THREADS)
k_head_fwd(const float *__restrict__ f, int N, int HW, const float *__restrict__ lin, double *__restrict__ partial) {
    constexpr int C = CPL * 32;
    __shared__ double red[HD_WARPS];
    const int img = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float w[CPL];
#pragma unroll
    for (int k = 0; k < CPL; k++) w[k] = lin[lane + 32 * k];
    double acc = 0.0;
    for (int px = blockIdx.x * HD_WARPS + warp; px < HW; px += LP_HEAD_BLOCKS * HD_WARPS) {
        const float *p0 = f + ((int64_t)img * HW + px) * C + lane, *p1 = f + ((int64_t)(img + N) * HW + px) * C + lane;
        float a[CPL], b[CPL], sa = 0.f, sb = 0.f;
#pragma unroll
        for (int k = 0; k < CPL; k++) {
            a[k] = p0[32 * k];
            b[k] = p1[32 * k];
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
template <int CPL>
__global__ void __launch_bounds__(HD_THREADS)
k_head_bwd(const float *__restrict__ f, int N, int i0, int HW, const float *__restrict__ lin,
           const float *__restrict__ dout, float *__restrict__ g) {
    constexpr int C = CPL * 32;
    const int lane = threadIdx.x & 31, px = blockIdx.x * HD_WARPS + (threadIdx.x >> 5);
    if (px >= HW) return;
    const int img = i0 + blockIdx.y, other = img < N ? img + N : img - N;
    const float scale = 2.f * dout[img < N ? img : img - N] / (float)HW;
    const float *p0 = f + ((int64_t)img * HW + px) * C + lane, *p1 = f + ((int64_t)other * HW + px) * C + lane;
    float a[CPL], b[CPL], sa = 0.f, sb = 0.f;
#pragma unroll
    for (int k = 0; k < CPL; k++) {
        a[k] = p0[32 * k];
        b[k] = p1[32 * k];
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
    float *dst = g + ((int64_t)(img - i0) * HW + px) * C + lane;
#pragma unroll
    for (int k = 0; k < CPL; k++) dst[32 * k] = !(a[k] <= 0.f) ? tf32_round((gn[k] - (a[k] / na) * proj) / na) : 0.f;
}

// ---------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------
int64_t align64(int64_t floats) { return (floats + 63) & ~(int64_t)63; }

// workspace carve-up (offsets in floats; every region 256-byte aligned)
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
    int64_t off = 0;
    auto take = [&](int64_t floats) { const int64_t o = off; off += align64(floats); return o; };
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
    p.partial = take(2 * (int64_t)LP_NTAPS * p.N * LP_HEAD_BLOCKS);  // doubles
    p.total = off;
    return p;
}

int check_config(const GsLpipsConfig *c, const char *who) {
    if (!c) return gs_set_error(GS_ERR_INVALID, who);
    if (c->batch < 0 || c->batch > 32767 || c->height < 16 || c->width < 16 || c->height > 16384 || c->width > 16384 ||
        (c->normalize != 0 && c->normalize != 1) || c->grads < 0 || c->grads > 3)
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

int launch_head_fwd(const float *f, int C, int N, int HW, const float *lin, double *partial, cudaStream_t st) {
    const dim3 grid(LP_HEAD_BLOCKS, N);
    switch (C) {
        case 64: k_head_fwd<2><<<grid, HD_THREADS, 0, st>>>(f, N, HW, lin, partial); break;
        case 128: k_head_fwd<4><<<grid, HD_THREADS, 0, st>>>(f, N, HW, lin, partial); break;
        case 256: k_head_fwd<8><<<grid, HD_THREADS, 0, st>>>(f, N, HW, lin, partial); break;
        default: k_head_fwd<16><<<grid, HD_THREADS, 0, st>>>(f, N, HW, lin, partial); break;
    }
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}

int launch_head_bwd(const float *f, int C, int N, int i0, int nb, int HW, const float *lin, const float *dout, float *g,
                    cudaStream_t st) {
    const dim3 grid(blocks_for(HW, HD_WARPS), nb);
    switch (C) {
        case 64: k_head_bwd<2><<<grid, HD_THREADS, 0, st>>>(f, N, i0, HW, lin, dout, g); break;
        case 128: k_head_bwd<4><<<grid, HD_THREADS, 0, st>>>(f, N, i0, HW, lin, dout, g); break;
        case 256: k_head_bwd<8><<<grid, HD_THREADS, 0, st>>>(f, N, i0, HW, lin, dout, g); break;
        default: k_head_bwd<16><<<grid, HD_THREADS, 0, st>>>(f, N, i0, HW, lin, dout, g); break;
    }
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}

}  // namespace

struct GsLpipsWeights {
    void *base;
    const float *fwd[LP_LAYERS], *rot[LP_LAYERS], *bias[LP_LAYERS];  // fwd[0] = conv1_1's [27][64]; rot[0] unused
    const float *lin[LP_NTAPS], *shift, *scale;
};

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

extern "C" GS_API void gs_lpips_weights_destroy(GsLpipsWeights *w) {
    if (!w) return;
    cudaFree(w->base);  // synchronises with the device: no kernel still reads the weights
    delete w;
}

extern "C" GS_API int64_t gs_lpips_workspace_bytes(const GsLpipsConfig *cfg) {
    if (check_config(cfg, "bad GsLpipsConfig") != GS_OK) return -1;
    return (int64_t)sizeof(float) * make_plan(*cfg).total;
}

extern "C" GS_API int gs_lpips_forward(const GsLpipsWeights *w, const GsLpipsConfig *cfg, const float *in0,
                                       const float *in1, void *workspace, float *out, void *stream) {
    if (int rc = check_config(cfg, "bad GsLpipsConfig for gs_lpips_forward")) return rc;
    if (!w || !in0 || !in1 || !workspace || !out)
        return gs_set_error(GS_ERR_INVALID, "gs_lpips_forward: null pointer argument");
    if (reinterpret_cast<uintptr_t>(workspace) & 255u)
        return gs_set_error(GS_ERR_INVALID, "gs_lpips_forward: the workspace must be 256-byte aligned");
    if (cfg->batch == 0) return GS_OK;
    const Plan p = make_plan(*cfg);
    float *ws = static_cast<float *>(workspace);
    double *partial = reinterpret_cast<double *>(ws + p.partial);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int N = p.N, nimg = p.nimg;
    const int64_t in0_stride = cfg->batch > 1 ? cfg->in0_stride : 0, in1_stride = cfg->batch > 1 ? cfg->in1_stride : 0;

    int pp = 0;  // ping-pong buffer the next output goes to (activations not kept)
    auto next_buf = [&](int64_t kept) { if (p.full) return ws + kept; float *r = ws + p.ping[pp]; pp ^= 1; return r; };

    float *cur = next_buf(p.act[0]);
    k_conv0_fwd<<<blocks_for((int64_t)nimg * p.h[0] * p.w[0] * 8, C0_THREADS), C0_THREADS, 0, st>>>(
        in0, in1, in0_stride, in1_stride, N, p.h[0], p.w[0], cfg->normalize, w->fwd[0], w->bias[0], w->shift, w->scale, cur);
    GS_CUDA_OK(cudaGetLastError());
    int pi = 0;
    for (int l = 1; l < LP_LAYERS; l++) {
        const int v = LP_LEVEL[l];
        if (lp_pooled_input(l)) {
            float *pooled = next_buf(p.full ? p.pool[pi] : 0);
            pi++;
            k_pool<<<blocks_for((int64_t)nimg * p.h[v] * p.w[v] * (LP_CIN[l] / 4), EW_THREADS), EW_THREADS, 0, st>>>(
                cur, nimg, p.h[v - 1], p.w[v - 1], LP_CIN[l], pooled);
            GS_CUDA_OK(cudaGetLastError());
            cur = pooled;
        }
        float *o = next_buf(p.act[l]);
        if (int rc = launch_conv(cur, w->fwd[l], w->bias[l], nullptr, o, nimg, p.h[v], p.w[v], LP_CIN[l], LP_COUT[l], st)) return rc;
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

extern "C" GS_API int gs_lpips_backward(const GsLpipsWeights *w, const GsLpipsConfig *cfg, const float *dL_dout,
                                        void *workspace, float *dL_din0, float *dL_din1, void *stream) {
    if (int rc = check_config(cfg, "bad GsLpipsConfig for gs_lpips_backward")) return rc;
    if (!w || !dL_dout || !workspace) return gs_set_error(GS_ERR_INVALID, "gs_lpips_backward: null pointer argument");
    if (reinterpret_cast<uintptr_t>(workspace) & 255u)
        return gs_set_error(GS_ERR_INVALID, "gs_lpips_backward: the workspace must be 256-byte aligned");
    if ((dL_din0 && !(cfg->grads & 1)) || (dL_din1 && !(cfg->grads & 2)))
        return gs_set_error(GS_ERR_INVALID, "gs_lpips_backward: a gradient the forward's config did not provide for (grads)");
    if (cfg->batch == 0 || (!dL_din0 && !dL_din1)) return GS_OK;
    const Plan p = make_plan(*cfg);
    float *ws = static_cast<float *>(workspace);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int N = p.N;
    const int i0 = dL_din0 ? 0 : N, nb = (dL_din0 && dL_din1) ? 2 * N : N;
    // activations of images [i0, i0 + nb)
    auto act = [&](int l) { const int v = LP_LEVEL[l]; return ws + p.act[l] + (int64_t)i0 * p.h[v] * p.w[v] * LP_COUT[l]; };
    float *cur = ws + p.grad[0], *oth = ws + p.grad[1];

    if (int rc = launch_head_bwd(ws + p.act[12], 512, N, i0, nb, p.h[4] * p.w[4], w->lin[4], dL_dout, cur, st)) return rc;
    for (int l = LP_LAYERS - 1; l >= 1; l--) {
        const int v = LP_LEVEL[l];
        // cur = dL/d(pre-activation of layer l) -> oth = dL/d(input of layer l)
        if (int rc = launch_conv(cur, w->rot[l], nullptr, lp_pooled_input(l) ? nullptr : act(l - 1), oth, nb, p.h[v], p.w[v],
                                 LP_COUT[l], LP_CIN[l], st))
            return rc;
        if (lp_pooled_input(l)) {
            const int u = v - 1, t = LP_TAP_OF[l - 1], C = LP_COUT[l - 1];
            if (int rc = launch_head_bwd(ws + p.act[l - 1], C, N, i0, nb, p.h[u] * p.w[u], w->lin[t], dL_dout, cur, st)) return rc;
            k_unpool_bwd<<<blocks_for((int64_t)nb * p.h[u] * p.w[u] * (C / 4), EW_THREADS), EW_THREADS, 0, st>>>(
                act(l - 1), oth, nb, p.h[u], p.w[u], C, cur);
            GS_CUDA_OK(cudaGetLastError());
        } else {
            std::swap(cur, oth);
        }
    }
    k_conv0_bwd<<<blocks_for((int64_t)nb * p.h[0] * p.w[0], C0_THREADS), C0_THREADS, 0, st>>>(
        cur, nb, p.h[0], p.w[0], w->fwd[0], w->scale, cfg->normalize ? 2.f : 1.f, dL_din0 ? dL_din0 : dL_din1, dL_din1,
        dL_din0 ? N : nb);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}
