// gs_optimizer.cu -- PF3plat's optimizer step on the device, DESIGN.md 5.19: the NaN-gradient skip of
// ModelWrapper.optimizer_step (src/model/model_wrapper.py:224-238), Lightning's clip_grad_norm_ and torch.optim.Adam's
// foreach update, then zero_grad, over a multi-tensor chunk table in three launches:
//   k_adam_norm    one CTA per chunk: the chunk's sum of squares of its gradient, in fp64, and its NaN flag (x != x,
//                  so an Inf is not mistaken for a NaN).
//   k_adam_reduce  one CTA: the partials in a fixed order -> the skip verdict and coef = min(max_norm / (total + 1e-6),
//                  1) in fp32 as torch forms it (reciprocal, then product).  total is the fp64 sum's square root
//                  rounded to fp32 once, independent of the summation order up to fp64 rounding (torch sums in fp32);
//                  a sum past FLT_MAX gives total = inf, as torch's fp32 squares overflow.  Unless skipped, every
//                  listed tensor's step + 1 and its step size -lr / (1 - beta1^step) and sqrt(1 - beta2^step) in fp64,
//                  rounded to fp32 once where torch's foreach kernels round their Python scalars.  A skip adds one to
//                  the caller's counter.
//   k_adam_update  one CTA per chunk: nothing but the zeroing of the gradient when the step is skipped; otherwise
//                  grad, param and both moments read once, param and both moments written, the gradient zeroed.
// No float atomics: every result is the same bit for bit from run to run.  Nothing is read back by the host.
#include <float.h>

#include "gs_common.cuh"

namespace {

constexpr int THREADS = 256;
constexpr int REDUCE_THREADS = 1024;
constexpr size_t ALIGN = 256;

struct AdamVerdict {
    int skip;
    float coef;
};

// torch's float32 view of the Python scalars of _multi_tensor_adam (non-capturable) and clip_grad_norm_
struct AdamScalars {
    float lerp_w;        // 1 - beta1: _foreach_lerp_(exp_avgs, grads, 1 - beta1)
    float lerp_w_c;      // 1 - lerp_w in fp32, the other side of torch's lerp
    float beta2;         // _foreach_mul_(exp_avg_sqs, beta2)
    float one_m_beta2;   // _foreach_addcmul_(exp_avg_sqs, grads, grads, 1 - beta2)
    float eps;           // _foreach_add_(denom, eps)
    int clip;            // max_norm >= 0: grads were multiplied by coef
    int zero_grads;
};

struct ScratchLayout {
    size_t partial, flags, verdict, tensor_scalars, total;
};

size_t align_up(size_t x) { return (x + ALIGN - 1) / ALIGN * ALIGN; }

ScratchLayout layout_of(const GsAdamConfig *c) {
    ScratchLayout l;
    l.partial = 0;
    l.flags = l.partial + align_up((size_t)c->chunks * sizeof(double));
    l.verdict = l.flags + align_up((size_t)c->chunks * sizeof(int));
    l.tensor_scalars = l.verdict + ALIGN;
    l.total = l.tensor_scalars + align_up((size_t)c->tensors * sizeof(float2));
    return l;
}

__device__ __forceinline__ bool aligned16(const void *p) { return ((uintptr_t)p & 15) == 0; }

// sum over a CTA's threads in a fixed order: a shuffle tree per warp, then the warps' sums in index order by thread 0
template <int NT>
__device__ __forceinline__ double block_sum(double s, double *warp_sums) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = s;
    __syncthreads();
    double total = 0.0;
    if (threadIdx.x == 0)
#pragma unroll
        for (int w = 0; w < NT / 32; w++) total += warp_sums[w];
    return total;  // thread 0 only
}

__global__ void __launch_bounds__(THREADS) k_adam_norm(const GsAdamChunk *__restrict__ chunks, double *partial,
                                                        int *nan_flags) {
    __shared__ double warp_sums[THREADS / 32];
    const GsAdamChunk c = chunks[blockIdx.x];
    const float *g = c.grad + c.begin;
    const int n = c.count;
    double s = 0.0;
    bool nan = false;
    int i0 = 0;
    if (aligned16(g)) {
        const float4 *g4 = reinterpret_cast<const float4 *>(g);
        const int n4 = n >> 2;
#pragma unroll 4
        for (int i = threadIdx.x; i < n4; i += THREADS) {
            const float4 x = g4[i];
            s = fma((double)x.x, (double)x.x, s);
            s = fma((double)x.y, (double)x.y, s);
            s = fma((double)x.z, (double)x.z, s);
            s = fma((double)x.w, (double)x.w, s);
            nan |= (x.x != x.x) | (x.y != x.y) | (x.z != x.z) | (x.w != x.w);
        }
        i0 = n4 << 2;
    }
    for (int i = i0 + threadIdx.x; i < n; i += THREADS) {  // the tail, or the whole of an unaligned chunk
        const double x = g[i];
        s = fma(x, x, s);
        nan |= x != x;
    }
    nan = __syncthreads_or(nan);
    const double total = block_sum<THREADS>(s, warp_sums);
    if (threadIdx.x == 0) {
        partial[blockIdx.x] = total;
        nan_flags[blockIdx.x] = nan ? 1 : 0;
    }
}

__global__ void __launch_bounds__(REDUCE_THREADS) k_adam_reduce(const GsAdamChunk *__restrict__ chunks, int n_chunks,
                                                                int n_tensors, const double *partial,
                                                                const int *nan_flags, double beta1, double beta2,
                                                                float max_norm, float *steps, const float *lr,
                                                                int32_t *skipped, AdamVerdict *verdict,
                                                                float2 *tensor_scalars) {
    __shared__ double warp_sums[REDUCE_THREADS / 32];
    double s = 0.0;
    int nan = 0;
    for (int c = threadIdx.x; c < n_chunks; c += REDUCE_THREADS) {
        s += partial[c];
        nan |= nan_flags[c];
    }
    const bool skip = __syncthreads_or(nan);
    const double sumsq = block_sum<REDUCE_THREADS>(s, warp_sums);
    if (threadIdx.x == 0) {
        float coef = 1.0f;
        if (max_norm >= 0.0f) {  // clip_grads_with_norm_: max_norm / (total + 1e-6) is reciprocal() * max_norm
            const float total = sumsq > (double)FLT_MAX ? INFINITY : (float)sqrt(sumsq);
            coef = fminf((1.0f / (total + 1e-6f)) * max_norm, 1.0f);
        }
        verdict->skip = skip ? 1 : 0;
        verdict->coef = coef;
        if (skip) *skipped += 1;
    }
    if (skip) return;
    const double lr_d = (double)*lr;
    for (int c = threadIdx.x; c < n_chunks; c += REDUCE_THREADS) {
        const int t = chunks[c].tensor;
        if ((c > 0 && chunks[c - 1].tensor == t) || t < 0 || t >= n_tensors) continue;  // once per tensor
        const float step = steps[t] + 1.0f;  // _foreach_add_(state_steps, 1) on float32 steps
        steps[t] = step;
        const double bc1 = 1.0 - pow(beta1, (double)step);
        const double bc2 = 1.0 - pow(beta2, (double)step);
        tensor_scalars[t] = make_float2((float)(-(lr_d / bc1)), (float)sqrt(bc2));
    }
}

// one element of _multi_tensor_adam after the clip, each foreach op's arithmetic as torch's CUDA functors form it
__device__ __forceinline__ void adam_element(float &p, float g, float &m, float &v, float step_size, float bc2_sqrt,
                                             const AdamScalars &k) {
    // at::native::lerp: self + w (end - self) for |w| < 0.5, else end - (end - self) (1 - w)
    m = k.lerp_w < 0.5f ? fmaf(k.lerp_w, g - m, m) : fmaf(-(g - m), k.lerp_w_c, g);
    v = fmaf(k.one_m_beta2, g * g, v * k.beta2);   // mul_(beta2), then self + value (g g)
    const float denom = sqrtf(v) / bc2_sqrt + k.eps;
    p = fmaf(step_size, m / denom, p);             // addcdiv: self + value (m / denom)
}

__global__ void __launch_bounds__(THREADS) k_adam_update(const GsAdamChunk *__restrict__ chunks, int n_tensors,
                                                          const AdamVerdict *verdict,
                                                          const float2 *__restrict__ tensor_scalars, AdamScalars k) {
    const GsAdamChunk c = chunks[blockIdx.x];
    const AdamVerdict vd = *verdict;
    const int n = c.count;
    float *gp = c.grad + c.begin;
    if (vd.skip || c.tensor < 0 || c.tensor >= n_tensors) {
        if (!k.zero_grads) return;
        int i0 = 0;
        if (aligned16(gp)) {
            float4 *g4 = reinterpret_cast<float4 *>(gp);
            for (int i = threadIdx.x; i < (n >> 2); i += THREADS) g4[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
            i0 = n & ~3;
        }
        for (int i = i0 + threadIdx.x; i < n; i += THREADS) gp[i] = 0.0f;
        return;
    }
    const float coef = vd.coef;
    const float2 ts = tensor_scalars[c.tensor];
    float *pp = c.param + c.begin, *mp = c.exp_avg + c.begin, *vp = c.exp_avg_sq + c.begin;
    const bool store_g = k.zero_grads || k.clip;  // clip_grad_norm_ leaves the clipped gradient behind
    int i0 = 0;
    if (aligned16(gp) && aligned16(pp) && aligned16(mp) && aligned16(vp)) {
        float4 *g4 = reinterpret_cast<float4 *>(gp), *p4 = reinterpret_cast<float4 *>(pp);
        float4 *m4 = reinterpret_cast<float4 *>(mp), *v4 = reinterpret_cast<float4 *>(vp);
        const int n4 = n >> 2;
#pragma unroll 2
        for (int i = threadIdx.x; i < n4; i += THREADS) {
            float4 g = g4[i], p = p4[i], m = m4[i], v = v4[i];
            if (k.clip) g = make_float4(g.x * coef, g.y * coef, g.z * coef, g.w * coef);
            adam_element(p.x, g.x, m.x, v.x, ts.x, ts.y, k);
            adam_element(p.y, g.y, m.y, v.y, ts.x, ts.y, k);
            adam_element(p.z, g.z, m.z, v.z, ts.x, ts.y, k);
            adam_element(p.w, g.w, m.w, v.w, ts.x, ts.y, k);
            p4[i] = p;
            m4[i] = m;
            v4[i] = v;
            if (store_g) g4[i] = k.zero_grads ? make_float4(0.0f, 0.0f, 0.0f, 0.0f) : g;
        }
        i0 = n4 << 2;
    }
    for (int i = i0 + threadIdx.x; i < n; i += THREADS) {  // the tail, or the whole of a misaligned chunk
        float g = gp[i], p = pp[i], m = mp[i], v = vp[i];
        if (k.clip) g *= coef;
        adam_element(p, g, m, v, ts.x, ts.y, k);
        pp[i] = p;
        mp[i] = m;
        vp[i] = v;
        if (store_g) gp[i] = k.zero_grads ? 0.0f : g;
    }
}

int check_config(const GsAdamConfig *c) {
    if (!c) return gs_set_error(GS_ERR_INVALID, "gs_adam: null config");
    if (c->tensors < 1 || c->chunks < 1) return gs_set_error(GS_ERR_INVALID, "gs_adam: need tensors >= 1 and chunks >= 1");
    if (!(c->beta1 >= 0.0 && c->beta1 < 1.0) || !(c->beta2 >= 0.0 && c->beta2 < 1.0))
        return gs_set_error(GS_ERR_INVALID, "gs_adam: beta1 and beta2 must lie in [0, 1)");
    if (!(c->eps >= 0.0 && c->eps < INFINITY)) return gs_set_error(GS_ERR_INVALID, "gs_adam: eps must be finite and >= 0");
    if (c->max_norm != c->max_norm || c->max_norm == INFINITY || c->max_norm == -INFINITY)
        return gs_set_error(GS_ERR_INVALID, "gs_adam: max_norm must be finite (< 0: no clip)");
    if (c->zero_grads != 0 && c->zero_grads != 1) return gs_set_error(GS_ERR_INVALID, "gs_adam: zero_grads must be 0 or 1");
    return GS_OK;
}

}  // namespace

extern "C" GS_API int64_t gs_adam_scratch_bytes(const GsAdamConfig *cfg) {
    if (check_config(cfg)) return -1;
    return (int64_t)layout_of(cfg).total;
}

extern "C" GS_API int gs_adam_step(const GsAdamConfig *cfg, const GsAdamChunk *chunks, float *steps, const float *lr,
                                   int32_t *skipped, void *scratch, void *stream) {
    if (int rc = check_config(cfg)) return rc;
    if (!chunks || !steps || !lr || !skipped || !scratch) return gs_set_error(GS_ERR_INVALID, "gs_adam_step: null pointer");
    if ((uintptr_t)scratch % ALIGN) return gs_set_error(GS_ERR_INVALID, "gs_adam_step: scratch must be 256-byte aligned");
    const ScratchLayout l = layout_of(cfg);
    char *base = static_cast<char *>(scratch);
    double *partial = reinterpret_cast<double *>(base + l.partial);
    int *flags = reinterpret_cast<int *>(base + l.flags);
    AdamVerdict *verdict = reinterpret_cast<AdamVerdict *>(base + l.verdict);
    float2 *tensor_scalars = reinterpret_cast<float2 *>(base + l.tensor_scalars);
    AdamScalars k;
    k.lerp_w = (float)(1.0 - cfg->beta1);
    k.lerp_w_c = 1.0f - k.lerp_w;
    k.beta2 = (float)cfg->beta2;
    k.one_m_beta2 = (float)(1.0 - cfg->beta2);
    k.eps = (float)cfg->eps;
    k.clip = cfg->max_norm >= 0.0;
    k.zero_grads = cfg->zero_grads;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    k_adam_norm<<<cfg->chunks, THREADS, 0, st>>>(chunks, partial, flags);
    GS_CUDA_OK(cudaGetLastError());
    k_adam_reduce<<<1, REDUCE_THREADS, 0, st>>>(chunks, cfg->chunks, cfg->tensors, partial, flags, cfg->beta1,
                                                cfg->beta2, k.clip ? (float)cfg->max_norm : -1.0f, steps, lr, skipped,
                                                verdict, tensor_scalars);
    GS_CUDA_OK(cudaGetLastError());
    k_adam_update<<<cfg->chunks, THREADS, 0, st>>>(chunks, cfg->tensors, verdict, tensor_scalars, k);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}
