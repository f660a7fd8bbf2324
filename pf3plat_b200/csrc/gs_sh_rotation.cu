// gs_sh_rotation.cu -- every camera's block-diagonal Wigner-D matrix after the reference's rotation guard, DESIGN.md 5.17:
// PF3plat's src/misc/sh_rotation.py:10-36 as pf3plat_b200/sh_rotation.py evaluates it without e3nn.
//   k_sh_rotation_guard   one CTA: torch.allclose(torch.det(R), 1) over the whole call (rtol 1e-5, atol 1e-8), with
//                         det in fp64 from the fp32 entries; a NaN or +-Inf determinant fails.  Writes one int flag.
//   k_sh_rotation_blocks  one CTA per camera: R (or I when the flag is 0, substituted before the fit, as the tensor
//                         route does), then per degree l <= 4 D_l = Y_l(R X) pinv(Y_l(X)^T) over the 64 fixed unit
//                         vectors of gs_sh_fit.h, all in fp64 with fixed-order sums, rounded to fp32 once.  Every
//                         element of [d_sh, d_sh] is written, the exact zeros off the diagonal blocks included.
// Two launches, no atomics, no memset, nothing read back by the host; a camera's matrix depends on its rotation and
// the flag only, not on N or on its position in the batch.
#include "gs_common.cuh"
#include "gs_sh_fit.h"

namespace {

constexpr int GUARD_THREADS = 1024;
constexpr int BLOCK_THREADS = GS_SH_FIT_NPTS;  // one thread per fit point
constexpr int MAX_D_SH = 25;
constexpr int YS_ROW = BLOCK_THREADS + 1;     // doubles per row of the basis table in shared memory

struct ShRotParams {
    const float *base;
    int64_t outer_stride, inner_stride;
    int32_t inner, row_stride, d_sh, degrees;
};

__device__ __forceinline__ const float *matrix_at(const ShRotParams &p, int cam) {
    const int i = cam / p.inner, s = cam - i * p.inner;
    return p.base + (int64_t)i * p.outer_stride + (int64_t)s * p.inner_stride;
}

// isclose(det, 1) as allclose applies it: |det - 1| <= atol + rtol |1|; a NaN or infinite det compares false
__device__ __forceinline__ bool det_is_one(const float *m, int rs) {
    const double a = m[0], b = m[1], c = m[2];
    const double d = m[rs], e = m[rs + 1], f = m[rs + 2];
    const double g = m[2 * rs], h = m[2 * rs + 1], i = m[2 * rs + 2];
    const double det = a * (e * i - f * h) - b * (d * i - f * g) + c * (d * h - e * g);
    return fabs(det - 1.0) <= 1e-8 + 1e-5;
}

__global__ void __launch_bounds__(GUARD_THREADS) k_sh_rotation_guard(ShRotParams p, int n, int *flag) {
    bool ok = true;
#pragma unroll 4
    for (int cam = threadIdx.x; cam < n; cam += GUARD_THREADS) ok &= det_is_one(matrix_at(p, cam), p.row_stride);
    ok = __syncthreads_and(ok);
    if (threadIdx.x == 0) *flag = ok ? 1 : 0;
}

// real_sh_basis(degree, m) of sh_rotation.py, statement for statement (left-to-right products), written to
// y[i * YS_ROW] for the 2 degree + 1 components
__device__ __forceinline__ void real_sh_basis(int degree, const double m[3], double *y) {
    const double x = m[2], yv = m[0], z = m[1];
    const double xx = x * x, yy = yv * yv, zz = z * z;
    constexpr int S = YS_ROW;
    if (degree == 0) {
        y[0] = 0.28209479177387814;
    } else if (degree == 1) {
        const double c = 0.4886025119029199;
        y[0] = c * yv;
        y[S] = c * z;
        y[2 * S] = c * x;
    } else if (degree == 2) {
        y[0] = 1.0925484305920792 * x * yv;
        y[S] = 1.0925484305920792 * yv * z;
        y[2 * S] = 0.31539156525252005 * (2 * zz - xx - yy);
        y[3 * S] = 1.0925484305920792 * x * z;
        y[4 * S] = 0.5462742152960396 * (xx - yy);
    } else if (degree == 3) {
        y[0] = 0.5900435899266435 * yv * (3 * xx - yy);
        y[S] = 2.890611442640554 * x * yv * z;
        y[2 * S] = 0.4570457994644658 * yv * (4 * zz - xx - yy);
        y[3 * S] = 0.3731763325901154 * z * (2 * zz - 3 * xx - 3 * yy);
        y[4 * S] = 0.4570457994644658 * x * (4 * zz - xx - yy);
        y[5 * S] = 1.445305721320277 * z * (xx - yy);
        y[6 * S] = 0.5900435899266435 * x * (xx - 3 * yy);
    } else {
        const double rr = xx + yy + zz;
        y[0] = 2.5033429417967046 * x * yv * (xx - yy);
        y[S] = 1.7701307697799304 * yv * z * (3 * xx - yy);
        y[2 * S] = 0.9461746957575601 * x * yv * (7 * zz - rr);
        y[3 * S] = 0.6690465435572892 * yv * z * (7 * zz - 3 * rr);
        y[4 * S] = 0.10578554691520431 * (35 * zz * zz - 30 * zz * rr + 3 * rr * rr);
        y[5 * S] = 0.6690465435572892 * x * z * (7 * zz - 3 * rr);
        y[6 * S] = 0.47308734787878004 * (xx - yy) * (7 * zz - rr);
        y[7 * S] = 1.7701307697799304 * x * z * (xx - 3 * yy);
        y[8 * S] = 0.6258357354491761 * (xx * (xx - 3 * yy) - yy * (3 * xx - yy));
    }
}

__device__ __forceinline__ int degree_of(int row) {
    int l = 0;
    while ((l + 1) * (l + 1) <= row) l++;
    return l;
}

// entries of the blocks of degrees < l: sum_{m < l} (2m + 1)^2 = l (2l - 1) (2l + 1) / 3
__device__ __forceinline__ int block_entries(int l) { return l * (2 * l - 1) * (2 * l + 1) / 3; }

__global__ void __launch_bounds__(BLOCK_THREADS) k_sh_rotation_blocks(ShRotParams p, const int *flag, float *out) {
    // ys[l^2 + i][k] = Y_l,i(R x_k); rows padded by one so that lanes on different rows hit different banks
    __shared__ double ys[MAX_D_SH][YS_ROW];
    const int cam = blockIdx.x, k = threadIdx.x;
    double r[9] = {1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0};
    if (*flag) {
        const float *m = matrix_at(p, cam);
#pragma unroll
        for (int a = 0; a < 3; a++)
#pragma unroll
            for (int c = 0; c < 3; c++) r[3 * a + c] = m[a * p.row_stride + c];
    }
    for (int l = 0; l < p.degrees; l++) {
        const double *x = GS_SH_FIT_POINTS[l][k];
        const double x0 = x[0], x1 = x[1], x2 = x[2];
        double moved[3];
#pragma unroll
        for (int a = 0; a < 3; a++) moved[a] = r[3 * a] * x0 + r[3 * a + 1] * x1 + r[3 * a + 2] * x2;  // R x_k
        real_sh_basis(l, moved, &ys[l * l][k]);
    }
    const int d = p.d_sh, dd = d * d;
    float *o = out + (int64_t)cam * dd;
    for (int e = k; e < dd; e += BLOCK_THREADS) {  // the exact zeros off the diagonal blocks
        const int i = e / d, j = e - i * d;
        if (degree_of(i) != degree_of(j)) o[e] = 0.0f;
    }
    __syncthreads();
    // the blocks' entries only, sum_l (2l + 1)^2 of them, so that no lane idles on a zero
    const int nnz = block_entries(p.degrees);
    for (int t = k; t < nnz; t += BLOCK_THREADS) {
        int l = 0;
        while (t >= block_entries(l + 1)) l++;
        const int n = 2 * l + 1, local = t - block_entries(l);
        const int i = l * l + local / n, jl = local - (local / n) * n;
        const double *pinv = GS_SH_FIT_PINV + GS_SH_FIT_NPTS * l * l + jl;
        const double *yi = ys[i];
        double acc = 0.0;
        for (int q = 0; q < GS_SH_FIT_NPTS; q++) acc += yi[q] * pinv[q * n];  // fixed order
        o[i * d + l * l + jl] = (float)acc;
    }
}

int sh_params(const GsShRotationConfig *c, const float *rotations, ShRotParams *p) {
    if (!c) return gs_set_error(GS_ERR_INVALID, "gs_sh_rotation: null config");
    if (c->d_sh != 1 && c->d_sh != 4 && c->d_sh != 9 && c->d_sh != 16 && c->d_sh != 25)
        return gs_set_error(GS_ERR_INVALID, "gs_sh_rotation: d_sh must be 1, 4, 9, 16 or 25");
    if (c->outer < 1 || c->inner < 1 || (int64_t)c->outer * c->inner > INT32_MAX)
        return gs_set_error(GS_ERR_INVALID, "gs_sh_rotation: need outer, inner >= 1 and N = outer inner < 2^31");
    if (c->row_stride != 3 && c->row_stride != 4)
        return gs_set_error(GS_ERR_INVALID, "gs_sh_rotation: row_stride must be 3 or 4");
    p->base = rotations;
    p->outer_stride = c->outer_stride;
    p->inner_stride = c->inner_stride;
    p->inner = c->inner;
    p->row_stride = c->row_stride;
    p->d_sh = c->d_sh;
    p->degrees = c->d_sh == 1 ? 1 : c->d_sh == 4 ? 2 : c->d_sh == 9 ? 3 : c->d_sh == 16 ? 4 : 5;
    return GS_OK;
}

}  // namespace

extern "C" GS_API int64_t gs_sh_rotation_workspace_bytes(const GsShRotationConfig *cfg) {
    ShRotParams p;
    if (sh_params(cfg, nullptr, &p)) return -1;
    return 16;
}

extern "C" GS_API int gs_sh_rotation_blocks(const GsShRotationConfig *cfg, const float *rotations, float *out,
                                            void *workspace, void *stream) {
    ShRotParams p;
    if (int rc = sh_params(cfg, rotations, &p)) return rc;
    if (!rotations || !out || !workspace) return gs_set_error(GS_ERR_INVALID, "gs_sh_rotation_blocks: null pointer");
    const int n = cfg->outer * cfg->inner;
    int *flag = static_cast<int *>(workspace);
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    k_sh_rotation_guard<<<1, GUARD_THREADS, 0, st>>>(p, n, flag);
    GS_CUDA_OK(cudaGetLastError());
    k_sh_rotation_blocks<<<n, BLOCK_THREADS, 0, st>>>(p, flag, out);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}
