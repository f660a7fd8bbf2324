// gs_cameras.cu -- the camera glue of the render boundary for all views of a call in ONE tiny kernel.
//
// Restates what render_cuda does before its per-view loop, PF3plat's src/model/decoder/cuda_splatting.py:64-87,
// with the helpers it calls: get_fov (PF3plat's src/geometry/projection.py:233-247) and get_projection_matrix
// (cuda_splatting.py:17-44).  The reference spends ~50 small tensor ops here (two matrix inversions through cuSOLVER,
// four host-built constants copied to the device, per-view `.item()` syncs); at PF3plat's call sizes that host-side
// time is comparable to the rasterizer itself.  One thread per view, arithmetic in fp64, results rounded to fp32.
#include "gs_common.cuh"
#include "gs_inverse.cuh"

namespace {

__device__ double ray_dot(const double *kinv, double ax, double ay, double bx, double by) {
    double a[3], b[3];
    for (int i = 0; i < 3; i++) {
        a[i] = kinv[i * 3] * ax + kinv[i * 3 + 1] * ay + kinv[i * 3 + 2];
        b[i] = kinv[i * 3] * bx + kinv[i * 3 + 1] * by + kinv[i * 3 + 2];
    }
    const double na = sqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]), nb = sqrt(b[0] * b[0] + b[1] * b[1] + b[2] * b[2]);
    return (a[0] * b[0] + a[1] * b[1] + a[2] * b[2]) / (na * nb);
}

__global__ void k_view_batch(int B, int scale_invariant, const float *__restrict__ extrinsics,
                             const float *__restrict__ intrinsics, const float *__restrict__ near_,
                             const float *__restrict__ far_, float *__restrict__ viewmatrix, float *__restrict__ projmatrix,
                             float *__restrict__ campos, float *__restrict__ tanfov, float *__restrict__ scale_out) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= B) return;
    double e[16], k[9], kinv[9], w2c[16];
    for (int i = 0; i < 16; i++) e[i] = extrinsics[(size_t)v * 16 + i];
    for (int i = 0; i < 9; i++) k[i] = intrinsics[(size_t)v * 9 + i];
    double nr = near_[v], fr = far_[v], s = 1.0;
    if (scale_invariant) {                       // cuda_splatting.py:64-71: the scene is rescaled by 1/near
        s = 1.0 / nr;
        e[3] *= s; e[7] *= s; e[11] *= s;
        nr *= s;
        fr *= s;
    }
    inverse3(k, kinv);
    // get_fov: angle between the rays through the mid-points of opposite image edges
    const double fov_x = acos(ray_dot(kinv, 0.0, 0.5, 1.0, 0.5)), fov_y = acos(ray_dot(kinv, 0.5, 0.0, 0.5, 1.0));
    const double tx = tan(0.5 * fov_x), ty = tan(0.5 * fov_y);
    // get_projection_matrix (row-major p), then both matrices transposed as the rasterizer expects them
    const double top = ty * nr, right = tx * nr;
    double p[16] = {0};
    p[0] = 2.0 * nr / (2.0 * right);
    p[5] = 2.0 * nr / (2.0 * top);
    p[14] = 1.0;
    p[10] = fr / (fr - nr);
    p[11] = -(fr * nr) / (fr - nr);
    inverse4(e, w2c);
    float *vm = viewmatrix + (size_t)v * 16, *pm = projmatrix + (size_t)v * 16;
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++) {
            vm[i * 4 + j] = (float)w2c[j * 4 + i];  // view^T
            double acc = 0.0;                      // full = view^T @ proj^T  ->  full[i][j] = sum_k w2c[k][i] * p[j][k]
            for (int q = 0; q < 4; q++) acc += w2c[q * 4 + i] * p[j * 4 + q];
            pm[i * 4 + j] = (float)acc;
        }
    campos[(size_t)v * 3 + 0] = (float)e[3];
    campos[(size_t)v * 3 + 1] = (float)e[7];
    campos[(size_t)v * 3 + 2] = (float)e[11];
    tanfov[(size_t)v * 2 + 0] = (float)tx;
    tanfov[(size_t)v * 2 + 1] = (float)ty;
    scale_out[v] = (float)s;
}

}  // namespace

extern "C" GS_API int gs_view_batch(int32_t B, int32_t scale_invariant, const float *extrinsics, const float *intrinsics,
                                    const float *near_, const float *far_, float *viewmatrix, float *projmatrix, float *campos,
                                    float *tanfov, float *view_scale, void *stream) {
    if (B < 0) return gs_set_error(GS_ERR_INVALID, "negative view count");
    if (B == 0) return GS_OK;
    if (!extrinsics || !intrinsics || !near_ || !far_ || !viewmatrix || !projmatrix || !campos || !tanfov || !view_scale)
        return gs_set_error(GS_ERR_INVALID, "gs_view_batch: null argument");
    k_view_batch<<<(B + 63) / 64, 64, 0, static_cast<cudaStream_t>(stream)>>>(B, scale_invariant, extrinsics, intrinsics, near_,
                                                                               far_, viewmatrix, projmatrix, campos, tanfov,
                                                                               view_scale);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}
