// gs_poses.cu -- the encoder's pose path between PnP and the networks that read it, DESIGN.md 5.14:
//   gs_pose_sync      PF3plat's camera_synchronization (src/flow_util.py:623-743) at its default arguments
//   gs_refine_poses   encoder_costvolume.py:465-473 (r6d2mat and the 4x4 assembly) and the .inverse() of the result
//   gs_plucker_rays   plucker_embedding(get_world_rays(grid, abspose.inverse(), K)) (encoder_costvolume.py:387-392)
// As stock PyTorch this stretch is ~100 small launches with host reads in between (mass.min().item(), and the
// synchronising torch.linalg.svd / inv).  Here it is two launches for the synchronisation and one for each other op,
// all arithmetic in fp64 from float32 inputs, no atomics and nothing read back by the host.
#include "gs_common.cuh"
#include "gs_inverse.cuh"

namespace {

constexpr int SYNC_THREADS = 256;
constexpr int SYNC_SQUARES = 10;  // camera_synchronization's `squares`: L is raised to the power 2^10

struct SyncParams {
    int batch, views, pairs;
    int8_t pi[GS_POSES_MAX_PAIRS], pj[GS_POSES_MAX_PAIRS];
    int8_t chain[GS_POSES_MAX_VIEWS];  // chain[k]: the pair (k, k+1)
};

__device__ __forceinline__ double nan_min(double m, double x) { return (x < m || isnan(x)) ? x : m; }

// One CTA per scene.  L [4N, 4N] is built in float32 exactly as the reference builds it (the confidences in pair
// order, c/2 added on both diagonals, normalised per column with the sum clamped at 1e-9, c * SE3_inverse(P) and
// c * P), widened to fp64 and squared ten times in shared memory.  Writes column block 0 [N, 4, 4] and the scene's
// smallest mass L[v][3][3] (NaN if anything in the scene is non-finite).
__global__ void __launch_bounds__(SYNC_THREADS)
k_pose_sync_power(SyncParams p, const float *__restrict__ Ps, const float *__restrict__ conf, double *__restrict__ Lc,
                  double *__restrict__ scene_min) {
    extern __shared__ double sm[];
    __shared__ float cf[GS_POSES_MAX_VIEWS][GS_POSES_MAX_VIEWS];
    __shared__ int16_t blk[GS_POSES_MAX_VIEWS][GS_POSES_MAX_VIEWS];  // -1: zero block, 2q: c SE3_inverse(P_q), 2q+1: c P_q
    const int s = blockIdx.x, N = p.views, M = 4 * N;
    double *A = sm, *B = sm + M * M;
    if (threadIdx.x == 0) {
        for (int i = 0; i < N; i++)
            for (int j = 0; j < N; j++) {
                cf[i][j] = 0.0f;
                blk[i][j] = -1;
            }
        for (int q = 0; q < p.pairs; q++) {
            const int i = p.pi[q], j = p.pj[q];
            const float c = conf[(size_t)q * p.batch + s];
            cf[i][j] = c;
            cf[j][i] = c;
            cf[i][i] = cf[i][i] + c / 2.0f;
            cf[j][j] = cf[j][j] + c / 2.0f;
            blk[i][j] = (int16_t)(2 * q);
            blk[j][i] = (int16_t)(2 * q + 1);
        }
        for (int j = 0; j < N; j++) {
            float sum = 0.0f;
            for (int i = 0; i < N; i++) sum += cf[i][j];
            sum = sum < 1e-9f ? 1e-9f : sum;  // clamp(min=1e-9), NaN passes through
            for (int i = 0; i < N; i++) cf[i][j] = cf[i][j] / sum;
        }
    }
    __syncthreads();
    bool bad = false;
    for (int e = threadIdx.x; e < M * M; e += SYNC_THREADS) {
        const int r = e / M, col = e % M, bi = r >> 2, bj = col >> 2, rr = r & 3, cc = col & 3;
        float val;
        if (bi == bj) {
            val = __fmul_rn(cf[bi][bi], rr == cc ? 1.0f : 0.0f);
        } else if (blk[bi][bj] < 0) {
            val = 0.0f;
        } else {
            const int q = blk[bi][bj] >> 1;
            const float *P = Ps + ((size_t)q * p.batch + s) * 16;
            float m;
            if (blk[bi][bj] & 1) {
                m = P[rr * 4 + cc];
            } else if (rr == 3) {
                m = P[12 + cc];  // SE3_inverse keeps P's bottom row
            } else if (cc < 3) {
                m = P[cc * 4 + rr];  // R^T
            } else {
                // (-1 * R^T) @ t, rounded product by product and summed in order (no contraction), so that L's
                // float32 bits are fixed by this definition and the test oracle can restate them exactly
                m = __fadd_rn(__fadd_rn(__fmul_rn(-P[rr], P[3]), __fmul_rn(-P[4 + rr], P[7])), __fmul_rn(-P[8 + rr], P[11]));
            }
            val = __fmul_rn(cf[bi][bj], m);
        }
        bad |= !isfinite(val);
        A[e] = (double)val;
    }
    bad = __syncthreads_or(bad);
    for (int it = 0; it < SYNC_SQUARES; it++) {
        const int cols = it == SYNC_SQUARES - 1 ? 4 : M;  // the last square is read in column block 0 only
        for (int e = threadIdx.x; e < M * cols; e += SYNC_THREADS) {
            const int r = e / cols, c = e % cols;
            double acc = 0.0;
            for (int k = 0; k < M; k++) acc = fma(A[r * M + k], A[k * M + c], acc);
            B[r * M + c] = acc;
        }
        __syncthreads();
        double *t = A;
        A = B;
        B = t;
    }
    bool nonfinite = false;
    for (int e = threadIdx.x; e < 16 * N; e += SYNC_THREADS) {
        const double x = A[((e >> 4) * 4 + ((e >> 2) & 3)) * M + (e & 3)];
        nonfinite |= !isfinite(x);
        Lc[(size_t)s * 16 * N + e] = x;
    }
    bad = __syncthreads_or(bad || nonfinite);
    if (threadIdx.x == 0) {
        double m = A[3 * M + 3];
        for (int v = 1; v < N; v++) m = nan_min(m, A[(4 * v + 3) * M + 3]);
        scene_min[s] = bad ? __longlong_as_double(0x7ff8000000000000ll) : m;
    }
}

__device__ void mat4_mul(const double *a, const double *b, double *o) {
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++) {
            double acc = 0.0;
            for (int k = 0; k < 4; k++) acc = fma(a[i * 4 + k], b[k * 4 + j], acc);
            o[i * 4 + j] = acc;
        }
}

double __device__ det3(const double u[3][3]) {
    return u[0][0] * (u[1][1] * u[2][2] - u[1][2] * u[2][1]) - u[0][1] * (u[1][0] * u[2][2] - u[1][2] * u[2][0]) +
           u[0][2] * (u[1][0] * u[2][1] - u[1][1] * u[2][0]);
}

// R = U diag(1, 1, det(U V^T)) V^T of A = U S V^T, the smallest singular value's direction flipped, by one-sided
// Jacobi on A's columns (W = A V converges to U S).  `a` and `R` are row-major 3x3.
__device__ void so3_project(const double *a, double *R) {
    double W[3][3], V[3][3];
    for (int r = 0; r < 3; r++)
        for (int c = 0; c < 3; c++) {
            W[r][c] = a[r * 3 + c];
            V[r][c] = r == c ? 1.0 : 0.0;
        }
    for (int sweep = 0; sweep < 32; sweep++) {
        bool rotated = false;
        for (int pq = 0; pq < 3; pq++) {
            const int P = pq == 2 ? 1 : 0, Q = pq == 0 ? 1 : 2;
            double al = 0.0, be = 0.0, ga = 0.0;
            for (int r = 0; r < 3; r++) {
                al += W[r][P] * W[r][P];
                be += W[r][Q] * W[r][Q];
                ga += W[r][P] * W[r][Q];
            }
            if (!(fabs(ga) > 1e-15 * sqrt(al * be))) continue;
            rotated = true;
            const double zeta = (be - al) / (2.0 * ga);
            const double t = copysign(1.0, zeta) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
            const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
            for (int r = 0; r < 3; r++) {
                const double wp = W[r][P], wq = W[r][Q], vp = V[r][P], vq = V[r][Q];
                W[r][P] = c * wp - s * wq;
                W[r][Q] = s * wp + c * wq;
                V[r][P] = c * vp - s * vq;
                V[r][Q] = s * vp + c * vq;
            }
        }
        if (!rotated) break;
    }
    double sig[3];
    for (int c = 0; c < 3; c++) sig[c] = sqrt(W[0][c] * W[0][c] + W[1][c] * W[1][c] + W[2][c] * W[2][c]);
    int kmin = 0;
    for (int c = 1; c < 3; c++)
        if (sig[c] < sig[kmin]) kmin = c;
    for (int c = 0; c < 3; c++)
        if (sig[c] > 0.0)
            for (int r = 0; r < 3; r++) W[r][c] /= sig[c];
    for (int c = 0; c < 3; c++) {
        if (c == kmin || sig[c] > 0.0) continue;
        // rank <= 1: a zero column besides kmin becomes a unit vector orthogonal to the other non-kmin column o: e_c if
        // o is zero too (so the zero block projects to I, as LAPACK's SVD of zeros gives), else the axis least aligned
        // with o minus its projection on o
        const int o = 3 - c - kmin;
        double e[3] = {0.0, 0.0, 0.0};
        if (sig[o] > 0.0) {
            int m = 0;
            for (int r = 1; r < 3; r++)
                if (fabs(W[r][o]) < fabs(W[m][o])) m = r;
            for (int r = 0; r < 3; r++) e[r] = (r == m ? 1.0 : 0.0) - W[m][o] * W[r][o];
            const double n = sqrt(e[0] * e[0] + e[1] * e[1] + e[2] * e[2]);
            for (int r = 0; r < 3; r++) e[r] /= n;
        } else {
            e[c] = 1.0;
        }
        for (int r = 0; r < 3; r++) W[r][c] = e[r];
    }
    if (!(sig[kmin] > 0.0)) {  // rank 2 or less: complete U by the cross product of its other two columns
        const int k1 = (kmin + 1) % 3, k2 = (kmin + 2) % 3;
        for (int r = 0; r < 3; r++)
            W[r][kmin] = W[(r + 1) % 3][k1] * W[(r + 2) % 3][k2] - W[(r + 2) % 3][k1] * W[(r + 1) % 3][k2];
    }
    const double d = det3(W) * det3(V);
    for (int r = 0; r < 3; r++)
        for (int c = 0; c < 3; c++) {
            double acc = 0.0;
            for (int k = 0; k < 3; k++) acc += (k == kmin ? d : 1.0) * W[r][k] * V[c][k];
            R[r * 3 + c] = acc;
        }
}

// One thread per (scene, view).  The batch-wide smallest mass is reduced in scene order by every thread; if it is
// exactly 0 (or views == 2) the scene is chained, P(v-1, v) ... P(0, 1) I, otherwise column block 0 is divided by its
// mass (clamped at 1e-9) and its rotation projected onto SO(3).
__global__ void k_pose_sync_finish(SyncParams p, int chain_only, const float *__restrict__ Ps,
                                   const double *__restrict__ Lc, const double *__restrict__ scene_min,
                                   float *__restrict__ out) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= p.batch * p.views) return;
    const int s = t / p.views, v = t % p.views;
    float *o = out + (size_t)t * 16;
    bool chain = chain_only != 0;
    if (!chain) {
        double g = scene_min[0];
        for (int q = 1; q < p.batch; q++) g = nan_min(g, scene_min[q]);
        chain = g == 0.0;
    }
    if (chain) {
        double Mx[16], P[16], T[16];
        for (int i = 0; i < 16; i++) Mx[i] = (i % 5 == 0) ? 1.0 : 0.0;
        for (int k = 0; k < v; k++) {
            const float *src = Ps + ((size_t)p.chain[k] * p.batch + s) * 16;
            for (int i = 0; i < 16; i++) P[i] = src[i];
            mat4_mul(P, Mx, T);
            for (int i = 0; i < 16; i++) Mx[i] = T[i];
        }
        for (int i = 0; i < 16; i++) o[i] = (float)Mx[i];
        return;
    }
    if (isnan(scene_min[s])) {
        for (int i = 0; i < 16; i++) o[i] = __int_as_float(0x7fc00000);
        return;
    }
    double L[16], Rp[9], R[9];
    const double *src = Lc + (size_t)t * 16;
    const double mass = src[15] < 1e-9 ? 1e-9 : src[15];
    for (int i = 0; i < 16; i++) L[i] = src[i] / mass;
    for (int r = 0; r < 3; r++)
        for (int c = 0; c < 3; c++) Rp[r * 3 + c] = L[r * 4 + c];
    so3_project(Rp, R);
    for (int r = 0; r < 3; r++) {
        for (int c = 0; c < 3; c++) o[r * 4 + c] = (float)R[r * 3 + c];
        o[r * 4 + 3] = (float)L[r * 4 + 3];
    }
    for (int c = 0; c < 4; c++) o[12 + c] = (float)L[12 + c];
}

// ---- refined poses ----

constexpr double NORMALIZE_EPS = 1e-12;  // F.normalize's default eps

struct Refined {
    double x[9], n1, b1[3], s, c[3], n2, b2[3], b3[3], A[16], Ai[16];
};

__device__ void cross3(const double *a, const double *b, double *o) {
    o[0] = a[1] * b[2] - a[2] * b[1];
    o[1] = a[2] * b[0] - a[0] * b[2];
    o[2] = a[0] * b[1] - a[1] * b[0];
}

__device__ void refine(const float *pose_enc, const float *delta, double gamma, int item, int v, Refined &f) {
    for (int k = 0; k < 9; k++) {
        f.x[k] = pose_enc[(size_t)item * 9 + k];
        if (v > 0) f.x[k] += (double)delta[(size_t)item * 9 + k] * gamma;
    }
    const double *a1 = f.x, *a2 = f.x + 3;
    f.n1 = sqrt(a1[0] * a1[0] + a1[1] * a1[1] + a1[2] * a1[2]);
    const double m1 = fmax(f.n1, NORMALIZE_EPS);
    for (int k = 0; k < 3; k++) f.b1[k] = a1[k] / m1;
    f.s = f.b1[0] * a2[0] + f.b1[1] * a2[1] + f.b1[2] * a2[2];
    for (int k = 0; k < 3; k++) f.c[k] = a2[k] - f.s * f.b1[k];
    f.n2 = sqrt(f.c[0] * f.c[0] + f.c[1] * f.c[1] + f.c[2] * f.c[2]);
    const double m2 = fmax(f.n2, NORMALIZE_EPS);
    for (int k = 0; k < 3; k++) f.b2[k] = f.c[k] / m2;
    cross3(f.b1, f.b2, f.b3);
    const double *rows[3] = {f.b1, f.b2, f.b3};
    for (int r = 0; r < 3; r++) {
        for (int k = 0; k < 3; k++) f.A[r * 4 + k] = rows[r][k];
        f.A[r * 4 + 3] = f.x[6 + r];
    }
    f.A[12] = f.A[13] = f.A[14] = 0.0;
    f.A[15] = 1.0;
    inverse4(f.A, f.Ai);
}

__global__ void k_refine_forward(int items, int views, const float *__restrict__ pose_enc,
                                 const float *__restrict__ delta, const float *__restrict__ gamma,
                                 float *__restrict__ abspose, float *__restrict__ abspose_inv) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= items) return;
    Refined f;
    refine(pose_enc, delta, gamma[0], t, t % views, f);
    for (int i = 0; i < 16; i++) {
        abspose[(size_t)t * 16 + i] = (float)f.A[i];
        abspose_inv[(size_t)t * 16 + i] = (float)f.Ai[i];
    }
}

// F.normalize's backward: y = x / max(|x|, eps); the clamp passes the norm's gradient where |x| >= eps
__device__ void normalize_bwd(const double *y, double n, const double *g, double *gx) {
    if (n >= NORMALIZE_EPS) {
        const double yg = y[0] * g[0] + y[1] * g[1] + y[2] * g[2];
        for (int k = 0; k < 3; k++) gx[k] = (g[k] - y[k] * yg) / n;
    } else {
        for (int k = 0; k < 3; k++) gx[k] = g[k] / NORMALIZE_EPS;
    }
}

constexpr int REFINE_BWD_THREADS = 256;

// One CTA: every (scene, view) is a loop iteration of one thread, and dL/dgamma is reduced in fp64 in a fixed order.
__global__ void __launch_bounds__(REFINE_BWD_THREADS)
k_refine_backward(int items, int views, const float *__restrict__ pose_enc, const float *__restrict__ delta,
                  const float *__restrict__ gamma, const float *__restrict__ g_abs, const float *__restrict__ g_inv,
                  float *__restrict__ d_pose_enc, float *__restrict__ d_delta, float *__restrict__ d_gamma) {
    __shared__ double red[REFINE_BWD_THREADS];
    const double gm = gamma[0];
    double part = 0.0;
    for (int t = threadIdx.x; t < items; t += REFINE_BWD_THREADS) {
        const int v = t % views;
        Refined f;
        refine(pose_enc, delta, gm, t, v, f);
        double G[16];
        for (int i = 0; i < 16; i++) G[i] = g_abs ? (double)g_abs[(size_t)t * 16 + i] : 0.0;
        if (g_inv) {  // d(A^-1) -> -A^-T G A^-T
            double Gi[16], T[16];
            for (int i = 0; i < 16; i++) Gi[i] = g_inv[(size_t)t * 16 + i];
            for (int k = 0; k < 4; k++)
                for (int c = 0; c < 4; c++) {
                    double acc = 0.0;
                    for (int l = 0; l < 4; l++) acc += Gi[k * 4 + l] * f.Ai[c * 4 + l];
                    T[k * 4 + c] = acc;
                }
            for (int r = 0; r < 4; r++)
                for (int c = 0; c < 4; c++) {
                    double acc = 0.0;
                    for (int k = 0; k < 4; k++) acc += f.Ai[k * 4 + r] * T[k * 4 + c];
                    G[r * 4 + c] -= acc;
                }
        }
        double gb1[3], gb2[3], gb3[3], gx[9], tmp[3], gc[3];
        for (int k = 0; k < 3; k++) {
            gb1[k] = G[k];
            gb2[k] = G[4 + k];
            gb3[k] = G[8 + k];
            gx[6 + k] = G[k * 4 + 3];
        }
        cross3(f.b2, gb3, tmp);  // b3 = b1 x b2
        for (int k = 0; k < 3; k++) gb1[k] += tmp[k];
        cross3(gb3, f.b1, tmp);
        for (int k = 0; k < 3; k++) gb2[k] += tmp[k];
        normalize_bwd(f.b2, f.n2, gb2, gc);
        const double gcb1 = gc[0] * f.b1[0] + gc[1] * f.b1[1] + gc[2] * f.b1[2];
        for (int k = 0; k < 3; k++) {  // c = a2 - (b1 . a2) b1
            gx[3 + k] = gc[k] - gcb1 * f.b1[k];
            gb1[k] += -f.s * gc[k] - gcb1 * f.x[3 + k];
        }
        normalize_bwd(f.b1, f.n1, gb1, gx);
        for (int k = 0; k < 9; k++) {
            const double dk = delta[(size_t)t * 9 + k];
            d_pose_enc[(size_t)t * 9 + k] = (float)gx[k];
            d_delta[(size_t)t * 9 + k] = v > 0 ? (float)(gx[k] * gm) : 0.0f;
            if (v > 0) part += gx[k] * dk;
        }
    }
    red[threadIdx.x] = part;
    __syncthreads();
    for (int w = REFINE_BWD_THREADS / 2; w > 0; w >>= 1) {
        if (threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
        __syncthreads();
    }
    if (threadIdx.x == 0) d_gamma[0] = (float)red[0];
}

// ---- Plücker rays ----

constexpr int PLUCKER_THREADS = 256;

__global__ void __launch_bounds__(PLUCKER_THREADS)
k_plucker_rays(int height, int width, const float *__restrict__ abspose, const float *__restrict__ intrinsics,
               float *__restrict__ out) {
    __shared__ double c2w[16], kinv[9];
    const int vb = blockIdx.y;
    if (threadIdx.x == 0) {
        double e[16], k[9];
        for (int i = 0; i < 16; i++) e[i] = abspose[(size_t)vb * 16 + i];
        for (int i = 0; i < 9; i++) k[i] = intrinsics[(size_t)vb * 9 + i];
        inverse4(e, c2w);
        inverse3(k, kinv);
    }
    __syncthreads();
    const int hw = height * width, px = blockIdx.x * PLUCKER_THREADS + threadIdx.x;
    if (px >= hw) return;
    const double x = ((px % width) + 0.5) / width, y = ((px / width) + 0.5) / height;
    double d[3], dw[3], o[3], m[3];
    for (int i = 0; i < 3; i++) d[i] = kinv[i * 3] * x + kinv[i * 3 + 1] * y + kinv[i * 3 + 2];
    const double n = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
    for (int i = 0; i < 3; i++) d[i] /= n;
    for (int i = 0; i < 3; i++) {  // homogeneous w = 0: c2w[i][3] * 0 is kept, so a non-finite origin poisons the ray
        dw[i] = c2w[i * 4] * d[0] + c2w[i * 4 + 1] * d[1] + c2w[i * 4 + 2] * d[2] + c2w[i * 4 + 3] * 0.0;
        o[i] = c2w[i * 4 + 3];
    }
    cross3(o, dw, m);
    float *dst = out + (size_t)vb * 6 * hw + px;
    for (int i = 0; i < 3; i++) {
        dst[(size_t)i * hw] = (float)dw[i];
        dst[(size_t)(3 + i) * hw] = (float)m[i];
    }
}

size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

// validates the pairs and fills the kernels' parameter block
int sync_params(const GsPoseSyncConfig *c, SyncParams *sp) {
    if (!c) return gs_set_error(GS_ERR_INVALID, "pose sync: null config");
    const int N = c->views;
    if (N < 2 || N > GS_POSES_MAX_VIEWS || c->batch < 1 || c->batch > 65535 || c->pairs < 1 ||
        c->pairs > N * (N - 1) / 2)
        return gs_set_error(GS_ERR_INVALID, "pose sync: need 2 <= views <= 16, 1 <= batch <= 65535, "
                                            "1 <= pairs <= views (views - 1) / 2");
    SyncParams p{};
    p.batch = c->batch;
    p.views = N;
    p.pairs = c->pairs;
    bool seen[GS_POSES_MAX_VIEWS][GS_POSES_MAX_VIEWS] = {}, covered[GS_POSES_MAX_VIEWS] = {};
    for (int k = 0; k < GS_POSES_MAX_VIEWS; k++) p.chain[k] = -1;
    for (int q = 0; q < c->pairs; q++) {
        const int i = c->pair_i[q], j = c->pair_j[q];
        if (i < 0 || j < 0 || i >= N || j >= N || i == j)
            return gs_set_error(GS_ERR_INVALID, "pose sync: a pair (i, j) needs 0 <= i, j < views and i != j");
        if (seen[i][j] || seen[j][i]) return gs_set_error(GS_ERR_INVALID, "pose sync: a pair repeats");
        seen[i][j] = covered[i] = covered[j] = true;
        p.pi[q] = (int8_t)i;
        p.pj[q] = (int8_t)j;
        if (j == i + 1) p.chain[i] = (int8_t)q;
    }
    for (int k = 0; k < N; k++)
        if (!covered[k]) return gs_set_error(GS_ERR_INVALID, "pose sync: a view is in no pair");
    for (int k = 0; k + 1 < N; k++)
        if (p.chain[k] < 0) return gs_set_error(GS_ERR_INVALID, "pose sync: the chain needs every pair (k, k+1)");
    *sp = p;
    return GS_OK;
}

size_t sync_scratch(const GsPoseSyncConfig *c, char *base, double **Lc, double **mins) {
    const size_t a = align256(sizeof(double) * 16 * c->batch * c->views);
    if (base) {
        *Lc = reinterpret_cast<double *>(base);
        *mins = reinterpret_cast<double *>(base + a);
    }
    return a + align256(sizeof(double) * c->batch);
}

int check_refine(const GsRefinePosesConfig *c, const GsRefinePosesInputs *in) {
    if (!c || c->batch < 1 || c->views < 1 || (int64_t)c->batch * c->views > (1 << 24))
        return gs_set_error(GS_ERR_INVALID, "refine poses: need batch >= 1, views >= 1, batch views <= 2^24");
    if (!in || !in->pose_enc || !in->delta || !in->gamma)
        return gs_set_error(GS_ERR_INVALID, "refine poses: null input pointer");
    return GS_OK;
}

}  // namespace

extern "C" GS_API int64_t gs_pose_sync_scratch_bytes(const GsPoseSyncConfig *cfg) {
    SyncParams p;
    if (sync_params(cfg, &p)) return -1;
    return (int64_t)sync_scratch(cfg, nullptr, nullptr, nullptr);
}

extern "C" GS_API int gs_pose_sync(const GsPoseSyncConfig *cfg, const float *Ps, const float *confidence, float *out,
                                   void *scratch, void *stream) {
    SyncParams p;
    if (int rc = sync_params(cfg, &p)) return rc;
    const bool chain_only = cfg->views == 2;
    if (!Ps || !out || (!chain_only && !confidence))
        return gs_set_error(GS_ERR_INVALID, "gs_pose_sync: null pointer");
    if (!chain_only && (!scratch || (reinterpret_cast<uintptr_t>(scratch) & 255u)))
        return gs_set_error(GS_ERR_INVALID, "gs_pose_sync: scratch must be non-null and 256-byte aligned");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    double *Lc = nullptr, *mins = nullptr;
    if (!chain_only) {
        sync_scratch(cfg, static_cast<char *>(scratch), &Lc, &mins);
        const int M = 4 * cfg->views;
        const size_t smem = 2 * sizeof(double) * M * M;
        GS_CUDA_OK(cudaFuncSetAttribute(k_pose_sync_power, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        k_pose_sync_power<<<cfg->batch, SYNC_THREADS, smem, st>>>(p, Ps, confidence, Lc, mins);
        GS_CUDA_OK(cudaGetLastError());
    }
    const int n = cfg->batch * cfg->views;
    k_pose_sync_finish<<<(n + 127) / 128, 128, 0, st>>>(p, chain_only ? 1 : 0, Ps, Lc, mins, out);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}

extern "C" GS_API int gs_refine_poses_forward(const GsRefinePosesConfig *cfg, const GsRefinePosesInputs *in,
                                              float *abspose, float *abspose_inv, void *stream) {
    if (int rc = check_refine(cfg, in)) return rc;
    if (!abspose || !abspose_inv) return gs_set_error(GS_ERR_INVALID, "gs_refine_poses_forward: null output pointer");
    const int n = cfg->batch * cfg->views;
    k_refine_forward<<<(n + 127) / 128, 128, 0, static_cast<cudaStream_t>(stream)>>>(
        n, cfg->views, in->pose_enc, in->delta, in->gamma, abspose, abspose_inv);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}

extern "C" GS_API int gs_refine_poses_backward(const GsRefinePosesConfig *cfg, const GsRefinePosesInputs *in,
                                               const GsRefinePosesGrads *grads, void *stream) {
    if (int rc = check_refine(cfg, in)) return rc;
    if (!grads || !grads->dL_dpose_enc || !grads->dL_ddelta || !grads->dL_dgamma)
        return gs_set_error(GS_ERR_INVALID, "gs_refine_poses_backward: null gradient pointer");
    k_refine_backward<<<1, REFINE_BWD_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
        cfg->batch * cfg->views, cfg->views, in->pose_enc, in->delta, in->gamma, grads->dL_dabspose,
        grads->dL_dabspose_inv, grads->dL_dpose_enc, grads->dL_ddelta, grads->dL_dgamma);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}

extern "C" GS_API int gs_plucker_rays(const GsPluckerConfig *cfg, const float *abspose, const float *intrinsics,
                                      float *out, void *stream) {
    if (!cfg || cfg->batch < 1 || cfg->views < 1 || cfg->height < 1 || cfg->width < 1 ||
        (int64_t)cfg->batch * cfg->views > 65535 || (int64_t)cfg->height * cfg->width > (1 << 28))
        return gs_set_error(GS_ERR_INVALID, "gs_plucker_rays: need batch, views, height, width >= 1, batch views <= "
                                            "65535, height width <= 2^28");
    if (!abspose || !intrinsics || !out) return gs_set_error(GS_ERR_INVALID, "gs_plucker_rays: null pointer");
    const int hw = cfg->height * cfg->width;
    const dim3 grid((hw + PLUCKER_THREADS - 1) / PLUCKER_THREADS, cfg->batch * cfg->views);
    k_plucker_rays<<<grid, PLUCKER_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(cfg->height, cfg->width, abspose,
                                                                                   intrinsics, out);
    GS_CUDA_OK(cudaGetLastError());
    return GS_OK;
}
