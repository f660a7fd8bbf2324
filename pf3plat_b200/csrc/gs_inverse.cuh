// gs_inverse.cuh -- fp64 inverses of row-major 3x3 and 4x4 matrices by cofactors, shared by the camera glue
// (gs_cameras.cu) and the pose path (gs_poses.cu).  A singular matrix divides by a zero determinant: the result is
// non-finite, nothing traps.
#pragma once

static __device__ void inverse3(const double *m, double *o) {
    const double c00 = m[4] * m[8] - m[5] * m[7], c01 = m[5] * m[6] - m[3] * m[8], c02 = m[3] * m[7] - m[4] * m[6];
    const double inv = 1.0 / (m[0] * c00 + m[1] * c01 + m[2] * c02);
    o[0] = c00 * inv; o[1] = (m[2] * m[7] - m[1] * m[8]) * inv; o[2] = (m[1] * m[5] - m[2] * m[4]) * inv;
    o[3] = c01 * inv; o[4] = (m[0] * m[8] - m[2] * m[6]) * inv; o[5] = (m[2] * m[3] - m[0] * m[5]) * inv;
    o[6] = c02 * inv; o[7] = (m[1] * m[6] - m[0] * m[7]) * inv; o[8] = (m[0] * m[4] - m[1] * m[3]) * inv;
}

// general 4x4 inverse (the reference calls .inverse() on camera matrices, not a rigid-body shortcut)
static __device__ void inverse4(const double *m, double *o) {
    const double s0 = m[0] * m[5] - m[4] * m[1], s1 = m[0] * m[6] - m[4] * m[2], s2 = m[0] * m[7] - m[4] * m[3];
    const double s3 = m[1] * m[6] - m[5] * m[2], s4 = m[1] * m[7] - m[5] * m[3], s5 = m[2] * m[7] - m[6] * m[3];
    const double c5 = m[10] * m[15] - m[14] * m[11], c4 = m[9] * m[15] - m[13] * m[11], c3 = m[9] * m[14] - m[13] * m[10];
    const double c2 = m[8] * m[15] - m[12] * m[11], c1 = m[8] * m[14] - m[12] * m[10], c0 = m[8] * m[13] - m[12] * m[9];
    const double inv = 1.0 / (s0 * c5 - s1 * c4 + s2 * c3 + s3 * c2 - s4 * c1 + s5 * c0);
    o[0] = (m[5] * c5 - m[6] * c4 + m[7] * c3) * inv;
    o[1] = (-m[1] * c5 + m[2] * c4 - m[3] * c3) * inv;
    o[2] = (m[13] * s5 - m[14] * s4 + m[15] * s3) * inv;
    o[3] = (-m[9] * s5 + m[10] * s4 - m[11] * s3) * inv;
    o[4] = (-m[4] * c5 + m[6] * c2 - m[7] * c1) * inv;
    o[5] = (m[0] * c5 - m[2] * c2 + m[3] * c1) * inv;
    o[6] = (-m[12] * s5 + m[14] * s2 - m[15] * s1) * inv;
    o[7] = (m[8] * s5 - m[10] * s2 + m[11] * s1) * inv;
    o[8] = (m[4] * c4 - m[5] * c2 + m[7] * c0) * inv;
    o[9] = (-m[0] * c4 + m[1] * c2 - m[3] * c0) * inv;
    o[10] = (m[12] * s4 - m[13] * s2 + m[15] * s0) * inv;
    o[11] = (-m[8] * s4 + m[9] * s2 - m[11] * s0) * inv;
    o[12] = (-m[4] * c3 + m[5] * c1 - m[6] * c0) * inv;
    o[13] = (m[0] * c3 - m[1] * c1 + m[2] * c0) * inv;
    o[14] = (-m[12] * s3 + m[13] * s1 - m[14] * s0) * inv;
    o[15] = (m[8] * s3 - m[9] * s1 + m[10] * s0) * inv;
}
