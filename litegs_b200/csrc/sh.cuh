// sh.cuh -- real spherical-harmonics basis (degree 0..3) and the camera-centre helper.
// Constants and coefficient order follow the reference (GR/compact.cu:554-653): sh_rest rows are
// l=1 (-y, z, -x), l=2 (xy, yz, 2zz-xx-yy, xz, xx-yy), l=3 (7 terms).
#pragma once

template <int DEG>
__device__ __forceinline__ void lgs_sh_basis(float x, float y, float z, float* b)
{
    b[0] = 0.28209479177387814f;
    if (DEG > 0) {
        const float C1 = 0.4886025119029199f;
        b[1] = -C1 * y; b[2] = C1 * z; b[3] = -C1 * x;
        if (DEG > 1) {
            float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
            b[4] = 1.0925484305920792f * xy;
            b[5] = -1.0925484305920792f * yz;
            b[6] = 0.31539156525252005f * (2.0f * zz - xx - yy);
            b[7] = -1.0925484305920792f * xz;
            b[8] = 0.5462742152960396f * (xx - yy);
            if (DEG > 2) {
                b[9] = -0.5900435899266435f * y * (3.0f * xx - yy);
                b[10] = 2.890611442640554f * xy * z;
                b[11] = -0.4570457994644658f * y * (4.0f * zz - xx - yy);
                b[12] = 0.3731763325901154f * z * (2.0f * zz - 3.0f * xx - 3.0f * yy);
                b[13] = -0.4570457994644658f * x * (4.0f * zz - xx - yy);
                b[14] = 1.445305721320277f * z * (xx - yy);
                b[15] = -0.5900435899266435f * x * (xx - 3.0f * yy);
            }
        }
    }
}

// g = sum_k w[k] * d b_k / d(x, y, z) for k = 1 .. (DEG+1)^2 - 1 (b_0 is constant), the polynomial derivatives of
// lgs_sh_basis at the point (x, y, z) (not projected onto the sphere: the caller applies the normalisation's Jacobian).
template <int DEG>
__device__ __forceinline__ void lgs_sh_basis_grad(float x, float y, float z, const float* w, float* g)
{
    g[0] = 0.f; g[1] = 0.f; g[2] = 0.f;
    if constexpr (DEG > 0) {
        const float C1 = 0.4886025119029199f;
        g[0] -= C1 * w[3]; g[1] -= C1 * w[1]; g[2] += C1 * w[2];
        if constexpr (DEG > 1) {
            const float C20 = 1.0925484305920792f, C22 = 0.31539156525252005f, C24 = 0.5462742152960396f;
            g[0] += C20 * (y * w[4] - z * w[7]) + 2.0f * x * (C24 * w[8] - C22 * w[6]);
            g[1] += C20 * (x * w[4] - z * w[5]) - 2.0f * y * (C22 * w[6] + C24 * w[8]);
            g[2] += -C20 * (y * w[5] + x * w[7]) + 4.0f * C22 * z * w[6];
            if constexpr (DEG > 2) {
                const float C30 = -0.5900435899266435f, C31 = 2.890611442640554f, C32 = -0.4570457994644658f;
                const float C33 = 0.3731763325901154f, C34 = -0.4570457994644658f, C35 = 1.445305721320277f;
                const float C36 = -0.5900435899266435f;
                // __fmul_rn: products the compiler cannot share with lgs_sh_basis's, whose FMA contraction (and so the sh_rest
                // gradient) must not depend on whether this function is called
                const float xx = __fmul_rn(x, x), yy = __fmul_rn(y, y), zz = __fmul_rn(z, z);
                const float xy = __fmul_rn(x, y), yz = __fmul_rn(y, z), xz = __fmul_rn(x, z);
                g[0] += 6.0f * C30 * xy * w[9] + C31 * yz * w[10] - 2.0f * C32 * xy * w[11] - 6.0f * C33 * xz * w[12] +
                        C34 * (4.0f * zz - 3.0f * xx - yy) * w[13] + 2.0f * C35 * xz * w[14] + 3.0f * C36 * (xx - yy) * w[15];
                g[1] += 3.0f * C30 * (xx - yy) * w[9] + C31 * xz * w[10] + C32 * (4.0f * zz - xx - 3.0f * yy) * w[11] -
                        6.0f * C33 * yz * w[12] - 2.0f * C34 * xy * w[13] - 2.0f * C35 * yz * w[14] - 6.0f * C36 * xy * w[15];
                g[2] += C31 * xy * w[10] + 8.0f * C32 * yz * w[11] + C33 * (6.0f * zz - 3.0f * xx - 3.0f * yy) * w[12] +
                        8.0f * C34 * xz * w[13] + C35 * (xx - yy) * w[14];
            }
        }
    }
}

// camera centre = -t . R^T with t = V[3,:3], R = V[:3,:3]   (GR/compact.cu:875-879)
__device__ __forceinline__ void lgs_camera_center(const float* __restrict__ Vm, float* c)
{
    float tx = -Vm[12], ty = -Vm[13], tz = -Vm[14];
    c[0] = tx * Vm[0] + ty * Vm[1] + tz * Vm[2];
    c[1] = tx * Vm[4] + ty * Vm[5] + tz * Vm[6];
    c[2] = tx * Vm[8] + ty * Vm[9] + tz * Vm[10];
}
