// projection.cuh -- the per-Gaussian projection formulas, one device definition each, called by both the op-level kernels
// (per_gaussian.cu) and the fused projection (fused.cu), so the oracle tests of the op-level kernels check the code the
// fused path runs (fused.cu names the two it writes out).  Plain values in and out: each caller keeps its own loads and stores (the SH colour excepted, which
// reads its coefficients through base pointers and a stride).  Matrices are row-vector, [i*4+j]; per-Gaussian small
// matrices are row-major in registers.
#pragma once
#include "sh.cuh"

// activation (GR/compact.cu:825-893): scale exp(s_raw), unit quaternion qn = q_raw * rn (returns rn = 1/|q_raw|), opacity
// sigmoid(o_raw)
__device__ __forceinline__ void lgs_activate_scale(const float* s_raw, float* s)
{
#pragma unroll
    for (int k = 0; k < 3; k++) s[k] = expf(s_raw[k]);
}

__device__ __forceinline__ float lgs_normalize_quat(const float* q_raw, float* qn)
{
    const float rn = 1.0f / sqrtf(q_raw[0] * q_raw[0] + q_raw[1] * q_raw[1] + q_raw[2] * q_raw[2] + q_raw[3] * q_raw[3] + 1e-12f);
#pragma unroll
    for (int k = 0; k < 4; k++) qn[k] = q_raw[k] * rn;
    return rn;
}

__device__ __forceinline__ float lgs_sigmoid(float o_raw) { return 1.0f / (1.0f + expf(-o_raw)); }

// d q_raw of a gradient dq at the unit quaternion qn = q_raw * rn
__device__ __forceinline__ void lgs_quat_normalize_backward(const float* dq, const float* qn, float rn, float* d)
{
    const float dot = dq[0] * qn[0] + dq[1] * qn[1] + dq[2] * qn[2] + dq[3] * qn[3];
#pragma unroll
    for (int k = 0; k < 4; k++) d[k] = rn * (dq[k] - dot * qn[k]);
}

// d o_raw of d o.  true_sigmoid = 0 keeps the reference's d_o * sigma(x) (GR/compact.cu:952, SURVEY Q15); 1 gives the analytic
// sigma (1 - sigma).  1 - sig is u itself: forming it from the rounded sig cancels for saturated logits.
__device__ __forceinline__ float lgs_sigmoid_backward(float d_o, float o_raw, int true_sigmoid)
{
    const float u = 1.0f / (1.0f + expf(o_raw)), sig = 1.0f - u;
    return d_o * (true_sigmoid ? sig * u : sig);
}

// unit view direction dirn of the world position p from the camera centre of Vm (GR/compact.cu:875-881); returns 1/|p - cc|
__device__ __forceinline__ float lgs_view_dir(const float* __restrict__ Vm, const float* p, float* dirn)
{
    float cc[3];
    lgs_camera_center(Vm, cc);
    const float d0 = p[0] - cc[0], d1 = p[1] - cc[1], d2 = p[2] - cc[2];
    const float dn = 1.0f / sqrtf(d0 * d0 + d1 * d1 + d2 * d2 + 1e-12f);
    dirn[0] = d0 * dn; dirn[1] = d1 * dn; dirn[2] = d2 * dn;
    return dn;
}

// colour of direction (x, y, z) (GR/compact.cu:573-653), no clamp: coefficient k of channel c is sh0[c * stride + i] (k = 0) or
// shr[((k - 1) * 3 + c) * stride + i]
template <int DEG>
__device__ __forceinline__ void lgs_sh_color(float x, float y, float z, const float* __restrict__ sh0, const float* __restrict__ shr,
                                             size_t i, size_t stride, float* col)
{
    constexpr int K = (DEG + 1) * (DEG + 1);
    float b[16];
    lgs_sh_basis<DEG>(x, y, z, b);
#pragma unroll
    for (int c = 0; c < 3; c++) {
        float acc = b[0] * sh0[c * stride + i];
#pragma unroll
        for (int k = 1; k < K; k++) acc += b[k] * shr[((size_t)(k - 1) * 3 + c) * stride + i];
        col[c] = acc + 0.5f;
    }
}

// MVP (GR/transform.cu:398-436): view position v = w . Vm of the homogeneous world position w
__device__ __forceinline__ void lgs_mvp_view(const float* __restrict__ Vm, const float* w, float* v)
{
#pragma unroll
    for (int k = 0; k < 4; k++) v[k] = w[0] * Vm[k] + w[1] * Vm[4 + k] + w[2] * Vm[8 + k] + w[3] * Vm[12 + k];
}

// clip position h = v . P; returns iw = 1/h_w (0 when |h_w| <= 1e-12), ndc = h * iw
__device__ __forceinline__ float lgs_mvp_clip(const float* __restrict__ P, const float* v, float* h)
{
#pragma unroll
    for (int k = 0; k < 4; k++) h[k] = v[0] * P[k] + v[1] * P[4 + k] + v[2] * P[8 + k] + v[3] * P[12 + k];
    return (fabsf(h[3]) > 1e-12f) ? (1.0f / h[3]) : 0.0f;
}

// MVP backward (GR/transform.cu:517-558), clip half: dh and dv = dh . P^T + gv from d ndc (x, y, z) gn and a view-space
// gradient gv
__device__ __forceinline__ void lgs_mvp_clip_backward(const float* __restrict__ P, const float* h, float iw, const float* gn,
                                                      const float* gv, float* dh, float* dv)
{
    const float n0 = h[0] * iw, n1 = h[1] * iw, n2 = h[2] * iw;
    dh[0] = gn[0] * iw; dh[1] = gn[1] * iw; dh[2] = gn[2] * iw;
    dh[3] = -(gn[0] * n0 + gn[1] * n1 + gn[2] * n2) * iw;
#pragma unroll
    for (int k = 0; k < 4; k++) dv[k] = dh[0] * P[k * 4] + dh[1] * P[k * 4 + 1] + dh[2] * P[k * 4 + 2] + dh[3] * P[k * 4 + 3] + gv[k];
}

// view half: d w = dv . Vm^T
__device__ __forceinline__ void lgs_mvp_view_backward(const float* __restrict__ Vm, const float* dv, float* dw)
{
#pragma unroll
    for (int k = 0; k < 4; k++) dw[k] = dv[0] * Vm[k * 4] + dv[1] * Vm[k * 4 + 1] + dv[2] * Vm[k * 4 + 2] + dv[3] * Vm[k * 4 + 3];
}

// rotation R of the unit quaternion (r, x, y, z) (GR/transform.cu:106-125); row a of T = diag(s) R is R's row a times s_a
__device__ __forceinline__ void lgs_quat_R(float r, float x, float y, float z, float* R)
{
    R[0] = 1 - 2 * (y * y + z * z); R[1] = 2 * (x * y + r * z);     R[2] = 2 * (x * z - r * y);
    R[3] = 2 * (x * y - r * z);     R[4] = 1 - 2 * (x * x + z * z); R[5] = 2 * (y * z + r * x);
    R[6] = 2 * (x * z + r * y);     R[7] = 2 * (y * z - r * x);     R[8] = 1 - 2 * (x * x + y * y);
}

// d (r, x, y, z) of a gradient dR of lgs_quat_R's output (GR/transform.cu:185-226)
__device__ __forceinline__ void lgs_quat_R_backward(float r, float x, float y, float z, const float* dR, float* dq)
{
    dq[0] = 2 * z * (dR[1] - dR[3]) + 2 * y * (dR[6] - dR[2]) + 2 * x * (dR[5] - dR[7]);
    dq[1] = 2 * y * (dR[3] + dR[1]) + 2 * z * (dR[6] + dR[2]) + 2 * r * (dR[5] - dR[7]) - 4 * x * (dR[8] + dR[4]);
    dq[2] = 2 * x * (dR[3] + dR[1]) + 2 * r * (dR[6] - dR[2]) + 2 * z * (dR[5] + dR[7]) - 4 * y * (dR[8] + dR[0]);
    dq[3] = 2 * r * (dR[1] - dR[3]) + 2 * x * (dR[6] + dR[2]) + 2 * y * (dR[5] + dR[7]) - 4 * z * (dR[4] + dR[0]);
}

// row a of T = diag(s) R backward: returns d s_a from the gradient dT of the row, and scales dT in place to the gradient of R's row
__device__ __forceinline__ float lgs_scale_rot_backward(const float* R, float s, float* dT)
{
    const float ds = R[0] * dT[0] + R[1] * dT[1] + R[2] * dT[2];
    dT[0] *= s; dT[1] *= s; dT[2] *= s;
    return ds;
}

// ray-space Jacobian J[a*2+c] (a = 0..2, c = 0..1) at the view position v (GR/transform.cu:36-50): only (0,0), (1,1), (2,0)
// and (2,1) are non-zero
__device__ __forceinline__ void lgs_ray_J(const float* __restrict__ P, const float* v, int H, int W, float* J)
{
    float p00 = P[0], p11 = P[5];
    float fx = p00 * W * 0.5f, fy = p11 * H * 0.5f;
    float tx = v[0], ty = v[1], tz = v[2];
    float lx = tz / p00 * 1.3f, ly = tz / p11 * 1.3f;
    tx = fmaxf(fminf(tx, lx), -lx);
    ty = fmaxf(fminf(ty, ly), -ly);
    float rz = 1.0f / fmaxf(tz, 1e-2f);
    float rz2 = rz * rz;
    J[0] = fx * rz; J[1] = 0.f; J[2] = 0.f; J[3] = fy * rz; J[4] = -fx * tx * rz2; J[5] = -fy * ty * rz2;
}

// VJ = V3x3 . J and M = T . VJ (GR/transform.cu:761-769) with T = diag(s) R, R row-major [9] (a caller holding T itself passes it
// as R with s = 1)
__device__ __forceinline__ void lgs_cov_M(const float* __restrict__ Vm, const float* J, const float* R, const float* s, float* VJ,
                                          float* M)
{
#pragma unroll
    for (int a = 0; a < 3; a++)
#pragma unroll
        for (int c = 0; c < 2; c++) {
            float acc = 0.f;
#pragma unroll
            for (int k = 0; k < 3; k++) acc += Vm[a * 4 + k] * J[k * 2 + c];
            VJ[a * 2 + c] = acc;
        }
#pragma unroll
    for (int a = 0; a < 3; a++)
#pragma unroll
        for (int c = 0; c < 2; c++) {
            float acc = 0.f;
#pragma unroll
            for (int k = 0; k < 3; k++) acc += (R[a * 3 + k] * s[a]) * VJ[k * 2 + c];
            M[a * 2 + c] = acc;
        }
}

// 2D covariance M^T M + 0.3 I: (c00, c01 = c10, c11)
__device__ __forceinline__ void lgs_cov2d(const float* M, float& c00, float& c01, float& c11)
{
    c00 = M[0] * M[0] + M[2] * M[2] + M[4] * M[4] + 0.3f;
    c01 = M[0] * M[1] + M[2] * M[3] + M[4] * M[5];
    c11 = M[1] * M[1] + M[3] * M[3] + M[5] * M[5] + 0.3f;
}

// guarded inverse of [[m00, m01], [m10, m11]] (GR/transform.cu:1379-1419), inv row-major [4]
__device__ __forceinline__ void lgs_inv2x2(float m00, float m01, float m10, float m11, float* inv)
{
    float det = m00 * m11 - m01 * m10;
    float det1 = (m00 - m01) * (m11 - m01) + m01 * (m00 + m11 - 2 * m01);
    det = (fabsf(det) < fabsf(1e-5f * m01 * m10)) ? det1 : det;
    det = (fabsf(det) < 1e-9f) ? 1e-9f : det;
    float dr = 1.0f / det;
    inv[0] = m11 * dr; inv[1] = -m01 * dr; inv[2] = -m10 * dr; inv[3] = m00 * dr;
}

// inverse backward d m = -(inv . d inv . inv) (GR/transform.cu:1446-1450), all row-major [4]
__device__ __forceinline__ void lgs_inv2x2_backward(const float* A, const float* G, float* d)
{
    const float t0 = A[0] * G[0] + A[1] * G[2], t1 = A[0] * G[1] + A[1] * G[3];
    const float t2 = A[2] * G[0] + A[3] * G[2], t3 = A[2] * G[1] + A[3] * G[3];
    d[0] = -(t0 * A[0] + t1 * A[2]);
    d[1] = -(t0 * A[1] + t1 * A[3]);
    d[2] = -(t2 * A[0] + t3 * A[2]);
    d[3] = -(t2 * A[1] + t3 * A[3]);
}

// 2D covariance backward (GR/transform.cu:861-880): dM = 2 M G for the gradient G [4] of M^T M, and dT = dM . VJ^T
__device__ __forceinline__ void lgs_cov2d_backward(const float* M, const float* VJ, const float* G, float* dM, float* dT)
{
#pragma unroll
    for (int a = 0; a < 3; a++) {
#pragma unroll
        for (int c = 0; c < 2; c++) dM[a * 2 + c] = 2.f * (M[a * 2] * G[c] + M[a * 2 + 1] * G[2 + c]);
#pragma unroll
        for (int k = 0; k < 3; k++) dT[a * 3 + k] = dM[a * 2] * VJ[k * 2] + dM[a * 2 + 1] * VJ[k * 2 + 1];
    }
}
