/*
 * oracle_core.h -- CPU restatement of the LiteGS render hot path (TEST INFRASTRUCTURE ONLY).
 *
 * This file is included twice by oracle.c: once with REAL=float (the fp32 parity oracle)
 * and once with REAL=double (finite-difference / gradcheck tier).  It is NOT part of the
 * product: nothing under litegs_b200/ may include, link or call it.
 *
 * Every function cites the reference file:line (relative to the reference's litegs/submodules/
 * gaussian_raster/, abbreviated GR/) whose arithmetic it restates.  Layouts are the reference's:
 * SoA with the point index innermost, row-vector matrices.
 *
 * PARITY PINNING: the reference ships no CPU path, no golden vectors and no test for this path
 * (SURVEY.md section 8c).  The restatement is pinned against the reference's own CUDA kernels run on
 * an H100 (oracle/build_ref.py -> oracle/_ref, fixtures under tests/golden/) -- see DESIGN.md.
 */

#ifndef REAL
#error "include from oracle.c"
#endif

/* ---- helpers ------------------------------------------------------------------------- */

/* CUDA float->int conversion semantics (cvt.rzi.s32.f32): NaN -> 0, saturating. The reference
 * relies on them implicitly in GR/binning.cu:345-352 and GR/speedy_splat.cuh:122-127. */
static inline int SUF(f2i_rz)(REAL x)
{
    if (x != x) return 0;
    if (x >= (REAL)2147483647.0) return 2147483647;
    if (x <= (REAL)-2147483648.0) return (-2147483647 - 1);
    return (int)x;
}
static inline int SUF(imin)(int a, int b) { return a < b ? a : b; }
static inline int SUF(imax)(int a, int b) { return a > b ? a : b; }

/* ---- frustum culling of chunk AABBs ---------------------------------------------------- */
/* GR/compact.cu:419-501 (visibility test) ; ids are emitted in ascending order (the reference's
 * atomics give an arbitrary order, which is semantically irrelevant). */
void SUF(orc_frustum_culling_aabb)(const REAL* origin, const REAL* ext, const REAL* planes,
                                  int M, int V, uint8_t* visibility, int64_t* ids, int32_t* count)
{
    int c = 0;
    for (int m = 0; m < M; m++) {
        int gv = 0;
        for (int n = 0; n < V; n++) {
            int vis = 1;
            for (int p = 0; p < 6; p++) {
                const REAL* pl = planes + (n * 6 + p) * 4;
                REAL d0 = pl[0] * origin[0 * M + m] + pl[1] * origin[1 * M + m] + pl[2] * origin[2 * M + m] + pl[3];
                REAL de = FABS(pl[0]) * ext[0 * M + m] + FABS(pl[1]) * ext[1 * M + m] + FABS(pl[2]) * ext[2 * M + m];
                vis &= ((d0 + de) >= 0);
            }
            gv |= vis;
        }
        visibility[m] = (uint8_t)gv;
        if (gv) ids[c++] = m;
    }
    *count = c;
}

/* ---- spherical harmonics -------------------------------------------------------------- */
/* constants GR/compact.cu:554-571 ; basis GR/compact.cu:573-653 (== GR/transform.cu:951-1037) */
#ifndef ORC_SH_CONSTS
#define ORC_SH_CONSTS
static const double ORC_SH_C0 = 0.28209479177387814;
static const double ORC_SH_C1 = 0.4886025119029199;
static const double ORC_SH_C2[5] = { 1.0925484305920792, -1.0925484305920792, 0.31539156525252005,
                                     -1.0925484305920792, 0.5462742152960396 };
static const double ORC_SH_C3[7] = { -0.5900435899266435, 2.890611442640554, -0.4570457994644658,
                                     0.3731763325901154, -0.4570457994644658, 1.445305721320277,
                                     -0.5900435899266435 };
#endif

/* basis[0..K) for direction (x,y,z); basis[0] = C0. Order of sh_rest rows follows the reference. */
static inline void SUF(sh_basis)(int deg, REAL x, REAL y, REAL z, REAL* b)
{
    b[0] = (REAL)ORC_SH_C0;
    if (deg > 0) {
        b[1] = -(REAL)ORC_SH_C1 * y;
        b[2] = (REAL)ORC_SH_C1 * z;
        b[3] = -(REAL)ORC_SH_C1 * x;
        if (deg > 1) {
            REAL xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
            b[4] = (REAL)ORC_SH_C2[0] * xy;
            b[5] = (REAL)ORC_SH_C2[1] * yz;
            b[6] = (REAL)ORC_SH_C2[2] * ((REAL)2.0 * zz - xx - yy);
            b[7] = (REAL)ORC_SH_C2[3] * xz;
            b[8] = (REAL)ORC_SH_C2[4] * (xx - yy);
            if (deg > 2) {
                b[9] = (REAL)ORC_SH_C3[0] * y * ((REAL)3.0 * xx - yy);
                b[10] = (REAL)ORC_SH_C3[1] * xy * z;
                b[11] = (REAL)ORC_SH_C3[2] * y * ((REAL)4.0 * zz - xx - yy);
                b[12] = (REAL)ORC_SH_C3[3] * z * ((REAL)2.0 * zz - (REAL)3.0 * xx - (REAL)3.0 * yy);
                b[13] = (REAL)ORC_SH_C3[4] * x * ((REAL)4.0 * zz - xx - yy);
                b[14] = (REAL)ORC_SH_C3[5] * z * (xx - yy);
                b[15] = (REAL)ORC_SH_C3[6] * x * (xx - (REAL)3.0 * yy);
            }
        }
    }
}

/* camera centre = -t . R^T with t = V[3,:3], R = V[:3,:3]  (GR/compact.cu:875-879) */
static inline void SUF(camera_center)(const REAL* Vm, REAL* c)
{
    REAL tx = -Vm[3 * 4 + 0], ty = -Vm[3 * 4 + 1], tz = -Vm[3 * 4 + 2];
    c[0] = tx * Vm[0 * 4 + 0] + ty * Vm[0 * 4 + 1] + tz * Vm[0 * 4 + 2];
    c[1] = tx * Vm[1 * 4 + 0] + ty * Vm[1 * 4 + 1] + tz * Vm[1 * 4 + 2];
    c[2] = tx * Vm[2 * 4 + 0] + ty * Vm[2 * 4 + 1] + tz * Vm[2 * 4 + 2];
}

/* standalone SH->RGB, non-cluster path: GR/transform.cu:951-1037 ; sh [K,3,N], dirs [V,3,N] */
void SUF(orc_sh2rgb_forward)(int deg, const REAL* sh0, const REAL* shr, const REAL* dirs,
                            int V, int N, REAL* rgb)
{
    int K = (deg + 1) * (deg + 1);
#pragma omp parallel for
    for (int i = 0; i < N; i++) {
        for (int v = 0; v < V; v++) {
            REAL b[16];
            SUF(sh_basis)(deg, dirs[(v * 3 + 0) * (size_t)N + i], dirs[(v * 3 + 1) * (size_t)N + i],
                          dirs[(v * 3 + 2) * (size_t)N + i], b);
            for (int c = 0; c < 3; c++) {
                REAL r = b[0] * sh0[c * (size_t)N + i];
                for (int k = 1; k < K; k++) r += b[k] * shr[((k - 1) * 3 + c) * (size_t)N + i];
                rgb[(v * 3 + c) * (size_t)N + i] = r + (REAL)0.5;
            }
        }
    }
}

/* GR/transform.cu:1090-1296 : d sh = basis * d rgb, written for every view in turn (the last view
 * wins in the reference: it assigns, not accumulates); dir gradient is zero (commented out there). */
void SUF(orc_sh2rgb_backward)(int deg, const REAL* rgb_grad, int rest_dim, const REAL* dirs,
                             int V, int N, REAL* sh0_grad, REAL* shr_grad)
{
    int K = (deg + 1) * (deg + 1);
    for (size_t j = 0; j < (size_t)rest_dim * 3 * N; j++) shr_grad[j] = 0;
#pragma omp parallel for
    for (int i = 0; i < N; i++) {
        for (int v = 0; v < V; v++) {
            REAL b[16];
            SUF(sh_basis)(deg, dirs[(v * 3 + 0) * (size_t)N + i], dirs[(v * 3 + 1) * (size_t)N + i],
                          dirs[(v * 3 + 2) * (size_t)N + i], b);
            for (int c = 0; c < 3; c++) {
                REAL g = rgb_grad[(v * 3 + c) * (size_t)N + i];
                sh0_grad[c * (size_t)N + i] = b[0] * g;
                for (int k = 1; k < K; k++) shr_grad[((k - 1) * 3 + c) * (size_t)N + i] = b[k] * g;
            }
        }
    }
}

/* ---- cull + compact + activate (cluster path) ------------------------------------------- */
/* GR/compact.cu:825-893. params [..,C,S]; outputs [..,A,S]; chunks >= nvis only get opacity 0. */
void SUF(orc_cull_compact_activate)(int deg, const int64_t* chunk_ids, int nvis, const REAL* view, int V,
                                   const REAL* pos, const REAL* scale, const REAL* rot, const REAL* sh0,
                                   const REAL* shr, const REAL* opac, int C, int S, int A,
                                   REAL* apos, REAL* ascale, REAL* arot, REAL* color, REAL* aopac)
{
    int K = (deg + 1) * (deg + 1);
    size_t CS = (size_t)C * S, AS = (size_t)A * S;
#pragma omp parallel for
    for (int a = 0; a < A; a++) {
        if (a >= nvis) {
            for (int s = 0; s < S; s++) aopac[(size_t)a * S + s] = 0;
            continue;
        }
        size_t src = (size_t)chunk_ids[a] * S, dst = (size_t)a * S;
        for (int s = 0; s < S; s++) {
            REAL p[3] = { pos[0 * CS + src + s], pos[1 * CS + src + s], pos[2 * CS + src + s] };
            apos[0 * AS + dst + s] = p[0];
            apos[1 * AS + dst + s] = p[1];
            apos[2 * AS + dst + s] = p[2];
            apos[3 * AS + dst + s] = 1;
            for (int k = 0; k < 3; k++) ascale[k * AS + dst + s] = EXP(scale[k * CS + src + s]);
            REAL q[4];
            for (int k = 0; k < 4; k++) q[k] = rot[k * CS + src + s];
            REAL rn = (REAL)1.0 / SQRT(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3] + (REAL)1e-12);
            for (int k = 0; k < 4; k++) arot[k * AS + dst + s] = q[k] * rn;
            aopac[dst + s] = (REAL)1.0 / ((REAL)1.0 + EXP(-opac[src + s]));
            for (int v = 0; v < V; v++) {
                REAL cc[3];
                SUF(camera_center)(view + v * 16, cc);
                REAL d[3] = { p[0] - cc[0], p[1] - cc[1], p[2] - cc[2] };
                REAL dn = (REAL)1.0 / SQRT(d[0] * d[0] + d[1] * d[1] + d[2] * d[2] + (REAL)1e-12);
                REAL b[16];
                SUF(sh_basis)(deg, d[0] * dn, d[1] * dn, d[2] * dn, b);
                for (int c = 0; c < 3; c++) {
                    REAL r = b[0] * sh0[c * CS + src + s];
                    for (int k = 1; k < K; k++) r += b[k] * shr[((size_t)(k - 1) * 3 + c) * CS + src + s];
                    color[((size_t)v * 3 + c) * AS + dst + s] = r + (REAL)0.5;
                }
            }
        }
    }
}

/* GR/compact.cu:895-980.  true_sigmoid=0 reproduces the reference's opacity-logit gradient
 * d o * sigma(x) (GR/compact.cu:952, SURVEY Q15); true_sigmoid=1 is the analytic d o * s(1-s).
 * grads are compacted [..,A,S]; sh_rest rows >= K-1 stay zero. rest_dim = sh_rest.shape[0]. */
void SUF(orc_activate_backward)(int deg, const int64_t* chunk_ids, int nvis, const REAL* view, int V,
                               const REAL* pos, const REAL* scale, const REAL* rot, const REAL* opac,
                               int C, int S, int A, int rest_dim, int true_sigmoid,
                               const REAL* g_apos, const REAL* g_ascale, const REAL* g_arot,
                               const REAL* g_color, const REAL* g_aopac,
                               REAL* g_pos, REAL* g_scale, REAL* g_rot, REAL* g_sh0, REAL* g_shr, REAL* g_opac)
{
    int K = (deg + 1) * (deg + 1);
    size_t CS = (size_t)C * S, AS = (size_t)A * S;
    for (size_t j = 0; j < (size_t)rest_dim * 3 * AS; j++) g_shr[j] = 0;
#pragma omp parallel for
    for (int a = 0; a < nvis; a++) {
        size_t src = (size_t)chunk_ids[a] * S, dst = (size_t)a * S;
        for (int s = 0; s < S; s++) {
            for (int k = 0; k < 3; k++) g_pos[k * AS + dst + s] = g_apos[k * AS + dst + s];
            for (int k = 0; k < 3; k++)
                g_scale[k * AS + dst + s] = EXP(scale[k * CS + src + s]) * g_ascale[k * AS + dst + s];
            REAL q[4], g[4], o[4];
            for (int k = 0; k < 4; k++) { q[k] = rot[k * CS + src + s]; g[k] = g_arot[k * AS + dst + s]; }
            REAL rn = (REAL)1.0 / SQRT(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3] + (REAL)1e-12);
            for (int k = 0; k < 4; k++) o[k] = q[k] * rn;
            REAL dot = g[0] * o[0] + g[1] * o[1] + g[2] * o[2] + g[3] * o[3];
            for (int k = 0; k < 4; k++) g_rot[k * AS + dst + s] = rn * (g[k] - dot * o[k]);
            REAL x = opac[src + s];
            REAL u = (REAL)1.0 / ((REAL)1.0 + EXP(x)), sig = (REAL)1.0 - u;   /* 1 - sig = u, not formed from the rounded sig */
            REAL fac = true_sigmoid ? sig * u : sig;
            g_opac[dst + s] = g_aopac[dst + s] * fac;
            REAL p[3] = { pos[0 * CS + src + s], pos[1 * CS + src + s], pos[2 * CS + src + s] };
            for (int v = 0; v < V; v++) {
                REAL cc[3];
                SUF(camera_center)(view + v * 16, cc);
                REAL d[3] = { p[0] - cc[0], p[1] - cc[1], p[2] - cc[2] };
                REAL dn = (REAL)1.0 / SQRT(d[0] * d[0] + d[1] * d[1] + d[2] * d[2] + (REAL)1e-12);
                REAL b[16];
                SUF(sh_basis)(deg, d[0] * dn, d[1] * dn, d[2] * dn, b);
                for (int c = 0; c < 3; c++) {
                    REAL gc = g_color[((size_t)v * 3 + c) * AS + dst + s];
                    if (v == 0) g_sh0[c * AS + dst + s] = b[0] * gc;
                    else g_sh0[c * AS + dst + s] += b[0] * gc;
                    for (int k = 1; k < K; k++) {
                        size_t o_ = ((size_t)(k - 1) * 3 + c) * AS + dst + s;
                        if (v == 0) g_shr[o_] = b[k] * gc; else g_shr[o_] += b[k] * gc;
                    }
                }
            }
        }
    }
}

/* ---- per-Gaussian projection ops -------------------------------------------------------- */

/* GR/transform.cu:378-438.  pos [4,N] -> view,ndc [V,4,N]. Entries >= valid are left untouched. */
void SUF(orc_mvp_forward)(const REAL* pos, const REAL* view, const REAL* proj, int V, int N, int valid,
                         REAL* vpos, REAL* ndc)
{
#pragma omp parallel for
    for (int i = 0; i < valid; i++) {
        for (int b = 0; b < V; b++) {
            const REAL* Vm = view + b * 16; const REAL* P = proj + b * 16;
            REAL w[4], v[4], h[4];
            for (int k = 0; k < 4; k++) w[k] = pos[(size_t)k * N + i];
            for (int k = 0; k < 4; k++)
                v[k] = w[0] * Vm[0 * 4 + k] + w[1] * Vm[1 * 4 + k] + w[2] * Vm[2 * 4 + k] + w[3] * Vm[3 * 4 + k];
            for (int k = 0; k < 4; k++)
                h[k] = v[0] * P[0 * 4 + k] + v[1] * P[1 * 4 + k] + v[2] * P[2 * 4 + k] + v[3] * P[3 * 4 + k];
            REAL iw = (FABS(h[3]) > (REAL)1e-12) ? ((REAL)1.0 / h[3]) : (REAL)0.0;
            for (int k = 0; k < 4; k++) vpos[((size_t)b * 4 + k) * N + i] = v[k];
            ndc[((size_t)b * 4 + 0) * N + i] = h[0] * iw;
            ndc[((size_t)b * 4 + 1) * N + i] = h[1] * iw;
            ndc[((size_t)b * 4 + 2) * N + i] = h[2] * iw;
            ndc[((size_t)b * 4 + 3) * N + i] = 1;
        }
    }
}

/* GR/transform.cu:472-560 : d pos [4,N], summed over views. */
void SUF(orc_mvp_backward)(const REAL* g_ndc, const REAL* g_view, const REAL* view, const REAL* proj,
                          const REAL* vpos, int V, int N, int valid, REAL* g_pos)
{
#pragma omp parallel for
    for (int i = 0; i < valid; i++) {
        REAL acc[4] = { 0, 0, 0, 0 };
        for (int b = 0; b < V; b++) {
            const REAL* Vm = view + b * 16; const REAL* P = proj + b * 16;
            REAL v[4], h[4], gn[4], dh[4], dv[4];
            for (int k = 0; k < 4; k++) v[k] = vpos[((size_t)b * 4 + k) * N + i];
            for (int k = 0; k < 4; k++)
                h[k] = v[0] * P[0 * 4 + k] + v[1] * P[1 * 4 + k] + v[2] * P[2 * 4 + k] + v[3] * P[3 * 4 + k];
            REAL iw = (FABS(h[3]) > (REAL)1e-12) ? ((REAL)1.0 / h[3]) : (REAL)0.0;
            REAL n0 = h[0] * iw, n1 = h[1] * iw, n2 = h[2] * iw;
            for (int k = 0; k < 4; k++) gn[k] = g_ndc[((size_t)b * 4 + k) * N + i];
            dh[0] = gn[0] * iw; dh[1] = gn[1] * iw; dh[2] = gn[2] * iw;
            dh[3] = -(gn[0] * n0 + gn[1] * n1 + gn[2] * n2) * iw;
            for (int k = 0; k < 4; k++)
                dv[k] = dh[0] * P[k * 4 + 0] + dh[1] * P[k * 4 + 1] + dh[2] * P[k * 4 + 2] + dh[3] * P[k * 4 + 3]
                      + g_view[((size_t)b * 4 + k) * N + i];
            for (int k = 0; k < 4; k++)
                acc[k] += dv[0] * Vm[k * 4 + 0] + dv[1] * Vm[k * 4 + 1] + dv[2] * Vm[k * 4 + 2] + dv[3] * Vm[k * 4 + 3];
        }
        for (int k = 0; k < 4; k++) g_pos[(size_t)k * N + i] = acc[k];
    }
}

/* rotation matrix of unit quaternion (r,x,y,z), GR/transform.cu:115-125 */
static inline void SUF(quat_R)(REAL r, REAL x, REAL y, REAL z, REAL R[9])
{
    R[0] = 1 - 2 * (y * y + z * z); R[1] = 2 * (x * y + r * z);     R[2] = 2 * (x * z - r * y);
    R[3] = 2 * (x * y - r * z);     R[4] = 1 - 2 * (x * x + z * z); R[5] = 2 * (y * z + r * x);
    R[6] = 2 * (x * z + r * y);     R[7] = 2 * (y * z - r * x);     R[8] = 1 - 2 * (x * x + y * y);
}

/* GR/transform.cu:92-127 : T[a][b] = s_a R[a][b], [3,3,N] */
void SUF(orc_transform_forward)(const REAL* quat, const REAL* scale, int N, int valid, REAL* T)
{
#pragma omp parallel for
    for (int i = 0; i < valid; i++) {
        REAL R[9];
        SUF(quat_R)(quat[0 * (size_t)N + i], quat[1 * (size_t)N + i], quat[2 * (size_t)N + i], quat[3 * (size_t)N + i], R);
        for (int a = 0; a < 3; a++)
            for (int b = 0; b < 3; b++) T[((size_t)a * 3 + b) * N + i] = R[a * 3 + b] * scale[(size_t)a * N + i];
    }
}

/* GR/transform.cu:151-228 */
void SUF(orc_transform_backward)(const REAL* gT, const REAL* quat, const REAL* scale, int N, int valid,
                                REAL* g_quat, REAL* g_scale)
{
#pragma omp parallel for
    for (int i = 0; i < valid; i++) {
        REAL r = quat[0 * (size_t)N + i], x = quat[1 * (size_t)N + i], y = quat[2 * (size_t)N + i], z = quat[3 * (size_t)N + i];
        REAL R[9], dt[9];
        SUF(quat_R)(r, x, y, z, R);
        for (int k = 0; k < 9; k++) dt[k] = gT[(size_t)k * N + i];
        for (int a = 0; a < 3; a++)
            g_scale[(size_t)a * N + i] = R[a * 3 + 0] * dt[a * 3 + 0] + R[a * 3 + 1] * dt[a * 3 + 1] + R[a * 3 + 2] * dt[a * 3 + 2];
        for (int a = 0; a < 3; a++)
            for (int b = 0; b < 3; b++) dt[a * 3 + b] *= scale[(size_t)a * N + i];
        g_quat[0 * (size_t)N + i] = 2 * z * (dt[1] - dt[3]) + 2 * y * (dt[6] - dt[2]) + 2 * x * (dt[5] - dt[7]);
        g_quat[1 * (size_t)N + i] = 2 * y * (dt[3] + dt[1]) + 2 * z * (dt[6] + dt[2]) + 2 * r * (dt[5] - dt[7]) - 4 * x * (dt[8] + dt[4]);
        g_quat[2 * (size_t)N + i] = 2 * x * (dt[3] + dt[1]) + 2 * r * (dt[6] - dt[2]) + 2 * z * (dt[5] + dt[7]) - 4 * y * (dt[8] + dt[0]);
        g_quat[3 * (size_t)N + i] = 2 * r * (dt[1] - dt[3]) + 2 * x * (dt[6] + dt[2]) + 2 * y * (dt[5] + dt[7]) - 4 * z * (dt[4] + dt[0]);
    }
}

/* GR/transform.cu:22-52 : J [V,3,3,N], zero except (0,0),(1,1),(2,0),(2,1). */
void SUF(orc_jacobian_rayspace)(const REAL* vpos, const REAL* proj, int V, int N, int valid, int H, int W, REAL* J)
{
    for (size_t j = 0; j < (size_t)V * 9 * N; j++) J[j] = 0;
#pragma omp parallel for
    for (int i = 0; i < valid; i++) {
        for (int b = 0; b < V; b++) {
            REAL p00 = proj[b * 16 + 0], p11 = proj[b * 16 + 5];
            REAL fx = p00 * W * (REAL)0.5, fy = p11 * H * (REAL)0.5;
            REAL tx = vpos[((size_t)b * 4 + 0) * N + i], ty = vpos[((size_t)b * 4 + 1) * N + i], tz = vpos[((size_t)b * 4 + 2) * N + i];
            REAL lx = tz / p00 * (REAL)1.3, ly = tz / p11 * (REAL)1.3;
            tx = FMAX(FMIN(tx, lx), -lx);
            ty = FMAX(FMIN(ty, ly), -ly);
            REAL rz = (REAL)1.0 / FMAX(tz, (REAL)1e-2);
            REAL rz2 = rz * rz;
            J[(((size_t)b * 3 + 0) * 3 + 0) * N + i] = fx * rz;
            J[(((size_t)b * 3 + 1) * 3 + 1) * N + i] = fy * rz;
            J[(((size_t)b * 3 + 2) * 3 + 0) * N + i] = -fx * tx * rz2;
            J[(((size_t)b * 3 + 2) * 3 + 1) * N + i] = -fy * ty * rz2;
        }
    }
}

/* M = T . V3x3 . J3x2 (GR/transform.cu:761-769) */
static inline void SUF(cov_M)(const REAL* T, int N, int i, const REAL* Vm, const REAL* Jb, REAL VJ[6], REAL M[6])
{
    REAL Jl[6];
    for (int a = 0; a < 3; a++) for (int c = 0; c < 2; c++) Jl[a * 2 + c] = Jb[((size_t)a * 3 + c) * N + i];
    for (int a = 0; a < 3; a++) for (int c = 0; c < 2; c++) {
        REAL t = 0;
        for (int k = 0; k < 3; k++) t += Vm[a * 4 + k] * Jl[k * 2 + c];
        VJ[a * 2 + c] = t;
    }
    for (int a = 0; a < 3; a++) for (int c = 0; c < 2; c++) {
        REAL t = 0;
        for (int k = 0; k < 3; k++) t += T[((size_t)a * 3 + k) * N + i] * VJ[k * 2 + c];
        M[a * 2 + c] = t;
    }
}

/* GR/transform.cu:736-780 : cov2d = M^T M + 0.3 I, [V,2,2,N] */
void SUF(orc_cov2d_forward)(const REAL* J, const REAL* view, const REAL* T, int V, int N, int valid, REAL* cov)
{
#pragma omp parallel for
    for (int i = 0; i < valid; i++) {
        for (int b = 0; b < V; b++) {
            REAL VJ[6], M[6];
            SUF(cov_M)(T, N, i, view + b * 16, J + (size_t)b * 9 * N, VJ, M);
            for (int p = 0; p < 2; p++) for (int q = 0; q < 2; q++) {
                REAL t = 0;
                for (int k = 0; k < 3; k++) t += M[k * 2 + p] * M[k * 2 + q];
                if (p == q) t += (REAL)0.3;
                cov[(((size_t)b * 2 + p) * 2 + q) * N + i] = t;
            }
        }
    }
}

/* GR/transform.cu:823-890 : dT = 2 M dCov (VJ)^T summed over views ; [3,3,N] (entries >= valid: 0) */
void SUF(orc_cov2d_backward)(const REAL* g_cov, const REAL* J, const REAL* view, const REAL* T,
                            int V, int N, int valid, REAL* gT)
{
#pragma omp parallel for
    for (int i = 0; i < N; i++) {
        REAL acc[9] = { 0 };
        if (i < valid) {
            for (int b = 0; b < V; b++) {
                REAL VJ[6], M[6], G[4], dM[6];
                SUF(cov_M)(T, N, i, view + b * 16, J + (size_t)b * 9 * N, VJ, M);
                for (int k = 0; k < 4; k++) G[k] = g_cov[((size_t)b * 4 + k) * N + i];
                for (int a = 0; a < 3; a++) for (int c = 0; c < 2; c++)
                    dM[a * 2 + c] = 2 * (M[a * 2 + 0] * G[0 * 2 + c] + M[a * 2 + 1] * G[1 * 2 + c]);
                for (int a = 0; a < 3; a++) for (int k = 0; k < 3; k++)
                    acc[a * 3 + k] += dM[a * 2 + 0] * VJ[k * 2 + 0] + dM[a * 2 + 1] * VJ[k * 2 + 1];
            }
        }
        for (int k = 0; k < 9; k++) gT[(size_t)k * N + i] = acc[k];
    }
}

/* GR/transform.cu:1364-1421 : eigenvalues, eigenvectors and guarded inverse of a 2x2. */
void SUF(orc_eigh_inv_forward)(const REAL* in, int V, int N, int valid, REAL* val, REAL* vec, REAL* inv)
{
#pragma omp parallel for
    for (int i = 0; i < valid; i++) {
        for (int b = 0; b < V; b++) {
            size_t o = (size_t)b * 4 * N + i;
            REAL m00 = in[o + 0 * (size_t)N], m01 = in[o + 1 * (size_t)N], m10 = in[o + 2 * (size_t)N], m11 = in[o + 3 * (size_t)N];
            REAL det = m00 * m11 - m01 * m10;
            REAL det1 = (m00 - m01) * (m11 - m01) + m01 * (m00 + m11 - 2 * m01);
            det = (FABS(det) < FABS((REAL)1e-5 * m01 * m10)) ? det1 : det;
            REAL t0 = m00 + m11;
            REAL t1 = SQRT((m00 - m11) * (m00 - m11) + 4 * m01 * m01);
            t1 = FMAX(t1, (REAL)1e-9);
            REAL e0 = (REAL)0.5 * (t0 - t1), e1 = (REAL)0.5 * (t0 + t1);
            val[((size_t)b * 2 + 0) * N + i] = e0;
            val[((size_t)b * 2 + 1) * N + i] = e1;
            REAL v0[2], v1[2];
            if (FABS(e0 - m00) > FABS(e0 - m11)) {
                v0[0] = -m01; v0[1] = m00 - e0; v1[0] = e1 - m11; v1[1] = m01;
            } else {
                v0[0] = m11 - e0; v0[1] = -m01; v1[0] = m01; v1[1] = e1 - m00;
            }
            REAL l0 = (REAL)1.0 / SQRT(v0[0] * v0[0] + v0[1] * v0[1]);
            REAL l1 = (REAL)1.0 / SQRT(v1[0] * v1[0] + v1[1] * v1[1]);
            vec[o + 0 * (size_t)N] = v0[0] * l0; vec[o + 1 * (size_t)N] = v1[0] * l1;
            vec[o + 2 * (size_t)N] = v0[1] * l0; vec[o + 3 * (size_t)N] = v1[1] * l1;
            det = (FABS(det) < (REAL)1e-9) ? (REAL)1e-9 : det;
            REAL dr = 1 / det;
            inv[o + 1 * (size_t)N] = -m01 * dr;
            inv[o + 2 * (size_t)N] = -m10 * dr;
            inv[o + 0 * (size_t)N] = m11 * dr;
            inv[o + 3 * (size_t)N] = m00 * dr;
        }
    }
}

/* GR/transform.cu:1424-1454 : dM = -(inv . dInv . inv) */
void SUF(orc_inv2x2_backward)(const REAL* inv, const REAL* g_inv, int V, int N, int valid, REAL* g_in)
{
#pragma omp parallel for
    for (int i = 0; i < valid; i++) {
        for (int b = 0; b < V; b++) {
            size_t o = (size_t)b * 4 * N + i;
            REAL A[4], G[4], t[4], r[4];
            for (int k = 0; k < 4; k++) { A[k] = inv[o + k * (size_t)N]; G[k] = g_inv[o + k * (size_t)N]; }
            for (int p = 0; p < 2; p++) for (int q = 0; q < 2; q++) t[p * 2 + q] = A[p * 2 + 0] * G[0 * 2 + q] + A[p * 2 + 1] * G[1 * 2 + q];
            for (int p = 0; p < 2; p++) for (int q = 0; q < 2; q++) r[p * 2 + q] = t[p * 2 + 0] * A[0 * 2 + q] + t[p * 2 + 1] * A[1 * 2 + q];
            for (int k = 0; k < 4; k++) g_in[o + k * (size_t)N] = -r[k];
        }
    }
}

/* ---- binning -------------------------------------------------------------------------- */

/* GR/speedy_splat.cuh:16-31.  The two quotients by A (or C) are taken as products with the once-rounded reciprocal
 * inv_A = 1/A (inv_C = 1/C) of the splat: the reference's own build does the same (--use_fast_math turns x/c into
 * x * rcp(c), GR/setup.py:35), and one division per splat and axis replaces two per tile row.  The CUDA kernels
 * (csrc/splat_geom.cuh) use the identical operation sequence, so tile decisions stay bit-identical CPU <-> GPU. */
static inline void SUF(ellipse_isect)(REAL A, REAL B, REAL Cc, REAL inv_A, REAL inv_C, REAL disc, REAL t, REAL px, REAL py,
                                      int isY, REAL coord, REAL* lo, REAL* hi)
{
    REAL p_u = isY ? py : px;
    REAL p_v = isY ? px : py;
    REAL coeff = isY ? A : Cc;
    REAL inv = isY ? inv_A : inv_C;
    REAL h = coord - p_u;
    REAL sq = SQRT(disc * h * h + t * coeff);
    *lo = (-B * h - sq) * inv + p_v;
    *hi = (-B * h + sq) * inv + p_v;
}

typedef struct {
    REAL A, B, C, inv_A, inv_C, disc, t, px, py;
    REAL bbox_min[2], bbox_max[2], argmin[2], argmax[2];
    int rect_min[2], rect_max[2];
    int visible;
} SUF(splat_geom);

/* visibility + bounding box + tile rectangle: GR/binning.cu:309-355 (== :46-89).
 * 2*log(255 o) is evaluated in double and rounded to REAL so that the CPU and GPU (which does the
 * same) make bit-identical tile decisions; the reference's own value comes from fast-math __logf.
 * exact_bound=1: the rectangle ends after the tile holding bbox_max, floor((bbox_max + T) / T);
 * 0: the reference's floor((bbox_max + T - 1) / T), which drops tile k when the ellipse reaches
 * pixel centre kT with bbox_max < kT + 1 (DESIGN.md section 7, D14). */
static inline void SUF(splat_setup)(REAL ndcx, REAL ndcy, REAL viewz, REAL A, REAL B, REAL Cc, REAL o,
                                    int H, int W, int TH, int TW, int gx, int gy, int exact_bound, SUF(splat_geom)* g)
{
    g->A = A; g->B = B; g->C = Cc;
    g->disc = B * B - A * Cc;
    g->px = (ndcx * (REAL)0.5 + (REAL)0.5) * W - (REAL)0.5;
    g->py = (ndcy * (REAL)0.5 + (REAL)0.5) * H - (REAL)0.5;
    int vis = !((ndcx < (REAL)-1.3) || (ndcx > (REAL)1.3) || (ndcy < (REAL)-1.3) || (ndcy > (REAL)1.3) ||
                (viewz <= (REAL)0.2) || (o < (REAL)1.0 / 255));
    vis &= ((A > 0) & (Cc > 0) & (g->disc < 0));
    g->visible = vis;
    if (!vis) return;
    REAL t = (REAL)(2.0 * log((double)(o * (REAL)255.0)));
    g->t = t;
    g->inv_A = (REAL)1 / A; g->inv_C = (REAL)1 / Cc;
    REAL xt = SQRT(-(B * B * t) / (g->disc * A));
    xt = (B < 0) ? xt : -xt;
    REAL yt = SQRT(-(B * B * t) / (g->disc * Cc));
    yt = (B < 0) ? yt : -yt;
    g->argmin[0] = g->py - yt; g->argmin[1] = g->px - xt;
    g->argmax[0] = g->py + yt; g->argmax[1] = g->px + xt;
    REAL lo, hi;
    SUF(ellipse_isect)(A, B, Cc, g->inv_A, g->inv_C, g->disc, t, g->px, g->py, 1, g->argmin[0], &lo, &hi); g->bbox_min[0] = lo;
    SUF(ellipse_isect)(A, B, Cc, g->inv_A, g->inv_C, g->disc, t, g->px, g->py, 0, g->argmin[1], &lo, &hi); g->bbox_min[1] = lo;
    SUF(ellipse_isect)(A, B, Cc, g->inv_A, g->inv_C, g->disc, t, g->px, g->py, 1, g->argmax[0], &lo, &hi); g->bbox_max[0] = hi;
    SUF(ellipse_isect)(A, B, Cc, g->inv_A, g->inv_C, g->disc, t, g->px, g->py, 0, g->argmax[1], &lo, &hi); g->bbox_max[1] = hi;
    g->rect_min[0] = SUF(imax)(0, SUF(imin)(gx, SUF(f2i_rz)(g->bbox_min[0] / TW)));
    g->rect_min[1] = SUF(imax)(0, SUF(imin)(gy, SUF(f2i_rz)(g->bbox_min[1] / TH)));
    REAL ex = g->bbox_max[0] + TW, ey = g->bbox_max[1] + TH;
    if (!exact_bound) { ex = ex - 1; ey = ey - 1; }
    g->rect_max[0] = SUF(imax)(0, SUF(imin)(gx, SUF(f2i_rz)(ex / TW)));
    g->rect_max[1] = SUF(imax)(0, SUF(imin)(gy, SUF(f2i_rz)(ey / TH)));
}

/* Attribution: the overlap walk restated below is speedy-splat's "AccuTile" procedure (https://github.com/j-alex-hanson/
 * speedy-splat, based on Inria/MPII "gaussian-splatting", Gaussian-Splatting License, non-commercial research and evaluation
 * use; notice carried over from GR/speedy_splat.cuh:1-13, see NOTICE.md). */
/* GR/speedy_splat.cuh:33-149 ; returns the tile count, optionally emits (tile+1, idx) at keys/vals[off..] */
static inline int SUF(process_tiles)(const SUF(splat_geom)* g, int TH, int TW, int gx,
                                     int32_t idx, int off, int cap, int32_t* keys, int32_t* vals)
{
    int y_span = g->rect_max[1] - g->rect_min[1], x_span = g->rect_max[0] - g->rect_min[0];
    if (y_span * x_span <= 0) return 0;
    int isY = y_span < x_span;
    REAL BU = isY ? TH : TW, BV = isY ? TW : TH;
    int rmin[2] = { g->rect_min[0], g->rect_min[1] }, rmax[2] = { g->rect_max[0], g->rect_max[1] };
    REAL bmin[2] = { g->bbox_min[0], g->bbox_min[1] }, bmax[2] = { g->bbox_max[0], g->bbox_max[1] };
    REAL amin[2] = { g->argmin[0], g->argmin[1] }, amax[2] = { g->argmax[0], g->argmax[1] };
    if (isY) {
        int ti; REAL tr;
        ti = rmin[0]; rmin[0] = rmin[1]; rmin[1] = ti;
        ti = rmax[0]; rmax[0] = rmax[1]; rmax[1] = ti;
        tr = bmin[0]; bmin[0] = bmin[1]; bmin[1] = tr;
        tr = bmax[0]; bmax[0] = bmax[1]; bmax[1] = tr;
        tr = amin[0]; amin[0] = amin[1]; amin[1] = tr;
        tr = amax[0]; amax[0] = amax[1]; amax[1] = tr;
    }
    int count = 0;
    REAL imax_lo = bmax[1], imax_hi = bmin[1];   /* intersect_max_line = {bbox_max.y, bbox_min.y} */
    REAL imin_lo, imin_hi;
    REAL min_line = rmin[0] * BU, max_line;
    if (bmin[0] <= min_line)
        SUF(ellipse_isect)(g->A, g->B, g->C, g->inv_A, g->inv_C, g->disc, g->t, g->px, g->py, isY, rmin[0] * BU, &imin_lo, &imin_hi);
    else { imin_lo = imax_lo; imin_hi = imax_hi; }
    for (int u = rmin[0]; u < rmax[0]; ++u) {
        max_line = min_line + BU;
        if (max_line <= bmax[0])
            SUF(ellipse_isect)(g->A, g->B, g->C, g->inv_A, g->inv_C, g->disc, g->t, g->px, g->py, isY, max_line, &imax_lo, &imax_hi);
        REAL emin, emax;
        if (min_line <= amin[1] && amin[1] < max_line) emin = bmin[1];
        else emin = FMIN(imin_lo, imax_lo);
        if (min_line <= amax[1] && amax[1] < max_line) emax = bmax[1];
        else emax = FMAX(imin_hi, imax_hi);
        int min_v = SUF(imax)(rmin[1], SUF(imin)(rmax[1], SUF(f2i_rz)(emin / BV)));
        int max_v = SUF(imin)(rmax[1], SUF(imax)(rmin[1], SUF(f2i_rz)(emax / BV + 1)));
        count += max_v - min_v;
        if (keys) {
            for (int v = min_v; v < max_v; v++) {
                int key = isY ? (u * gx + v) : (v * gx + u);
                if (off < cap) { keys[off] = key + 1; vals[off] = idx; }
                off++;
            }
        }
        imin_lo = imax_lo; imin_hi = imax_hi;
        min_line = max_line;
    }
    return count;
}

/* GR/binning.cu:289-385 : per-splat pixel bbox + tile count.  [V,*,N]; entries >= valid untouched
 * (the caller pre-zeroes `alloc`, as the reference does with torch::zeros). */
void SUF(orc_get_allocate_size)(const REAL* ndc, const REAL* viewz, const REAL* inv_cov, const REAL* opac,
                               int V, int N, int valid, int H, int W, int TH, int TW, int exact_bound,
                               int32_t* left_up, int32_t* right_down, int32_t* alloc)
{
    int gx = (W + TW - 1) / TW, gy = (H + TH - 1) / TH;
#pragma omp parallel for
    for (int i = 0; i < valid; i++) {
        for (int b = 0; b < V; b++) {
            SUF(splat_geom) g;
            size_t o4 = (size_t)b * 4 * N + i;
            SUF(splat_setup)(ndc[o4], ndc[o4 + N], viewz[(size_t)b * N + i], inv_cov[o4], inv_cov[o4 + N],
                             inv_cov[o4 + 3 * (size_t)N], opac[i], H, W, TH, TW, gx, gy, exact_bound, &g);
            size_t o2 = (size_t)b * 2 * N + i;
            if (g.visible) {
                left_up[o2] = SUF(f2i_rz)(CEIL(g.bbox_min[0])); left_up[o2 + N] = SUF(f2i_rz)(CEIL(g.bbox_min[1]));
                right_down[o2] = SUF(f2i_rz)(FLOOR(g.bbox_max[0])); right_down[o2 + N] = SUF(f2i_rz)(FLOOR(g.bbox_max[1]));
                alloc[(size_t)b * N + i] = SUF(process_tiles)(&g, TH, TW, gx, i, 0, 0, NULL, NULL);
            } else {
                left_up[o2] = -1; left_up[o2 + N] = -1; right_down[o2] = -1; right_down[o2 + N] = -1;
                alloc[(size_t)b * N + i] = 0;
            }
        }
    }
}

/* GR/binning.cu:33-110 + :199-221 : emit (tile+1, splat) pairs in depth order at `offset`
 * (inclusive scan of the depth-ordered counts), then a STABLE sort on the tile key.  Slots that are
 * never written keep key 0 and sort to the front (SURVEY Q2).  keys_out/vals_out [V,cap]. */
void SUF(orc_create_table)(const REAL* ndc, const REAL* inv_cov, const REAL* opac, const int32_t* offset,
                          const int64_t* sorted_id, int V, int N, int cap, int H, int W, int TH, int TW,
                          int exact_bound, int32_t* keys_out, int32_t* vals_out)
{
    int gx = (W + TW - 1) / TW, gy = (H + TH - 1) / TH;
    int ntile = gx * gy + 1;
    int32_t* keys = (int32_t*)calloc((size_t)cap, sizeof(int32_t));
    int32_t* vals = (int32_t*)calloc((size_t)cap, sizeof(int32_t));
    int* hist = (int*)malloc(sizeof(int) * (size_t)(ntile + 1));
    for (int b = 0; b < V; b++) {
        memset(keys, 0, sizeof(int32_t) * (size_t)cap);
        memset(vals, 0, sizeof(int32_t) * (size_t)cap);
#pragma omp parallel for
        for (int j = 0; j < N; j++) {
            int off = j == 0 ? 0 : offset[(size_t)b * N + j - 1];
            int asz = offset[(size_t)b * N + j] - off;
            int i = (int)sorted_id[(size_t)b * N + j];
            if (asz > 0 && off + asz <= cap) {
                SUF(splat_geom) g;
                size_t o4 = (size_t)b * 4 * N + i;
                /* the emit kernel skips the visibility test: it trusts asz>0 (GR/binning.cu:63) */
                SUF(splat_setup)(ndc[o4], ndc[o4 + N], (REAL)1.0, inv_cov[o4], inv_cov[o4 + N],
                                 inv_cov[o4 + 3 * (size_t)N], opac[i], H, W, TH, TW, gx, gy, exact_bound, &g);
                if (g.visible) SUF(process_tiles)(&g, TH, TW, gx, i, off, cap, keys, vals);
            }
        }
        /* stable counting sort by key */
        memset(hist, 0, sizeof(int) * (size_t)(ntile + 1));
        for (int j = 0; j < cap; j++) hist[keys[j] + 1]++;
        for (int t = 0; t < ntile; t++) hist[t + 1] += hist[t];
        for (int j = 0; j < cap; j++) {
            int p = hist[keys[j]]++;
            keys_out[(size_t)b * cap + p] = keys[j];
            vals_out[(size_t)b * cap + p] = vals[j];
        }
    }
    free(keys); free(vals); free(hist);
}

/* GR/binning.cu:228-287 : range[t] = first index of key t, -1 when absent; range[t+1] doubles as the
 * end marker.  fix_last=1 additionally closes the last populated tile (the reference leaves it -1 so
 * that tile renders empty -- SURVEY Q3); fix_last=0 reproduces the reference bit for bit. */
void SUF(orc_tile_range)(const int32_t* keys, int V, int L, int max_tile, int fix_last, int32_t* range)
{
    for (int b = 0; b < V; b++) {
        int32_t* r = range + (size_t)b * (max_tile + 2);
        const int32_t* k = keys + (size_t)b * L;
        for (int t = 0; t < max_tile + 2; t++) r[t] = -1;
        if (L <= 0) continue;
        r[k[0]] = 0;
        r[max_tile + 1] = L;
        for (int j = 0; j < L - 1; j++) {
            int cur = k[j], nxt = k[j + 1];
            if (cur != nxt) {
                if (cur + 1 < nxt) r[cur + 1] = j + 1;
                r[nxt] = j + 1;
            }
        }
        if (fix_last && k[L - 1] + 1 <= max_tile + 1) r[k[L - 1] + 1] = L;
    }
}

/* ---- rasterisation ---------------------------------------------------------------------- */

/* GR/raster.cu:334-356 but WITHOUT the half quantisation: rec = {px,py,A,B,C,o,r,g,b} per splat. */
typedef struct { REAL px, py, A, B, C, o, r, g, b; } SUF(splat_rec);

static inline SUF(splat_rec) SUF(load_rec)(const REAL* ndc, const REAL* inv_cov, const REAL* color,
                                            const REAL* opac, int b, int N, int i, int H, int W)
{
    SUF(splat_rec) s;
    size_t o4 = (size_t)b * 4 * N + i, o3 = (size_t)b * 3 * N + i;
    s.px = (ndc[o4] + (REAL)1.0) * (REAL)0.5 * W - (REAL)0.5;
    s.py = (ndc[o4 + N] + (REAL)1.0) * (REAL)0.5 * H - (REAL)0.5;
    s.A = inv_cov[o4]; s.B = inv_cov[o4 + N]; s.C = inv_cov[o4 + 3 * (size_t)N];
    s.o = opac[i];
    s.r = color[o3]; s.g = color[o3 + N]; s.b = color[o3 + 2 * (size_t)N];
    return s;
}

/* GR/raster.cu:161-332 (thresholds :260-270, outputs :306-330).  Images are padded to whole tiles:
 * img [V,3,Hp,Wp], T [V,1,Hp,Wp], last [V,1,Hp,Wp] int16.  Optional stats: frag_count/frag_weight
 * [V,1,N] (GR/raster.cu:273-301).  fragile (optional, [V,Hp,Wp] u8) marks pixels that came within
 * `eps` of a step-function threshold (SURVEY Appendix B) so that tests can mask them. */
void SUF(orc_raster_forward)(const int32_t* sorted, const int32_t* range, const REAL* ndc, const REAL* inv_cov,
                            const REAL* color, const REAL* opac, const int32_t* tiles, int ntiles_sel,
                            int V, int N, int cap, int H, int W, int TH, int TW,
                            REAL* img, REAL* Tout, int16_t* last, int32_t* frag_count, REAL* frag_weight,
                            uint8_t* fragile, REAL eps)
{
    int gx = (W + TW - 1) / TW, gy = (H + TH - 1) / TH;
    int Hp = gy * TH, Wp = gx * TW, ntile = gx * gy;
    int nrender = tiles ? ntiles_sel : ntile;
    for (int b = 0; b < V; b++) {
        const int32_t* rg = range + (size_t)b * (ntile + 2);
#pragma omp parallel for schedule(dynamic, 4)
        for (int ti = 0; ti < nrender; ti++) {
            int tid = tiles ? tiles[(size_t)b * ntiles_sel + ti] : ti + 1;
            if (tid == 0 || tid >= ntile + 1) continue;
            int start = rg[tid], end = rg[tid + 1];
            int tx = (tid - 1) % gx, ty = (tid - 1) / gx;
            for (int py = 0; py < TH; py++) for (int px = 0; px < TW; px++) {
                int x = tx * TW + px, y = ty * TH + py;
                REAL T = 1, C0 = 0, C1 = 0, C2 = 0; int n = 0; int frag = 0;
                if (start != -1) {
                    for (int k = start; k < end; k++) {
                        if (!(T > (REAL)1.0 / 8192)) break;
                        if (FABS(T - (REAL)1.0 / 8192) < eps * (REAL)1e-3) frag = 1;
                        n++;
                        int i = sorted[(size_t)b * cap + k];
                        SUF(splat_rec) s = SUF(load_rec)(ndc, inv_cov, color, opac, b, N, i, H, W);
                        REAL dx = s.px - x, dy = s.py - y;
                        REAL pw = (REAL)-0.5 * (s.A * dx * dx + 2 * s.B * dx * dy + s.C * dy * dy);
                        REAL a = s.o * EXP(pw);
                        if (FABS(a - (REAL)1.0 / 256) < eps) frag = 1;
                        if (a < (REAL)1.0 / 256) continue;
                        a = FMIN(a, (REAL)255.0 / 256);
                        REAL w = a * T;
                        C0 += s.r * w; C1 += s.g * w; C2 += s.b * w;
                        if (frag_count) {
#pragma omp atomic
                            frag_count[(size_t)b * N + i] += 1;
#pragma omp atomic
                            frag_weight[(size_t)b * N + i] += w;
                        }
                        T = T * (1 - a);
                    }
                    if (FABS(T - (REAL)1.0 / 8192) < eps * (REAL)1e-3) frag = 1;
                }
                size_t po = (size_t)y * Wp + x, plane = (size_t)Hp * Wp;
                img[((size_t)b * 3 + 0) * plane + po] = FMIN(C0, (REAL)1.0);
                img[((size_t)b * 3 + 1) * plane + po] = FMIN(C1, (REAL)1.0);
                img[((size_t)b * 3 + 2) * plane + po] = FMIN(C2, (REAL)1.0);
                Tout[(size_t)b * plane + po] = T;
                last[(size_t)b * plane + po] = (int16_t)(uint16_t)(n > 65535 ? 65535 : n);   /* 16-bit count, read back unsigned (GR/raster.cu:683-686) */
                if (fragile) fragile[(size_t)b * plane + po] = (uint8_t)frag;
            }
        }
    }
}

/* GR/raster.cu:599-853 + unpack_gradient :855-886.  d_img [V,3,Hp,Wp] is the (already max-normalised)
 * image gradient, `scaler` the de-normaliser (wrapper.py:490-494).  Outputs: d_ndc [V,4,N],
 * d_inv_cov [V,2,2,N], d_color [V,3,N], d_opac [1,N] (view 0 only, GR/raster.cu:881-884),
 * err_sq [V,1,N] when stats are requested (sum over pixels of (running d_opacity)^2, :779-784). */
void SUF(orc_raster_backward)(const int32_t* sorted, const int32_t* range, const REAL* ndc, const REAL* inv_cov,
                             const REAL* color, const REAL* opac, const int32_t* tiles, int ntiles_sel,
                             const REAL* Tfinal, const int16_t* last, const REAL* d_img, const REAL* d_trans,
                             REAL scaler, int V, int N, int cap, int H, int W, int TH, int TW,
                             REAL* d_ndc, REAL* d_inv_cov, REAL* d_color, REAL* d_opac, REAL* err_sq)
{
    int gx = (W + TW - 1) / TW, gy = (H + TH - 1) / TH;
    int Hp = gy * TH, Wp = gx * TW, ntile = gx * gy;
    int nrender = tiles ? ntiles_sel : ntile;
    size_t plane = (size_t)Hp * Wp;
    /* accumulate in double irrespective of REAL: the oracle is the accuracy anchor */
    double* acc = (double*)calloc((size_t)V * N * 9, sizeof(double));
    double* acc_err = err_sq ? (double*)calloc((size_t)V * N, sizeof(double)) : NULL;
    for (int b = 0; b < V; b++) {
        const int32_t* rg = range + (size_t)b * (ntile + 2);
#pragma omp parallel for schedule(dynamic, 4)
        for (int ti = 0; ti < nrender; ti++) {
            int tid = tiles ? tiles[(size_t)b * ntiles_sel + ti] : ti + 1;
            if (tid == 0 || tid >= ntile + 1) continue;
            int start = rg[tid];
            if (start == -1) continue;
            int tx = (tid - 1) % gx, ty = (tid - 1) / gx;
            for (int py = 0; py < TH; py++) for (int px = 0; px < TW; px++) {
                int x = tx * TW + px, y = ty * TH + py;
                size_t po = (size_t)y * Wp + x;
                REAL T = Tfinal[(size_t)b * plane + po];
                REAL Tf = T;
                REAL g0 = d_img[((size_t)b * 3 + 0) * plane + po], g1 = d_img[((size_t)b * 3 + 1) * plane + po],
                     g2 = d_img[((size_t)b * 3 + 2) * plane + po];
                REAL gT = d_trans ? d_trans[(size_t)b * plane + po] : 0;
                REAL R0 = 0, R1 = 0, R2 = 0;
                int n = (int)(uint16_t)last[(size_t)b * plane + po];
                for (int k = n - 1; k >= 0; k--) {
                    int i = sorted[(size_t)b * cap + start + k];
                    SUF(splat_rec) s = SUF(load_rec)(ndc, inv_cov, color, opac, b, N, i, H, W);
                    REAL dx = s.px - x, dy = s.py - y;
                    REAL pw = (REAL)-0.5 * (s.A * dx * dx + 2 * s.B * dx * dy + s.C * dy * dy);
                    REAL G = EXP(pw);
                    REAL a = s.o * G;
                    if (a < (REAL)1.0 / 256) continue;
                    a = FMIN(a, (REAL)255.0 / 256);
                    T = FMIN((REAL)1.0, T / (1 - a));
                    REAL w = a * T;
                    REAL da = T * ((s.r - R0) * g0 + (s.g - R1) * g1 + (s.b - R2) * g2);
                    if (d_trans) da -= gT * Tf / (1 - a);
                    R0 += a * (s.r - R0); R1 += a * (s.g - R1); R2 += a * (s.b - R2);
                    REAL dpw = s.o * G * da;
                    double* A9 = acc + ((size_t)b * N + i) * 9;
#pragma omp atomic
                    A9[0] += -(s.A * dx + s.B * dy) * dpw;
#pragma omp atomic
                    A9[1] += -(s.B * dx + s.C * dy) * dpw;
#pragma omp atomic
                    A9[2] += (REAL)-0.5 * dx * dx * dpw;
#pragma omp atomic
                    A9[3] += -dx * dy * dpw;          /* total d/dB; split in halves below */
#pragma omp atomic
                    A9[4] += (REAL)-0.5 * dy * dy * dpw;
#pragma omp atomic
                    A9[5] += w * g0;
#pragma omp atomic
                    A9[6] += w * g1;
#pragma omp atomic
                    A9[7] += w * g2;
#pragma omp atomic
                    A9[8] += G * da;
                    if (acc_err) {
                        double e = (double)(G * da);
#pragma omp atomic
                        acc_err[(size_t)b * N + i] += e * e;
                    }
                }
            }
        }
    }
    for (int b = 0; b < V; b++) for (int i = 0; i < N; i++) {
        const double* A9 = acc + ((size_t)b * N + i) * 9;
        size_t o4 = (size_t)b * 4 * N + i, o3 = (size_t)b * 3 * N + i;
        d_ndc[o4] = (REAL)(A9[0] * 0.5 * W * scaler);
        d_ndc[o4 + N] = (REAL)(A9[1] * 0.5 * H * scaler);
        d_ndc[o4 + 2 * (size_t)N] = 0; d_ndc[o4 + 3 * (size_t)N] = 0;
        d_inv_cov[o4] = (REAL)(A9[2] * scaler);
        d_inv_cov[o4 + N] = (REAL)(A9[3] * 0.5 * scaler);
        d_inv_cov[o4 + 2 * (size_t)N] = (REAL)(A9[3] * 0.5 * scaler);
        d_inv_cov[o4 + 3 * (size_t)N] = (REAL)(A9[4] * scaler);
        d_color[o3] = (REAL)(A9[5] * scaler); d_color[o3 + N] = (REAL)(A9[6] * scaler); d_color[o3 + 2 * (size_t)N] = (REAL)(A9[7] * scaler);
        if (b == 0) d_opac[i] = (REAL)(A9[8] * scaler);
        if (err_sq) err_sq[(size_t)b * N + i] = (REAL)acc_err[(size_t)b * N + i];
    }
    free(acc); if (acc_err) free(acc_err);
}

/* err_square_sum exactly as the reference accumulates it (GR/raster.cu:744-784,812-820): one warp owns a tile, lane l owns
 * the column strip x = l % TW, rows (l / TW) * PPT .. + PPT - 1 with PPT = TH*TW/32 (:644-645), handled as PPT/2 vertical
 * PAIRS (rows 2i, 2i+1).  Per splat the lane keeps a running sum of G*dalpha over its even rows and one over its odd rows;
 * after every pair that ANY lane of the warp reaches (:758) the two running sums are squared and added (:779-784), and the
 * lanes' totals are summed into err_square_sum (:812-818) when any lane has a non-zero d_opacity (:796).  This is NOT the
 * sum over pixels of (G dalpha)^2: it depends on the lane layout, which is part of the reference's contract for the
 * densification score (densify.py:286-292).  Same inputs as orc_raster_backward; err_sq [V,1,N] is overwritten. */
void SUF(orc_raster_err_square_ref)(const int32_t* sorted, const int32_t* range, const REAL* ndc, const REAL* inv_cov,
                                   const REAL* color, const REAL* opac, const int32_t* tiles, int ntiles_sel,
                                   const REAL* Tfinal, const int16_t* last, const REAL* d_img, const REAL* d_trans,
                                   int V, int N, int cap, int H, int W, int TH, int TW, REAL* err_sq)
{
    int gx = (W + TW - 1) / TW, gy = (H + TH - 1) / TH;
    int Hp = gy * TH, Wp = gx * TW, ntile = gx * gy;
    int nrender = tiles ? ntiles_sel : ntile;
    int PPT = TH * TW / 32, NPAIR = PPT / 2, npx = TH * TW;
    size_t plane = (size_t)Hp * Wp;
    double* acc = (double*)calloc((size_t)V * N, sizeof(double));
    for (int b = 0; b < V; b++) {
        const int32_t* rg = range + (size_t)b * (ntile + 2);
#pragma omp parallel for schedule(dynamic, 4)
        for (int ti = 0; ti < nrender; ti++) {
            int tid = tiles ? tiles[(size_t)b * ntiles_sel + ti] : ti + 1;
            if (tid == 0 || tid >= ntile + 1) continue;
            int start = rg[tid];
            if (start == -1) continue;
            int tx = (tid - 1) % gx, ty = (tid - 1) / gx;
            /* per-pixel state of the back-to-front walk, pixel index = lane * PPT + j */
            REAL* T = (REAL*)malloc(sizeof(REAL) * npx * 6);
            REAL* R0 = T + npx; REAL* R1 = R0 + npx; REAL* R2 = R1 + npx; REAL* go = R2 + npx; REAL* Tf = go + npx;
            int* nn = (int*)malloc(sizeof(int) * npx);
            unsigned char* ok = (unsigned char*)malloc(npx);
            int kmax = 0;
            for (int l = 0; l < 32; l++) for (int j = 0; j < PPT; j++) {
                int x = tx * TW + l % TW, y = ty * TH + (l / TW) * PPT + j;
                size_t po = (size_t)y * Wp + x;
                int q = l * PPT + j;
                T[q] = Tfinal[(size_t)b * plane + po]; Tf[q] = T[q];
                R0[q] = R1[q] = R2[q] = 0;
                nn[q] = (int)(uint16_t)last[(size_t)b * plane + po];
                if (nn[q] > kmax) kmax = nn[q];
            }
            for (int k = kmax - 1; k >= 0; k--) {
                int i = sorted[(size_t)b * cap + start + k];
                SUF(splat_rec) s = SUF(load_rec)(ndc, inv_cov, color, opac, b, N, i, H, W);
                int any_nonzero = 0;
                for (int l = 0; l < 32; l++) for (int j = 0; j < PPT; j++) {
                    int x = tx * TW + l % TW, y = ty * TH + (l / TW) * PPT + j;
                    size_t po = (size_t)y * Wp + x;
                    int q = l * PPT + j;
                    ok[q] = 0; go[q] = 0;
                    if (k >= nn[q]) continue;
                    REAL dx = s.px - x, dy = s.py - y;
                    REAL pw = (REAL)-0.5 * (s.A * dx * dx + 2 * s.B * dx * dy + s.C * dy * dy);
                    REAL G = EXP(pw);
                    REAL a = s.o * G;
                    if (a < (REAL)1.0 / 256) continue;
                    a = FMIN(a, (REAL)255.0 / 256);
                    T[q] = FMIN((REAL)1.0, T[q] / (1 - a));
                    REAL g0 = d_img[((size_t)b * 3 + 0) * plane + po], g1 = d_img[((size_t)b * 3 + 1) * plane + po],
                         g2 = d_img[((size_t)b * 3 + 2) * plane + po];
                    REAL da = T[q] * ((s.r - R0[q]) * g0 + (s.g - R1[q]) * g1 + (s.b - R2[q]) * g2);
                    if (d_trans) da -= d_trans[(size_t)b * plane + po] * Tf[q] / (1 - a);
                    R0[q] += a * (s.r - R0[q]); R1[q] += a * (s.g - R1[q]); R2[q] += a * (s.b - R2[q]);
                    ok[q] = 1; go[q] = G * da;
                    if (go[q] != 0) any_nonzero = 1;
                }
                if (!any_nonzero) continue;
                double e = 0;
                /* which pairs does the warp execute? (any lane valid in rows 2i, 2i+1) */
                for (int l = 0; l < 32; l++) {
                    double runx = 0, runy = 0;
                    for (int pi = 0; pi < NPAIR; pi++) {
                        int exec = 0;
                        for (int l2 = 0; l2 < 32 && !exec; l2++) exec = ok[l2 * PPT + 2 * pi] | ok[l2 * PPT + 2 * pi + 1];
                        if (!exec) continue;
                        runx += go[l * PPT + 2 * pi]; runy += go[l * PPT + 2 * pi + 1];
                        e += runx * runx + runy * runy;
                    }
                }
#pragma omp atomic
                acc[(size_t)b * N + i] += e;
            }
            free(T); free(nn); free(ok);
        }
    }
    for (size_t q = 0; q < (size_t)V * N; q++) err_sq[q] = (REAL)acc[q];
    free(acc);
}

/* ---- optimiser / statistics (next rows, SURVEY 8f) --------------------------------------- */

/* GR/compact.cu:320-344 : Adam without bias correction on the visible chunks. param [R,C,S],
 * grad [R,A,S] */
void SUF(orc_adam_chunk)(REAL* param, const REAL* grad, REAL* m, REAL* v2, const int64_t* ids, int nvis,
                        int R, int C, int S, int A, REAL lr, REAL b1, REAL b2, REAL eps)
{
    for (int r = 0; r < R; r++) for (int a = 0; a < nvis; a++) for (int s = 0; s < S; s++) {
        size_t p = ((size_t)r * C + ids[a]) * S + s;
        REAL g = grad[((size_t)r * A + a) * S + s];
        REAL e1 = b1 * m[p] + ((REAL)1.0 - b1) * g;
        REAL e2 = b2 * v2[p] + ((REAL)1.0 - b2) * g * g;
        param[p] += -lr * e1 / (SQRT(e2) + eps);
        m[p] = e1; v2[p] = e2;
    }
}

/* ---- fused L1 + SSIM loss (next row, SURVEY 8f rank 2) ---------------------------------------
 * fused_ssim/ssim.cu:64-274 (ssim map + partial derivatives), :277-437 (backward), :528-712 and
 * :719-850 (the L1 + SSIM loss variants).  11-tap Gaussian (sigma 1.5, the constants of ssim.cu:12-24),
 * zero padding, separable: horizontal pass first, symmetric pairs from the centre outwards then the
 * centre tap (ssim.cu:135-160), vertical pass the same way (:216-240).  Images are [B,CH,H,W]. */
#ifndef ORC_SSIM_CONSTS
#define ORC_SSIM_CONSTS
static const float ORC_GAUSS11[11] = { 0.001028380123898387f, 0.0075987582094967365f, 0.036000773310661316f,
    0.10936068743467331f, 0.21300552785396576f, 0.26601171493530273f, 0.21300552785396576f,
    0.10936068743467331f, 0.036000773310661316f, 0.0075987582094967365f, 0.001028380123898387f };
#endif

static inline REAL SUF(pix0)(const REAL* plane, int H, int W, int y, int x)
{
    return (x < 0 || x >= W || y < 0 || y >= H) ? (REAL)0 : plane[(size_t)y * W + x];
}

/* l1_mode 0: map = ssim (ssim.cu:251-254); 1: map = w (1 - ssim) + (1 - w) |x - y| (ssim.cu:586-588,691).
 * dm_* may be NULL (train = false). */
void SUF(orc_ssim_forward)(const REAL* img1, const REAL* img2, int B, int CH, int H, int W, REAL C1, REAL C2,
                           int l1_mode, REAL ssim_weight, REAL* map, REAL* dm_dmu1, REAL* dm_dsigma1_sq,
                           REAL* dm_dsigma12)
{
    const size_t np = (size_t)H * W;
#pragma omp parallel for schedule(static)
    for (int pc = 0; pc < B * CH; pc++) {
        const REAL* X = img1 + (size_t)pc * np;
        const REAL* Y = img2 + (size_t)pc * np;
        REAL* hx = (REAL*)malloc(sizeof(REAL) * 5 * (size_t)(H + 10) * W);   /* horizontal sums for rows -5..H+4 */
        for (int yy = 0; yy < H + 10; yy++) for (int x = 0; x < W; x++) {
            int y = yy - 5;
            REAL s[5] = { 0, 0, 0, 0, 0 };
            for (int d = 1; d <= 5; d++) {
                REAL w = (REAL)ORC_GAUSS11[5 - d];
                REAL xl = SUF(pix0)(X, H, W, y, x - d), yl = SUF(pix0)(Y, H, W, y, x - d);
                REAL xr = SUF(pix0)(X, H, W, y, x + d), yr = SUF(pix0)(Y, H, W, y, x + d);
                s[0] += (xl + xr) * w;
                s[1] += ((xl * xl) + (xr * xr)) * w;
                s[2] += (yl + yr) * w;
                s[3] += ((yl * yl) + (yr * yr)) * w;
                s[4] += ((xl * yl) + (xr * yr)) * w;
            }
            REAL cx = SUF(pix0)(X, H, W, y, x), cy = SUF(pix0)(Y, H, W, y, x), wc = (REAL)ORC_GAUSS11[5];
            s[0] += cx * wc; s[1] += (cx * cx) * wc; s[2] += cy * wc; s[3] += (cy * cy) * wc; s[4] += (cx * cy) * wc;
            for (int k = 0; k < 5; k++) hx[((size_t)yy * W + x) * 5 + k] = s[k];
        }
        for (int y = 0; y < H; y++) for (int x = 0; x < W; x++) {
            REAL o[5] = { 0, 0, 0, 0, 0 };
            for (int d = 1; d <= 5; d++) {
                REAL w = (REAL)ORC_GAUSS11[5 - d];
                const REAL* top = hx + ((size_t)(y + 5 - d) * W + x) * 5;
                const REAL* bot = hx + ((size_t)(y + 5 + d) * W + x) * 5;
                for (int k = 0; k < 5; k++) o[k] += (top[k] + bot[k]) * w;
            }
            const REAL* ctr = hx + ((size_t)(y + 5) * W + x) * 5;
            for (int k = 0; k < 5; k++) o[k] += ctr[k] * (REAL)ORC_GAUSS11[5];
            REAL mu1 = o[0], mu2 = o[2];
            REAL mu1_sq = mu1 * mu1, mu2_sq = mu2 * mu2;
            REAL sigma1_sq = o[1] - mu1_sq, sigma2_sq = o[3] - mu2_sq, sigma12 = o[4] - mu1 * mu2;
            REAL A = mu1_sq + mu2_sq + C1, Bv = sigma1_sq + sigma2_sq + C2;
            REAL Cv = (REAL)2 * mu1 * mu2 + C1, Dv = (REAL)2 * sigma12 + C2;
            REAL val = (Cv * Dv) / (A * Bv);
            size_t gi = (size_t)pc * np + (size_t)y * W + x;
            if (l1_mode) {
                REAL l1 = FABS(X[(size_t)y * W + x] - Y[(size_t)y * W + x]);
                map[gi] = ssim_weight * ((REAL)1 - val) + ((REAL)1 - ssim_weight) * l1;
            } else {
                map[gi] = val;
            }
            if (dm_dmu1) {
                dm_dmu1[gi] = (mu2 * (REAL)2 * Dv) / (A * Bv) - (mu2 * (REAL)2 * Cv) / (A * Bv)
                            - (mu1 * (REAL)2 * Cv * Dv) / (A * A * Bv) + (mu1 * (REAL)2 * Cv * Dv) / (A * Bv * Bv);
                dm_dsigma1_sq[gi] = (-Cv * Dv) / (A * Bv * Bv);
                dm_dsigma12[gi] = ((REAL)2 * Cv) / (A * Bv);
            }
        }
        free(hx);
    }
}

/* dL/dimg1 from dL/dmap and the saved partials: each partial x chain is filtered with the same separable
 * Gaussian, then  dL/dpix = sum0 + 2 p1 sum1 + p2 sum2  (ssim.cu:417-424).  l1_mode 1 scales the partials by
 * -ssim_weight and adds (1 - w) sign(p1 - p2) chain (ssim.cu:775-779,833-844). */
void SUF(orc_ssim_backward)(const REAL* img1, const REAL* img2, const REAL* dL_dmap, const REAL* dm_dmu1,
                            const REAL* dm_dsigma1_sq, const REAL* dm_dsigma12, int B, int CH, int H, int W,
                            int l1_mode, REAL ssim_weight, REAL* dL_dimg1)
{
    const size_t np = (size_t)H * W;
    const REAL scale = l1_mode ? -ssim_weight : (REAL)1;
#pragma omp parallel for schedule(static)
    for (int pc = 0; pc < B * CH; pc++) {
        const REAL* ch = dL_dmap + (size_t)pc * np;
        const REAL* m[3] = { dm_dmu1 + (size_t)pc * np, dm_dsigma1_sq + (size_t)pc * np, dm_dsigma12 + (size_t)pc * np };
        REAL* hx = (REAL*)malloc(sizeof(REAL) * 3 * (size_t)(H + 10) * W);
        for (int yy = 0; yy < H + 10; yy++) for (int x = 0; x < W; x++) {
            int y = yy - 5;
            for (int k = 0; k < 3; k++) {
                REAL acc = 0;
                for (int d = 1; d <= 5; d++) {
                    REAL l = scale * SUF(pix0)(m[k], H, W, y, x - d) * SUF(pix0)(ch, H, W, y, x - d);
                    REAL r = scale * SUF(pix0)(m[k], H, W, y, x + d) * SUF(pix0)(ch, H, W, y, x + d);
                    acc += (l + r) * (REAL)ORC_GAUSS11[5 - d];
                }
                acc += (scale * SUF(pix0)(m[k], H, W, y, x) * SUF(pix0)(ch, H, W, y, x)) * (REAL)ORC_GAUSS11[5];
                hx[((size_t)yy * W + x) * 3 + k] = acc;
            }
        }
        for (int y = 0; y < H; y++) for (int x = 0; x < W; x++) {
            REAL s[3] = { 0, 0, 0 };
            for (int d = 1; d <= 5; d++) {
                const REAL* top = hx + ((size_t)(y + 5 - d) * W + x) * 3;
                const REAL* bot = hx + ((size_t)(y + 5 + d) * W + x) * 3;
                for (int k = 0; k < 3; k++) s[k] += (top[k] + bot[k]) * (REAL)ORC_GAUSS11[5 - d];
            }
            const REAL* ctr = hx + ((size_t)(y + 5) * W + x) * 3;
            for (int k = 0; k < 3; k++) s[k] += ctr[k] * (REAL)ORC_GAUSS11[5];
            size_t gi = (size_t)pc * np + (size_t)y * W + x;
            REAL p1 = img1[gi], p2 = img2[gi];
            REAL g = s[0] + ((REAL)2 * p1) * s[1] + p2 * s[2];
            if (l1_mode) {
                REAL sg = (p1 == p2) ? (REAL)0 : (p1 > p2 ? (REAL)1 : (REAL)-1);
                g += ((REAL)1 - ssim_weight) * sg * ch[(size_t)y * W + x];
            }
            dL_dimg1[gi] = g;
        }
        free(hx);
    }
}
