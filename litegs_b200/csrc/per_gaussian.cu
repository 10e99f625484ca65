// per_gaussian.cu -- the per-Gaussian (elementwise) operators of the render hot path, op-compatible
// with the reference's `litegs_fused` entry points.  One thread per Gaussian, SoA with the point index
// innermost (every load/store is a coalesced 128-byte row), current-stream launches, checked.
//
// These are the "Level A" kernels (SURVEY.md section 7): they keep the reference's tensor contract so
// litegs/utils/wrapper.py runs on them unchanged.  The fused projection in fused.cu never
// materialises the intermediates these kernels exchange through HBM.
#include <stdarg.h>
#include "common.cuh"
#include "sh.cuh"

// ------------------------------------------------------------------------------------------------
// error string plumbing
// ------------------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";
void lgs_set_error(const char* fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
extern "C" const char* lgs_last_error(void) { return g_err; }
extern "C" int lgs_abi_version(void) { return 3; }

#define VALID_GUARD(idx, n)                                                \
    if ((idx) >= (n) || (valid_length != nullptr && (idx) >= valid_length[0])) return;

// ------------------------------------------------------------------------------------------------
// frustum culling of chunk AABBs + ordered stream compaction.   replaces GR/compact.cu:419-551
// One CTA of 1024 threads; a block-wide ballot scan gives every visible chunk its rank, so the compacted ids come
// out in ascending order (deterministic; the reference's atomics give an arbitrary order).  M is ~8k at 1M
// Gaussians, i.e. 8 slabs of 1024 chunks: the kernel is pure latency, so the 8 slabs' AABB loads are issued together
// (one round trip instead of eight) and the 8 per-slab warp-count scans run in parallel on 8 warps (two barriers per
// 8192 chunks instead of 24).
// ------------------------------------------------------------------------------------------------
constexpr int CULL_U = 8;
__global__ void __launch_bounds__(1024) frustum_cull_kernel(
    const float* __restrict__ origin, const float* __restrict__ ext, const float* __restrict__ planes,
    int M, int V, uint8_t* __restrict__ visibility, int* __restrict__ visible_num, int64_t* __restrict__ ids)
{
    __shared__ int warp_counts[CULL_U][32];     // visible chunks per warp, per slab; then their exclusive prefix
    __shared__ int slab_total[CULL_U];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int running = 0;                            // chunks emitted by earlier groups (same value in every thread)
    for (int base0 = 0; base0 < M; base0 += 1024 * CULL_U) {
        float o[CULL_U][3], e[CULL_U][3];
#pragma unroll
        for (int u = 0; u < CULL_U; u++) {
            const int m = base0 + u * 1024 + threadIdx.x;
            const bool in = m < M;
#pragma unroll
            for (int k = 0; k < 3; k++) { o[u][k] = in ? origin[k * M + m] : 0.0f; e[u][k] = in ? ext[k * M + m] : 0.0f; }
        }
        unsigned ballots[CULL_U];
#pragma unroll
        for (int u = 0; u < CULL_U; u++) {
            const int m = base0 + u * 1024 + threadIdx.x;
            bool vis = false;
            if (m < M) {
                for (int n = 0; n < V; n++) {
                    bool in = true;
#pragma unroll
                    for (int p = 0; p < 6; p++) {
                        const float* pl = planes + (n * 6 + p) * 4;
                        // plain IEEE expression order (no FMA contraction) so the decision is reproducible
                        float d0 = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(pl[0], o[u][0]), __fmul_rn(pl[1], o[u][1])), __fmul_rn(pl[2], o[u][2])), pl[3]);
                        float de = __fadd_rn(__fadd_rn(__fmul_rn(fabsf(pl[0]), e[u][0]), __fmul_rn(fabsf(pl[1]), e[u][1])), __fmul_rn(fabsf(pl[2]), e[u][2]));
                        in &= (__fadd_rn(d0, de) >= 0.0f);
                    }
                    vis |= in;
                }
                visibility[m] = vis ? 1 : 0;
            }
            ballots[u] = __ballot_sync(0xffffffffu, vis);
            if (lane == 0) warp_counts[u][warp] = __popc(ballots[u]);
        }
        __syncthreads();
        if (warp < CULL_U) {                    // warp u scans slab u's 32 warp counts
            const int c = warp_counts[warp][lane];
            int inc = c;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) { int t = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= d) inc += t; }
            warp_counts[warp][lane] = inc - c;
            if (lane == 31) slab_total[warp] = inc;
        }
        __syncthreads();
        int before = running;
#pragma unroll
        for (int u = 0; u < CULL_U; u++) {
            const int m = base0 + u * 1024 + threadIdx.x;
            if ((ballots[u] >> lane) & 1u) ids[before + warp_counts[u][warp] + __popc(ballots[u] & ((1u << lane) - 1u))] = m;
            before += slab_total[u];
        }
        running = before;
        __syncthreads();                        // the shared arrays are rewritten by the next group
    }
    if (threadIdx.x == 0) visible_num[0] = running;
}

extern "C" int lgs_frustum_culling_aabb(const float* aabb_origin, const float* aabb_ext, const float* frustumplane,
                                        int M, int V, uint8_t* visibility, int* visible_num, int64_t* visible_chunk_id,
                                        void* stream)
{
    LGS_REQUIRE(M >= 0 && V >= 1, "frustum_culling_aabb: bad sizes M=%d V=%d", M, V);
    frustum_cull_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(aabb_origin, aabb_ext, frustumplane, M, V, visibility,
                                                             visible_num, visible_chunk_id);
    LGS_CHECK_LAUNCH("frustum_cull_kernel");
    return LGS_OK;
}

// ------------------------------------------------------------------------------------------------
// cull + compact + activate (+ SH -> RGB).                          replaces GR/compact.cu:825-1085
// grid = allocated chunks, block = chunk size.  exp/sigmoid use the accurate expf (1M evaluations per
// view are free next to the 236 B/Gaussian this kernel reads).
// ------------------------------------------------------------------------------------------------
template <int DEG>
__global__ void activate_forward_kernel(
    const int64_t* __restrict__ chunk_ids, const int* __restrict__ visible_num, const float* __restrict__ view, int V,
    const float* __restrict__ pos, const float* __restrict__ scale, const float* __restrict__ rot,
    const float* __restrict__ sh0, const float* __restrict__ shr, const float* __restrict__ opac, int C, int S, int A,
    float* __restrict__ apos, float* __restrict__ ascale, float* __restrict__ arot, float* __restrict__ color,
    float* __restrict__ aopac)
{
    const int a = blockIdx.x, s = threadIdx.x;
    const size_t CS = (size_t)C * S, AS = (size_t)A * S;
    const size_t dst = (size_t)a * S + s;
    if (a >= visible_num[0]) {  // tail chunk: harmless, invisible (GR/compact.cu:888-891)
        aopac[dst] = 0.0f;
        return;
    }
    const size_t src = (size_t)chunk_ids[a] * S + s;
    float p[3] = { pos[src], pos[CS + src], pos[2 * CS + src] };
    apos[dst] = p[0]; apos[AS + dst] = p[1]; apos[2 * AS + dst] = p[2]; apos[3 * AS + dst] = 1.0f;
#pragma unroll
    for (int k = 0; k < 3; k++) ascale[k * AS + dst] = expf(scale[k * CS + src]);
    float q0 = rot[src], q1 = rot[CS + src], q2 = rot[2 * CS + src], q3 = rot[3 * CS + src];
    float rn = 1.0f / sqrtf(q0 * q0 + q1 * q1 + q2 * q2 + q3 * q3 + 1e-12f);
    arot[dst] = q0 * rn; arot[AS + dst] = q1 * rn; arot[2 * AS + dst] = q2 * rn; arot[3 * AS + dst] = q3 * rn;
    aopac[dst] = 1.0f / (1.0f + expf(-opac[src]));
    for (int v = 0; v < V; v++) {
        float cc[3];
        lgs_camera_center(view + v * 16, cc);
        float d0 = p[0] - cc[0], d1 = p[1] - cc[1], d2 = p[2] - cc[2];
        float dn = 1.0f / sqrtf(d0 * d0 + d1 * d1 + d2 * d2 + 1e-12f);
        float b[16];
        lgs_sh_basis<DEG>(d0 * dn, d1 * dn, d2 * dn, b);
        constexpr int K = (DEG + 1) * (DEG + 1);
#pragma unroll
        for (int c = 0; c < 3; c++) {
            float r = b[0] * sh0[c * CS + src];
#pragma unroll
            for (int k = 1; k < K; k++) r += b[k] * shr[((size_t)(k - 1) * 3 + c) * CS + src];
            color[((size_t)v * 3 + c) * AS + dst] = r + 0.5f;
        }
    }
}

extern "C" int lgs_cull_compact_activate(int sh_degree, const int64_t* visible_chunk_id, const int* visible_chunks_num,
                                         const float* view_matrix, int V, const float* position, const float* scale,
                                         const float* rotation, const float* sh_base, const float* sh_rest,
                                         const float* opacity, int C, int S, int A, float* act_position, float* act_scale,
                                         float* act_rotation, float* color, float* act_opacity, void* stream)
{
    LGS_REQUIRE(sh_degree >= 0 && sh_degree <= 3, "cull_compact_activate: sh_degree %d not in 0..3", sh_degree);
    LGS_REQUIRE(S >= 1 && S <= 1024 && V >= 1, "cull_compact_activate: chunk size %d / views %d unsupported", S, V);
    if (A == 0) return LGS_OK;
    cudaStream_t st = (cudaStream_t)stream;
    lgs_with_degree(sh_degree, [&](auto deg) {
        activate_forward_kernel<deg><<<A, S, 0, st>>>(visible_chunk_id, visible_chunks_num, view_matrix, V, position, scale, rotation,
                                                      sh_base, sh_rest, opacity, C, S, A, act_position, act_scale, act_rotation, color,
                                                      act_opacity);
        return LGS_OK;
    });
    LGS_CHECK_LAUNCH("activate_forward_kernel");
    return LGS_OK;
}

// replaces GR/compact.cu:895-980 / 1087-1212.  true_sigmoid=0 keeps the reference's opacity-logit
// gradient d_o * sigma(x) (GR/compact.cu:952, SURVEY Q15); 1 gives the analytic sigma(1-sigma).
template <int DEG>
__global__ void activate_backward_kernel(
    const int64_t* __restrict__ chunk_ids, const int* __restrict__ visible_num, const float* __restrict__ view, int V,
    const float* __restrict__ pos, const float* __restrict__ scale, const float* __restrict__ rot,
    const float* __restrict__ opac, int C, int S, int A, int rest_dim, int true_sigmoid,
    const float* __restrict__ g_apos, const float* __restrict__ g_ascale, const float* __restrict__ g_arot,
    const float* __restrict__ g_color, const float* __restrict__ g_aopac,
    float* __restrict__ g_pos, float* __restrict__ g_scale, float* __restrict__ g_rot, float* __restrict__ g_sh0,
    float* __restrict__ g_shr, float* __restrict__ g_opac)
{
    const int a = blockIdx.x, s = threadIdx.x;
    if (a >= visible_num[0]) return;
    const size_t CS = (size_t)C * S, AS = (size_t)A * S;
    const size_t dst = (size_t)a * S + s, src = (size_t)chunk_ids[a] * S + s;
#pragma unroll
    for (int k = 0; k < 3; k++) g_pos[k * AS + dst] = g_apos[k * AS + dst];
#pragma unroll
    for (int k = 0; k < 3; k++) g_scale[k * AS + dst] = expf(scale[k * CS + src]) * g_ascale[k * AS + dst];
    float q[4], g[4], o[4];
#pragma unroll
    for (int k = 0; k < 4; k++) { q[k] = rot[k * CS + src]; g[k] = g_arot[k * AS + dst]; }
    float rn = 1.0f / sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3] + 1e-12f);
#pragma unroll
    for (int k = 0; k < 4; k++) o[k] = q[k] * rn;
    float dot = g[0] * o[0] + g[1] * o[1] + g[2] * o[2] + g[3] * o[3];
#pragma unroll
    for (int k = 0; k < 4; k++) g_rot[k * AS + dst] = rn * (g[k] - dot * o[k]);
    const float u = 1.0f / (1.0f + expf(opac[src])), sig = 1.0f - u;     // 1 - sig = u, not formed from the rounded sig
    g_opac[dst] = g_aopac[dst] * (true_sigmoid ? sig * u : sig);

    float p[3] = { pos[src], pos[CS + src], pos[2 * CS + src] };
    constexpr int K = (DEG + 1) * (DEG + 1);
    float acc[3][K];
#pragma unroll
    for (int c = 0; c < 3; c++)
#pragma unroll
        for (int k = 0; k < K; k++) acc[c][k] = 0.0f;
    for (int v = 0; v < V; v++) {
        float cc[3];
        lgs_camera_center(view + v * 16, cc);
        float d0 = p[0] - cc[0], d1 = p[1] - cc[1], d2 = p[2] - cc[2];
        float dn = 1.0f / sqrtf(d0 * d0 + d1 * d1 + d2 * d2 + 1e-12f);
        float b[16];
        lgs_sh_basis<DEG>(d0 * dn, d1 * dn, d2 * dn, b);
#pragma unroll
        for (int c = 0; c < 3; c++) {
            float gc = g_color[((size_t)v * 3 + c) * AS + dst];
#pragma unroll
            for (int k = 0; k < K; k++) acc[c][k] += b[k] * gc;
        }
    }
#pragma unroll
    for (int c = 0; c < 3; c++) {
        g_sh0[c * AS + dst] = acc[c][0];
#pragma unroll
        for (int k = 1; k < K; k++) g_shr[((size_t)(k - 1) * 3 + c) * AS + dst] = acc[c][k];
    }
    (void)rest_dim;
}

extern "C" int lgs_activate_backward(int sh_degree, const int64_t* visible_chunk_id, const int* visible_chunks_num,
                                     const float* view_matrix, int V, const float* position, const float* scale,
                                     const float* rotation, const float* opacity, int C, int S, int A, int rest_dim,
                                     int true_sigmoid_grad, const float* g_act_position, const float* g_act_scale,
                                     const float* g_act_rotation, const float* g_color, const float* g_act_opacity,
                                     float* g_position, float* g_scale, float* g_rotation, float* g_sh_base,
                                     float* g_sh_rest, float* g_opacity, void* stream)
{
    LGS_REQUIRE(sh_degree >= 0 && sh_degree <= 3, "activate_backward: sh_degree %d not in 0..3", sh_degree);
    LGS_REQUIRE(S >= 1 && S <= 1024 && V >= 1, "activate_backward: chunk size %d / views %d unsupported", S, V);
    LGS_REQUIRE(rest_dim >= (sh_degree + 1) * (sh_degree + 1) - 1, "activate_backward: sh_rest has %d rows, degree %d needs %d",
                rest_dim, sh_degree, (sh_degree + 1) * (sh_degree + 1) - 1);
    if (A == 0) return LGS_OK;
    cudaStream_t st = (cudaStream_t)stream;
    // rows of sh_rest above the active degree (and tail chunks) must read as zero, as with the
    // reference's torch::zeros allocation (GR/compact.cu:1107).
    LGS_CUDA(cudaMemsetAsync(g_sh_rest, 0, sizeof(float) * (size_t)rest_dim * 3 * A * S, st));
    lgs_with_degree(sh_degree, [&](auto deg) {
        activate_backward_kernel<deg><<<A, S, 0, st>>>(visible_chunk_id, visible_chunks_num, view_matrix, V, position, scale, rotation,
                                                       opacity, C, S, A, rest_dim, true_sigmoid_grad, g_act_position, g_act_scale,
                                                       g_act_rotation, g_color, g_act_opacity, g_position, g_scale, g_rotation, g_sh_base,
                                                       g_sh_rest, g_opacity);
        return LGS_OK;
    });
    LGS_CHECK_LAUNCH("activate_backward_kernel");
    return LGS_OK;
}

// ------------------------------------------------------------------------------------------------
// world -> view -> NDC.                                              replaces GR/transform.cu:378-598
// ------------------------------------------------------------------------------------------------
__global__ void mvp_forward_kernel(const float* __restrict__ view, const float* __restrict__ proj,
                                   const float* __restrict__ pos, const int* __restrict__ valid_length,
                                   float* __restrict__ vpos, float* __restrict__ ndc, int N)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    VALID_GUARD(i, N);
    const float* Vm = view + b * 16; const float* P = proj + b * 16;
    float w[4], v[4], h[4];
#pragma unroll
    for (int k = 0; k < 4; k++) w[k] = pos[(size_t)k * N + i];
#pragma unroll
    for (int k = 0; k < 4; k++) v[k] = w[0] * Vm[k] + w[1] * Vm[4 + k] + w[2] * Vm[8 + k] + w[3] * Vm[12 + k];
#pragma unroll
    for (int k = 0; k < 4; k++) h[k] = v[0] * P[k] + v[1] * P[4 + k] + v[2] * P[8 + k] + v[3] * P[12 + k];
    float iw = (fabsf(h[3]) > 1e-12f) ? (1.0f / h[3]) : 0.0f;
    size_t o = (size_t)b * 4 * N + i;
#pragma unroll
    for (int k = 0; k < 4; k++) vpos[o + (size_t)k * N] = v[k];
    ndc[o] = h[0] * iw; ndc[o + N] = h[1] * iw; ndc[o + 2 * (size_t)N] = h[2] * iw; ndc[o + 3 * (size_t)N] = 1.0f;
}

extern "C" int lgs_mvp_transform_forward(const float* world_position, const float* view_matrix, const float* proj_matrix,
                                         const int* valid_length, int V, int N, float* view_position, float* ndc_position,
                                         void* stream)
{
    LGS_REQUIRE(V >= 1 && N >= 0, "mvp_transform_forward: bad sizes V=%d N=%d", V, N);
    if (N == 0) return LGS_OK;
    mvp_forward_kernel<<<dim3(lgs_cdiv(N, 256), V), 256, 0, (cudaStream_t)stream>>>(view_matrix, proj_matrix, world_position,
                                                                                  valid_length, view_position, ndc_position, N);
    LGS_CHECK_LAUNCH("mvp_forward_kernel");
    return LGS_OK;
}

__global__ void mvp_backward_kernel(const float* __restrict__ g_ndc, const float* __restrict__ g_view,
                                    const float* __restrict__ view, const float* __restrict__ proj,
                                    const float* __restrict__ vpos, const int* __restrict__ valid_length,
                                    float* __restrict__ g_pos, int V, int N)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    VALID_GUARD(i, N);
    float acc[4] = { 0.f, 0.f, 0.f, 0.f };
    for (int b = 0; b < V; b++) {
        const float* Vm = view + b * 16; const float* P = proj + b * 16;
        size_t o = (size_t)b * 4 * N + i;
        float v[4], h[4], gn[4], dh[4], dv[4];
#pragma unroll
        for (int k = 0; k < 4; k++) v[k] = vpos[o + (size_t)k * N];
#pragma unroll
        for (int k = 0; k < 4; k++) h[k] = v[0] * P[k] + v[1] * P[4 + k] + v[2] * P[8 + k] + v[3] * P[12 + k];
        float iw = (fabsf(h[3]) > 1e-12f) ? (1.0f / h[3]) : 0.0f;
        float n0 = h[0] * iw, n1 = h[1] * iw, n2 = h[2] * iw;
#pragma unroll
        for (int k = 0; k < 4; k++) gn[k] = g_ndc[o + (size_t)k * N];
        dh[0] = gn[0] * iw; dh[1] = gn[1] * iw; dh[2] = gn[2] * iw;
        dh[3] = -(gn[0] * n0 + gn[1] * n1 + gn[2] * n2) * iw;
#pragma unroll
        for (int k = 0; k < 4; k++)
            dv[k] = dh[0] * P[k * 4] + dh[1] * P[k * 4 + 1] + dh[2] * P[k * 4 + 2] + dh[3] * P[k * 4 + 3] + g_view[o + (size_t)k * N];
#pragma unroll
        for (int k = 0; k < 4; k++)
            acc[k] += dv[0] * Vm[k * 4] + dv[1] * Vm[k * 4 + 1] + dv[2] * Vm[k * 4 + 2] + dv[3] * Vm[k * 4 + 3];
    }
#pragma unroll
    for (int k = 0; k < 4; k++) g_pos[(size_t)k * N + i] = acc[k];
}

extern "C" int lgs_mvp_transform_backward(const float* grad_ndc_pos, const float* grad_view_pos, const float* view_matrix,
                                          const float* proj_matrix, const float* view_pos, const int* valid_length, int V,
                                          int N, float* grad_world_pos, void* stream)
{
    LGS_REQUIRE(V >= 1 && N >= 0, "mvp_transform_backward: bad sizes V=%d N=%d", V, N);
    if (N == 0) return LGS_OK;
    mvp_backward_kernel<<<lgs_cdiv(N, 256), 256, 0, (cudaStream_t)stream>>>(grad_ndc_pos, grad_view_pos, view_matrix, proj_matrix,
                                                                          view_pos, valid_length, grad_world_pos, V, N);
    LGS_CHECK_LAUNCH("mvp_backward_kernel");
    return LGS_OK;
}

// ------------------------------------------------------------------------------------------------
// T = diag(s) R(q).                                                   replaces GR/transform.cu:92-256
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void quat_R(float r, float x, float y, float z, float* R)
{
    R[0] = 1 - 2 * (y * y + z * z); R[1] = 2 * (x * y + r * z);     R[2] = 2 * (x * z - r * y);
    R[3] = 2 * (x * y - r * z);     R[4] = 1 - 2 * (x * x + z * z); R[5] = 2 * (y * z + r * x);
    R[6] = 2 * (x * z + r * y);     R[7] = 2 * (y * z - r * x);     R[8] = 1 - 2 * (x * x + y * y);
}

__global__ void transform_forward_kernel(const float* __restrict__ quat, const float* __restrict__ scale,
                                         const int* __restrict__ valid_length, float* __restrict__ T, int N)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    VALID_GUARD(i, N);
    float R[9];
    quat_R(quat[i], quat[(size_t)N + i], quat[2 * (size_t)N + i], quat[3 * (size_t)N + i], R);
#pragma unroll
    for (int a = 0; a < 3; a++) {
        float s = scale[(size_t)a * N + i];
#pragma unroll
        for (int b = 0; b < 3; b++) T[((size_t)a * 3 + b) * N + i] = R[a * 3 + b] * s;
    }
}

extern "C" int lgs_create_transform_matrix_forward(const float* quaternion, const float* scale, const int* valid_length,
                                                   int N, float* transform, void* stream)
{
    LGS_REQUIRE(N >= 0, "createTransformMatrix_forward: bad N=%d", N);
    if (N == 0) return LGS_OK;
    transform_forward_kernel<<<lgs_cdiv(N, 256), 256, 0, (cudaStream_t)stream>>>(quaternion, scale, valid_length, transform, N);
    LGS_CHECK_LAUNCH("transform_forward_kernel");
    return LGS_OK;
}

__global__ void transform_backward_kernel(const float* __restrict__ gT, const float* __restrict__ quat,
                                          const float* __restrict__ scale, const int* __restrict__ valid_length,
                                          float* __restrict__ g_quat, float* __restrict__ g_scale, int N)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    VALID_GUARD(i, N);
    float r = quat[i], x = quat[(size_t)N + i], y = quat[2 * (size_t)N + i], z = quat[3 * (size_t)N + i];
    float R[9], dt[9];
    quat_R(r, x, y, z, R);
#pragma unroll
    for (int k = 0; k < 9; k++) dt[k] = gT[(size_t)k * N + i];
#pragma unroll
    for (int a = 0; a < 3; a++) {
        g_scale[(size_t)a * N + i] = R[a * 3] * dt[a * 3] + R[a * 3 + 1] * dt[a * 3 + 1] + R[a * 3 + 2] * dt[a * 3 + 2];
        float s = scale[(size_t)a * N + i];
        dt[a * 3] *= s; dt[a * 3 + 1] *= s; dt[a * 3 + 2] *= s;
    }
    g_quat[i] = 2 * z * (dt[1] - dt[3]) + 2 * y * (dt[6] - dt[2]) + 2 * x * (dt[5] - dt[7]);
    g_quat[(size_t)N + i] = 2 * y * (dt[3] + dt[1]) + 2 * z * (dt[6] + dt[2]) + 2 * r * (dt[5] - dt[7]) - 4 * x * (dt[8] + dt[4]);
    g_quat[2 * (size_t)N + i] = 2 * x * (dt[3] + dt[1]) + 2 * r * (dt[6] - dt[2]) + 2 * z * (dt[5] + dt[7]) - 4 * y * (dt[8] + dt[0]);
    g_quat[3 * (size_t)N + i] = 2 * r * (dt[1] - dt[3]) + 2 * x * (dt[6] + dt[2]) + 2 * y * (dt[5] + dt[7]) - 4 * z * (dt[4] + dt[0]);
}

extern "C" int lgs_create_transform_matrix_backward(const float* transform_grad, const float* quaternion, const float* scale,
                                                    const int* valid_length, int N, float* grad_quaternion, float* grad_scale,
                                                    void* stream)
{
    LGS_REQUIRE(N >= 0, "createTransformMatrix_backward: bad N=%d", N);
    if (N == 0) return LGS_OK;
    transform_backward_kernel<<<lgs_cdiv(N, 256), 256, 0, (cudaStream_t)stream>>>(transform_grad, quaternion, scale, valid_length,
                                                                               grad_quaternion, grad_scale, N);
    LGS_CHECK_LAUNCH("transform_backward_kernel");
    return LGS_OK;
}

// ------------------------------------------------------------------------------------------------
// ray-space Jacobian.                                                  replaces GR/transform.cu:22-90
// The output is [V,3,3,N] with five structurally-zero rows; the kernel writes all nine so the caller
// does not need a separate memset pass (the reference allocates with torch::zeros).
// ------------------------------------------------------------------------------------------------
__global__ void jacobian_kernel(const float* __restrict__ vpos, const float* __restrict__ proj,
                                const int* __restrict__ valid_length, int H, int W, float* __restrict__ J, int N)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    if (i >= N) return;
    size_t o = (size_t)b * 9 * N + i;
    bool live = !(valid_length != nullptr && i >= valid_length[0]);
    float j00 = 0.f, j11 = 0.f, j20 = 0.f, j21 = 0.f;
    if (live) {
        float p00 = proj[b * 16], p11 = proj[b * 16 + 5];
        float fx = p00 * W * 0.5f, fy = p11 * H * 0.5f;
        size_t vo = (size_t)b * 4 * N + i;
        float tx = vpos[vo], ty = vpos[vo + N], tz = vpos[vo + 2 * (size_t)N];
        float lx = tz / p00 * 1.3f, ly = tz / p11 * 1.3f;
        tx = fmaxf(fminf(tx, lx), -lx);
        ty = fmaxf(fminf(ty, ly), -ly);
        float rz = 1.0f / fmaxf(tz, 1e-2f);
        float rz2 = rz * rz;
        j00 = fx * rz; j11 = fy * rz; j20 = -fx * tx * rz2; j21 = -fy * ty * rz2;
    }
    J[o] = j00; J[o + (size_t)N] = 0.f; J[o + 2 * (size_t)N] = 0.f;
    J[o + 3 * (size_t)N] = 0.f; J[o + 4 * (size_t)N] = j11; J[o + 5 * (size_t)N] = 0.f;
    J[o + 6 * (size_t)N] = j20; J[o + 7 * (size_t)N] = j21; J[o + 8 * (size_t)N] = 0.f;
}

extern "C" int lgs_jacobian_rayspace(const float* view_pos, const float* proj_matrix, const int* valid_length, int V, int N,
                                     int output_h, int output_w, float* jacobian, void* stream)
{
    LGS_REQUIRE(V >= 1 && N >= 0, "jacobianRayspace: bad sizes V=%d N=%d", V, N);
    if (N == 0) return LGS_OK;
    jacobian_kernel<<<dim3(lgs_cdiv(N, 256), V), 256, 0, (cudaStream_t)stream>>>(view_pos, proj_matrix, valid_length, output_h,
                                                                               output_w, jacobian, N);
    LGS_CHECK_LAUNCH("jacobian_kernel");
    return LGS_OK;
}

// ------------------------------------------------------------------------------------------------
// cov2d = (T V3 J)^T (T V3 J) + 0.3 I and its backward.              replaces GR/transform.cu:736-927
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void cov_M(const float* __restrict__ T, int N, int i, const float* __restrict__ Vm,
                                      const float* __restrict__ Jb, float* VJ, float* M)
{
    float Jl[6];
#pragma unroll
    for (int a = 0; a < 3; a++)
#pragma unroll
        for (int c = 0; c < 2; c++) Jl[a * 2 + c] = Jb[((size_t)a * 3 + c) * N + i];
#pragma unroll
    for (int a = 0; a < 3; a++)
#pragma unroll
        for (int c = 0; c < 2; c++) {
            float t = 0.f;
#pragma unroll
            for (int k = 0; k < 3; k++) t += Vm[a * 4 + k] * Jl[k * 2 + c];
            VJ[a * 2 + c] = t;
        }
#pragma unroll
    for (int a = 0; a < 3; a++)
#pragma unroll
        for (int c = 0; c < 2; c++) {
            float t = 0.f;
#pragma unroll
            for (int k = 0; k < 3; k++) t += T[((size_t)a * 3 + k) * N + i] * VJ[k * 2 + c];
            M[a * 2 + c] = t;
        }
}

__global__ void cov2d_forward_kernel(const float* __restrict__ J, const float* __restrict__ view, const float* __restrict__ T,
                                     const int* __restrict__ valid_length, float* __restrict__ cov, int N)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    VALID_GUARD(i, N);
    float VJ[6], M[6];
    cov_M(T, N, i, view + b * 16, J + (size_t)b * 9 * N, VJ, M);
    float c00 = M[0] * M[0] + M[2] * M[2] + M[4] * M[4] + 0.3f;
    float c01 = M[0] * M[1] + M[2] * M[3] + M[4] * M[5];
    float c11 = M[1] * M[1] + M[3] * M[3] + M[5] * M[5] + 0.3f;
    size_t o = (size_t)b * 4 * N + i;
    cov[o] = c00; cov[o + N] = c01; cov[o + 2 * (size_t)N] = c01; cov[o + 3 * (size_t)N] = c11;
}

extern "C" int lgs_create_cov2d_forward(const float* J, const float* view_matrix, const float* transform_matrix,
                                        const int* valid_length, int V, int N, float* cov2d, void* stream)
{
    LGS_REQUIRE(V >= 1 && N >= 0, "createCov2dDirectly_forward: bad sizes V=%d N=%d", V, N);
    if (N == 0) return LGS_OK;
    cov2d_forward_kernel<<<dim3(lgs_cdiv(N, 256), V), 256, 0, (cudaStream_t)stream>>>(J, view_matrix, transform_matrix, valid_length,
                                                                                    cov2d, N);
    LGS_CHECK_LAUNCH("cov2d_forward_kernel");
    return LGS_OK;
}

__global__ void cov2d_backward_kernel(const float* __restrict__ g_cov, const float* __restrict__ J, const float* __restrict__ view,
                                      const float* __restrict__ T, const int* __restrict__ valid_length, float* __restrict__ gT,
                                      int V, int N)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    float acc[9];
#pragma unroll
    for (int k = 0; k < 9; k++) acc[k] = 0.f;
    if (!(valid_length != nullptr && i >= valid_length[0])) {
        for (int b = 0; b < V; b++) {
            float VJ[6], M[6], G[4], dM[6];
            cov_M(T, N, i, view + b * 16, J + (size_t)b * 9 * N, VJ, M);
#pragma unroll
            for (int k = 0; k < 4; k++) G[k] = g_cov[((size_t)b * 4 + k) * N + i];
#pragma unroll
            for (int a = 0; a < 3; a++)
#pragma unroll
                for (int c = 0; c < 2; c++) dM[a * 2 + c] = 2.f * (M[a * 2] * G[c] + M[a * 2 + 1] * G[2 + c]);
#pragma unroll
            for (int a = 0; a < 3; a++)
#pragma unroll
                for (int k = 0; k < 3; k++) acc[a * 3 + k] += dM[a * 2] * VJ[k * 2] + dM[a * 2 + 1] * VJ[k * 2 + 1];
        }
    }
#pragma unroll
    for (int k = 0; k < 9; k++) gT[(size_t)k * N + i] = acc[k];
}

extern "C" int lgs_create_cov2d_backward(const float* cov2d_grad, const float* J, const float* view_matrix,
                                         const float* transform_matrix, const int* valid_length, int V, int N,
                                         float* transform_matrix_grad, void* stream)
{
    LGS_REQUIRE(V >= 1 && N >= 0, "createCov2dDirectly_backward: bad sizes V=%d N=%d", V, N);
    if (N == 0) return LGS_OK;
    cov2d_backward_kernel<<<lgs_cdiv(N, 256), 256, 0, (cudaStream_t)stream>>>(cov2d_grad, J, view_matrix, transform_matrix, valid_length,
                                                                           transform_matrix_grad, V, N);
    LGS_CHECK_LAUNCH("cov2d_backward_kernel");
    return LGS_OK;
}

// ------------------------------------------------------------------------------------------------
// eigen-decomposition + guarded inverse of the 2x2 covariance.       replaces GR/transform.cu:1364-1518
// ------------------------------------------------------------------------------------------------
__global__ void eigh_inv_forward_kernel(const float* __restrict__ in, const int* __restrict__ valid_length,
                                        float* __restrict__ val, float* __restrict__ vec, float* __restrict__ inv, int N)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    VALID_GUARD(i, N);
    size_t o = (size_t)b * 4 * N + i;
    float m00 = in[o], m01 = in[o + N], m10 = in[o + 2 * (size_t)N], m11 = in[o + 3 * (size_t)N];
    float det = m00 * m11 - m01 * m10;
    float det1 = (m00 - m01) * (m11 - m01) + m01 * (m00 + m11 - 2 * m01);
    det = (fabsf(det) < fabsf(1e-5f * m01 * m10)) ? det1 : det;
    float t0 = m00 + m11;
    float t1 = sqrtf((m00 - m11) * (m00 - m11) + 4 * m01 * m01);
    t1 = fmaxf(t1, 1e-9f);
    float e0 = 0.5f * (t0 - t1), e1 = 0.5f * (t0 + t1);
    val[((size_t)b * 2) * N + i] = e0;
    val[((size_t)b * 2 + 1) * N + i] = e1;
    float v00, v01, v10, v11;
    if (fabsf(e0 - m00) > fabsf(e0 - m11)) { v00 = -m01; v01 = m00 - e0; v10 = e1 - m11; v11 = m01; }
    else { v00 = m11 - e0; v01 = -m01; v10 = m01; v11 = e1 - m00; }
    float l0 = 1.0f / sqrtf(v00 * v00 + v01 * v01), l1 = 1.0f / sqrtf(v10 * v10 + v11 * v11);
    vec[o] = v00 * l0; vec[o + N] = v10 * l1; vec[o + 2 * (size_t)N] = v01 * l0; vec[o + 3 * (size_t)N] = v11 * l1;
    det = (fabsf(det) < 1e-9f) ? 1e-9f : det;
    float dr = 1.0f / det;
    inv[o] = m11 * dr; inv[o + N] = -m01 * dr; inv[o + 2 * (size_t)N] = -m10 * dr; inv[o + 3 * (size_t)N] = m00 * dr;
}

extern "C" int lgs_eigh_and_inv_2x2_forward(const float* input, const int* valid_length, int V, int N, float* val, float* vec,
                                            float* inv, void* stream)
{
    LGS_REQUIRE(V >= 1 && N >= 0, "eigh_and_inv_2x2matrix_forward: bad sizes V=%d N=%d", V, N);
    if (N == 0) return LGS_OK;
    eigh_inv_forward_kernel<<<dim3(lgs_cdiv(N, 256), V), 256, 0, (cudaStream_t)stream>>>(input, valid_length, val, vec, inv, N);
    LGS_CHECK_LAUNCH("eigh_inv_forward_kernel");
    return LGS_OK;
}

__global__ void inv2x2_backward_kernel(const float* __restrict__ inv, const float* __restrict__ g_inv,
                                       const int* __restrict__ valid_length, float* __restrict__ g_in, int N)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    VALID_GUARD(i, N);
    size_t o = (size_t)b * 4 * N + i;
    float A[4], G[4], t[4];
#pragma unroll
    for (int k = 0; k < 4; k++) { A[k] = inv[o + (size_t)k * N]; G[k] = g_inv[o + (size_t)k * N]; }
    t[0] = A[0] * G[0] + A[1] * G[2]; t[1] = A[0] * G[1] + A[1] * G[3];
    t[2] = A[2] * G[0] + A[3] * G[2]; t[3] = A[2] * G[1] + A[3] * G[3];
    g_in[o] = -(t[0] * A[0] + t[1] * A[2]);
    g_in[o + N] = -(t[0] * A[1] + t[1] * A[3]);
    g_in[o + 2 * (size_t)N] = -(t[2] * A[0] + t[3] * A[2]);
    g_in[o + 3 * (size_t)N] = -(t[2] * A[1] + t[3] * A[3]);
}

extern "C" int lgs_inv_2x2_backward(const float* inv_matrix, const float* grad_inv, const int* valid_length, int V, int N,
                                    float* grad_matrix, void* stream)
{
    LGS_REQUIRE(V >= 1 && N >= 0, "inv_2x2matrix_backward: bad sizes V=%d N=%d", V, N);
    if (N == 0) return LGS_OK;
    inv2x2_backward_kernel<<<dim3(lgs_cdiv(N, 256), V), 256, 0, (cudaStream_t)stream>>>(inv_matrix, grad_inv, valid_length, grad_matrix, N);
    LGS_CHECK_LAUNCH("inv2x2_backward_kernel");
    return LGS_OK;
}

// ------------------------------------------------------------------------------------------------
// standalone SH -> RGB for the cluster_size=0 path.                 replaces GR/transform.cu:951-1361
// ------------------------------------------------------------------------------------------------
template <int DEG>
__global__ void sh2rgb_forward_kernel(const float* __restrict__ sh0, const float* __restrict__ shr, const float* __restrict__ dirs,
                                      float* __restrict__ rgb, int N)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x, v = blockIdx.y;
    if (i >= N) return;
    constexpr int K = (DEG + 1) * (DEG + 1);
    float b[16];
    size_t od = (size_t)v * 3 * N + i;
    lgs_sh_basis<DEG>(dirs[od], dirs[od + N], dirs[od + 2 * (size_t)N], b);
#pragma unroll
    for (int c = 0; c < 3; c++) {
        float r = b[0] * sh0[(size_t)c * N + i];
#pragma unroll
        for (int k = 1; k < K; k++) r += b[k] * shr[((size_t)(k - 1) * 3 + c) * N + i];
        rgb[od + (size_t)c * N] = r + 0.5f;
    }
}

extern "C" int lgs_sh2rgb_forward(int degree, const float* sh_base, const float* sh_rest, const float* dirs, int V, int N,
                                  float* rgb, void* stream)
{
    LGS_REQUIRE(degree >= 0 && degree <= 3, "sh2rgb_forward: degree %d not in 0..3", degree);
    if (N == 0) return LGS_OK;
    dim3 grid(lgs_cdiv(N, 256), V);
    cudaStream_t st = (cudaStream_t)stream;
    lgs_with_degree(degree, [&](auto deg) {
        sh2rgb_forward_kernel<deg><<<grid, 256, 0, st>>>(sh_base, sh_rest, dirs, rgb, N);
        return LGS_OK;
    });
    LGS_CHECK_LAUNCH("sh2rgb_forward_kernel");
    return LGS_OK;
}

// The reference assigns (not accumulates) per view, so the last view wins (GR/transform.cu:1106-1115);
// V is 1 in every caller.  Kept as is.
template <int DEG>
__global__ void sh2rgb_backward_kernel(const float* __restrict__ dirs, const float* __restrict__ rgb_grad, int V, int N,
                                       float* __restrict__ g0, float* __restrict__ gr)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    constexpr int K = (DEG + 1) * (DEG + 1);
    for (int v = 0; v < V; v++) {
        float b[16];
        size_t od = (size_t)v * 3 * N + i;
        lgs_sh_basis<DEG>(dirs[od], dirs[od + N], dirs[od + 2 * (size_t)N], b);
#pragma unroll
        for (int c = 0; c < 3; c++) {
            float g = rgb_grad[od + (size_t)c * N];
            g0[(size_t)c * N + i] = b[0] * g;
#pragma unroll
            for (int k = 1; k < K; k++) gr[((size_t)(k - 1) * 3 + c) * N + i] = b[k] * g;
        }
    }
}

extern "C" int lgs_sh2rgb_backward(int degree, const float* rgb_grad, int sh_rest_dim, const float* dirs, int V, int N,
                                   float* sh_base_grad, float* sh_rest_grad, float* dir_grad, void* stream)
{
    LGS_REQUIRE(degree >= 0 && degree <= 3, "sh2rgb_backward: degree %d not in 0..3", degree);
    LGS_REQUIRE(sh_rest_dim >= (degree + 1) * (degree + 1) - 1, "sh2rgb_backward: sh_rest_dim %d too small for degree %d", sh_rest_dim, degree);
    if (N == 0) return LGS_OK;
    cudaStream_t st = (cudaStream_t)stream;
    LGS_CUDA(cudaMemsetAsync(sh_rest_grad, 0, sizeof(float) * (size_t)sh_rest_dim * 3 * N, st));
    if (dir_grad) LGS_CUDA(cudaMemsetAsync(dir_grad, 0, sizeof(float) * (size_t)V * 3 * N, st));
    int grid = lgs_cdiv(N, 256);
    lgs_with_degree(degree, [&](auto deg) {
        sh2rgb_backward_kernel<deg><<<grid, 256, 0, st>>>(dirs, rgb_grad, V, N, sh_base_grad, sh_rest_grad);
        return LGS_OK;
    });
    LGS_CHECK_LAUNCH("sh2rgb_backward_kernel");
    return LGS_OK;
}

// ------------------------------------------------------------------------------------------------
// sparse Adam (no bias correction) and the chunk scatter op.   replaces GR/compact.cu:320-417,1221-1336
// ------------------------------------------------------------------------------------------------
__global__ void adam_chunk_kernel(float* __restrict__ param, const float* __restrict__ grad, float* __restrict__ m,
                                  float* __restrict__ v2, const int64_t* __restrict__ ids, const int* __restrict__ valid_length,
                                  int C, int S, int A, float lr, float b1, float b2, float eps)
{
    int a = blockIdx.x, r = blockIdx.y, s = threadIdx.x;
    if (valid_length != nullptr && a >= valid_length[0]) return;
    size_t p = ((size_t)r * C + ids[a]) * S + s;
    float g = grad[((size_t)r * A + a) * S + s];
    float e1 = b1 * m[p] + (1.0f - b1) * g;
    float e2 = b2 * v2[p] + (1.0f - b2) * g * g;
    param[p] += -lr * e1 / (sqrtf(e2) + eps);
    m[p] = e1; v2[p] = e2;
}

// Same update with 16-byte accesses: a thread owns 4 consecutive Gaussians of a chunk, a CTA covers ROWS rows of one visible
// chunk (S/4 x ROWS threads).  Four times fewer threads and four times more bytes in flight per thread than the one-element
// form (which is what the reference launches: GR/compact.cu:320-344) -- the six launches of an optimiser step are bandwidth
// bound, not latency bound, this way.
template <int ROWS>
__global__ void adam_chunk_vec4_kernel(float* __restrict__ param, const float* __restrict__ grad, float* __restrict__ m,
                                       float* __restrict__ v2, const int64_t* __restrict__ ids, const int* __restrict__ valid_length,
                                       int R, int C, int S, int A, float lr, float b1, float b2, float eps)
{
    const int a = blockIdx.x, r = blockIdx.y * ROWS + threadIdx.y;
    if (r >= R || (valid_length != nullptr && a >= valid_length[0])) return;
    const size_t p = ((size_t)r * C + ids[a]) * S + 4 * threadIdx.x;
    const float4 g4 = *reinterpret_cast<const float4*>(grad + ((size_t)r * A + a) * S + 4 * threadIdx.x);
    float4 m4 = *reinterpret_cast<const float4*>(m + p), v4 = *reinterpret_cast<const float4*>(v2 + p);
    float4 p4 = *reinterpret_cast<const float4*>(param + p);
    const float* gp = &g4.x; float* mp = &m4.x; float* vp = &v4.x; float* pq = &p4.x;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const float g = gp[i];
        const float e1 = b1 * mp[i] + (1.0f - b1) * g;
        const float e2 = b2 * vp[i] + (1.0f - b2) * g * g;
        pq[i] += -lr * e1 / (sqrtf(e2) + eps);
        mp[i] = e1; vp[i] = e2;
    }
    *reinterpret_cast<float4*>(param + p) = p4;
    *reinterpret_cast<float4*>(m + p) = m4;
    *reinterpret_cast<float4*>(v2 + p) = v4;
}

extern "C" int lgs_adam_update_chunk(float* param, const float* grad, float* exp_avg, float* exp_avg_sq,
                                     const int64_t* visible_index, const int* valid_length, int R, int C, int S, int A,
                                     double lr, double b1, double b2, double eps, void* stream)
{
    LGS_REQUIRE(S >= 1 && S <= 1024, "adamUpdate: chunk size %d unsupported", S);
    if (A == 0 || R == 0) return LGS_OK;
    const bool aligned = ((((uintptr_t)param | (uintptr_t)grad | (uintptr_t)exp_avg | (uintptr_t)exp_avg_sq) & 15) == 0) && S % 4 == 0 &&
                         S / 4 <= 128;
    if (aligned) {
        constexpr int ROWS = 8;
        adam_chunk_vec4_kernel<ROWS><<<dim3(A, lgs_cdiv(R, ROWS)), dim3(S / 4, ROWS), 0, (cudaStream_t)stream>>>(
            param, grad, exp_avg, exp_avg_sq, visible_index, valid_length, R, C, S, A, (float)lr, (float)b1, (float)b2, (float)eps);
        LGS_CHECK_LAUNCH("adam_chunk_vec4_kernel");
        return LGS_OK;
    }
    adam_chunk_kernel<<<dim3(A, R), S, 0, (cudaStream_t)stream>>>(param, grad, exp_avg, exp_avg_sq, visible_index, valid_length, C, S, A,
                                                                 (float)lr, (float)b1, (float)b2, (float)eps);
    LGS_CHECK_LAUNCH("adam_chunk_kernel");
    return LGS_OK;
}

__global__ void adam_primitive_kernel(float* __restrict__ param, const float* __restrict__ grad, float* __restrict__ m,
                                      float* __restrict__ v2, const int64_t* __restrict__ visible, int R, int N, float lr,
                                      float b1, float b2, float eps)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N || !visible[i]) return;
    for (int r = 0; r < R; r++) {
        size_t p = (size_t)r * N + i;
        float g = grad[p];
        float e1 = b1 * m[p] + (1.0f - b1) * g;
        float e2 = b2 * v2[p] + (1.0f - b2) * g * g;
        param[p] += -lr * e1 / (sqrtf(e2) + eps);
        m[p] = e1; v2[p] = e2;
    }
}

extern "C" int lgs_adam_update_primitive(float* param, const float* grad, float* exp_avg, float* exp_avg_sq,
                                         const int64_t* primitive_visible, int R, int N, double lr, double b1, double b2,
                                         double eps, void* stream)
{
    if (N == 0 || R == 0) return LGS_OK;
    adam_primitive_kernel<<<lgs_cdiv(N, 256), 256, 0, (cudaStream_t)stream>>>(param, grad, exp_avg, exp_avg_sq, primitive_visible, R, N,
                                                                           (float)lr, (float)b1, (float)b2, (float)eps);
    LGS_CHECK_LAUNCH("adam_primitive_kernel");
    return LGS_OK;
}

template <typename T, int OP>
__global__ void sparse_scatter_kernel(T* __restrict__ A, const T* __restrict__ B, const int64_t* __restrict__ ids,
                                      const int* __restrict__ valid, int chunks, int alloc_chunks)
{
    int src = blockIdx.x, e = blockIdx.y;
    if (src >= valid[0]) return;
    size_t ob = ((size_t)e * alloc_chunks + src) * blockDim.x + threadIdx.x;
    size_t oa = ((size_t)e * chunks + ids[src]) * blockDim.x + threadIdx.x;
    T b = B[ob];
    if (OP == 0) A[oa] += b;
    else if (OP == 1) A[oa] = min(A[oa], b);
    else A[oa] = max(A[oa], b);
}

// dtype: 0 float32, 1 int32, 2 float64, 3 int64, 4 int16, 5 int8, 6 uint8 (the reference dispatches AT_DISPATCH_ALL_TYPES,
// GR/compact.cu:1305); op: 0 add, 1 min, 2 max
extern "C" int lgs_sparse_chunk_op(void* A, const void* B, const int64_t* visible_chunk_ids, const int* visible_count, int dtype,
                                   int op, int ele_num, int chunks, int alloc_chunks, int chunk_size, void* stream)
{
    LGS_REQUIRE(chunk_size >= 1 && chunk_size <= 1024, "gpu_driven_pipeline_sparse_op: chunk_size %d exceeds max threads per block", chunk_size);
    LGS_REQUIRE(op >= 0 && op <= 2, "gpu_driven_pipeline_sparse_op: unsupported op %d (expected add, min, max)", op);
    LGS_REQUIRE(dtype >= 0 && dtype <= 6, "gpu_driven_pipeline_sparse_op: unsupported dtype code %d", dtype);
    if (alloc_chunks == 0 || ele_num == 0) return LGS_OK;
    dim3 grid(alloc_chunks, ele_num);
    cudaStream_t st = (cudaStream_t)stream;
    const auto scatter = [&](auto zero) {       // the element type is zero's type
        using T = decltype(zero);
        const auto launch = [&](auto o) {
            sparse_scatter_kernel<T, o><<<grid, chunk_size, 0, st>>>((T*)A, (const T*)B, visible_chunk_ids, visible_count, chunks,
                                                                      alloc_chunks);
        };
        if (op == 0) launch(std::integral_constant<int, 0>{});
        else if (op == 1) launch(std::integral_constant<int, 1>{});
        else launch(std::integral_constant<int, 2>{});
    };
    switch (dtype) {
        case 0: scatter(0.0f); break;
        case 1: scatter(0); break;
        case 2: scatter(0.0); break;
        case 3: scatter(0LL); break;
        case 4: scatter((short)0); break;
        case 5: scatter((signed char)0); break;
        default: scatter((unsigned char)0); break;
    }
    LGS_CHECK_LAUNCH("sparse_scatter_kernel");
    return LGS_OK;
}
