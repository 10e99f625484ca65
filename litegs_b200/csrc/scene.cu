// scene.cu -- chunk maintenance between optimisation epochs (SURVEY 8f rank 4): Morton codes for the spatial re-clustering,
// the permutation of every per-Gaussian row by the sorted order, and the chunk AABBs the frustum culling reads.
//                                  replaces the PyTorch passes of litegs/scene/point.py:22-154 and litegs/scene/cluster.py:29-46
// Not on the per-view hot path (the reference runs them every densification_interval epochs, trainer.py:103-106); they are
// HBM-bound single passes here instead of ~20 elementwise PyTorch kernels plus one indexing kernel per tensor.
#include "common.cuh"

// 3 x `bits` interleaved Morton code of each point, exactly as _gen_morton_code (point.py:38-81): fp32 normalisation
// ((p - min) / max(max - min, 1e-12)) * (2^bits - 1), truncation to integer, clamp, bit i of x/y/z to bits 3i, 3i+1, 3i+2.
__global__ void morton_kernel(const float* __restrict__ xyz, const float* __restrict__ lo, const float* __restrict__ hi, int N, int bits,
                              long long* __restrict__ codes)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const float scale = (float)((1ll << bits) - 1);
    unsigned long long q[3];
#pragma unroll
    for (int a = 0; a < 3; a++) {
        float denom = fmaxf(__fsub_rn(hi[a], lo[a]), 1e-12f);
        float nrm = __fmul_rn(__fdiv_rn(__fsub_rn(xyz[(size_t)a * N + i], lo[a]), denom), scale);
        long long v = (long long)nrm;                            // .long(): truncation toward zero
        v = v < 0 ? 0 : (v > (long long)scale ? (long long)scale : v);
        q[a] = (unsigned long long)v;
    }
    unsigned long long code = 0;
    for (int b = 0; b < bits; b++)
        code |= ((q[0] >> b) & 1ull) << (3 * b) | ((q[1] >> b) & 1ull) << (3 * b + 1) | ((q[2] >> b) & 1ull) << (3 * b + 2);
    codes[i] = (long long)code;
}

extern "C" int lgs_morton_codes(const float* xyz, const float* lo3, const float* hi3, int N, int bits, long long* codes, void* stream)
{
    LGS_REQUIRE(bits >= 1 && bits <= 21, "morton_codes: %d bits per axis not in 1..21", bits);
    if (N <= 0) return LGS_OK;
    morton_kernel<<<lgs_cdiv(N, 256), 256, 0, (cudaStream_t)stream>>>(xyz, lo3, hi3, N, bits, codes);
    LGS_CHECK_LAUNCH("morton_kernel");
    return LGS_OK;
}

// dst[r, j] = src[r, idx[j]] for every row r: ONE launch permutes all R rows of a [R, N] matrix (parameters, gradients and the
// two Adam moments are [rows, N] views of their storage), reading idx once per column.
__global__ void permute_rows_kernel(const float* __restrict__ src, const long long* __restrict__ idx, int R, int N, float* __restrict__ dst)
{
    int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= N) return;
    const size_t s = (size_t)idx[j];
    for (int r = blockIdx.y; r < R; r += gridDim.y) dst[(size_t)r * N + j] = src[(size_t)r * N + s];
}

extern "C" int lgs_permute_rows(const float* src, const long long* idx, int R, int N, float* dst, void* stream)
{
    LGS_REQUIRE(src != dst, "permute_rows: in-place permutation is not supported");
    if (R <= 0 || N <= 0) return LGS_OK;
    dim3 grid(lgs_cdiv(N, 256), R < 64 ? R : 64);
    permute_rows_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(src, idx, R, N, dst);
    LGS_CHECK_LAUNCH("permute_rows_kernel");
    return LGS_OK;
}

// Chunk AABBs (cluster.py:29-46): per Gaussian the half extent along each world axis is sqrt(2 ln 255) * sum_a |s_a R[a][k]|
// (the S.R rows scaled: GR/transform.cu:106-125), the chunk's box is the union of [p - e, p + e].  One CTA per chunk, the
// chunk's S Gaussians reduced through shared memory.  Inputs are the RAW parameters (log scale, unnormalised quaternion).
__global__ void cluster_aabb_kernel(const float* __restrict__ xyz, const float* __restrict__ scale, const float* __restrict__ rot, int C,
                                    int S, float* __restrict__ origin, float* __restrict__ extend)
{
    __shared__ float s_lo[3][32], s_hi[3][32];
    const int c = blockIdx.x, t = threadIdx.x;
    const size_t CS = (size_t)C * S;
    float lo[3] = { 3.4028235e38f, 3.4028235e38f, 3.4028235e38f }, hi[3] = { -3.4028235e38f, -3.4028235e38f, -3.4028235e38f };
    for (int s = t; s < S; s += blockDim.x) {
        const size_t i = (size_t)c * S + s;
        float q[4] = { rot[i], rot[CS + i], rot[2 * CS + i], rot[3 * CS + i] };
        float inv = 1.0f / sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);       // F.normalize(rot, dim=0), trainer.py:106
        const float r = q[0] * inv, x = q[1] * inv, y = q[2] * inv, z = q[3] * inv;
        const float R[9] = { 1 - 2 * (y * y + z * z), 2 * (x * y + r * z), 2 * (x * z - r * y),
                             2 * (x * y - r * z), 1 - 2 * (x * x + z * z), 2 * (y * z + r * x),
                             2 * (x * z + r * y), 2 * (y * z - r * x), 1 - 2 * (x * x + y * y) };
        const float sc[3] = { expf(scale[i]), expf(scale[CS + i]), expf(scale[2 * CS + i]) };
        const float k = 3.3290429115295410f;                     // sqrt(2 ln 255)
#pragma unroll
        for (int d = 0; d < 3; d++) {
            float e = (fabsf(sc[0] * R[0 * 3 + d]) + fabsf(sc[1] * R[1 * 3 + d]) + fabsf(sc[2] * R[2 * 3 + d])) * k;
            float p = xyz[(size_t)d * CS + i];
            lo[d] = fminf(lo[d], p - e); hi[d] = fmaxf(hi[d], p + e);
        }
    }
#pragma unroll
    for (int d = 0; d < 3; d++) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            lo[d] = fminf(lo[d], __shfl_xor_sync(0xffffffffu, lo[d], o));
            hi[d] = fmaxf(hi[d], __shfl_xor_sync(0xffffffffu, hi[d], o));
        }
        if ((t & 31) == 0) { s_lo[d][t >> 5] = lo[d]; s_hi[d][t >> 5] = hi[d]; }
    }
    __syncthreads();
    if (t < 3) {
        const int nw = (blockDim.x + 31) >> 5;
        float a = s_lo[t][0], b = s_hi[t][0];
        for (int w = 1; w < nw; w++) { a = fminf(a, s_lo[t][w]); b = fmaxf(b, s_hi[t][w]); }
        origin[(size_t)t * C + c] = (b + a) * 0.5f;
        extend[(size_t)t * C + c] = (b - a) * 0.5f;
    }
}

// Mip-Splatting's 3D smoothing filter (DESIGN.md section 1, "3D smoothing filter"), computed from the training cameras.
// Per Gaussian p and camera v, every op single-rounded and without contraction:
//   x/y/z_v = ((p0 V[0][c] + p1 V[1][c]) + p2 V[2][c]) + V[3][c]     (c = 0, 1, 2)
//   fx = (P[0][0] W) 0.5, fy = (P[1][1] H) 0.5, zc = max(z_v, 0.001), u = (x_v / zc) fx + W 0.5, w = (y_v / zc) fy + H 0.5
//   valid: z_v > 0.2 and (-0.15 W) <= u <= (1.15 W) and (-0.15 H) <= w <= (1.15 H)
//   dist = min(100000, z_v over the valid cameras), focal = max of fx over all cameras, f = (dist / focal) 0.4472136
// A Gaussian no camera sees gets the largest f of the seen ones (division and product by positive constants are monotone
// under rounding, so that is the f of the largest seen dist), or 0 when no Gaussian is seen.
constexpr int LGS_F3D_THREADS = 256;
constexpr int LGS_F3D_CAM_FLOATS = 20;     // V[0..3][0..2], fx, fy, W/2, H/2, the four screen bounds

__global__ void __launch_bounds__(LGS_F3D_THREADS) filter_3d_kernel(const float* __restrict__ xyz, int N, const float* __restrict__ view,
                                                                    const float* __restrict__ proj, const int* __restrict__ hw, int V,
                                                                    float* __restrict__ out, unsigned* __restrict__ max_bits)
{
    __shared__ float s_cam[LGS_F3D_THREADS][LGS_F3D_CAM_FLOATS + 1];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = i < N;
    const float p0 = live ? xyz[i] : 0.f, p1 = live ? xyz[(size_t)N + i] : 0.f, p2 = live ? xyz[2 * (size_t)N + i] : 0.f;
    float dist = 100000.0f, focal = 0.0f;
    bool seen = false;
    for (int base = 0; base < V; base += LGS_F3D_THREADS) {
        const int v = base + threadIdx.x;
        if (v < V) {
            const float* Vm = view + (size_t)v * 16;
            const float H = (float)hw[2 * v], W = (float)hw[2 * v + 1];
            float* c = s_cam[threadIdx.x];
#pragma unroll
            for (int r = 0; r < 4; r++)
#pragma unroll
                for (int k = 0; k < 3; k++) c[r * 3 + k] = Vm[r * 4 + k];
            c[12] = __fmul_rn(__fmul_rn(proj[(size_t)v * 16], W), 0.5f);
            c[13] = __fmul_rn(__fmul_rn(proj[(size_t)v * 16 + 5], H), 0.5f);
            c[14] = __fmul_rn(W, 0.5f); c[15] = __fmul_rn(H, 0.5f);
            c[16] = __fmul_rn(-0.15f, W); c[17] = __fmul_rn(1.15f, W);
            c[18] = __fmul_rn(-0.15f, H); c[19] = __fmul_rn(1.15f, H);
        }
        __syncthreads();
        const int nb = min(LGS_F3D_THREADS, V - base);
        for (int j = 0; j < nb; j++) {
            const float* c = s_cam[j];
            focal = fmaxf(focal, c[12]);
            const float z = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(p0, c[2]), __fmul_rn(p1, c[5])), __fmul_rn(p2, c[8])), c[11]);
            if (!(z > 0.2f)) continue;
            const float x = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(p0, c[0]), __fmul_rn(p1, c[3])), __fmul_rn(p2, c[6])), c[9]);
            const float y = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(p0, c[1]), __fmul_rn(p1, c[4])), __fmul_rn(p2, c[7])), c[10]);
            const float zc = fmaxf(z, 0.001f);
            const float u = __fadd_rn(__fmul_rn(__fdiv_rn(x, zc), c[12]), c[14]);
            const float w = __fadd_rn(__fmul_rn(__fdiv_rn(y, zc), c[13]), c[15]);
            if (u >= c[16] && u <= c[17] && w >= c[18] && w <= c[19]) {
                dist = fminf(dist, z);
                seen = true;
            }
        }
        __syncthreads();
    }
    const float f = __fmul_rn(__fdiv_rn(dist, focal), 0.4472136f);
    // seen f > 0 (dist > 0.2): positive floats order like their bit patterns, so the integer maximum is exact and order-free
    const unsigned wmax = __reduce_max_sync(0xffffffffu, (live && seen) ? __float_as_uint(f) : 0u);
    if ((threadIdx.x & 31) == 0 && wmax != 0u) atomicMax(max_bits, wmax);
    if (live) out[i] = seen ? f : -1.0f;
}

// fills the unseen Gaussians (marked -1 by filter_3d_kernel) with the largest seen f
__global__ void filter_3d_fill_kernel(float* __restrict__ out, int N, const unsigned* __restrict__ max_bits)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < N && out[i] < 0.0f) out[i] = __uint_as_float(*max_bits);
}

extern "C" int lgs_filter_3d(const float* position, int C, int S, const float* view, const float* proj, const int* hw, int V,
                             float* filter_3d, void* stream)
{
    LGS_REQUIRE(C >= 0 && S >= 1 && V >= 1, "filter_3d: bad sizes C=%d S=%d V=%d", C, S, V);
    LGS_REQUIRE((long long)C * S < (1ll << 31), "filter_3d: %lld Gaussians exceed the 32-bit index", (long long)C * S);
    const int N = C * S;
    if (N == 0) return LGS_OK;
    cudaStream_t st = (cudaStream_t)stream;
    unsigned* max_bits = nullptr;
    LGS_CUDA(cudaMallocAsync((void**)&max_bits, sizeof(unsigned), st));
    LGS_CUDA(cudaMemsetAsync(max_bits, 0, sizeof(unsigned), st));
    filter_3d_kernel<<<lgs_cdiv(N, LGS_F3D_THREADS), LGS_F3D_THREADS, 0, st>>>(position, N, view, proj, hw, V, filter_3d, max_bits);
    LGS_CHECK_LAUNCH("filter_3d_kernel");
    filter_3d_fill_kernel<<<lgs_cdiv(N, 256), 256, 0, st>>>(filter_3d, N, max_bits);
    LGS_CHECK_LAUNCH("filter_3d_fill_kernel");
    LGS_CUDA(cudaFreeAsync(max_bits, st));
    return LGS_OK;
}

extern "C" int lgs_cluster_aabb(const float* xyz, const float* scale, const float* rot, int C, int S, float* origin, float* extend,
                                void* stream)
{
    LGS_REQUIRE(S >= 1, "cluster_aabb: bad chunk size %d", S);
    if (C <= 0) return LGS_OK;
    int threads = S >= 1024 ? 1024 : ((S + 31) / 32) * 32;
    cluster_aabb_kernel<<<C, threads, 0, (cudaStream_t)stream>>>(xyz, scale, rot, C, S, origin, extend);
    LGS_CHECK_LAUNCH("cluster_aabb_kernel");
    return LGS_OK;
}
