// optim.cu -- the optimizer step of the data-parallel path: ONE launch applies Adam to all six parameter tensors from the
// dense (all-reduced) gradient buffer.      replaces six adamUpdate launches per step (optimizer.py:14-44 ->
// GR/compact.cu:320-417), one per parameter group, each on a compacted gradient
//
// Semantics are the reference's sparse Adam (GR/compact.cu:320-344): no bias correction,
//     m = b1 m + (1-b1) g;  v = b2 v + (1-b2) g^2;  p -= lr m / (sqrt(v) + eps)
// and only chunks that were visible update (moments of the others do not decay).  With several views per step "visible"
// means visible in at least one view on any rank: every backward marks its visible chunks in a float row that is
// all-reduced together with the gradients (it is the tail of the same flat buffer).  The kernel also clears the
// gradient rows and the marks of the chunks it consumed, so the 236 B/Gaussian buffer never needs a separate memset.
// HBM-bound: 28 B (+4 B clear) per element and step.
#include "common.cuh"

namespace {

constexpr int NGROUP = 6;

struct AdamGroups {
    float* param[NGROUP];     // [rows_k, C, S] each
    int row0[NGROUP + 1];     // first row of each group inside the flat [rows, C, S] gradient / moment buffers
    float lr[NGROUP];
};

__global__ void mark_chunks_kernel(const int64_t* __restrict__ ids, const int* __restrict__ count, int A, float* __restrict__ touched)
{
    int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < A && j < count[0]) touched[ids[j]] = 1.0f;
}

// grid = chunks, block = S/4 threads (float4 along the chunk)
template <bool CLEAR>
__global__ void adam_dense_kernel(AdamGroups G, float* __restrict__ grad, float* __restrict__ m, float* __restrict__ v,
                                  float* __restrict__ touched, int C, int S, float b1, float b2, float eps)
{
    const int c = blockIdx.x;
    if (touched != nullptr && touched[c] == 0.0f) return;
    const size_t CS = (size_t)C * S;
    const size_t off = (size_t)c * S + 4 * threadIdx.x;
#pragma unroll
    for (int k = 0; k < NGROUP; k++) {          // static group index: G stays in the constant bank (no local copy of the struct)
        const float lr = G.lr[k];
        float* const pbase = G.param[k];
        for (int r = G.row0[k]; r < G.row0[k + 1]; r++) {
            const size_t f = (size_t)r * CS + off;
            float4 g4 = *reinterpret_cast<const float4*>(grad + f);
            float4 m4 = *reinterpret_cast<const float4*>(m + f);
            float4 v4 = *reinterpret_cast<const float4*>(v + f);
            float* pp = pbase + (size_t)(r - G.row0[k]) * CS + off;
            float4 p4 = *reinterpret_cast<const float4*>(pp);
            float* gp = &g4.x; float* mp = &m4.x; float* vp = &v4.x; float* pq = &p4.x;
#pragma unroll
            for (int i = 0; i < 4; i++) {
                float g = gp[i];
                float e1 = b1 * mp[i] + (1.0f - b1) * g;
                float e2 = b2 * vp[i] + (1.0f - b2) * g * g;
                pq[i] += -lr * e1 / (sqrtf(e2) + eps);
                mp[i] = e1; vp[i] = e2;
            }
            *reinterpret_cast<float4*>(m + f) = m4;
            *reinterpret_cast<float4*>(v + f) = v4;
            *reinterpret_cast<float4*>(pp) = p4;
            if (CLEAR) *reinterpret_cast<float4*>(grad + f) = make_float4(0.f, 0.f, 0.f, 0.f);
        }
    }
    if (CLEAR && touched != nullptr) {
        __syncthreads();
        if (threadIdx.x == 0) touched[c] = 0.0f;
    }
}

}  // namespace

/* touched[ids[j]] = 1 for j < min(A, *count)  (the visible chunks of one view) */
extern "C" int lgs_mark_visible_chunks(const int64_t* visible_chunk_id, const int* visible_chunks_num, int A, float* touched, void* stream)
{
    if (A <= 0) return LGS_OK;
    LGS_REQUIRE(visible_chunk_id && visible_chunks_num && touched, "mark_visible_chunks: null pointer");
    mark_chunks_kernel<<<lgs_cdiv(A, 256), 256, 0, (cudaStream_t)stream>>>(visible_chunk_id, visible_chunks_num, A, touched);
    LGS_CHECK_LAUNCH("mark_chunks_kernel");
    return LGS_OK;
}

extern "C" int lgs_adam_step_dense(float* const* params, const int* rows_per_param, const float* lr_per_param, float* grad,
                                   float* exp_avg, float* exp_avg_sq, float* touched, int C, int S, double b1, double b2, double eps,
                                   int clear_grad, void* stream)
{
    LGS_REQUIRE(params && rows_per_param && lr_per_param && grad && exp_avg && exp_avg_sq, "adam_step_dense: null pointer");
    LGS_REQUIRE(C >= 1 && S >= 4 && S % 4 == 0 && S <= 4096, "adam_step_dense: chunk size %d must be a multiple of 4 in 4..4096", S);
    AdamGroups G;
    G.row0[0] = 0;
    for (int k = 0; k < NGROUP; k++) {
        LGS_REQUIRE(params[k] != nullptr && rows_per_param[k] >= 1, "adam_step_dense: parameter group %d is empty", k);
        LGS_REQUIRE(((uintptr_t)params[k] & 15) == 0, "adam_step_dense: parameter %d is not 16-byte aligned", k);
        G.param[k] = params[k];
        G.row0[k + 1] = G.row0[k] + rows_per_param[k];
        G.lr[k] = lr_per_param[k];
    }
    LGS_REQUIRE((((uintptr_t)grad | (uintptr_t)exp_avg | (uintptr_t)exp_avg_sq) & 15) == 0, "adam_step_dense: buffers must be 16-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    lgs_with_flags([&](auto clear) {
        adam_dense_kernel<clear><<<C, S / 4, 0, st>>>(G, grad, exp_avg, exp_avg_sq, touched, C, S, (float)b1, (float)b2, (float)eps);
        return LGS_OK;
    }, clear_grad != 0);
    LGS_CHECK_LAUNCH("adam_dense_kernel");
    return LGS_OK;
}
