// nvls.cu -- the data path's only exchange, the per-step all-reduce of the dense gradient buffer (SURVEY 8e), as ONE kernel over
// the NVSwitch multicast address of the buffer (NVLink SHARP): every rank owns 1/world of the buffer, pulls the switch-reduced
// sum of its slice from all replicas with multimem.ld_reduce and pushes it back to all replicas with multimem.st -- "two-shot"
// all-reduce with the reduction done inside the switch, 16 bytes per instruction.  Per GPU and direction the links carry the
// buffer once (+1/world), the NVLS algorithm NCCL uses; what the own kernel removes is the protocol / channel overhead of the
// library call.
//
// The buffer must be symmetric memory mapped for multicast (torch.distributed._symmetric_memory: empty + rendezvous ->
// multicast_ptr); the caller brackets the launch with cross-GPU barriers on the same stream (all replicas complete before the
// reduction reads them; all slices broadcast before anyone reads the result).  Every element is reduced exactly once, by its
// owner, so all replicas receive bit-identical sums.  The reference has no multi-GPU path at all (SURVEY fact 3).
#include "common.cuh"

#define LGS_NVLS_UNROLL 4
__global__ void __launch_bounds__(512) nvls_allreduce_f32_kernel(float* __restrict__ mc, size_t n4, int rank, int world)
{
    const size_t per = (n4 + (size_t)world - 1) / (size_t)world;
    const size_t lo = (size_t)rank * per;
    const size_t hi = lo + per < n4 ? lo + per : n4;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    // LGS_NVLS_UNROLL independent switch reductions in flight per thread before the first store: the round trip through the
    // switch is long, the loop is otherwise a dependent load -> store chain
    for (size_t i0 = lo + (size_t)blockIdx.x * blockDim.x + threadIdx.x; i0 < hi; i0 += stride * LGS_NVLS_UNROLL) {
        float v[LGS_NVLS_UNROLL][4];
#pragma unroll
        for (int u = 0; u < LGS_NVLS_UNROLL; u++) {
            const size_t i = i0 + (size_t)u * stride;
            if (i < hi)
                asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
                             : "=f"(v[u][0]), "=f"(v[u][1]), "=f"(v[u][2]), "=f"(v[u][3]) : "l"(mc + 4 * i) : "memory");
        }
#pragma unroll
        for (int u = 0; u < LGS_NVLS_UNROLL; u++) {
            const size_t i = i0 + (size_t)u * stride;
            if (i < hi)
                asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(mc + 4 * i), "f"(v[u][0]), "f"(v[u][1]),
                             "f"(v[u][2]), "f"(v[u][3]) : "memory");
        }
    }
}

// multicast_ptr: the multicast (NVSwitch) address of the symmetric buffer; n_floats: its length, a multiple of 4; ctas: grid size
// (0 = default).  The launch itself neither waits for nor signals the other ranks.
extern "C" int lgs_nvls_allreduce_f32(float* multicast_ptr, size_t n_floats, int rank, int world, int ctas, void* stream)
{
    LGS_REQUIRE(multicast_ptr != nullptr && world >= 1 && rank >= 0 && rank < world, "nvls_allreduce: bad arguments (rank %d of %d)", rank, world);
    LGS_REQUIRE(n_floats % 4 == 0 && ((uintptr_t)multicast_ptr & 15) == 0, "nvls_allreduce: length %zu / address not 16-byte granular", n_floats);
    if (n_floats == 0) return LGS_OK;
    if (ctas <= 0) ctas = 128;
    nvls_allreduce_f32_kernel<<<ctas, 512, 0, (cudaStream_t)stream>>>(multicast_ptr, n_floats / 4, rank, world);
    LGS_CHECK_LAUNCH("nvls_allreduce_f32_kernel");
    return LGS_OK;
}
