// geometry.cu -- depth-normal consistency on the fused path's depth, transmittance and normal images (ours; DESIGN.md section 1,
// "Depth-normal consistency"): the normal n_d taken from the unprojected expected depth by central differences, and the loss
// L = weight / (H W) sum_p (1 - n_d . N_p / |N_p|) with its exact gradient with respect to D, T and N, in one pass.
//
// Gather form, no atomics.  A CTA owns a TX x TY tile of output pixels and
//   1. stages alpha = 1 - T and ED = D / alpha of the tile plus a 2-pixel halo in shared memory;
//   2. for every pixel p of the tile plus a 1-pixel halo forms a, b, c = b x a, n_d and, with the loss, the gradient of l_p with
//      respect to a and b (ga, gb: 6 floats, shared memory); tile pixels also write n_d, dL/dN and their share of the loss;
//   3. every tile pixel q collects dL/dED_q = r_q . (ga(q-x) - ga(q+x) + gb(q-y) - gb(q+y)) from its four neighbours and
//      writes dL/dD = dL/dED / alpha and dL/dT = dL/dD ED.
// The inputs are read through row (and channel) strides, so the [..., :H, :W] views of padded planes need no copy; proj[0][0]
// and proj[1][1] are read on the device, so nothing synchronises with the host.
#include "common.cuh"

namespace {

constexpr int TX = 64, TY = 16;           // output tile
constexpr int NT = 256;                   // threads per CTA
constexpr int EX = TX + 4, EY = TY + 4;   // ED and alpha: the tile and a 2-pixel halo
constexpr int GX = TX + 2, GY = TY + 2;   // per-pixel stencil terms: the tile and a 1-pixel halo

struct V3 { float x, y, z; };

__device__ __forceinline__ V3 cross(V3 p, V3 q) { return { p.y * q.z - p.z * q.y, p.z * q.x - p.x * q.z, p.x * q.y - p.y * q.x }; }
__device__ __forceinline__ float dot(V3 p, V3 q) { return p.x * q.x + p.y * q.y + p.z * q.z; }

// GRAD: write d_depth, d_trans, d_normal.  The n_d map and the block sums are nullable; normal is needed for GRAD or block sums.
// The minimum of 4 CTAs per SM only caps registers at 64: without it ptxas gives the map-only form 32 registers and a spill.
template <bool NMAP, bool GRAD>
__global__ void __launch_bounds__(NT, 4) depth_normal_kernel(const float* __restrict__ D, int ds, const float* __restrict__ T, int ts,
                                                          const float* __restrict__ N, int ns, int ncs, const float* __restrict__ proj,
                                                          int H, int W, float alpha_min, float scale, float* __restrict__ nd,
                                                          float* __restrict__ dD, float* __restrict__ dT, float* __restrict__ dN,
                                                          float* __restrict__ block_sums)
{
    __shared__ float sE[EY][EX], sA[EY][EX];
    __shared__ float sG[GRAD ? 6 : 1][GRAD ? GY : 1][GRAD ? GX : 1];     // ga (0..2) and gb (3..5)
    const int t = threadIdx.x;
    const int u0 = (int)blockIdx.x * TX, v0 = (int)blockIdx.y * TY;
    const size_t HW = (size_t)H * W;
    const bool loss = block_sums != nullptr;
    const float fx = (proj[0] * (float)W) * 0.5f, fy = (proj[5] * (float)H) * 0.5f;
    const float hx = 2.0f / fx, hy = 2.0f / fy;               // r(u+1) - r(u-1) and r(v+1) - r(v-1)
    const float cx = 0.5f * (float)W, cy = 0.5f * (float)H;
    auto rx = [&](int u) { return ((float)u + 0.5f - cx) / fx; };
    auto ry = [&](int v) { return ((float)v + 0.5f - cy) / fy; };

    // 1. alpha and ED; alpha = 0 outside the image, which no alpha_min >= 0 accepts
    for (int i = t; i < EX * EY; i += NT) {
        const int y = i / EX, x = i - y * EX;
        const int u = u0 - 2 + x, v = v0 - 2 + y;
        float a = 0.0f, e = 0.0f;
        if (u >= 0 && u < W && v >= 0 && v < H) {
            a = 1.0f - T[(size_t)v * ts + u];
            if (a > alpha_min) e = D[(size_t)v * ds + u] / a;
        }
        sA[y][x] = a;
        sE[y][x] = e;
    }
    __syncthreads();

    // 2. n_d, the loss, dL/dN and the stencil terms ga, gb
    float lsum = 0.0f;
    for (int i = t; i < GX * GY; i += NT) {
        const int y = i / GX, x = i - y * GX;
        const int u = u0 - 1 + x, v = v0 - 1 + y;
        const int ey = y + 1, ex = x + 1;                     // p in sE / sA
        const bool in_tile = x >= 1 && x <= TX && y >= 1 && y <= TY && u < W && v < H;
        bool m = u >= 1 && u <= W - 2 && v >= 1 && v <= H - 2 && sA[ey][ex] > alpha_min && sA[ey][ex - 1] > alpha_min &&
                 sA[ey][ex + 1] > alpha_min && sA[ey - 1][ex] > alpha_min && sA[ey + 1][ex] > alpha_min;
        V3 a = {}, b = {}, n = {}, ga = {}, gb = {};
        float ic = 0.0f;
        if (m) {
            const float eL = sE[ey][ex - 1], eR = sE[ey][ex + 1], eT = sE[ey - 1][ex], eB = sE[ey + 1][ex];
            const float dx = eR - eL, dy = eB - eT;
            a = { dx * rx(u - 1) + eR * hx, dx * ry(v), dx };
            b = { dy * rx(u), dy * ry(v - 1) + eB * hy, dy };
            const V3 c = cross(b, a);
            const float cc = dot(c, c);
            m = cc > 0.0f;
            if (m) {
                ic = 1.0f / sqrtf(cc);
                n = { c.x * ic, c.y * ic, c.z * ic };
            }
        }
        if (NMAP && in_tile) {
            const size_t o = (size_t)v * W + u;
            nd[o] = n.x; nd[HW + o] = n.y; nd[2 * HW + o] = n.z;
        }
        V3 gN = {};
        if (m && (GRAD || (loss && in_tile))) {
            const size_t o = (size_t)v * ns + u;
            const V3 q = { N[o], N[ncs + o], N[2 * (size_t)ncs + o] };
            const float nn = dot(q, q);
            if (nn > 1e-12f) {
                const float iN = 1.0f / sqrtf(nn);
                const V3 mq = { q.x * iN, q.y * iN, q.z * iN };
                const float cs = dot(n, mq);
                if (in_tile) lsum += 1.0f - cs;
                if (GRAD) {
                    const float sN = scale * iN, sc = scale * ic;
                    gN = { sN * (cs * mq.x - n.x), sN * (cs * mq.y - n.y), sN * (cs * mq.z - n.z) };
                    const V3 gc = { sc * (cs * n.x - mq.x), sc * (cs * n.y - mq.y), sc * (cs * n.z - mq.z) };
                    ga = cross(gc, b);
                    gb = cross(a, gc);
                }
            }
        }
        if (GRAD) {
            if (in_tile) {
                const size_t o = (size_t)v * W + u;
                dN[o] = gN.x; dN[HW + o] = gN.y; dN[2 * HW + o] = gN.z;
            }
            sG[0][y][x] = ga.x; sG[1][y][x] = ga.y; sG[2][y][x] = ga.z;
            sG[3][y][x] = gb.x; sG[4][y][x] = gb.y; sG[5][y][x] = gb.z;
        }
    }

    // 3. dL/dED of every tile pixel from its four neighbours' terms
    if (GRAD) {
        __syncthreads();
        for (int i = t; i < TX * TY; i += NT) {
            const int y = i / TX, x = i - y * TX;
            const int u = u0 + x, v = v0 + y;
            if (u >= W || v >= H) continue;
            const int gy = y + 1, gx = x + 1;
            float G[3];
#pragma unroll
            for (int k = 0; k < 3; k++)
                G[k] = (sG[k][gy][gx - 1] - sG[k][gy][gx + 1]) + (sG[3 + k][gy - 1][gx] - sG[3 + k][gy + 1][gx]);
            const float gE = (G[0] * rx(u) + G[1] * ry(v)) + G[2];
            const float a = sA[y + 2][x + 2];
            float gd = 0.0f, gt = 0.0f;
            if (a > alpha_min) {
                gd = gE / a;
                gt = gd * sE[y + 2][x + 2];
            }
            const size_t o = (size_t)v * W + u;
            dD[o] = gd;
            dT[o] = gt;
        }
    }

    if (loss) {
        __shared__ float s_part[NT / 32];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) lsum += __shfl_xor_sync(0xffffffffu, lsum, o);
        if ((t & 31) == 0) s_part[t >> 5] = lsum;
        __syncthreads();
        if (t == 0) {
            float s = 0.0f;
#pragma unroll
            for (int k = 0; k < NT / 32; k++) s += s_part[k];
            block_sums[blockIdx.y * gridDim.x + blockIdx.x] = s;
        }
    }
}

}  // namespace

extern "C" int lgs_depth_normal_num_block_sums(int H, int W, int* count)
{
    LGS_REQUIRE(H >= 1 && W >= 1 && count != nullptr, "depth_normal_num_block_sums: bad arguments");
    *count = ((H + TY - 1) / TY) * ((W + TX - 1) / TX);
    return LGS_OK;
}

extern "C" int lgs_depth_normal(const float* depth, int depth_row_stride, const float* trans, int trans_row_stride, const float* normal,
                                int normal_row_stride, int normal_channel_stride, const float* proj, int H, int W, float alpha_min,
                                float grad_scale, float* n_d, float* d_depth, float* d_trans, float* d_normal, float* block_sums,
                                void* stream)
{
    LGS_REQUIRE(H >= 1 && W >= 1, "depth_normal: bad shape [%d,%d]", H, W);
    LGS_REQUIRE(depth != nullptr && trans != nullptr && proj != nullptr, "depth_normal: null depth, transmittance or projection");
    LGS_REQUIRE(depth_row_stride >= W && trans_row_stride >= W, "depth_normal: row strides must be at least W = %d", W);
    LGS_REQUIRE(alpha_min >= 0.0f && alpha_min < 1.0f, "depth_normal: alpha_min = %g outside [0, 1)", (double)alpha_min);
    const bool grad = d_depth != nullptr;
    LGS_REQUIRE(grad == (d_trans != nullptr) && grad == (d_normal != nullptr), "depth_normal: the three gradients come together");
    LGS_REQUIRE(n_d != nullptr || grad || block_sums != nullptr, "depth_normal: nothing to compute");
    if (grad || block_sums != nullptr) {
        LGS_REQUIRE(normal != nullptr, "depth_normal: the loss and its gradient need the normal image");
        LGS_REQUIRE(normal_row_stride >= W && (size_t)normal_channel_stride >= (size_t)(H - 1) * normal_row_stride + W,
                    "depth_normal: bad normal strides (%d, %d) for [%d,%d]", normal_channel_stride, normal_row_stride, H, W);
    }
    cudaStream_t st = (cudaStream_t)stream;
    dim3 grid((W + TX - 1) / TX, (H + TY - 1) / TY);
    lgs_with_flags([&](auto nmap, auto g) {
        depth_normal_kernel<nmap, g><<<grid, NT, 0, st>>>(depth, depth_row_stride, trans, trans_row_stride, normal, normal_row_stride,
                                                          normal_channel_stride, proj, H, W, alpha_min, grad_scale, n_d, d_depth, d_trans,
                                                          d_normal, block_sums);
        return LGS_OK;
    }, n_d != nullptr, grad);
    LGS_CHECK_LAUNCH("depth_normal_kernel");
    return LGS_OK;
}
