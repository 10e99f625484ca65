// ssim.cu -- fused SSIM / L1+SSIM loss maps and their backward: the step either side of the rasterizer in a
// training iteration (consumes the rendered image, produces dL/dimage).
// replaces fused_ssim/ssim.cu:64-274, 277-437 (SSIM), 528-712, 719-850 (L1 + SSIM loss) and their hosts :444-524, 855-942.
//
// Same maths as the reference (11-tap sigma-1.5 Gaussian, zero padding, separable, per channel; the partial derivatives
// dm/dmu1, dm/dsigma1^2, dm/dsigma12 are saved by the forward and filtered again by the backward), different schedule.
// The reference stages a 26x26 window per 16x16 tile and keeps a 5-channel intermediate image in shared memory; that costs
// ~130 shared-memory accesses and ~440 issued instructions per output.  Here a CTA is a band of 128 columns x 32 rows and every thread streams DOWN
// one column:
//   * vertical pass in registers, straight from global memory (coalesced across the warp, 11 rows of loads in flight):
//     each incoming row is scattered into the 11 pending output rows of a register ring (statically indexed: the row loop
//     is unrolled by 11), so no intermediate image exists;
//   * when a ring slot completes, the 4 vertically filtered moments of that row go to a double-buffered 2 KB row buffer
//     (one __syncthreads per row) and each thread finishes its own pixel with the horizontal pass (44 conflict-free LDS);
//   * 4 moments instead of 5: SSIM only needs sigma1^2 + sigma2^2, so x^2 + y^2 is filtered as ONE image.
// ~190 instructions and ~48 shared-memory accesses per output, ~100 registers, 2 KB of shared memory per CTA.
// The loss map itself is optional: the training path only needs its mean, so the kernel can emit one partial sum per
// CTA instead (summed on the host side in a fixed order -> deterministic).
#include "common.cuh"

namespace {

constexpr int CT = 128;                 // threads = columns per CTA (incl. 2 x 5 halo columns)
constexpr int HALO = 5;
constexpr int CO = CT - 2 * HALO;       // 118 output columns per CTA
#ifndef LGS_SSIM_BH
#define LGS_SSIM_BH 32
#endif
constexpr int BH = LGS_SSIM_BH;         // output rows per CTA
constexpr int RIN = BH + 2 * HALO;      // input rows a thread streams

__device__ __forceinline__ float gauss(int k)
{
    // fused_ssim/ssim.cu:12-24 (normalised exp(-(k-5)^2 / 4.5), rounded to fp32)
    constexpr float G[11] = { 0.001028380123898387f, 0.0075987582094967365f, 0.036000773310661316f, 0.10936068743467331f,
                              0.21300552785396576f,  0.26601171493530273f,   0.21300552785396576f,  0.10936068743467331f,
                              0.036000773310661316f, 0.0075987582094967365f, 0.001028380123898387f };
    return G[k];
}

__device__ __forceinline__ float rcp_approx(float x)
{
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

// L1: loss map w (1 - ssim) + (1 - w) |x - y| instead of the ssim map.   TRAIN: write the three partials.
template <bool L1, bool TRAIN>
__global__ void __launch_bounds__(CT) ssim_forward_kernel(const float* __restrict__ img1, const float* __restrict__ img2, int H, int W,
                                                          float C1, float C2, float ssim_weight, float* __restrict__ map,
                                                          float* __restrict__ dm_dmu1, float* __restrict__ dm_dsigma1_sq,
                                                          float* __restrict__ dm_dsigma12, float* __restrict__ block_sums)
{
    constexpr int NM = 4;                                  // x, y, x^2 + y^2, x y
    __shared__ float rowbuf[2][NM][CT];
    const size_t plane = (size_t)blockIdx.z * H * W;
    const float* X = img1 + plane;
    const float* Y = img2 + plane;
    const int t = threadIdx.x;
    const int gx = (int)blockIdx.x * CO - HALO + t;        // this thread's column
    const int y0 = (int)blockIdx.y * BH;                   // first output row
    const bool col_in = gx >= 0 && gx < W;
    const bool col_out = t >= HALO && t < CT - HALO && gx < W;
    float acc[11][NM];
    float l1v[11];
#pragma unroll
    for (int i = 0; i < 11; i++) {
        l1v[i] = 0.0f;
#pragma unroll
        for (int m = 0; m < NM; m++) acc[i][m] = 0.0f;
    }
    float lsum = 0.0f;
    int emitted = 0;
    for (int r0 = 0; r0 < RIN; r0 += 11) {
        float xs[11], ys[11];
#pragma unroll
        for (int i = 0; i < 11; i++) {                     // 11 rows of loads in flight
            const int gy = y0 - HALO + r0 + i;
            const bool in = col_in && r0 + i < RIN && gy >= 0 && gy < H;
            xs[i] = in ? X[(size_t)gy * W + gx] : 0.0f;
            ys[i] = in ? Y[(size_t)gy * W + gx] : 0.0f;
        }
#pragma unroll
        for (int i = 0; i < 11; i++) {
            if (r0 + i < RIN) {                            // uniform across the CTA
                const float x = xs[i], y = ys[i];
                const float q[NM] = { x, y, fmaf(x, x, y * y), x * y };
                if (L1) l1v[i] = fabsf(x - y);
                // input row r = r0 + i feeds output rows r - j with tap j; output row o lives in slot o % 11
#pragma unroll
                for (int j = 0; j < 11; j++) {
                    const int slot = (i - j + 11) % 11;
#pragma unroll
                    for (int m = 0; m < NM; m++) acc[slot][m] = fmaf(gauss(j), q[m], acc[slot][m]);
                }
                // slot (i + 1) % 11 now holds output row o = r - 10: complete if o >= 0, otherwise the partial sums of a
                // row above the band, to be discarded; either way the slot restarts at zero for output row r + 1
                float done[NM];
#pragma unroll
                for (int m = 0; m < NM; m++) { done[m] = acc[(i + 1) % 11][m]; acc[(i + 1) % 11][m] = 0.0f; }
                if (r0 + i >= 10) {
                    const int buf = emitted & 1;
#pragma unroll
                    for (int m = 0; m < NM; m++) rowbuf[buf][m][t] = done[m];
                    __syncthreads();
                    const int gy = y0 + r0 + i - 10;
                    if (col_out && gy < H) {
                        float mom[NM];
#pragma unroll
                        for (int m = 0; m < NM; m++) {
                            float a = gauss(0) * rowbuf[buf][m][t - HALO];
#pragma unroll
                            for (int k = 1; k < 11; k++) a = fmaf(gauss(k), rowbuf[buf][m][t - HALO + k], a);
                            mom[m] = a;
                        }
                        const float mu1 = mom[0], mu2 = mom[1];
                        const float mu1_sq = mu1 * mu1, mu2_sq = mu2 * mu2;
                        const float A = mu1_sq + mu2_sq + C1;
                        const float B = (mom[2] - mu1_sq - mu2_sq) + C2;           // sigma1^2 + sigma2^2 + C2
                        const float sigma12 = mom[3] - mu1 * mu2;
                        const float C = 2.0f * mu1 * mu2 + C1, D = 2.0f * sigma12 + C2;
                        const float iA = rcp_approx(A), iB = rcp_approx(B);       // MUFU.RCP, 1 ulp: A, B >= C1, C2 > 0
                        const float iAB = iA * iB;
                        const float val = (C * D) * iAB;
                        float out = val;
                        if (L1) out = ssim_weight * (1.0f - val) + (1.0f - ssim_weight) * l1v[(i + 6) % 11];   // centre row r - 5
                        const size_t gi = plane + (size_t)gy * W + gx;
                        if (map != nullptr) map[gi] = out;
                        lsum += out;
                        if (TRAIN) {
                            // fused_ssim/ssim.cu:258-268 with the common factor 1/(A B) pulled out
                            dm_dmu1[gi] = 2.0f * iAB * (mu2 * (D - C) + mu1 * C * D * (iB - iA));
                            dm_dsigma1_sq[gi] = -(C * D) * iAB * iB;
                            dm_dsigma12[gi] = 2.0f * C * iAB;
                        }
                    }
                    emitted++;
                }
            }
        }
    }
    if (block_sums != nullptr) {
        __shared__ float s_part[CT / 32];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) lsum += __shfl_xor_sync(0xffffffffu, lsum, o);
        if ((t & 31) == 0) s_part[t >> 5] = lsum;
        __syncthreads();
        if (t == 0) {
            float s = 0.0f;
#pragma unroll
            for (int k = 0; k < CT / 32; k++) s += s_part[k];
            block_sums[((size_t)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x] = s;
        }
    }
}

// UNIFORM: dL_dmap == nullptr, the upstream gradient is the constant `chain` (loss = mean of the map): one load stream
// and 22 registers fewer than with a per-pixel upstream gradient
template <bool L1, bool UNIFORM>
__global__ void __launch_bounds__(CT) ssim_backward_kernel(const float* __restrict__ img1, const float* __restrict__ img2,
                                                           const float* __restrict__ dL_dmap, float chain,
                                                           const float* __restrict__ dm_dmu1, const float* __restrict__ dm_dsigma1_sq,
                                                           const float* __restrict__ dm_dsigma12, int H, int W, float ssim_weight,
                                                           float* __restrict__ dL_dimg1)
{
    constexpr int NM = 3;
    __shared__ float rowbuf[2][NM][CT];
    const size_t plane = (size_t)blockIdx.z * H * W;
    const int t = threadIdx.x;
    const int gx = (int)blockIdx.x * CO - HALO + t;
    const int y0 = (int)blockIdx.y * BH;
    const bool col_in = gx >= 0 && gx < W;
    const bool col_out = t >= HALO && t < CT - HALO && gx < W;
    const float scale = L1 ? -ssim_weight : 1.0f;                  // d loss / d ssim  (fused_ssim/ssim.cu:775-779)
    float acc[11][NM];
    float cv[UNIFORM ? 1 : 11];                                     // upstream gradient of the last 11 input rows
#pragma unroll
    for (int i = 0; i < 11; i++) {
        if (!UNIFORM) cv[i] = 0.0f;
#pragma unroll
        for (int m = 0; m < NM; m++) acc[i][m] = 0.0f;
    }
    int emitted = 0;
    for (int r0 = 0; r0 < RIN; r0 += 11) {
        float q[11][NM], cn[UNIFORM ? 1 : 11];
#pragma unroll
        for (int i = 0; i < 11; i++) {
            const int gy = y0 - HALO + r0 + i;
            const bool in = col_in && r0 + i < RIN && gy >= 0 && gy < H;
            const size_t gi = plane + (size_t)(in ? gy : 0) * W + (in ? gx : 0);
            const float c = UNIFORM ? chain : (in ? dL_dmap[gi] : 0.0f);
            if (!UNIFORM) cn[i] = c;
            q[i][0] = in ? dm_dmu1[gi] * (scale * c) : 0.0f;
            q[i][1] = in ? dm_dsigma1_sq[gi] * (scale * c) : 0.0f;
            q[i][2] = in ? dm_dsigma12[gi] * (scale * c) : 0.0f;
        }
#pragma unroll
        for (int i = 0; i < 11; i++) {
            if (r0 + i < RIN) {
                if (!UNIFORM) cv[i] = cn[i];                        // slot i is free: its row (r - 11) was last used 6 rows ago
#pragma unroll
                for (int j = 0; j < 11; j++) {
                    const int slot = (i - j + 11) % 11;
#pragma unroll
                    for (int m = 0; m < NM; m++) acc[slot][m] = fmaf(gauss(j), q[i][m], acc[slot][m]);
                }
                float done[NM];
#pragma unroll
                for (int m = 0; m < NM; m++) { done[m] = acc[(i + 1) % 11][m]; acc[(i + 1) % 11][m] = 0.0f; }
                if (r0 + i >= 10) {
                    const int buf = emitted & 1;
#pragma unroll
                    for (int m = 0; m < NM; m++) rowbuf[buf][m][t] = done[m];
                    __syncthreads();
                    const int gy = y0 + r0 + i - 10;
                    if (col_out && gy < H) {
                        float s[NM];
#pragma unroll
                        for (int m = 0; m < NM; m++) {
                            float a = gauss(0) * rowbuf[buf][m][t - HALO];
#pragma unroll
                            for (int k = 1; k < 11; k++) a = fmaf(gauss(k), rowbuf[buf][m][t - HALO + k], a);
                            s[m] = a;
                        }
                        const size_t gi = plane + (size_t)gy * W + gx;
                        const float p1 = img1[gi], p2 = img2[gi];
                        float g = s[0] + (2.0f * p1) * s[1] + p2 * s[2];                   // fused_ssim/ssim.cu:417-421
                        if (L1) {
                            const float sg = (p1 == p2) ? 0.0f : copysignf(1.0f, p1 - p2);  // fused_ssim/ssim.cu:840-841
                            g += (1.0f - ssim_weight) * sg * (UNIFORM ? chain : cv[UNIFORM ? 0 : (i + 6) % 11]);   // upstream of the centre row r - 5
                        }
                        dL_dimg1[gi] = g;
                    }
                    emitted++;
                }
            }
        }
    }
}

}  // namespace

/* number of per-CTA partial sums lgs_ssim_forward writes for this shape */
extern "C" int lgs_ssim_num_block_sums(int B, int CH, int H, int W, int* count)
{
    LGS_REQUIRE(B >= 1 && CH >= 1 && H >= 1 && W >= 1 && count != nullptr, "ssim_num_block_sums: bad arguments");
    *count = B * CH * ((H + BH - 1) / BH) * ((W + CO - 1) / CO);
    return LGS_OK;
}

extern "C" int lgs_ssim_forward(const float* img1, const float* img2, int B, int CH, int H, int W, float C1, float C2, int l1_mode,
                                float ssim_weight, float* map, float* dm_dmu1, float* dm_dsigma1_sq, float* dm_dsigma12,
                                float* block_sums, void* stream)
{
    LGS_REQUIRE(B >= 1 && CH >= 1 && H >= 1 && W >= 1, "ssim_forward: bad shape [%d,%d,%d,%d]", B, CH, H, W);
    LGS_REQUIRE(img1 != nullptr && img2 != nullptr, "ssim_forward: null image");
    LGS_REQUIRE((size_t)B * CH <= 65535, "ssim_forward: B*CH = %d exceeds the grid z limit", B * CH);
    const bool train = dm_dmu1 != nullptr;
    LGS_REQUIRE(!train || (dm_dsigma1_sq != nullptr && dm_dsigma12 != nullptr), "ssim_forward: the three partial maps come together");
    LGS_REQUIRE(map != nullptr || block_sums != nullptr || train, "ssim_forward: nothing to compute");
    cudaStream_t st = (cudaStream_t)stream;
    dim3 grid((W + CO - 1) / CO, (H + BH - 1) / BH, B * CH);
#define FWD(L, T) ssim_forward_kernel<L, T><<<grid, CT, 0, st>>>(img1, img2, H, W, C1, C2, ssim_weight, map, dm_dmu1, dm_dsigma1_sq, \
                                                                 dm_dsigma12, block_sums)
    if (l1_mode) { if (train) FWD(true, true); else FWD(true, false); }
    else { if (train) FWD(false, true); else FWD(false, false); }
#undef FWD
    LGS_CHECK_LAUNCH("ssim_forward_kernel");
    return LGS_OK;
}

extern "C" int lgs_ssim_backward(const float* img1, const float* img2, const float* dL_dmap, float uniform_chain, const float* dm_dmu1,
                                 const float* dm_dsigma1_sq, const float* dm_dsigma12, int B, int CH, int H, int W, int l1_mode,
                                 float ssim_weight, float* dL_dimg1, void* stream)
{
    LGS_REQUIRE(B >= 1 && CH >= 1 && H >= 1 && W >= 1, "ssim_backward: bad shape [%d,%d,%d,%d]", B, CH, H, W);
    LGS_REQUIRE(img1 && img2 && dm_dmu1 && dm_dsigma1_sq && dm_dsigma12 && dL_dimg1, "ssim_backward: null tensor");
    LGS_REQUIRE((size_t)B * CH <= 65535, "ssim_backward: B*CH = %d exceeds the grid z limit", B * CH);
    cudaStream_t st = (cudaStream_t)stream;
    dim3 grid((W + CO - 1) / CO, (H + BH - 1) / BH, B * CH);
#define BWD(L, U) ssim_backward_kernel<L, U><<<grid, CT, 0, st>>>(img1, img2, dL_dmap, uniform_chain, dm_dmu1, dm_dsigma1_sq, dm_dsigma12, H, \
                                                                  W, ssim_weight, dL_dimg1)
    if (dL_dmap == nullptr) { if (l1_mode) BWD(true, true); else BWD(false, true); }
    else { if (l1_mode) BWD(true, false); else BWD(false, false); }
#undef BWD
    LGS_CHECK_LAUNCH("ssim_backward_kernel");
    return LGS_OK;
}
