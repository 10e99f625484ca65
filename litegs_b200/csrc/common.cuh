// common.cuh -- shared helpers for the litegs_b200 CUDA library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#define LGS_OK 0
#define LGS_ERR_ARG 10001      // bad argument (size, null pointer, unsupported tile size ...)
#define LGS_ERR_WORKSPACE 10002 // caller-provided workspace too small

void lgs_set_error(const char* fmt, ...);

#define LGS_REQUIRE(cond, ...)                                   \
    do {                                                         \
        if (!(cond)) {                                           \
            lgs_set_error(__VA_ARGS__);                          \
            return LGS_ERR_ARG;                                  \
        }                                                        \
    } while (0)

// Launch check: the reference never checks launches (SURVEY Q10); we do, on every entry point.
#define LGS_CHECK_LAUNCH(what)                                                               \
    do {                                                                                     \
        cudaError_t e__ = cudaGetLastError();                                                \
        if (e__ != cudaSuccess) {                                                            \
            lgs_set_error("%s: %s (%s:%d)", what, cudaGetErrorString(e__), __FILE__, __LINE__); \
            return (int)e__;                                                                 \
        }                                                                                    \
    } while (0)

#define LGS_CUDA(...)                                                                        \
    do {                                                                                     \
        cudaError_t e__ = (__VA_ARGS__);                                                     \
        if (e__ != cudaSuccess) {                                                            \
            lgs_set_error("%s: %s (%s:%d)", "cuda call", cudaGetErrorString(e__), __FILE__, __LINE__); \
            return (int)e__;                                                                 \
        }                                                                                    \
    } while (0)

static inline int lgs_cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }
static inline bool lgs_tile_ok(int th, int tw)
{
    return (th == 8 && tw == 16) || (th == 12 && tw == 16) || (th == 16 && tw == 16) || (th == 8 && tw == 8);
}

// Dispatch on the four tile shapes the reference compiles (GR/raster.cu:375-383).
#define LGS_DISPATCH_TILE(th, tw, ...)                                   \
    if (th == 8 && tw == 16) { constexpr int TH = 8, TW = 16; __VA_ARGS__ }      \
    else if (th == 12 && tw == 16) { constexpr int TH = 12, TW = 16; __VA_ARGS__ } \
    else if (th == 16 && tw == 16) { constexpr int TH = 16, TW = 16; __VA_ARGS__ } \
    else { constexpr int TH = 8, TW = 8; __VA_ARGS__ }

// 48-byte fp32 splat record produced by pack/project and consumed by both raster kernels.
// (The reference packs colour/opacity to half in a 32-byte record, GR/raster.cu:19-29; the fp32
//  parity gate of BASELINE.json needs full precision, so ours is 12 floats.)
struct __align__(16) SplatRec {
    float px, py, A, B;     // screen mean, inverse covariance (A=[0][0], B=[0][1])
    float C, o, r, g;       // C=[1][1], activated opacity, colour r,g
    float b, depth, pad0, pad1;
};
static_assert(sizeof(SplatRec) == 48, "SplatRec must be 48 bytes");
#define LGS_REC_FLOATS 12

// 12-float gradient accumulator, same indexing as raster_backward's RED targets.  The geometry slots hold RAW moments
// of dL/dpower over the splat's pixels (dx = mu_x - x_pixel, dy = mu_y - y_pixel, s_k = sum_pixels dpw dy^k per column):
//   0: sum dx s0   1: sum s1   2: sum dx^2 s0   3: sum dx s1   4: sum s2   5,6,7: d colour   8: sum s0   9: err_sq
// and the consumer (unpack_kernel / project_backward_kernel) turns them into the gradients of GR/raster.cu:826-841 with the
// splat's conic (A, B, C) and opacity o once per splat:
//   dmu_x = -(A m0 + B m1)  dmu_y = -(B m0 + C m1)  dA = -m2/2  dB(total) = -m3  dC = -m4/2  do = m8 / o
#define LGS_GRAD_FLOATS 12
struct LgsRasterGrad { float dmx, dmy, dA, dB, dC, dop; };
#ifdef __CUDACC__
__device__ __forceinline__ void lgs_finish_raster_grad(const float4& a, const float4& c, const float4& e, float A, float B, float C,
                                                       float o, LgsRasterGrad& g)
{
    g.dmx = -(A * a.x + B * a.y);
    g.dmy = -(B * a.x + C * a.y);
    g.dA = -0.5f * a.z;
    g.dB = -a.w;
    g.dC = -0.5f * c.x;
    g.dop = (o > 0.0f) ? e.x / o : 0.0f;
}
#endif
