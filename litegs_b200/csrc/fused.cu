// fused.cu -- "Level B" of the render hot path: the per-view projection chain collapsed into one kernel
// per direction (SURVEY.md section 7).
//
// project_forward : gather visible chunk -> activate -> SH colour -> MVP -> S.R -> J -> cov2d -> inverse ->
//                   visibility + exact tile count -> 48-byte record + depth key + count.
//                   It replaces cull_compact_activate + mvp_transform_forward + createTransformMatrix_forward +
//                   jacobianRayspace + createCov2dDirectly_forward + eigh_and_inv_2x2matrix_forward +
//                   get_allocate_size + pack_forward_params (GR/compact.cu:825-893, GR/transform.cu:22-127,
//                   378-438,736-780,1364-1421, GR/binning.cu:289-385, GR/raster.cu:334-356) and never writes
//                   their ~230 B/Gaussian of intermediates (view_pos, ndc, T, J, cov2d, eig, inv, bbox) to HBM.
// project_backward: record gradient -> (recomputed chain) -> the six compacted parameter gradients; replaces
//                   unpack_gradient + inv_2x2matrix_backward + createCov2dDirectly_backward +
//                   createTransformMatrix_backward + mvp_transform_backward + activate_backward.
// emit_pairs_rec  : the (tile, splat) emission pass reading the record instead of three SoA tensors.
//
// The projection formulas are the functions of projection.cuh (and lgs_record_grad of common.cuh) that the op-level kernels
// in per_gaussian.cu and raster.cu call too, so both levels are checked against the same oracle.  Two are written out in
// project_backward_kernel with the expressions of the shared function, because calling it changes that kernel's register
// allocation: the inverse backward (lgs_inv2x2_backward) and the covariance backward (lgs_cov2d_backward).
// One view per launch (the reference's effective configuration, SURVEY Q1); batches of views loop on the host.
#include "common.cuh"
#include "projection.cuh"
#include "splat_geom.cuh"

struct ProjIntermediates {
    float s[3], qn[4], rn, o;       // activated scale, unit quaternion, 1/|q|, opacity
    float v[4], h[4], iw;           // view position, homogeneous clip position, 1/w
    float R[9];                     // rotation of the unit quaternion
    float VJ[6], M[6];              // V3x3.J and T.V3x3.J
    float inv[3];                   // A, B, C of the inverse 2D covariance
    float dirn[3];                  // unit view direction (for SH)
};

// Exact gradient mode (DESIGN.md section 1): one axis of lgs_ray_J backwards, as written.  p = P00 (P11), n = W (H), t = tx (ty);
// dJd = d J00 (J11), dJ2 = d J20 (J21), rz and rz2 as in lgs_ray_J.  Each clamp passes the gradient to the operand it returned;
// at a tie that is the position, not the limit.  Adds to d t, d tz and d rz; returns d p.
__device__ __forceinline__ float fused_J_axis_backward(float p, float n, float t, float tz, float rz, float rz2, float dJd, float dJ2,
                                                       float& dt, float& dtz, float& drz)
{
    const float f = p * n * 0.5f;
    const float l = tz / p * 1.3f;
    const float m = fminf(t, l);
    const float th = fmaxf(m, -l);
    const float df = dJd * rz - dJ2 * th * rz2;              // J_d = f rz, J_2 = -f th rz2
    const float dth = -dJ2 * f * rz2;
    drz += dJd * f - 2.0f * dJ2 * f * th * rz;
    float dm = dth, dl = 0.0f;
    if (m < -l) { dm = 0.0f; dl = -dth; }
    float dtt = dm;
    if (t > l) { dtt = 0.0f; dl += dm; }
    dt += dtt;
    dtz += dl * 1.3f / p;
    return df * n * 0.5f - dl * l / p;
}

// Mip-Splatting's 3D smoothing filter (DESIGN.md section 1, "3D smoothing filter"): s'_k = sqrt(s_k^2 + f^2) and
// rho3 = sqrt((r_0 r_1) r_2) with r_k = s_k^2 / (s_k^2 + f^2), every step one correctly rounded op in this order, so that
// tests/filter3d_oracle.py reproduces it bit for bit.  With f = 0, s' = s and rho3 = 1 exactly (s^2 normal).
struct Filter3D {
    float s[3];                     // the unfiltered activated scale
    float qf[3];                    // s_k^2 + f^2
    float f2, rho3;
};

__device__ __forceinline__ void filter_3d_factor(float f, const float* s, Filter3D& F)
{
    F.f2 = __fmul_rn(f, f);
    float r[3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const float q = __fmul_rn(s[k], s[k]);
        F.s[k] = s[k];
        F.qf[k] = __fadd_rn(q, F.f2);
        r[k] = __fdiv_rn(q, F.qf[k]);
    }
    F.rho3 = __fsqrt_rn(__fmul_rn(__fmul_rn(r[0], r[1]), r[2]));
}

// The forward chain shared by both directions.  Vm/P are the view / projection matrices (row-vector).
// F3D: the 3D filter f3d is applied: t.s holds the filtered scale s' and t.o the filtered opacity sigma(o_raw) * rho3; F keeps
// the unfiltered scale and the factors the backward needs.
template <bool F3D = false>
__device__ __forceinline__ void project_chain(const float* __restrict__ Vm, const float* __restrict__ P, const float* p,
                                              const float* s_raw, const float* q_raw, float o_raw, int H, int W,
                                              ProjIntermediates& t, float f3d = 0.0f, Filter3D* F = nullptr)
{
    lgs_activate_scale(s_raw, t.s);
    if constexpr (F3D) {
        filter_3d_factor(f3d, t.s, *F);
#pragma unroll
        for (int k = 0; k < 3; k++) t.s[k] = __fsqrt_rn(F->qf[k]);
    }
    t.rn = lgs_normalize_quat(q_raw, t.qn);
    t.o = lgs_sigmoid(o_raw);
    if constexpr (F3D) t.o = __fmul_rn(t.o, F->rho3);
    lgs_view_dir(Vm, p, t.dirn);
    const float w[4] = { p[0], p[1], p[2], 1.0f };       // the world position, w = 1
    lgs_mvp_view(Vm, w, t.v);
    t.iw = lgs_mvp_clip(P, t.v, t.h);
    // S.R (GR/transform.cu:106-125)
    lgs_quat_R(t.qn[0], t.qn[1], t.qn[2], t.qn[3], t.R);
    float J[6];
    lgs_ray_J(P, t.v, H, W, J);
    lgs_cov_M(Vm, J, t.R, t.s, t.VJ, t.M);
    float c00, c01, c11;
    lgs_cov2d(t.M, c00, c01, c11);
    float inv[4];
    lgs_inv2x2(c00, c01, c01, c11, inv);
    t.inv[0] = inv[0]; t.inv[1] = inv[1]; t.inv[2] = inv[3];
}

// Normals (DESIGN.md section 1, "Normals"): the view-space normal of the shortest scale axis, turned to face the camera.
// ax = argmin of the RAW log-scales (first index wins a tie; the 3D filter never changes it), n_w = row ax of R,
// n_c[j] = (n_w0 V[0][j] + n_w1 V[1][j]) + n_w2 V[2][j], sg = -1 if (n_c0 v0 + n_c1 v1) + n_c2 v2 > 0 else +1; n = sg n_c.
// n_c and the facing test are single-rounded ops in this order, so that tests/normal_oracle.py reproduces sg bit for bit.
// R is indexed with selects: a dynamic index would put the array in local memory.
struct NormalFrame {
    float nw[3], nc[3], sg;
    int ax;
};

__device__ __forceinline__ void normal_frame(const float* s_raw, const float* R, const float* __restrict__ Vm, const float* v,
                                             NormalFrame& f)
{
    int ax = (s_raw[1] < s_raw[0]) ? 1 : 0;
    ax = (s_raw[2] < (ax == 1 ? s_raw[1] : s_raw[0])) ? 2 : ax;
    f.ax = ax;
#pragma unroll
    for (int k = 0; k < 3; k++) f.nw[k] = (ax == 0) ? R[k] : ((ax == 1) ? R[3 + k] : R[6 + k]);
#pragma unroll
    for (int j = 0; j < 3; j++)
        f.nc[j] = __fadd_rn(__fadd_rn(__fmul_rn(f.nw[0], Vm[j]), __fmul_rn(f.nw[1], Vm[4 + j])), __fmul_rn(f.nw[2], Vm[8 + j]));
    const float dv = __fadd_rn(__fadd_rn(__fmul_rn(f.nc[0], v[0]), __fmul_rn(f.nc[1], v[1])), __fmul_rn(f.nc[2], v[2]));
    f.sg = (dv > 0.0f) ? -1.0f : 1.0f;
}

// Antialiased mode (DESIGN.md section 1): the opacity compensation of the 2D low-pass filter,
// rho = sqrt(det(M^T M) / det(M^T M + 0.3 I)).  Every step is one correctly rounded op in a fixed order, so that the
// opacity the tile decision sees is the oracle's bit for bit.
struct AAFactor {
    float a00, a01, a11;            // M^T M (unfiltered 2D covariance)
    float c00, c11;                 // diagonal of the filtered covariance
    float det_o, det_b, r2, rho;
};

__device__ __forceinline__ void antialias_factor(const float* M, AAFactor& f)
{
    f.a00 = __fadd_rn(__fadd_rn(__fmul_rn(M[0], M[0]), __fmul_rn(M[2], M[2])), __fmul_rn(M[4], M[4]));
    f.a01 = __fadd_rn(__fadd_rn(__fmul_rn(M[0], M[1]), __fmul_rn(M[2], M[3])), __fmul_rn(M[4], M[5]));
    f.a11 = __fadd_rn(__fadd_rn(__fmul_rn(M[1], M[1]), __fmul_rn(M[3], M[3])), __fmul_rn(M[5], M[5]));
    f.c00 = __fadd_rn(f.a00, 0.3f);
    f.c11 = __fadd_rn(f.a11, 0.3f);
    const float a01sq = __fmul_rn(f.a01, f.a01);
    f.det_o = __fsub_rn(__fmul_rn(f.a00, f.a11), a01sq);
    f.det_b = __fsub_rn(__fmul_rn(f.c00, f.c11), a01sq);
    f.r2 = __fdiv_rn(f.det_o, f.det_b);
    f.rho = __fsqrt_rn(fmaxf(f.r2, 0.0f));
}

// grid = allocated chunks (all M: chunks >= *visible_num write an invisible record), block = chunk size
// AA: the record's opacity is sigma(o_raw) * rho (antialiased mode); everything downstream reads it from the record.
// F3D: the 3D smoothing filter filter_3d[src] widens the scale and scales the opacity by rho3 before AA sees either.
// NORMAL: also the camera-facing view-space normal n of the shortest axis (normal_frame) into normal_rec f32[A*S,4] as
// (n0, n1, n2, 0); slots of chunks at or past the visible count get zeros, as their record does.
template <int DEG, int TH, int TW, bool AA, bool F3D, bool NORMAL = false>
__global__ void project_forward_kernel(
    const int64_t* __restrict__ chunk_ids, const int* __restrict__ visible_num, const float* __restrict__ view,
    const float* __restrict__ proj, const float* __restrict__ pos, const float* __restrict__ scale,
    const float* __restrict__ rot, const float* __restrict__ sh0, const float* __restrict__ shr,
    const float* __restrict__ opac, int C, int S, int H, int W, int gx, int gy, SplatRec* __restrict__ recs,
    unsigned* __restrict__ depth_key, unsigned* __restrict__ iota, int* __restrict__ tile_count, int* __restrict__ totals,
    const float* __restrict__ filter_3d, float4* __restrict__ normal_rec)
{
    const int a = blockIdx.x, s = threadIdx.x;
    const size_t dst = (size_t)a * S + s;
    int count = 0;
    unsigned key = 0xFFFFFFFFu;
    SplatRec r;
    r.px = r.py = 0.f; r.A = r.B = r.C = 0.f; r.o = 0.f; r.r = r.g = r.b = 0.f; r.depth = 0.f; r.pad0 = r.pad1 = 0.f;
    float4 nrm = make_float4(0.f, 0.f, 0.f, 0.f);
    if (a < visible_num[0]) {
        const size_t CS = (size_t)C * S;
        const size_t src = (size_t)chunk_ids[a] * S + s;
        float p[3] = { pos[src], pos[CS + src], pos[2 * CS + src] };
        float sr_[3] = { scale[src], scale[CS + src], scale[2 * CS + src] };
        float q[4] = { rot[src], rot[CS + src], rot[2 * CS + src], rot[3 * CS + src] };
        ProjIntermediates t;
        if constexpr (F3D) {
            Filter3D F;
            project_chain<true>(view, proj, p, sr_, q, opac[src], H, W, t, filter_3d[src], &F);
        } else {
            project_chain(view, proj, p, sr_, q, opac[src], H, W, t);
        }
        if constexpr (AA) {
            AAFactor f;
            antialias_factor(t.M, f);
            t.o = __fmul_rn(t.o, f.rho);
        }
        if constexpr (NORMAL) {
            NormalFrame nf;
            normal_frame(sr_, t.R, view, t.v, nf);
            nrm = make_float4(nf.sg * nf.nc[0], nf.sg * nf.nc[1], nf.sg * nf.nc[2], 0.f);
        }
        // colour (GR/compact.cu:573-653), no clamp on this path (SURVEY Q13)
        float col[3];
        lgs_sh_color<DEG>(t.dirn[0], t.dirn[1], t.dirn[2], sh0, shr, src, CS, col);
        const float ndcx = t.h[0] * t.iw, ndcy = t.h[1] * t.iw, ndcz = t.h[2] * t.iw;
        SplatGeom g;
        lgs_splat_setup<TH, TW>(ndcx, ndcy, t.v[2], t.inv[0], t.inv[1], t.inv[2], t.o, H, W, gx, gy, true, g);
        if (g.visible) count = lgs_process_tiles<TH, TW, false>(g, gx, 0, 0, 0, (int*)nullptr, (int*)nullptr);
        if (count > 0) key = __float_as_uint(t.v[2]);       // v.z > 0.2 here: positive floats order as unsigned
        r.px = __fsub_rn(__fmul_rn(__fmul_rn(__fadd_rn(ndcx, 1.0f), 0.5f), (float)W), 0.5f);   // GR/raster.cu:347-348
        r.py = __fsub_rn(__fmul_rn(__fmul_rn(__fadd_rn(ndcy, 1.0f), 0.5f), (float)H), 0.5f);
        r.A = t.inv[0]; r.B = t.inv[1]; r.C = t.inv[2]; r.o = t.o;
        r.r = col[0]; r.g = col[1]; r.b = col[2]; r.depth = t.v[2]; r.pad0 = ndcx; r.pad1 = ndcy;   // depth slot: view-space z (the sort key)
        (void)ndcz;
    }
    recs[dst] = r;
    if constexpr (NORMAL) normal_rec[dst] = nrm;
    depth_key[dst] = key;
    iota[dst] = (unsigned)dst;
    tile_count[dst] = count;
    // total number of (tile, splat) pairs: integer sum, order independent -> deterministic
    // totals: pair count (integer sum: order independent, deterministic) and the range of the depth keys that matter
    // (splats with pairs) so that the host can sort only the bits of that range.  totals[1] holds max(~key) so that a
    // zero fill initialises both.  One set of atomics per block.
    __shared__ int s_sum[32];
    __shared__ unsigned s_min[32], s_max[32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    int wsum = __reduce_add_sync(0xffffffffu, count);
    unsigned wmin = __reduce_min_sync(0xffffffffu, count > 0 ? key : 0xFFFFFFFFu);
    unsigned wmax = __reduce_max_sync(0xffffffffu, count > 0 ? key : 0u);
    if (lane == 0) { s_sum[wid] = wsum; s_min[wid] = wmin; s_max[wid] = wmax; }
    __syncthreads();
    if (wid == 0) {
        int bs = lane < nw ? s_sum[lane] : 0;
        unsigned bmin = lane < nw ? s_min[lane] : 0xFFFFFFFFu, bmax = lane < nw ? s_max[lane] : 0u;
        bs = __reduce_add_sync(0xffffffffu, bs);
        bmin = __reduce_min_sync(0xffffffffu, bmin);
        bmax = __reduce_max_sync(0xffffffffu, bmax);
        if (lane == 0 && bs != 0) {
            atomicAdd(&totals[0], bs);
            atomicMax((unsigned*)&totals[1], ~bmin);
            atomicMax((unsigned*)&totals[2], bmax);
        }
    }
}

// normal_rec f32[A*S,4] or NULL: normal mode, the camera-facing view-space normal of each record (DESIGN.md section 1, "Normals").
extern "C" int lgs_project_forward(int sh_degree, const int64_t* visible_chunk_id, const int* visible_chunks_num,
                                   const float* view_matrix, const float* proj_matrix, const float* position,
                                   const float* scale, const float* rotation, const float* sh_base, const float* sh_rest,
                                   const float* opacity, int C, int S, int A, int img_h, int img_w, int tile_h, int tile_w,
                                   float* packed_params, unsigned* depth_key, unsigned* iota, int* tile_count, int* totals,
                                   const float* filter_3d, int antialiased, float* normal_rec, void* stream)
{
    LGS_REQUIRE(sh_degree >= 0 && sh_degree <= 3, "project_forward: sh_degree %d not in 0..3", sh_degree);
    LGS_REQUIRE(lgs_tile_ok(tile_h, tile_w), "project_forward: tile %dx%d not one of 8x16, 12x16, 16x16, 8x8", tile_h, tile_w);
    LGS_REQUIRE(S >= 32 && S <= 1024 && S % 32 == 0, "project_forward: chunk size %d must be a multiple of 32 in 32..1024", S);
    cudaStream_t st = (cudaStream_t)stream;
    LGS_CUDA(cudaMemsetAsync(totals, 0, 3 * sizeof(int), st));
    if (A == 0) return LGS_OK;
    int gx = (img_w + tile_w - 1) / tile_w, gy = (img_h + tile_h - 1) / tile_h;
    const int rc = lgs_with_flags([&](auto nm, auto f3, auto aa) { return lgs_with_tile(tile_h, tile_w, [&](auto th, auto tw) {
        return lgs_with_degree(sh_degree, [&](auto deg) {
            constexpr auto kernel = project_forward_kernel<deg, th, tw, aa, f3, nm>;
            // the heaviest NORMAL instantiations use 72 registers, which allows 896 threads instead of 1024 (DESIGN.md section 1,
            // "Normals")
            if constexpr (nm) {
                const int mt = lgs_max_threads<kernel>();
                LGS_REQUIRE(S <= mt, "project_forward: normals with this configuration support chunk sizes up to %d, got %d", mt, S);
            }
            kernel<<<A, S, 0, st>>>(visible_chunk_id, visible_chunks_num, view_matrix, proj_matrix, position, scale, rotation, sh_base,
                                    sh_rest, opacity, C, S, img_h, img_w, gx, gy, (SplatRec*)packed_params, depth_key, iota, tile_count,
                                    totals, filter_3d, (float4*)normal_rec);
            return LGS_OK;
        }); }); }, normal_rec != nullptr, filter_3d != nullptr, antialiased != 0);
    if (rc != LGS_OK) return rc;
    LGS_CHECK_LAUNCH("project_forward_kernel");
    return LGS_OK;
}

// (tile+1, splat) emission in depth order from the packed record.    replaces GR/binning.cu:33-110
// One splat per lane.  A warp's 32 splats own one contiguous run [wbase, wend) of the pair list (the offsets
// are a scan in the same order), so the lanes stage their pairs in a per-warp shared-memory window and the
// warp then copies the window out with fully coalesced stores; without the staging every lane streams its own
// run and the kernel sits on the LSU queue (ncu: lg_throttle was the top stall).  Runs longer than the window
// are handled by walking again per window (rare: near-camera splats).
constexpr int LGS_EMIT_WARPS = 8;
#ifndef LGS_EMIT_WINDOW
#define LGS_EMIT_WINDOW 512
#endif
template <int TH, int TW, typename KeyT>
__global__ void __launch_bounds__(LGS_EMIT_WARPS * 32) emit_pairs_rec_kernel(const SplatRec* __restrict__ recs, const int* __restrict__ offset,
                                                             const unsigned* __restrict__ order, int n, int cap, int H, int W,
                                                             int gx, int gy, KeyT* __restrict__ keys, int* __restrict__ vals,
                                                             const int* __restrict__ n_dev, int* __restrict__ valid_pairs)
{
    __shared__ KeyT s_keys[LGS_EMIT_WARPS][LGS_EMIT_WINDOW];
    __shared__ int s_vals[LGS_EMIT_WARPS][LGS_EMIT_WINDOW];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (n_dev != nullptr) n = min(n, max(*n_dev, 0));         // GPU-driven sizing: n is the capacity, *n_dev the live count
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j - lane >= n) return;                               // whole warp past the end
    int off = 0, asz = 0, i = 0;
    if (j < n) {
        off = j == 0 ? 0 : offset[j - 1];
        asz = offset[j] - off;
        // the first run that crosses the capacity: everything from here on is dropped, so the list is valid up to `off`
        // exactly (offsets are monotone: this thread is unique) -- the sort and the tile ranges must not look further
        if (valid_pairs != nullptr && asz > 0 && off <= cap && off + asz > cap) *valid_pairs = off;
        if (asz <= 0 || off + asz > cap) asz = 0;
        i = (int)order[j];
    }
    SplatGeom g;
    g.visible = false;
    if (asz > 0) {
        const SplatRec r = recs[i];
        lgs_splat_setup<TH, TW>(r.pad0, r.pad1, 1.0f, r.A, r.B, r.C, r.o, H, W, gx, gy, false, g);
    }
    const bool live = asz > 0 && g.visible;
    const int wbase = __reduce_min_sync(0xffffffffu, live ? off : 0x7fffffff);
    const int wend = __reduce_max_sync(0xffffffffu, live ? off + asz : 0);
    KeyT* sk = s_keys[wid];
    int* sv = s_vals[wid];
    for (int lo = wbase; lo < wend; lo += LGS_EMIT_WINDOW) {
        if (live && off < lo + LGS_EMIT_WINDOW && off + asz > lo)
            lgs_process_tiles<TH, TW, true, KeyT>(g, gx, i, off, LGS_EMIT_WINDOW, sk, sv, lo);
        __syncwarp();
        const int m = min(LGS_EMIT_WINDOW, wend - lo);
        for (int k = lane; k < m; k += 32) { keys[lo + k] = sk[k]; vals[lo + k] = sv[k]; }
        __syncwarp();
    }
}

// n_capacity bounds the launch, *n_dev is the live splat count; runs that would cross `cap` are dropped (and flagged by
// lgs_view_params) and *valid_pairs (nullable; normally &params[1]) is lowered to the length of the list that WAS written, so
// that nothing downstream reads an unwritten slot.  key_bits = 16 (requires tiles + 1 < 65536) or 32.
extern "C" int lgs_emit_pairs_dev(const float* packed_params, const int* offset, const unsigned* order, int n_capacity, const int* n_dev,
                                  int cap, int img_h, int img_w, int tile_h, int tile_w, int key_bits, void* keys, int* vals,
                                  int* valid_pairs, void* stream)
{
    LGS_REQUIRE(lgs_tile_ok(tile_h, tile_w), "emit_pairs_dev: tile %dx%d not one of 8x16, 12x16, 16x16, 8x8", tile_h, tile_w);
    LGS_REQUIRE(n_dev != nullptr && (key_bits == 16 || key_bits == 32), "emit_pairs_dev: bad arguments");
    if (n_capacity <= 0 || cap <= 0) return LGS_OK;
    int gx = (img_w + tile_w - 1) / tile_w, gy = (img_h + tile_h - 1) / tile_h;
    LGS_REQUIRE(key_bits == 32 || gx * gy + 1 < 65536, "emit_pairs_dev: %d tiles do not fit 16-bit keys", gx * gy);
    cudaStream_t st = (cudaStream_t)stream;
    const int grid = lgs_cdiv(n_capacity, LGS_EMIT_WARPS * 32);
    lgs_with_flags([&](auto k16) { return lgs_with_tile(tile_h, tile_w, [&](auto th, auto tw) {
        using KeyT = std::conditional_t<k16, unsigned short, int>;
        emit_pairs_rec_kernel<th, tw, KeyT><<<grid, LGS_EMIT_WARPS * 32, 0, st>>>((const SplatRec*)packed_params, offset, order, n_capacity,
                                                                              cap, img_h, img_w, gx, gy, (KeyT*)keys, vals, n_dev, valid_pairs);
        return LGS_OK;
    }); }, key_bits == 16);
    LGS_CHECK_LAUNCH("emit_pairs_rec_kernel(dev)");
    return LGS_OK;
}

// Derived launch parameters of one view, computed ON THE DEVICE from the counters project_forward leaves behind, so that the rest
// of the view can be enqueued without reading anything back:
//   params[0] = live splat slots (visible chunks * S)      params[1] = pairs, clamped to the pair capacity
//   params[2] = depth-key bias (smallest key of a splat that owns pairs)
//   params[3] = bits of the depth-key range                 params[4] = flags: 1 = pairs exceed the capacity (list truncated),
//   params[5] = pairs (unclamped)                                        2 = depth-key range needs more bits than planned
//   params[6] = visible chunks                              params[7] = planned depth bits
// counters = i32[4] as written by lgs_frustum_culling_aabb ([0]) and lgs_project_forward ([1..3]).
// sticky (i32[4], nullable) accumulates over views: [0] |= flags, [1] = max pairs, [2] = max depth bits, [3] += 1 -- one read-back
// per BATCH of views tells whether any of them overflowed and how large the next workspace has to be.
__global__ void view_params_kernel(const int* __restrict__ counters, int S, int pair_capacity, int planned_bits, int* __restrict__ params,
                                   int* __restrict__ sticky)
{
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    const int nvis = counters[0], D = counters[1];
    const unsigned kmin = ~(unsigned)counters[2], kmax = (unsigned)counters[3];
    int bits = 1;
    if (D > 0 && kmax >= kmin) { unsigned r = kmax - kmin; bits = (r == 0) ? 1 : (32 - __clz(r)); }
    int flags = 0;
    if (D > pair_capacity) flags |= 1;
    if (bits > planned_bits) flags |= 2;
    params[0] = nvis * S; params[1] = min(D, pair_capacity); params[2] = (int)kmin; params[3] = bits;
    params[4] = flags; params[5] = D; params[6] = nvis; params[7] = planned_bits;
    if (sticky != nullptr) {
        atomicOr(&sticky[0], flags); atomicMax(&sticky[1], D); atomicMax(&sticky[2], bits); atomicAdd(&sticky[3], 1);
    }
}

extern "C" int lgs_view_params(const int* counters, int S, int pair_capacity, int planned_depth_bits, int* params, int* sticky,
                               void* stream)
{
    LGS_REQUIRE(counters != nullptr && params != nullptr && planned_depth_bits >= 1 && planned_depth_bits <= 32, "view_params: bad arguments");
    view_params_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(counters, S, pair_capacity, planned_depth_bits, params, sticky);
    LGS_CHECK_LAUNCH("view_params_kernel");
    return LGS_OK;
}

__device__ __forceinline__ float nan_to_num0(float x)
{
    if (x != x) return 0.0f;                               // torch.nan_to_num_(0) of wrapper.py:591
    if (isinf(x)) return x > 0 ? 3.4028234663852886e38f : -3.4028234663852886e38f;
    return x;
}

// Sum of 32 per-thread values over a warp: lane l returns the sum of v[l] (transposing butterfly, 31 shuffles).
// The order of the additions depends on nothing but the lane: the result is bit-reproducible.
template <int OFF>
__device__ __forceinline__ void warp_sum_transposed_step(float* v, int lane)
{
    const bool upper = (lane & OFF) != 0;
#pragma unroll
    for (int i = 0; i < OFF; i++) {
        const float send = upper ? v[i] : v[i + OFF];
        const float keep = upper ? v[i + OFF] : v[i];
        v[i] = keep + __shfl_xor_sync(0xffffffffu, send, OFF);
    }
}

__device__ __forceinline__ float warp_sum32_transposed(float* v)
{
    const int lane = threadIdx.x & 31;
    warp_sum_transposed_step<16>(v, lane);
    warp_sum_transposed_step<8>(v, lane);
    warp_sum_transposed_step<4>(v, lane);
    warp_sum_transposed_step<2>(v, lane);
    warp_sum_transposed_step<1>(v, lane);
    return v[0];
}

// CAM: also the camera gradient (DESIGN.md section 1, "Camera gradient").  Each thread forms its contribution to
// d_view[16] and d_proj[16]; the block sums them in a fixed order and writes one row of cam_partials f32[A,32] per
// chunk (chunks at or past the visible count write zeros); camera_grad_sum_kernel folds the rows.
// AA: antialiased mode.  The record gradient is taken at o_eff = sigma(o_raw) * rho; d o = d o_eff * rho, and the rho path
// adds d det(M^T M) and d det(M^T M + 0.3 I) to d cov2d before dM = 2 M G, so ds, dq and the camera path all see it.
// F3D: 3D smoothing filter.  With g = d o3 (after the AA step), d sigma = g rho3 and
// d s_raw_k = s_k (ds'_k (s_k / s'_k)) + (g o3) (f^2 / qf_k); f is held constant.
// EXACT: exact gradient mode.  d xyz (and, with CAM, the camera gradient) gain the terms through J (dJ = V3x3^T (T^T dM),
// back through lgs_ray_J to the view-space position and P00, P11) and through the SH view direction (reads sh_rest of the
// active degree).  The other gradients are the same instructions as without it.
// DEPTH: depth mode.  Record slot LGS_GRAD_DEPTH (d view-space z) joins dv.z: it reaches d xyz through V and the camera gradient as
// dV[k][2] += p~_k dz, and nothing reaches d proj.  A Gaussian whose only gradient is that slot is not skipped.
// NORMAL: normal mode.  grad_normal f32[A*S,4] (dL/dn from the raster backward) gives dn_c = sg dn and dn_w = V3x3 dn_c, which is
// added to row ax of the rotation-matrix gradient (dT after its product with s) and so reaches rot; with CAM,
// dV[k][j] += n_w[k] dn_c[j] (k, j < 3).  Nothing reaches xyz, the scales or d proj; ax and sg are held constant.  A Gaussian
// whose only gradient is a normal row is not skipped.
template <int DEG, bool CAM, bool AA, bool F3D, bool EXACT, bool DEPTH, bool NORMAL = false>
__global__ void project_backward_kernel(
    const int64_t* __restrict__ chunk_ids, const int* __restrict__ visible_num, const float* __restrict__ view,
    const float* __restrict__ proj, const float* __restrict__ pos, const float* __restrict__ scale,
    const float* __restrict__ rot, const float* __restrict__ opac, int C, int S, int A, int rest_dim, int H, int W,
    int true_sigmoid, int accumulate, const float* __restrict__ grad /*[A*S,12]*/, const float* __restrict__ inv_scaler,
    float* __restrict__ g_pos, float* __restrict__ g_scale, float* __restrict__ g_rot, float* __restrict__ g_sh0,
    float* __restrict__ g_shr, float* __restrict__ g_opac, float* __restrict__ touched, float* __restrict__ cam_partials,
    const float* __restrict__ filter_3d, const float* __restrict__ shr, const float4* __restrict__ grad_normal)
{
    const int a = blockIdx.x, s = threadIdx.x;
    if (a >= visible_num[0]) {
        if constexpr (CAM) {
            if (s < 32) cam_partials[(size_t)a * 32 + s] = 0.f;
        }
        return;
    }
    const size_t CS = (size_t)C * S, AS = (size_t)A * S;
    const size_t dst = (size_t)a * S + s, src = (size_t)chunk_ids[a] * S + s;
    if (touched != nullptr && s == 0) touched[chunk_ids[a]] = 1.0f;     // chunk mark for the fused optimizer step
    constexpr int K = (DEG + 1) * (DEG + 1);
    const float sc = inv_scaler ? inv_scaler[0] : 1.0f;
    const float4* g4 = reinterpret_cast<const float4*>(grad + dst * LGS_GRAD_FLOATS);
    const float4 ga = g4[0], gb = g4[1], gc = g4[2];
    const float4 gn = NORMAL ? grad_normal[dst] : make_float4(0.f, 0.f, 0.f, 0.f);
    const bool any = (ga.x != 0.f) | (ga.y != 0.f) | (ga.z != 0.f) | (ga.w != 0.f) | (gb.x != 0.f) | (gb.y != 0.f) |
                     (gb.z != 0.f) | (gb.w != 0.f) | (gc.x != 0.f) | (DEPTH && gc.z != 0.f) |
                     (NORMAL && ((gn.x != 0.f) | (gn.y != 0.f) | (gn.z != 0.f)));
    float o_pos[3] = { 0.f, 0.f, 0.f }, o_sc[3] = { 0.f, 0.f, 0.f }, o_q[4] = { 0.f, 0.f, 0.f, 0.f }, o_op = 0.f;
    float shb[16], dcol3[3] = { 0.f, 0.f, 0.f };       // SH basis and colour gradient: d sh[k][c] = shb[k] * dcol3[c]
#pragma unroll
    for (int k = 0; k < 16; k++) shb[k] = 0.f;
    float cam[CAM ? 32 : 1];        // d_view[k*4+j] then d_proj[16 + k*4+j] of this Gaussian
    if constexpr (CAM) {
#pragma unroll
        for (int k = 0; k < 32; k++) cam[k] = 0.f;
    }
    if (any) {
        float p[3] = { pos[src], pos[CS + src], pos[2 * CS + src] };
        float sr_[3] = { scale[src], scale[CS + src], scale[2 * CS + src] };
        float q[4] = { rot[src], rot[CS + src], rot[2 * CS + src], rot[3 * CS + src] };
        const float o_raw = opac[src];
        ProjIntermediates t;
        Filter3D F;
        if constexpr (F3D) {
            project_chain<true>(view, proj, p, sr_, q, o_raw, H, W, t, filter_3d[src], &F);
        } else {
            project_chain(view, proj, p, sr_, q, o_raw, H, W, t);
        }
        AAFactor f;
        float o_rec = t.o;                                  // the record's opacity
        if constexpr (AA) {
            antialias_factor(t.M, f);
            o_rec = __fmul_rn(t.o, f.rho);
        }
        // raw moments -> record gradient (GR/raster.cu:826-841), then unpack (GR/raster.cu:870-884)
        LgsRecordGrad rg;
        lgs_record_grad(ga, gb, gc, t.inv[0], t.inv[1], t.inv[2], o_rec, H, W, sc, rg);
        const float d_ndcx = rg.dndcx, d_ndcy = rg.dndcy, dA = rg.dA, dBh = rg.dBh, dC = rg.dC;
        const float* dcol = rg.dcol;
        float d_o = rg.dop;
        // inverse backward: dCov = -(inv . dInv . inv), the expressions of lgs_inv2x2_backward with A = [iA iB; iB iC] (a call
        // moves the register count of 111 backward instantiations by -21 to +11), NaN -> 0
        const float iA = t.inv[0], iB = t.inv[1], iC = t.inv[2];
        float t00 = iA * dA + iB * dBh, t01 = iA * dBh + iB * dC, t10 = iB * dA + iC * dBh, t11 = iB * dBh + iC * dC;
        float G[4];
        G[0] = nan_to_num0(-(t00 * iA + t01 * iB)); G[1] = nan_to_num0(-(t00 * iB + t01 * iC));
        G[2] = nan_to_num0(-(t10 * iA + t11 * iB)); G[3] = nan_to_num0(-(t10 * iB + t11 * iC));
        if constexpr (AA) {
            // o_eff = o sqrt(r2), r2 = det_o / det_b; rho = 0 means an invisible record, which gets no gradient
            if (f.rho > 0.0f) {
                const float d_r2 = d_o * t.o / (2.0f * f.rho);
                const float d_det_o = d_r2 / f.det_b;
                const float d_det_b = -d_r2 * f.r2 / f.det_b;
                const float d_a01_half = -f.a01 * (d_det_o + d_det_b);
                G[0] += d_det_o * f.a11 + d_det_b * f.c11;
                G[3] += d_det_o * f.a00 + d_det_b * f.c00;
                G[1] += d_a01_half;
                G[2] += d_a01_half;
            }
            d_o = d_o * f.rho;
        }
        // cov2d backward: dT = 2 M G (VJ)^T, the expressions of lgs_cov2d_backward (a call moves the register count of 27
        // backward instantiations by -19 to +4)
        float dT[9];
        float dM[(CAM || EXACT) ? 6 : 1];
#pragma unroll
        for (int r = 0; r < 3; r++) {
            float dM0 = 2.f * (t.M[r * 2] * G[0] + t.M[r * 2 + 1] * G[2]);
            float dM1 = 2.f * (t.M[r * 2] * G[1] + t.M[r * 2 + 1] * G[3]);
            if constexpr (CAM || EXACT) { dM[r * 2] = dM0; dM[r * 2 + 1] = dM1; }
#pragma unroll
            for (int k = 0; k < 3; k++) dT[r * 3 + k] = dM0 * t.VJ[k * 2] + dM1 * t.VJ[k * 2 + 1];
        }
        // transform backward (GR/transform.cu:185-226) on the ACTIVATED scale / unit quaternion
        float ds[3];
#pragma unroll
        for (int r = 0; r < 3; r++) ds[r] = lgs_scale_rot_backward(t.R + r * 3, t.s[r], dT + r * 3);
        NormalFrame nf;
        float dnc[3], dqn[4];
        if constexpr (NORMAL) {
            // the rotation-matrix gradient of the normal term: row ax is dn_w[k] = sum_j V[k][j] dn_c[j] with dn_c = sg dn, the
            // other rows zero.  It goes through its own quaternion backward and is added to the rot gradient at the end: by
            // linearity the same as adding it to dT here, and the other terms keep their instructions (g_N = 0 leaves their bits).
            normal_frame(sr_, t.R, view, t.v, nf);
            dnc[0] = nf.sg * (gn.x * sc); dnc[1] = nf.sg * (gn.y * sc); dnc[2] = nf.sg * (gn.z * sc);
            float dRn[9];
#pragma unroll
            for (int k = 0; k < 3; k++) {
                const float dnw = view[k * 4] * dnc[0] + view[k * 4 + 1] * dnc[1] + view[k * 4 + 2] * dnc[2];
#pragma unroll
                for (int r = 0; r < 3; r++) dRn[r * 3 + k] = (r == nf.ax) ? dnw : 0.0f;
            }
            lgs_quat_R_backward(t.qn[0], t.qn[1], t.qn[2], t.qn[3], dRn, dqn);
        }
        float dq[4];
        lgs_quat_R_backward(t.qn[0], t.qn[1], t.qn[2], t.qn[3], dT, dq);
        // activation chain (GR/compact.cu:925-952)
        if constexpr (F3D) {
            // ds is the gradient at s' (t.s); t.o is o3 and d_o is d o3
            const float go3 = __fmul_rn(d_o, t.o);
#pragma unroll
            for (int k = 0; k < 3; k++)
                o_sc[k] = __fadd_rn(__fmul_rn(F.s[k], __fmul_rn(ds[k], __fdiv_rn(F.s[k], t.s[k]))), __fmul_rn(go3, __fdiv_rn(F.f2, F.qf[k])));
            d_o = __fmul_rn(d_o, F.rho3);
        } else {
#pragma unroll
            for (int k = 0; k < 3; k++) o_sc[k] = t.s[k] * ds[k];
        }
        lgs_quat_normalize_backward(dq, t.qn, t.rn, o_q);
        if constexpr (NORMAL) {
            float o_qn[4];
            lgs_quat_normalize_backward(dqn, t.qn, t.rn, o_qn);
#pragma unroll
            for (int k = 0; k < 4; k++) o_q[k] = __fadd_rn(o_q[k], o_qn[k]);   // no contraction into o_q
        }
        o_op = lgs_sigmoid_backward(d_o, o_raw, true_sigmoid);
        // MVP backward (GR/transform.cu:517-558) with d_ndc.z = d_ndc.w = 0 and no view-space gradient
        const float* P = proj; const float* Vm = view;
        const float dndc[3] = { d_ndcx, d_ndcy, 0.f }, dv_view[4] = { 0.f, 0.f, 0.f, 0.f };
        float dh[4], dv[4];
        lgs_mvp_clip_backward(P, t.h, t.iw, dndc, dv_view, dh, dv);
        if constexpr (DEPTH) dv[2] += gc.z * sc;          // d view-space z of the depth channel (slot LGS_GRAD_DEPTH = gc.z)
        float dp00 = 0.f, dp11 = 0.f;
        if constexpr (EXACT) {
            // J term: dVJ = T^T dM, dJ[k][c] = sum_a V3[a][k] dVJ[a][c]; only J00, J11, J20, J21 depend on anything
            float dVJ[6];
#pragma unroll
            for (int r = 0; r < 3; r++)
#pragma unroll
                for (int c = 0; c < 2; c++)
                    dVJ[r * 2 + c] = t.R[r] * t.s[0] * dM[c] + t.R[3 + r] * t.s[1] * dM[2 + c] + t.R[6 + r] * t.s[2] * dM[4 + c];
            const float dJ00 = Vm[0] * dVJ[0] + Vm[4] * dVJ[2] + Vm[8] * dVJ[4];
            const float dJ11 = Vm[1] * dVJ[1] + Vm[5] * dVJ[3] + Vm[9] * dVJ[5];
            const float dJ20 = Vm[2] * dVJ[0] + Vm[6] * dVJ[2] + Vm[10] * dVJ[4];
            const float dJ21 = Vm[2] * dVJ[1] + Vm[6] * dVJ[3] + Vm[10] * dVJ[5];
            const float tz = t.v[2];
            const float rz = 1.0f / fmaxf(tz, 1e-2f), rz2 = rz * rz;
            float dtz = 0.f, drz = 0.f;
            dp00 = fused_J_axis_backward(P[0], (float)W, t.v[0], tz, rz, rz2, dJ00, dJ20, dv[0], dtz, drz);
            dp11 = fused_J_axis_backward(P[5], (float)H, t.v[1], tz, rz, rz2, dJ11, dJ21, dv[1], dtz, drz);
            if (!(tz < 1e-2f)) dtz -= rz2 * drz;             // below the depth floor rz is constant
            dv[2] += dtz;
        }
        float dw[4];
        lgs_mvp_view_backward(Vm, dv, dw);
#pragma unroll
        for (int k = 0; k < 3; k++) o_pos[k] = dw[k];
        if constexpr (CAM) {
            // NDC path: v = p~ . Vm and h = v . P  ->  dVm[k][j] = p~_k dv_j, dP[k][j] = v_k dh_j
            const float pt[4] = { p[0], p[1], p[2], 1.0f };
#pragma unroll
            for (int k = 0; k < 4; k++)
#pragma unroll
                for (int j = 0; j < 4; j++) { cam[k * 4 + j] = pt[k] * dv[j]; cam[16 + k * 4 + j] = t.v[k] * dh[j]; }
            if constexpr (EXACT) { cam[16] += dp00; cam[21] += dp11; }
            // Sigma2 path through the V3x3 factor of M = T.V3x3.J, J frozen: dVJ = T^T dM, dV3[a][k] = sum_c dVJ[a][c] J[k][c]
            float J[6];
            lgs_ray_J(P, t.v, H, W, J);
#pragma unroll
            for (int r = 0; r < 3; r++) {
                float dVJ[2];
#pragma unroll
                for (int c = 0; c < 2; c++)
                    dVJ[c] = t.R[r] * t.s[0] * dM[c] + t.R[3 + r] * t.s[1] * dM[2 + c] + t.R[6 + r] * t.s[2] * dM[4 + c];
#pragma unroll
                for (int k = 0; k < 3; k++) cam[r * 4 + k] += dVJ[0] * J[k * 2] + dVJ[1] * J[k * 2 + 1];
            }
            if constexpr (NORMAL) {
                // n_c[j] = sum_k n_w[k] V[k][j]  ->  dV[k][j] += n_w[k] dn_c[j]
#pragma unroll
                for (int k = 0; k < 3; k++)
#pragma unroll
                    for (int j = 0; j < 3; j++) cam[k * 4 + j] = __fmaf_rn(nf.nw[k], dnc[j], cam[k * 4 + j]);
            }
        }
        // SH coefficients (GR/compact.cu:655-823); the direction is treated as constant
        lgs_sh_basis<DEG>(t.dirn[0], t.dirn[1], t.dirn[2], shb);
        dcol3[0] = dcol[0]; dcol3[1] = dcol[1]; dcol3[2] = dcol[2];
        if constexpr (EXACT && DEG > 0) {
            // SH direction term: w_k = sum_c sh[k][c] dcol_c, g_u = sum_k w_k d b_k / du, g_d = n (g_u - u (u . g_u)) with
            // d = p - cc and n = 1 / sqrt(|d|^2 + 1e-12) as in project_chain; d xyz += g_d, d cc = -g_d
            float w[K];
            w[0] = 0.f;
#pragma unroll
            for (int k = 1; k < K; k++) {
                const float* sk = shr + (size_t)(k - 1) * 3 * CS + src;
                w[k] = sk[0] * dcol[0] + sk[CS] * dcol[1] + sk[2 * CS] * dcol[2];
            }
            float gu[3];
            lgs_sh_basis_grad<DEG>(t.dirn[0], t.dirn[1], t.dirn[2], w, gu);
            float ud[3];
            const float dn = lgs_view_dir(Vm, p, ud);
            const float ug = t.dirn[0] * gu[0] + t.dirn[1] * gu[1] + t.dirn[2] * gu[2];
            float gd[3];
#pragma unroll
            for (int m = 0; m < 3; m++) { gd[m] = dn * (gu[m] - t.dirn[m] * ug); o_pos[m] += gd[m]; }
            if constexpr (CAM) {
                // cc_m = sum_k (-V[3][k]) V[m][k]: d V[3][k] += sum_m g_d[m] V[m][k], d V[m][k] += g_d[m] V[3][k]
#pragma unroll
                for (int k = 0; k < 3; k++) {
                    cam[12 + k] += gd[0] * Vm[k] + gd[1] * Vm[4 + k] + gd[2] * Vm[8 + k];
#pragma unroll
                    for (int m = 0; m < 3; m++) cam[m * 4 + k] += gd[m] * Vm[12 + k];
                }
            }
        }
    }
    if constexpr (CAM) {
        // chunk sum in a fixed order: warps by the transposing butterfly, then warp 0..nw-1 in sequence (S % 32 == 0)
        __shared__ float s_cam[32][33];
        const int lane = s & 31, wid = s >> 5, nw = blockDim.x >> 5;
        s_cam[wid][lane] = warp_sum32_transposed(cam);
        __syncthreads();
        if (s < 32) {
            float acc = s_cam[0][s];
            for (int w = 1; w < nw; w++) acc += s_cam[w][s];
            cam_partials[(size_t)a * 32 + s] = acc;
        }
    }
    if (accumulate) {
        // dense accumulation: outputs are the full [..,C,S] gradient tensors, this view's contribution is added at
        // the SOURCE chunk (each Gaussian is owned by exactly one thread of one launch: no atomics needed);
        // Gaussians that received no gradient are not touched at all.
        // The read-modify-writes are issued in batches (all loads of a batch first, then the stores) so that 11-16
        // independent L2 round trips are in flight per thread instead of one dependent load->add->store chain each.
        if (any) {
            float old[11];
#pragma unroll
            for (int k = 0; k < 3; k++) old[k] = g_pos[k * CS + src];
#pragma unroll
            for (int k = 0; k < 3; k++) old[3 + k] = g_scale[k * CS + src];
#pragma unroll
            for (int k = 0; k < 4; k++) old[6 + k] = g_rot[k * CS + src];
            old[10] = g_opac[src];
#pragma unroll
            for (int k = 0; k < 3; k++) g_pos[k * CS + src] = old[k] + o_pos[k];
#pragma unroll
            for (int k = 0; k < 3; k++) g_scale[k * CS + src] = old[3 + k] + o_sc[k];
#pragma unroll
            for (int k = 0; k < 4; k++) g_rot[k * CS + src] = old[6 + k] + o_q[k];
            g_opac[src] = old[10] + o_op;
#pragma unroll
            for (int c = 0; c < 3; c++) {
                float osh[K];
                osh[0] = g_sh0[c * CS + src];
#pragma unroll
                for (int k = 1; k < K; k++) osh[k] = g_shr[((size_t)(k - 1) * 3 + c) * CS + src];
                g_sh0[c * CS + src] = fmaf(shb[0], dcol3[c], osh[0]);
#pragma unroll
                for (int k = 1; k < K; k++) g_shr[((size_t)(k - 1) * 3 + c) * CS + src] = fmaf(shb[k], dcol3[c], osh[k]);
            }
        }
        return;
    }
#pragma unroll
    for (int k = 0; k < 3; k++) g_pos[k * AS + dst] = o_pos[k];
#pragma unroll
    for (int k = 0; k < 3; k++) g_scale[k * AS + dst] = o_sc[k];
#pragma unroll
    for (int k = 0; k < 4; k++) g_rot[k * AS + dst] = o_q[k];
    g_opac[dst] = o_op;
#pragma unroll
    for (int c = 0; c < 3; c++) {
        g_sh0[c * AS + dst] = shb[0] * dcol3[c];
#pragma unroll
        for (int k = 1; k < K; k++) g_shr[((size_t)(k - 1) * 3 + c) * AS + dst] = shb[k] * dcol3[c];
    }
    (void)rest_dim;
}

// d_cam[j] = sum over the A rows of partials[a*32 + j], in a fixed order: 32 row groups (a = g, g+32, ...) per column,
// then the groups in sequence.  Rows of chunks past the visible count are zero, so capacity-sized launches give the
// same bits as exact ones.
__global__ void __launch_bounds__(1024) camera_grad_sum_kernel(const float* __restrict__ partials, int A, float* __restrict__ d_cam)
{
    __shared__ float s_acc[32][33];
    const int j = threadIdx.x & 31, g = threadIdx.x >> 5;
    float acc = 0.0f;
    for (int a = g; a < A; a += 32) acc += partials[(size_t)a * 32 + j];
    s_acc[g][j] = acc;
    __syncthreads();
    if (g == 0) {
        float sum = s_acc[0][j];
        for (int k = 1; k < 32; k++) sum += s_acc[k][j];
        d_cam[j] = sum;
    }
}

// mode 0: outputs are compacted [..,A,S] and assigned; mode 1: same, cleared first (rows of chunks >= *visible_num and
// sh_rest rows above the active degree must read as zero); mode 2: outputs are the DENSE [..,C,S] gradient tensors and
// this view's gradients are accumulated into them (the multi-view / data-parallel path: no compacted round trip).
// depth: 1 = the record gradient carries a depth slot (lgs_rasterize_backward was given d_depth), 0 = it does not.
// grad_normal: f32[A*S,4] normal gradient of lgs_rasterize_backward (normal mode), or NULL = no normal term.
extern "C" int lgs_project_backward(int sh_degree, const int64_t* visible_chunk_id, const int* visible_chunks_num,
                                    const float* view_matrix, const float* proj_matrix, const float* position,
                                    const float* scale, const float* rotation, const float* opacity, int C, int S, int A,
                                    int rest_dim, int img_h, int img_w, int true_sigmoid_grad, const float* packed_grad,
                                    const float* grad_inv_scaler, int zero_outputs, float* g_position, float* g_scale,
                                    float* g_rotation, float* g_sh_base, float* g_sh_rest, float* g_opacity, float* touched,
                                    float* cam_partials, float* d_cam, const float* filter_3d, int antialiased,
                                    const float* sh_base, const float* sh_rest, int exact_grad, int depth,
                                    const float* grad_normal, void* stream)
{
    LGS_REQUIRE(sh_degree >= 0 && sh_degree <= 3, "project_backward: sh_degree %d not in 0..3", sh_degree);
    LGS_REQUIRE(rest_dim >= (sh_degree + 1) * (sh_degree + 1) - 1, "project_backward: sh_rest has %d rows, degree %d needs %d", rest_dim,
                sh_degree, (sh_degree + 1) * (sh_degree + 1) - 1);
    LGS_REQUIRE(S >= 1 && S <= 1024, "project_backward: chunk size %d unsupported", S);
    const bool cam = d_cam != nullptr;
    LGS_REQUIRE((cam_partials != nullptr) == cam, "project_backward: cam_partials and d_cam are both given or both NULL");
    LGS_REQUIRE(!cam || S % 32 == 0, "project_backward: the camera gradient needs a chunk size that is a multiple of 32, got %d", S);
    LGS_REQUIRE(!exact_grad || sh_degree == 0 || sh_rest != nullptr, "project_backward: exact_grad at SH degree %d needs sh_rest",
                sh_degree);
    (void)sh_base;                                  // the constant band has no direction term
    cudaStream_t st = (cudaStream_t)stream;
    if (A == 0) {
        if (cam) LGS_CUDA(cudaMemsetAsync(d_cam, 0, 32 * sizeof(float), st));
        return LGS_OK;
    }
    size_t AS = (size_t)A * S;
    const int accumulate = (zero_outputs == 2) ? 1 : 0;
    if (zero_outputs == 1) {
        LGS_CUDA(cudaMemsetAsync(g_position, 0, sizeof(float) * 3 * AS, st));
        LGS_CUDA(cudaMemsetAsync(g_scale, 0, sizeof(float) * 3 * AS, st));
        LGS_CUDA(cudaMemsetAsync(g_rotation, 0, sizeof(float) * 4 * AS, st));
        LGS_CUDA(cudaMemsetAsync(g_sh_base, 0, sizeof(float) * 3 * AS, st));
        LGS_CUDA(cudaMemsetAsync(g_sh_rest, 0, sizeof(float) * (size_t)rest_dim * 3 * AS, st));
        LGS_CUDA(cudaMemsetAsync(g_opacity, 0, sizeof(float) * AS, st));
    }
    const int rc = lgs_with_flags([&](auto nm, auto ex, auto z, auto f3, auto aa, auto k) {
        return lgs_with_degree(sh_degree, [&](auto deg) {
            constexpr auto kernel = project_backward_kernel<deg, k, aa, f3, ex, z, nm>;
            // The kernel has no launch bounds (the default instantiations must keep their code), and the heaviest EXACT ones use up
            // to 168 registers, which allows 384 threads instead of 1024 (DESIGN.md section 1, "Exact gradient mode"); NORMAL
            // instantiations use up to 138 without EXACT (DESIGN.md section 1, "Normals").
            if constexpr (ex || nm) {
                const int mt = lgs_max_threads<kernel>();
                LGS_REQUIRE(S <= mt, "project_backward: %s with this configuration supports chunk sizes up to %d, got %d",
                            ex ? "exact_grad" : "the normal gradient", mt, S);
            }
            kernel<<<A, S, 0, st>>>(visible_chunk_id, visible_chunks_num, view_matrix, proj_matrix, position, scale, rotation, opacity, C,
                                    S, A, rest_dim, img_h, img_w, true_sigmoid_grad, accumulate, packed_grad, grad_inv_scaler, g_position,
                                    g_scale, g_rotation, g_sh_base, g_sh_rest, g_opacity, touched, cam_partials, filter_3d, sh_rest,
                                    (const float4*)grad_normal);
            return LGS_OK;
        }); }, grad_normal != nullptr, exact_grad != 0, depth != 0, filter_3d != nullptr, antialiased != 0, cam);
    if (rc != LGS_OK) return rc;
    LGS_CHECK_LAUNCH("project_backward_kernel");
    if (cam) {
        camera_grad_sum_kernel<<<1, 1024, 0, st>>>(cam_partials, A, d_cam);
        LGS_CHECK_LAUNCH("camera_grad_sum_kernel");
    }
    return LGS_OK;
}

// ---------------------------------------------------------------------------------------------------
// Camera matrices from learnable view parameters: create_viewproj (GR/compact.cu:17-141, 143-316)
// ---------------------------------------------------------------------------------------------------

struct ViewProjMats {
    float r, x, y, z;               // normalised quaternion
    float view[16], proj[16];       // row-vector convention, [i*4+j]
};

__device__ __forceinline__ void viewproj_mats(const float* __restrict__ vp /*[7]*/, float recp_tan_half_fov_x, int img_h, int img_w,
                                              float z_near, float z_far, ViewProjMats& m)
{
    float r = vp[0], x = vp[1], y = vp[2], z = vp[3];
    const float recp = rsqrtf(r * r + x * x + y * y + z * z + 1e-12f);      // as GR/compact.cu:35
    r *= recp; x *= recp; y *= recp; z *= recp;
    m.r = r; m.x = x; m.y = y; m.z = z;
    const float V[16] = { 1 - 2 * (y * y + z * z), 2 * (x * y + r * z), 2 * (x * z - r * y), 0,
                          2 * (x * y - r * z), 1 - 2 * (x * x + z * z), 2 * (y * z + r * x), 0,
                          2 * (x * z + r * y), 2 * (y * z - r * x), 1 - 2 * (x * x + y * y), 0,
                          vp[4], vp[5], vp[6], 1.0f };
    const float p00 = recp_tan_half_fov_x;
    const float p11 = p00 * img_w / img_h;                                 // float arithmetic here (GR/compact.cu:55)
    const float P[16] = { p00, 0, 0, 0,
                          0, p11, 0, 0,
                          0, 0, z_far / (z_far - z_near), 1,
                          0, 0, -z_far * z_near / (z_far - z_near), 0 };
#pragma unroll
    for (int k = 0; k < 16; k++) { m.view[k] = V[k]; m.proj[k] = P[k]; }
}

// one thread per view; outputs view, proj, viewproj f32[V,4,4] and frustumplane f32[V,6,4]
__global__ void create_viewproj_forward_kernel(const float* __restrict__ view_params, const float* __restrict__ recp_tan_half_fov_x, int V,
                                               int img_h, int img_w, float z_near, float z_far, float* __restrict__ view,
                                               float* __restrict__ proj, float* __restrict__ viewproj, float* __restrict__ planes)
{
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    ViewProjMats m;
    viewproj_mats(view_params + (size_t)v * 7, recp_tan_half_fov_x[0], img_h, img_w, z_near, z_far, m);
    float vp[16];
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) {
            float acc = 0.0f;
#pragma unroll
            for (int k = 0; k < 4; k++) acc += m.view[i * 4 + k] * m.proj[k * 4 + j];
            vp[i * 4 + j] = acc;
        }
#pragma unroll
    for (int k = 0; k < 16; k++) {
        view[(size_t)v * 16 + k] = m.view[k]; proj[(size_t)v * 16 + k] = m.proj[k]; viewproj[(size_t)v * 16 + k] = vp[k];
    }
    // planes (GR/compact.cu:90-118): column combinations of viewproj, row i of the plane = row i of the matrix
    float* pl = planes + (size_t)v * 24;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const float c0 = vp[i * 4 + 0], c1 = vp[i * 4 + 1], c2 = vp[i * 4 + 2], c3 = vp[i * 4 + 3];
        pl[0 * 4 + i] = c3 + c0; pl[1 * 4 + i] = c3 - c0;
        pl[2 * 4 + i] = c3 + c1; pl[3 * 4 + i] = c3 - c1;
        pl[4 * 4 + i] = c2;      pl[5 * 4 + i] = c3 - c2;
    }
}

// One block; thread t handles views t, t + blockDim, ...  The fov gradient is summed per thread in view order and then
// over threads in a fixed order (the reference's += on one global word races across views, GR/compact.cu:275-276).
constexpr int LGS_VIEWPROJ_THREADS = 128;
__global__ void __launch_bounds__(LGS_VIEWPROJ_THREADS) create_viewproj_backward_kernel(
    const float* __restrict__ view_grad, const float* __restrict__ proj_grad, const float* __restrict__ viewproj_grad,
    const float* __restrict__ view_params, const float* __restrict__ recp_tan_half_fov_x, int V, int img_h, int img_w, float z_near,
    float z_far, float* __restrict__ grad_view_params, float* __restrict__ grad_recp)
{
    __shared__ float s_fov[LGS_VIEWPROJ_THREADS];
    float fov = 0.0f;
    for (int v = threadIdx.x; v < V; v += blockDim.x) {
        ViewProjMats m;
        viewproj_mats(view_params + (size_t)v * 7, recp_tan_half_fov_x[0], img_h, img_w, z_near, z_far, m);
        // d viewproj -> d view (= dVP . P^T) and d proj (= V^T . dVP), plus the incoming gradients (GR/compact.cu:191-212)
        float gv[16], gp[16];
#pragma unroll
        for (int k = 0; k < 16; k++) { gv[k] = 0.f; gp[k] = 0.f; }
#pragma unroll
        for (int i = 0; i < 4; i++)
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const float g = viewproj_grad[(size_t)v * 16 + i * 4 + j];
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    gv[i * 4 + k] += g * m.proj[k * 4 + j];
                    gp[k * 4 + j] += g * m.view[i * 4 + k];
                }
            }
#pragma unroll
        for (int k = 0; k < 16; k++) {
            gv[k] = view_grad[(size_t)v * 16 + k] + gv[k];
            gp[k] = proj_grad[(size_t)v * 16 + k] + gp[k];
        }
        // rotation block -> normalised quaternion (GR/compact.cu:215-267)
        const float r = m.r, x = m.x, y = m.y, z = m.z;
        float gr = 0, gx = 0, gy = 0, gz = 0, g;
        g = gv[0];  gy += g * (-4 * y); gz += g * (-4 * z);
        g = gv[1];  gx += g * (2 * y); gy += g * (2 * x); gr += g * (2 * z); gz += g * (2 * r);
        g = gv[2];  gx += g * (2 * z); gz += g * (2 * x); gr += g * (-2 * y); gy += g * (-2 * r);
        g = gv[4];  gx += g * (2 * y); gy += g * (2 * x); gr += g * (-2 * z); gz += g * (-2 * r);
        g = gv[5];  gx += g * (-4 * x); gz += g * (-4 * z);
        g = gv[6];  gy += g * (2 * z); gz += g * (2 * y); gr += g * (2 * x); gx += g * (2 * r);
        g = gv[8];  gx += g * (2 * z); gz += g * (2 * x); gr += g * (2 * y); gy += g * (2 * r);
        g = gv[9];  gy += g * (2 * z); gz += g * (2 * y); gr += g * (-2 * x); gx += g * (-2 * r);
        g = gv[10]; gx += g * (-4 * x); gy += g * (-4 * y);
        float* out = grad_view_params + (size_t)v * 7;
        out[4] = gv[12]; out[5] = gv[13]; out[6] = gv[14];
        // fov: proj_11 = proj_00 * w / h, but the backward scales by the INTEGER quotient img_w / img_h (GR/compact.cu:276)
        fov = fov + gp[0];
        fov = fov + gp[5] * (float)(img_w / img_h);
        // normalisation backward on the already normalised quaternion (GR/compact.cu:279-285): the true derivative times |q|
        const float norm = sqrtf(r * r + x * x + y * y + z * z);
        const float dot = (r * gr + x * gx + y * gy + z * gz) / (norm * norm);
        out[0] = gr / norm - r * dot; out[1] = gx / norm - x * dot; out[2] = gy / norm - y * dot; out[3] = gz / norm - z * dot;
    }
    s_fov[threadIdx.x] = fov;
    __syncthreads();
    if (threadIdx.x == 0) {
        float acc = 0.0f;
        for (int t = 0; t < LGS_VIEWPROJ_THREADS; t++) acc += s_fov[t];
        grad_recp[0] = acc;
    }
}

extern "C" int lgs_create_viewproj_forward(const float* view_params, const float* recp_tan_half_fov_x, int V, int img_h, int img_w,
                                           float z_near, float z_far, float* view_matrix, float* proj_matrix, float* viewproj_matrix,
                                           float* frustumplane, void* stream)
{
    LGS_REQUIRE(V >= 0 && img_h > 0 && img_w > 0, "create_viewproj_forward: bad arguments (V %d, %dx%d)", V, img_h, img_w);
    if (V == 0) return LGS_OK;
    create_viewproj_forward_kernel<<<lgs_cdiv(V, 128), 128, 0, (cudaStream_t)stream>>>(view_params, recp_tan_half_fov_x, V, img_h, img_w,
                                                                                      z_near, z_far, view_matrix, proj_matrix,
                                                                                      viewproj_matrix, frustumplane);
    LGS_CHECK_LAUNCH("create_viewproj_forward_kernel");
    return LGS_OK;
}

extern "C" int lgs_create_viewproj_backward(const float* view_matrix_grad, const float* proj_matrix_grad, const float* viewproj_matrix_grad,
                                            const float* view_params, const float* recp_tan_half_fov_x, int V, int img_h, int img_w,
                                            float z_near, float z_far, float* grad_view_params, float* grad_recp_tan_half_fov_x,
                                            void* stream)
{
    LGS_REQUIRE(V >= 0 && img_h > 0 && img_w > 0, "create_viewproj_backward: bad arguments (V %d, %dx%d)", V, img_h, img_w);
    create_viewproj_backward_kernel<<<1, LGS_VIEWPROJ_THREADS, 0, (cudaStream_t)stream>>>(view_matrix_grad, proj_matrix_grad,
        viewproj_matrix_grad, view_params, recp_tan_half_fov_x, V, img_h, img_w, z_near, z_far, grad_view_params, grad_recp_tan_half_fov_x);
    LGS_CHECK_LAUNCH("create_viewproj_backward_kernel");
    return LGS_OK;
}
