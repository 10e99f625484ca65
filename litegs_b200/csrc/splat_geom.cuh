// splat_geom.cuh -- per-splat visibility test, alpha=1/255 iso-ellipse bounding box and the exact
// ellipse/tile overlap walk ("AccuTile").  Restates GR/binning.cu:309-355 and GR/speedy_splat.cuh:16-149.
//
// These are step functions of fp32 quantities that decide WHICH (tile, splat) pairs exist, i.e. integer
// results.  To make them bit-reproducible (and bit-comparable with the CPU oracle) every operation is a
// single correctly-rounded IEEE op (__fmul_rn & co are never contracted into FMAs, sqrt/div are the
// IEEE ones) in the reference's expression order, and 2*ln(255 o) is evaluated in double and rounded
// once.  The reference's own build uses --use_fast_math here (GR/setup.py:35), which is why its lists
// can differ from ours on pairs that graze a tile corner (SURVEY Appendix B).
// Attribution (carried over from the file this restates, GR/speedy_splat.cuh:1-13): the ellipse/tile overlap walk is the
// "AccuTile" procedure of speedy-splat (https://github.com/j-alex-hanson/speedy-splat), itself based on "gaussian-splatting"
// by Inria and the Max Planck Institut fuer Informatik (MPII).  Original work (c) Inria and MPII, licensed under the
// Gaussian-Splatting License: use, reproduction and distribution of that work and its derivatives for non-commercial
// research and evaluation purposes only.  See NOTICE.md at the repository root.
#pragma once

struct SplatGeom {
    float A, B, C, inv_A, inv_C, disc, t, px, py;
    float bbox_min[2], bbox_max[2], argmin[2], argmax[2];  // [0]=x-ish, [1]=y-ish exactly as the reference's float2
    int rect_min[2], rect_max[2];
    bool visible;
};

__device__ __forceinline__ int lgs_f2i_rz(float x) { return __float2int_rz(x); }  // NaN -> 0, saturating

// x / T, correctly rounded.  For a power-of-two tile side the quotient is x * 2^-k, which is the same correctly rounded
// real number, so one FMUL replaces the ~10-instruction IEEE division sequence bit for bit (8x16, 16x16, 8x8 tiles).
template <int T>
__device__ __forceinline__ float lgs_div_tile(float x)
{
    if ((T & (T - 1)) == 0) return __fmul_rn(x, 1.0f / (float)T);
    return __fdiv_rn(x, (float)T);
}

// The two quotients by A (or C) are products with the splat's once-rounded reciprocal inv_A = 1/A (inv_C = 1/C): what the
// reference's own fast-math build does (x/c -> x * rcp(c)), one IEEE division per splat and axis instead of two per tile
// row, and the same operation sequence as the oracle (oracle_core.h: ellipse_isect).
__device__ __forceinline__ void lgs_ellipse_isect(float A, float B, float C, float inv_A, float inv_C, float disc, float t, float px,
                                                  float py, bool isY, float coord, float& lo, float& hi)
{
    float p_u = isY ? py : px;
    float p_v = isY ? px : py;
    float coeff = isY ? A : C;
    float inv = isY ? inv_A : inv_C;
    float h = __fsub_rn(coord, p_u);
    float sq = __fsqrt_rn(__fadd_rn(__fmul_rn(__fmul_rn(disc, h), h), __fmul_rn(t, coeff)));
    float nbh = __fmul_rn(-B, h);
    lo = __fadd_rn(__fmul_rn(__fsub_rn(nbh, sq), inv), p_v);
    hi = __fadd_rn(__fmul_rn(__fadd_rn(nbh, sq), inv), p_v);
}

// check_visibility=false reproduces the emit kernel, which trusts the count it was given
// (GR/binning.cu:63) and skips the ndc / depth tests.
// exact_bound: the last tile row / column of the rectangle is the one holding bbox_max, floor((bbox_max + T) / T), so a
// splat whose ellipse reaches pixel centre kT keeps tile k even when bbox_max < kT + 1.  false = the reference's
// floor((bbox_max + T - 1) / T) (GR/binning.cu:88-91), which treats bbox_max as an integer pixel bound and drops that tile
// (DESIGN.md section 7, D14).  The count and the emit of one list must use the same rule.
template <int TH, int TW>
__device__ __forceinline__ void lgs_splat_setup(float ndcx, float ndcy, float viewz, float A, float B, float C, float o,
                                                int H, int W, int gx, int gy, bool check_visibility, SplatGeom& g,
                                                bool exact_bound = true)
{
    g.A = A; g.B = B; g.C = C;
    g.disc = __fsub_rn(__fmul_rn(B, B), __fmul_rn(A, C));
    g.px = __fsub_rn(__fmul_rn(__fadd_rn(__fmul_rn(ndcx, 0.5f), 0.5f), (float)W), 0.5f);
    g.py = __fsub_rn(__fmul_rn(__fadd_rn(__fmul_rn(ndcy, 0.5f), 0.5f), (float)H), 0.5f);
    bool vis = true;
    if (check_visibility)
        vis = !((ndcx < -1.3f) || (ndcx > 1.3f) || (ndcy < -1.3f) || (ndcy > 1.3f) || (viewz <= 0.2f));
    vis = vis && !(o < __fdiv_rn(1.0f, 255.0f));
    vis = vis && (A > 0.0f) && (C > 0.0f) && (g.disc < 0.0f);
    g.visible = vis;
    if (!vis) return;
    float t = (float)(2.0 * log((double)__fmul_rn(o, 255.0f)));
    g.t = t;
    g.inv_A = __fdiv_rn(1.0f, A); g.inv_C = __fdiv_rn(1.0f, C);
    float bbt = __fmul_rn(__fmul_rn(B, B), t);
    float xt = __fsqrt_rn(__fdiv_rn(-bbt, __fmul_rn(g.disc, A)));
    xt = (B < 0.0f) ? xt : -xt;
    float yt = __fsqrt_rn(__fdiv_rn(-bbt, __fmul_rn(g.disc, C)));
    yt = (B < 0.0f) ? yt : -yt;
    g.argmin[0] = __fsub_rn(g.py, yt); g.argmin[1] = __fsub_rn(g.px, xt);
    g.argmax[0] = __fadd_rn(g.py, yt); g.argmax[1] = __fadd_rn(g.px, xt);
    float lo, hi;
    lgs_ellipse_isect(A, B, C, g.inv_A, g.inv_C, g.disc, t, g.px, g.py, true, g.argmin[0], lo, hi);  g.bbox_min[0] = lo;
    lgs_ellipse_isect(A, B, C, g.inv_A, g.inv_C, g.disc, t, g.px, g.py, false, g.argmin[1], lo, hi); g.bbox_min[1] = lo;
    lgs_ellipse_isect(A, B, C, g.inv_A, g.inv_C, g.disc, t, g.px, g.py, true, g.argmax[0], lo, hi);  g.bbox_max[0] = hi;
    lgs_ellipse_isect(A, B, C, g.inv_A, g.inv_C, g.disc, t, g.px, g.py, false, g.argmax[1], lo, hi); g.bbox_max[1] = hi;
    g.rect_min[0] = max(0, min(gx, lgs_f2i_rz(lgs_div_tile<TW>(g.bbox_min[0]))));
    g.rect_min[1] = max(0, min(gy, lgs_f2i_rz(lgs_div_tile<TH>(g.bbox_min[1]))));
    const float ex = __fadd_rn(g.bbox_max[0], (float)TW), ey = __fadd_rn(g.bbox_max[1], (float)TH);
    g.rect_max[0] = max(0, min(gx, lgs_f2i_rz(lgs_div_tile<TW>(exact_bound ? ex : __fsub_rn(ex, 1.0f)))));
    g.rect_max[1] = max(0, min(gy, lgs_f2i_rz(lgs_div_tile<TH>(exact_bound ? ey : __fsub_rn(ey, 1.0f)))));
}

// Walks the tile slices of one splat; returns the number of tiles and, when EMIT, writes
// (tile id + 1, idx) pairs number off, off+1, ... to keys/vals[k - lo] for those k inside the window
// [lo, lo + cap)  (lo = 0: plain bounds guard; lo > 0: staging a window of the list in shared memory).
template <int TH, int TW, bool EMIT, typename KeyT = int>
__device__ __forceinline__ int lgs_process_tiles(const SplatGeom& g, int gx, int idx, int off, int cap,
                                                 KeyT* __restrict__ keys, int* __restrict__ vals, int lo = 0)
{
    int y_span = g.rect_max[1] - g.rect_min[1], x_span = g.rect_max[0] - g.rect_min[0];
    if (y_span * x_span <= 0) return 0;
    const bool isY = y_span < x_span;
    const float BU = isY ? (float)TH : (float)TW;
    int rmin0 = isY ? g.rect_min[1] : g.rect_min[0], rmin1 = isY ? g.rect_min[0] : g.rect_min[1];
    int rmax0 = isY ? g.rect_max[1] : g.rect_max[0], rmax1 = isY ? g.rect_max[0] : g.rect_max[1];
    float bmin0 = isY ? g.bbox_min[1] : g.bbox_min[0], bmin1 = isY ? g.bbox_min[0] : g.bbox_min[1];
    float bmax0 = isY ? g.bbox_max[1] : g.bbox_max[0], bmax1 = isY ? g.bbox_max[0] : g.bbox_max[1];
    float amin1 = isY ? g.argmin[0] : g.argmin[1];
    float amax1 = isY ? g.argmax[0] : g.argmax[1];
    int count = 0;
    float imax_lo = bmax1, imax_hi = bmin1;
    float imin_lo, imin_hi;
    float min_line = __fmul_rn((float)rmin0, BU), max_line;
    if (bmin0 <= min_line) lgs_ellipse_isect(g.A, g.B, g.C, g.inv_A, g.inv_C, g.disc, g.t, g.px, g.py, isY, min_line, imin_lo, imin_hi);
    else { imin_lo = imax_lo; imin_hi = imax_hi; }
    for (int u = rmin0; u < rmax0; ++u) {
        max_line = __fadd_rn(min_line, BU);
        if (max_line <= bmax0) lgs_ellipse_isect(g.A, g.B, g.C, g.inv_A, g.inv_C, g.disc, g.t, g.px, g.py, isY, max_line, imax_lo, imax_hi);
        float emin, emax;
        if (min_line <= amin1 && amin1 < max_line) emin = bmin1; else emin = fminf(imin_lo, imax_lo);
        if (min_line <= amax1 && amax1 < max_line) emax = bmax1; else emax = fmaxf(imin_hi, imax_hi);
        // the slice runs along v: divide by the tile side in that direction (TW when slicing by rows, TH by columns)
        const float qmin = isY ? lgs_div_tile<TW>(emin) : lgs_div_tile<TH>(emin);
        const float qmax = isY ? lgs_div_tile<TW>(emax) : lgs_div_tile<TH>(emax);
        int min_v = max(rmin1, min(rmax1, lgs_f2i_rz(qmin)));
        int max_v = min(rmax1, max(rmin1, lgs_f2i_rz(__fadd_rn(qmax, 1.0f))));
        count += max_v - min_v;
        if (EMIT) {
            for (int v = min_v; v < max_v; v++) {
                int key = isY ? (u * gx + v) : (v * gx + u);
                unsigned rel = (unsigned)(off - lo);
                if (rel < (unsigned)cap) { keys[rel] = (KeyT)(key + 1); vals[rel] = idx; }
                off++;
            }
        }
        imin_lo = imax_lo; imin_hi = imax_hi;
        min_line = max_line;
    }
    return count;
}
