// binning.cu -- visibility + exact tile-overlap count, (tile, splat) pair emission in depth order,
// stable radix sort on the tile bits, tile ranges.      replaces GR/binning.cu (all of it)
//
// Ordering scheme (the reference's, because it moves the fewest bytes when pairs >> splats): splats are
// depth-sorted once (N keys), pairs are emitted in that order at scanned offsets, then ONE stable LSD
// radix sort over only the ceil(log2(tiles))+1 tile bits (2 passes at 1080p) groups them by tile while
// preserving depth order.  cub::DeviceRadixSort (CCCL, header-only) provides the onesweep passes.
#include <cub/device/device_radix_sort.cuh>   // lgs_create_table (reference-compatible Level A path)
#include <cub/device/device_scan.cuh>
#include <cub/iterator/transform_input_iterator.cuh>
#include <cub/iterator/counting_input_iterator.cuh>
#include "common.cuh"
#include "splat_geom.cuh"

// Level A tile rectangle: 1 = floor((bbox_max + T) / T), 0 = the reference's rule (lgs_set_exact_tile_bound, DESIGN.md D14)
static int g_exact_tile_bound = 1;
extern "C" int lgs_set_exact_tile_bound(int on) { g_exact_tile_bound = on ? 1 : 0; return LGS_OK; }

// ------------------------------------------------------------------------------------------------
// per-splat pixel bbox + tile count.                                  replaces GR/binning.cu:289-440
// ------------------------------------------------------------------------------------------------
template <int TH, int TW>
__global__ void __launch_bounds__(256) allocate_size_kernel(
    const float* __restrict__ ndc, const float* __restrict__ viewz, const float* __restrict__ inv_cov,
    const float* __restrict__ opac, const int* __restrict__ valid_length, int N, int H, int W, int gx, int gy, bool exact_bound,
    int* __restrict__ left_up, int* __restrict__ right_down, int* __restrict__ alloc)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    if (i >= N || (valid_length != nullptr && i >= valid_length[0])) return;
    size_t o4 = (size_t)b * 4 * N + i, o2 = (size_t)b * 2 * N + i;
    SplatGeom g;
    lgs_splat_setup<TH, TW>(ndc[o4], ndc[o4 + N], viewz[(size_t)b * N + i], inv_cov[o4], inv_cov[o4 + N],
                            inv_cov[o4 + 3 * (size_t)N], opac[i], H, W, gx, gy, true, g, exact_bound);
    if (g.visible) {
        left_up[o2] = lgs_f2i_rz(ceilf(g.bbox_min[0])); left_up[o2 + N] = lgs_f2i_rz(ceilf(g.bbox_min[1]));
        right_down[o2] = lgs_f2i_rz(floorf(g.bbox_max[0])); right_down[o2 + N] = lgs_f2i_rz(floorf(g.bbox_max[1]));
        alloc[(size_t)b * N + i] = lgs_process_tiles<TH, TW, false>(g, gx, i, 0, 0, (int*)nullptr, (int*)nullptr);
    } else {
        left_up[o2] = -1; left_up[o2 + N] = -1; right_down[o2] = -1; right_down[o2 + N] = -1;
        alloc[(size_t)b * N + i] = 0;
    }
}

extern "C" int lgs_get_allocate_size(const float* ndc, const float* view_space_z, const float* inv_cov2d, const float* opacity,
                                     const int* valid_length, int V, int N, int height, int width, int tile_h, int tile_w,
                                     int* left_up, int* right_down, int* allocate_size, void* stream)
{
    LGS_REQUIRE(lgs_tile_ok(tile_h, tile_w), "get_allocate_size: tile %dx%d not one of 8x16, 12x16, 16x16, 8x8", tile_h, tile_w);
    LGS_REQUIRE(V >= 1 && N >= 0, "get_allocate_size: bad sizes V=%d N=%d", V, N);
    cudaStream_t st = (cudaStream_t)stream;
    if (N == 0) return LGS_OK;
    // entries past valid_length read as 0 (the reference allocates the counts with torch::zeros)
    LGS_CUDA(cudaMemsetAsync(allocate_size, 0, sizeof(int) * (size_t)V * N, st));
    int gx = (width + tile_w - 1) / tile_w, gy = (height + tile_h - 1) / tile_h;
    dim3 grid(lgs_cdiv(N, 256), V);
    lgs_with_tile(tile_h, tile_w, [&](auto th, auto tw) {
        allocate_size_kernel<th, tw><<<grid, 256, 0, st>>>(ndc, view_space_z, inv_cov2d, opacity, valid_length, N, height, width,
                                                          gx, gy, g_exact_tile_bound != 0, left_up, right_down, allocate_size);
        return LGS_OK;
    });
    LGS_CHECK_LAUNCH("allocate_size_kernel");
    return LGS_OK;
}

// ------------------------------------------------------------------------------------------------
// emit (tile+1, splat) pairs in depth order.                          replaces GR/binning.cu:33-110
// ------------------------------------------------------------------------------------------------
template <int TH, int TW>
__global__ void __launch_bounds__(256) emit_pairs_kernel(
    const float* __restrict__ ndc, const float* __restrict__ inv_cov, const float* __restrict__ opac,
    const int* __restrict__ offset /*inclusive scan, depth order*/, const int64_t* __restrict__ sorted_id,
    int N, int cap, int H, int W, int gx, int gy, bool exact_bound, int* __restrict__ keys, int* __restrict__ vals)
{
    int j = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    if (j >= N) return;
    int off = j == 0 ? 0 : offset[(size_t)b * N + j - 1];
    int asz = offset[(size_t)b * N + j] - off;
    if (asz <= 0 || off + asz > cap) return;   // overflow beyond the allocation is dropped (GR/binning.cu:63)
    int i = (int)sorted_id[(size_t)b * N + j];
    size_t o4 = (size_t)b * 4 * N + i;
    SplatGeom g;
    lgs_splat_setup<TH, TW>(ndc[o4], ndc[o4 + N], 1.0f, inv_cov[o4], inv_cov[o4 + N], inv_cov[o4 + 3 * (size_t)N], opac[i],
                            H, W, gx, gy, false, g, exact_bound);
    if (g.visible) lgs_process_tiles<TH, TW, true>(g, gx, i, off, cap, keys + (size_t)b * cap, vals + (size_t)b * cap);
}

static inline int tile_bits(int tiles)
{
    int bit = 0;
    unsigned t = (unsigned)tiles;
    while (t >>= 1) bit++;
    return bit + 1;     // GR/binning.cu:199-202
}

extern "C" int lgs_create_table_workspace_bytes(int V, int cap, size_t* bytes)
{
    size_t tmp = 0;
    cub::DeviceRadixSort::SortPairs<int, int>(nullptr, tmp, nullptr, nullptr, nullptr, nullptr, cap, 0, 32);
    *bytes = ((tmp + 255) / 256) * 256 + 2 * sizeof(int) * (size_t)V * cap + 512;
    return LGS_OK;
}

// offset: inclusive scan of the depth-ordered counts [V,N]; depth_sorted_pointid int64 [V,N];
// outputs sorted_tile_id / sorted_point_id int32 [V,cap].
extern "C" int lgs_create_table(const float* ndc, const float* inv_cov2d, const float* opacity, const int* offset,
                                const int64_t* depth_sorted_pointid, int V, int N, int cap, int height, int width, int tile_h,
                                int tile_w, int* sorted_tile_id, int* sorted_point_id, void* workspace, size_t workspace_bytes,
                                void* stream)
{
    LGS_REQUIRE(lgs_tile_ok(tile_h, tile_w), "create_table: tile %dx%d not one of 8x16, 12x16, 16x16, 8x8", tile_h, tile_w);
    LGS_REQUIRE(cap > 0, "create_table: error pred_allocate_size (%d)", cap);
    size_t need = 0;
    lgs_create_table_workspace_bytes(V, cap, &need);
    if (workspace == nullptr || workspace_bytes < need) {
        lgs_set_error("create_table: workspace of %zu bytes needed, %zu given", need, workspace_bytes);
        return LGS_ERR_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    char* ws = (char*)(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
    int* keys = (int*)ws;
    int* vals = keys + (size_t)V * cap;
    void* cub_tmp = (void*)(((uintptr_t)(vals + (size_t)V * cap) + 255) & ~(uintptr_t)255);
    size_t cub_bytes = 0;
    cub::DeviceRadixSort::SortPairs<int, int>(nullptr, cub_bytes, nullptr, nullptr, nullptr, nullptr, cap, 0, 32);
    // unused slots keep key 0 and sort to the front (SURVEY Q2)
    LGS_CUDA(cudaMemsetAsync(keys, 0, sizeof(int) * (size_t)V * cap, st));
    LGS_CUDA(cudaMemsetAsync(vals, 0, sizeof(int) * (size_t)V * cap, st));
    int gx = (width + tile_w - 1) / tile_w, gy = (height + tile_h - 1) / tile_h;
    if (N > 0) {
        dim3 grid(lgs_cdiv(N, 256), V);
        lgs_with_tile(tile_h, tile_w, [&](auto th, auto tw) {
            emit_pairs_kernel<th, tw><<<grid, 256, 0, st>>>(ndc, inv_cov2d, opacity, offset, depth_sorted_pointid, N, cap, height,
                                                           width, gx, gy, g_exact_tile_bound != 0, keys, vals);
            return LGS_OK;
        });
        LGS_CHECK_LAUNCH("emit_pairs_kernel");
    }
    int bits = tile_bits(gx * gy);
    for (int b = 0; b < V; b++) {
        LGS_CUDA(cub::DeviceRadixSort::SortPairs<int, int>(cub_tmp, cub_bytes, keys + (size_t)b * cap, sorted_tile_id + (size_t)b * cap,
                                                           vals + (size_t)b * cap, sorted_point_id + (size_t)b * cap, cap, 0, bits, st));
    }
    return LGS_OK;
}

// ------------------------------------------------------------------------------------------------
// tile ranges.                                                        replaces GR/binning.cu:228-287
// range[t] = first index of key t or -1; range[t+1] is the end marker.  fix_last closes the last
// populated tile, which the reference leaves open so that it renders empty (SURVEY Q3).
// ------------------------------------------------------------------------------------------------
__global__ void fill_int_kernel(int* __restrict__ p, int v, size_t n)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}

// The table by search: entry t only depends on where key t would be inserted in the sorted list, so one warp per tile does
// one lower_bound instead of the whole list being streamed once -- 16k warps x 5 probe rounds instead of 22 MB at 1080p.
// KeyT = int (op-level table) or unsigned short (fused pipeline when tiles+1 < 65536).  The rules:
//   populated t                      -> first index of t
//   empty t right after a populated  -> that tile's end (its successor's start); for the LAST populated tile only if fix_last
//   t = max_tile + 1                 -> L
//   anything else                    -> -1
template <typename KeyT>
__global__ void __launch_bounds__(256) tile_range_bsearch_kernel(const KeyT* __restrict__ keys, int L, int max_tile, int fix_last,
                                                                 int* __restrict__ range, const int* __restrict__ L_dev)
{
    if (L_dev != nullptr) L = min(L, max(*L_dev, 0));         // GPU-driven sizing: L is the capacity, *L_dev the live length
    // one WARP per tile: a 32-ary search (each lane probes the last key of one of 32 segments, a ballot counts the segments
    // that lie entirely below t) needs 5 rounds of independent loads at 1080p where a binary search needs 24 dependent ones
    const int lane = threadIdx.x & 31;
    const int t = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), b = blockIdx.y;
    if (t > max_tile + 1) return;
    const KeyT* k = keys + (size_t)b * L;
    int lo = 0, hi = L;                                     // lower_bound(t) lies in [lo, hi]
    while (hi - lo > 32) {
        const int stride = (hi - lo + 31) >> 5;
        const int probe = min(hi - 1, lo + lane * stride + stride - 1);
        const int c = __popc(__ballot_sync(0xffffffffu, (int)k[probe] < t));     // keys are sorted: the predicate is 1..1 0..0
        lo = min(hi, lo + c * stride);
        hi = min(hi, lo + stride);
    }
    {
        const bool below = lo + lane < hi && (int)k[lo + lane] < t;
        lo += __popc(__ballot_sync(0xffffffffu, below));
    }
    if (lane != 0) return;
    int r = -1;
    if (lo < L && (int)k[lo] == t) r = lo;
    else if (t >= 1 && lo > 0 && (int)k[lo - 1] == t - 1 && (lo < L || fix_last)) r = lo;
    if (t == max_tile + 1) r = L;
    range[(size_t)b * (max_tile + 2) + t] = r;
}

template <typename KeyT>
static int tile_range_launch(const KeyT* keys, int V, int L, int max_tile, int fix_last, int* range, cudaStream_t st,
                             const int* L_dev = nullptr)
{
    if (L_dev != nullptr) {
        LGS_REQUIRE(V == 1, "tile_range: the device-side length form handles one view per call");
        tile_range_bsearch_kernel<KeyT><<<dim3(lgs_cdiv(max_tile + 2, 8), V), 256, 0, st>>>(keys, L, max_tile, fix_last, range, L_dev);
        LGS_CHECK_LAUNCH("tile_range_bsearch_kernel");
        return LGS_OK;
    }
    if (L <= 0) {
        size_t n = (size_t)V * (max_tile + 2);
        fill_int_kernel<<<lgs_cdiv((long long)n, 256), 256, 0, st>>>(range, -1, n);
        LGS_CHECK_LAUNCH("fill_int_kernel");
        return LGS_OK;
    }
    tile_range_bsearch_kernel<KeyT><<<dim3(lgs_cdiv(max_tile + 2, 8), V), 256, 0, st>>>(keys, L, max_tile, fix_last, range, nullptr);
    LGS_CHECK_LAUNCH("tile_range_bsearch_kernel");
    return LGS_OK;
}

extern "C" int lgs_tile_range(const int* table_tile_id, int V, int table_length, int max_tile_id, int fix_last, int* tile_range,
                              void* stream)
{
    LGS_REQUIRE(V >= 1 && table_length >= 0 && max_tile_id >= 0, "tileRange: bad sizes V=%d L=%d max_tile=%d", V, table_length, max_tile_id);
    return tile_range_launch<int>(table_tile_id, V, table_length, max_tile_id, fix_last, tile_range, (cudaStream_t)stream);
}

// device-side length forms (GPU-driven sizing: `capacity` bounds the launch, *length_dev is the live length)
extern "C" int lgs_tile_range_u16_dev(const unsigned short* table_tile_id, int capacity, const int* length_dev, int max_tile_id,
                                      int fix_last, int* tile_range, void* stream)
{
    LGS_REQUIRE(capacity >= 0 && length_dev != nullptr && max_tile_id >= 0 && max_tile_id < 65535, "tileRange(u16,dev): bad arguments");
    return tile_range_launch<unsigned short>(table_tile_id, 1, capacity, max_tile_id, fix_last, tile_range, (cudaStream_t)stream, length_dev);
}

extern "C" int lgs_tile_range_dev(const int* table_tile_id, int capacity, const int* length_dev, int max_tile_id, int fix_last,
                                  int* tile_range, void* stream)
{
    LGS_REQUIRE(capacity >= 0 && length_dev != nullptr && max_tile_id >= 0, "tileRange(dev): bad arguments");
    return tile_range_launch<int>(table_tile_id, 1, capacity, max_tile_id, fix_last, tile_range, (cudaStream_t)stream, length_dev);
}

// ------------------------------------------------------------------------------------------------
// building block for the fused pipeline: "gather + inclusive scan"   (the radix sorts live in sort.cu)
// ------------------------------------------------------------------------------------------------
struct GatherCount {
    const int* counts; const unsigned* order; const int* n_dev;     // n_dev (nullable): items at or past *n_dev count as 0
    __host__ __device__ int operator()(int j) const
    {
#ifdef __CUDA_ARCH__
        if (n_dev != nullptr && j >= *n_dev) return 0;
#endif
        return counts[order[j]];
    }
};

extern "C" int lgs_scan_gathered_workspace_bytes(int n, size_t* bytes)
{
    size_t tmp = 0;
    cub::CountingInputIterator<int> cnt(0);
    GatherCount op{ nullptr, nullptr, nullptr };
    cub::TransformInputIterator<int, GatherCount, cub::CountingInputIterator<int>> it(cnt, op);
    cub::DeviceScan::InclusiveSum(nullptr, tmp, it, (int*)nullptr, n);
    *bytes = tmp + 256;
    return LGS_OK;
}

// out[j] = sum_{k<=j} counts[order[k]]   (inclusive, int32) over `capacity` items; items at or past *n_dev contribute 0
// (their `order` entries are never read)
extern "C" int lgs_scan_gathered_dev(const int* counts, const unsigned* order, int capacity, const int* n_dev, int* out, void* workspace,
                                     size_t workspace_bytes, void* stream)
{
    LGS_REQUIRE(n_dev != nullptr, "scan_gathered_dev: n_dev is NULL");
    if (capacity <= 0) return LGS_OK;
    cub::CountingInputIterator<int> cnt(0);
    GatherCount op{ counts, order, n_dev };
    cub::TransformInputIterator<int, GatherCount, cub::CountingInputIterator<int>> it(cnt, op);
    size_t need = 0;
    cub::DeviceScan::InclusiveSum(nullptr, need, it, out, capacity);
    void* ws = (void*)(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
    if (workspace == nullptr || workspace_bytes < need + 256) {
        lgs_set_error("scan_gathered: workspace of %zu bytes needed, %zu given", need + 256, workspace_bytes);
        return LGS_ERR_WORKSPACE;
    }
    LGS_CUDA(cub::DeviceScan::InclusiveSum(ws, need, it, out, capacity, (cudaStream_t)stream));
    return LGS_OK;
}
