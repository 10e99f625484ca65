// sort.cu -- stable LSD radix sort of (key, value) pairs on a bit range: the depth sort (N float-bit keys)
// and the tile sort (D pairs, tile bits only) of the fused pipeline.     replaces torch.sort at
// wrapper.py:739 and cub::DeviceRadixSort::SortPairs at GR/binning.cu:204-221
//
// Two implementations behind the same entry points (lgs_set_sort_impl / env LGS_SORT):
//   * "lgs" (default): per pass   histogram (digit x block table) -> per-digit exclusive scan over the blocks ->
//     scatter.  The scatter ranks a block's tile of keys warp by warp with same-digit lane masks built by
//     shared-memory atomicOr (stable, and never worse than a 32-way conflict on a constant digit),
//     orders the tile in shared memory and writes it out as one coalesced run per digit.  Digit width is
//     chosen per call so that ceil(bits / passes) bits are sorted per pass: 14 tile bits = 2 x 7,
//     16 = 2 x 8, 24 depth bits = 3 x 8.  Blocks are 256 threads x 8 or 16 keys, so a 1M-key depth sort
//     still launches 490 blocks (cub's onesweep launches 109 blocks of 384 x 23 keys on the same input).
//   * "cub": cub::DeviceRadixSort::SortPairs (onesweep), kept as the cross-check and fallback.
// Both are stable and sort exactly the bits [begin_bit, end_bit); results are bit-identical.
#include <cub/device/device_radix_sort.cuh>
#include <cub/block/block_scan.cuh>
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include "common.cuh"

namespace {

constexpr int RS_THREADS = 256;
constexpr int RS_WARPS = RS_THREADS / 32;
constexpr int RS_MAXBINS = 256;          // == RS_THREADS: thread t owns digit t in the block-wide steps

int g_sort_impl = -1;                    // -1: read LGS_SORT on first use; 0 cub; 1 lgs
bool g_sort_forced = false;              // LGS_SORT / lgs_set_sort_impl given: no automatic choice

int sort_impl()
{
    if (g_sort_impl < 0) {
        const char* e = getenv("LGS_SORT");
        g_sort_forced = e != nullptr;
        g_sort_impl = (e != nullptr && strcmp(e, "cub") == 0) ? 0 : 1;
    }
    return g_sort_impl;
}

// Automatic choice when nothing is forced: the own passes up to 7-bit digits (1080p: 14 tile bits = 2 x 7), cub's onesweep when
// the tile ids need 8-bit digits on more than 8 M pairs (4K: 16 bits, 71.7 M pairs) -- profiles/microbench/dev_count_bench.py
// times both.
int sort_impl_for(int n, int bits)
{
    int impl = sort_impl();
    if (!g_sort_forced && impl == 1 && bits > 14 && n > (8 << 20)) impl = 0;
    return impl;
}

__device__ __forceinline__ unsigned lanemask_lt()
{
    unsigned m;
    asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
    return m;
}

// table[digit * nblocks + block] = number of keys of this block's tile with that digit.  Per-warp private
// shared-memory histograms fed by one ATOMS per key (16-byte key loads when the tile is whole and aligned).
template <typename KeyT, int IPT, bool VEC>
__global__ void __launch_bounds__(RS_THREADS) rs_hist_kernel(const KeyT* __restrict__ keys, int n, int shift, int nbins, int nblocks,
                                                             int* __restrict__ table, unsigned bias, const int* __restrict__ n_dev,
                                                             const unsigned* __restrict__ bias_dev)
{
    constexpr int TILE = RS_THREADS * IPT;
    constexpr int KPV = 16 / (int)sizeof(KeyT);                 // keys per 16-byte vector
    __shared__ int h[RS_WARPS][RS_MAXBINS];
    const int t = threadIdx.x, w = t >> 5;
    // GPU-driven sizing: the launch covers the CAPACITY n, the live count / key bias are read on the device (no host sync)
    if (n_dev != nullptr) n = min(n, max(*n_dev, 0));
    if (bias_dev != nullptr) bias = *bias_dev;
    const int base = blockIdx.x * TILE;
    if (base >= n) {                                            // block past the live range: an all-zero column
        if (t < nbins) table[(size_t)t * nblocks + blockIdx.x] = 0;
        return;
    }
#pragma unroll
    for (int k = 0; k < RS_WARPS; k++) h[k][t] = 0;
    __syncthreads();
    const unsigned mask = (unsigned)nbins - 1u;
    int* hw = h[w];
    if (VEC && base + TILE <= n) {
        const uint4* v = reinterpret_cast<const uint4*>(keys + base);
#pragma unroll
        for (int j = 0; j < IPT / KPV; j++) {
            uint4 q = v[j * RS_THREADS + t];
            unsigned x[4] = { q.x, q.y, q.z, q.w };
#pragma unroll
            for (int c = 0; c < 4; c++) {
                if (sizeof(KeyT) == 2) {
                    atomicAdd(&hw[(((x[c] & 0xffffu) - bias) >> shift) & mask], 1);
                    atomicAdd(&hw[(((x[c] >> 16) - bias) >> shift) & mask], 1);
                } else {
                    atomicAdd(&hw[((x[c] - bias) >> shift) & mask], 1);
                }
            }
        }
    } else {
#pragma unroll
        for (int i = 0; i < IPT; i++) {
            int idx = base + i * RS_THREADS + t;
            if (idx < n) atomicAdd(&hw[(((unsigned)keys[idx] - bias) >> shift) & mask], 1);
        }
    }
    __syncthreads();
    if (t < nbins) {
        int c = 0;
#pragma unroll
        for (int k = 0; k < RS_WARPS; k++) c += h[k][t];
        table[(size_t)t * nblocks + blockIdx.x] = c;
    }
}

// one block per digit: table row -> its exclusive scan over the blocks, totals[digit] = row sum
__global__ void __launch_bounds__(RS_THREADS) rs_scan_rows_kernel(int* __restrict__ table, int nblocks, int* __restrict__ totals)
{
    using BlockScan = cub::BlockScan<int, RS_THREADS>;
    __shared__ typename BlockScan::TempStorage s_scan;
    int* row = table + (size_t)blockIdx.x * nblocks;
    const int per = (nblocks + RS_THREADS - 1) / RS_THREADS;
    const int lo = min(nblocks, (int)threadIdx.x * per), hi = min(nblocks, lo + per);
    int sum = 0;
    for (int k = lo; k < hi; k++) sum += row[k];
    int pre, tot;
    BlockScan(s_scan).ExclusiveSum(sum, pre, tot);
    for (int k = lo; k < hi; k++) { int c = row[k]; row[k] = pre; pre += c; }
    if (threadIdx.x == 0) totals[blockIdx.x] = tot;
}

// table[d * nblocks + b] = keys with digit d in blocks before b;  totals[d] = keys with digit d
// NS = keys of a lane ranked per round of the warp-level ranking (1, 2 or 4): each of the NS items ORs its lane bit into its OWN set
// of match slots, one __syncwarp later item j reads the count of its digit, the group sizes of that digit in the items before it
// and its own group's mask -- all independent loads -- and the highest lane of every group publishes the group size with one
// ATOMS.ADD.  The three warp barriers and the dependent ATOMS -> LDS -> STS chain of a round are paid once per NS keys instead of
// once per key (the per-key form is latency bound).
template <typename KeyT, int IPT, int NS>
__global__ void __launch_bounds__(RS_THREADS, IPT == 16 ? 3 : 4) rs_scatter_kernel(const KeyT* __restrict__ kin, const unsigned* __restrict__ vin,
                                                                KeyT* __restrict__ kout, unsigned* __restrict__ vout, int n, int shift,
                                                                int nbins, int nblocks, const int* __restrict__ table,
                                                                const int* __restrict__ totals, unsigned bias,
                                                                const int* __restrict__ n_dev, const unsigned* __restrict__ bias_dev)
{
    constexpr int TILE = RS_THREADS * IPT;
    static_assert(IPT % NS == 0, "the ranking rounds must tile the items of a lane");
    if (n_dev != nullptr) n = min(n, max(*n_dev, 0));
    if (bias_dev != nullptr) bias = *bias_dev;
    if ((int)blockIdx.x * TILE >= n) return;
    using BlockScan = cub::BlockScan<int, RS_THREADS>;
    __shared__ int s_cnt[RS_WARPS][RS_MAXBINS];
    __shared__ int s_gofs[RS_MAXBINS];
    __shared__ KeyT s_k[TILE];
    __shared__ unsigned s_v[TILE];
    unsigned* s_match = s_v;                 // [NS][RS_WARPS][nbins] match slots, live only while ranking (host: NS*RS_WARPS*nbins <= TILE)
    __shared__ typename BlockScan::TempStorage s_scan;
    const int t = threadIdx.x, lane = t & 31, w = t >> 5;
    const int base = blockIdx.x * TILE;
    const int nvalid = min(TILE, n - base);
    const unsigned mask = (unsigned)nbins - 1u;
    const unsigned lt = lanemask_lt();
#pragma unroll
    for (int k = 0; k < RS_WARPS; k++) s_cnt[k][t] = 0;
    for (int k = t; k < NS * RS_WARPS * nbins; k += RS_THREADS) s_match[k] = 0u;
    // warp-striped tile: item i of lane l of warp w is element w*32*IPT + i*32 + l, so (w, i, l) order is index order
    KeyT key[IPT];
    unsigned val[IPT];
    unsigned short rank[IPT];
#pragma unroll
    for (int i = 0; i < IPT; i++) {
        int loc = w * 32 * IPT + i * 32 + lane;
        bool valid = loc < nvalid;
        key[i] = valid ? kin[base + loc] : (KeyT)(bias - 1u);   // padding: digit of all ones, ranks after every real key of it
        val[i] = valid ? vin[base + loc] : 0u;
    }
    // first output slot of each digit (exclusive scan of the totals) + this block's offset inside the digit
    int gdig;
    {
        int tot_d = t < nbins ? totals[t] : 0;
        BlockScan(s_scan).ExclusiveSum(tot_d, gdig);
        if (t < nbins) gdig += table[(size_t)t * nblocks + blockIdx.x];
    }
    __syncthreads();
    unsigned* mw = s_match + w * nbins;            // this warp's slots of set 0; set q is NS-strided by RS_WARPS * nbins
    const int set_stride = RS_WARPS * nbins;
#pragma unroll
    for (int i0 = 0; i0 < IPT; i0 += NS) {
        // lanes of this warp holding the same digit: OR the lane bits into the digit's slot (one ATOMS; MATCH.ANY
        // issues at a low rate and alone bounded this kernel, eight ballots cost ~32 issue slots)
        unsigned d[NS];
#pragma unroll
        for (int q = 0; q < NS; q++) {
            d[q] = (((unsigned)key[i0 + q] - bias) >> shift) & mask;
            atomicOr(&mw[q * set_stride + d[q]], 1u << lane);
        }
        __syncwarp();
        unsigned own[NS];
#pragma unroll
        for (int j = 0; j < NS; j++) {
            int r = s_cnt[w][d[j]];
#pragma unroll
            for (int q = 0; q < j; q++) r += __popc(mw[q * set_stride + d[j]]);     // same digit in the earlier items of the round
            own[j] = mw[j * set_stride + d[j]];
            rank[i0 + j] = (unsigned short)(r + __popc(own[j] & lt));
        }
        __syncwarp();
#pragma unroll
        for (int j = 0; j < NS; j++) {
            if ((own[j] >> lane) <= 1u) {          // highest lane of the group publishes the group size and clears the slot
                if (NS == 1) s_cnt[w][d[j]] = (int)rank[i0 + j] + 1;
                else atomicAdd(&s_cnt[w][d[j]], __popc(own[j]));
                mw[j * set_stride + d[j]] = 0u;
            }
        }
        __syncwarp();
    }
    __syncthreads();
    // digit t: exclusive scan of the per-warp counts, then of the digit totals across the block
    int tot = 0;
#pragma unroll
    for (int k = 0; k < RS_WARPS; k++) { int c = s_cnt[k][t]; s_cnt[k][t] = tot; tot += c; }
    int dbase;
    BlockScan(s_scan).ExclusiveSum(tot, dbase);
#pragma unroll
    for (int k = 0; k < RS_WARPS; k++) s_cnt[k][t] += dbase;
    s_gofs[t] = gdig - dbase;
    __syncthreads();
#pragma unroll
    for (int i = 0; i < IPT; i++) {
        unsigned d = (((unsigned)key[i] - bias) >> shift) & mask;
        int p = s_cnt[w][d] + rank[i];
        s_k[p] = key[i];
        s_v[p] = val[i];
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < IPT; i++) {
        int k = i * RS_THREADS + t;
        if (k < nvalid) {
            KeyT kk = s_k[k];
            int dst = s_gofs[(((unsigned)kk - bias) >> shift) & mask] + k;
            kout[dst] = kk;
            vout[dst] = s_v[k];
        }
    }
}

// ---- single-read-per-pass form ("onesweep"): global digit histograms of ALL passes in one read of the keys, then one kernel
// per pass that ranks a tile, obtains the number of same-digit keys in all EARLIER tiles by decoupled look-back (each tile
// publishes its per-digit counts, then its inclusive prefix, in one 32-bit word per digit: 2 flag bits + 30-bit count) and
// scatters.  Against the histogram / row-scan / scatter passes above this removes, per pass, one full read of the keys and two
// latency-bound launches.
// The ranking and the shared-memory reorder are the ones of rs_scatter_kernel.  Tiles take their index from an atomic ticket, so a
// tile's predecessors have always started: the look-back cannot dead-lock whatever order the hardware dispatches CTAs in.
constexpr unsigned LB_AGG = 1u << 30, LB_INC = 2u << 30, LB_MASK = (1u << 30) - 1u;
constexpr int RS_MAXPASS = 4;

struct GhistArgs { int shift[RS_MAXPASS]; int nbins[RS_MAXPASS]; int passes; };

template <typename KeyT, int IPT>
__global__ void __launch_bounds__(RS_THREADS) rs_ghist_kernel(const KeyT* __restrict__ keys, int n, GhistArgs A, int* __restrict__ ghist,
                                                              unsigned bias, const int* __restrict__ n_dev,
                                                              const unsigned* __restrict__ bias_dev)
{
    constexpr int TILE = RS_THREADS * IPT;
    __shared__ int h[RS_MAXPASS][RS_MAXBINS];
    const int t = threadIdx.x;
    if (n_dev != nullptr) n = min(n, max(*n_dev, 0));
    if (bias_dev != nullptr) bias = *bias_dev;
    const int base = blockIdx.x * TILE;
    if (base >= n) return;
    for (int p = 0; p < A.passes; p++) h[p][t] = 0;
    __syncthreads();
#pragma unroll
    for (int i = 0; i < IPT; i++) {
        const int idx = base + i * RS_THREADS + t;
        if (idx < n) {
            const unsigned k = (unsigned)keys[idx] - bias;
            for (int p = 0; p < A.passes; p++) atomicAdd(&h[p][(k >> A.shift[p]) & (unsigned)(A.nbins[p] - 1)], 1);
        }
    }
    __syncthreads();
    for (int p = 0; p < A.passes; p++)
        if (t < A.nbins[p] && h[p][t] != 0) atomicAdd(&ghist[p * RS_MAXBINS + t], h[p][t]);
}

template <typename KeyT, int IPT>
__global__ void __launch_bounds__(RS_THREADS) rs_onesweep_kernel(const KeyT* __restrict__ kin, const unsigned* __restrict__ vin,
                                                                 KeyT* __restrict__ kout, unsigned* __restrict__ vout, int n, int shift,
                                                                 int nbins, const int* __restrict__ ghist /* this pass: [RS_MAXBINS] */,
                                                                 unsigned* __restrict__ status /* this pass: [tiles][nbins] */,
                                                                 int* __restrict__ ticket, unsigned bias, const int* __restrict__ n_dev,
                                                                 const unsigned* __restrict__ bias_dev)
{
    constexpr int TILE = RS_THREADS * IPT;
    using BlockScan = cub::BlockScan<int, RS_THREADS>;
    __shared__ int s_cnt[RS_WARPS][RS_MAXBINS];
    __shared__ int s_gofs[RS_MAXBINS];
    __shared__ KeyT s_k[TILE];
    __shared__ unsigned s_v[TILE];
    __shared__ int s_tile;
    static_assert(TILE >= RS_WARPS * RS_MAXBINS, "the match slots alias the value staging buffer");
    unsigned (*s_match)[RS_MAXBINS] = reinterpret_cast<unsigned (*)[RS_MAXBINS]>(s_v);
    __shared__ typename BlockScan::TempStorage s_scan;
    const int t = threadIdx.x, lane = t & 31, w = t >> 5;
    if (n_dev != nullptr) n = min(n, max(*n_dev, 0));
    if (bias_dev != nullptr) bias = *bias_dev;
    if (t == 0) s_tile = atomicAdd(ticket, 1);
#pragma unroll
    for (int k = 0; k < RS_WARPS; k++) { s_cnt[k][t] = 0; s_match[k][t] = 0u; }
    __syncthreads();
    const int tile = s_tile;
    const int base = tile * TILE;
    if (base >= n) return;                                   // (uniform) tickets past the live range have nothing to do
    const int nvalid = min(TILE, n - base);
    const unsigned mask = (unsigned)nbins - 1u;
    const unsigned lt = lanemask_lt();
    KeyT key[IPT];
    unsigned val[IPT];
    unsigned short rank[IPT];
#pragma unroll
    for (int i = 0; i < IPT; i++) {
        int loc = w * 32 * IPT + i * 32 + lane;
        bool valid = loc < nvalid;
        key[i] = valid ? kin[base + loc] : (KeyT)(bias - 1u);   // padding: digit of all ones, ranks after every real key of it
        val[i] = valid ? vin[base + loc] : 0u;
    }
    // first output slot of each digit over the whole input (exclusive scan of the global histogram)
    int gdig;
    {
        int tot_d = t < nbins ? ghist[t] : 0;
        BlockScan(s_scan).ExclusiveSum(tot_d, gdig);
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < IPT; i++) {
        unsigned d = (((unsigned)key[i] - bias) >> shift) & mask;
        atomicOr(&s_match[w][d], 1u << lane);
        __syncwarp();
        unsigned m = s_match[w][d];
        int r = s_cnt[w][d] + __popc(m & lt);
        rank[i] = (unsigned short)r;
        __syncwarp();
        if ((m >> lane) <= 1u) { s_cnt[w][d] = r + 1; s_match[w][d] = 0u; }
        __syncwarp();
    }
    __syncthreads();
    // digit t: exclusive scan of the per-warp counts -> this tile's count of digit t (padding keys excluded below)
    int tot = 0;
#pragma unroll
    for (int k = 0; k < RS_WARPS; k++) { int c = s_cnt[k][t]; s_cnt[k][t] = tot; tot += c; }
    // real keys of digit t in this tile: the padding keys all carry the all-ones digit of (bias - 1) - bias = 0xffff.. -> mask
    int real = tot;
    if (t == (int)mask) real -= (TILE - nvalid);
    // decoupled look-back over the earlier tiles
    if (t < nbins) {
        volatile unsigned* st_ = status + (size_t)tile * nbins;
        st_[t] = LB_AGG | (unsigned)real;
        unsigned prefix = 0u;
        for (int i = tile - 1; i >= 0;) {
            const unsigned v = *((volatile unsigned*)(status + (size_t)i * nbins + t));
            const unsigned flag = v & ~LB_MASK;
            if (flag == 0u) continue;                        // predecessor has not published yet (it has started: tickets)
            prefix += v & LB_MASK;
            if (flag == LB_INC) break;
            i--;
        }
        st_[t] = LB_INC | (prefix + (unsigned)real);
        gdig += (int)prefix;
    }
    int dbase;
    BlockScan(s_scan).ExclusiveSum(tot, dbase);
#pragma unroll
    for (int k = 0; k < RS_WARPS; k++) s_cnt[k][t] += dbase;
    s_gofs[t] = gdig - dbase;
    __syncthreads();
#pragma unroll
    for (int i = 0; i < IPT; i++) {
        unsigned d = (((unsigned)key[i] - bias) >> shift) & mask;
        int p = s_cnt[w][d] + rank[i];
        s_k[p] = key[i];
        s_v[p] = val[i];
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < IPT; i++) {
        int k = i * RS_THREADS + t;
        if (k < nvalid) {
            KeyT kk = s_k[k];
            int dst = s_gofs[(((unsigned)kk - bias) >> shift) & mask] + k;
            kout[dst] = kk;
            vout[dst] = s_v[k];
        }
    }
}

struct RsPlan {
    int ipt, tile, nblocks, passes, dbits;
    size_t table_bytes, scan_bytes, total_bytes, off_scan, off_keys, off_vals;
};

inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

template <typename KeyT>
RsPlan rs_plan(int n, int begin_bit, int end_bit)
{
    RsPlan p;
    static const int forced_ipt = getenv("LGS_RS_IPT") ? atoi(getenv("LGS_RS_IPT")) : 0;      // A/B knob: 8 | 16
    p.ipt = (forced_ipt == 8 || forced_ipt == 16) ? forced_ipt : (n > (1 << 22) ? 16 : 8);
    p.tile = RS_THREADS * p.ipt;
    p.nblocks = (n + p.tile - 1) / p.tile;
    int bits = end_bit - begin_bit;
    p.passes = bits <= 0 ? 0 : (bits + 7) / 8;
    p.dbits = p.passes == 0 ? 0 : (bits + p.passes - 1) / p.passes;
    // table: [digit][block] counts of one pass (pass form)  |  look-back status words of up to RS_MAXPASS passes (onesweep form)
    p.table_bytes = align256((size_t)RS_MAXPASS * RS_MAXBINS * p.nblocks * sizeof(int));
    p.scan_bytes = align256((RS_MAXPASS * RS_MAXBINS + 64) * sizeof(int));          // digit totals | global histograms + tickets
    p.off_scan = p.table_bytes;
    p.off_keys = p.off_scan + p.scan_bytes;
    p.off_vals = p.off_keys + align256((size_t)n * sizeof(KeyT));
    p.total_bytes = p.off_vals + align256((size_t)n * sizeof(unsigned));
    return p;
}

bool rs_use_onesweep();
template <typename KeyT>
int rs_sort_onesweep(const KeyT* keys_in, KeyT* keys_out, const unsigned* vals_in, unsigned* vals_out, int n, int begin_bit, int end_bit,
                     unsigned bias, char* ws, cudaStream_t st, const int* n_dev, const unsigned* bias_dev);

template <typename KeyT>
int rs_sort(const KeyT* keys_in, KeyT* keys_out, const unsigned* vals_in, unsigned* vals_out, int n, int begin_bit, int end_bit,
            unsigned bias, char* ws, cudaStream_t st, const int* n_dev = nullptr, const unsigned* bias_dev = nullptr)
{
    RsPlan p = rs_plan<KeyT>(n, begin_bit, end_bit);
    if (p.passes == 0) {
        LGS_REQUIRE(n_dev == nullptr, "sort_pairs: a device-side count needs at least one pass");
        LGS_CUDA(cudaMemcpyAsync(keys_out, keys_in, (size_t)n * sizeof(KeyT), cudaMemcpyDeviceToDevice, st));
        LGS_CUDA(cudaMemcpyAsync(vals_out, vals_in, (size_t)n * sizeof(unsigned), cudaMemcpyDeviceToDevice, st));
        return LGS_OK;
    }
    if (rs_use_onesweep())
        return rs_sort_onesweep<KeyT>(keys_in, keys_out, vals_in, vals_out, n, begin_bit, end_bit, bias, ws, st, n_dev, bias_dev);
    int* table = (int*)ws;
    int* totals = (int*)(ws + p.off_scan);
    KeyT* ktmp = (KeyT*)(ws + p.off_keys);
    unsigned* vtmp = (unsigned*)(ws + p.off_vals);
    const KeyT* ksrc = keys_in;
    const unsigned* vsrc = vals_in;
    int bit = begin_bit;
    for (int pass = 0; pass < p.passes; pass++) {
        int dbits = min(p.dbits, end_bit - bit);
        int nbins = 1 << dbits;
        bool to_out = ((p.passes - 1 - pass) & 1) == 0;
        KeyT* kdst = to_out ? keys_out : ktmp;
        unsigned* vdst = to_out ? vals_out : vtmp;
        const bool vec = ((uintptr_t)ksrc & 15) == 0;
        lgs_with_flags([&](auto ipt16, auto v) {
            rs_hist_kernel<KeyT, ipt16 ? 16 : 8, v><<<p.nblocks, RS_THREADS, 0, st>>>(ksrc, n, bit, nbins, p.nblocks, table, bias, n_dev,
                                                                                     bias_dev);
            return LGS_OK;
        }, p.ipt == 16, vec);
        LGS_CHECK_LAUNCH("rs_hist_kernel");
        rs_scan_rows_kernel<<<nbins, RS_THREADS, 0, st>>>(table, p.nblocks, totals);
        LGS_CHECK_LAUNCH("rs_scan_rows_kernel");
        // keys ranked per round: as many as the match slots fit in the value staging buffer they alias (env LGS_RS_RANK caps it: A/B)
        static const int rank_cap = getenv("LGS_RS_RANK") ? atoi(getenv("LGS_RS_RANK")) : 2;
        int ns = 1;
        while (ns < 4 && ns * 2 <= rank_cap && ns * 2 * RS_WARPS * nbins <= p.tile) ns *= 2;
        lgs_with_flags([&](auto ipt16, auto ns4, auto ns2) {
            rs_scatter_kernel<KeyT, ipt16 ? 16 : 8, ns4 ? 4 : ns2 ? 2 : 1><<<p.nblocks, RS_THREADS, 0, st>>>(
                ksrc, vsrc, kdst, vdst, n, bit, nbins, p.nblocks, table, totals, bias, n_dev, bias_dev);
            return LGS_OK;
        }, p.ipt == 16, ns == 4, ns == 2);
        LGS_CHECK_LAUNCH("rs_scatter_kernel");
        ksrc = kdst; vsrc = vdst;
        bit += dbits;
    }
    return LGS_OK;
}

// 0 = histogram / row-scan / scatter passes (default), 1 = onesweep form.  env LGS_RS=passes|onesweep
// With one thread per digit walking back one predecessor per dependent load, the look-back of the concurrently resident tiles
// costs more than the histogram read and the row scan it saves (profiles/microbench/dev_count_bench.py times both forms).
int g_rs_onesweep = -1;
bool rs_use_onesweep()
{
    if (g_rs_onesweep < 0) {
        const char* e = getenv("LGS_RS");
        g_rs_onesweep = (e != nullptr && e[0] == 'o') ? 1 : 0;
    }
    return g_rs_onesweep == 1;
}

template <typename KeyT>
int rs_sort_onesweep(const KeyT* keys_in, KeyT* keys_out, const unsigned* vals_in, unsigned* vals_out, int n, int begin_bit, int end_bit,
                     unsigned bias, char* ws, cudaStream_t st, const int* n_dev, const unsigned* bias_dev)
{
    RsPlan p = rs_plan<KeyT>(n, begin_bit, end_bit);
    unsigned* status = (unsigned*)ws;
    int* ghist = (int*)(ws + p.off_scan);
    int* tickets = ghist + RS_MAXPASS * RS_MAXBINS;
    KeyT* ktmp = (KeyT*)(ws + p.off_keys);
    unsigned* vtmp = (unsigned*)(ws + p.off_vals);
    GhistArgs A;
    A.passes = p.passes;
    size_t status_words = 0;
    int bit = begin_bit;
    for (int pass = 0; pass < p.passes; pass++) {
        int dbits = min(p.dbits, end_bit - bit);
        A.shift[pass] = bit; A.nbins[pass] = 1 << dbits;
        status_words += (size_t)p.nblocks * A.nbins[pass];
        bit += dbits;
    }
    LGS_CUDA(cudaMemsetAsync(status, 0, status_words * sizeof(unsigned), st));
    LGS_CUDA(cudaMemsetAsync(ghist, 0, (RS_MAXPASS * RS_MAXBINS + 64) * sizeof(int), st));
    lgs_with_flags([&](auto ipt16) {
        rs_ghist_kernel<KeyT, ipt16 ? 16 : 8><<<p.nblocks, RS_THREADS, 0, st>>>(keys_in, n, A, ghist, bias, n_dev, bias_dev);
        return LGS_OK;
    }, p.ipt == 16);
    LGS_CHECK_LAUNCH("rs_ghist_kernel");
    const KeyT* ksrc = keys_in;
    const unsigned* vsrc = vals_in;
    size_t soff = 0;
    for (int pass = 0; pass < p.passes; pass++) {
        bool to_out = ((p.passes - 1 - pass) & 1) == 0;
        KeyT* kdst = to_out ? keys_out : ktmp;
        unsigned* vdst = to_out ? vals_out : vtmp;
        lgs_with_flags([&](auto ipt16) {
            rs_onesweep_kernel<KeyT, ipt16 ? 16 : 8><<<p.nblocks, RS_THREADS, 0, st>>>(ksrc, vsrc, kdst, vdst, n, A.shift[pass],
                A.nbins[pass], ghist + pass * RS_MAXBINS, status + soff, tickets + pass, bias, n_dev, bias_dev);
            return LGS_OK;
        }, p.ipt == 16);
        LGS_CHECK_LAUNCH("rs_onesweep_kernel");
        soff += (size_t)p.nblocks * A.nbins[pass];
        ksrc = kdst; vsrc = vdst;
    }
    return LGS_OK;
}

template <typename KeyT>
size_t sort_workspace_bytes(int n, int max_bits)
{
    size_t cubb = 0;
    cub::DeviceRadixSort::SortPairs<KeyT, unsigned>(nullptr, cubb, nullptr, nullptr, nullptr, nullptr, n, 0, max_bits);
    size_t own = rs_plan<KeyT>(n, 0, max_bits).total_bytes;      // independent of the bit range
    return std::max(cubb, own) + 256;
}

template <typename KeyT>
int sort_pairs(const char* who, const KeyT* keys_in, KeyT* keys_out, const unsigned* vals_in, unsigned* vals_out, int n, int begin_bit,
               int end_bit, void* workspace, size_t workspace_bytes, void* stream)
{
    if (n <= 0) return LGS_OK;
    LGS_REQUIRE(begin_bit >= 0 && end_bit >= begin_bit && end_bit <= (int)(8 * sizeof(KeyT)), "%s: bad bit range [%d, %d)", who, begin_bit,
                end_bit);
    char* ws = (char*)(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
    size_t need;
    const int impl = sort_impl_for(n, end_bit - begin_bit);
    if (impl == 0) {
        need = 0;
        cub::DeviceRadixSort::SortPairs<KeyT, unsigned>(nullptr, need, nullptr, nullptr, nullptr, nullptr, n, begin_bit, end_bit);
    } else {
        need = rs_plan<KeyT>(n, begin_bit, end_bit).total_bytes;
    }
    if (workspace == nullptr || workspace_bytes < need + 256) {
        lgs_set_error("%s: workspace of %zu bytes needed, %zu given", who, need + 256, workspace_bytes);
        return LGS_ERR_WORKSPACE;
    }
    if (impl == 0) {
        LGS_CUDA(cub::DeviceRadixSort::SortPairs<KeyT, unsigned>(ws, need, keys_in, keys_out, vals_in, vals_out, n, begin_bit, end_bit,
                                                                 (cudaStream_t)stream));
        return LGS_OK;
    }
    return rs_sort<KeyT>(keys_in, keys_out, vals_in, vals_out, n, begin_bit, end_bit, 0u, ws, (cudaStream_t)stream);
}

}  // namespace

// 0 = cub::DeviceRadixSort, 1 = the histogram/scan/scatter passes above (default; env LGS_SORT=cub|lgs); both force the choice.
// -1 = unforced again: LGS_SORT is read on the next sort and, without it, sort_impl_for chooses per call.
extern "C" int lgs_set_sort_impl(int impl)
{
    LGS_REQUIRE(impl == -1 || impl == 0 || impl == 1, "set_sort_impl: %d is not -1 (unforced), 0 (cub) or 1 (lgs)", impl);
    g_sort_impl = impl;
    g_sort_forced = impl >= 0;
    return LGS_OK;
}

// 1 = onesweep form of the own radix sort, 0 = histogram / row-scan / scatter passes (default); env LGS_RS=passes|onesweep
extern "C" int lgs_set_radix_form(int onesweep)
{
    g_rs_onesweep = onesweep ? 1 : 0;
    return LGS_OK;
}

extern "C" int lgs_sort_pairs_u32_workspace_bytes(int n, size_t* bytes)
{
    *bytes = sort_workspace_bytes<unsigned>(n < 1 ? 1 : n, 32);
    return LGS_OK;
}

extern "C" int lgs_sort_pairs_u32(const unsigned* keys_in, unsigned* keys_out, const unsigned* vals_in, unsigned* vals_out, int n,
                                  int begin_bit, int end_bit, void* workspace, size_t workspace_bytes, void* stream)
{
    return sort_pairs<unsigned>("sort_pairs_u32", keys_in, keys_out, vals_in, vals_out, n, begin_bit, end_bit, workspace, workspace_bytes,
                                stream);
}

// 16-bit tile keys (tiles+1 < 65536, i.e. anything up to 4K at 8x16): 6 instead of 8 bytes per pair and pass
extern "C" int lgs_sort_pairs_u16_workspace_bytes(int n, size_t* bytes)
{
    *bytes = sort_workspace_bytes<unsigned short>(n < 1 ? 1 : n, 16);
    return LGS_OK;
}

extern "C" int lgs_sort_pairs_u16(const unsigned short* keys_in, unsigned short* keys_out, const unsigned* vals_in, unsigned* vals_out,
                                  int n, int begin_bit, int end_bit, void* workspace, size_t workspace_bytes, void* stream)
{
    return sort_pairs<unsigned short>("sort_pairs_u16", keys_in, keys_out, vals_in, vals_out, n, begin_bit, end_bit, workspace,
                                      workspace_bytes, stream);
}

// ---- GPU-driven variants: capacity on the host, live count (and key bias) on the device -------------------------------------
// The launch geometry covers `capacity` items; every kernel reads the live count from *n_dev (clamped to the capacity) and,
// for the rebased depth sort, the bias from *bias_dev -- no read-back, so a whole view can be enqueued (or captured in a
// CUDA graph) without a host synchronisation (SURVEY 7 "GPU-driven sizing"; the reference hides its two read-backs behind last
// epoch's feedback values instead, GR/compact.cu:527-549, GR/binning.cu:137-163).  Own radix sort only.
// The depth sort orders by (key - *bias_dev) on the bits [0, end_bit): for keys known to lie in [bias, bias + 2^end_bit) this is
// the order of the full keys at fewer passes (view-space z in [1.3, 4.7) spans 31 bits of float pattern but only 24 bits of
// range).  Keys outside that interval land in unspecified places.
extern "C" int lgs_sort_pairs_u32_dev(const unsigned* keys_in, unsigned* keys_out, const unsigned* vals_in, unsigned* vals_out,
                                      int capacity, const int* n_dev, const unsigned* bias_dev, int end_bit, void* workspace,
                                      size_t workspace_bytes, void* stream)
{
    if (capacity <= 0) return LGS_OK;
    LGS_REQUIRE(n_dev != nullptr && end_bit >= 1 && end_bit <= 32, "sort_pairs_u32_dev: bad arguments (end_bit %d)", end_bit);
    char* ws = (char*)(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
    size_t need = rs_plan<unsigned>(capacity, 0, end_bit).total_bytes;
    if (workspace == nullptr || workspace_bytes < need + 256) {
        lgs_set_error("sort_pairs_u32_dev: workspace of %zu bytes needed, %zu given", need + 256, workspace_bytes);
        return LGS_ERR_WORKSPACE;
    }
    return rs_sort<unsigned>(keys_in, keys_out, vals_in, vals_out, capacity, 0, end_bit, 0u, ws, (cudaStream_t)stream, n_dev, bias_dev);
}

extern "C" int lgs_sort_pairs_u16_dev(const unsigned short* keys_in, unsigned short* keys_out, const unsigned* vals_in,
                                      unsigned* vals_out, int capacity, const int* n_dev, int begin_bit, int end_bit, void* workspace,
                                      size_t workspace_bytes, void* stream)
{
    if (capacity <= 0) return LGS_OK;
    LGS_REQUIRE(n_dev != nullptr && begin_bit >= 0 && end_bit > begin_bit && end_bit <= 16, "sort_pairs_u16_dev: bad bit range [%d, %d)",
                begin_bit, end_bit);
    char* ws = (char*)(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
    size_t need = rs_plan<unsigned short>(capacity, begin_bit, end_bit).total_bytes;
    if (workspace == nullptr || workspace_bytes < need + 256) {
        lgs_set_error("sort_pairs_u16_dev: workspace of %zu bytes needed, %zu given", need + 256, workspace_bytes);
        return LGS_ERR_WORKSPACE;
    }
    return rs_sort<unsigned short>(keys_in, keys_out, vals_in, vals_out, capacity, begin_bit, end_bit, 0u, ws, (cudaStream_t)stream, n_dev,
                                   nullptr);
}

extern "C" int lgs_sort_pairs_u32k_dev(const unsigned* keys_in, unsigned* keys_out, const unsigned* vals_in, unsigned* vals_out,
                                       int capacity, const int* n_dev, int begin_bit, int end_bit, void* workspace, size_t workspace_bytes,
                                       void* stream)
{   // 32-bit tile keys (more than 65534 tiles), device-side count
    if (capacity <= 0) return LGS_OK;
    LGS_REQUIRE(n_dev != nullptr && begin_bit >= 0 && end_bit > begin_bit && end_bit <= 32, "sort_pairs_u32k_dev: bad bit range [%d, %d)",
                begin_bit, end_bit);
    char* ws = (char*)(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
    size_t need = rs_plan<unsigned>(capacity, begin_bit, end_bit).total_bytes;
    if (workspace == nullptr || workspace_bytes < need + 256) {
        lgs_set_error("sort_pairs_u32k_dev: workspace of %zu bytes needed, %zu given", need + 256, workspace_bytes);
        return LGS_ERR_WORKSPACE;
    }
    return rs_sort<unsigned>(keys_in, keys_out, vals_in, vals_out, capacity, begin_bit, end_bit, 0u, ws, (cudaStream_t)stream, n_dev, nullptr);
}
