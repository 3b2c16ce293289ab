// K2 — blocked CSR x CSR^T, thresholded, top-n per left row, for sm_90a.
//
// Replaces StringGrouper._build_matches
// (string_grouper/string_grouper.py:709-752): the per block
// pair sp_matmul_topn products (:737-743), the zip over right blocks (:746)
// and the vstack over left blocks (:750).  See DESIGN.md §K2 for the layout.
//
//   postings_build   right matrix  -> (feature, column-tile) bucketed postings + directory with block maxima
//   candidates       block-max test of 128 tiles at a time, then the Gustavson row-wise product of the pruned left
//                    row over the surviving tiles into a shared-memory accumulator tile per warp (16-bit fixed
//                    point or fp32); emits (row, col) with partial score > the (row, tile) candidate threshold
//   rescore          exact sorted-merge dot product of every candidate pair; rescore_refined first drops the
//                    candidates whose partial score + grouped bound of the pruned part cannot reach the threshold
//   topn_select      strict threshold, top-n per row, value-descending
#include <cub/cub.cuh>
#include <cuda_fp16.h>

#include "sg_common.cuh"

namespace sg {

// ---------------------------------------------------------------------------
// postings build: one column tile at a time
// ---------------------------------------------------------------------------
// Column tile t holds the right rows perm[t*W .. t*W + W) of the processing order.  Its postings lie contiguously at
// tile_off[t], sorted by feature; bucket (f, t) is the run of feature f among them.  Only the directory is
// feature-major, dir[f * T + t]: the entries a left row reads for one of its features over consecutive column tiles
// are neighbours.  Nothing is built per (feature, tile) pair beyond that: the caller clears the directory and the
// block maxima, and every tile writes the entries of the features it holds.
//
// A posting is 4 bytes: the column inside the tile (16 bits) and the weight rounded to fp16 (16 bits).  The
// candidate scores only have to be within CAND_MARGIN of the exact ones (every candidate is re-scored in the
// matrix dtype): an fp16 weight is off by at most 2^-11 relative, so a score by at most 4.9e-4.  The order inside a
// bucket is arbitrary (a bucket holds every column once; the fixed-point tiles add integers, so the candidate set
// does not depend on it).  A nonzero weight below fp16's range keeps its sign and becomes the smallest subnormal
// (2^-24) instead of zero, which is no further from it than rounding to nearest: with the candidate threshold at 0
// (thresholds below the margin) a pair of non-negative rows is found exactly when it shares a feature.
constexpr int PB_THREADS = 1024;
constexpr int PB_ITEMS = 8;
constexpr int PB_CAP = PB_THREADS * PB_ITEMS;   // postings of a tile sorted in shared memory; larger tiles: global
constexpr size_t PB_SMEM = (size_t)PB_CAP * 8;  // keys + postings (the block sort's scratch reuses them)

__device__ __forceinline__ uint32_t make_posting(float v, float w_scale, uint32_t local) {
    const float x = v * w_scale;
    const float y = x != 0.f && fabsf(x) < 0x1p-24f ? copysignf(0x1p-24f, x) : x;
    return ((uint32_t)__half_as_ushort(__float2half_rn(y)) << 16) | local;
}

// postings per tile, one warp per tile; tile_cnt[T] = 0 closes the exclusive scan into tile_off
__global__ void postings_tile_count_kernel(int64_t n_rows, int64_t T, int W, const int64_t *__restrict__ indptr,
                                           const int32_t *__restrict__ perm, int32_t *__restrict__ tile_cnt) {
    const int64_t t = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (t > T) return;
    int s = 0;      // < nnz < 2^31
    if (t < T) {
        const int64_t p1 = (t + 1) * W < n_rows ? (t + 1) * W : n_rows;
        for (int64_t p = t * W + lane_id(); p < p1; p += 32) {
            const int64_t row = perm ? perm[p] : p;
            s += (int)(indptr[row + 1] - indptr[row]);
        }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(FULL, s, o);
    if (lane_id() == 0) tile_cnt[t] = s;
}

// The directory entries of the runs of sorted keys[0, n) (postings pst[0, n), the first at posting index `start`):
// one aligned 8-byte entry per (feature, tile) so that a lane fetches it in one load,
// {int32 start, u16 length | fp16 largest |weight| << 16}, and the same maxima as fp16 rows of Tp tiles per feature
// (what the block-max test streams).  |round(w)| = round(|w|), and non-negative halves order like integers.
__device__ __forceinline__ void postings_emit_runs(const uint32_t *keys, const uint32_t *pst, int n, int start,
                                                   int64_t t, int64_t T, int64_t Tp, int2 *__restrict__ dir,
                                                   unsigned short *__restrict__ maxw_rows) {
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const uint32_t f = keys[i];
        if (i > 0 && keys[i - 1] == f) continue;
        uint32_t m = 0;
        int j = i;
        for (; j < n && keys[j] == f; ++j) m = max(m, (pst[j] >> 16) & 0x7fffu);
        dir[(int64_t)f * T + t] = make_int2(start + i, (int)(((uint32_t)(j - i) & 0xffffu) | (m << 16)));
        maxw_rows[(int64_t)f * Tp + t] = (unsigned short)m;
    }
}

// Block radix sort by feature of the n <= PB_THREADS * ITEMS (key, posting) pairs in skey / spost, in place; the
// sort's scratch reuses the same shared memory.  Items are taken in striped order and sorted as if blocked: a fixed
// permutation of the input, so the result is still deterministic.  Padding keys (all key_bits set, above every
// feature) sort behind the n postings.
template <int ITEMS>
__device__ __forceinline__ void postings_sort_tile(uint32_t *skey, uint32_t *spost, int n, int key_bits) {
    typedef cub::BlockRadixSort<uint32_t, PB_THREADS, ITEMS, uint32_t> Sort;
    static_assert(sizeof(typename Sort::TempStorage) <= PB_SMEM, "block sort scratch exceeds the tile buffers");
    const uint32_t pad = (uint32_t)((1ull << key_bits) - 1);
    uint32_t keys[ITEMS], vals[ITEMS];
#pragma unroll
    for (int k = 0; k < ITEMS; ++k) {
        const int i = k * PB_THREADS + threadIdx.x;
        keys[k] = i < n ? skey[i] : pad;
        vals[k] = i < n ? spost[i] : 0u;
    }
    __syncthreads();
    Sort(*reinterpret_cast<typename Sort::TempStorage *>(skey)).SortBlockedToStriped(keys, vals, 0, key_bits);
    __syncthreads();
#pragma unroll
    for (int k = 0; k < ITEMS; ++k) {
        const int i = k * PB_THREADS + threadIdx.x;
        skey[i] = keys[k];
        spost[i] = vals[k];
    }
}

// One CTA per tile: the tile's (feature, posting) pairs in row order, then
//   * up to PB_CAP of them: sorted by feature in shared memory, postings and directory entries written;
//   * more: copied to big_key / big_post at tile_off[t] and big_end[t] = tile_off[t + 1], for the segmented sort
//     (postings_big_dir_kernel finishes them); every other tile sets big_end[t] = tile_off[t], an empty segment.
__global__ void __launch_bounds__(PB_THREADS)
postings_tile_build_kernel(int64_t n_rows, int64_t T, int64_t Tp, int W, int key_bits,
                           const int64_t *__restrict__ indptr, const int32_t *__restrict__ indices,
                           const float *__restrict__ val, const int32_t *__restrict__ perm, float w_scale,
                           const int32_t *__restrict__ tile_off, uint32_t *__restrict__ post, int2 *__restrict__ dir,
                           unsigned short *__restrict__ maxw_rows, uint32_t *__restrict__ big_key,
                           uint32_t *__restrict__ big_post, int32_t *__restrict__ big_end, int32_t *n_spilled) {
    typedef cub::BlockScan<int, PB_THREADS> Scan;
    __shared__ typename Scan::TempStorage scan_tmp;
    __shared__ int64_t row_p0[PB_THREADS];
    __shared__ int row_off[PB_THREADS];
    extern __shared__ __align__(16) uint32_t pb_smem[];
    uint32_t *skey = pb_smem, *spost = pb_smem + PB_CAP;

    const int64_t t = blockIdx.x;
    const int off0 = tile_off[t], n = tile_off[t + 1] - off0;
    const bool big = n > PB_CAP;
    if (threadIdx.x == 0) {
        big_end[t] = big ? off0 + n : off0;
        if (big && n_spilled) atomicAdd(n_spilled, 1);
    }
    uint32_t *kdst = big ? big_key + off0 : skey, *pdst = big ? big_post + off0 : spost;

    // gather, PB_THREADS rows at a time: offsets by a block scan of the row lengths, then one entry per thread (its
    // row by a binary search over the offsets: rows past the tile's end are empty and start at `total`)
    const int64_t p0 = t * W;
    const int nr = (int)((p0 + W < n_rows ? p0 + W : n_rows) - p0);
    int base = 0;
    for (int r0 = 0; r0 < nr; r0 += PB_THREADS) {
        const int r = r0 + threadIdx.x;
        int len = 0;
        int64_t q = 0;
        if (r < nr) {
            const int64_t row = perm ? perm[p0 + r] : p0 + r;
            q = indptr[row];
            len = (int)(indptr[row + 1] - q);
        }
        int o, total;
        Scan(scan_tmp).ExclusiveSum(len, o, total);
        row_p0[threadIdx.x] = q;
        row_off[threadIdx.x] = o;
        __syncthreads();
#pragma unroll 4
        for (int j = threadIdx.x; j < total; j += PB_THREADS) {
            int k = 0;          // the last row starting at or before j
#pragma unroll
            for (int s = PB_THREADS / 2; s; s >>= 1)
                if (row_off[k + s] <= j) k += s;
            const int64_t p = row_p0[k] + (j - row_off[k]);
            kdst[base + j] = (uint32_t)indices[p];
            pdst[base + j] = make_posting(val[p], w_scale, (uint32_t)(r0 + k));
        }
        base += total;
        __syncthreads();
    }
    if (big) return;

    // the smallest sort that holds the tile: the work of every radix pass grows with the items per thread
    if (n <= PB_THREADS * 2) postings_sort_tile<2>(skey, spost, n, key_bits);
    else if (n <= PB_THREADS * 4) postings_sort_tile<4>(skey, spost, n, key_bits);
    else postings_sort_tile<PB_ITEMS>(skey, spost, n, key_bits);
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += PB_THREADS) post[off0 + i] = spost[i];
    postings_emit_runs(skey, spost, n, off0, t, T, Tp, dir, maxw_rows);
}

// Tiles of more than PB_CAP postings after the segmented sort of [tile_off[t], big_end[t]): keys / pst are the sorted
// buffers (pst may be `post` itself); every other tile has an empty segment and returns.
__global__ void __launch_bounds__(256)
postings_big_dir_kernel(int64_t T, int64_t Tp, const int32_t *__restrict__ tile_off,
                        const int32_t *__restrict__ big_end, const uint32_t *keys, const uint32_t *pst, uint32_t *post,
                        int2 *__restrict__ dir, unsigned short *__restrict__ maxw_rows) {
    const int64_t t = blockIdx.x;
    const int off0 = tile_off[t], n = big_end[t] - off0;
    if (n == 0) return;
    if (pst != post)
        for (int i = threadIdx.x; i < n; i += blockDim.x) post[off0 + i] = pst[off0 + i];
    postings_emit_runs(keys + off0, pst + off0, n, off0, t, T, Tp, dir, maxw_rows);
}

__device__ __forceinline__ float post_w(uint32_t e) { return __half2float(__ushort_as_half((unsigned short)(e >> 16))); }
__device__ __forceinline__ int post_c(uint32_t e) { return (int)(e & 0xffffu); }

__device__ __forceinline__ int dir_len(int2 d) { return d.y & 0xffff; }
__device__ __forceinline__ float dir_maxw(int2 d) {
    return __half2float(__ushort_as_half((unsigned short)((unsigned)d.y >> 16)));
}

// ---------------------------------------------------------------------------
// candidate generation
// ---------------------------------------------------------------------------
constexpr int LONG_BUCKET = 64;  // buckets from this length on are streamed by the whole warp, one at a time
#ifndef SG_WALK_MLP
#define SG_WALK_MLP 1            // steps of the concatenated walk whose posting loads are in flight together
#endif

// Resident CTAs per SM the register allocation is made for (the accumulator tiles are small, registers decide):
// 32 warps/CTA x 2 = 64 warps at 32 registers; 16 x 3 = 48 warps at 40; 8 x 5 = 40 warps at 48; 4 x 8 = 32 warps at 64.
constexpr int min_ctas(int nw) { return nw == 32 ? 2 : nw == 16 ? 3 : nw == 8 ? 5 : 8; }

// Accumulator tile element.
//   float    : fp32 scores, read-modify-write in the long-bucket path, CAS-loop atomics in the short one.
//   uint16_t : 16-bit fixed point (1/32768 units, scores in [0, 2)), two columns per 32-bit word, every update
//              one native integer ATOMS.ADD on the word.  Twice the columns per shared-memory byte: half the
//              directory look-ups and half the clearing per column.  Each product is rounded once (<= 2^-16),
//              sums are exact; the caller widens the candidate margin by 2e-5 per kept feature.
constexpr float FIX_ONE = 32768.f;

template <typename AccT>
struct AccOps;
template <>
struct AccOps<float> {
    typedef float val_t;
    static constexpr int PER16 = 4;           // elements per 16-byte vector
    static __device__ __forceinline__ float left_weight(float a) { return a; }
    static __device__ __forceinline__ float threshold(float thr) { return thr; }
    static __device__ __forceinline__ float fma_store(float *acc, int col, float a, float w) {
        const float v = fmaf(a, w, acc[col]);
        acc[col] = v;
        return v;
    }
    static __device__ __forceinline__ float atomic_add(float *acc, int col, float a, float w) {
        const float x = a * w;
        return atomicAdd(acc + col, x) + x;
    }
    static __device__ __forceinline__ float vmax(float a, float b) { return fmaxf(a, b); }
    // bit i set when element i of the 16-byte vector exceeds thr
    static __device__ __forceinline__ unsigned above(const uint4 &v, float thr) {
        return (__uint_as_float(v.x) > thr ? 1u : 0u) | (__uint_as_float(v.y) > thr ? 2u : 0u) |
               (__uint_as_float(v.z) > thr ? 4u : 0u) | (__uint_as_float(v.w) > thr ? 8u : 0u);
    }
    // element i of the vector as a score
    static __device__ __forceinline__ float value(const uint4 &v, int i) {
        return __uint_as_float(i < 2 ? (i == 0 ? v.x : v.y) : (i == 2 ? v.z : v.w));
    }
};
template <>
struct AccOps<uint16_t> {
    typedef int val_t;
    static constexpr int PER16 = 8;
    static __device__ __forceinline__ float left_weight(float a) { return a * FIX_ONE; }
    // v > floor(thr * 32768)  <=>  v / 32768 > thr  for integer v
    static __device__ __forceinline__ int threshold(float thr) { return (int)floorf(thr * FIX_ONE); }
    static __device__ __forceinline__ int atomic_add(uint16_t *acc, int col, float a, float w) {
        const int x = __float2int_rn(a * w);
        const unsigned sh = ((unsigned)col & 1u) << 4;
        const unsigned old = atomicAdd(reinterpret_cast<unsigned *>(acc) + (col >> 1), (unsigned)x << sh);
        return (int)((old >> sh) & 0xffffu) + x;
    }
    static __device__ __forceinline__ int fma_store(uint16_t *acc, int col, float a, float w) {
        return atomic_add(acc, col, a, w);
    }
    static __device__ __forceinline__ int vmax(int a, int b) { return max(a, b); }
    static __device__ __forceinline__ unsigned pair_above(unsigned u, int thr) {
        return ((int)(u & 0xffffu) > thr ? 1u : 0u) | ((int)(u >> 16) > thr ? 2u : 0u);
    }
    static __device__ __forceinline__ unsigned above(const uint4 &v, int thr) {
        return pair_above(v.x, thr) | (pair_above(v.y, thr) << 2) | (pair_above(v.z, thr) << 4) |
               (pair_above(v.w, thr) << 6);
    }
    static __device__ __forceinline__ float value(const uint4 &v, int i) {
        const unsigned w = i < 4 ? (i < 2 ? v.x : v.y) : (i < 6 ? v.z : v.w);
        return (float)((w >> ((i & 1) << 4)) & 0xffffu) * (1.f / FIX_ONE);
    }
};

// One bucket-directory batch of a row (32 features, one per lane: bucket [b0, b0+len) and left weight a)
// applied to the accumulator tile.
//   * buckets of LONG_BUCKET postings or more: the whole warp streams one bucket at a time;
//   * all the others are walked as ONE concatenated list, 32 postings per step whatever the bucket boundaries
//     (after pruning a row keeps its rarer features, whose buckets hold a dozen postings per tile: one bucket
//     per step would leave most lanes idle).  Lane -> bucket by a 5-step binary search over the running
//     sums; two lanes of a step may meet on one column, hence shared-memory atomics.
template <typename AccT>
__device__ __forceinline__ void apply_buckets(AccT *__restrict__ acc, const uint32_t *__restrict__ post, int b0,
                                              int len, float a, int lane,
                                              typename AccOps<AccT>::val_t &seen) {
    typedef AccOps<AccT> Ops;
    unsigned m = __ballot_sync(FULL, len >= LONG_BUCKET);
    while (m) {
        const int src = __ffs(m) - 1;
        m &= m - 1;
        const int s = __shfl_sync(FULL, b0, src);
        const int e = s + __shfl_sync(FULL, len, src);
        const float ak = __shfl_sync(FULL, a, src);
        int p = s + lane;
        for (; p + 96 < e; p += 128) {
            const uint32_t e0 = post[p], e1 = post[p + 32], e2 = post[p + 64], e3 = post[p + 96];
            const typename Ops::val_t v0 = Ops::fma_store(acc, post_c(e0), ak, post_w(e0));
            const typename Ops::val_t v1 = Ops::fma_store(acc, post_c(e1), ak, post_w(e1));
            const typename Ops::val_t v2 = Ops::fma_store(acc, post_c(e2), ak, post_w(e2));
            const typename Ops::val_t v3 = Ops::fma_store(acc, post_c(e3), ak, post_w(e3));
            seen = Ops::vmax(Ops::vmax(Ops::vmax(seen, v0), Ops::vmax(v1, v2)), v3);
        }
        for (; p < e; p += 32) {
            const uint32_t e0 = post[p];
            seen = Ops::vmax(seen, Ops::fma_store(acc, post_c(e0), ak, post_w(e0)));
        }
        __syncwarp();
    }
    // the concatenated walk over the remaining buckets
    const int ln = len >= LONG_BUCKET ? 0 : len;
    int incl = ln;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int up = __shfl_up_sync(FULL, incl, o);
        if (lane >= o) incl += up;
    }
    const int total = __shfl_sync(FULL, incl, 31);
    const int d = b0 - (incl - ln);                    // posting index = d + position in the concatenated list
    // SG_WALK_MLP steps at a time: the posting loads of all of them are issued before the first accumulator update
    // (the kernel is bound by the latency of these L2 loads, not by issue slots)
    for (int base = 0; base < total; base += 32 * SG_WALK_MLP) {
        uint32_t e[SG_WALK_MLP];
        float ak[SG_WALK_MLP];
#pragma unroll
        for (int u = 0; u < SG_WALK_MLP; ++u) {
            const int item = base + 32 * u + lane;
            int k = 0;                                 // number of buckets that end at or before `item`
#pragma unroll
            for (int st = 16; st; st >>= 1) {
                const int v = __shfl_sync(FULL, incl, k + st - 1);
                if (v <= item) k += st;
            }
            const int dk = __shfl_sync(FULL, d, k);
            ak[u] = __shfl_sync(FULL, a, k);
            e[u] = 0u;
            if (item < total) e[u] = post[dk + item];
        }
#pragma unroll
        for (int u = 0; u < SG_WALK_MLP; ++u) {
            const int item = base + 32 * u + lane;
            if (item < total) seen = Ops::vmax(seen, Ops::atomic_add(acc, post_c(e[u]), ak[u], post_w(e[u])));
        }
    }
    __syncwarp();
}

// Pruned left operand (sg_prune_rows; all three optional together): row i keeps only its first a_len[i] stored
// features; a pair (i, j) is reported when its partial score exceeds
//     thr_row[i] - xp_norm[i] * tile_bound[tile of j]
// = the row's threshold minus what the pruned features can still add for the columns of that tile.
//
// Block-max test (`maxw_h`, the fp16 largest |weight| of every (feature, tile) bucket, feature-major, rows padded to
// Tp tiles): no column of tile t can collect more than ub(t) = sum_f |a_f| * max|w_(f,t)|.  The bounds of 128 tiles
// are evaluated in one pass, four consecutive tiles per lane: per kept feature one 8-byte load of their maxima and two
// HFMA2 in packed fp16, at an address that is the feature's row offset (held by its lane for the whole row) plus the
// pass's column.  Only the tiles whose bound can exceed their candidate threshold are walked at all: nothing is
// accumulated, cleared or swept for the others.
//
// Triangle of a self-match (`diag_rank` != NULL, left and right rows the same matrix in the same processing order):
// row i only reports columns whose position in that order is >= diag_rank[i], so every unordered pair is found
// once, from the row that comes first (the caller mirrors the kept pairs).  Tiles wholly below the rank are left
// out of the block-max ballot; in the tile holding the rank the columns below it are not reported.
// `group_items` (with diag_rank): exclusive offsets of the work items per column-tile group (diag_items_kernel), so
// that no item is handed out whose row has no tile at or above its rank in the group.
//
// Position range (cossim_candidates_range_kernel, `hi_pos` != NULL, with diag_rank as the lower end): row i reports
// only the columns at positions in [diag_rank[i], hi_pos[i]) of the right processing order (a blocked product: both
// sides sorted by block id first, the range is the row's block among the right rows).  Tiles wholly at or above hi
// are left out of the block-max ballot, and in the tile holding hi the columns at or above it are not reported.
// `group_items` then holds 2 * n_groups + 1 entries: the exclusive offsets of the work items per column-tile group and
// the first ridx of each group (range_items_kernel); the items of group g are the rows first[g], first[g] + 1, ...
//
// Top-n floor (cossim_candidates_floor_kernel, top_n <= 32, non-negative weights): floor[row] is a proven lower bound
// of the exact score of the row's top_n-th best pair; it only rises.  A pair whose exact score is below it cannot be
// in the row's output, so the candidate threshold of the row becomes max(thr_row, floor - E_r - FLOOR_EPS), read again
// at every 128-tile pass (block-max test and sweep).  E_r = margin + margin_pf * kept features bounds how far the
// accumulated partial p^ can differ from the kept-feature product x_S.y in EITHER direction (the fp16 posting weights
// and the fixed-point / fp32 roundings are symmetric; the same constants give thr_row), and x_S.y <= exact for
// non-negative weights.  So p^ - E_r (rounded down) is a lower bound of the exact score of every reported pair: the
// warp keeps the best 32 of them per work item, one per lane, and once top_n exist publishes the top_n-th with
// atomicMax (non-negative floats order like their bits).  The pairs of one item are distinct columns.
// Self-match (`self_rank` = every row's position in the common processing order): `seed` = 1 walks only the row's own
// column-tile group, starting at the 128-tile pass that holds the row (clusters of identical names sit next to each
// other in that order, so this is where floors rise first); `seed` = 0 walks every other group.
// Both (cossim_candidates_range_floor_kernel, a keyed arg-max): the floor is raised only from pairs inside the row's
// range, which the sweep's lo / hi cut has already masked, so it stays a bound of eligible pairs.  A self-match's seed
// takes no group_items (one item per row, in the group holding self_rank[row], which lies in [lo, hi)); without the
// seed the items come from group_items as for the range alone, and the row's own group is skipped.
//
// Long rows (more than 32 kept features: long records rows, names without a threshold): only the first 32 stay in
// registers, but ub(t) is taken over ALL kept features, the later ones 32 at a time, their {row offset, weight} loaded
// once per 128-tile pass, with the same fp16 round-up and a slack of 5e-4 per feature.  Every hfma2
// rounds once; while the running sum stays below 2 (ulp 2^-10) that is at most 2^-11 < 5e-4, and once it reaches 2
// it stays there (non-negative terms, monotone rounding), above any threshold of scores in [0, 1].
// `b_scale` (a power of two, 1 for rows of norm <= 1) keeps that argument for any operands: the left weights of the
// bound and the thresholds it is tested against are multiplied by it, so the bound is evaluated in units of a power
// of two at or above the largest possible score, where every term and every threshold lies below 2 (and nothing
// overflows fp16).  The accumulated partial scores stay in score units.
struct FloorArgs {
    float *floor;
    const int32_t *self_rank;
    int seed, top_n;
    float margin, margin_pf;
};

// kept: the best 32 values so far, descending over the lanes; x: one new value per lane.  Sort x ascending, the lane-wise
// maxima are the best 32 of the union as a bitonic sequence, five merge stages sort them (as sel_rows_kernel does).
__device__ __forceinline__ void floor_merge(float &kept, float x, int lane) {
#pragma unroll
    for (int k = 2; k <= 32; k <<= 1) {
#pragma unroll
        for (int j = k >> 1; j > 0; j >>= 1) {
            const float o = __shfl_xor_sync(FULL, x, j);
            x = (((lane & k) == 0) == ((lane & j) == 0)) ? fminf(x, o) : fmaxf(x, o);
        }
    }
    kept = fmaxf(kept, x);
#pragma unroll
    for (int j = 16; j > 0; j >>= 1) {
        const float o = __shfl_xor_sync(FULL, kept, j);
        kept = (lane & j) == 0 ? fmaxf(kept, o) : fminf(kept, o);
    }
}

template <int NW, typename AccT, bool FLOOR, bool RANGE = false>
__device__ __forceinline__ void
candidates_body(const int64_t *__restrict__ a_indptr, const int32_t *__restrict__ a_len,
                const int32_t *__restrict__ a_idx, const float *__restrict__ a_val, int64_t row_begin,
                int64_t row_end, const int32_t *__restrict__ perm_a, int64_t n_right,
                const int2 *__restrict__ bdir, const uint32_t *__restrict__ maxw_h,
                const uint32_t *__restrict__ post, const int32_t *__restrict__ perm_b, int Tp, int W,
                int64_t T, int64_t tiles_per_group, float a_scale, float b_scale, float thr_all,
                const float *__restrict__ thr_row, const float *__restrict__ xp_norm,
                const float *__restrict__ tile_bound, const int32_t *__restrict__ diag_rank,
                const unsigned long long *__restrict__ group_items, int32_t *__restrict__ cand_row,
                int32_t *__restrict__ cand_col, float *__restrict__ cand_partial, unsigned long long cap,
                unsigned long long *__restrict__ cand_count, unsigned long long *__restrict__ row_queue,
                const FloorArgs &fa, const int32_t *__restrict__ hi_pos = nullptr) {
    typedef AccOps<AccT> Ops;
    typedef typename Ops::val_t val_t;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    AccT *acc = reinterpret_cast<AccT *>(smem_raw) + (size_t)warp * W;
    uint4 *acc16 = reinterpret_cast<uint4 *>(acc);
    const int n16 = W / Ops::PER16;                         // 16-byte vectors per tile
    const uint4 zero4 = make_uint4(0u, 0u, 0u, 0u);

    for (int c = lane; c < n16; c += 32) acc16[c] = zero4;
    __syncwarp();

    // Work item = (column-tile group, left row), groups outermost: at any moment every CTA of the grid streams
    // posting buckets of the same few column tiles, so the live posting set stays L2-resident however
    // large the right matrix is.  tiles_per_group is a multiple of 64.
    const int64_t n_rows = row_end - row_begin;
    const int64_t n_groups = (T + tiles_per_group - 1) / tiles_per_group;
    unsigned long long n_items =
        group_items ? group_items[n_groups] : (unsigned long long)n_rows * (unsigned long long)n_groups;
    if constexpr (FLOOR && RANGE) {
        if (fa.seed) n_items = (unsigned long long)n_rows;      // the seed takes no group_items: one item per row
    } else if constexpr (FLOOR) {
        if (fa.self_rank) n_items = (unsigned long long)n_rows * (unsigned long long)(fa.seed ? 1 : n_groups - 1);
    }
    const int n_tiles = (int)T;
    int group = 0;              // with group_items: items arrive in increasing order, so the group only moves forward
    for (;;) {
        unsigned long long item = 0;
        if (lane == 0) item = atomicAdd(row_queue, 1ull);
        item = __shfl_sync(FULL, item, 0);
        if (item >= n_items) break;
        int64_t ridx;
        if (group_items) {
            while (item >= group_items[group + 1]) ++group;
            ridx = (int64_t)(item - group_items[group]);
            if constexpr (RANGE) ridx += (int64_t)group_items[n_groups + 1 + group];
        } else {
            group = (int)(item / (unsigned long long)n_rows);
            ridx = (int64_t)(item % (unsigned long long)n_rows);
        }
        const int64_t row = perm_a ? perm_a[ridx] : row_begin + ridx;   // processing order: neighbours share buckets
        int own_pass = 0;       // floor seed: the walk starts at the 128-tile pass holding the row
        if constexpr (FLOOR) {
            if (fa.self_rank) {
                const int64_t pos = fa.self_rank[row];
                const int64_t own = pos / (tiles_per_group * W);
                if (fa.seed) {
                    group = (int)own;
                    own_pass = (int)((pos / W - own * tiles_per_group) >> 7);
                } else if constexpr (RANGE) {
                    if (group == own) continue;     // group_items hand out the own group too: the seed walked it
                } else if (group >= own) {
                    ++group;
                }
            }
        }
        const int64_t p0 = a_indptr[row];
        const int nf = a_len ? a_len[row] : (int)(a_indptr[row + 1] - p0);
        if (nf == 0) continue;
        float thr_r = thr_row ? thr_row[row] : thr_all;
        // floor: E_r rounded up, the best 32 lower bounds of this item (descending over the lanes), the floor last seen
        float e_r = 0.f, kept = 0.f, floor_seen = 0.f;
        if constexpr (FLOOR) e_r = __fmaf_ru(fa.margin_pf, (float)nf, fa.margin);
        const float xp = xp_norm ? xp_norm[row] : 0.f;
        // tile ids, directory slots (T * V1 < 2^31, checked by sg_postings_build) and positions fit 32 bits
        const int t_begin = (int)(group * tiles_per_group);
        int t_end = (int)(t_begin + tiles_per_group < T ? t_begin + tiles_per_group : T);
        // first column position this row reports (0: the full product); tile t holds positions [t*W, t*W + W)
        const int dr = diag_rank ? diag_rank[row] : 0;
        int hr = 0;             // range: one past the last position the row reports; no tile from ceil(hr / W) on
        if constexpr (RANGE) {
            hr = hi_pos[row];
            const int t_hi = (int)(((int64_t)hr + W - 1) / W);
            if (t_hi < t_end) t_end = t_hi;
        }
        const int t_first = (int)(((int64_t)dr / W) & ~127);           // the 128-tile pass holding the rank
        const int tb_begin = t_first > t_begin ? t_first : t_begin;
        if constexpr (FLOOR && RANGE) {
            // the passes start at tb_begin, which lo may have moved past the group's first tile; the row's own
            // position lies in [lo, hi) and in its group, so its pass is one of them
            if (fa.seed) own_pass = (int)(((int64_t)fa.self_rank[row] / W - tb_begin) >> 7);
        }

        // the first 32 features of the row stay in registers; lane k also holds where its feature's block maxima row
        // starts, in 4-tile (8-byte) units: below T * V1 < 2^31 (checked by sg_postings_build), so 32 bits
        int f0 = 0;
        float a0 = 0.f;
        __half2 a2 = __float2half2_rn(0.f);
        unsigned mo = 0u;
        if (lane < nf) {
            f0 = a_idx[p0 + lane];
            const float a = a_val[p0 + lane] * a_scale;
            a0 = Ops::left_weight(a);
            a2 = __half2half2(__float2half_ru(fabsf(a * b_scale)));   // rounded up: the bound must not fall short
            mo = (unsigned)f0 * (unsigned)(Tp >> 2);
        }
        const int2 *drow = bdir + f0 * n_tiles;
        const int nk = nf < 32 ? nf : 32;
        // fp16 arithmetic of the bound: one rounding of at most 2^-11 (values below 2) per kept feature
        const float slack = 5e-4f * (float)nf + 1e-4f;

        for (int tb0 = tb_begin; tb0 < t_end; tb0 += 128) {
            int tb = tb0;
            if constexpr (FLOOR) {
                tb += own_pass * 128;           // passes of the group in rotated order
                if (tb >= t_end) tb -= (t_end - tb_begin + 127) / 128 * 128;
                const float f = __shfl_sync(FULL, __ldcg(fa.floor + row), 0);
                if (f > floor_seen) {
                    floor_seen = f;
                    thr_r = fmaxf(thr_r, __fsub_rd(__fsub_rd(f, e_r), FLOOR_EPS));
                }
            }
            // ---- bounds of tiles t0 = tb + 4*lane .. t0 + 3 (tiles wholly below the rank are not taken).  A lane
            // whose tiles all lie at or past t_end reads lane 0's maxima instead (the same sectors, so no extra
            // traffic, and never past Tp) and passes none of them.
            unsigned pass4;         // bit j: tile t0 + j passes
            const int t0 = tb + 4 * lane;
            {
                const unsigned q = (unsigned)(tb >> 2) + (t0 < t_end ? lane : 0);   // + row offset: < 2^31
                const uint2 *maxw4 = reinterpret_cast<const uint2 *>(maxw_h);
                __half2 ub01 = __float2half2_rn(0.f), ub23 = __float2half2_rn(0.f);
                for (int kk = 0; kk < nk; ++kk) {
                    const unsigned o = __shfl_sync(FULL, mo, kk);
                    const __half2 ak = __shfl_sync(FULL, a2, kk);
                    const uint2 mv = maxw4[o + q];
                    ub01 = __hfma2(ak, *reinterpret_cast<const __half2 *>(&mv.x), ub01);
                    ub23 = __hfma2(ak, *reinterpret_cast<const __half2 *>(&mv.y), ub23);
                }
                // the kept features after the first 32, one chunk of 32 at a time
                for (int base = 32; base < nf; base += 32) {
                    unsigned ol = 0u;
                    __half2 al = __float2half2_rn(0.f);
                    if (base + lane < nf) {
                        ol = (unsigned)a_idx[p0 + base + lane] * (unsigned)(Tp >> 2);
                        al = __half2half2(__float2half_ru(fabsf(a_val[p0 + base + lane] * a_scale * b_scale)));
                    }
                    const int nc = nf - base < 32 ? nf - base : 32;
                    for (int kk = 0; kk < nc; ++kk) {
                        const unsigned o = __shfl_sync(FULL, ol, kk);
                        const __half2 ak = __shfl_sync(FULL, al, kk);
                        const uint2 mv = maxw4[o + q];
                        ub01 = __hfma2(ak, *reinterpret_cast<const __half2 *>(&mv.x), ub01);
                        ub23 = __hfma2(ak, *reinterpret_cast<const __half2 *>(&mv.y), ub23);
                    }
                }
                const float2 u01 = __half22float2(ub01), u23 = __half22float2(ub23);
                const float4 tb4 = reinterpret_cast<const float4 *>(tile_bound)[q];
                const float thr0 = xp > 0.f ? fmaxf(fmaf(-xp, tb4.x, thr_r), 0.f) : thr_r;
                const float thr1 = xp > 0.f ? fmaxf(fmaf(-xp, tb4.y, thr_r), 0.f) : thr_r;
                const float thr2 = xp > 0.f ? fmaxf(fmaf(-xp, tb4.z, thr_r), 0.f) : thr_r;
                const float thr3 = xp > 0.f ? fmaxf(fmaf(-xp, tb4.w, thr_r), 0.f) : thr_r;
                pass4 = (t0 < t_end && (t0 + 1) * W > dr && u01.x + slack > thr0 * b_scale ? 1u : 0u) |
                        (t0 + 1 < t_end && (t0 + 2) * W > dr && u01.y + slack > thr1 * b_scale ? 2u : 0u) |
                        (t0 + 2 < t_end && (t0 + 3) * W > dr && u23.x + slack > thr2 * b_scale ? 4u : 0u) |
                        (t0 + 3 < t_end && (t0 + 4) * W > dr && u23.y + slack > thr3 * b_scale ? 8u : 0u);
            }
            // ---- walk the surviving tiles in increasing order; the directory entry of the next one is fetched
            // ahead.  Each lane keeps only its own four bits (one register where warp-wide masks would take four).
            auto next_tile = [&]() -> int {
                const unsigned m = __ballot_sync(FULL, pass4 != 0u);
                if (!m) return -1;
                const int s = __ffs(m) - 1;
                const int j = __ffs(__shfl_sync(FULL, pass4, s)) - 1;
                if (lane == s) pass4 &= pass4 - 1u;
                return tb + 4 * s + j;
            };
            int t = next_tile();
            int2 d_cur = make_int2(0, 0);
            if (t >= 0 && lane < nf) d_cur = drow[t];
            while (t >= 0) {
                const int t_next = next_tile();
                int2 d_next = make_int2(0, 0);
                if (t_next >= 0 && lane < nf) d_next = drow[t_next];

                const float thr_f = xp > 0.f ? fmaxf(fmaf(-xp, tile_bound[t], thr_r), 0.f) : thr_r;
                const val_t thr_c = Ops::threshold(thr_f);
                val_t seen = 0;        // largest value this lane wrote into the tile
                apply_buckets<AccT>(acc, post, d_cur.x, dir_len(d_cur), a0, lane, seen);
                if (nf > 32) {
                    for (int base = 32; base < nf; base += 32) {
                        const int k = base + lane;
                        int b0 = 0, len = 0;
                        float a = 0.f;
                        if (k < nf) {
                            const int2 d = bdir[a_idx[p0 + k] * n_tiles + t];
                            a = Ops::left_weight(a_val[p0 + k] * a_scale);
                            b0 = d.x;
                            len = dir_len(d);
                        }
                        apply_buckets<AccT>(acc, post, b0, len, a, lane, seen);
                    }
                }
                if (!__any_sync(FULL, seen > thr_c)) {
                    // No value written into this tile exceeded the candidate threshold: clearing is enough
                    for (int c = lane; c < n16; c += 32) acc16[c] = zero4;
                } else {
                    // sweep: report scores above the candidate threshold, clear the tile; one atomic per warp step
                    for (int c0 = 0; c0 < n16; c0 += 32) {
                        const int c = c0 + lane;
                        unsigned m = 0;
                        uint4 v = zero4;
                        if (c < n16) {
                            v = acc16[c];
                            if (v.x | v.y | v.z | v.w) {
                                acc16[c] = zero4;
                                m = Ops::above(v, thr_c);
                                // the tile holding the rank: columns before it belong to earlier rows
                                const int below = dr - (t * W + c * Ops::PER16);
                                if (below > 0) m = below >= Ops::PER16 ? 0u : m & (~0u << below);
                                if constexpr (RANGE) {      // the tile holding hi: columns from it on are not the row's
                                    const int room = hr - (t * W + c * Ops::PER16);
                                    if (room < Ops::PER16) m = room <= 0 ? 0u : m & ((1u << room) - 1u);
                                }
                            }
                        }
                        if constexpr (FLOOR) {
                            // the lane's best new lower bound p^ - E_r joins the item's best 32
                            float best = 0.f;
                            for (unsigned mm = m; mm; mm &= mm - 1) best = fmaxf(best, Ops::value(v, __ffs(mm) - 1));
                            const float lb = fmaxf(__fsub_rd(best, e_r), 0.f);
                            if (__any_sync(FULL, lb > __shfl_sync(FULL, kept, fa.top_n - 1))) {
                                floor_merge(kept, lb, lane);
                                const float kth = __shfl_sync(FULL, kept, fa.top_n - 1);
                                if (kth > floor_seen) {
                                    floor_seen = kth;
                                    if (lane == 0) atomicMax(reinterpret_cast<int *>(fa.floor + row), __float_as_int(kth));
                                    thr_r = fmaxf(thr_r, __fsub_rd(__fsub_rd(kth, e_r), FLOOR_EPS));
                                }
                            }
                        }
                        if (__any_sync(FULL, m != 0)) {
                            const int cnt = __popc(m);
                            int incl = cnt;
#pragma unroll
                            for (int o = 1; o < 32; o <<= 1) {
                                const int up = __shfl_up_sync(FULL, incl, o);
                                if (lane >= o) incl += up;
                            }
                            unsigned long long slot = 0;
                            if (lane == 31) slot = atomicAdd(cand_count, (unsigned long long)incl);
                            slot = __shfl_sync(FULL, slot, 31) + (unsigned long long)(incl - cnt);
                            while (m) {
                                const int i = __ffs(m) - 1;
                                m &= m - 1;
                                if (slot < cap) {
                                    const int col = t * W + c * Ops::PER16 + i;
                                    cand_row[slot] = (int32_t)row;
                                    cand_col[slot] = perm_b ? perm_b[col] : col;
                                    if (cand_partial) cand_partial[slot] = Ops::value(v, i);
                                }
                                ++slot;
                            }
                        }
                    }
                }
                __syncwarp();
                t = t_next;
                d_cur = d_next;
            }
        }
    }
}

#define SG_CAND_PARAMS                                                                                              \
    const int64_t *__restrict__ a_indptr, const int32_t *__restrict__ a_len, const int32_t *__restrict__ a_idx,     \
        const float *__restrict__ a_val, int64_t row_begin, int64_t row_end, const int32_t *__restrict__ perm_a,    \
        int64_t n_right, const int2 *__restrict__ bdir, const uint32_t *__restrict__ maxw_h,                        \
        const uint32_t *__restrict__ post, const int32_t *__restrict__ perm_b, int Tp, int W, int64_t T,            \
        int64_t tiles_per_group, float a_scale, float b_scale, float thr_all, const float *__restrict__ thr_row,    \
        const float *__restrict__ xp_norm, const float *__restrict__ tile_bound,                                    \
        const int32_t *__restrict__ diag_rank, const unsigned long long *__restrict__ group_items,                  \
        int32_t *__restrict__ cand_row, int32_t *__restrict__ cand_col, float *__restrict__ cand_partial,           \
        unsigned long long cap, unsigned long long *__restrict__ cand_count,                                        \
        unsigned long long *__restrict__ row_queue
#define SG_CAND_ARGS                                                                                              \
    a_indptr, a_len, a_idx, a_val, row_begin, row_end, perm_a, n_right, bdir, maxw_h, post, perm_b, Tp, W, T,     \
        tiles_per_group, a_scale, b_scale, thr_all, thr_row, xp_norm, tile_bound, diag_rank, group_items, cand_row, \
        cand_col, cand_partial, cap, cand_count, row_queue

template <int NW, typename AccT>
__global__ void __launch_bounds__(NW * 32, min_ctas(NW)) cossim_candidates_kernel(SG_CAND_PARAMS) {
    candidates_body<NW, AccT, false>(SG_CAND_ARGS, FloorArgs{});
}

template <int NW, typename AccT>
__global__ void __launch_bounds__(NW * 32, min_ctas(NW)) cossim_candidates_floor_kernel(SG_CAND_PARAMS, FloorArgs fa) {
    candidates_body<NW, AccT, true>(SG_CAND_ARGS, fa);
}

template <int NW, typename AccT>
__global__ void __launch_bounds__(NW * 32, min_ctas(NW))
    cossim_candidates_range_kernel(SG_CAND_PARAMS, const int32_t *__restrict__ hi_pos) {
    candidates_body<NW, AccT, false, true>(SG_CAND_ARGS, FloorArgs{}, hi_pos);
}

template <int NW, typename AccT>
__global__ void __launch_bounds__(NW * 32, min_ctas(NW))
    cossim_candidates_range_floor_kernel(SG_CAND_PARAMS, FloorArgs fa, const int32_t *__restrict__ hi_pos) {
    candidates_body<NW, AccT, true, true>(SG_CAND_ARGS, fa, hi_pos);
}
#undef SG_CAND_PARAMS
#undef SG_CAND_ARGS

// Work items of the triangle.  A row has work in the groups from the one holding its rank on, so group g needs the
// items ridx < last[g] = 1 + the largest ridx whose first group is <= g (a prefix of the launch; exact when the ranks
// grow with ridx, as for the whole processing order and its slices and strides).
// Pass 1: last[first group of ridx] = max(ridx + 1), one atomic per warp and group.
__global__ void diag_last_kernel(int64_t n_rows, const int32_t *__restrict__ perm_a, int64_t row_begin,
                                 const int32_t *__restrict__ diag_rank, int64_t group_cols,
                                 unsigned long long *__restrict__ last) {
    const int64_t ridx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    long long g = -1;
    if (ridx < n_rows) g = diag_rank[perm_a ? perm_a[ridx] : row_begin + ridx] / group_cols;
    const unsigned peers = __match_any_sync(FULL, g);
    if (g >= 0 && lane_id() == 31 - __clz(peers)) atomicMax(last + g, (unsigned long long)(ridx + 1));
}

// Pass 2 (one warp): running maximum of last[] = items of each group, then their exclusive sum, in place;
// items[n_groups] = all items.
__global__ void diag_items_kernel(int64_t n_groups, unsigned long long *__restrict__ items) {
    const int lane = threadIdx.x;
    unsigned long long run_max = 0, run_sum = 0;
    for (int64_t g0 = 0; g0 < n_groups; g0 += 32) {
        const int64_t g = g0 + lane;
        unsigned long long v = g < n_groups ? items[g] : 0ull;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long up = __shfl_up_sync(FULL, v, o);
            if (lane >= o && up > v) v = up;
        }
        if (run_max > v) v = run_max;
        run_max = __shfl_sync(FULL, v, 31);
        if (g >= n_groups) v = 0;                       // lanes past the last group add nothing
        unsigned long long s = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long up = __shfl_up_sync(FULL, s, o);
            if (lane >= o) s += up;
        }
        if (g < n_groups) items[g] = run_sum + s - v;
        run_sum += __shfl_sync(FULL, s, 31);
    }
    if (lane == 0) items[n_groups] = run_sum;
}

// Work items of a position-range product.  Row ridx has work in the groups from lo / group_cols to (hi - 1) / group_cols
// (none when hi <= lo), so group g needs the items first[g] <= ridx < last[g], with last[g] = 1 + the largest ridx whose
// first group is <= g and first[g] = the smallest ridx whose last group is >= g.  Every row with work in g lies in that
// range whatever the order; the range holds no other row with work when lo and hi grow with ridx (the blocked
// processing order and its slices and strides).
// Pass 1: last[first group of ridx] = max(ridx + 1) in items[0, n_groups), (n_rows - first)[last group of ridx] =
// max(n_rows - ridx) in items[n_groups + 1, 2 n_groups + 1), one atomic per warp and group.
__global__ void range_groups_kernel(int64_t n_rows, const int32_t *__restrict__ perm_a, int64_t row_begin,
                                    const int32_t *__restrict__ lo_pos, const int32_t *__restrict__ hi_pos,
                                    int64_t group_cols, int64_t n_groups, unsigned long long *__restrict__ items) {
    const int64_t ridx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    long long g0 = -1, g1 = -1;
    if (ridx < n_rows) {
        const int64_t row = perm_a ? perm_a[ridx] : row_begin + ridx;
        const int64_t lo = lo_pos[row], hi = hi_pos[row];
        if (hi > lo) {
            g0 = lo / group_cols;
            g1 = (hi - 1) / group_cols;
        }
    }
    unsigned peers = __match_any_sync(FULL, g0);
    if (g0 >= 0 && lane_id() == 31 - __clz(peers)) atomicMax(items + g0, (unsigned long long)(ridx + 1));
    peers = __match_any_sync(FULL, g1);
    if (g1 >= 0 && lane_id() == __ffs(peers) - 1)
        atomicMax(items + n_groups + 1 + g1, (unsigned long long)(n_rows - ridx));
}

// Pass 2 (one warp): first[g] = n_rows - the suffix maximum of pass 1's second half, in place; then the prefix maximum
// of last[], the items max(last[g] - first[g], 0) of each group and their exclusive sum in items[0, n_groups];
// items[n_groups] = all items.
__global__ void range_items_kernel(int64_t n_rows, int64_t n_groups, unsigned long long *__restrict__ items) {
    const int lane = threadIdx.x;
    unsigned long long *first = items + n_groups + 1;
    unsigned long long run = 0;
    for (int64_t g0 = 0; g0 < n_groups; g0 += 32) {           // from the last group down
        const int64_t g = n_groups - 1 - g0 - lane;
        unsigned long long v = g >= 0 ? first[g] : 0ull;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long up = __shfl_up_sync(FULL, v, o);
            if (lane >= o && up > v) v = up;
        }
        if (run > v) v = run;
        run = __shfl_sync(FULL, v, 31);
        if (g >= 0) first[g] = (unsigned long long)n_rows - v;
    }
    unsigned long long run_max = 0, run_sum = 0;
    for (int64_t g0 = 0; g0 < n_groups; g0 += 32) {
        const int64_t g = g0 + lane;
        unsigned long long v = g < n_groups ? items[g] : 0ull;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long up = __shfl_up_sync(FULL, v, o);
            if (lane >= o && up > v) v = up;
        }
        if (run_max > v) v = run_max;
        run_max = __shfl_sync(FULL, v, 31);
        const unsigned long long c = (g < n_groups && v > first[g]) ? v - first[g] : 0ull;
        unsigned long long s = c;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long up = __shfl_up_sync(FULL, s, o);
            if (lane >= o) s += up;
        }
        if (g < n_groups) items[g] = run_sum + s - c;
        run_sum += __shfl_sync(FULL, s, 31);
    }
    if (lane == 0) items[n_groups] = run_sum;
}

// ---------------------------------------------------------------------------
// exact re-scoring
// ---------------------------------------------------------------------------
template <typename T>
struct ExactOps;
template <>
struct ExactOps<double> {
    static __device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
    static __device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
};
template <>
struct ExactOps<float> {
    static __device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
    static __device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
};

template <typename T>
__device__ __forceinline__ T merge_dot(const int32_t *__restrict__ ai, const T *__restrict__ av, int64_t pa,
                                       int64_t ea, const int32_t *__restrict__ bi,
                                       const T *__restrict__ bv, int64_t pb, int64_t eb) {
    T sum = (T)0;
    if (pa >= ea || pb >= eb) return sum;
    int32_t fa = ai[pa], fb = bi[pb];
    for (;;) {
        if (fa == fb) {
            sum = ExactOps<T>::add(sum, ExactOps<T>::mul(av[pa], bv[pb]));
            ++pa;
            ++pb;
            if (pa >= ea || pb >= eb) break;
            fa = ai[pa];
            fb = bi[pb];
        } else if (fa < fb) {
            if (++pa >= ea) break;
            fa = ai[pa];
        } else {
            if (++pb >= eb) break;
            fb = bi[pb];
        }
    }
    return sum;
}

// Same sum, same order, fewer L1 wavefronts: the right row's indices are the scattered loads of this kernel (every
// lane its own row), so they come four at a time as aligned 16-byte vectors (elements of the neighbouring row in the
// first vector are skipped; the last, partial vector is read by scalar loads so nothing beyond the row is touched).
// The left row is shared by most lanes of a warp (candidates arrive grouped by row): its loads are broadcasts.
template <typename T>
__device__ __forceinline__ T merge_dot_vec(const int32_t *__restrict__ ai, const T *__restrict__ av, int64_t pa,
                                           int64_t ea, const int32_t *__restrict__ bi,
                                           const T *__restrict__ bv, int64_t pb, int64_t eb) {
    T sum = (T)0;
    if (pa >= ea || pb >= eb) return sum;
    const int32_t END = 0x7fffffff;
    int32_t fa = ai[pa];
    for (int64_t k = pb & ~(int64_t)3; k < eb; k += 4) {
        int32_t f[4];
        if (k + 4 <= eb) {
            const int4 q = __ldg(reinterpret_cast<const int4 *>(bi + k));
            f[0] = q.x, f[1] = q.y, f[2] = q.z, f[3] = q.w;
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) f[j] = k + j < eb ? bi[k + j] : END;
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int64_t p = k + j;
            if (p < pb || p >= eb) continue;
            const int32_t fb = f[j];
            while (fa < fb) {
                if (++pa >= ea) return sum;
                fa = ai[pa];
            }
            if (fa == fb) sum = ExactOps<T>::add(sum, ExactOps<T>::mul(av[pa], bv[p]));
        }
    }
    return sum;
}

// `keep_count` == NULL: out[i] = exact score of candidate i.  Otherwise only the candidates whose exact score
// exceeds `keep_thr` (strict, string_grouper.py:729/:740) survive, appended in no particular order to
// (keep_row, keep_col, out) through one warp-aggregated atomic per warp: the selection sorts that follow then
// work on the matches-to-be instead of on every candidate the pruned traversal had to report.
//
// Mirror (`mirror_count` != NULL, the triangle of a self-match): every kept pair (r, c) with r != c is also written
// as (c, r) with the same score, right behind the warp's own pairs.  The mirrored score is the exact one: the
// sorted merge multiplies the same two values in the other order (IEEE products commute) and adds the products in
// the same ascending feature order, so score(c, r) is score(r, c) bit for bit.
__device__ __forceinline__ void keep_pairs(bool keep, bool mir, int32_t r, int32_t c, double sc, int lane,
                                           int32_t *__restrict__ keep_row, int32_t *__restrict__ keep_col,
                                           double *__restrict__ out, unsigned long long *__restrict__ keep_count,
                                           unsigned long long *__restrict__ mirror_count,
                                           int32_t *__restrict__ row_cnt, int64_t row_begin) {
    const unsigned m = __ballot_sync(FULL, keep);
    if (!m) return;
    const unsigned mm = __ballot_sync(FULL, mir);
    const int leader = __ffs(m) - 1;
    unsigned long long base = 0;
    if (lane == leader) {
        base = atomicAdd(keep_count, (unsigned long long)(__popc(m) + __popc(mm)));
        if (mm) atomicAdd(mirror_count, (unsigned long long)__popc(mm));
    }
    base = __shfl_sync(FULL, base, leader);
    const unsigned lt = (1u << lane) - 1u;
    if (keep) {
        const unsigned long long w = base + __popc(m & lt);
        keep_row[w] = r;
        keep_col[w] = c;
        out[w] = sc;
        if (row_cnt) atomicAdd(row_cnt + (r - row_begin), 1);       // survivors per row: sizes the row buckets of
                                                                    // sg_topn_select_rows
    }
    if (mir) {
        const unsigned long long w = base + __popc(m) + __popc(mm & lt);
        keep_row[w] = c;
        keep_col[w] = r;
        out[w] = sc;
        if (row_cnt) atomicAdd(row_cnt + (c - row_begin), 1);
    }
}

// Top-n floor of the re-score (sg_rescore_floor / sg_rescore_refined_floor): a pair above the threshold is kept only
// if its exact score is >= floor[r] (at least top_n pairs of the row score that much, so it changes no output);
// `dropped` (optional) counts the pairs above the threshold the floor removed.  The refined kernel's grouped bound
// tests against max(row_threshold[r], floor[r] - FLOOR_EPS - E_r), E_r = margin + margin_pf * row_len[r] as in the
// candidates kernel.
struct RescoreFloor {
    const float *floor;
    const int32_t *row_len;
    float margin, margin_pf;
    unsigned long long *dropped;
};

__device__ __forceinline__ bool floor_keep(bool keep, int32_t r, double sc, const RescoreFloor &rf) {
    const bool drop = keep && sc < (double)rf.floor[r];
    if (rf.dropped) {
        const unsigned m = __ballot_sync(FULL, drop);
        if (m && lane_id() == __ffs(m) - 1) atomicAdd(rf.dropped, (unsigned long long)__popc(m));
    }
    return keep && !drop;
}

// Arg-max re-score (sg_rescore_nearest / sg_rescore_refined_nearest): best[r - row_begin] holds the order-preserving
// bits of the largest exact score row r has met so far (atomicMax; zero = none yet).  A pair above the threshold (and
// the floor) is written only if its score is at least that running best.  The best only rises, so every pair whose
// score equals the row's final best is written; sg_nearest_master then takes the lowest column among them.
struct RescoreNearest : RescoreFloor {
    unsigned long long *best;
};

__device__ __forceinline__ unsigned long long score_order_bits(double x) {
    const unsigned long long b = (unsigned long long)__double_as_longlong(x);
    return (b >> 63) ? ~b : (b | 0x8000000000000000ull);      // order-preserving map of IEEE doubles to unsigned
}

__device__ __forceinline__ bool nearest_keep(bool keep, int32_t r, int64_t row_begin, double sc,
                                             const RescoreFloor &) {
    return keep;
}
__device__ __forceinline__ bool nearest_keep(bool keep, int32_t r, int64_t row_begin, double sc,
                                             const RescoreNearest &rn) {
    if (!keep) return false;
    const unsigned long long b = score_order_bits(sc);
    return atomicMax(rn.best + (r - row_begin), b) <= b;
}

template <typename T, int VEC, typename RF = RescoreFloor>
__global__ void __launch_bounds__(256, 8) rescore_kernel(int64_t n, const int32_t *__restrict__ cr, const int32_t *__restrict__ cc,
                               const int64_t *__restrict__ a_indptr, const int32_t *__restrict__ a_idx,
                               const T *__restrict__ a_val, const int64_t *__restrict__ b_indptr,
                               const int32_t *__restrict__ b_idx, const T *__restrict__ b_val,
                               double *__restrict__ out, double keep_thr, int32_t *__restrict__ keep_row,
                               int32_t *__restrict__ keep_col, unsigned long long *__restrict__ keep_count,
                               unsigned long long *__restrict__ mirror_count, int32_t *__restrict__ row_cnt,
                               int64_t row_begin, RF rf) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int32_t r = 0, c = 0;
    double sc = 0.0;
    bool keep = false;
    if (i < n) {
        r = cr[i];
        c = cc[i];
        sc = VEC ? (double)merge_dot_vec<T>(a_idx, a_val, a_indptr[r], a_indptr[r + 1], b_idx, b_val, b_indptr[c],
                                            b_indptr[c + 1])
                 : (double)merge_dot<T>(a_idx, a_val, a_indptr[r], a_indptr[r + 1], b_idx, b_val, b_indptr[c],
                                        b_indptr[c + 1]);
        if (!keep_count) out[i] = sc;
        keep = keep_count && sc > keep_thr;
    }
    if (!keep_count) return;
    if (rf.floor) keep = floor_keep(keep, r, sc, rf);
    keep = nearest_keep(keep, r, row_begin, sc, rf);
    keep_pairs(keep, keep && mirror_count && r != c, r, c, sc, threadIdx.x & 31, keep_row, keep_col, out, keep_count,
               mirror_count, row_cnt, row_begin);
}

// sg_rescore_refined: a CTA takes REFINE_CHUNK consecutive candidates.  Pass 1 re-tests each with the grouped bound
// (one 32-byte sector of the column's group norms, the row's are shared by neighbours) and compacts the survivors'
// positions into shared memory; pass 2 scores the survivors with full warps, exactly as rescore_kernel does.
constexpr int REFINE_CHUNK = 2048;

__device__ __forceinline__ float group_dot8(const uint4 &x, const uint4 &y, float d) {
    const __half2 *xh = reinterpret_cast<const __half2 *>(&x);
    const __half2 *yh = reinterpret_cast<const __half2 *>(&y);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float2 a = __half22float2(xh[k]), b = __half22float2(yh[k]);
        d = fmaf(a.x, b.x, d);          // products of two fp16 values are exact in fp32
        d = fmaf(a.y, b.y, d);
    }
    return d;
}
// sum over the 16 groups of |x_P,g| |y_H,g| (fp16[16] per row, csrc/sg_prune.cu), the fp32 additions rounded up
__device__ __forceinline__ float group_dot(const uint4 *__restrict__ x, const uint4 *__restrict__ y) {
    const float d = group_dot8(x[1], __ldg(y + 1), group_dot8(x[0], __ldg(y), 0.f));
    return d * (1.f + 1e-5f) + 1e-6f;
}

template <typename T, int VEC, typename RF = RescoreFloor>
__global__ void __launch_bounds__(256, 8)
rescore_refined_kernel(int64_t n, const int32_t *__restrict__ cr, const int32_t *__restrict__ cc,
                       const float *__restrict__ partial, const uint4 *__restrict__ xg,
                       const uint4 *__restrict__ yg, const float *__restrict__ thr_row,
                       const int64_t *__restrict__ a_indptr, const int32_t *__restrict__ a_idx,
                       const T *__restrict__ a_val, const int64_t *__restrict__ b_indptr,
                       const int32_t *__restrict__ b_idx, const T *__restrict__ b_val, double *__restrict__ out,
                       double keep_thr, int32_t *__restrict__ keep_row, int32_t *__restrict__ keep_col,
                       unsigned long long *__restrict__ keep_count, unsigned long long *__restrict__ refined_count,
                       unsigned long long *__restrict__ mirror_count, int32_t *__restrict__ row_cnt,
                       int64_t row_begin, RF rf) {
    __shared__ uint16_t live[REFINE_CHUNK];
    __shared__ int n_live;
    const int lane = threadIdx.x & 31;
    const int64_t base = (int64_t)blockIdx.x * REFINE_CHUNK;
    if (threadIdx.x == 0) n_live = 0;
    __syncthreads();
    for (int o = threadIdx.x; o < REFINE_CHUNK; o += 256) {          // uniform trip count: the ballots need every lane
        const int64_t i = base + o;
        bool pass = false;
        if (i < n) {
            const int32_t r = cr[i], c = cc[i];
            float thr = thr_row[r];
            if (rf.floor) {
                const float e_r = __fmaf_ru(rf.margin_pf, (float)rf.row_len[r], rf.margin);
                thr = fmaxf(thr, __fsub_rd(__fsub_rd(rf.floor[r], e_r), FLOOR_EPS));
            }
            pass = partial[i] + group_dot(xg + 2 * (int64_t)r, yg + 2 * (int64_t)c) > thr;
        }
        const unsigned m = __ballot_sync(FULL, pass);
        if (m) {
            int w = 0;
            if (lane == 0) w = atomicAdd(&n_live, __popc(m));
            w = __shfl_sync(FULL, w, 0);
            if (pass) live[w + __popc(m & ((1u << lane) - 1u))] = (uint16_t)o;
        }
    }
    __syncthreads();
    const int total = n_live;
    if (refined_count && threadIdx.x == 0 && total) atomicAdd(refined_count, (unsigned long long)total);
    for (int j0 = 0; j0 < total; j0 += 256) {
        const int j = j0 + threadIdx.x;
        int32_t r = 0, c = 0;
        double sc = 0.0;
        bool keep = false;
        if (j < total) {
            const int64_t i = base + live[j];
            r = cr[i];
            c = cc[i];
            sc = VEC ? (double)merge_dot_vec<T>(a_idx, a_val, a_indptr[r], a_indptr[r + 1], b_idx, b_val, b_indptr[c],
                                                b_indptr[c + 1])
                     : (double)merge_dot<T>(a_idx, a_val, a_indptr[r], a_indptr[r + 1], b_idx, b_val, b_indptr[c],
                                            b_indptr[c + 1]);
            keep = sc > keep_thr;
        }
        if (rf.floor) keep = floor_keep(keep, r, sc, rf);
        keep = nearest_keep(keep, r, row_begin, sc, rf);
        keep_pairs(keep, keep && mirror_count && r != c, r, c, sc, lane, keep_row, keep_col, out, keep_count,
                   mirror_count, row_cnt, row_begin);
    }
}

// The products of a row pair (common features in ascending order, each multiplied in T), one at a time.
template <typename T>
struct CommonProducts {
    const int32_t *ai, *bi;
    const T *av, *bv;
    int64_t pa, ea, pb, eb;
    __device__ __forceinline__ T next() {      // the caller knows how many there are
        for (;;) {
            const int32_t fa = ai[pa], fb = bi[pb];
            if (fa == fb) return ExactOps<T>::mul(av[pa++], bv[pb++]);
            if (fa < fb) ++pa; else ++pb;
        }
    }
};

template <typename T>
__device__ int64_t count_common(const int32_t *__restrict__ ai, int64_t pa, int64_t ea,
                                const int32_t *__restrict__ bi, int64_t pb, int64_t eb) {
    int64_t k = 0;
    while (pa < ea && pb < eb) {
        const int32_t fa = ai[pa], fb = bi[pb];
        k += fa == fb;
        pa += fa <= fb;
        pb += fb <= fa;
    }
    return k;
}

constexpr int PW_BLOCKSIZE = 128;     // numpy's pairwise-sum block (numpy/_core/src/umath/loops_utils.h.src)

// numpy's pairwise sum of the next n (<= PW_BLOCKSIZE) products: a plain loop below 8 terms, else 8 accumulators over
// the multiple of 8, combined as ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), then the rest one by one
template <typename T>
__device__ __forceinline__ T pairwise_block(CommonProducts<T> &p, int64_t n) {
    T res = (T)0;
    if (n < 8) {
        for (int64_t i = 0; i < n; ++i) res = ExactOps<T>::add(res, p.next());
        return res;
    }
    T r[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = p.next();
    int64_t i = 8;
    for (; i < n - (n % 8); i += 8) {
#pragma unroll
        for (int j = 0; j < 8; ++j) r[j] = ExactOps<T>::add(r[j], p.next());
    }
    res = ExactOps<T>::add(ExactOps<T>::add(ExactOps<T>::add(r[0], r[1]), ExactOps<T>::add(r[2], r[3])),
                           ExactOps<T>::add(ExactOps<T>::add(r[4], r[5]), ExactOps<T>::add(r[6], r[7])));
    for (; i < n; ++i) res = ExactOps<T>::add(res, p.next());
    return res;
}

// StringGrouper.dot = master.multiply(dup).sum(axis=1): scipy reduces a row with np.add.reduceat, i.e. p0 + numpy's
// pairwise sum of p1..pk-1.  Above PW_BLOCKSIZE terms numpy splits n into n2 = n/2 rounded down to a multiple of 8 and
// n - n2 and adds the two halves; the recursion runs here on an explicit stack of pending right halves (the leaves are
// visited left to right, i.e. in the order the merge walk produces the products).
template <typename T>
__global__ void rowwise_dot_kernel(int64_t n, const int64_t *__restrict__ a_indptr,
                                   const int32_t *__restrict__ a_idx, const T *__restrict__ a_val,
                                   const int64_t *__restrict__ b_indptr, const int32_t *__restrict__ b_idx,
                                   const T *__restrict__ b_val, double *__restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t pa = a_indptr[i], ea = a_indptr[i + 1], pb = b_indptr[i], eb = b_indptr[i + 1];
    const int64_t k = count_common<T>(a_idx, pa, ea, b_idx, pb, eb);
    if (k == 0) {
        out[i] = 0.0;
        return;
    }
    CommonProducts<T> p{a_idx, b_idx, a_val, b_val, pa, ea, pb, eb};
    const T p0 = p.next();
    if (k == 1) {
        out[i] = (double)p0;
        return;
    }
    int64_t right[32];       // a row has fewer than 2^31 entries: at most 24 halvings down to a block
    T left[32];
    bool have_left[32];
    int sp = 0;
    int64_t m = k - 1;
    T res;
    for (;;) {
        while (m > PW_BLOCKSIZE) {
            int64_t m2 = m / 2;
            m2 -= m2 % 8;
            right[sp] = m - m2;
            have_left[sp] = false;
            ++sp;
            m = m2;
        }
        res = pairwise_block<T>(p, m);
        while (sp > 0 && have_left[sp - 1]) res = ExactOps<T>::add(left[--sp], res);
        if (sp == 0) break;
        left[sp - 1] = res;
        have_left[sp - 1] = true;
        m = right[sp - 1];
    }
    out[i] = (double)ExactOps<T>::add(p0, res);
}

// ---------------------------------------------------------------------------
// top-n selection
// ---------------------------------------------------------------------------
// Candidates are ordered by (row asc, score desc, column desc) with three stable LSD radix-sort passes
// (column, score, row); candidates at or below the threshold are parked behind the last row.  The first
// min(top_n, count) entries of a row segment are then exactly the survivors: larger score first and, among
// EQUAL scores, the larger column (sp_matmul_topn walks its touched-column list in reverse first-touch order
// and only replaces the heap minimum on a strictly greater score, so among exact ties - identical strings -
// it keeps the highest column ids; SURVEY.md Appendix A.3).  They are written score-descending with ties in
// ascending column order (sort=True, string_grouper.py:730/:741).
__global__ void select_init_kernel(int64_t n, const int32_t *__restrict__ cc, uint32_t *__restrict__ key_col,
                                   uint32_t *__restrict__ idx) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    key_col[i] = ~(uint32_t)cc[i];          // descending column
    idx[i] = (uint32_t)i;
}

__global__ void select_score_keys_kernel(int64_t n, const uint32_t *__restrict__ idx, const double *__restrict__ score,
                                         uint64_t *__restrict__ key_score) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint64_t b = (uint64_t)__double_as_longlong(score[idx[i]]);
    b = (b >> 63) ? ~b : (b | 0x8000000000000000ull);   // order-preserving map of IEEE doubles to unsigned
    key_score[i] = ~b;                                  // descending score
}

__global__ void select_row_keys_kernel(int64_t n, const uint32_t *__restrict__ idx, const int32_t *__restrict__ cr,
                                       const double *__restrict__ score, double thr, int64_t row_begin,
                                       int64_t n_rows, uint32_t *__restrict__ key_row) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t c = idx[i];
    key_row[i] = score[c] > thr ? (uint32_t)(cr[c] - (int32_t)row_begin) : (uint32_t)n_rows;
}

__global__ void select_segments_kernel(int64_t n, const uint32_t *__restrict__ key_row, int64_t n_rows,
                                       int64_t *__restrict__ seg) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r > n_rows) return;
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if ((int64_t)key_row[mid] < r) lo = mid + 1; else hi = mid;
    }
    seg[r] = lo;
}

__global__ void select_count_kernel(int64_t n_rows, const int64_t *__restrict__ seg, int top_n,
                                    int64_t *__restrict__ out_cnt, int32_t *__restrict__ out_max) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_rows) return;
    const int64_t c = seg[r + 1] - seg[r];
    const int k = (int)(c < top_n ? c : top_n);
    out_cnt[r] = k;
    if (k > 0) atomicMax(out_max, k);
}

// one thread per output entry; position inside the row = k, mirrored inside its run of equal scores
__global__ void select_write_kernel(int64_t n_rows, int64_t row_begin, const int64_t *__restrict__ seg,
                                    const uint32_t *__restrict__ idx, const int32_t *__restrict__ cc,
                                    const double *__restrict__ score, const int64_t *__restrict__ out_indptr,
                                    int32_t *__restrict__ out_row, int32_t *__restrict__ out_col,
                                    double *__restrict__ out_score) {
    const int64_t o = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= out_indptr[n_rows]) return;
    // row of this output slot: largest r with out_indptr[r] <= o
    int64_t lo = 0, hi = n_rows;
    while (lo < hi) {
        const int64_t mid = (lo + hi + 1) >> 1;
        if (out_indptr[mid] <= o) lo = mid; else hi = mid - 1;
    }
    const int64_t r = lo;
    const int64_t k = o - out_indptr[r];
    const int64_t n_out = out_indptr[r + 1] - out_indptr[r];
    const int64_t base = seg[r];
    const uint32_t c = idx[base + k];
    const double sc = score[c];
    int64_t a = k, b = k + 1;                       // run [a, b) of equal scores among the survivors
    while (a > 0 && score[idx[base + a - 1]] == sc) --a;
    while (b < n_out && score[idx[base + b]] == sc) ++b;
    const int64_t w = out_indptr[r] + a + (b - 1 - k);
    out_row[w] = (int32_t)(r + row_begin);
    out_col[w] = cc[c];
    out_score[w] = sc;
}

__global__ void select_finish_kernel(int64_t n_rows, const int64_t *__restrict__ out_indptr,
                                     int64_t *__restrict__ out_nnz) {
    if (threadIdx.x == 0 && blockIdx.x == 0) *out_nnz = out_indptr[n_rows];
}

static int bits_for(uint64_t v) {
    int b = 0;
    while (v) { ++b; v >>= 1; }
    return b < 1 ? 1 : b;
}

}  // namespace sg

using namespace sg;

extern "C" {

int64_t sg_num_tiles(int64_t n_right, int tile_w) {
    if (tile_w <= 0) return 0;
    const int64_t t = (n_right + tile_w - 1) / tile_w;
    return t < 1 ? 1 : t;
}

// scratch of sg_postings_build: tile counts, offsets and segment ends, the segmented sort's key / posting buffers,
// the scratch of the scan and of the segmented sort
static size_t postings_scan_bytes(int64_t n_tiles) {
    size_t b = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, b, (int32_t *)nullptr, (int32_t *)nullptr, n_tiles + 1);
    return b;
}
static size_t postings_sort_bytes(int64_t nnz, int64_t n_cols, int64_t n_tiles) {
    size_t b = 0;
    cub::DoubleBuffer<uint32_t> k(nullptr, nullptr), v(nullptr, nullptr);
    cub::DeviceSegmentedRadixSort::SortPairs(nullptr, b, k, v, (int)nnz, (int)n_tiles, (int32_t *)nullptr,
                                             (int32_t *)nullptr, 0, bits_for((uint64_t)n_cols));
    return b;
}

size_t sg_postings_workspace_bytes(int64_t nnz, int64_t n_cols, int64_t n_tiles) {
    return 3 * align_up((size_t)(n_tiles + 1) * 4, 256) + 3 * align_up((size_t)(nnz > 0 ? nnz : 1) * 4, 256) +
           align_up(postings_scan_bytes(n_tiles), 256) + align_up(postings_sort_bytes(nnz, n_cols, n_tiles), 256) +
           4096;
}

int64_t sg_num_tiles_padded(int64_t n_right, int tile_w) {
    return (sg_num_tiles(n_right, tile_w) + 63) / 64 * 64;
}

int sg_postings_build(int64_t n_rows, int64_t n_cols, int64_t nnz, const int64_t *indptr, const int32_t *indices,
                      const float *val32, const int32_t *perm, int tile_w, int64_t indptr_base, float w_scale,
                      void *bucket_dir, void *bucket_maxw, void *postings, int32_t *n_spilled, void *ws,
                      size_t ws_bytes, void *stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    (void)indptr_base;      // indptr holds absolute positions into indices / val32
    if (tile_w <= 0 || (tile_w & 31) || tile_w > 32768)
        return fail(SG_ERR_INVALID, "tile_w must be a multiple of 32 up to 32768 (16-bit bucket lengths)");
    if (nnz >= (int64_t)0x7fffffff)
        return fail(SG_ERR_OVERFLOW, "right matrix nnz %lld does not fit int32 postings", (long long)nnz);
    if (!bucket_dir || !bucket_maxw || !postings) return fail(SG_ERR_INVALID, "postings outputs must not be NULL");
    const int64_t T = sg_num_tiles(n_rows, tile_w);
    const int64_t Tp = sg_num_tiles_padded(n_rows, tile_w);
    const int64_t V1 = n_cols + 1;
    if (T * V1 >= (int64_t)0x7fffffff) return fail(SG_ERR_OVERFLOW, "bucket table %lld too large", (long long)(T * V1));
    const int key_bits = bits_for((uint64_t)n_cols);
    Arena ar(ws, ws_bytes);
    int32_t *tile_cnt = ar.take<int32_t>((size_t)T + 1);
    int32_t *tile_off = ar.take<int32_t>((size_t)T + 1);
    int32_t *big_end = ar.take<int32_t>((size_t)T + 1);
    const size_t n_buf = (size_t)(nnz > 0 ? nnz : 1);
    uint32_t *big_key = ar.take<uint32_t>(n_buf), *big_key2 = ar.take<uint32_t>(n_buf);
    uint32_t *big_post = ar.take<uint32_t>(n_buf);
    size_t scan_bytes = postings_scan_bytes(T), sort_bytes = postings_sort_bytes(nnz, n_cols, T);
    char *scan_tmp = ar.take<char>(scan_bytes), *sort_tmp = ar.take<char>(sort_bytes);
    if (!ar.ok()) return fail(SG_ERR_INVALID, "postings workspace too small (%zu < %zu)", ws_bytes, ar.off);

    // empty buckets and the padding tiles up to Tp stay zero
    SG_CUDA_TRY(cudaMemsetAsync(bucket_dir, 0, (size_t)(T * V1) * 8, st));
    SG_CUDA_TRY(cudaMemsetAsync(bucket_maxw, 0, (size_t)(V1 * Tp) * 2, st));
    if (n_rows <= 0 || nnz <= 0) return SG_OK;
    postings_tile_count_kernel<<<(unsigned)((T + 1 + 7) / 8), 256, 0, st>>>(n_rows, T, tile_w, indptr, perm,
                                                                            tile_cnt);
    SG_LAUNCH_CHECK();
    SG_CUDA_TRY(cub::DeviceScan::ExclusiveSum(scan_tmp, scan_bytes, tile_cnt, tile_off, T + 1, st));
    SG_CUDA_TRY(cudaFuncSetAttribute(postings_tile_build_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)PB_SMEM));
    postings_tile_build_kernel<<<(unsigned)T, PB_THREADS, PB_SMEM, st>>>(
        n_rows, T, Tp, tile_w, key_bits, indptr, indices, val32, perm, w_scale, tile_off, (uint32_t *)postings,
        (int2 *)bucket_dir, (unsigned short *)bucket_maxw, big_key, big_post, big_end, n_spilled);
    SG_LAUNCH_CHECK();
    // tiles of more than PB_CAP postings: sorted in global memory; the other segments are empty
    cub::DoubleBuffer<uint32_t> keys(big_key, big_key2), vals(big_post, (uint32_t *)postings);
    SG_CUDA_TRY(cub::DeviceSegmentedRadixSort::SortPairs(sort_tmp, sort_bytes, keys, vals, (int)nnz, (int)T, tile_off,
                                                         big_end, 0, key_bits, st));
    postings_big_dir_kernel<<<(unsigned)T, 256, 0, st>>>(T, Tp, tile_off, big_end, keys.Current(), vals.Current(),
                                                         (uint32_t *)postings, (int2 *)bucket_dir,
                                                         (unsigned short *)bucket_maxw);
    SG_LAUNCH_CHECK();
    return SG_OK;
}

}  // extern "C"

template <int NW, typename AccT, bool FLOOR, bool RANGE = false>
static int launch_candidates(const int64_t *a_indptr, const int32_t *a_len, const int32_t *a_indices,
                             const float *a_val32, int64_t row_begin, int64_t row_end, const int32_t *perm_a,
                             int64_t n_right, int64_t n_cols, const void *bucket_dir, const void *bucket_maxw,
                             const void *postings, const int32_t *perm_b, int tile_w, int64_t tiles_per_group,
                             float a_scale, float b_scale,
                             float thr_c, const float *thr_row, const float *xp_norm, const float *tile_bound,
                             const int32_t *diag_rank, unsigned long long *group_items,
                             int32_t *cand_row, int32_t *cand_col, float *cand_partial,
                             int64_t cand_cap, unsigned long long *cand_count, unsigned long long *row_queue,
                             int n_sm, cudaStream_t st, const FloorArgs &fa, const int32_t *hi_pos = nullptr) {
    const size_t smem = (size_t)NW * tile_w * sizeof(AccT);
    const void *kern;
    if constexpr (RANGE && FLOOR) kern = (const void *)cossim_candidates_range_floor_kernel<NW, AccT>;
    else if constexpr (RANGE) kern = (const void *)cossim_candidates_range_kernel<NW, AccT>;
    else if constexpr (FLOOR) kern = (const void *)cossim_candidates_floor_kernel<NW, AccT>;
    else kern = (const void *)cossim_candidates_kernel<NW, AccT>;
    SG_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int64_t T = sg_num_tiles(n_right, tile_w);
    const int64_t n_rows = row_end - row_begin;
    // the seed of a keyed floor launch hands out one item per row without group_items (candidates_body)
    const bool items = !(RANGE && FLOOR && fa.seed);
    if constexpr (RANGE) {
        if (items) {
            const int64_t n_groups = (T + tiles_per_group - 1) / tiles_per_group;
            SG_CUDA_TRY(cudaMemsetAsync(group_items, 0, (size_t)(2 * n_groups + 1) * sizeof(unsigned long long), st));
            range_groups_kernel<<<(unsigned)((n_rows + 255) / 256), 256, 0, st>>>(
                n_rows, perm_a, row_begin, diag_rank, hi_pos, tiles_per_group * tile_w, n_groups, group_items);
            SG_LAUNCH_CHECK();
            range_items_kernel<<<1, 32, 0, st>>>(n_rows, n_groups, group_items);
            SG_LAUNCH_CHECK();
        }
    } else if (diag_rank) {
        const int64_t n_groups = (T + tiles_per_group - 1) / tiles_per_group;
        SG_CUDA_TRY(cudaMemsetAsync(group_items, 0, (size_t)(n_groups + 1) * sizeof(unsigned long long), st));
        diag_last_kernel<<<(unsigned)((n_rows + 255) / 256), 256, 0, st>>>(n_rows, perm_a, row_begin, diag_rank,
                                                                           tiles_per_group * tile_w, group_items);
        SG_LAUNCH_CHECK();
        diag_items_kernel<<<1, 32, 0, st>>>(n_groups, group_items);
        SG_LAUNCH_CHECK();
    }
    int per_sm = 1;
    SG_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, NW * 32, smem));
    if (per_sm < 1) per_sm = 1;
    int64_t ctas = (n_rows + NW - 1) / NW;
    if (ctas > (int64_t)n_sm * per_sm) ctas = (int64_t)n_sm * per_sm;   // persistent grid: resident CTAs x SMs
    if (ctas < 1) ctas = 1;
#define SG_KARGS                                                                                                    \
    a_indptr, a_len, a_indices, a_val32, row_begin, row_end, perm_a, n_right, (const int2 *)bucket_dir,               \
        (const uint32_t *)bucket_maxw, (const uint32_t *)postings, perm_b, (int)sg_num_tiles_padded(n_right, tile_w), \
        tile_w, T, tiles_per_group, a_scale, b_scale, thr_c, thr_row, xp_norm, tile_bound, diag_rank,                \
        diag_rank && items ? group_items : nullptr, cand_row, cand_col, cand_partial, (unsigned long long)cand_cap,  \
        cand_count, row_queue
    if constexpr (RANGE && FLOOR)
        cossim_candidates_range_floor_kernel<NW, AccT><<<(unsigned)ctas, NW * 32, smem, st>>>(SG_KARGS, fa, hi_pos);
    else if constexpr (RANGE)
        cossim_candidates_range_kernel<NW, AccT><<<(unsigned)ctas, NW * 32, smem, st>>>(SG_KARGS, hi_pos);
    else if constexpr (FLOOR)
        cossim_candidates_floor_kernel<NW, AccT><<<(unsigned)ctas, NW * 32, smem, st>>>(SG_KARGS, fa);
    else
        cossim_candidates_kernel<NW, AccT><<<(unsigned)ctas, NW * 32, smem, st>>>(SG_KARGS);
#undef SG_KARGS
    SG_LAUNCH_CHECK();
    return SG_OK;
}

// fa == NULL: cossim_candidates_kernel, or with `hi_pos` the position-range variant; otherwise the floor variant,
// with `hi_pos` the floor over a position range
static int cossim_candidates(const int64_t *a_indptr, const int32_t *a_len, const int32_t *a_indices,
                             const float *a_val32, int64_t row_begin, int64_t row_end, const int32_t *perm_a,
                             int64_t n_right, int64_t n_cols, const void *bucket_dir, const void *bucket_maxw,
                             const void *postings, const int32_t *perm_b, int tile_w, int acc_dtype, float a_scale,
                             float b_scale, float cand_threshold,
                             const float *cand_threshold_row, const float *pruned_norm_row, const float *tile_bound,
                             int64_t tiles_per_group, const int32_t *diag_rank, unsigned long long *group_items,
                             int32_t *cand_row, int32_t *cand_col, float *cand_partial, int64_t cand_cap,
                             unsigned long long *cand_count, unsigned long long *row_queue, int warps_per_cta,
                             void *stream_, const FloorArgs *fa, const int32_t *hi_pos = nullptr) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (row_end <= row_begin || n_right <= 0) return SG_OK;
    if (acc_dtype != SG_ACC_F32 && acc_dtype != SG_ACC_U16)
        return fail(SG_ERR_INVALID, "acc_dtype must be SG_ACC_F32 or SG_ACC_U16");
    if (!tile_bound || !bucket_maxw) return fail(SG_ERR_INVALID, "tile_bound and bucket_maxw are required");
    if (diag_rank && !group_items) return fail(SG_ERR_INVALID, "diag_rank needs group_items");
    if (tiles_per_group < 64 || tiles_per_group % 64)
        return fail(SG_ERR_INVALID, "tiles_per_group must be a positive multiple of 64");
    const int acc_bytes = acc_dtype == SG_ACC_U16 ? 2 : 4;
    if (tile_w <= 0 || ((size_t)tile_w * acc_bytes) % 256 || (tile_w & 31))
        return fail(SG_ERR_INVALID, "tile_w must be a multiple of 32 and tile_w * accumulator size a multiple of 256 bytes");
    if (tile_w > 32768) return fail(SG_ERR_INVALID, "tile_w must not exceed 32768 (16-bit bucket lengths)");
    if (!(cand_threshold >= 0.f)) return fail(SG_ERR_INVALID, "cand_threshold must be >= 0");
    if (!(b_scale > 0.f && b_scale <= 1.f)) return fail(SG_ERR_INVALID, "b_scale must be in (0, 1]");
    int dev = 0, n_sm = 0, smem_optin = 0;
    SG_CUDA_TRY(cudaGetDevice(&dev));
    SG_CUDA_TRY(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
    SG_CUDA_TRY(cudaDeviceGetAttribute(&smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    if ((size_t)warps_per_cta * tile_w * acc_bytes > (size_t)smem_optin)
        return fail(SG_ERR_INVALID, "warps_per_cta*tile_w*%d = %zu exceeds %d bytes of shared memory", acc_bytes,
                    (size_t)warps_per_cta * tile_w * acc_bytes, smem_optin);
#define SG_ARGS                                                                                              \
    a_indptr, a_len, a_indices, a_val32, row_begin, row_end, perm_a, n_right, n_cols, bucket_dir, bucket_maxw, \
        postings, perm_b, tile_w, tiles_per_group, a_scale, b_scale, cand_threshold, cand_threshold_row,           \
        pruned_norm_row, tile_bound, diag_rank, group_items, cand_row, cand_col, cand_partial, cand_cap, cand_count, \
        row_queue, n_sm, st
    if (hi_pos) {
        // the range variant is built for the default 8 warps only
        if (warps_per_cta != 8) return fail(SG_ERR_INVALID, "the position-range variant runs with 8 warps per CTA");
        if (!diag_rank || !group_items) return fail(SG_ERR_INVALID, "the position range needs lo_pos and group_items");
        if (fa)
            return acc_dtype == SG_ACC_U16 ? launch_candidates<8, uint16_t, true, true>(SG_ARGS, *fa, hi_pos)
                                           : launch_candidates<8, float, true, true>(SG_ARGS, *fa, hi_pos);
        return acc_dtype == SG_ACC_U16 ? launch_candidates<8, uint16_t, false, true>(SG_ARGS, FloorArgs{}, hi_pos)
                                       : launch_candidates<8, float, false, true>(SG_ARGS, FloorArgs{}, hi_pos);
    }
    if (fa) {
        // the floor variant is built for the default 8 warps only
        if (warps_per_cta != 8) return fail(SG_ERR_INVALID, "the top-n floor variant runs with 8 warps per CTA");
        return acc_dtype == SG_ACC_U16 ? launch_candidates<8, uint16_t, true>(SG_ARGS, *fa)
                                       : launch_candidates<8, float, true>(SG_ARGS, *fa);
    }
    const FloorArgs none{};
#define SG_CASE(NW)                                                                                          \
    case NW:                                                                                                 \
        return acc_dtype == SG_ACC_U16 ? launch_candidates<NW, uint16_t, false>(SG_ARGS, none)              \
                                       : launch_candidates<NW, float, false>(SG_ARGS, none);
    switch (warps_per_cta) {
        SG_CASE(4)
        SG_CASE(8)
        SG_CASE(16)
        SG_CASE(32)
        default:
            return fail(SG_ERR_INVALID, "warps_per_cta must be one of 4, 8, 16, 32");
    }
#undef SG_CASE
#undef SG_ARGS
}

// FloorArgs of sg_cossim_candidates_floor and sg_cossim_candidates_range_floor from their arguments, checked
static int floor_args(FloorArgs &fa, float *row_floor, int top_n, float floor_margin, float floor_margin_per_feature,
                      const int32_t *self_rank, const int32_t *perm_a, int flags) {
    if (!row_floor) return fail(SG_ERR_INVALID, "row_floor is required");
    if (flags & ~(SG_FLOOR_SEED | SG_FLOOR_LONG_ROWS)) return fail(SG_ERR_INVALID, "unknown flags %d", flags);
    const bool seed = (flags & SG_FLOOR_SEED) != 0;
    if (top_n < 1 || top_n > 32) return fail(SG_ERR_INVALID, "the top-n floor supports 1 <= top_n <= 32, got %d", top_n);
    if (!(floor_margin >= 0.f) || !(floor_margin_per_feature >= 0.f))
        return fail(SG_ERR_INVALID, "floor margins must be >= 0");
    if (seed && !self_rank) return fail(SG_ERR_INVALID, "seed needs self_rank");
    if (self_rank && !perm_a) return fail(SG_ERR_INVALID, "self_rank needs perm_a");
    fa = FloorArgs{row_floor, self_rank, seed ? 1 : 0, top_n, floor_margin, floor_margin_per_feature};
    return SG_OK;
}

extern "C" {

int sg_cossim_candidates(const int64_t *a_indptr, const int32_t *a_len, const int32_t *a_indices,
                         const float *a_val32, int64_t row_begin, int64_t row_end, const int32_t *perm_a,
                         int64_t n_right, int64_t n_cols, const void *bucket_dir, const void *bucket_maxw,
                         const void *postings, const int32_t *perm_b, int tile_w, int acc_dtype, float a_scale,
                         float b_scale, float cand_threshold,
                         const float *cand_threshold_row, const float *pruned_norm_row, const float *tile_bound,
                         int64_t tiles_per_group, const int32_t *diag_rank, unsigned long long *group_items,
                         int32_t *cand_row, int32_t *cand_col, float *cand_partial, int64_t cand_cap,
                         unsigned long long *cand_count, unsigned long long *row_queue, int warps_per_cta,
                         void *stream_) {
    return cossim_candidates(a_indptr, a_len, a_indices, a_val32, row_begin, row_end, perm_a, n_right, n_cols,
                             bucket_dir, bucket_maxw, postings, perm_b, tile_w, acc_dtype, a_scale, b_scale,
                             cand_threshold, cand_threshold_row, pruned_norm_row, tile_bound, tiles_per_group,
                             diag_rank, group_items,
                             cand_row, cand_col, cand_partial, cand_cap, cand_count, row_queue, warps_per_cta, stream_,
                             nullptr);
}

int sg_cossim_candidates_floor(const int64_t *a_indptr, const int32_t *a_len, const int32_t *a_indices,
                               const float *a_val32, int64_t row_begin, int64_t row_end, const int32_t *perm_a,
                               int64_t n_right, int64_t n_cols, const void *bucket_dir, const void *bucket_maxw,
                               const void *postings, const int32_t *perm_b, int tile_w, int acc_dtype, float a_scale,
                               float b_scale, float cand_threshold, const float *cand_threshold_row,
                               const float *pruned_norm_row,
                               const float *tile_bound, int64_t tiles_per_group, int32_t *cand_row,
                               int32_t *cand_col, float *cand_partial, int64_t cand_cap,
                               unsigned long long *cand_count, unsigned long long *row_queue, int warps_per_cta,
                               float *row_floor, int top_n, float floor_margin, float floor_margin_per_feature,
                               const int32_t *self_rank, int flags, void *stream_) {
    FloorArgs fa{};
    const int rc = floor_args(fa, row_floor, top_n, floor_margin, floor_margin_per_feature, self_rank, perm_a, flags);
    if (rc != SG_OK) return rc;
    return cossim_candidates(a_indptr, a_len, a_indices, a_val32, row_begin, row_end, perm_a, n_right, n_cols,
                             bucket_dir, bucket_maxw, postings, perm_b, tile_w, acc_dtype, a_scale, b_scale,
                             cand_threshold, cand_threshold_row, pruned_norm_row, tile_bound, tiles_per_group,
                             nullptr, nullptr,
                             cand_row, cand_col, cand_partial, cand_cap, cand_count, row_queue, warps_per_cta, stream_,
                             &fa);
}

int sg_cossim_candidates_range(const int64_t *a_indptr, const int32_t *a_len, const int32_t *a_indices,
                               const float *a_val32, int64_t row_begin, int64_t row_end, const int32_t *perm_a,
                               int64_t n_right, int64_t n_cols, const void *bucket_dir, const void *bucket_maxw,
                               const void *postings, const int32_t *perm_b, int tile_w, int acc_dtype, float a_scale,
                               float b_scale, float cand_threshold, const float *cand_threshold_row,
                               const float *pruned_norm_row,
                               const float *tile_bound, int64_t tiles_per_group, const int32_t *lo_pos,
                               const int32_t *hi_pos, unsigned long long *group_items, int32_t *cand_row,
                               int32_t *cand_col, float *cand_partial, int64_t cand_cap,
                               unsigned long long *cand_count, unsigned long long *row_queue, int warps_per_cta,
                               void *stream_) {
    if (!lo_pos || !hi_pos || !group_items) return fail(SG_ERR_INVALID, "lo_pos, hi_pos and group_items are required");
    return cossim_candidates(a_indptr, a_len, a_indices, a_val32, row_begin, row_end, perm_a, n_right, n_cols,
                             bucket_dir, bucket_maxw, postings, perm_b, tile_w, acc_dtype, a_scale, b_scale,
                             cand_threshold, cand_threshold_row, pruned_norm_row, tile_bound, tiles_per_group,
                             lo_pos, group_items,
                             cand_row, cand_col, cand_partial, cand_cap, cand_count, row_queue, warps_per_cta, stream_,
                             nullptr, hi_pos);
}

int sg_cossim_candidates_range_floor(const int64_t *a_indptr, const int32_t *a_len, const int32_t *a_indices,
                                     const float *a_val32, int64_t row_begin, int64_t row_end, const int32_t *perm_a,
                                     int64_t n_right, int64_t n_cols, const void *bucket_dir, const void *bucket_maxw,
                                     const void *postings, const int32_t *perm_b, int tile_w, int acc_dtype,
                                     float a_scale, float b_scale, float cand_threshold,
                                     const float *cand_threshold_row, const float *pruned_norm_row,
                                     const float *tile_bound, int64_t tiles_per_group, const int32_t *lo_pos,
                                     const int32_t *hi_pos, unsigned long long *group_items, int32_t *cand_row,
                                     int32_t *cand_col, float *cand_partial, int64_t cand_cap,
                                     unsigned long long *cand_count, unsigned long long *row_queue, int warps_per_cta,
                                     float *row_floor, int top_n, float floor_margin, float floor_margin_per_feature,
                                     const int32_t *self_rank, int flags, void *stream_) {
    if (!lo_pos || !hi_pos || !group_items) return fail(SG_ERR_INVALID, "lo_pos, hi_pos and group_items are required");
    FloorArgs fa{};
    const int rc = floor_args(fa, row_floor, top_n, floor_margin, floor_margin_per_feature, self_rank, perm_a, flags);
    if (rc != SG_OK) return rc;
    return cossim_candidates(a_indptr, a_len, a_indices, a_val32, row_begin, row_end, perm_a, n_right, n_cols,
                             bucket_dir, bucket_maxw, postings, perm_b, tile_w, acc_dtype, a_scale, b_scale,
                             cand_threshold, cand_threshold_row, pruned_norm_row, tile_bound, tiles_per_group,
                             lo_pos, group_items,
                             cand_row, cand_col, cand_partial, cand_cap, cand_count, row_queue, warps_per_cta, stream_,
                             &fa, hi_pos);
}

}  // extern "C"

template <typename RF>
static int rescore(int64_t n_cand, const int32_t *cand_row, const int32_t *cand_col, const int64_t *a_indptr,
                   const int32_t *a_indices, const void *a_val, const int64_t *b_indptr, const int32_t *b_indices,
                   const void *b_val, int dtype, double *score_out, double keep_threshold, int32_t *keep_row,
                   int32_t *keep_col, unsigned long long *keep_count, unsigned long long *mirror_count,
                   int32_t *row_cnt, int64_t row_begin, void *stream_, const RF &rf) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (n_cand <= 0) return SG_OK;
    if (keep_count && (!keep_row || !keep_col)) return fail(SG_ERR_INVALID, "keep_count needs keep_row and keep_col");
    if (row_cnt && !keep_count) return fail(SG_ERR_INVALID, "row_cnt needs keep_count");
    if (mirror_count && !keep_count) return fail(SG_ERR_INVALID, "mirror_count needs keep_count");
    const unsigned grid = (unsigned)((n_cand + 255) / 256);
    const bool vec = ((uintptr_t)b_indices & 15) == 0;      // merge_dot_vec reads aligned 16-byte index vectors
#define SG_RESCORE(T, VEC)                                                                                        \
    rescore_kernel<T, VEC, RF><<<grid, 256, 0, st>>>(n_cand, cand_row, cand_col, a_indptr, a_indices,               \
                                                     (const T *)a_val, b_indptr, b_indices, (const T *)b_val,       \
                                                     score_out, keep_threshold, keep_row, keep_col, keep_count,     \
                                                     mirror_count, row_cnt, row_begin, rf)
    if (rf.floor && !keep_count) return fail(SG_ERR_INVALID, "row_floor needs keep_count");
    if (dtype == SG_DTYPE_F64) {
        if (vec) SG_RESCORE(double, 1);
        else SG_RESCORE(double, 0);
    } else if (dtype == SG_DTYPE_F32) {
        if (vec) SG_RESCORE(float, 1);
        else SG_RESCORE(float, 0);
    } else {
        return fail(SG_ERR_INVALID, "dtype must be SG_DTYPE_F32 or SG_DTYPE_F64");
    }
#undef SG_RESCORE
    SG_LAUNCH_CHECK();
    return SG_OK;
}

template <typename RF>
static int rescore_refined(int64_t n_cand, const int32_t *cand_row, const int32_t *cand_col, const float *cand_partial,
                           const void *left_group_norms, const void *right_group_norms, const float *row_threshold,
                           const int64_t *a_indptr, const int32_t *a_indices, const void *a_val,
                           const int64_t *b_indptr, const int32_t *b_indices, const void *b_val, int dtype,
                           double *score_out, double keep_threshold, int32_t *keep_row, int32_t *keep_col,
                           unsigned long long *keep_count, unsigned long long *refined_count,
                           unsigned long long *mirror_count, int32_t *row_cnt, int64_t row_begin, void *stream_,
                           const RF &rf) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (n_cand <= 0) return SG_OK;
    if (!keep_count || !keep_row || !keep_col) return fail(SG_ERR_INVALID, "keep_count, keep_row and keep_col are required");
    if (!cand_partial || !left_group_norms || !right_group_norms || !row_threshold)
        return fail(SG_ERR_INVALID, "partial scores, group norms and row thresholds are required");
    if (((uintptr_t)left_group_norms | (uintptr_t)right_group_norms) & 31)
        return fail(SG_ERR_INVALID, "group norms must be 32-byte aligned");
    const unsigned grid = (unsigned)((n_cand + REFINE_CHUNK - 1) / REFINE_CHUNK);
    const bool vec = ((uintptr_t)b_indices & 15) == 0;
#define SG_RESCORE(T, VEC)                                                                                         \
    rescore_refined_kernel<T, VEC, RF><<<grid, 256, 0, st>>>(                                                       \
        n_cand, cand_row, cand_col, cand_partial, (const uint4 *)left_group_norms, (const uint4 *)right_group_norms, \
        row_threshold, a_indptr, a_indices, (const T *)a_val, b_indptr, b_indices, (const T *)b_val, score_out,      \
        keep_threshold, keep_row, keep_col, keep_count, refined_count, mirror_count, row_cnt, row_begin, rf)
    if (rf.floor && !rf.row_len) return fail(SG_ERR_INVALID, "row_floor needs row_len");
    if (dtype == SG_DTYPE_F64) {
        if (vec) SG_RESCORE(double, 1);
        else SG_RESCORE(double, 0);
    } else if (dtype == SG_DTYPE_F32) {
        if (vec) SG_RESCORE(float, 1);
        else SG_RESCORE(float, 0);
    } else {
        return fail(SG_ERR_INVALID, "dtype must be SG_DTYPE_F32 or SG_DTYPE_F64");
    }
#undef SG_RESCORE
    SG_LAUNCH_CHECK();
    return SG_OK;
}

extern "C" {

int sg_rescore(int64_t n_cand, const int32_t *cand_row, const int32_t *cand_col, const int64_t *a_indptr,
               const int32_t *a_indices, const void *a_val, const int64_t *b_indptr, const int32_t *b_indices,
               const void *b_val, int dtype, double *score_out, double keep_threshold, int32_t *keep_row,
               int32_t *keep_col, unsigned long long *keep_count, unsigned long long *mirror_count,
               int32_t *row_cnt, int64_t row_begin, void *stream_) {
    return rescore(n_cand, cand_row, cand_col, a_indptr, a_indices, a_val, b_indptr, b_indices, b_val, dtype,
                   score_out, keep_threshold, keep_row, keep_col, keep_count, mirror_count, row_cnt, row_begin, stream_,
                   RescoreFloor{});
}

int sg_rescore_floor(int64_t n_cand, const int32_t *cand_row, const int32_t *cand_col, const int64_t *a_indptr,
                     const int32_t *a_indices, const void *a_val, const int64_t *b_indptr, const int32_t *b_indices,
                     const void *b_val, int dtype, double *score_out, double keep_threshold, int32_t *keep_row,
                     int32_t *keep_col, unsigned long long *keep_count, int32_t *row_cnt, int64_t row_begin,
                     const float *row_floor, unsigned long long *floor_dropped, void *stream_) {
    if (!row_floor) return fail(SG_ERR_INVALID, "row_floor is required");
    return rescore(n_cand, cand_row, cand_col, a_indptr, a_indices, a_val, b_indptr, b_indices, b_val, dtype,
                   score_out, keep_threshold, keep_row, keep_col, keep_count, nullptr, row_cnt, row_begin, stream_,
                   RescoreFloor{row_floor, nullptr, 0.f, 0.f, floor_dropped});
}

int sg_rescore_refined(int64_t n_cand, const int32_t *cand_row, const int32_t *cand_col, const float *cand_partial,
                       const void *left_group_norms, const void *right_group_norms, const float *row_threshold,
                       const int64_t *a_indptr, const int32_t *a_indices, const void *a_val,
                       const int64_t *b_indptr, const int32_t *b_indices, const void *b_val, int dtype,
                       double *score_out, double keep_threshold, int32_t *keep_row, int32_t *keep_col,
                       unsigned long long *keep_count, unsigned long long *refined_count,
                       unsigned long long *mirror_count, int32_t *row_cnt, int64_t row_begin, void *stream_) {
    return rescore_refined(n_cand, cand_row, cand_col, cand_partial, left_group_norms, right_group_norms,
                           row_threshold, a_indptr, a_indices, a_val, b_indptr, b_indices, b_val, dtype, score_out,
                           keep_threshold, keep_row, keep_col, keep_count, refined_count, mirror_count, row_cnt,
                           row_begin, stream_, RescoreFloor{});
}

int sg_rescore_refined_floor(int64_t n_cand, const int32_t *cand_row, const int32_t *cand_col,
                             const float *cand_partial, const void *left_group_norms, const void *right_group_norms,
                             const float *row_threshold, const int64_t *a_indptr, const int32_t *a_indices,
                             const void *a_val, const int64_t *b_indptr, const int32_t *b_indices, const void *b_val,
                             int dtype, double *score_out, double keep_threshold, int32_t *keep_row,
                             int32_t *keep_col, unsigned long long *keep_count, unsigned long long *refined_count,
                             int32_t *row_cnt, int64_t row_begin, const float *row_floor, const int32_t *row_len,
                             float floor_margin, float floor_margin_per_feature, unsigned long long *floor_dropped,
                             void *stream_) {
    if (!row_floor) return fail(SG_ERR_INVALID, "row_floor is required");
    return rescore_refined(n_cand, cand_row, cand_col, cand_partial, left_group_norms, right_group_norms,
                           row_threshold, a_indptr, a_indices, a_val, b_indptr, b_indices, b_val, dtype, score_out,
                           keep_threshold, keep_row, keep_col, keep_count, refined_count, nullptr, row_cnt, row_begin,
                           stream_, RescoreFloor{row_floor, row_len, floor_margin, floor_margin_per_feature,
                                                 floor_dropped});
}

int sg_rescore_nearest(int64_t n_cand, const int32_t *cand_row, const int32_t *cand_col, const int64_t *a_indptr,
                       const int32_t *a_indices, const void *a_val, const int64_t *b_indptr, const int32_t *b_indices,
                       const void *b_val, int dtype, double *score_out, double keep_threshold, int32_t *keep_row,
                       int32_t *keep_col, unsigned long long *keep_count, unsigned long long *row_best,
                       int64_t row_begin, const float *row_floor, unsigned long long *floor_dropped, void *stream_) {
    if (!keep_count || !row_best) return fail(SG_ERR_INVALID, "keep_count and row_best are required");
    RescoreNearest rn{};
    rn.floor = row_floor;
    rn.dropped = floor_dropped;
    rn.best = row_best;
    return rescore(n_cand, cand_row, cand_col, a_indptr, a_indices, a_val, b_indptr, b_indices, b_val, dtype,
                   score_out, keep_threshold, keep_row, keep_col, keep_count, nullptr, nullptr, row_begin, stream_, rn);
}

int sg_rescore_refined_nearest(int64_t n_cand, const int32_t *cand_row, const int32_t *cand_col,
                               const float *cand_partial, const void *left_group_norms, const void *right_group_norms,
                               const float *row_threshold, const int64_t *a_indptr, const int32_t *a_indices,
                               const void *a_val, const int64_t *b_indptr, const int32_t *b_indices, const void *b_val,
                               int dtype, double *score_out, double keep_threshold, int32_t *keep_row,
                               int32_t *keep_col, unsigned long long *keep_count, unsigned long long *refined_count,
                               unsigned long long *row_best, int64_t row_begin, const float *row_floor,
                               const int32_t *row_len, float floor_margin, float floor_margin_per_feature,
                               unsigned long long *floor_dropped, void *stream_) {
    if (!row_best) return fail(SG_ERR_INVALID, "row_best is required");
    RescoreNearest rn{};
    rn.floor = row_floor;
    rn.row_len = row_len;
    rn.margin = floor_margin;
    rn.margin_pf = floor_margin_per_feature;
    rn.dropped = floor_dropped;
    rn.best = row_best;
    return rescore_refined(n_cand, cand_row, cand_col, cand_partial, left_group_norms, right_group_norms,
                           row_threshold, a_indptr, a_indices, a_val, b_indptr, b_indices, b_val, dtype, score_out,
                           keep_threshold, keep_row, keep_col, keep_count, refined_count, nullptr, nullptr, row_begin,
                           stream_, rn);
}

int sg_rowwise_dot(int64_t n_rows, const int64_t *a_indptr, const int32_t *a_indices, const void *a_val,
                   const int64_t *b_indptr, const int32_t *b_indices, const void *b_val, int dtype, double *out,
                   void *stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (n_rows <= 0) return SG_OK;
    const unsigned grid = (unsigned)((n_rows + 255) / 256);
    if (dtype == SG_DTYPE_F64)
        rowwise_dot_kernel<double><<<grid, 256, 0, st>>>(n_rows, a_indptr, a_indices, (const double *)a_val,
                                                         b_indptr, b_indices, (const double *)b_val, out);
    else if (dtype == SG_DTYPE_F32)
        rowwise_dot_kernel<float><<<grid, 256, 0, st>>>(n_rows, a_indptr, a_indices, (const float *)a_val,
                                                        b_indptr, b_indices, (const float *)b_val, out);
    else
        return fail(SG_ERR_INVALID, "dtype must be SG_DTYPE_F32 or SG_DTYPE_F64");
    SG_LAUNCH_CHECK();
    return SG_OK;
}

size_t sg_topn_select_workspace_bytes(int64_t n_cand, int64_t n_rows) {
    size_t s32 = 0, s64 = 0, scan_bytes = 0;
    const int64_t n = n_cand < 1 ? 1 : n_cand;
    cub::DeviceRadixSort::SortPairs(nullptr, s32, (uint32_t *)nullptr, (uint32_t *)nullptr, (uint32_t *)nullptr,
                                    (uint32_t *)nullptr, n);
    cub::DeviceRadixSort::SortPairs(nullptr, s64, (uint64_t *)nullptr, (uint64_t *)nullptr, (uint32_t *)nullptr,
                                    (uint32_t *)nullptr, n);
    cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (int64_t *)nullptr, (int64_t *)nullptr, n_rows + 1);
    const size_t sort_bytes = s32 > s64 ? s32 : s64;
    return 2 * align_up((size_t)n * 8, 256) + 4 * align_up((size_t)n * 4, 256) +
           2 * align_up((size_t)(n_rows + 2) * 8, 256) + align_up(sort_bytes, 256) + align_up(scan_bytes, 256) + 4096;
}

int sg_topn_select(int64_t n_cand, const int32_t *cand_row, const int32_t *cand_col, const double *score,
                   int64_t row_begin, int64_t n_rows, int top_n, double threshold, int64_t *out_indptr,
                   int32_t *out_row, int32_t *out_col, double *out_score, int64_t *out_nnz,
                   int32_t *out_max_row, void *ws, size_t ws_bytes, void *stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (n_rows < 0 || n_cand < 0) return fail(SG_ERR_INVALID, "negative size");
    if (n_cand >= (int64_t)0xfffffff0u) return fail(SG_ERR_OVERFLOW, "too many candidates: %lld", (long long)n_cand);
    SG_CUDA_TRY(cudaMemsetAsync(out_max_row, 0, sizeof(int32_t), st));
    if (n_cand == 0 || top_n <= 0) {
        SG_CUDA_TRY(cudaMemsetAsync(out_indptr, 0, (size_t)(n_rows + 1) * sizeof(int64_t), st));
        SG_CUDA_TRY(cudaMemsetAsync(out_nnz, 0, sizeof(int64_t), st));
        return SG_OK;
    }
    Arena ar(ws, ws_bytes);
    uint64_t *k64_in = ar.take<uint64_t>((size_t)n_cand);
    uint64_t *k64_out = ar.take<uint64_t>((size_t)n_cand);
    uint32_t *k32_in = ar.take<uint32_t>((size_t)n_cand);
    uint32_t *k32_out = ar.take<uint32_t>((size_t)n_cand);
    uint32_t *idx_a = ar.take<uint32_t>((size_t)n_cand);
    uint32_t *idx_b = ar.take<uint32_t>((size_t)n_cand);
    int64_t *seg = ar.take<int64_t>((size_t)n_rows + 2);
    int64_t *cnt = ar.take<int64_t>((size_t)n_rows + 2);
    size_t s32 = 0, s64 = 0, scan_bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, s32, k32_in, k32_out, idx_a, idx_b, n_cand);
    cub::DeviceRadixSort::SortPairs(nullptr, s64, k64_in, k64_out, idx_a, idx_b, n_cand);
    cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, cnt, out_indptr, n_rows + 1);
    size_t sort_bytes = s32 > s64 ? s32 : s64;
    char *sort_tmp = ar.take<char>(sort_bytes);
    char *scan_tmp = ar.take<char>(scan_bytes);
    if (!ar.ok()) return fail(SG_ERR_INVALID, "select workspace too small (%zu < %zu)", ws_bytes, ar.off);

    const unsigned g1 = (unsigned)((n_cand + 255) / 256);
    // pass 1: column descending
    select_init_kernel<<<g1, 256, 0, st>>>(n_cand, cand_col, k32_in, idx_a);
    SG_LAUNCH_CHECK();
    SG_CUDA_TRY(cub::DeviceRadixSort::SortPairs(sort_tmp, sort_bytes, k32_in, k32_out, idx_a, idx_b, n_cand, 0, 32, st));
    // pass 2: score descending (stable)
    select_score_keys_kernel<<<g1, 256, 0, st>>>(n_cand, idx_b, score, k64_in);
    SG_LAUNCH_CHECK();
    SG_CUDA_TRY(cub::DeviceRadixSort::SortPairs(sort_tmp, sort_bytes, k64_in, k64_out, idx_b, idx_a, n_cand, 0, 64, st));
    // pass 3: row ascending (stable); candidates not above the threshold go behind the last row
    select_row_keys_kernel<<<g1, 256, 0, st>>>(n_cand, idx_a, cand_row, score, threshold, row_begin, n_rows, k32_in);
    SG_LAUNCH_CHECK();
    SG_CUDA_TRY(cub::DeviceRadixSort::SortPairs(sort_tmp, sort_bytes, k32_in, k32_out, idx_a, idx_b, n_cand, 0,
                                                bits_for((uint64_t)n_rows), st));
    const unsigned g2 = (unsigned)((n_rows + 1 + 255) / 256);
    select_segments_kernel<<<g2, 256, 0, st>>>(n_cand, k32_out, n_rows, seg);
    SG_LAUNCH_CHECK();
    SG_CUDA_TRY(cudaMemsetAsync(cnt, 0, (size_t)(n_rows + 2) * sizeof(int64_t), st));
    if (n_rows > 0) {
        select_count_kernel<<<(unsigned)((n_rows + 255) / 256), 256, 0, st>>>(n_rows, seg, top_n, cnt, out_max_row);
        SG_LAUNCH_CHECK();
    }
    SG_CUDA_TRY(cub::DeviceScan::ExclusiveSum(scan_tmp, scan_bytes, cnt, out_indptr, n_rows + 1, st));
    if (n_rows > 0) {
        // at most min(n_cand, n_rows * top_n) outputs; one thread each (threads beyond the total exit)
        int64_t max_out = n_rows * (int64_t)top_n;
        if (max_out > n_cand) max_out = n_cand;
        select_write_kernel<<<(unsigned)((max_out + 255) / 256), 256, 0, st>>>(n_rows, row_begin, seg, idx_b, cand_col,
                                                                              score, out_indptr, out_row, out_col,
                                                                              out_score);
        SG_LAUNCH_CHECK();
    }
    select_finish_kernel<<<1, 32, 0, st>>>(n_rows, out_indptr, out_nnz);
    SG_LAUNCH_CHECK();
    return SG_OK;
}


// K3 — per-row top-n merge of column-block results: zip_sp_matmul_topn (string_grouper.py:746).  The block results
// arrive concatenated as COO with block column offsets already applied; like the reference's heap (initial minimum =
// the smallest positive normal of the value type, strict >) entries that are not strictly positive are dropped.
size_t sg_topn_merge_workspace_bytes(int64_t n_entries, int64_t n_rows) {
    return sg_topn_select_workspace_bytes(n_entries, n_rows);
}

int sg_topn_merge(int64_t n_entries, const int32_t *row, const int32_t *col, const double *score, int64_t n_rows,
                  int top_n, int dtype, int64_t *out_indptr, int32_t *out_row, int32_t *out_col, double *out_score,
                  int64_t *out_nnz, int32_t *out_max_row, void *ws, size_t ws_bytes, void *stream_) {
    if (dtype != SG_DTYPE_F32 && dtype != SG_DTYPE_F64) return fail(SG_ERR_INVALID, "dtype must be SG_DTYPE_F32 or SG_DTYPE_F64");
    const double tiny = dtype == SG_DTYPE_F32 ? 1.17549435082228750797e-38 : 2.22507385850720138309e-308;
    return sg_topn_select(n_entries, row, col, score, 0, n_rows, top_n, tiny, out_indptr, out_row, out_col, out_score,
                          out_nnz, out_max_row, ws, ws_bytes, stream_);
}

}  // extern "C"
