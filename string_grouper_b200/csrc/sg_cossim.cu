// K2 — blocked CSR x CSR^T, thresholded, top-n per left row, for sm_90a.
//
// Replaces StringGrouper._build_matches
// (string_grouper/string_grouper.py:709-752): the per block
// pair sp_matmul_topn products (:737-743), the zip over right blocks (:746)
// and the vstack over left blocks (:750).  See DESIGN.md §K2 for the layout.
//
//   postings_build   right matrix  -> (feature, column-tile) bucketed postings + directory with block maxima
//   candidates       block-max test of 64 tiles at a time, then the Gustavson row-wise product of the pruned left
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
// postings build: feature-major buckets (feature, column tile) over the processing order of the right rows
// ---------------------------------------------------------------------------
// bucket = f * T + t (feature-major: the buckets a left row walks for one of its features over consecutive column
// tiles are neighbours in the directory and in the posting array), t = rank[doc] / tile_w.
// Pass 1: bucket sizes and the largest |weight| of every bucket.
__global__ void postings_count_kernel(int64_t n_rows, const int64_t *__restrict__ indptr,
                                      const int32_t *__restrict__ indices, const float *__restrict__ val,
                                      const int32_t *__restrict__ rank, int W, int64_t T, float w_scale,
                                      int32_t *__restrict__ cnt, uint32_t *__restrict__ maxw) {
    const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= n_rows) return;
    const int64_t t = (rank ? rank[row] : row) / W;
    const int64_t p1 = indptr[row + 1];
    for (int64_t p = indptr[row] + lane_id(); p < p1; p += 32) {
        const int64_t b = (int64_t)indices[p] * T + t;
        atomicAdd(cnt + b, 1);
        // largest |weight| of the bucket as the fp16 value the kernel will see (non-negative halves order like integers)
        atomicMax(maxw + b, (uint32_t)__half_as_ushort(__float2half_rn(fabsf(val[p] * w_scale))));
    }
}

// Pass 2 (after the scan of the sizes): every posting takes the next free slot of its bucket, counting `cnt` down.
// A posting is 4 bytes: the column inside the tile (16 bits) and the weight rounded to fp16 (16 bits).  The
// candidate scores only have to be within CAND_MARGIN of the exact ones (every candidate is re-scored in the
// matrix dtype): an fp16 weight is off by at most 2^-11 relative, so a score by at most 4.9e-4.  The order inside a
// bucket is whatever the atomics make it (a bucket holds every column once; the fixed-point tiles add integers, so
// the candidate set does not depend on it) — this replaced a 44-bit radix sort of all postings (1.1 of 2.6 ms).
__global__ void postings_scatter_kernel(int64_t n_rows, const int64_t *__restrict__ indptr,
                                        const int32_t *__restrict__ indices, const float *__restrict__ val,
                                        const int32_t *__restrict__ rank, int W, int64_t T, float w_scale,
                                        const int32_t *__restrict__ ptr, int32_t *__restrict__ cnt,
                                        uint32_t *__restrict__ post) {
    const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= n_rows) return;
    const int64_t pos = rank ? rank[row] : row;
    const int64_t t = pos / W;
    const uint32_t local = (uint32_t)(pos - t * W);
    const int64_t p1 = indptr[row + 1];
    for (int64_t p = indptr[row] + lane_id(); p < p1; p += 32) {
        const int64_t b = (int64_t)indices[p] * T + t;
        const int slot = ptr[b] + atomicSub(cnt + b, 1) - 1;
        post[slot] = ((uint32_t)__half_as_ushort(__float2half_rn(val[p] * w_scale)) << 16) | local;
    }
}

__device__ __forceinline__ float post_w(uint32_t e) { return __half2float(__ushort_as_half((unsigned short)(e >> 16))); }
__device__ __forceinline__ int post_c(uint32_t e) { return (int)(e & 0xffffu); }

// bucket directory: one aligned 8-byte entry per (feature, tile) so that a lane fetches it in one load:
// {int32 start, u16 length | fp16 largest |weight| << 16}
__global__ void postings_dir_kernel(int64_t nb, const int32_t *__restrict__ ptr, const uint32_t *__restrict__ maxw,
                                    int2 *__restrict__ dir, int64_t T, int64_t Tp,
                                    unsigned short *__restrict__ maxw_rows) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nb) return;
    dir[i] = make_int2(ptr[i], (int)(((uint32_t)(ptr[i + 1] - ptr[i]) & 0xffffu) | (maxw[i] << 16)));
    // the same maxima as fp16 rows of Tp tiles per feature (zero padded): what the block-max test streams
    if (maxw_rows) maxw_rows[(i / T) * Tp + (i % T)] = (unsigned short)maxw[i];
}

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
#ifndef SG_FILTER_MLP
#define SG_FILTER_MLP 1          // block-maxima loads in flight per lane in the block-max test
// With 40 resident warps the load latency is covered; more loads in flight cost registers and issue slots.
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
// Tp tiles): no column of tile t can collect more than ub(t) = sum_f |a_f| * max|w_(f,t)|.  The bounds of 64 tiles
// are evaluated at once, two tiles per lane in packed fp16 (one HFMA2 per kept feature and tile pair), and only
// the tiles whose bound can exceed their candidate threshold are walked at all: nothing is accumulated, cleared
// or swept for the others.
template <int NW, typename AccT>
__global__ void __launch_bounds__(NW * 32, min_ctas(NW))
cossim_candidates_kernel(const int64_t *__restrict__ a_indptr, const int32_t *__restrict__ a_len,
                         const int32_t *__restrict__ a_idx, const float *__restrict__ a_val, int64_t row_begin,
                         int64_t row_end, const int32_t *__restrict__ perm_a, int64_t n_right,
                         const int2 *__restrict__ bdir, const uint32_t *__restrict__ maxw_h,
                         const uint32_t *__restrict__ post, const int32_t *__restrict__ perm_b, int Tp, int W,
                         int64_t T, int64_t tiles_per_group, float a_scale, float thr_all,
                         const float *__restrict__ thr_row, const float *__restrict__ xp_norm,
                         const float *__restrict__ tile_bound, int32_t *__restrict__ cand_row,
                         int32_t *__restrict__ cand_col, float *__restrict__ cand_partial, unsigned long long cap,
                         unsigned long long *__restrict__ cand_count, unsigned long long *__restrict__ row_queue) {
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
    const unsigned long long n_items = (unsigned long long)n_rows * (unsigned long long)n_groups;
    const int n_tiles = (int)T;
    for (;;) {
        unsigned long long item = 0;
        if (lane == 0) item = atomicAdd(row_queue, 1ull);
        item = __shfl_sync(FULL, item, 0);
        if (item >= n_items) break;
        const int64_t group = (int64_t)(item / (unsigned long long)n_rows);
        const int64_t ridx = (int64_t)(item % (unsigned long long)n_rows);
        const int64_t row = perm_a ? perm_a[ridx] : row_begin + ridx;   // processing order: neighbours share buckets
        const int64_t p0 = a_indptr[row];
        const int nf = a_len ? a_len[row] : (int)(a_indptr[row + 1] - p0);
        if (nf == 0) continue;
        const float thr_r = thr_row ? thr_row[row] : thr_all;
        const float xp = xp_norm ? xp_norm[row] : 0.f;
        // tile ids, directory slots (T * V1 < 2^31, checked by sg_postings_build) and positions fit 32 bits
        const int t_begin = (int)(group * tiles_per_group);
        const int t_end = (int)(t_begin + tiles_per_group < T ? t_begin + tiles_per_group : T);

        // the first 32 features of the row stay in registers
        int f0 = 0;
        float a0 = 0.f;
        __half2 a2 = __float2half2_rn(0.f);
        if (lane < nf) {
            f0 = a_idx[p0 + lane];
            const float a = a_val[p0 + lane] * a_scale;
            a0 = Ops::left_weight(a);
            a2 = __half2half2(__float2half_ru(fabsf(a)));   // rounded up: the bound must not fall short
        }
        const int2 *drow = bdir + f0 * n_tiles;
        const int nk = nf < 32 ? nf : 32;
        // fp16 arithmetic of the bound: one rounding of at most 2^-11 (values below 2) per kept feature
        const float slack = 5e-4f * (float)nk + 1e-4f;

        for (int tb = t_begin; tb < t_end; tb += 64) {
            // ---- bounds of tiles tb + 2*lane and tb + 2*lane + 1
            unsigned m_even, m_odd;
            if (nf <= 32) {
                __half2 ub2 = __float2half2_rn(0.f);
                const uint32_t *mrow = maxw_h + (tb >> 1) + lane;
                // SG_FILTER_MLP block-maxima loads in flight per lane
                for (int k0 = 0; k0 < nk; k0 += SG_FILTER_MLP) {
                    uint32_t m[SG_FILTER_MLP];
                    __half2 ak2[SG_FILTER_MLP];
#pragma unroll
                    for (int u = 0; u < SG_FILTER_MLP; ++u) {
                        const int kk = k0 + u;
                        const int fk = __shfl_sync(FULL, f0, kk & 31);
                        ak2[u] = __shfl_sync(FULL, a2, kk & 31);
                        m[u] = kk < nk ? mrow[fk * (Tp >> 1)] : 0u;
                    }
#pragma unroll
                    for (int u = 0; u < SG_FILTER_MLP; ++u)
                        ub2 = __hfma2(ak2[u], *reinterpret_cast<const __half2 *>(&m[u]), ub2);
                }
                const float2 ub = __half22float2(ub2);
                const float2 tb2 = reinterpret_cast<const float2 *>(tile_bound)[(tb >> 1) + lane];
                const int t0 = tb + 2 * lane;
                const float thr0 = xp > 0.f ? fmaxf(fmaf(-xp, tb2.x, thr_r), 0.f) : thr_r;
                const float thr1 = xp > 0.f ? fmaxf(fmaf(-xp, tb2.y, thr_r), 0.f) : thr_r;
                m_even = __ballot_sync(FULL, t0 < t_end && ub.x + slack > thr0);
                m_odd = __ballot_sync(FULL, t0 + 1 < t_end && ub.y + slack > thr1);
            } else {        // rows with more than 32 kept features: every tile is walked
                const int t0 = tb + 2 * lane;
                m_even = __ballot_sync(FULL, t0 < t_end);
                m_odd = __ballot_sync(FULL, t0 + 1 < t_end);
            }
            // ---- walk the surviving tiles; the directory entry of the next one is fetched ahead
            int t = -1;
            if (m_even) { t = tb + 2 * (__ffs(m_even) - 1); m_even &= m_even - 1; }
            else if (m_odd) { t = tb + 2 * (__ffs(m_odd) - 1) + 1; m_odd &= m_odd - 1; }
            int2 d_cur = make_int2(0, 0);
            if (t >= 0 && lane < nf) d_cur = drow[t];
            while (t >= 0) {
                int t_next = -1;
                if (m_even) { t_next = tb + 2 * (__ffs(m_even) - 1); m_even &= m_even - 1; }
                else if (m_odd) { t_next = tb + 2 * (__ffs(m_odd) - 1) + 1; m_odd &= m_odd - 1; }
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
template <typename T, int VEC>
__global__ void __launch_bounds__(256, 8) rescore_kernel(int64_t n, const int32_t *__restrict__ cr, const int32_t *__restrict__ cc,
                               const int64_t *__restrict__ a_indptr, const int32_t *__restrict__ a_idx,
                               const T *__restrict__ a_val, const int64_t *__restrict__ b_indptr,
                               const int32_t *__restrict__ b_idx, const T *__restrict__ b_val,
                               double *__restrict__ out, double keep_thr, int32_t *__restrict__ keep_row,
                               int32_t *__restrict__ keep_col, unsigned long long *__restrict__ keep_count,
                               int32_t *__restrict__ row_cnt, int64_t row_begin) {
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
    const unsigned m = __ballot_sync(FULL, keep);
    if (!m) return;
    const int lane = threadIdx.x & 31;
    unsigned long long base = 0;
    if (lane == __ffs(m) - 1) base = atomicAdd(keep_count, (unsigned long long)__popc(m));
    base = __shfl_sync(FULL, base, __ffs(m) - 1);
    if (keep) {
        const unsigned long long w = base + __popc(m & ((1u << lane) - 1u));
        keep_row[w] = r;
        keep_col[w] = c;
        out[w] = sc;
        if (row_cnt) atomicAdd(row_cnt + (r - row_begin), 1);       // survivors per row: sizes the row buckets of
                                                                    // sg_topn_select_rows
    }
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

template <typename T, int VEC>
__global__ void __launch_bounds__(256, 8)
rescore_refined_kernel(int64_t n, const int32_t *__restrict__ cr, const int32_t *__restrict__ cc,
                       const float *__restrict__ partial, const uint4 *__restrict__ xg,
                       const uint4 *__restrict__ yg, const float *__restrict__ thr_row,
                       const int64_t *__restrict__ a_indptr, const int32_t *__restrict__ a_idx,
                       const T *__restrict__ a_val, const int64_t *__restrict__ b_indptr,
                       const int32_t *__restrict__ b_idx, const T *__restrict__ b_val, double *__restrict__ out,
                       double keep_thr, int32_t *__restrict__ keep_row, int32_t *__restrict__ keep_col,
                       unsigned long long *__restrict__ keep_count, unsigned long long *__restrict__ refined_count,
                       int32_t *__restrict__ row_cnt, int64_t row_begin) {
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
            pass = partial[i] + group_dot(xg + 2 * (int64_t)r, yg + 2 * (int64_t)c) > thr_row[r];
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
        const unsigned m = __ballot_sync(FULL, keep);
        if (!m) continue;
        unsigned long long w0 = 0;
        if (lane == __ffs(m) - 1) w0 = atomicAdd(keep_count, (unsigned long long)__popc(m));
        w0 = __shfl_sync(FULL, w0, __ffs(m) - 1);
        if (keep) {
            const unsigned long long w = w0 + __popc(m & ((1u << lane) - 1u));
            keep_row[w] = r;
            keep_col[w] = c;
            out[w] = sc;
            if (row_cnt) atomicAdd(row_cnt + (r - row_begin), 1);
        }
    }
}

template <typename T>
__global__ void rowwise_dot_kernel(int64_t n, const int64_t *__restrict__ a_indptr,
                                   const int32_t *__restrict__ a_idx, const T *__restrict__ a_val,
                                   const int64_t *__restrict__ b_indptr, const int32_t *__restrict__ b_idx,
                                   const T *__restrict__ b_val, double *__restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    out[i] = (double)merge_dot<T>(a_idx, a_val, a_indptr[i], a_indptr[i + 1], b_idx, b_val, b_indptr[i],
                                  b_indptr[i + 1]);
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

size_t sg_postings_workspace_bytes(int64_t nnz, int64_t n_cols, int64_t n_tiles) {
    (void)nnz;
    const int64_t nb = n_tiles * (n_cols + 1) + 1;
    size_t b2 = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, b2, (int32_t *)nullptr, (int32_t *)nullptr, nb);
    return 2 * align_up((size_t)nb * 4, 256) + align_up(b2, 256) + 4096;
}

int64_t sg_num_tiles_padded(int64_t n_right, int tile_w) {
    return (sg_num_tiles(n_right, tile_w) + 63) / 64 * 64;
}

int sg_postings_build(int64_t n_rows, int64_t n_cols, int64_t nnz, const int64_t *indptr, const int32_t *indices,
                      const float *val32, const int32_t *rank, int tile_w, int64_t indptr_base, float w_scale,
                      int32_t *bucket_ptr, void *bucket_dir, void *bucket_maxw, void *postings, void *ws,
                      size_t ws_bytes, void *stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    (void)indptr_base;      // indptr holds absolute positions into indices / val32
    if (tile_w <= 0 || (tile_w & 31) || tile_w > 32768)
        return fail(SG_ERR_INVALID, "tile_w must be a multiple of 32 up to 32768 (16-bit bucket lengths)");
    if (nnz >= (int64_t)0x7fffffff)
        return fail(SG_ERR_OVERFLOW, "right matrix nnz %lld does not fit int32 postings", (long long)nnz);
    const int64_t T = sg_num_tiles(n_rows, tile_w);
    const int64_t V1 = n_cols + 1;
    const int64_t nb = T * V1 + 1;
    if (nb >= (int64_t)0x7fffffff) return fail(SG_ERR_OVERFLOW, "bucket table %lld too large", (long long)nb);
    Arena ar(ws, ws_bytes);
    int32_t *cnt = ar.take<int32_t>((size_t)nb);
    uint32_t *maxw = ar.take<uint32_t>((size_t)nb);
    size_t cub_bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, cub_bytes, cnt, bucket_ptr, nb);
    char *tmp = ar.take<char>(cub_bytes);
    if (!ar.ok()) return fail(SG_ERR_INVALID, "postings workspace too small (%zu < %zu)", ws_bytes, ar.off);
    SG_CUDA_TRY(cudaMemsetAsync(cnt, 0, (size_t)nb * 4, st));
    SG_CUDA_TRY(cudaMemsetAsync(maxw, 0, (size_t)nb * 4, st));
    const unsigned row_grid = (unsigned)((n_rows + 7) / 8);
    if (n_rows > 0 && nnz > 0) {
        postings_count_kernel<<<row_grid, 256, 0, st>>>(n_rows, indptr, indices, val32, rank, tile_w, T, w_scale, cnt,
                                                        maxw);
        SG_LAUNCH_CHECK();
    }
    SG_CUDA_TRY(cub::DeviceScan::ExclusiveSum(tmp, cub_bytes, cnt, bucket_ptr, nb, st));
    if (bucket_dir) {
        const int64_t Tp = sg_num_tiles_padded(n_rows, tile_w);
        if (bucket_maxw) SG_CUDA_TRY(cudaMemsetAsync(bucket_maxw, 0, (size_t)(V1 * Tp) * 2, st));
        postings_dir_kernel<<<(unsigned)((nb - 1 + 255) / 256), 256, 0, st>>>(nb - 1, bucket_ptr, maxw,
                                                                              (int2 *)bucket_dir, T, Tp,
                                                                              (unsigned short *)bucket_maxw);
        SG_LAUNCH_CHECK();
    }
    if (n_rows > 0 && nnz > 0) {
        postings_scatter_kernel<<<row_grid, 256, 0, st>>>(n_rows, indptr, indices, val32, rank, tile_w, T, w_scale,
                                                          bucket_ptr, cnt, (uint32_t *)postings);
        SG_LAUNCH_CHECK();
    }
    return SG_OK;
}

}  // extern "C"

template <int NW, typename AccT>
static int launch_candidates(const int64_t *a_indptr, const int32_t *a_len, const int32_t *a_indices,
                             const float *a_val32, int64_t row_begin, int64_t row_end, const int32_t *perm_a,
                             int64_t n_right, int64_t n_cols, const void *bucket_dir, const void *bucket_maxw,
                             const void *postings, const int32_t *perm_b, int tile_w, int64_t tiles_per_group,
                             float a_scale,
                             float thr_c, const float *thr_row, const float *xp_norm, const float *tile_bound,
                             int32_t *cand_row, int32_t *cand_col, float *cand_partial,
                             int64_t cand_cap, unsigned long long *cand_count, unsigned long long *row_queue,
                             int n_sm, cudaStream_t st) {
    const size_t smem = (size_t)NW * tile_w * sizeof(AccT);
    SG_CUDA_TRY(cudaFuncSetAttribute(cossim_candidates_kernel<NW, AccT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)smem));
    const int64_t T = sg_num_tiles(n_right, tile_w);
    const int64_t n_rows = row_end - row_begin;
    int per_sm = 1;
    SG_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, cossim_candidates_kernel<NW, AccT>, NW * 32,
                                                              smem));
    if (per_sm < 1) per_sm = 1;
    int64_t ctas = (n_rows + NW - 1) / NW;
    if (ctas > (int64_t)n_sm * per_sm) ctas = (int64_t)n_sm * per_sm;   // persistent grid: resident CTAs x SMs
    if (ctas < 1) ctas = 1;
    cossim_candidates_kernel<NW, AccT><<<(unsigned)ctas, NW * 32, smem, st>>>(
        a_indptr, a_len, a_indices, a_val32, row_begin, row_end, perm_a, n_right, (const int2 *)bucket_dir,
        (const uint32_t *)bucket_maxw, (const uint32_t *)postings, perm_b, (int)sg_num_tiles_padded(n_right, tile_w),
        tile_w, T, tiles_per_group,
        a_scale, thr_c, thr_row, xp_norm, tile_bound, cand_row, cand_col, cand_partial, (unsigned long long)cand_cap,
        cand_count, row_queue);
    SG_LAUNCH_CHECK();
    return SG_OK;
}

extern "C" {

int sg_cossim_candidates(const int64_t *a_indptr, const int32_t *a_len, const int32_t *a_indices,
                         const float *a_val32, int64_t row_begin, int64_t row_end, const int32_t *perm_a,
                         int64_t n_right, int64_t n_cols, const void *bucket_dir, const void *bucket_maxw,
                         const void *postings, const int32_t *perm_b, int tile_w, int acc_dtype, float a_scale,
                         float cand_threshold,
                         const float *cand_threshold_row, const float *pruned_norm_row, const float *tile_bound,
                         int64_t tiles_per_group, int32_t *cand_row,
                         int32_t *cand_col, float *cand_partial, int64_t cand_cap, unsigned long long *cand_count,
                         unsigned long long *row_queue, int warps_per_cta, void *stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (row_end <= row_begin || n_right <= 0) return SG_OK;
    if (acc_dtype != SG_ACC_F32 && acc_dtype != SG_ACC_U16)
        return fail(SG_ERR_INVALID, "acc_dtype must be SG_ACC_F32 or SG_ACC_U16");
    if (!tile_bound || !bucket_maxw) return fail(SG_ERR_INVALID, "tile_bound and bucket_maxw are required");
    if (tiles_per_group < 64 || tiles_per_group % 64)
        return fail(SG_ERR_INVALID, "tiles_per_group must be a positive multiple of 64");
    const int acc_bytes = acc_dtype == SG_ACC_U16 ? 2 : 4;
    if (tile_w <= 0 || ((size_t)tile_w * acc_bytes) % 256 || (tile_w & 31))
        return fail(SG_ERR_INVALID, "tile_w must be a multiple of 32 and tile_w * accumulator size a multiple of 256 bytes");
    if (tile_w > 32768) return fail(SG_ERR_INVALID, "tile_w must not exceed 32768 (16-bit bucket lengths)");
    if (!(cand_threshold >= 0.f)) return fail(SG_ERR_INVALID, "cand_threshold must be >= 0");
    int dev = 0, n_sm = 0, smem_optin = 0;
    SG_CUDA_TRY(cudaGetDevice(&dev));
    SG_CUDA_TRY(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
    SG_CUDA_TRY(cudaDeviceGetAttribute(&smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    if ((size_t)warps_per_cta * tile_w * acc_bytes > (size_t)smem_optin)
        return fail(SG_ERR_INVALID, "warps_per_cta*tile_w*%d = %zu exceeds %d bytes of shared memory", acc_bytes,
                    (size_t)warps_per_cta * tile_w * acc_bytes, smem_optin);
#define SG_ARGS                                                                                              \
    a_indptr, a_len, a_indices, a_val32, row_begin, row_end, perm_a, n_right, n_cols, bucket_dir, bucket_maxw, \
        postings, perm_b, tile_w, tiles_per_group, a_scale, cand_threshold, cand_threshold_row, pruned_norm_row,      \
        tile_bound, cand_row, cand_col, cand_partial, cand_cap, cand_count, row_queue, n_sm, st
#define SG_CASE(NW)                                                                                          \
    case NW:                                                                                                 \
        return acc_dtype == SG_ACC_U16 ? launch_candidates<NW, uint16_t>(SG_ARGS)                           \
                                       : launch_candidates<NW, float>(SG_ARGS);
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

int sg_rescore(int64_t n_cand, const int32_t *cand_row, const int32_t *cand_col, const int64_t *a_indptr,
               const int32_t *a_indices, const void *a_val, const int64_t *b_indptr, const int32_t *b_indices,
               const void *b_val, int dtype, double *score_out, double keep_threshold, int32_t *keep_row,
               int32_t *keep_col, unsigned long long *keep_count, int32_t *row_cnt, int64_t row_begin,
               void *stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (n_cand <= 0) return SG_OK;
    if (keep_count && (!keep_row || !keep_col)) return fail(SG_ERR_INVALID, "keep_count needs keep_row and keep_col");
    if (row_cnt && !keep_count) return fail(SG_ERR_INVALID, "row_cnt needs keep_count");
    const unsigned grid = (unsigned)((n_cand + 255) / 256);
    const bool vec = ((uintptr_t)b_indices & 15) == 0;      // merge_dot_vec reads aligned 16-byte index vectors
#define SG_RESCORE(T, VEC)                                                                                        \
    rescore_kernel<T, VEC><<<grid, 256, 0, st>>>(n_cand, cand_row, cand_col, a_indptr, a_indices, (const T *)a_val, \
                                                 b_indptr, b_indices, (const T *)b_val, score_out, keep_threshold,  \
                                                 keep_row, keep_col, keep_count, row_cnt, row_begin)
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

int sg_rescore_refined(int64_t n_cand, const int32_t *cand_row, const int32_t *cand_col, const float *cand_partial,
                       const void *left_group_norms, const void *right_group_norms, const float *row_threshold,
                       const int64_t *a_indptr, const int32_t *a_indices, const void *a_val,
                       const int64_t *b_indptr, const int32_t *b_indices, const void *b_val, int dtype,
                       double *score_out, double keep_threshold, int32_t *keep_row, int32_t *keep_col,
                       unsigned long long *keep_count, unsigned long long *refined_count, int32_t *row_cnt,
                       int64_t row_begin, void *stream_) {
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
    rescore_refined_kernel<T, VEC><<<grid, 256, 0, st>>>(                                                           \
        n_cand, cand_row, cand_col, cand_partial, (const uint4 *)left_group_norms, (const uint4 *)right_group_norms, \
        row_threshold, a_indptr, a_indices, (const T *)a_val, b_indptr, b_indices, (const T *)b_val, score_out,      \
        keep_threshold, keep_row, keep_col, keep_count, refined_count, row_cnt, row_begin)
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
