// K2, tile-centric formulation for sm_90a: right-matrix row segments staged through TMA into shared memory.
//
// Replaces the block loop of StringGrouper._build_matches
// (string_grouper/string_grouper.py:734-750: `Bs` = row blocks of the right matrix, one
// sp_matmul_topn per (left block, right block) pair, :737-743) for L2-normalised non-negative matrices
// (the K1 output).  Where the reference slices ~4000-row right blocks so that the accumulators of
// sparse_dot_topn stay cache-resident (:387-389), this kernel takes 256-row right blocks ("column tiles"
// of the product) whose whole inverted index fits in shared memory:
//
//   tiles_build      right matrix -> per tile one contiguous blob: the tile's postings sorted by (feature,
//                    column) as 4-byte {fixed-point weight, column}, a bitmap over the features present, its
//                    rank table and the bucket offsets; plus the fp16 block maxima the filter streams
//   pack_left        pruned left rows (sg_prune_rows) -> {feature, fixed-point weight} pairs and one 16-byte
//                    record {start, kept features, threshold, pruned norm} per row in processing order
//   tile_filter      block-max test of every (left row, tile) pair: no column of tile t can collect more than
//                    ub = sum_f |a_f| max|w_(f,t)|; pairs that cannot reach their candidate threshold are
//                    dropped.  Output: one bit per pair, transposed ([tile word][left rank]) so that a tile
//                    reads the ranks that survive for it with coalesced loads
//   tile_candidates  one CTA per (tile, segment of left ranks): the tile's blob is copied into shared memory
//                    by cp.async.bulk (TMA, completion on an mbarrier); every warp then takes surviving left
//                    rows, finds the buckets of the row's kept features through the bitmap (two shared-memory
//                    loads), walks their concatenation 32 postings per step and adds integer products
//                    a_q * w_q (2^-30 units) into a 256-column accumulator tile with native shared-memory
//                    atomics.  All weights are non-negative, so a column's partial score only grows: the step
//                    in which it crosses the candidate threshold reports the pair — no sweep of the tile.
//
// Every candidate is re-scored exactly (sg_rescore), so the result is identical to the plain traversal.
#include <cub/cub.cuh>
#include <cuda_fp16.h>

#include "sg_common.cuh"

namespace sg {

struct __align__(16) TileDesc {
    long long blob_off;     // byte offset of the tile's blob (16-byte aligned)
    int n_post;             // postings of the tile
    int n_dist;             // distinct features of the tile = buckets
};

constexpr int TL_LONG = 64;          // buckets from this length on are streamed by the whole warp
constexpr int TL_W = 256;            // columns per tile (accumulator: 256 x u32 = 1 KB per warp)
constexpr int TL_CBUF = 96;          // candidate buffer entries per warp
constexpr float TL_FIX = 32768.f;    // weights in 2^-15 units, products in 2^-30 units
constexpr int TL_WARP_BYTES = TL_W * 4 + 64 * 4 + 32 * 8 + TL_CBUF * 8;
constexpr int TL_HEAD_BYTES = 128;   // mbarrier, item broadcast, survivor count

__host__ __device__ __forceinline__ int a16(int x) { return (x + 15) & ~15; }
// bitmap words per tile: one bit per feature, rounded up to 16 bytes
__host__ __device__ __forceinline__ int bitmap_words(int64_t n_cols) { return (int)(((n_cols + 31) / 32 + 3) & ~(int64_t)3); }
__host__ __device__ __forceinline__ int blob_bytes(int n_post, int n_dist, int bw) {
    return a16(4 * n_post) + 4 * bw + a16(2 * bw) + a16(2 * (n_dist + 1));
}

// ---------------------------------------------------------------------------
// mbarrier / bulk-copy (TMA) primitives
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, unsigned bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, unsigned parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "SG_WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra SG_DONE_%=;\n"
        "bra SG_WAIT_%=;\n"
        "SG_DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}

// ---------------------------------------------------------------------------
// build: right matrix -> tile blobs
// ---------------------------------------------------------------------------
// key = ((tile * V + feature) << 16) | column inside the tile; value = weight bits
__global__ void tiles_keys_kernel(int64_t n_rows, const int64_t *__restrict__ indptr,
                                  const int32_t *__restrict__ indices, const float *__restrict__ val,
                                  const int32_t *__restrict__ rank, int W, int64_t V, int64_t base, float w_scale,
                                  uint64_t *__restrict__ keys, uint32_t *__restrict__ vals) {
    const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= n_rows) return;
    const int64_t pos = rank ? rank[row] : row;
    const int64_t t = pos / W;
    const uint64_t local = (uint64_t)(pos - t * W);
    const int64_t p1 = indptr[row + 1];
    for (int64_t p = indptr[row] + lane_id(); p < p1; p += 32) {
        keys[p - base] = ((uint64_t)(t * V + indices[p]) << 16) | local;
        vals[p - base] = __float_as_uint(val[p] * w_scale);
    }
}

__global__ void tiles_ptr_kernel(int64_t T, int64_t V, int64_t nnz, const uint64_t *__restrict__ keys,
                                 int32_t *__restrict__ tile_ptr) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t > T) return;
    const uint64_t k = ((uint64_t)(t * V)) << 16;
    int64_t lo = 0, hi = nnz;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (keys[mid] < k) lo = mid + 1; else hi = mid;
    }
    tile_ptr[t] = (int32_t)lo;
}

// one CTA per tile: distinct features -> blob size; also the largest blob / posting count over all tiles
__global__ void tiles_count_kernel(int64_t T, const int32_t *__restrict__ tile_ptr, const uint64_t *__restrict__ keys,
                                   int bw, int32_t *__restrict__ n_dist, int64_t *__restrict__ bytes,
                                   int32_t *__restrict__ maxima) {
    const int64_t t = blockIdx.x;
    const int b = tile_ptr[t], e = tile_ptr[t + 1];
    int c = 0;
    for (int p = b + threadIdx.x; p < e; p += blockDim.x)
        c += (p == b || (keys[p] >> 16) != (keys[p - 1] >> 16)) ? 1 : 0;
    typedef cub::BlockReduce<int, 256> Red;
    __shared__ typename Red::TempStorage tmp;
    const int total = Red(tmp).Sum(c);
    if (threadIdx.x == 0) {
        n_dist[t] = total;
        const int bb = blob_bytes(e - b, total, bw);
        bytes[t] = bb;
        atomicMax(maxima, bb);
        atomicMax(maxima + 1, e - b);
    }
}

// one CTA (256 threads) per tile
__global__ void __launch_bounds__(256)
tiles_fill_kernel(int64_t T, int64_t V, int64_t Tp, const int32_t *__restrict__ tile_ptr,
                  const uint64_t *__restrict__ keys, const uint32_t *__restrict__ vals,
                  const int32_t *__restrict__ n_dist, const int64_t *__restrict__ blob_off, int bw,
                  unsigned char *__restrict__ blob, TileDesc *__restrict__ desc,
                  unsigned short *__restrict__ maxw_rows) {
    extern __shared__ uint32_t s_bitmap[];          // bw words
    typedef cub::BlockScan<int, 256> Scan;
    __shared__ typename Scan::TempStorage tmp;
    __shared__ int s_running;
    const int64_t t = blockIdx.x;
    const int b = tile_ptr[t], e = tile_ptr[t + 1];
    const int n_post = e - b, nd = n_dist[t];
    const long long boff = blob_off[t];
    uint32_t *post = reinterpret_cast<uint32_t *>(blob + boff);
    uint32_t *bm_out = reinterpret_cast<uint32_t *>(blob + boff + a16(4 * n_post));
    unsigned short *prefix = reinterpret_cast<unsigned short *>(blob + boff + a16(4 * n_post) + 4 * bw);
    unsigned short *off = reinterpret_cast<unsigned short *>(blob + boff + a16(4 * n_post) + 4 * bw + a16(2 * bw));
    for (int i = threadIdx.x; i < bw; i += 256) s_bitmap[i] = 0u;
    if (threadIdx.x == 0) {
        s_running = 0;
        desc[t].blob_off = boff;
        desc[t].n_post = n_post;
        desc[t].n_dist = nd;
    }
    __syncthreads();
    const uint64_t fbase = (uint64_t)(t * V);
    for (int base = 0; base < n_post; base += 256) {
        const int p = b + base + threadIdx.x;
        int head = 0;
        uint64_t kf = 0;
        if (p < e) {
            const uint64_t key = keys[p];
            kf = key >> 16;
            head = (p == b || (keys[p - 1] >> 16) != kf) ? 1 : 0;
            float w = __uint_as_float(vals[p]);
            w = w < 0.f ? 0.f : w;
            unsigned wq = (unsigned)__float2int_rn(w * TL_FIX);
            wq = wq > 65535u ? 65535u : wq;
            post[p - b] = (wq << 16) | ((unsigned)(key & 0xffffu) << 2);
        }
        int excl = 0;
        Scan(tmp).ExclusiveSum(head, excl);
        const int running = s_running;
        if (head) {
            const unsigned f = (unsigned)(kf - fbase);
            atomicOr(&s_bitmap[f >> 5], 1u << (f & 31));
            off[running + excl] = (unsigned short)(p - b);
            // largest fixed-point weight of the bucket (the run of equal features starting here)
            unsigned mq = 0;
            for (int q = p; q < e && (keys[q] >> 16) == kf; ++q) {
                float w = __uint_as_float(vals[q]);
                w = w < 0.f ? 0.f : w;
                unsigned wq = (unsigned)__float2int_rn(w * TL_FIX);
                mq = wq > mq ? wq : mq;
            }
            mq = mq > 65535u ? 65535u : mq;
            // what the kernel accumulates is w_q / 32768: the fp16 bound must not fall short of it
            maxw_rows[(int64_t)f * Tp + t] = __half_as_ushort(__float2half_ru((float)mq * (1.f / TL_FIX)));
        }
        __syncthreads();
        if (threadIdx.x == 255) s_running = running + excl + head;
        __syncthreads();
    }
    if (threadIdx.x == 0) off[nd] = (unsigned short)n_post;
    // zero padding of the posting section (never walked; keeps the blob deterministic)
    for (int i = n_post + threadIdx.x; i < (a16(4 * n_post) >> 2); i += 256) post[i] = 0u;
    __syncthreads();
    // rank table: prefix[w] = set bits before word w
    if (threadIdx.x == 0) s_running = 0;
    __syncthreads();
    for (int base = 0; base < bw; base += 256) {
        const int i = base + threadIdx.x;
        const uint32_t word = i < bw ? s_bitmap[i] : 0u;
        int excl = 0;
        Scan(tmp).ExclusiveSum(__popc(word), excl);
        const int running = s_running;
        if (i < bw) {
            bm_out[i] = word;
            prefix[i] = (unsigned short)(running + excl);
        }
        __syncthreads();
        if (threadIdx.x == 255) s_running = running + excl + __popc(word);
        __syncthreads();
    }
}

// ---------------------------------------------------------------------------
// left operand: pruned rows -> packed {feature, fixed-point weight}, 16-byte row records in processing order
// ---------------------------------------------------------------------------
__global__ void pack_left_kernel(int64_t n_ranks, const int32_t *__restrict__ perm, int64_t row_begin,
                                 const int64_t *__restrict__ indptr, const int32_t *__restrict__ p_len,
                                 const int32_t *__restrict__ p_idx, const float *__restrict__ p_val,
                                 const float *__restrict__ p_thr, const float *__restrict__ p_xp, float a_scale,
                                 int2 *__restrict__ lpack, int4 *__restrict__ rowinfo) {
    const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (r >= n_ranks) return;
    const int64_t row = perm ? perm[r] : row_begin + r;
    const int64_t p0 = indptr[row];
    const int nf = p_len ? p_len[row] : (int)(indptr[row + 1] - p0);
    for (int k = lane_id(); k < nf; k += 32) {
        float a = p_val[p0 + k] * a_scale;
        a = a < 0.f ? 0.f : a;
        lpack[p0 + k] = make_int2(p_idx[p0 + k], __float2int_rn(a * TL_FIX));
    }
    if (lane_id() == 0)
        rowinfo[r] = make_int4((int)p0, nf, __float_as_int(p_thr[row]), __float_as_int(p_xp ? p_xp[row] : 0.f));
}

// ---------------------------------------------------------------------------
// block-max filter: one bit per (left rank, tile), transposed
// ---------------------------------------------------------------------------
// Word layout: the 64 tiles of batch b = [64b, 64b+64) occupy words 2b (even tiles) and 2b+1 (odd tiles), bit
// (tile & 63) >> 1 — the bounds of two neighbouring tiles are evaluated in one packed fp16 lane.
constexpr int FL_WARPS = 8;
constexpr int FL_RANKS = 32;      // ranks per CTA (4 per warp)
constexpr int FL_WORDS = 128;     // mask words per pass through shared memory (4096 tiles)

__global__ void __launch_bounds__(FL_WARPS * 32)
tile_filter_kernel(int64_t n_ranks, const int4 *__restrict__ rowinfo, const int2 *__restrict__ lpack,
                   const uint32_t *__restrict__ maxw_h, int Tp, int64_t T, const float *__restrict__ tile_bound,
                   uint32_t *__restrict__ mask, int64_t mask_stride) {
    __shared__ uint32_t buf[FL_WORDS][FL_RANKS + 1];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t rank0 = (int64_t)blockIdx.x * FL_RANKS;
    const int n_words = Tp >> 5;
    const int half_tp = Tp >> 1;
    for (int w0 = 0; w0 < n_words; w0 += FL_WORDS) {
        const int w1 = w0 + FL_WORDS < n_words ? w0 + FL_WORDS : n_words;
        for (int ri = 0; ri < FL_RANKS / FL_WARPS; ++ri) {
            const int rr = warp * (FL_RANKS / FL_WARPS) + ri;
            const int64_t r = rank0 + rr;
            int nf = 0;
            float thr_r = 0.f, xp = 0.f;
            int f0 = 0;
            __half2 a2 = __float2half2_rn(0.f);
            if (r < n_ranks) {
                const int4 info = rowinfo[r];
                nf = info.y;
                thr_r = __int_as_float(info.z);
                xp = __int_as_float(info.w);
                if (lane < nf) {
                    const int2 fa = lpack[(int64_t)info.x + lane];
                    f0 = fa.x;
                    // rounded up: the bound must not fall short
                    a2 = __half2half2(__float2half_ru((float)fa.y * (1.f / TL_FIX)));
                }
            }
            const int nk = nf < 32 ? nf : 32;
            const float slack = 5e-4f * (float)nk + 1e-4f;    // fp16 arithmetic of the bound
            for (int wd = w0; wd < w1; wd += 2) {
                const int tb = wd << 5;                       // first tile of the batch
                unsigned m_even = 0, m_odd = 0;
                const int t0 = tb + 2 * lane;
                if (nf > 32) {                                // more kept features than lanes: every tile is walked
                    m_even = __ballot_sync(FULL, t0 < T);
                    m_odd = __ballot_sync(FULL, t0 + 1 < T);
                } else if (nf > 0) {
                    __half2 ub2 = __float2half2_rn(0.f);
                    const uint32_t *mrow = maxw_h + (tb >> 1) + lane;
                    for (int k = 0; k < nk; ++k) {
                        const int fk = __shfl_sync(FULL, f0, k);
                        const __half2 ak2 = __shfl_sync(FULL, a2, k);
                        const uint32_t m = mrow[(int64_t)fk * half_tp];
                        ub2 = __hfma2(ak2, *reinterpret_cast<const __half2 *>(&m), ub2);
                    }
                    const float2 ub = __half22float2(ub2);
                    const float2 tb2 = reinterpret_cast<const float2 *>(tile_bound)[(tb >> 1) + lane];
                    const float thr0 = xp > 0.f ? fmaxf(fmaf(-xp, tb2.x, thr_r), 0.f) : thr_r;
                    const float thr1 = xp > 0.f ? fmaxf(fmaf(-xp, tb2.y, thr_r), 0.f) : thr_r;
                    m_even = __ballot_sync(FULL, t0 < T && ub.x + slack > thr0);
                    m_odd = __ballot_sync(FULL, t0 + 1 < T && ub.y + slack > thr1);
                }
                if (lane == 0) {
                    buf[wd - w0][rr] = m_even;
                    buf[wd - w0 + 1][rr] = m_odd;
                }
            }
        }
        __syncthreads();
        for (int wd = w0 + warp; wd < w1; wd += FL_WARPS)
            if (rank0 + lane < mask_stride) mask[(int64_t)wd * mask_stride + rank0 + lane] = buf[wd - w0][lane];
        __syncthreads();
    }
}

// ---------------------------------------------------------------------------
// candidates
// ---------------------------------------------------------------------------
constexpr int tl_min_ctas(int nw) { return nw == 16 ? 1 : 3; }

struct WarpCtx {
    uint32_t *acc;          // TL_W partial scores, 2^-30 units
    uint32_t *flags;        // bucket-start bits of the concatenated list
    int2 *dk;               // per non-empty short bucket: {posting index - start in the list, left weight}
    int2 *cbuf;             // buffered candidates {left rank, column position}
    int ccount;
};

__device__ __forceinline__ void flush_candidates(WarpCtx &cx, int lane, const int32_t *__restrict__ perm_a,
                                                 int64_t row_begin, const int32_t *__restrict__ perm_b,
                                                 int32_t *__restrict__ cand_row, int32_t *__restrict__ cand_col,
                                                 unsigned long long cap, unsigned long long *cand_count) {
    __syncwarp();
    if (cx.ccount > 0) {
        unsigned long long base = 0;
        if (lane == 0) base = atomicAdd(cand_count, (unsigned long long)cx.ccount);
        base = __shfl_sync(FULL, base, 0);
        for (int i = lane; i < cx.ccount; i += 32) {
            const int2 c = cx.cbuf[i];
            if (base + i < cap) {
                cand_row[base + i] = (int32_t)(perm_a ? perm_a[c.x] : row_begin + c.x);
                cand_col[base + i] = perm_b ? perm_b[c.y] : c.y;
            }
        }
        cx.ccount = 0;
    }
    __syncwarp();
}

// report the columns whose partial score crossed the threshold in this step
#define TL_EMIT(crossed_, colbyte_)                                                                       \
    do {                                                                                                  \
        const unsigned em_ = __ballot_sync(FULL, (crossed_));                                             \
        if (em_) {                                                                                        \
            if ((crossed_)) cx.cbuf[cx.ccount + __popc(em_ & lt_mask)] = make_int2(rank_id, col0 + ((int)(colbyte_) >> 2)); \
            cx.ccount += __popc(em_);                                                                     \
            if (cx.ccount > TL_CBUF - 32)                                                                 \
                flush_candidates(cx, lane, perm_a, row_begin, perm_b, cand_row, cand_col, cap, cand_count);   \
        }                                                                                                 \
    } while (0)

// One (left row, tile) pair: buckets of the row's kept features through the bitmap directory, long buckets streamed
// by the warp, all others walked as one concatenated list; columns whose partial score crosses the threshold are
// buffered as candidates.
#define TL_PAIR(rank_id_, info_, fa_first_)                                                                         \
    do {                                                                                                            \
        const int rank_id = (rank_id_);                                                                             \
        const int cur_p0 = (info_).x, cur_nf = (info_).y;                                                           \
        const float thr_r = __int_as_float((info_).z);                                                              \
        const float xp = __int_as_float((info_).w);                                                                 \
        const float thr_f = xp > 0.f ? fmaxf(fmaf(-xp, tbound, thr_r), 0.f) : thr_r;                                \
        const unsigned thr_c = (unsigned)__float2uint_rd(fminf(thr_f, 3.9f) * (TL_FIX * TL_FIX));                   \
        bool touched = false;                                                                                       \
        ++n_pairs;                                                                                                  \
        for (int fb = 0; fb < cur_nf; fb += 32) {                                                                   \
            int2 e_fa = (fa_first_);                                                                                \
            if (fb > 0) {                                                                                           \
                e_fa = make_int2(0, 0);                                                                             \
                if (fb + lane < cur_nf) e_fa = lpack[(int64_t)cur_p0 + fb + lane];                                  \
            }                                                                                                       \
            int len = 0, o0 = 0;                                                                                    \
            if (fb + lane < cur_nf) {                                                                               \
                const unsigned f = (unsigned)e_fa.x;                                                                \
                const uint32_t bmw = bitmap[f >> 5];                                                                \
                if ((bmw >> (f & 31)) & 1u) {                                                                       \
                    const int jb = (int)prefix[f >> 5] + __popc(bmw & ((1u << (f & 31)) - 1u));                     \
                    o0 = off[jb];                                                                                   \
                    len = (int)off[jb + 1] - o0;                                                                    \
                }                                                                                                   \
            }                                                                                                       \
            const unsigned aq = (unsigned)e_fa.y;                                                                   \
            unsigned lm = __ballot_sync(FULL, len >= TL_LONG);                                                      \
            while (lm) {                                                                                            \
                const int s_ = __ffs(lm) - 1;                                                                       \
                lm &= lm - 1;                                                                                       \
                const int b0 = __shfl_sync(FULL, o0, s_);                                                           \
                const int b1 = b0 + __shfl_sync(FULL, len, s_);                                                     \
                const unsigned ak = __shfl_sync(FULL, aq, s_);                                                      \
                n_walked += (unsigned)(b1 - b0);                                                                    \
                for (int p = b0; p < b1; p += 32) {                                                                 \
                    bool crossed = false;                                                                           \
                    unsigned cb = 0;                                                                                \
                    if (p + lane < b1) {                                                                            \
                        const uint32_t e = post[p + lane];                                                          \
                        const unsigned x = (e >> 16) * ak;                                                          \
                        cb = e & 0xffffu;                                                                           \
                        const unsigned old = atomicAdd(                                                             \
                            reinterpret_cast<unsigned *>(reinterpret_cast<unsigned char *>(cx.acc) + cb), x);       \
                        crossed = old <= thr_c && old + x > thr_c;                                                  \
                    }                                                                                               \
                    TL_EMIT(crossed, cb);                                                                           \
                }                                                                                                   \
                touched = true;                                                                                     \
            }                                                                                                       \
            const int ln = len >= TL_LONG ? 0 : len;                                                                \
            int incl = ln;                                                                                          \
            _Pragma("unroll") for (int o = 1; o < 32; o <<= 1) {                                                    \
                const int up = __shfl_up_sync(FULL, incl, o);                                                       \
                if (lane >= o) incl += up;                                                                          \
            }                                                                                                       \
            const int total = __shfl_sync(FULL, incl, 31);                                                          \
            if (total > 0) {                                                                                        \
                touched = true;                                                                                     \
                n_walked += (unsigned)total;                                                                        \
                const unsigned nz = __ballot_sync(FULL, ln > 0);                                                    \
                if (ln > 0) {                                                                                       \
                    const int st = incl - ln;                                                                       \
                    cx.dk[__popc(nz & lt_mask)] = make_int2(o0 - st, (int)aq);                                      \
                    atomicOr(&cx.flags[st >> 5], 1u << (st & 31));                                                  \
                }                                                                                                   \
                __syncwarp();                                                                                       \
                int kbase = -1;                                                                                     \
                for (int s0 = 0; s0 < total; s0 += 32) {                                                            \
                    const uint32_t fw = cx.flags[s0 >> 5];                                                          \
                    const int k = kbase + __popc(fw & le_mask);                                                     \
                    kbase += __popc(fw);                                                                            \
                    __syncwarp();                                                                                   \
                    if (lane == 0) cx.flags[s0 >> 5] = 0u;                                                          \
                    bool crossed = false;                                                                           \
                    unsigned cb = 0;                                                                                \
                    if (s0 + lane < total) {                                                                        \
                        const int2 dd = cx.dk[k];                                                                   \
                        const uint32_t e = post[dd.x + s0 + lane];                                                  \
                        const unsigned x = (e >> 16) * (unsigned)dd.y;                                              \
                        cb = e & 0xffffu;                                                                           \
                        const unsigned old = atomicAdd(                                                             \
                            reinterpret_cast<unsigned *>(reinterpret_cast<unsigned char *>(cx.acc) + cb), x);       \
                        crossed = old <= thr_c && old + x > thr_c;                                                  \
                    }                                                                                               \
                    TL_EMIT(crossed, cb);                                                                           \
                }                                                                                                   \
                __syncwarp();                                                                                       \
            }                                                                                                       \
        }                                                                                                           \
        if (touched) {                                                                                              \
            __syncwarp();                                                                                           \
            _Pragma("unroll") for (int c = 0; c < TL_W * 4 / 16 / 32; ++c)                                          \
                reinterpret_cast<uint4 *>(cx.acc)[c * 32 + lane] = zero4;                                           \
            __syncwarp();                                                                                           \
        }                                                                                                           \
    } while (0)

__host__ __device__ constexpr int tl_list(int nw) { return nw * 256; }     // survivor ranks per scan round (every warp scans 256 ranks)

template <int NW>
__global__ void __launch_bounds__(NW * 32, tl_min_ctas(NW))
tile_candidates_kernel(const int32_t *__restrict__ perm_a, int64_t n_ranks, int64_t row_begin,
                       const int4 *__restrict__ rowinfo, const int2 *__restrict__ lpack,
                       const uint32_t *__restrict__ mask, int64_t mask_stride, const TileDesc *__restrict__ tdesc,
                       const unsigned char *__restrict__ blob, int64_t T, int bw,
                       const float *__restrict__ tile_bound, const int32_t *__restrict__ perm_b,
                       int64_t seg_ranks, int64_t n_seg, int32_t *__restrict__ cand_row,
                       int32_t *__restrict__ cand_col, unsigned long long cap,
                       unsigned long long *__restrict__ cand_count, unsigned long long *__restrict__ queue,
                       unsigned long long *__restrict__ walk_stats, int stage_bytes) {
    extern __shared__ __align__(128) unsigned char smem[];
    uint64_t *mbar = reinterpret_cast<uint64_t *>(smem);
    volatile long long *s_item = reinterpret_cast<volatile long long *>(smem + 16);
    int *s_count = reinterpret_cast<int *>(smem + 32);
    uint32_t *s_list = reinterpret_cast<uint32_t *>(smem + TL_HEAD_BYTES);
    unsigned char *stage = smem + TL_HEAD_BYTES + tl_list(NW) * 4;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned lt_mask = (1u << lane) - 1u, le_mask = lt_mask | (1u << lane);
    unsigned char *wa = stage + stage_bytes + (size_t)warp * TL_WARP_BYTES;
    WarpCtx cx;
    cx.acc = reinterpret_cast<uint32_t *>(wa);
    cx.flags = reinterpret_cast<uint32_t *>(wa + TL_W * 4);
    cx.dk = reinterpret_cast<int2 *>(wa + TL_W * 4 + 64 * 4);
    cx.cbuf = reinterpret_cast<int2 *>(wa + TL_W * 4 + 64 * 4 + 32 * 8);
    cx.ccount = 0;
    const uint4 zero4 = make_uint4(0u, 0u, 0u, 0u);
    for (int c = lane; c < (TL_W * 4 + 64 * 4) / 16; c += 32) reinterpret_cast<uint4 *>(wa)[c] = zero4;
    if (threadIdx.x == 0) {
        mbar_init(mbar, 1);
        *s_count = 0;
    }
    __syncthreads();

    const unsigned long long n_items = (unsigned long long)T * (unsigned long long)n_seg;
    unsigned parity = 0;
    unsigned long long n_pairs = 0, n_walked = 0;       // (row, tile) pairs taken / postings added by this warp
    for (;;) {
        // ---- next (tile, rank segment); its blob goes into shared memory by bulk copies (TMA)
        if (threadIdx.x == 0) {
            const unsigned long long it = atomicAdd(queue, 1ull);
            *s_item = (long long)it;
            if (it < n_items) {
                const TileDesc d = tdesc[it / (unsigned long long)n_seg];
                const unsigned bytes = (unsigned)blob_bytes(d.n_post, d.n_dist, bw);
                mbar_expect_tx(mbar, bytes);
                for (unsigned o = 0; o < bytes; o += 32768u) {      // pieces of at most 32 KB
                    const unsigned n = bytes - o < 32768u ? bytes - o : 32768u;
                    bulk_g2s(stage + o, blob + d.blob_off + o, n, mbar);
                }
            }
        }
        __syncthreads();
        const unsigned long long it = (unsigned long long)*s_item;
        if (it >= n_items) break;
        const int t = (int)(it / (unsigned long long)n_seg);
        const int64_t seg = (int64_t)(it % (unsigned long long)n_seg);
        const TileDesc d = tdesc[t];
        const uint32_t *post = reinterpret_cast<const uint32_t *>(stage);
        const uint32_t *bitmap = reinterpret_cast<const uint32_t *>(stage + a16(4 * d.n_post));
        const unsigned short *prefix = reinterpret_cast<const unsigned short *>(stage + a16(4 * d.n_post) + 4 * bw);
        const unsigned short *off =
            reinterpret_cast<const unsigned short *>(stage + a16(4 * d.n_post) + 4 * bw + a16(2 * bw));
        const float tbound = tile_bound[t];
        const int col0 = t * TL_W;
        const int64_t rank_lo = seg * seg_ranks;
        const int64_t rank_hi = rank_lo + seg_ranks < n_ranks ? rank_lo + seg_ranks : n_ranks;
        const uint32_t *mrow = mask + (int64_t)(((t >> 6) << 1) | (t & 1)) * mask_stride;
        const int bit = (t & 63) >> 1;
        bool staged = false;

        for (int64_t base = rank_lo; base < rank_hi; base += (int64_t)NW * 256) {
            // ---- scan round: every warp tests 256 ranks (eight coalesced mask words in flight) and appends the
            // survivors to the CTA's list.  Survivors cluster in rank order (similar rows are neighbours), so the list
            // is dealt out to the warps round-robin afterwards.
            const int64_t gbase = base + ((int64_t)warp << 8);
            uint32_t wsv[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int64_t r = gbase + j * 32 + lane;
                wsv[j] = r < rank_hi ? mrow[r] : 0u;
            }
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const unsigned sv = __ballot_sync(FULL, (wsv[j] >> bit) & 1u);
                if (sv) {
                    int pos = 0;
                    if (lane == 0) pos = atomicAdd(s_count, __popc(sv));
                    pos = __shfl_sync(FULL, pos, 0);
                    if ((sv >> lane) & 1u) s_list[pos + __popc(sv & lt_mask)] = (uint32_t)(gbase + j * 32 + lane);
                }
            }
            __syncthreads();
            const int count = *reinterpret_cast<volatile int *>(s_count);
            if (count > 0) {
                if (!staged) {
                    mbar_wait(mbar, parity);
                    staged = true;
                }
                // ---- this warp's pairs: list entries warp, warp + NW, ...; row record two ahead, features one ahead
                int i = warp;
                int r_c = 0, r_n = 0;
                int4 info_c = make_int4(0, 0, 0, 0), info_n = info_c;
                int2 fa_c = make_int2(0, 0);
                if (i < count) {
                    r_c = (int)s_list[i];
                    info_c = rowinfo[r_c];
                }
                if (i + NW < count) {
                    r_n = (int)s_list[i + NW];
                    info_n = rowinfo[r_n];
                }
                if (i < count && lane < info_c.y) fa_c = lpack[(int64_t)info_c.x + lane];
                while (i < count) {
                    int2 fa_n = make_int2(0, 0);
                    if (i + NW < count && lane < info_n.y) fa_n = lpack[(int64_t)info_n.x + lane];
                    int r_nn = 0;
                    int4 info_nn = make_int4(0, 0, 0, 0);
                    if (i + 2 * NW < count) {
                        r_nn = (int)s_list[i + 2 * NW];
                        info_nn = rowinfo[r_nn];
                    }
                    TL_PAIR(r_c, info_c, fa_c);
                    r_c = r_n; info_c = info_n; fa_c = fa_n;
                    r_n = r_nn; info_n = info_nn;
                    i += NW;
                }
            }
            __syncthreads();
            if (threadIdx.x == 0) *s_count = 0;
            // (the next round's appends come after the next __syncthreads-separated scan loads; the reset is ordered
            // before them by the barrier below)
            __syncthreads();
        }
        if (!staged) mbar_wait(mbar, parity);     // nothing survived: still consume the phase before the stage is reused
        parity ^= 1u;
        __syncthreads();      // every warp is done with the staged tile before the next one is copied over it
    }
    flush_candidates(cx, lane, perm_a, row_begin, perm_b, cand_row, cand_col, cap, cand_count);
    if (walk_stats && lane == 0) {
        atomicAdd(walk_stats, n_pairs);
        atomicAdd(walk_stats + 1, n_walked);
    }
}

static int bits_for64(uint64_t v) {
    int b = 0;
    while (v) { ++b; v >>= 1; }
    return b < 1 ? 1 : b;
}

}  // namespace sg

using namespace sg;

extern "C" {

int sg_tiles_tile_w(void) { return TL_W; }

int64_t sg_tiles_max_cols(void) { return (int64_t)1 << 18; }     // bitmap + rank table: 6 bytes per 32 features

/* upper bound of the blob array in bytes, known without a device read-back */
int64_t sg_tiles_blob_bound(int64_t nnz, int64_t n_rows, int64_t n_cols) {
    const int64_t T = sg_num_tiles(n_rows, TL_W);
    const int bw = bitmap_words(n_cols);
    return 6 * nnz + T * (int64_t)(4 * bw + a16(2 * bw) + 64) + 256;
}

size_t sg_tiles_workspace_bytes(int64_t nnz, int64_t n_rows, int64_t n_cols) {
    const int64_t T = sg_num_tiles(n_rows, TL_W);
    const int64_t n = nnz < 1 ? 1 : nnz;
    size_t b1 = 0, b2 = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, b1, (uint64_t *)nullptr, (uint64_t *)nullptr, (uint32_t *)nullptr,
                                    (uint32_t *)nullptr, n);
    cub::DeviceScan::ExclusiveSum(nullptr, b2, (int64_t *)nullptr, (int64_t *)nullptr, T + 1);
    return 2 * align_up((size_t)n * 8, 256) + 2 * align_up((size_t)n * 4, 256) + 4 * align_up((size_t)(T + 2) * 8, 256) +
           align_up(b1 > b2 ? b1 : b2, 256) + 4096;
}

/*
 * Right matrix -> tile blobs, descriptors, block maxima.  `maxima` [dev, 2 x int32] receives the largest blob in
 * bytes and the largest posting count of a tile (the caller sizes the shared-memory stage with the former).
 */
int sg_tiles_build(int64_t n_rows, int64_t n_cols, int64_t nnz, const int64_t *indptr, const int32_t *indices,
                   const float *val32, const int32_t *rank, int64_t indptr_base, float w_scale, void *tile_desc,
                   void *blob, int64_t blob_cap, void *bucket_maxw, int32_t *maxima, void *ws, size_t ws_bytes,
                   void *stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (n_cols > sg_tiles_max_cols())
        return fail(SG_ERR_UNSUPPORTED, "%lld features exceed the bitmap directory of the tile kernel", (long long)n_cols);
    if (nnz >= (int64_t)0x7fffffff)
        return fail(SG_ERR_OVERFLOW, "right matrix nnz %lld does not fit int32 postings", (long long)nnz);
    const int64_t T = sg_num_tiles(n_rows, TL_W);
    const int64_t Tp = sg_num_tiles_padded(n_rows, TL_W);
    const int bw = bitmap_words(n_cols);
    if (blob_cap < sg_tiles_blob_bound(nnz, n_rows, n_cols)) return fail(SG_ERR_INVALID, "blob buffer too small");
    Arena ar(ws, ws_bytes);
    const size_t n = (size_t)(nnz < 1 ? 1 : nnz);
    uint64_t *keys = ar.take<uint64_t>(n);
    uint64_t *keys_sorted = ar.take<uint64_t>(n);
    uint32_t *vals = ar.take<uint32_t>(n);
    uint32_t *vals_sorted = ar.take<uint32_t>(n);
    int32_t *tile_ptr = ar.take<int32_t>((size_t)T + 2);
    int32_t *n_dist = ar.take<int32_t>((size_t)T + 2);
    int64_t *bytes = ar.take<int64_t>((size_t)T + 2);
    int64_t *blob_off = ar.take<int64_t>((size_t)T + 2);
    size_t b1 = 0, b2 = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, b1, keys, keys_sorted, vals, vals_sorted, (int64_t)n);
    cub::DeviceScan::ExclusiveSum(nullptr, b2, bytes, blob_off, T + 1);
    size_t cub_bytes = b1 > b2 ? b1 : b2;
    char *tmp = ar.take<char>(cub_bytes);
    if (!ar.ok()) return fail(SG_ERR_INVALID, "tiles workspace too small (%zu < %zu)", ws_bytes, ar.off);
    SG_CUDA_TRY(cudaMemsetAsync(maxima, 0, 2 * sizeof(int32_t), st));
    SG_CUDA_TRY(cudaMemsetAsync(bucket_maxw, 0, (size_t)(n_cols + 1) * Tp * 2, st));
    SG_CUDA_TRY(cudaMemsetAsync(bytes, 0, (size_t)(T + 2) * 8, st));
    if (n_rows > 0 && nnz > 0) {
        tiles_keys_kernel<<<(unsigned)((n_rows + 7) / 8), 256, 0, st>>>(n_rows, indptr, indices, val32, rank, TL_W,
                                                                      n_cols, indptr_base, w_scale, keys, vals);
        SG_LAUNCH_CHECK();
        const int bits = 16 + bits_for64((uint64_t)(T * n_cols));
        SG_CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp, cub_bytes, keys, keys_sorted, vals, vals_sorted, nnz, 0,
                                                    bits > 64 ? 64 : bits, st));
    }
    tiles_ptr_kernel<<<(unsigned)((T + 1 + 255) / 256), 256, 0, st>>>(T, n_cols, nnz, keys_sorted, tile_ptr);
    SG_LAUNCH_CHECK();
    tiles_count_kernel<<<(unsigned)T, 256, 0, st>>>(T, tile_ptr, keys_sorted, bw, n_dist, bytes, maxima);
    SG_LAUNCH_CHECK();
    SG_CUDA_TRY(cub::DeviceScan::ExclusiveSum(tmp, cub_bytes, bytes, blob_off, T + 1, st));
    const size_t fill_smem = (size_t)bw * 4;
    SG_CUDA_TRY(cudaFuncSetAttribute(tiles_fill_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fill_smem));
    tiles_fill_kernel<<<(unsigned)T, 256, fill_smem, st>>>(T, n_cols, Tp, tile_ptr, keys_sorted, vals_sorted, n_dist,
                                                           blob_off, bw, (unsigned char *)blob, (TileDesc *)tile_desc,
                                                           (unsigned short *)bucket_maxw);
    SG_LAUNCH_CHECK();
    return SG_OK;
}

/* pruned left rows -> packed operand of the tile kernels; `perm` = processing order of the n_ranks rows (NULL:
 * rows row_begin, row_begin+1, ...) */
int sg_tiles_pack_left(int64_t n_ranks, const int32_t *perm, int64_t row_begin, const int64_t *indptr,
                       const int32_t *pruned_len, const int32_t *pruned_indices, const float *pruned_val32,
                       const float *threshold_row, const float *pruned_norm_row, float a_scale, void *lpack,
                       void *rowinfo, void *stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (n_ranks <= 0) return SG_OK;
    if (!threshold_row) return fail(SG_ERR_INVALID, "threshold_row is required");
    pack_left_kernel<<<(unsigned)((n_ranks + 7) / 8), 256, 0, st>>>(n_ranks, perm, row_begin, indptr, pruned_len,
                                                                   pruned_indices, pruned_val32, threshold_row,
                                                                   pruned_norm_row, a_scale, (int2 *)lpack,
                                                                   (int4 *)rowinfo);
    SG_LAUNCH_CHECK();
    return SG_OK;
}

int64_t sg_tiles_mask_words(int64_t n_right) { return sg_num_tiles_padded(n_right, TL_W) / 32; }

/* survivors of the block-max test: mask[word * mask_stride + rank], mask_stride = n_ranks rounded up to 32 */
int sg_tiles_filter(int64_t n_ranks, const void *rowinfo, const void *lpack, const void *bucket_maxw,
                    int64_t n_right, const float *tile_bound, uint32_t *mask, int64_t mask_stride, void *stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (n_ranks <= 0 || n_right <= 0) return SG_OK;
    if (mask_stride < n_ranks || (mask_stride & 31)) return fail(SG_ERR_INVALID, "mask_stride must be n_ranks rounded up to 32");
    const int64_t T = sg_num_tiles(n_right, TL_W);
    const int Tp = (int)sg_num_tiles_padded(n_right, TL_W);
    tile_filter_kernel<<<(unsigned)(mask_stride / FL_RANKS), FL_WARPS * 32, 0, st>>>(
        n_ranks, (const int4 *)rowinfo, (const int2 *)lpack, (const uint32_t *)bucket_maxw, Tp, T, tile_bound, mask,
        mask_stride);
    SG_LAUNCH_CHECK();
    return SG_OK;
}

size_t sg_tiles_smem_bytes(int stage_bytes, int warps_per_cta) {
    return (size_t)TL_HEAD_BYTES + (size_t)tl_list(warps_per_cta) * 4 + (size_t)a16(stage_bytes) + (size_t)warps_per_cta * TL_WARP_BYTES;
}

int sg_tiles_candidates(const int32_t *perm_a, int64_t n_ranks, int64_t row_begin, const void *rowinfo,
                        const void *lpack, const uint32_t *mask, int64_t mask_stride, const void *tile_desc,
                        const void *blob, int64_t n_right, int64_t n_cols, const float *tile_bound,
                        const int32_t *perm_b, int stage_bytes, int32_t *cand_row, int32_t *cand_col,
                        int64_t cand_cap, unsigned long long *cand_count, unsigned long long *queue,
                        unsigned long long *walk_stats, int warps_per_cta, void *stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (n_ranks <= 0 || n_right <= 0) return SG_OK;
    if (warps_per_cta != 8 && warps_per_cta != 16) return fail(SG_ERR_INVALID, "warps_per_cta must be 8 or 16");
    int dev = 0, n_sm = 0, smem_optin = 0;
    SG_CUDA_TRY(cudaGetDevice(&dev));
    SG_CUDA_TRY(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
    SG_CUDA_TRY(cudaDeviceGetAttribute(&smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    stage_bytes = a16(stage_bytes);
    const size_t smem = sg_tiles_smem_bytes(stage_bytes, warps_per_cta);
    if (smem > (size_t)smem_optin)
        return fail(SG_ERR_UNSUPPORTED, "a tile of the right matrix needs %zu bytes of shared memory (limit %d)", smem,
                    smem_optin);
    const int64_t T = sg_num_tiles(n_right, TL_W);
    const int bw = bitmap_words(n_cols);
    int per_sm = 1;
    int64_t ctas = 1, n_seg = 1, seg_ranks = 0;
#define SG_TL_LAUNCH(NW)                                                                                             \
    do {                                                                                                             \
        SG_CUDA_TRY(cudaFuncSetAttribute(tile_candidates_kernel<NW>, cudaFuncAttributeMaxDynamicSharedMemorySize,    \
                                         (int)smem));                                                                \
        SG_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, tile_candidates_kernel<NW>, NW * 32, smem)); \
        if (per_sm < 1) per_sm = 1;                                                                                  \
        ctas = (int64_t)n_sm * per_sm;                                                                               \
        /* about 16 work items per resident CTA; a segment holds at least 1024 left ranks */                         \
        n_seg = (16 * ctas + T - 1) / T;                                                                             \
        if (n_seg > (n_ranks + 1023) / 1024) n_seg = (n_ranks + 1023) / 1024;                                        \
        if (n_seg < 1) n_seg = 1;                                                                                    \
        seg_ranks = ((n_ranks + n_seg - 1) / n_seg + 255) / 256 * 256;                                               \
        n_seg = (n_ranks + seg_ranks - 1) / seg_ranks;                                                               \
        if (ctas > T * n_seg) ctas = T * n_seg;                                                                      \
        tile_candidates_kernel<NW><<<(unsigned)ctas, NW * 32, smem, st>>>(                                           \
            perm_a, n_ranks, row_begin, (const int4 *)rowinfo, (const int2 *)lpack, mask, mask_stride,               \
            (const TileDesc *)tile_desc, (const unsigned char *)blob, T, bw, tile_bound, perm_b, seg_ranks, n_seg,   \
            cand_row, cand_col, (unsigned long long)cand_cap, cand_count, queue, walk_stats, stage_bytes);           \
    } while (0)
    if (warps_per_cta == 16) SG_TL_LAUNCH(16); else SG_TL_LAUNCH(8);
#undef SG_TL_LAUNCH
    SG_LAUNCH_CHECK();
    return SG_OK;
}

}  // extern "C"
