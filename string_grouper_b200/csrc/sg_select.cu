// K2 tail — segmented per-row top-n selection, for sm_90a.
//
// The heap of sp_matmul_topn (call sites string_grouper/string_grouper.py:725-743; SURVEY.md Appendix
// A.3): per left row keep the `top_n` largest scores strictly above the threshold, emit them value-descending
// (sort=True).  sg_topn_select (sg_cossim.cu) does this with three global radix sorts over all survivors; here the
// survivors are bucketed by row (the exact re-score has already counted them per row), and every row is ranked on
// its own.  top_n <= 32 (max_n_matches defaults to 20): one warp per row streams the row 32 survivors at a time and
// keeps the best 32 in registers (shuffle bitonic sort + merge), whatever the row length.  Larger top_n: rows of up to
// 32 survivors by the warp network, up to 512 by one warp in shared memory, longer rows by one CTA (in pieces of
// SEL_BIG_CAP with the best top_n carried along, which needs top_n <= SEL_BIG_CAP / 2; otherwise the caller uses
// sg_topn_select).
//
// Order: score descending; among EQUAL scores the larger column wins the cut (what the upstream traversal keeps for
// identical strings) and the survivors of a tie are written in ascending column order — the rule of sg_topn_select.
#include <cub/cub.cuh>

#include "sg_common.cuh"

namespace sg {

constexpr int SEL_BIG_CAP = 4096;        // survivors of one row a CTA ranks in shared memory (12 bytes each)

__device__ __forceinline__ uint64_t score_key_desc(double s) {
    uint64_t b = (uint64_t)__double_as_longlong(s);
    b = (b >> 63) ? ~b : (b | 0x8000000000000000ull);     // order-preserving map of IEEE doubles to unsigned
    return ~b;                                            // ascending key == descending score
}

__global__ void sel_counts_kernel(int64_t n_rows, const int32_t *__restrict__ row_cnt, int top_n,
                                  int64_t *__restrict__ cnt64, int64_t *__restrict__ out_cnt,
                                  int32_t *__restrict__ out_max) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r > n_rows) return;
    const int c = r < n_rows ? row_cnt[r] : 0;
    const int k = c < top_n ? c : top_n;
    cnt64[r] = c;
    out_cnt[r] = k;
    if (k > 0) atomicMax(out_max, k);
}

// survivors -> row buckets (order inside a bucket is arbitrary; the ranking below is total)
__global__ void sel_scatter_kernel(int64_t n, const int32_t *__restrict__ cr, const int32_t *__restrict__ cc,
                                   const double *__restrict__ score, int64_t row_begin,
                                   const int64_t *__restrict__ row_start, int32_t *__restrict__ fill,
                                   int32_t *__restrict__ b_col, double *__restrict__ b_score) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t r = cr[i] - row_begin;
    const int64_t p = row_start[r] + atomicAdd(fill + r, 1);
    b_col[p] = cc[i];
    b_score[p] = score[i];
}

// compare-exchange on (key ascending, column descending)
__device__ __forceinline__ bool sel_before(uint64_t ka, int32_t ca, uint64_t kb, int32_t cb) {
    return ka < kb || (ka == kb && ca > cb);
}

// ascending bitonic sort of one (key, col, score) element per lane over (key, column descending)
__device__ __forceinline__ void warp_sort32(uint64_t &key, int32_t &col, double &sc, int lane) {
#pragma unroll
    for (int k = 2; k <= 32; k <<= 1) {
#pragma unroll
        for (int j = k >> 1; j > 0; j >>= 1) {
            const uint64_t ok = __shfl_xor_sync(FULL, key, j);
            const int32_t oc = __shfl_xor_sync(FULL, col, j);
            const double os = __shfl_xor_sync(FULL, sc, j);
            const bool up = ((lane & k) == 0);              // this pair sorts ascending
            const bool lower = ((lane & j) == 0);           // this lane keeps the smaller element of the pair
            const bool mine_first = sel_before(key, col, ok, oc);
            const bool keep = (lower == up) ? mine_first : !mine_first;
            if (!keep && !(key == ok && col == oc)) { key = ok; col = oc; sc = os; }
        }
    }
}

// One warp per row.  STREAM = true (top_n <= 32): a row of any length is taken 32 survivors at a time; the warp keeps
// the best 32 seen so far, sorted, one per lane — sort the new 32, C_i = min(best_i, new_{31-i}) are the best 32 of the
// union as a bitonic sequence, five merge stages sort them.  STREAM = false: rows with more than 32 survivors are
// appended to `big_rows` for the shared-memory kernels.
template <bool STREAM>
__global__ void __launch_bounds__(256)
sel_rows_small_kernel(int64_t n_rows, int64_t row_begin, const int64_t *__restrict__ row_start,
                      const int32_t *__restrict__ b_col, const double *__restrict__ b_score, int top_n,
                      const int64_t *__restrict__ out_indptr, int32_t *__restrict__ out_row,
                      int32_t *__restrict__ out_col, double *__restrict__ out_score, int32_t *__restrict__ big_rows,
                      int32_t *__restrict__ n_big) {
    const int lane = threadIdx.x & 31;
    const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (r >= n_rows) return;
    const int64_t s0 = row_start[r];
    const int m = (int)(row_start[r + 1] - s0);
    if (m == 0) return;
    if (!STREAM && m > 32) {
        if (lane == 0) big_rows[atomicAdd(n_big, 1)] = (int32_t)r;
        return;
    }
    uint64_t key = ~0ull;
    int32_t col = -1;
    double sc = 0.0;
    if (lane < m) {
        sc = b_score[s0 + lane];
        col = b_col[s0 + lane];
        key = score_key_desc(sc);
    }
    // idle lanes hold the largest key and sink to the end
    warp_sort32(key, col, sc, lane);
    if (STREAM) {
        for (int base = 32; base < m; base += 32) {
            uint64_t nk = ~0ull;
            int32_t nc = -1;
            double ns = 0.0;
            if (base + lane < m) {
                ns = b_score[s0 + base + lane];
                nc = b_col[s0 + base + lane];
                nk = score_key_desc(ns);
            }
            // nothing in this piece beats the current 32nd best: skip it
            const uint64_t worst_k = __shfl_sync(FULL, key, 31);
            const int32_t worst_c = __shfl_sync(FULL, col, 31);
            if (!__any_sync(FULL, sel_before(nk, nc, worst_k, worst_c))) continue;
            warp_sort32(nk, nc, ns, lane);
            const uint64_t rk = __shfl_sync(FULL, nk, 31 - lane);
            const int32_t rc = __shfl_sync(FULL, nc, 31 - lane);
            const double rs = __shfl_sync(FULL, ns, 31 - lane);
            if (sel_before(rk, rc, key, col)) { key = rk; col = rc; sc = rs; }
#pragma unroll
            for (int j = 16; j > 0; j >>= 1) {              // bitonic merge, ascending
                const uint64_t ok = __shfl_xor_sync(FULL, key, j);
                const int32_t oc = __shfl_xor_sync(FULL, col, j);
                const double os = __shfl_xor_sync(FULL, sc, j);
                const bool lower = ((lane & j) == 0);
                const bool mine_first = sel_before(key, col, ok, oc);
                const bool keep = lower ? mine_first : !mine_first;
                if (!keep && !(key == ok && col == oc)) { key = ok; col = oc; sc = os; }
            }
        }
    }
    const int kk = m < top_n ? m : top_n;
    // ties inside the kept set come out in ascending column order: mirror the position inside its run of equal scores
    const uint64_t prev = __shfl_up_sync(FULL, key, 1);
    const unsigned heads = __ballot_sync(FULL, lane < kk && (lane == 0 || key != prev));
    if (lane < kk) {
        const int a = 31 - __clz(heads & ((2u << lane) - 1u));            // start of my run
        const unsigned above = heads & ~((2u << lane) - 1u);
        const int b = above ? __ffs(above) - 1 : kk;                      // end of my run (exclusive)
        const int64_t w = out_indptr[r] + a + (b - 1 - lane);
        out_row[w] = (int32_t)(r + row_begin);
        out_col[w] = col;
        out_score[w] = sc;
    }
}

constexpr int SEL_MID_CAP = 512;         // survivors of one row a single warp ranks in shared memory
constexpr int SEL_MID_WARPS = 8;

// rows with 33 .. SEL_MID_CAP survivors: one warp per row (no block barriers), bitonic network in shared memory
__global__ void __launch_bounds__(SEL_MID_WARPS * 32)
sel_rows_mid_kernel(int64_t row_begin, const int64_t *__restrict__ row_start, const int32_t *__restrict__ b_col,
                    const double *__restrict__ b_score, int top_n, const int64_t *__restrict__ out_indptr,
                    int32_t *__restrict__ out_row, int32_t *__restrict__ out_col, double *__restrict__ out_score,
                    const int32_t *__restrict__ big_rows, const int32_t *__restrict__ n_big) {
    __shared__ uint64_t s_key[SEL_MID_WARPS][SEL_MID_CAP];
    __shared__ int32_t s_col[SEL_MID_WARPS][SEL_MID_CAP];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint64_t *key = s_key[warp];
    int32_t *col = s_col[warp];
    const int nb = *n_big;
    for (int bi = blockIdx.x * SEL_MID_WARPS + warp; bi < nb; bi += gridDim.x * SEL_MID_WARPS) {
        const int64_t r = big_rows[bi];
        const int64_t s0 = row_start[r];
        const int m = (int)(row_start[r + 1] - s0);
        if (m > SEL_MID_CAP) continue;          // sel_rows_big_kernel
        int P = 64;
        while (P < m) P <<= 1;
        for (int i = lane; i < P; i += 32) {
            key[i] = i < m ? score_key_desc(b_score[s0 + i]) : ~0ull;
            col[i] = i < m ? b_col[s0 + i] : -1;
        }
        __syncwarp();
        for (int k = 2; k <= P; k <<= 1) {
            for (int j = k >> 1; j > 0; j >>= 1) {
                for (int i = lane; i < P; i += 32) {
                    const int p = i ^ j;
                    if (p > i) {
                        const bool up = ((i & k) == 0);
                        const bool in_order = !sel_before(key[p], col[p], key[i], col[i]);
                        if (in_order != up) {
                            const uint64_t tk = key[i]; key[i] = key[p]; key[p] = tk;
                            const int32_t tc = col[i]; col[i] = col[p]; col[p] = tc;
                        }
                    }
                }
                __syncwarp();
            }
        }
        const int kk = m < top_n ? m : top_n;
        for (int i = lane; i < kk; i += 32) {
            const uint64_t kx = key[i];
            int a = i, b = i + 1;
            while (a > 0 && key[a - 1] == kx) --a;
            while (b < kk && key[b] == kx) ++b;
            const int64_t w = out_indptr[r] + a + (b - 1 - i);
            uint64_t bits = ~kx;                                    // back to the score
            bits = (bits >> 63) ? (bits & 0x7fffffffffffffffull) : ~bits;
            out_row[w] = (int32_t)(r + row_begin);
            out_col[w] = col[i];
            out_score[w] = __longlong_as_double((long long)bits);
        }
        __syncwarp();
    }
}

// rows with more than SEL_MID_CAP survivors: persistent CTAs; a row longer than SEL_BIG_CAP is taken in pieces, the
// best top_n so far carried along (needs top_n <= SEL_BIG_CAP / 2)
__global__ void __launch_bounds__(256)
sel_rows_big_kernel(int64_t row_begin, const int64_t *__restrict__ row_start, const int32_t *__restrict__ b_col,
                    const double *__restrict__ b_score, int top_n, const int64_t *__restrict__ out_indptr,
                    int32_t *__restrict__ out_row, int32_t *__restrict__ out_col, double *__restrict__ out_score,
                    const int32_t *__restrict__ big_rows, const int32_t *__restrict__ n_big) {
    __shared__ uint64_t s_key[SEL_BIG_CAP];
    __shared__ int32_t s_col[SEL_BIG_CAP];
    const int nb = *n_big;
    for (int bi = blockIdx.x; bi < nb; bi += gridDim.x) {
        const int64_t r = big_rows[bi];
        const int64_t s0 = row_start[r];
        const int m = (int)(row_start[r + 1] - s0);
        if (m <= SEL_MID_CAP) continue;         // sel_rows_mid_kernel
        int kept = 0;
        for (int start = 0; start < m;) {
            const int take = (SEL_BIG_CAP - kept) < (m - start) ? (SEL_BIG_CAP - kept) : (m - start);
            const int n_now = kept + take;
            int P = 64;
            while (P < n_now) P <<= 1;
            for (int i = kept + threadIdx.x; i < P; i += blockDim.x) {
                const int q = i - kept;
                s_key[i] = q < take ? score_key_desc(b_score[s0 + start + q]) : ~0ull;
                s_col[i] = q < take ? b_col[s0 + start + q] : -1;
            }
            __syncthreads();
            for (int k = 2; k <= P; k <<= 1) {
                for (int j = k >> 1; j > 0; j >>= 1) {
                    for (int i = threadIdx.x; i < P; i += blockDim.x) {
                        const int p = i ^ j;
                        if (p > i) {
                            const bool up = ((i & k) == 0);
                            const bool in_order = !sel_before(s_key[p], s_col[p], s_key[i], s_col[i]);
                            if (in_order != up) {
                                const uint64_t tk = s_key[i]; s_key[i] = s_key[p]; s_key[p] = tk;
                                const int32_t tc = s_col[i]; s_col[i] = s_col[p]; s_col[p] = tc;
                            }
                        }
                    }
                    __syncthreads();
                }
            }
            kept = n_now < top_n ? n_now : top_n;       // the best so far, in order, at the front
            start += take;
        }
        const int kk = kept;
        for (int i = threadIdx.x; i < kk; i += blockDim.x) {
            const uint64_t key = s_key[i];
            int a = i, b = i + 1;
            while (a > 0 && s_key[a - 1] == key) --a;
            while (b < kk && s_key[b] == key) ++b;
            const int64_t w = out_indptr[r] + a + (b - 1 - i);
            uint64_t bits = ~key;                                   // back to the score
            bits = (bits >> 63) ? (bits & 0x7fffffffffffffffull) : ~bits;
            out_row[w] = (int32_t)(r + row_begin);
            out_col[w] = s_col[i];
            out_score[w] = __longlong_as_double((long long)bits);
        }
        __syncthreads();
    }
}

__global__ void sel_finish_kernel(int64_t n_rows, const int64_t *__restrict__ out_indptr, int64_t *__restrict__ out_nnz) {
    if (threadIdx.x == 0 && blockIdx.x == 0) *out_nnz = out_indptr[n_rows];
}

__global__ void sel_max_count_kernel(int64_t n_rows, const int32_t *__restrict__ row_cnt, int32_t *__restrict__ out) {
    int m = 0;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n_rows; r += (int64_t)gridDim.x * blockDim.x)
        m = max(m, row_cnt[r]);
#pragma unroll
    for (int o = 16; o; o >>= 1) m = max(m, __shfl_xor_sync(FULL, m, o));
    if ((threadIdx.x & 31) == 0 && m > 0) atomicMax(out, m);
}

}  // namespace sg

using namespace sg;

extern "C" {

int sg_topn_rows_cap(void) { return SEL_BIG_CAP; }

/* *out_max [dev, zeroed by the caller] = largest row_cnt[r]: the caller compares it with sg_topn_rows_cap() */
int sg_row_count_max(int64_t n_rows, const int32_t *row_cnt, int32_t *out_max, void *stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (n_rows <= 0) return SG_OK;
    int64_t grid = (n_rows + 255) / 256;
    if (grid > 1184) grid = 1184;
    sel_max_count_kernel<<<(unsigned)grid, 256, 0, st>>>(n_rows, row_cnt, out_max);
    SG_LAUNCH_CHECK();
    return SG_OK;
}

size_t sg_topn_select_rows_workspace_bytes(int64_t n_cand, int64_t n_rows) {
    size_t scan_bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (int64_t *)nullptr, (int64_t *)nullptr, n_rows + 1);
    const int64_t n = n_cand < 1 ? 1 : n_cand;
    return align_up((size_t)n * 4, 256) + align_up((size_t)n * 8, 256) + 3 * align_up((size_t)(n_rows + 2) * 8, 256) +
           2 * align_up((size_t)(n_rows + 2) * 4, 256) + align_up(scan_bytes, 256) + 4096;
}

/*
 * Same contract as sg_topn_select; `row_cnt` [dev, n_rows] = survivors per row (relative to row_begin) as counted by
 * sg_rescore; every survivor must already be strictly above the threshold (sg_rescore keeps only those) and no row
 * may hold more than sg_topn_rows_cap() survivors.
 */
int sg_topn_select_rows(int64_t n_cand, const int32_t *cand_row, const int32_t *cand_col, const double *score,
                        int64_t row_begin, int64_t n_rows, int top_n, const int32_t *row_cnt, int64_t *out_indptr,
                        int32_t *out_row, int32_t *out_col, double *out_score, int64_t *out_nnz,
                        int32_t *out_max_row, void *ws, size_t ws_bytes, void *stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (n_rows < 0 || n_cand < 0) return fail(SG_ERR_INVALID, "negative size");
    SG_CUDA_TRY(cudaMemsetAsync(out_max_row, 0, sizeof(int32_t), st));
    if (n_cand == 0 || top_n <= 0 || n_rows == 0) {
        SG_CUDA_TRY(cudaMemsetAsync(out_indptr, 0, (size_t)(n_rows + 1) * sizeof(int64_t), st));
        SG_CUDA_TRY(cudaMemsetAsync(out_nnz, 0, sizeof(int64_t), st));
        return SG_OK;
    }
    Arena ar(ws, ws_bytes);
    int32_t *b_col = ar.take<int32_t>((size_t)n_cand);
    double *b_score = ar.take<double>((size_t)n_cand);
    int64_t *cnt64 = ar.take<int64_t>((size_t)n_rows + 2);
    int64_t *row_start = ar.take<int64_t>((size_t)n_rows + 2);
    int64_t *out_cnt = ar.take<int64_t>((size_t)n_rows + 2);
    int32_t *fill = ar.take<int32_t>((size_t)n_rows + 2);       // [n_rows + 1] = number of big rows
    int32_t *big_rows = ar.take<int32_t>((size_t)n_rows + 2);
    size_t scan_bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, cnt64, row_start, n_rows + 1);
    char *scan_tmp = ar.take<char>(scan_bytes);
    if (!ar.ok()) return fail(SG_ERR_INVALID, "select workspace too small (%zu < %zu)", ws_bytes, ar.off);
    int32_t *n_big = fill + n_rows + 1;
    SG_CUDA_TRY(cudaMemsetAsync(fill, 0, (size_t)(n_rows + 2) * sizeof(int32_t), st));
    sel_counts_kernel<<<(unsigned)((n_rows + 1 + 255) / 256), 256, 0, st>>>(n_rows, row_cnt, top_n, cnt64, out_cnt,
                                                                           out_max_row);
    SG_LAUNCH_CHECK();
    SG_CUDA_TRY(cub::DeviceScan::ExclusiveSum(scan_tmp, scan_bytes, cnt64, row_start, n_rows + 1, st));
    SG_CUDA_TRY(cub::DeviceScan::ExclusiveSum(scan_tmp, scan_bytes, out_cnt, out_indptr, n_rows + 1, st));
    sel_scatter_kernel<<<(unsigned)((n_cand + 255) / 256), 256, 0, st>>>(n_cand, cand_row, cand_col, score, row_begin,
                                                                        row_start, fill, b_col, b_score);
    SG_LAUNCH_CHECK();
    if (top_n <= 32) {
        // the common case (max_n_matches defaults to 20): every row, whatever its length, by one warp
        sel_rows_small_kernel<true><<<(unsigned)((n_rows + 7) / 8), 256, 0, st>>>(
            n_rows, row_begin, row_start, b_col, b_score, top_n, out_indptr, out_row, out_col, out_score, big_rows, n_big);
        SG_LAUNCH_CHECK();
    } else {
        sel_rows_small_kernel<false><<<(unsigned)((n_rows + 7) / 8), 256, 0, st>>>(
            n_rows, row_begin, row_start, b_col, b_score, top_n, out_indptr, out_row, out_col, out_score, big_rows, n_big);
        SG_LAUNCH_CHECK();
        int dev = 0, n_sm = 0;
        SG_CUDA_TRY(cudaGetDevice(&dev));
        SG_CUDA_TRY(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
        sel_rows_mid_kernel<<<(unsigned)(n_sm * 2), SEL_MID_WARPS * 32, 0, st>>>(row_begin, row_start, b_col, b_score,
                                                                                top_n, out_indptr, out_row, out_col,
                                                                                out_score, big_rows, n_big);
        SG_LAUNCH_CHECK();
        sel_rows_big_kernel<<<(unsigned)(n_sm * 2), 256, 0, st>>>(row_begin, row_start, b_col, b_score, top_n, out_indptr,
                                                                 out_row, out_col, out_score, big_rows, n_big);
        SG_LAUNCH_CHECK();
    }
    sel_finish_kernel<<<1, 32, 0, st>>>(n_rows, out_indptr, out_nnz);
    SG_LAUNCH_CHECK();
    return SG_OK;
}

}  // extern "C"
