// Row ordering by heavy-feature signature, for sm_90a.
//
// No reference counterpart: this is layout work for K2 (the reference's block loop,
// string_grouper/string_grouper.py:734-750, takes rows in input order).  The product
// C = A * B^T is invariant under row permutations of A and of B, so both sides are processed in an
// order that puts rows sharing the same frequent n-grams next to each other:
//   * left tiles of R consecutive rows then share most of their heavy features, so one posting read
//     serves several rows;
//   * the docs of a heavy feature form contiguous runs of (permuted) column ids, so the 32 lanes of a
//     posting chunk hit 32 different shared-memory banks.
// signature(row) = 64-bit mask over the 64 features with the largest document frequency in the RIGHT
// matrix (bit 63 = most frequent); rows are sorted by signature (stable: ties keep input order).
#include <cub/cub.cuh>

#include "sg_common.cuh"

namespace sg {

__global__ void order_df_kernel(int64_t n_rows, const int64_t *__restrict__ indptr,
                                const int32_t *__restrict__ indices, int32_t *__restrict__ df) {
    const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= n_rows) return;
    const int64_t p1 = indptr[row + 1];
    for (int64_t p = indptr[row] + lane_id(); p < p1; p += 32) atomicAdd(df + indices[p], 1);
}

__global__ void order_iota_kernel(int64_t n, int32_t *__restrict__ v) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) v[i] = (int32_t)i;
}

// hrank[f] = position of f among the 64 most frequent features, -1 otherwise
__global__ void order_hrank_kernel(int64_t n_cols, const int32_t *__restrict__ sorted_cols, int n_heavy,
                                   int8_t *__restrict__ hrank) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_cols) hrank[i] = -1;
}
__global__ void order_hrank_fill_kernel(const int32_t *__restrict__ sorted_cols, int n_heavy,
                                        int8_t *__restrict__ hrank) {
    const int i = threadIdx.x;
    if (i < n_heavy) hrank[sorted_cols[i]] = (int8_t)i;
}

// `row_norm` (optional): the row's norm over the heavy features (sg_heavy_norms).  Its 5-bit quantisation becomes
// the most significant part of the sort key (the 5 least frequent signature bits make room), so that the rows of
// a column tile have similar heavy norms: the per-tile bound of the pruned traversal (sg_tile_bounds) is then
// close to the bound of each column.
__global__ void order_signature_kernel(int64_t row_begin, int64_t n_rows, const int64_t *__restrict__ indptr,
                                       const int32_t *__restrict__ indices, const int8_t *__restrict__ hrank,
                                       const float *__restrict__ row_norm, float norm_scale,
                                       uint64_t *__restrict__ sig, int32_t *__restrict__ ids) {
    const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (r >= n_rows) return;
    const int64_t row = row_begin + r;
    const int64_t p1 = indptr[row + 1];
    uint64_t s = 0;
    for (int64_t p = indptr[row] + lane_id(); p < p1; p += 32) {
        const int h = hrank[indices[p]];
        if (h >= 0) s |= 1ull << (63 - h);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) s |= __shfl_xor_sync(FULL, s, o);
    if (lane_id() == 0) {
        if (row_norm) {
            int q = (int)ceilf(row_norm[r] * norm_scale * 31.f);
            q = q < 0 ? 0 : (q > 31 ? 31 : q);
            s = ((uint64_t)q << 59) | (s >> 5);
        }
        sig[r] = s;
        ids[r] = (int32_t)row;
    }
}

__global__ void order_inverse_kernel(int64_t n, int64_t row_begin, const int32_t *__restrict__ perm,
                                     int32_t *__restrict__ rank) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) rank[perm[i] - row_begin] = (int32_t)i;
}

}  // namespace sg

using namespace sg;

extern "C" {

size_t sg_order_workspace_bytes(int64_t n_rows, int64_t n_cols) {
    size_t b1 = 0, b2 = 0;
    cub::DeviceRadixSort::SortPairsDescending(nullptr, b1, (int32_t *)nullptr, (int32_t *)nullptr, (int32_t *)nullptr,
                                              (int32_t *)nullptr, n_cols);
    cub::DeviceRadixSort::SortPairs(nullptr, b2, (uint64_t *)nullptr, (uint64_t *)nullptr, (int32_t *)nullptr,
                                    (int32_t *)nullptr, n_rows);
    return 4 * align_up((size_t)n_cols * 4, 256) + 2 * align_up((size_t)n_rows * 8, 256) +
           align_up((size_t)n_rows * 4, 256) + align_up(b1 > b2 ? b1 : b2, 256) + 4096;
}

// hrank[n_cols] (int8): rank of each feature among the `n_heavy` (<= 64) most frequent features of the
// matrix (indptr, indices) with n_rows rows, -1 for the others.  df_in (optional): its document frequencies.
int sg_heavy_features(int64_t n_rows, int64_t n_cols, const int64_t *indptr, const int32_t *indices,
                      const int32_t *df_in, int n_heavy, int8_t *hrank, void *ws, size_t ws_bytes, void *stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (n_heavy < 0 || n_heavy > 64) return fail(SG_ERR_INVALID, "n_heavy must be in [0, 64]");
    if (n_cols <= 0) return SG_OK;
    if (n_heavy > n_cols) n_heavy = (int)n_cols;
    Arena ar(ws, ws_bytes);
    int32_t *df = ar.take<int32_t>((size_t)n_cols);
    int32_t *df_sorted = ar.take<int32_t>((size_t)n_cols);
    int32_t *cols = ar.take<int32_t>((size_t)n_cols);
    int32_t *cols_sorted = ar.take<int32_t>((size_t)n_cols);
    size_t b1 = 0;
    cub::DeviceRadixSort::SortPairsDescending(nullptr, b1, df, df_sorted, cols, cols_sorted, n_cols);
    char *tmp = ar.take<char>(b1);
    if (!ar.ok()) return fail(SG_ERR_INVALID, "order workspace too small (%zu < %zu)", ws_bytes, ar.off);
    if (!df_in) {      // no document frequencies at hand (sg_feature_df / the vectoriser's own): count them here
        SG_CUDA_TRY(cudaMemsetAsync(df, 0, (size_t)n_cols * 4, st));
        if (n_rows > 0) {
            order_df_kernel<<<(unsigned)((n_rows + 7) / 8), 256, 0, st>>>(n_rows, indptr, indices, df);
            SG_LAUNCH_CHECK();
        }
        df_in = df;
    }
    order_iota_kernel<<<(unsigned)((n_cols + 255) / 256), 256, 0, st>>>(n_cols, cols);
    SG_LAUNCH_CHECK();
    SG_CUDA_TRY(cub::DeviceRadixSort::SortPairsDescending(tmp, b1, df_in, df_sorted, cols, cols_sorted, n_cols, 0, 32, st));
    order_hrank_kernel<<<(unsigned)((n_cols + 255) / 256), 256, 0, st>>>(n_cols, cols_sorted, n_heavy, hrank);
    SG_LAUNCH_CHECK();
    if (n_heavy > 0) {
        order_hrank_fill_kernel<<<1, 64, 0, st>>>(cols_sorted, n_heavy, hrank);
        SG_LAUNCH_CHECK();
    }
    return SG_OK;
}

// perm[i] = id of the i-th row of [row_begin, row_end) in signature order; rank = inverse (relative to row_begin).
int sg_row_order(int64_t row_begin, int64_t row_end, const int64_t *indptr, const int32_t *indices,
                 const int8_t *hrank, const float *row_norm, float norm_scale, int32_t *perm, int32_t *rank,
                 void *ws, size_t ws_bytes, void *stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    const int64_t n = row_end - row_begin;
    if (n <= 0) return SG_OK;
    Arena ar(ws, ws_bytes);
    uint64_t *sig = ar.take<uint64_t>((size_t)n);
    uint64_t *sig_sorted = ar.take<uint64_t>((size_t)n);
    int32_t *ids = ar.take<int32_t>((size_t)n);
    size_t b2 = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, b2, sig, sig_sorted, ids, perm, n);
    char *tmp = ar.take<char>(b2);
    if (!ar.ok()) return fail(SG_ERR_INVALID, "order workspace too small (%zu < %zu)", ws_bytes, ar.off);
    order_signature_kernel<<<(unsigned)((n + 7) / 8), 256, 0, st>>>(row_begin, n, indptr, indices, hrank, row_norm,
                                                                   norm_scale, sig, ids);
    SG_LAUNCH_CHECK();
    SG_CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp, b2, sig, sig_sorted, ids, perm, n, 0, 64, st));
    if (rank) {
        order_inverse_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(n, row_begin, perm, rank);
        SG_LAUNCH_CHECK();
    }
    return SG_OK;
}

}  // extern "C"
