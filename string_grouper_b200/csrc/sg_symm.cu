// K4 — self-match post-processing on the device, for sm_90a.
//
// Replaces the LIL round trip of StringGrouper.fit
// (string_grouper/string_grouper.py:419-427) with
// _fix_diagonal (:955-958: M[r,r] = 1 for every r) and _symmetrize_matrix
// (:961-964: M[c,r] = M[r,c] for every stored (r,c)), followed by tocsr()
// which orders every row by ascending column.
//
// Device formulation: emit (r,c), (c,r) for every stored entry and (r,r) for
// every row as 64-bit keys (row << 32 | col) with the source entry as payload,
// radix-sort, keep the first of each run of equal keys; diagonal keys get
// exactly 1.0.  Where both (r,c) and (c,r) were stored the reference swaps
// the two values; they are the same sum of the same products, so either is
// kept.
#include <cub/cub.cuh>

#include "sg_common.cuh"

namespace sg {

// layout of the key array: [0,nnz) stored entries, then (mirror ? [nnz,2nnz) transposes : nothing),
// then (fix_diag ? n diagonal keys : nothing)
__global__ void symm_keys_kernel(int64_t n, int64_t nnz, int mirror, int fix_diag,
                                 const int32_t *__restrict__ row, const int32_t *__restrict__ col,
                                 uint64_t *__restrict__ keys, uint32_t *__restrict__ vals) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nnz) {
        const uint64_t r = (uint32_t)row[i], c = (uint32_t)col[i];
        keys[i] = (r << 32) | c;
        vals[i] = (uint32_t)i;
        if (mirror) {
            keys[nnz + i] = (c << 32) | r;
            vals[nnz + i] = (uint32_t)i;
        }
    } else if (fix_diag && i < nnz + n) {
        const uint64_t r = (uint64_t)(i - nnz);
        const int64_t o = (mirror ? 2 * nnz : nnz) + (i - nnz);
        keys[o] = (r << 32) | r;
        vals[o] = 0xffffffffu;
    }
}

__global__ void symm_flag_kernel(int64_t m, const uint64_t *__restrict__ keys, int64_t *__restrict__ flag) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    flag[i] = (i == 0 || keys[i] != keys[i - 1]) ? 1 : 0;
}

__global__ void symm_write_kernel(int64_t m, const uint64_t *__restrict__ keys, const uint32_t *__restrict__ vals,
                                  const int64_t *__restrict__ pos, const double *__restrict__ score,
                                  int fix_diag, int32_t *__restrict__ out_row, int32_t *__restrict__ out_col,
                                  double *__restrict__ out_score, int64_t *__restrict__ out_nnz) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const bool first = (i == 0 || keys[i] != keys[i - 1]);
    if (first) {
        const uint64_t k = keys[i];
        const int32_t r = (int32_t)(k >> 32), c = (int32_t)(k & 0xffffffffu);
        const int64_t o = pos[i];
        out_row[o] = r;
        out_col[o] = c;
        out_score[o] = (fix_diag && r == c) ? 1.0 : score[vals[i]];
    }
    if (i == m - 1) *out_nnz = pos[i] + (first ? 1 : 0);
}

static int bits_for64(uint64_t v) {
    int b = 0;
    while (v) { ++b; v >>= 1; }
    return b < 1 ? 1 : b;
}

}  // namespace sg

using namespace sg;

extern "C" {

size_t sg_symmetrize_workspace_bytes(int64_t nnz_in, int64_t n) {
    const int64_t m = 2 * nnz_in + n + 1;
    size_t sort_bytes = 0, scan_bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (uint64_t *)nullptr, (uint64_t *)nullptr,
                                    (uint32_t *)nullptr, (uint32_t *)nullptr, m);
    cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (int64_t *)nullptr, (int64_t *)nullptr, m);
    return 2 * align_up((size_t)m * 8, 256) + 2 * align_up((size_t)m * 4, 256) + 2 * align_up((size_t)m * 8, 256) +
           align_up(sort_bytes, 256) + align_up(scan_bytes, 256) + 4096;
}

int sg_symmetrize(int64_t n, int64_t nnz_in, int flags, const int32_t *in_row, const int32_t *in_col,
                  const double *in_score, int32_t *out_row, int32_t *out_col, double *out_score, int64_t *out_nnz,
                  void *ws, size_t ws_bytes, void *stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (n < 0 || nnz_in < 0) return fail(SG_ERR_INVALID, "negative size");
    const int fix_diag = (flags & SG_SYMM_FIX_DIAGONAL) ? 1 : 0, mirror = (flags & SG_SYMM_MIRROR) ? 1 : 0;
    const int64_t m = (mirror ? 2 : 1) * nnz_in + (fix_diag ? n : 0);
    if (m == 0) {
        SG_CUDA_TRY(cudaMemsetAsync(out_nnz, 0, sizeof(int64_t), st));
        return SG_OK;
    }
    if (m >= (int64_t)0xfffffff0u) return fail(SG_ERR_OVERFLOW, "too many matches to symmetrise: %lld", (long long)m);
    Arena ar(ws, ws_bytes);
    uint64_t *keys_in = ar.take<uint64_t>((size_t)m);
    uint64_t *keys = ar.take<uint64_t>((size_t)m);
    uint32_t *vals_in = ar.take<uint32_t>((size_t)m);
    uint32_t *vals = ar.take<uint32_t>((size_t)m);
    int64_t *flag = ar.take<int64_t>((size_t)m);
    int64_t *pos = ar.take<int64_t>((size_t)m);
    size_t sort_bytes = 0, scan_bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, keys_in, keys, vals_in, vals, m);
    cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, flag, pos, m);
    char *sort_tmp = ar.take<char>(sort_bytes);
    char *scan_tmp = ar.take<char>(scan_bytes);
    if (!ar.ok()) return fail(SG_ERR_INVALID, "symmetrize workspace too small (%zu < %zu)", ws_bytes, ar.off);

    const unsigned g0 = (unsigned)((nnz_in + n + 255) / 256);
    symm_keys_kernel<<<g0, 256, 0, st>>>(n, nnz_in, mirror, fix_diag, in_row, in_col, keys_in, vals_in);
    SG_LAUNCH_CHECK();
    const int end_bit = 32 + bits_for64((uint64_t)(n > 0 ? n - 1 : 0));
    SG_CUDA_TRY(cub::DeviceRadixSort::SortPairs(sort_tmp, sort_bytes, keys_in, keys, vals_in, vals, m, 0,
                                                end_bit > 64 ? 64 : end_bit, st));
    const unsigned g1 = (unsigned)((m + 255) / 256);
    symm_flag_kernel<<<g1, 256, 0, st>>>(m, keys, flag);
    SG_LAUNCH_CHECK();
    SG_CUDA_TRY(cub::DeviceScan::ExclusiveSum(scan_tmp, scan_bytes, flag, pos, m, st));
    symm_write_kernel<<<g1, 256, 0, st>>>(m, keys, vals, pos, in_score, fix_diag, out_row, out_col, out_score,
                                          out_nnz);
    SG_LAUNCH_CHECK();
    return SG_OK;
}

}  // extern "C"
