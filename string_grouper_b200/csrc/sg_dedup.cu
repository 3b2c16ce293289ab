// Groups of bit-identical rows of a CSR matrix, for sm_90a (the dedup path of a self-match, DESIGN.md §4).
//
// A self-match of a name list full of exact repeats computes the same row many times over: rows whose indices and
// values are bit-identical score bit-identically against every column (sg_rescore adds the same products in the same
// order).  sg_row_dedup puts such rows into groups, sg_rows_gather builds the matrix U of one representative per
// group; the product runs over U and sg_topn_select_groups (sg_select.cu) expands the result back to every row.
//
// Grouping: a 64-bit hash per row over (index, value bits), a stable radix sort of (hash, row), and a group starts
// at every sorted position whose hash differs from its predecessor's or whose row is not bit-identical to it (the
// hash is only a sort key; equality is verified).  A group is therefore a run of identical rows inside a run of equal
// hashes; two identical rows separated by a colliding different row land in two groups, which the expansion (a
// union of members) handles like any other pair of groups.  The groups are then renumbered by their first member, so
// U's rows are a subsequence of the matrix's in the original order.
#include <cub/cub.cuh>

#include "sg_common.cuh"

namespace sg {

__device__ __forceinline__ uint64_t mix64(uint64_t x) {      // splitmix64 finaliser
    x ^= x >> 30;
    x *= 0xbf58476d1ce4e5b9ull;
    x ^= x >> 27;
    x *= 0x94d049bb133111ebull;
    return x ^ (x >> 31);
}

// one warp per row; V = the value bits (uint64_t for float64, uint32_t for float32)
template <typename V>
__global__ void dedup_hash_kernel(int64_t n_rows, const int64_t *__restrict__ indptr,
                                  const int32_t *__restrict__ indices, const V *__restrict__ val, uint64_t mask,
                                  uint64_t *__restrict__ key, int32_t *__restrict__ row_id) {
    const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = lane_id();
    if (r >= n_rows) return;
    const int64_t s0 = indptr[r], len = indptr[r + 1] - s0;
    uint64_t h = 0;
    for (int64_t k = lane; k < len; k += 32) {
        const uint64_t i = (uint64_t)(uint32_t)indices[s0 + k] | ((uint64_t)k << 32);
        h += mix64(i ^ 0x9e3779b97f4a7c15ull) ^ mix64((uint64_t)val[s0 + k] + (uint64_t)k * 0x632be59bd9b4e019ull);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) h += __shfl_xor_sync(FULL, h, o);
    if (lane == 0) {
        key[r] = mix64(h ^ mix64((uint64_t)len)) & mask;
        row_id[r] = (int32_t)r;
    }
}

// head[p] = 1 where a group starts in sorted order: a new hash, or a row that is not bit-identical to its predecessor
template <typename V>
__global__ void dedup_head_kernel(int64_t n, const uint64_t *__restrict__ key, const int32_t *__restrict__ row,
                                  const int64_t *__restrict__ indptr, const int32_t *__restrict__ indices,
                                  const V *__restrict__ val, int32_t *__restrict__ head) {
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    int h = 1;
    if (p > 0 && key[p] == key[p - 1]) {
        const int64_t a = indptr[row[p]], len = indptr[row[p] + 1] - a;
        const int64_t b = indptr[row[p - 1]];
        if (indptr[row[p - 1] + 1] - b == len) {
            h = 0;
            for (int64_t k = 0; k < len; ++k)
                if (indices[a + k] != indices[b + k] || val[a + k] != val[b + k]) {
                    h = 1;
                    break;
                }
        }
    }
    head[p] = h;
}

// gsorted = inclusive scan of head: the group of sorted position p is gsorted[p] - 1 (hash order)
__global__ void dedup_mark_kernel(int64_t n, const int32_t *__restrict__ row, const int32_t *__restrict__ head,
                                  const int32_t *__restrict__ gsorted, int32_t *__restrict__ is_rep,
                                  int32_t *__restrict__ start, int64_t *__restrict__ out_sizes) {
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    is_rep[row[p]] = head[p];
    if (head[p]) start[gsorted[p] - 1] = (int32_t)p;
    if (p == n - 1) {
        start[gsorted[p]] = (int32_t)n;
        out_sizes[0] = gsorted[p];
    }
}

// per group (at its head): the new id (rank of its first member among the first members), size and representative
__global__ void dedup_groups_kernel(int64_t n, const int64_t *__restrict__ indptr, const int32_t *__restrict__ row,
                                    const int32_t *__restrict__ head, const int32_t *__restrict__ gsorted,
                                    const int32_t *__restrict__ start, const int32_t *__restrict__ new_id,
                                    int32_t *__restrict__ size_u, int32_t *__restrict__ rep,
                                    unsigned long long *__restrict__ rep_nnz) {
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint64_t len = 0;
    if (p < n && head[p]) {
        const int32_t g = gsorted[p] - 1, r = row[p], u = new_id[r];
        size_u[u] = start[g + 1] - start[g];
        rep[u] = r;
        len = (uint64_t)(indptr[r + 1] - indptr[r]);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) len += __shfl_xor_sync(FULL, len, o);
    if (lane_id() == 0 && len) atomicAdd(rep_nnz, (unsigned long long)len);
}

// every row: its group id and its place among the members (ascending rows: the sort is stable)
__global__ void dedup_members_kernel(int64_t n, const int32_t *__restrict__ row, const int32_t *__restrict__ gsorted,
                                     const int32_t *__restrict__ start, const int32_t *__restrict__ new_id,
                                     const int32_t *__restrict__ mem_ptr, int32_t *__restrict__ uid,
                                     int32_t *__restrict__ mem_rows) {
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    const int32_t s = start[gsorted[p] - 1];
    const int32_t u = new_id[row[s]];
    uid[row[p]] = u;
    mem_rows[mem_ptr[u] + (p - s)] = row[p];
}

__global__ void gather_row_len_kernel(int64_t m, const int32_t *__restrict__ rep, const int64_t *__restrict__ indptr,
                                      int64_t *__restrict__ len) {
    const int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (u < m) len[u] = indptr[rep[u] + 1] - indptr[rep[u]];
    else if (u == m) len[u] = 0;
}

// one warp per row of U
template <typename V>
__global__ void gather_rows_kernel(int64_t m, const int32_t *__restrict__ rep, const int64_t *__restrict__ indptr,
                                   const int32_t *__restrict__ indices, const V *__restrict__ val,
                                   const float *__restrict__ val32, const int64_t *__restrict__ out_indptr,
                                   int32_t *__restrict__ out_indices, V *__restrict__ out_val,
                                   float *__restrict__ out_val32) {
    const int64_t u = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (u >= m) return;
    const int64_t s = indptr[rep[u]], len = indptr[rep[u] + 1] - s, o = out_indptr[u];
    for (int64_t k = lane_id(); k < len; k += 32) {
        out_indices[o + k] = indices[s + k];
        out_val[o + k] = val[s + k];
        if (out_val32) out_val32[o + k] = val32[s + k];
    }
}

struct DedupWs {
    uint64_t *key_in, *key_out;
    int32_t *row_in, *row_out, *head, *gsorted, *start, *is_rep, *new_id, *size_u;
    char *sort_tmp, *scan_tmp;
    size_t sort_bytes, scan_bytes;
};

static size_t dedup_carve(Arena &ar, int64_t n, DedupWs *w) {
    DedupWs d{};
    const size_t n1 = (size_t)n + 2;
    d.key_in = ar.take<uint64_t>(n1);
    d.key_out = ar.take<uint64_t>(n1);
    d.row_in = ar.take<int32_t>(n1);
    d.row_out = ar.take<int32_t>(n1);
    d.head = ar.take<int32_t>(n1);
    d.gsorted = ar.take<int32_t>(n1);
    d.start = ar.take<int32_t>(n1);
    d.is_rep = ar.take<int32_t>(n1);
    d.new_id = ar.take<int32_t>(n1);
    d.size_u = ar.take<int32_t>(n1);
    cub::DeviceRadixSort::SortPairs(nullptr, d.sort_bytes, d.key_in, d.key_out, d.row_in, d.row_out, n);
    size_t a = 0, b = 0;
    cub::DeviceScan::InclusiveSum(nullptr, a, d.head, d.gsorted, n);
    cub::DeviceScan::ExclusiveSum(nullptr, b, d.is_rep, d.new_id, n + 1);
    d.scan_bytes = a > b ? a : b;
    d.sort_tmp = ar.take<char>(d.sort_bytes);
    d.scan_tmp = ar.take<char>(d.scan_bytes);
    if (w) *w = d;
    return ar.off;
}

}  // namespace sg

using namespace sg;

extern "C" {

size_t sg_row_dedup_workspace_bytes(int64_t n_rows) {
    Arena ar(nullptr, 0);
    return dedup_carve(ar, n_rows < 1 ? 1 : n_rows, nullptr) + 4096;
}

int sg_row_dedup(int64_t n_rows, const int64_t *indptr, const int32_t *indices, const void *val, int dtype,
                 uint64_t hash_mask, int32_t *uid, int32_t *mem_ptr, int32_t *mem_rows, int32_t *rep,
                 int64_t *out_sizes, void *ws, size_t ws_bytes, void *stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (n_rows < 0 || n_rows >= INT32_MAX) return fail(SG_ERR_INVALID, "row count %lld out of range", (long long)n_rows);
    if (dtype != SG_DTYPE_F32 && dtype != SG_DTYPE_F64) return fail(SG_ERR_INVALID, "bad dtype %d", dtype);
    SG_CUDA_TRY(cudaMemsetAsync(out_sizes, 0, 2 * sizeof(int64_t), st));
    if (n_rows == 0) {
        SG_CUDA_TRY(cudaMemsetAsync(mem_ptr, 0, sizeof(int32_t), st));
        return SG_OK;
    }
    const int64_t n = n_rows;
    Arena ar(ws, ws_bytes);
    DedupWs w;
    dedup_carve(ar, n, &w);
    if (!ar.ok()) return fail(SG_ERR_INVALID, "dedup workspace too small (%zu < %zu)", ws_bytes, ar.off);
    const bool f64 = dtype == SG_DTYPE_F64;
    const unsigned g_warp = (unsigned)((n + 7) / 8), g_thr = (unsigned)((n + 255) / 256);
    if (f64)
        dedup_hash_kernel<uint64_t><<<g_warp, 256, 0, st>>>(n, indptr, indices, (const uint64_t *)val, hash_mask,
                                                            w.key_in, w.row_in);
    else
        dedup_hash_kernel<uint32_t><<<g_warp, 256, 0, st>>>(n, indptr, indices, (const uint32_t *)val, hash_mask,
                                                            w.key_in, w.row_in);
    SG_LAUNCH_CHECK();
    const int end_bit = hash_mask ? 64 - __builtin_clzll(hash_mask) : 1;
    SG_CUDA_TRY(cub::DeviceRadixSort::SortPairs(w.sort_tmp, w.sort_bytes, w.key_in, w.key_out, w.row_in, w.row_out,
                                                n, 0, end_bit, st));
    if (f64)
        dedup_head_kernel<uint64_t><<<g_thr, 256, 0, st>>>(n, w.key_out, w.row_out, indptr, indices,
                                                           (const uint64_t *)val, w.head);
    else
        dedup_head_kernel<uint32_t><<<g_thr, 256, 0, st>>>(n, w.key_out, w.row_out, indptr, indices,
                                                           (const uint32_t *)val, w.head);
    SG_LAUNCH_CHECK();
    SG_CUDA_TRY(cub::DeviceScan::InclusiveSum(w.scan_tmp, w.scan_bytes, w.head, w.gsorted, n, st));
    dedup_mark_kernel<<<g_thr, 256, 0, st>>>(n, w.row_out, w.head, w.gsorted, w.is_rep, w.start, out_sizes);
    SG_LAUNCH_CHECK();
    SG_CUDA_TRY(cudaMemsetAsync(w.is_rep + n, 0, sizeof(int32_t), st));
    SG_CUDA_TRY(cub::DeviceScan::ExclusiveSum(w.scan_tmp, w.scan_bytes, w.is_rep, w.new_id, n + 1, st));
    // size_u[u] for u < m, zero above: the scan over n + 1 entries leaves mem_ptr[m..n] = n
    SG_CUDA_TRY(cudaMemsetAsync(w.size_u, 0, (size_t)(n + 1) * sizeof(int32_t), st));
    dedup_groups_kernel<<<g_thr, 256, 0, st>>>(n, indptr, w.row_out, w.head, w.gsorted, w.start, w.new_id, w.size_u,
                                               rep, (unsigned long long *)(out_sizes + 1));
    SG_LAUNCH_CHECK();
    SG_CUDA_TRY(cub::DeviceScan::ExclusiveSum(w.scan_tmp, w.scan_bytes, w.size_u, mem_ptr, n + 1, st));
    dedup_members_kernel<<<g_thr, 256, 0, st>>>(n, w.row_out, w.gsorted, w.start, w.new_id, mem_ptr, uid, mem_rows);
    SG_LAUNCH_CHECK();
    return SG_OK;
}

size_t sg_rows_gather_workspace_bytes(int64_t m) {
    size_t b = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, b, (int64_t *)nullptr, (int64_t *)nullptr, m + 1);
    return align_up((size_t)(m + 2) * 8, 256) + align_up(b, 256) + 1024;
}

int sg_rows_gather(int64_t m, const int32_t *rep, const int64_t *indptr, const int32_t *indices, const void *val,
                   const float *val32, int dtype, int64_t *out_indptr, int32_t *out_indices, void *out_val,
                   float *out_val32, void *ws, size_t ws_bytes, void *stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (m < 0) return fail(SG_ERR_INVALID, "negative row count");
    if (dtype != SG_DTYPE_F32 && dtype != SG_DTYPE_F64) return fail(SG_ERR_INVALID, "bad dtype %d", dtype);
    Arena ar(ws, ws_bytes);
    int64_t *len = ar.take<int64_t>((size_t)m + 2);
    size_t b = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, b, len, out_indptr, m + 1);
    char *tmp = ar.take<char>(b);
    if (!ar.ok()) return fail(SG_ERR_INVALID, "gather workspace too small (%zu < %zu)", ws_bytes, ar.off);
    gather_row_len_kernel<<<(unsigned)((m + 1 + 255) / 256), 256, 0, st>>>(m, rep, indptr, len);
    SG_LAUNCH_CHECK();
    SG_CUDA_TRY(cub::DeviceScan::ExclusiveSum(tmp, b, len, out_indptr, m + 1, st));
    if (m == 0) return SG_OK;
    const unsigned grid = (unsigned)((m + 7) / 8);
    if (dtype == SG_DTYPE_F64)
        gather_rows_kernel<uint64_t><<<grid, 256, 0, st>>>(m, rep, indptr, indices, (const uint64_t *)val, val32,
                                                           out_indptr, out_indices, (uint64_t *)out_val, out_val32);
    else
        gather_rows_kernel<uint32_t><<<grid, 256, 0, st>>>(m, rep, indptr, indices, (const uint32_t *)val, val32,
                                                           out_indptr, out_indices, (uint32_t *)out_val, out_val32);
    SG_LAUNCH_CHECK();
    return SG_OK;
}

}  // extern "C"
