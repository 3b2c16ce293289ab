// Group representatives on the device, for sm_90a  (SURVEY.md §8f row 2).
//
// Replaces the arithmetic of StringGrouper._deduplicate
// (string_grouper/string_grouper.py:851-904): weakly connected components of the match
// graph (scipy.sparse.csgraph.connected_components, :863), per-row similarity sums (:875-881) and the
// per-group choice of the representative: the first member ('first', :872-873) or the first member with
// the largest similarity sum ('centroid', :885-886, idxmax).
//
// Components: min-label hooking with atomicMin + pointer jumping until nothing changes; the label of a
// component ends up being its smallest member index, which is also the 'first' representative.
// Row sums are accumulated sequentially in storage order (the list is sorted by row, then column, exactly
// the order in which scipy's CSR row sum adds them), so 'centroid' ties resolve as in the reference.
#include "sg_common.cuh"

namespace sg {

__global__ void cc_init_kernel(int64_t n, int32_t *__restrict__ label) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) label[i] = (int32_t)i;
}

__global__ void cc_hook_kernel(int64_t nnz, const int32_t *__restrict__ row, const int32_t *__restrict__ col,
                               int32_t *__restrict__ label, int32_t *__restrict__ changed) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= nnz) return;
    const int32_t lu = label[row[e]], lv = label[col[e]];
    if (lu == lv) return;
    const int32_t hi = lu > lv ? lu : lv, lo = lu > lv ? lv : lu;
    atomicMin(label + hi, lo);
    *changed = 1;
}

__global__ void cc_compress_kernel(int64_t n, int32_t *__restrict__ label) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int32_t l = label[i];
    while (label[l] != l) l = label[l];
    label[i] = l;
}

__device__ __forceinline__ uint64_t orderable(double x) {
    const uint64_t b = (uint64_t)__double_as_longlong(x);
    return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}

// numpy's pairwise summation (numpy/_core/src/umath/loops_utils.h.src, *_pairwise_sum): fewer than 8 terms are
// added sequentially, up to 128 with eight interleaved accumulators, longer runs are split recursively.
// scipy's CSR row sum (`graph.sum(axis=1)`, string_grouper.py:880) is np.add.reduceat over the data array, which
// yields  data[first] + pairwise_sum(rest);  the 'centroid' representative among IDENTICAL strings is decided by
// exactly these rounding differences, so the same order of additions is used here.
__device__ double np_pairwise_sum(const double *a, int64_t n) {
    if (n < 8) {
        double res = 0.0;
        for (int64_t i = 0; i < n; ++i) res = __dadd_rn(res, a[i]);
        return res;
    }
    if (n <= 128) {
        double r[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) r[j] = a[j];
        int64_t i = 8;
        for (; i < n - (n % 8); i += 8) {
#pragma unroll
            for (int j = 0; j < 8; ++j) r[j] = __dadd_rn(r[j], a[i + j]);
        }
        double res = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])),
                               __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
        for (; i < n; ++i) res = __dadd_rn(res, a[i]);
        return res;
    }
    int64_t n2 = n / 2;
    n2 -= n2 % 8;
    return __dadd_rn(np_pairwise_sum(a, n2), np_pairwise_sum(a + n2, n - n2));
}

// one thread per row: segment [lower_bound(row, i), lower_bound(row, i+1)) of the row-sorted list
__global__ void cc_rowsum_kernel(int64_t n, int64_t nnz, const int32_t *__restrict__ row,
                                 const double *__restrict__ score, const int32_t *__restrict__ label,
                                 double *__restrict__ weight, unsigned long long *__restrict__ best) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int64_t lo = 0, hi = nnz;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (row[mid] < i) lo = mid + 1; else hi = mid;
    }
    int64_t hi2 = lo;      // upper bound of the segment (rows are contiguous)
    {
        int64_t a = lo, b = nnz;
        while (a < b) {
            const int64_t mid = (a + b) >> 1;
            if (row[mid] <= i) a = mid + 1; else b = mid;
        }
        hi2 = a;
    }
    const int64_t cnt = hi2 - lo;
    const double s = cnt == 0 ? 0.0 : (cnt == 1 ? score[lo] : __dadd_rn(score[lo], np_pairwise_sum(score + lo + 1, cnt - 1)));
    weight[i] = s;
    atomicMax(best + label[i], (unsigned long long)orderable(s));
}

__global__ void cc_pick_kernel(int64_t n, const int32_t *__restrict__ label, const double *__restrict__ weight,
                               const unsigned long long *__restrict__ best, int32_t *__restrict__ rep_of_root) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int32_t r = label[i];
    if ((unsigned long long)orderable(weight[i]) == best[r]) atomicMin(rep_of_root + r, (int32_t)i);
}

__global__ void cc_assign_kernel(int64_t n, const int32_t *__restrict__ label, const int32_t *__restrict__ rep_of_root,
                                 int32_t *__restrict__ rep) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) rep[i] = rep_of_root ? rep_of_root[label[i]] : label[i];
}

// ---------------------------------------------------------------------------
// nearest master per duplicate (StringGrouper._get_nearest_matches, string_grouper.py:783-849, the reduction of
// :803-807): for every right row the left row with the highest similarity, the smallest left index among equals.
// ---------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long ordered_bits(double x) {
    const unsigned long long b = (unsigned long long)__double_as_longlong(x);
    return (b >> 63) ? ~b : (b | 0x8000000000000000ull);      // order-preserving map of IEEE doubles to unsigned
}

__global__ void nearest_score_kernel(int64_t nnz, const int32_t *__restrict__ col, const double *__restrict__ score,
                                     unsigned long long *__restrict__ best_bits) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nnz) atomicMax(best_bits + col[i], ordered_bits(score[i]));
}

__global__ void nearest_row_kernel(int64_t nnz, const int32_t *__restrict__ row, const int32_t *__restrict__ col,
                                   const double *__restrict__ score, const unsigned long long *__restrict__ best_bits,
                                   int32_t *__restrict__ best_row) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nnz && ordered_bits(score[i]) == best_bits[col[i]]) atomicMin(best_row + col[i], row[i]);
}

__global__ void nearest_finish_kernel(int64_t n, int32_t *__restrict__ best_row) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && best_row[i] == 0x7f7f7f7f) best_row[i] = -1;      // the byte-wise 0x7f fill = "no row yet"
}

}  // namespace sg

using namespace sg;

extern "C" {

size_t sg_group_reps_workspace_bytes(int64_t n) {
    return 2 * align_up((size_t)(n + 1) * 4, 256) + 2 * align_up((size_t)(n + 1) * 8, 256) + 1024;
}

// Matches (row, col, score) sorted by (row, col) over n strings -> rep[i] = index of the representative of
// i's group.  centroid = 0: first member; 1: first member with the largest similarity sum.
// The component sweep reads one int32 back per round (a handful of rounds).
int sg_group_reps(int64_t n, int64_t nnz, const int32_t *row, const int32_t *col, const double *score, int centroid,
                  int32_t *rep, void *ws, size_t ws_bytes, void *stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (n <= 0) return SG_OK;
    Arena ar(ws, ws_bytes);
    int32_t *label = ar.take<int32_t>((size_t)n + 1);      // label[n] doubles as the "changed" flag
    int32_t *rep_of_root = ar.take<int32_t>((size_t)n + 1);
    double *weight = ar.take<double>((size_t)n + 1);
    unsigned long long *best = ar.take<unsigned long long>((size_t)n + 1);
    if (!ar.ok()) return fail(SG_ERR_INVALID, "group workspace too small (%zu < %zu)", ws_bytes, ar.off);
    int32_t *changed = label + n;
    const unsigned gn = (unsigned)((n + 255) / 256);
    const unsigned ge = (unsigned)((nnz + 255) / 256);
    cc_init_kernel<<<gn, 256, 0, st>>>(n, label);
    SG_LAUNCH_CHECK();
    for (int round = 0; nnz > 0 && round < 10000; ++round) {
        SG_CUDA_TRY(cudaMemsetAsync(changed, 0, sizeof(int32_t), st));
        cc_hook_kernel<<<ge, 256, 0, st>>>(nnz, row, col, label, changed);
        SG_LAUNCH_CHECK();
        cc_compress_kernel<<<gn, 256, 0, st>>>(n, label);
        SG_LAUNCH_CHECK();
        int32_t h = 0;
        SG_CUDA_TRY(cudaMemcpyAsync(&h, changed, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        SG_CUDA_TRY(cudaStreamSynchronize(st));
        if (!h) break;
    }
    if (centroid) {
        SG_CUDA_TRY(cudaMemsetAsync(best, 0, (size_t)n * 8, st));
        SG_CUDA_TRY(cudaMemsetAsync(rep_of_root, 0x7f, (size_t)n * 4, st));
        cc_rowsum_kernel<<<gn, 256, 0, st>>>(n, nnz, row, score, label, weight, best);
        SG_LAUNCH_CHECK();
        cc_pick_kernel<<<gn, 256, 0, st>>>(n, label, weight, best, rep_of_root);
        SG_LAUNCH_CHECK();
        cc_assign_kernel<<<gn, 256, 0, st>>>(n, label, rep_of_root, rep);
    } else {
        cc_assign_kernel<<<gn, 256, 0, st>>>(n, label, nullptr, rep);
    }
    SG_LAUNCH_CHECK();
    return SG_OK;
}

size_t sg_nearest_master_workspace_bytes(int64_t n_right) {
    return align_up((size_t)(n_right + 1) * 8, 256) + 1024;
}

// best[j] = left row with the highest similarity to right row j (smallest left index among equal scores), -1 when
// no match holds j.  Input: a match list in any order.
int sg_nearest_master(int64_t nnz, const int32_t *row, const int32_t *col, const double *score, int64_t n_right,
                      int32_t *best, void *ws, size_t ws_bytes, void *stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (n_right <= 0) return SG_OK;
    Arena ar(ws, ws_bytes);
    unsigned long long *best_bits = ar.take<unsigned long long>((size_t)n_right + 1);
    if (!ar.ok()) return fail(SG_ERR_INVALID, "nearest workspace too small (%zu < %zu)", ws_bytes, ar.off);
    SG_CUDA_TRY(cudaMemsetAsync(best_bits, 0, (size_t)n_right * 8, st));
    SG_CUDA_TRY(cudaMemsetAsync(best, 0xff, (size_t)n_right * 4, st));
    if (nnz > 0) {
        const unsigned ge = (unsigned)((nnz + 255) / 256);
        const unsigned gn = (unsigned)((n_right + 255) / 256);
        nearest_score_kernel<<<ge, 256, 0, st>>>(nnz, col, score, best_bits);
        SG_LAUNCH_CHECK();
        // 0x7f7f7f7f = "no row yet" for the atomicMin of the second pass (left row ids are far below it)
        SG_CUDA_TRY(cudaMemsetAsync(best, 0x7f, (size_t)n_right * 4, st));
        nearest_row_kernel<<<ge, 256, 0, st>>>(nnz, row, col, score, best_bits, best);
        SG_LAUNCH_CHECK();
        nearest_finish_kernel<<<gn, 256, 0, st>>>(n_right, best);
        SG_LAUNCH_CHECK();
    }
    return SG_OK;
}

}  // extern "C"
