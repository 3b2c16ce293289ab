// Weighted stacking of per-field TF-IDF matrices (match_records / group_similar_records), for sm_90a.
//
// A record has several string fields; each is vectorised on its own by K1.  Field k's rows are scaled by
// scale_k = sqrt(w_k / sum w) and the fields are laid side by side (field k's columns start after the vocabularies of
// fields 0..k-1), so the cosine of two stacked rows is sum_k (w_k / sum w) cos_k.  The stacked matrix is what K2 runs
// on, unchanged (DESIGN.md §3 "Stacked records", §4 "Fields").
//
// sg_fields_stack: indptr = exclusive scan of the summed row lengths; then one warp per row copies field after field
// to the row's running offset, adding the field's column offset and multiplying every value by scale_k in the matrix
// dtype (one IEEE rounding, __dmul_rn / __fmul_rn: no FMA can contract it).  Indices inside a row stay ascending,
// because the fields are laid out in order.  The fp32 copy is the rounded value, as K1 writes it.
#include <cub/cub.cuh>

#include "sg_common.cuh"

namespace sg {

struct FieldsArgs {
    const int64_t *indptr[SG_FIELDS_MAX];
    const int32_t *indices[SG_FIELDS_MAX];
    const void *val[SG_FIELDS_MAX];
    double scale[SG_FIELDS_MAX];
    int32_t col_offset[SG_FIELDS_MAX];
    int n_fields;
};

__global__ void fields_len_kernel(FieldsArgs f, int64_t n_rows, int64_t *__restrict__ len) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r < n_rows) {
        int64_t n = 0;
        for (int k = 0; k < f.n_fields; ++k) n += f.indptr[k][r + 1] - f.indptr[k][r];
        len[r] = n;
    } else if (r == n_rows) {
        len[r] = 0;
    }
}

__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }

// one warp per row
template <typename T>
__global__ void fields_scatter_kernel(FieldsArgs f, int64_t n_rows, const int64_t *__restrict__ out_indptr,
                                      int32_t *__restrict__ out_indices, T *__restrict__ out_val,
                                      float *__restrict__ out_val32) {
    const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (r >= n_rows) return;
    int64_t o = out_indptr[r];
    for (int k = 0; k < f.n_fields; ++k) {
        const int64_t s = f.indptr[k][r], n = f.indptr[k][r + 1] - s;
        const int32_t *__restrict__ idx = f.indices[k] + s;
        const T *__restrict__ val = static_cast<const T *>(f.val[k]) + s;
        const T sc = (T)f.scale[k];          // double -> float rounds to nearest, as numpy's astype(float32)
        const int32_t off = f.col_offset[k];
        for (int64_t j = lane_id(); j < n; j += 32) {
            const T x = mul_rn(val[j], sc);
            out_indices[o + j] = idx[j] + off;
            out_val[o + j] = x;
            if (out_val32) out_val32[o + j] = (float)x;
        }
        o += n;
    }
}

}  // namespace sg

using namespace sg;

extern "C" {

size_t sg_fields_stack_workspace_bytes(int64_t n_rows) {
    size_t b = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, b, (int64_t *)nullptr, (int64_t *)nullptr, n_rows + 1);
    return align_up((size_t)(n_rows + 2) * 8, 256) + align_up(b, 256) + 1024;
}

int sg_fields_stack(int n_fields, int64_t n_rows, const int64_t *const *indptr, const int32_t *const *indices,
                    const void *const *val, const double *scale, const int32_t *col_offset, int dtype,
                    int64_t *out_indptr, int32_t *out_indices, void *out_val, float *out_val32, void *ws,
                    size_t ws_bytes, void *stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (n_fields < 1 || n_fields > SG_FIELDS_MAX)
        return fail(SG_ERR_INVALID, "n_fields must be in [1, %d], got %d", SG_FIELDS_MAX, n_fields);
    if (n_rows < 0) return fail(SG_ERR_INVALID, "negative n_rows");
    if (dtype != SG_DTYPE_F32 && dtype != SG_DTYPE_F64)
        return fail(SG_ERR_INVALID, "dtype must be SG_DTYPE_F32 or SG_DTYPE_F64");
    FieldsArgs f{};
    f.n_fields = n_fields;
    for (int k = 0; k < n_fields; ++k) {
        if (!indptr[k] || !indices[k] || !val[k]) return fail(SG_ERR_INVALID, "field %d: missing array", k);
        if (!(scale[k] > 0.0 && scale[k] <= 1.0)) return fail(SG_ERR_INVALID, "field %d: scale must be in (0, 1]", k);
        if (col_offset[k] < 0) return fail(SG_ERR_INVALID, "field %d: negative column offset", k);
        f.indptr[k] = indptr[k];
        f.indices[k] = indices[k];
        f.val[k] = val[k];
        f.scale[k] = scale[k];
        f.col_offset[k] = col_offset[k];
    }
    Arena ar(ws, ws_bytes);
    int64_t *len = ar.take<int64_t>((size_t)n_rows + 2);
    size_t b = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, b, len, out_indptr, n_rows + 1);
    char *tmp = ar.take<char>(b);
    if (!ar.ok()) return fail(SG_ERR_INVALID, "fields workspace too small (%zu < %zu)", ws_bytes, ar.off);
    fields_len_kernel<<<(unsigned)((n_rows + 1 + 255) / 256), 256, 0, st>>>(f, n_rows, len);
    SG_LAUNCH_CHECK();
    SG_CUDA_TRY(cub::DeviceScan::ExclusiveSum(tmp, b, len, out_indptr, n_rows + 1, st));
    if (n_rows == 0) return SG_OK;
    const unsigned grid = (unsigned)((n_rows + 7) / 8);
    if (dtype == SG_DTYPE_F64)
        fields_scatter_kernel<double><<<grid, 256, 0, st>>>(f, n_rows, out_indptr, out_indices, (double *)out_val,
                                                            out_val32);
    else
        fields_scatter_kernel<float><<<grid, 256, 0, st>>>(f, n_rows, out_indptr, out_indices, (float *)out_val,
                                                           out_val32);
    SG_LAUNCH_CHECK();
    return SG_OK;
}

}  // extern "C"
