// Shared helpers for the libsg_b200.so translation units (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/sg_b200.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ < 900)
#error "libsg_b200 needs sm_90a or newer (TMA bulk copies, mbarrier transaction counts)"
#endif

namespace sg {

// per-thread error text, surfaced through sg_last_error()
char *err_buf();
int fail(int code, const char *fmt, ...);

#define SG_CUDA_TRY(expr)                                                                   \
    do {                                                                                    \
        cudaError_t _e = (expr);                                                            \
        if (_e != cudaSuccess)                                                              \
            return sg::fail(SG_ERR_CUDA, "%s:%d %s -> %s", __FILE__, __LINE__, #expr,       \
                            cudaGetErrorString(_e));                                        \
    } while (0)

#define SG_LAUNCH_CHECK() SG_CUDA_TRY(cudaGetLastError())

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// bump allocator over a caller-provided workspace
struct Arena {
    char *base;
    size_t off, cap;
    Arena(void *p, size_t bytes) : base((char *)p), off(0), cap(bytes) {}
    template <typename T>
    T *take(size_t n) {
        off = align_up(off, 256);
        T *r = (T *)(base + off);
        off += n * sizeof(T);
        return r;
    }
    bool ok() const { return off <= cap; }
};

constexpr unsigned FULL = 0xffffffffu;

// Top-n floor (sg_cossim_candidates_floor): a pair must stay a candidate when its exact score can be >= floor[row]
// (ties at the cut are resolved by column), so the thresholds derived from a floor f are those of "score > f - FLOOR_EPS".
constexpr float FLOOR_EPS = 1e-6f;

__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }

// K1 transform (sg_tfidf.cu): indptr = exclusive scan of the kept runs per row (row_nnz, n_docs + 1 slots; the last is
// zeroed here), workspace of sg_tfidf_transform_workspace_bytes
int transform_indptr(int64_t n_docs, int32_t *row_nnz, int64_t *indptr, void *ws, size_t ws_bytes, cudaStream_t st);

// sg_groups.cu: weight[i] = row i's similarity sum exactly as the 'centroid' representative uses it (row-sorted list);
// label and best are n-element scratch
int group_row_weights(int64_t n, int64_t nnz, const int32_t *row, const double *score, int32_t *label, double *weight,
                      unsigned long long *best, cudaStream_t st);

}  // namespace sg
