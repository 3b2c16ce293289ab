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

__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }

}  // namespace sg
