/*
 * TEST INFRASTRUCTURE — NOT PRODUCT CODE.
 *
 * CPU restatement (plain C + OpenMP) of the two operators that the reference
 * hot path delegates to the third-party package `sparse_dot_topn` (>=1.1.0,
 * un-pinned: pyproject.toml:30, setup.py:28 of the reference;
 * the wheel is not vendored with the reference):
 *
 *   sp_matmul_topn(A, B, top_n, threshold, sort, n_threads)
 *       call sites: string_grouper/string_grouper.py:725-732, :737-743
 *   zip_sp_matmul_topn(top_n, C_mats)
 *       call site:  string_grouper/string_grouper.py:746
 *
 * Published algorithm restated here (SURVEY.md Appendix A.3 / A.4):
 *   per output row i, Gustavson row-wise SpGEMM into a dense accumulator
 *   `sums[ncols]` with an intrusive linked list `next[ncols]` of touched
 *   columns (head insertion on first touch), then one walk over the list
 *   pushing every candidate with value STRICTLY greater than the running
 *   minimum into a fixed-size (top_n) min-heap that starts filled with
 *   `threshold`; optional final sort by value descending.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs may load this library; the product path
 * (string_grouper_b200/) never does.
 *
 * Parity status: pinned against the reference's own tests and tutorial
 * answers (tests/test_oracle_reference_suite.py, tests/golden/), which hold
 * only tiny inputs; there is no upstream binary to diff against here.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <float.h>
#ifdef _OPENMP
#include <omp.h>
#endif

typedef struct { double val; int64_t idx; } cand_t;

/* ---- fixed-capacity min-heap on val (root = smallest retained score) ---- */
static void heap_sift_down(cand_t *h, int64_t n, int64_t i) {
    for (;;) {
        int64_t l = 2 * i + 1, r = l + 1, m = i;
        if (l < n && h[l].val < h[m].val) m = l;
        if (r < n && h[r].val < h[m].val) m = r;
        if (m == i) return;
        cand_t t = h[i]; h[i] = h[m]; h[m] = t;
        i = m;
    }
}

/* replace the root by (idx,val) and return the new minimum */
static double heap_push_pop(cand_t *h, int64_t n, int64_t idx, double val) {
    h[0].val = val; h[0].idx = idx;
    heap_sift_down(h, n, 0);
    return h[0].val;
}

static int cmp_desc(const void *a, const void *b) {
    const cand_t *x = (const cand_t *)a, *y = (const cand_t *)b;
    if (x->val > y->val) return -1;
    if (x->val < y->val) return 1;
    /* tie order is unspecified upstream (std::sort); pick column ascending */
    return (x->idx > y->idx) - (x->idx < y->idx);
}

/* extract the real entries (idx >= 0) of a heap, optionally sorted */
static int64_t heap_drain(cand_t *h, int64_t n, int sort, int64_t *out_idx, double *out_val) {
    int64_t k = 0;
    for (int64_t j = 0; j < n; ++j) if (h[j].idx >= 0) h[k++] = h[j];
    if (sort) qsort(h, (size_t)k, sizeof(cand_t), cmp_desc);
    for (int64_t j = 0; j < k; ++j) { out_idx[j] = h[j].idx; out_val[j] = h[j].val; }
    return k;
}

/*
 * C = top_n_per_row(A * B, > threshold).
 * A: CSR nrows x K.  B: CSR K x ncols (this is what the python wrapper gets
 * after converting the CSC `Bi.T` back to CSR).  values are double; the f32
 * entry point below rounds through float the way a float32 kernel would.
 * Outputs: row_cnt[nrows], and per-row slabs out_idx/out_val[nrows*top_n].
 * Returns total nnz, or -1 on allocation failure.
 */
#define DEFINE_MATMUL(NAME, T)                                                              \
int64_t NAME(int64_t nrows, int64_t ncols, int64_t top_n, double threshold_d, int sort,    \
             int n_threads,                                                                 \
             const int64_t *a_indptr, const int64_t *a_idx, const T *a_val,                 \
             const int64_t *b_indptr, const int64_t *b_idx, const T *b_val,                 \
             int64_t *row_cnt, int64_t *out_idx, double *out_val)                           \
{                                                                                           \
    if (top_n > ncols) top_n = ncols;                                                       \
    if (top_n <= 0 || nrows <= 0) { for (int64_t i = 0; i < nrows; ++i) row_cnt[i] = 0; return 0; } \
    const T threshold = (T)threshold_d;                                                     \
    int failed = 0;                                                                         \
    int64_t total = 0;                                                                      \
    if (n_threads < 1) n_threads = 1;                                                       \
    _Pragma("omp parallel num_threads(n_threads) reduction(+:total)")                       \
    {                                                                                       \
        T *sums = (T *)calloc((size_t)ncols, sizeof(T));                                    \
        int64_t *next = (int64_t *)malloc((size_t)ncols * sizeof(int64_t));                 \
        cand_t *heap = (cand_t *)malloc((size_t)top_n * sizeof(cand_t));                    \
        if (!sums || !next || !heap) {                                                      \
            _Pragma("omp atomic write") failed = 1;                                         \
        } else {                                                                            \
            for (int64_t k = 0; k < ncols; ++k) next[k] = -1;                               \
            _Pragma("omp for schedule(dynamic, 64)")                                        \
            for (int64_t i = 0; i < nrows; ++i) {                                           \
                int64_t head = -2, length = 0;                                              \
                for (int64_t p = a_indptr[i]; p < a_indptr[i + 1]; ++p) {                   \
                    const int64_t j = a_idx[p];                                             \
                    const T v = a_val[p];                                                   \
                    for (int64_t q = b_indptr[j]; q < b_indptr[j + 1]; ++q) {               \
                        const int64_t k = b_idx[q];                                         \
                        sums[k] += v * b_val[q];                                            \
                        if (next[k] == -1) { next[k] = head; head = k; ++length; }          \
                    }                                                                       \
                }                                                                           \
                for (int64_t s = 0; s < top_n; ++s) { heap[s].val = (double)threshold; heap[s].idx = -1; } \
                T minv = threshold;                                                         \
                for (int64_t s = 0; s < length; ++s) {                                      \
                    const int64_t k = head;                                                 \
                    if (sums[k] > minv) minv = (T)heap_push_pop(heap, top_n, k, (double)sums[k]); \
                    head = next[k]; next[k] = -1; sums[k] = 0;                              \
                }                                                                           \
                const int64_t c = heap_drain(heap, top_n, sort, out_idx + i * top_n, out_val + i * top_n); \
                row_cnt[i] = c; total += c;                                                 \
            }                                                                               \
        }                                                                                   \
        free(sums); free(next); free(heap);                                                 \
    }                                                                                       \
    return failed ? -1 : total;                                                             \
}

DEFINE_MATMUL(sgo_sp_matmul_topn_f64, double)
DEFINE_MATMUL(sgo_sp_matmul_topn_f32, float)

/*
 * zip: per row, merge the (already thresholded, value-descending) rows of
 * nblk block results whose column ids are offset by the cumulative block
 * widths; blocks visited in REVERSE order, strict '>' against a heap that
 * starts at the smallest positive normal (exact zeros are dropped).
 * blk_indptr[b] / blk_idx[b] / blk_val[b] are arrays of pointers.
 */
int64_t sgo_zip_topn_f64(int64_t nrows, int64_t top_n, int64_t nblk,
                         const int64_t *const *blk_indptr, const int64_t *const *blk_idx,
                         const double *const *blk_val, const int64_t *blk_offset,
                         int use_float_min,
                         int64_t *row_cnt, int64_t *out_idx, double *out_val)
{
    if (top_n <= 0) { for (int64_t i = 0; i < nrows; ++i) row_cnt[i] = 0; return 0; }
    cand_t *heap = (cand_t *)malloc((size_t)top_n * sizeof(cand_t));
    if (!heap) return -1;
    const double floor_v = use_float_min ? (double)FLT_MIN : DBL_MIN;
    int64_t total = 0;
    for (int64_t i = 0; i < nrows; ++i) {
        for (int64_t s = 0; s < top_n; ++s) { heap[s].val = floor_v; heap[s].idx = -1; }
        double minv = floor_v;
        for (int64_t b = nblk - 1; b >= 0; --b) {
            const int64_t *ip = blk_indptr[b];
            for (int64_t p = ip[i]; p < ip[i + 1]; ++p) {
                const double v = blk_val[b][p];
                if (v > minv) minv = heap_push_pop(heap, top_n, blk_idx[b][p] + blk_offset[b], v);
            }
        }
        const int64_t c = heap_drain(heap, top_n, 1, out_idx + i * top_n, out_val + i * top_n);
        row_cnt[i] = c; total += c;
    }
    free(heap);
    return total;
}

int sgo_max_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}
