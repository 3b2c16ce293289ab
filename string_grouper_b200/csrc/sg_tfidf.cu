// K1 — character n-gram TF-IDF with the CSR emitted directly in HBM, for sm_90a.
//
// Replaces, for ASCII input (the Python host normalises the rare non-ASCII rows
// first, exactly string_grouper/string_grouper.py:372-375):
//   StringGrouper.n_grams                         string_grouper.py:365-378
//   TfidfVectorizer(min_df=1, analyzer=n_grams).fit / .transform
//                                                 string_grouper.py:305-308, :685-707
//   (sklearn text.py: _count_vocab, _sort_features, TfidfTransformer.fit/transform;
//    sparsefuncs_fast.pyx: _inplace_csr_row_normalize_l2)
//
// One warp per document:
//   strip / fold bytes  ->  pack n-grams into order-preserving keys (7 bits per
//   char, big endian: integer order == Python string order, so the rank of a key
//   among the keys present is sklearn's sorted-vocabulary column id)  ->  sort the
//   document's keys with a warp bitonic network  ->  run-length encode to
//   (key, tf)  ->  df[key] += 1 per distinct key.
// Then (sg_tfidf_vocab): rank = exclusive scan of (df > 0), indptr, V, nnz; the host reads df in column order back and
// computes idf exactly as scikit-learn does (numpy's log); (sg_tfidf_values) tf*idf, row L2 norm in double in column
// order; indices / values written coalesced at indptr[doc].
#include <cub/cub.cuh>

#include "sg_common.cuh"

namespace sg {

constexpr int K1_WARPS = 8;
constexpr int K1_CAP = 256;  // cleaned chars handled in shared memory; longer documents use HBM scratch

__device__ __forceinline__ bool is_stripped(unsigned c) {
    // default regex r'[,-./]|\s' (string_grouper.py:19): ',' '-' '.' '/' (0x2c..0x2f) and Python's
    // str-pattern \s restricted to ASCII: \t\n\v\f\r (0x09..0x0d), 0x1c..0x1f, space.
    return (c >= 0x2cu && c <= 0x2fu) || (c >= 0x09u && c <= 0x0du) || (c >= 0x1cu && c <= 0x20u);
}

// Bitonic sort (flip variant: every comparator is ascending, so positions >= G
// behave as +inf padding without being stored).  `keys` may be shared or global.
__device__ void warp_sort_keys(uint32_t *keys, int G, int lane) {
    if (G < 2) return;
    int P = 2;
    while (P < G) P <<= 1;
    const int half = P >> 1;
    for (int k = 2; k <= P; k <<= 1) {
        const int hk = k >> 1;
        for (int i = lane; i < half; i += 32) {
            const int blk = i / hk, o = i - blk * hk;
            const int a = blk * k + o, b = blk * k + (k - 1 - o);
            if (b < G) {
                const uint32_t ka = keys[a], kb = keys[b];
                if (ka > kb) { keys[a] = kb; keys[b] = ka; }
            }
        }
        __syncwarp();
        for (int j = k >> 2; j >= 1; j >>= 1) {
            for (int i = lane; i < half; i += 32) {
                const int a = (i / j) * 2 * j + (i % j), b = a + j;
                if (b < G) {
                    const uint32_t ka = keys[a], kb = keys[b];
                    if (ka > kb) { keys[a] = kb; keys[b] = ka; }
                }
            }
            __syncwarp();
        }
    }
}

// Run-length encode the sorted keys into (out_key, out_tf); one df increment per run when kDf (a fit; a transform
// through a fitted vocabulary leaves its df table alone).
template <bool kDf>
__device__ int warp_unique_count(const uint32_t *keys, int G, uint32_t *out_key, uint32_t *out_tf,
                                 int32_t *df, int lane) {
    int nheads = 0;
    for (int base = 0; base < G; base += 32) {
        const int j = base + lane;
        const bool valid = j < G;
        const uint32_t k = valid ? keys[j] : 0xffffffffu;
        uint32_t prev = __shfl_up_sync(FULL, k, 1);
        if (lane == 0) prev = base > 0 ? keys[base - 1] : ~k;
        const bool head = valid && (k != prev);
        const unsigned hb = __ballot_sync(FULL, head);
        const int nvalid = __popc(__ballot_sync(FULL, valid));
        const int first = hb ? __ffs(hb) - 1 : 32;
        const int carry = first < nvalid ? first : nvalid;
        if (lane == 0 && carry > 0 && nheads > 0) out_tf[nheads - 1] += (uint32_t)carry;
        if (head) {
            const unsigned above = hb & ~((2u << lane) - 1u);
            const int nxt = above ? __ffs(above) - 1 : 32;
            const int cnt = (nxt < nvalid ? nxt : nvalid) - lane;
            const int h = nheads + __popc(hb & ((1u << lane) - 1u));
            out_key[h] = k;
            out_tf[h] = (uint32_t)cnt;
            if (kDf) atomicAdd(df + k, 1);
        }
        nheads += __popc(hb);
        __syncwarp();
    }
    return nheads;
}

template <bool kDf>
__global__ void __launch_bounds__(K1_WARPS * 32)
tfidf_count_kernel(const uint8_t *__restrict__ bytes, const int64_t *__restrict__ offsets, int64_t n_docs,
                   int ngram, unsigned flags, int32_t *__restrict__ df, uint8_t *__restrict__ scratch_clean,
                   uint32_t *__restrict__ scratch_sort, uint32_t *__restrict__ scratch_key,
                   uint32_t *__restrict__ scratch_tf, int32_t *__restrict__ row_nnz) {
    __shared__ uint8_t s_clean[K1_WARPS][K1_CAP];
    __shared__ uint32_t s_keys[K1_WARPS][K1_CAP];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const bool fold = flags & SG_FLAG_IGNORE_CASE, strip = flags & SG_FLAG_STRIP_DEFAULT;
    for (int64_t doc = (int64_t)blockIdx.x * K1_WARPS + warp; doc < n_docs; doc += (int64_t)gridDim.x * K1_WARPS) {
        const int64_t s = offsets[doc];
        const int64_t len = offsets[doc + 1] - s;
        const bool small = len <= K1_CAP;
        uint8_t *clean = small ? s_clean[warp] : scratch_clean + s;
        uint32_t *keys = small ? s_keys[warp] : scratch_sort + s;
        int64_t L = 0;
        for (int64_t base = 0; base < len; base += 32) {
            const int64_t i = base + lane;
            unsigned c = i < len ? bytes[s + i] : 0u;
            if (fold && c >= 'A' && c <= 'Z') c |= 0x20u;
            const bool keep = i < len && !(strip && is_stripped(c));
            const unsigned kb = __ballot_sync(FULL, keep);
            if (keep) clean[L + __popc(kb & ((1u << lane) - 1u))] = (uint8_t)(c & 0x7fu);
            L += __popc(kb);
        }
        __syncwarp();
        const int64_t G64 = L - ngram + 1;
        const int G = G64 > 0 ? (int)G64 : 0;
        for (int j = lane; j < G; j += 32) {
            uint32_t key = 0;
            for (int q = 0; q < ngram; ++q) key = (key << 7) | clean[j + q];
            keys[j] = key;
        }
        __syncwarp();
        warp_sort_keys(keys, G, lane);
        const int nnz = warp_unique_count<kDf>(keys, G, scratch_key + s, scratch_tf + s, df, lane);
        if (lane == 0) row_nnz[doc] = nnz;
        __syncwarp();
    }
}

// Transform: keep the (key, tf) runs of a document whose key the fitted vocabulary holds (df > 0), compacted in place
// at the front of the document's scratch.  Keys stay ascending, so the kept runs are in column order.
__global__ void __launch_bounds__(K1_WARPS * 32)
tfidf_known_kernel(const int64_t *__restrict__ offsets, int64_t n_docs, const int32_t *__restrict__ df,
                   uint32_t *__restrict__ scratch_key, uint32_t *__restrict__ scratch_tf, int32_t *__restrict__ row_nnz) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int64_t doc = (int64_t)blockIdx.x * K1_WARPS + warp; doc < n_docs; doc += (int64_t)gridDim.x * K1_WARPS) {
        const int64_t s = offsets[doc];
        const int nnz = row_nnz[doc];
        int kept = 0;
        for (int base = 0; base < nnz; base += 32) {
            const int i = base + lane;
            uint32_t key = 0, tf = 0;
            bool keep = false;
            if (i < nnz) {
                key = scratch_key[s + i];
                tf = scratch_tf[s + i];
                keep = df[key] > 0;
            }
            // every lane has read its run before any writes: the writes land at or before the positions read
            const unsigned kb = __ballot_sync(FULL, keep);
            if (keep) {
                const int h = kept + __popc(kb & ((1u << lane) - 1u));
                scratch_key[s + h] = key;
                scratch_tf[s + h] = tf;
            }
            kept += __popc(kb);
            __syncwarp();
        }
        if (lane == 0) row_nnz[doc] = kept;
    }
}

__global__ void df_flag_kernel(int64_t slots, const int32_t *__restrict__ df, int32_t *__restrict__ flag) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < slots) flag[i] = df[i] > 0 ? 1 : 0;
}

__global__ void tfidf_tail_kernel(int64_t slots, const int32_t *__restrict__ df, const int32_t *__restrict__ rank,
                                  int64_t n_docs, const int64_t *__restrict__ indptr,
                                  int32_t *__restrict__ vocab_size, int64_t *__restrict__ nnz_total) {
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        *vocab_size = rank[slots - 1] + (df[slots - 1] > 0 ? 1 : 0);
        *nnz_total = indptr[n_docs];
    }
}

template <typename T>
struct NormMath;
template <>
struct NormMath<double> {
    static __device__ __forceinline__ double sq(double x) { return __dmul_rn(x, x); }
    static __device__ __forceinline__ double scale(double x, double norm) { return __ddiv_rn(x, norm); }
};
template <>
struct NormMath<float> {
    static __device__ __forceinline__ double sq(float x) { return (double)__fmul_rn(x, x); }
    static __device__ __forceinline__ float scale(float x, double norm) { return (float)__ddiv_rn((double)x, norm); }
};

// T = matrix dtype (tfidf_matrix_dtype, string_grouper.py:18).  Arithmetic follows sklearn: x = tf*idf in T (idf[V]
// computed on the host by numpy, exactly TfidfTransformer.fit); sum of squares in double in column order; x / sqrt(sum).
template <typename T>
__global__ void __launch_bounds__(K1_WARPS * 32)
tfidf_values_kernel(const int64_t *__restrict__ offsets, int64_t n_docs, const T *__restrict__ idf,
                    const int32_t *__restrict__ rank, const uint32_t *__restrict__ scratch_key,
                    const uint32_t *__restrict__ scratch_tf, const int32_t *__restrict__ row_nnz,
                    const int64_t *__restrict__ indptr, int32_t *__restrict__ indices,
                    double *__restrict__ val64, float *__restrict__ val32) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int64_t doc = (int64_t)blockIdx.x * K1_WARPS + warp; doc < n_docs; doc += (int64_t)gridDim.x * K1_WARPS) {
        const int nnz = row_nnz[doc];
        if (nnz == 0) continue;
        const int64_t s = offsets[doc], o = indptr[doc];
        double sum = 0.0;
        for (int base = 0; base < nnz; base += 32) {
            const int i = base + lane;
            double sq = 0.0;
            if (i < nnz) {
                const T x = (T)scratch_tf[s + i] * idf[rank[scratch_key[s + i]]];
                sq = NormMath<T>::sq(x);
            }
            const int m = nnz - base < 32 ? nnz - base : 32;
            for (int l = 0; l < m; ++l) sum = __dadd_rn(sum, __shfl_sync(FULL, sq, l));
        }
        const double norm = __dsqrt_rn(sum);
        for (int i = lane; i < nnz; i += 32) {
            const int32_t c = rank[scratch_key[s + i]];
            T x = (T)scratch_tf[s + i] * idf[c];
            if (sum != 0.0) x = NormMath<T>::scale(x, norm);
            indices[o + i] = c;
            if (val64) val64[o + i] = (double)x;
            val32[o + i] = (float)x;
        }
    }
}

__global__ void vocab_keys_kernel(int64_t slots, const int32_t *__restrict__ df, const int32_t *__restrict__ rank,
                                  uint32_t *__restrict__ keys_out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < slots && df[i] > 0) keys_out[rank[i]] = (uint32_t)i;
}

__global__ void vocab_df_kernel(int64_t slots, const int32_t *__restrict__ df, const int32_t *__restrict__ rank,
                                int32_t *__restrict__ df_out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < slots && df[i] > 0) df_out[rank[i]] = df[i];
}

// one warp per document, 8 resident CTAs of 8 warps per SM, grid-stride beyond
static int k1_grid(int64_t n_docs, unsigned *grid_out) {
    int dev = 0, n_sm = 0;
    SG_CUDA_TRY(cudaGetDevice(&dev));
    SG_CUDA_TRY(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
    int64_t grid = (n_docs + K1_WARPS - 1) / K1_WARPS;
    const int64_t cap = (int64_t)n_sm * 8;
    *grid_out = (unsigned)(grid > cap ? cap : grid);
    return SG_OK;
}

template <bool kDf>
static int launch_count(const uint8_t *bytes, const int64_t *offsets, int64_t n_docs, int ngram, unsigned flags,
                        int32_t *df_table, uint8_t *scratch_clean, uint32_t *scratch_sort, uint32_t *scratch_key,
                        uint32_t *scratch_tf, int32_t *row_nnz, cudaStream_t st) {
    if (ngram < 1 || ngram > 4)
        return fail(SG_ERR_UNSUPPORTED, "ngram_size %d: the device vectoriser packs 7-bit characters into 32-bit keys "
                                        "and supports 1 <= ngram_size <= 4", ngram);
    if (n_docs <= 0) return SG_OK;
    unsigned grid = 0;
    const int rc = k1_grid(n_docs, &grid);
    if (rc != SG_OK) return rc;
    tfidf_count_kernel<kDf><<<grid, K1_WARPS * 32, 0, st>>>(bytes, offsets, n_docs, ngram, flags, df_table,
                                                            scratch_clean, scratch_sort, scratch_key, scratch_tf,
                                                            row_nnz);
    SG_LAUNCH_CHECK();
    return SG_OK;
}

int transform_indptr(int64_t n_docs, int32_t *row_nnz, int64_t *indptr, void *ws, size_t ws_bytes, cudaStream_t st) {
    size_t b = 0;
    cub::DeviceScan::ExclusiveScan(nullptr, b, (int32_t *)nullptr, (int64_t *)nullptr, cub::Sum(), (int64_t)0,
                                   n_docs + 1);
    if (ws_bytes < b) return fail(SG_ERR_INVALID, "tfidf transform workspace too small (%zu < %zu)", ws_bytes, b);
    // row_nnz has n_docs+1 slots; the last one is a zero so that the scan yields indptr[n_docs]
    SG_CUDA_TRY(cudaMemsetAsync(row_nnz + n_docs, 0, sizeof(int32_t), st));
    SG_CUDA_TRY(cub::DeviceScan::ExclusiveScan(ws, b, row_nnz, indptr, cub::Sum(), (int64_t)0, n_docs + 1, st));
    return SG_OK;
}

}  // namespace sg

using namespace sg;

extern "C" {

int64_t sg_tfidf_table_slots(int ngram) { return (ngram >= 1 && ngram <= 4) ? ((int64_t)1 << (7 * ngram)) : -1; }

int sg_tfidf_count(const uint8_t *bytes, const int64_t *offsets, int64_t n_docs, int ngram, unsigned flags,
                   int32_t *df_table, uint8_t *scratch_clean, uint32_t *scratch_sort, uint32_t *scratch_key,
                   uint32_t *scratch_tf, int32_t *row_nnz, void *stream_) {
    return launch_count<true>(bytes, offsets, n_docs, ngram, flags, df_table, scratch_clean, scratch_sort,
                              scratch_key, scratch_tf, row_nnz, (cudaStream_t)stream_);
}

int sg_tfidf_transform_count(const uint8_t *bytes, const int64_t *offsets, int64_t n_docs, int ngram, unsigned flags,
                             uint8_t *scratch_clean, uint32_t *scratch_sort, uint32_t *scratch_key,
                             uint32_t *scratch_tf, int32_t *row_nnz, void *stream_) {
    return launch_count<false>(bytes, offsets, n_docs, ngram, flags, nullptr, scratch_clean, scratch_sort,
                               scratch_key, scratch_tf, row_nnz, (cudaStream_t)stream_);
}

size_t sg_tfidf_transform_workspace_bytes(int64_t n_docs) {
    size_t b = 0;
    cub::DeviceScan::ExclusiveScan(nullptr, b, (int32_t *)nullptr, (int64_t *)nullptr, cub::Sum(), (int64_t)0,
                                   n_docs + 1);
    return align_up(b, 256) + 256;
}

int sg_tfidf_known(const int64_t *offsets, int64_t n_docs, const int32_t *df_table, uint32_t *scratch_key,
                   uint32_t *scratch_tf, int32_t *row_nnz, int64_t *indptr, void *ws, size_t ws_bytes,
                   void *stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (n_docs < 0) return fail(SG_ERR_INVALID, "need n_docs >= 0");
    if (n_docs > 0) {
        unsigned grid = 0;
        const int rc = k1_grid(n_docs, &grid);
        if (rc != SG_OK) return rc;
        tfidf_known_kernel<<<grid, K1_WARPS * 32, 0, st>>>(offsets, n_docs, df_table, scratch_key, scratch_tf,
                                                           row_nnz);
        SG_LAUNCH_CHECK();
    }
    return transform_indptr(n_docs, row_nnz, indptr, ws, ws_bytes, st);
}

size_t sg_tfidf_vocab_workspace_bytes(int64_t n_docs, int ngram) {
    const int64_t slots = sg_tfidf_table_slots(ngram);
    if (slots < 0) return 0;
    size_t b1 = 0, b2 = 0;
    cub::DeviceScan::ExclusiveScan(nullptr, b1, (int32_t *)nullptr, (int64_t *)nullptr, cub::Sum(), (int64_t)0,
                                   n_docs + 1);
    cub::DeviceScan::ExclusiveSum(nullptr, b2, (int32_t *)nullptr, (int32_t *)nullptr, slots);
    return align_up((size_t)slots * 4, 256) + align_up(b1 > b2 ? b1 : b2, 256) + 1024;
}

int sg_tfidf_vocab(int64_t n_docs, int ngram, const int32_t *df_table, int32_t *rank_table, int32_t *row_nnz,
                   int64_t *indptr, int32_t *vocab_size, int64_t *nnz_total, void *ws, size_t ws_bytes,
                   void *stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    const int64_t slots = sg_tfidf_table_slots(ngram);
    if (slots < 0) return fail(SG_ERR_UNSUPPORTED, "ngram_size %d unsupported (1..4)", ngram);
    if (n_docs < 0) return fail(SG_ERR_INVALID, "need n_docs >= 0");
    Arena ar(ws, ws_bytes);
    int32_t *flag = ar.take<int32_t>((size_t)slots);
    size_t b1 = 0, b2 = 0;
    cub::DeviceScan::ExclusiveScan(nullptr, b1, (int32_t *)nullptr, (int64_t *)nullptr, cub::Sum(), (int64_t)0,
                                   n_docs + 1);
    cub::DeviceScan::ExclusiveSum(nullptr, b2, (int32_t *)nullptr, (int32_t *)nullptr, slots);
    size_t cub_bytes = b1 > b2 ? b1 : b2;
    char *cub_tmp = ar.take<char>(cub_bytes);
    if (!ar.ok()) return fail(SG_ERR_INVALID, "tfidf workspace too small (%zu < %zu)", ws_bytes, ar.off);

    // row_nnz has n_docs+1 slots; the last one is a zero so that the scan yields indptr[n_docs]
    SG_CUDA_TRY(cudaMemsetAsync(row_nnz + n_docs, 0, sizeof(int32_t), st));
    SG_CUDA_TRY(cub::DeviceScan::ExclusiveScan(cub_tmp, cub_bytes, row_nnz, indptr, cub::Sum(), (int64_t)0,
                                               n_docs + 1, st));
    df_flag_kernel<<<(unsigned)((slots + 255) / 256), 256, 0, st>>>(slots, df_table, flag);
    SG_LAUNCH_CHECK();
    SG_CUDA_TRY(cub::DeviceScan::ExclusiveSum(cub_tmp, cub_bytes, flag, rank_table, slots, st));
    tfidf_tail_kernel<<<1, 32, 0, st>>>(slots, df_table, rank_table, n_docs, indptr, vocab_size, nnz_total);
    SG_LAUNCH_CHECK();
    return SG_OK;
}

int sg_tfidf_values(const int64_t *offsets, int64_t n_docs, int dtype, const void *idf, const int32_t *rank_table,
                    const uint32_t *scratch_key, const uint32_t *scratch_tf, const int32_t *row_nnz,
                    const int64_t *indptr, int32_t *indices, double *val64, float *val32, void *stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (dtype != SG_DTYPE_F32 && dtype != SG_DTYPE_F64) return fail(SG_ERR_INVALID, "bad dtype");
    if (dtype == SG_DTYPE_F64 && !val64) return fail(SG_ERR_INVALID, "val64 is required for float64");
    if (n_docs <= 0) return SG_OK;
    int dev = 0, n_sm = 0;
    SG_CUDA_TRY(cudaGetDevice(&dev));
    SG_CUDA_TRY(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
    int64_t grid = (n_docs + K1_WARPS - 1) / K1_WARPS;
    const int64_t cap = (int64_t)n_sm * 8;
    if (grid > cap) grid = cap;
    if (dtype == SG_DTYPE_F64)
        tfidf_values_kernel<double><<<(unsigned)grid, K1_WARPS * 32, 0, st>>>(
            offsets, n_docs, (const double *)idf, rank_table, scratch_key, scratch_tf, row_nnz, indptr, indices, val64,
            val32);
    else
        tfidf_values_kernel<float><<<(unsigned)grid, K1_WARPS * 32, 0, st>>>(
            offsets, n_docs, (const float *)idf, rank_table, scratch_key, scratch_tf, row_nnz, indptr, indices,
            nullptr, val32);
    SG_LAUNCH_CHECK();
    return SG_OK;
}

int sg_tfidf_vocab_keys(const int32_t *df_table, const int32_t *rank_table, int ngram, uint32_t *keys_out,
                        void *stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    const int64_t slots = sg_tfidf_table_slots(ngram);
    if (slots < 0) return fail(SG_ERR_UNSUPPORTED, "ngram_size %d unsupported (1..4)", ngram);
    vocab_keys_kernel<<<(unsigned)((slots + 255) / 256), 256, 0, st>>>(slots, df_table, rank_table, keys_out);
    SG_LAUNCH_CHECK();
    return SG_OK;
}

int sg_tfidf_vocab_df(const int32_t *df_table, const int32_t *rank_table, int ngram, int32_t *df_out, void *stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    const int64_t slots = sg_tfidf_table_slots(ngram);
    if (slots < 0) return fail(SG_ERR_UNSUPPORTED, "ngram_size %d unsupported (1..4)", ngram);
    vocab_df_kernel<<<(unsigned)((slots + 255) / 256), 256, 0, st>>>(slots, df_table, rank_table, df_out);
    SG_LAUNCH_CHECK();
    return SG_OK;
}

}  // extern "C"
