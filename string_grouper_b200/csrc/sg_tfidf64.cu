// K1, general form — character n-gram TF-IDF with 64-bit keys and a sort-based vocabulary, for sm_90a.
//
// Same reference functions as sg_tfidf.cu (StringGrouper.n_grams string_grouper.py:365-378; TfidfVectorizer fit /
// transform :305-308, :685-707), for everything its dense 2^(7n) key table cannot hold: ngram_size >= 4 and text
// that keeps non-ASCII code points (normalize_to_ascii=False, :374-375 skipped).
//
// The host maps every distinct symbol of the cleaned text to its rank in sorted order (an order-preserving dense
// alphabet of S symbols, b = ceil(log2 S) bits each), so an n-gram packs big-endian into n*b <= 64 bits and integer
// order == Python string order (sklearn's sorted vocabulary, text.py:1209-1216):
//   * 1-byte input: a 256-entry table folds, strips and maps the bytes in one step (0xff = deleted);
//   * 4-byte input: already dense symbol ids (the host ran lower() / regex on the code points).
// One warp per document: keys -> warp bitonic sort -> run-length (key, tf).  Vocabulary: all (document, key) runs are
// radix-sorted once; run heads = the distinct n-grams in sorted order (column ids by a scan), run lengths = document
// frequencies.  No table proportional to the key space exists.
#include <cub/cub.cuh>

#include "sg_common.cuh"

namespace sg {

constexpr int K64_WARPS = 8;
constexpr int K64_CAP = 256;      // cleaned symbols handled in shared memory; longer documents use HBM scratch

__device__ void warp_sort_keys64(uint64_t *keys, int G, int lane) {
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
                const uint64_t ka = keys[a], kb = keys[b];
                if (ka > kb) { keys[a] = kb; keys[b] = ka; }
            }
        }
        __syncwarp();
        for (int j = k >> 2; j >= 1; j >>= 1) {
            for (int i = lane; i < half; i += 32) {
                const int a = (i / j) * 2 * j + (i % j), b = a + j;
                if (b < G) {
                    const uint64_t ka = keys[a], kb = keys[b];
                    if (ka > kb) { keys[a] = kb; keys[b] = ka; }
                }
            }
            __syncwarp();
        }
    }
}

// run-length encode sorted keys into (out_key, out_tf); returns the number of runs
__device__ int warp_unique_count64(const uint64_t *keys, int G, uint64_t *out_key, uint32_t *out_tf, int lane) {
    int nheads = 0;
    for (int base = 0; base < G; base += 32) {
        const int j = base + lane;
        const bool valid = j < G;
        const uint64_t k = valid ? keys[j] : ~0ull;
        uint64_t prev = __shfl_up_sync(FULL, k, 1);
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
        }
        nheads += __popc(hb);
        __syncwarp();
    }
    return nheads;
}

template <typename SymT>
__global__ void __launch_bounds__(K64_WARPS * 32)
tfidf64_count_kernel(const SymT *__restrict__ symbols, const int64_t *__restrict__ offsets, int64_t n_docs, int ngram,
                     int bits, const uint8_t *__restrict__ lut, uint32_t *__restrict__ scratch_clean,
                     uint64_t *__restrict__ scratch_sort, uint64_t *__restrict__ scratch_key,
                     uint32_t *__restrict__ scratch_tf, int32_t *__restrict__ row_nnz) {
    __shared__ uint32_t s_clean[K64_WARPS][K64_CAP];
    __shared__ uint64_t s_keys[K64_WARPS][K64_CAP];
    __shared__ uint8_t s_lut[256];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (sizeof(SymT) == 1) {
        for (int i = threadIdx.x; i < 256; i += blockDim.x) s_lut[i] = lut[i];
        __syncthreads();
    }
    for (int64_t doc = (int64_t)blockIdx.x * K64_WARPS + warp; doc < n_docs; doc += (int64_t)gridDim.x * K64_WARPS) {
        const int64_t s = offsets[doc];
        const int64_t len = offsets[doc + 1] - s;
        const bool small = len <= K64_CAP;
        uint32_t *clean = small ? s_clean[warp] : scratch_clean + s;
        uint64_t *keys = small ? s_keys[warp] : scratch_sort + s;
        int64_t L = 0;
        for (int64_t base = 0; base < len; base += 32) {
            const int64_t i = base + lane;
            unsigned c = 0;
            bool keep = false;
            if (i < len) {
                if (sizeof(SymT) == 1) {
                    c = s_lut[(unsigned)symbols[s + i] & 0xffu];
                    keep = c != 0xffu;
                } else {
                    c = (unsigned)symbols[s + i];
                    keep = true;
                }
            }
            const unsigned kb = __ballot_sync(FULL, keep);
            if (keep) clean[L + __popc(kb & ((1u << lane) - 1u))] = c;
            L += __popc(kb);
        }
        __syncwarp();
        const int64_t G64 = L - ngram + 1;
        const int G = G64 > 0 ? (int)G64 : 0;
        for (int j = lane; j < G; j += 32) {
            uint64_t key = 0;
            for (int q = 0; q < ngram; ++q) key = (key << bits) | (uint64_t)clean[j + q];
            keys[j] = key;
        }
        __syncwarp();
        warp_sort_keys64(keys, G, lane);
        const int nnz = warp_unique_count64(keys, G, scratch_key + s, scratch_tf + s, lane);
        if (lane == 0) row_nnz[doc] = nnz;
        __syncwarp();
    }
}

// (document, key) runs from their per-document scratch positions into CSR order
__global__ void tfidf64_compact_kernel(int64_t n_docs, const int64_t *__restrict__ offsets,
                                       const int64_t *__restrict__ indptr, const uint64_t *__restrict__ scratch_key,
                                       uint64_t *__restrict__ keys, uint32_t *__restrict__ pos) {
    const int64_t doc = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (doc >= n_docs) return;
    const int64_t s = offsets[doc], o = indptr[doc];
    const int nnz = (int)(indptr[doc + 1] - o);
    for (int i = lane_id(); i < nnz; i += 32) {
        keys[o + i] = scratch_key[s + i];
        pos[o + i] = (uint32_t)(o + i);
    }
}

// nnz lives on the device (indptr[n_docs]); the arrays are sized by the host-known upper bound `n`
__global__ void tfidf64_heads_kernel(int64_t n, const int64_t *__restrict__ nnz_ptr,
                                     const uint64_t *__restrict__ keys_sorted, int32_t *__restrict__ head) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) head[i] = (i < *nnz_ptr && (i == 0 || keys_sorted[i] != keys_sorted[i - 1])) ? 1 : 0;
}

// col_scan = inclusive scan of head; column of sorted position i = col_scan[i] - 1
__global__ void tfidf64_columns_kernel(const int64_t *__restrict__ nnz_ptr, const uint64_t *__restrict__ keys_sorted,
                                       const uint32_t *__restrict__ pos_sorted, const int32_t *__restrict__ head,
                                       const int32_t *__restrict__ col_scan, int32_t *__restrict__ col_of_entry,
                                       uint64_t *__restrict__ vocab_keys, int32_t *__restrict__ head_pos,
                                       int32_t *__restrict__ vocab_size) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t nnz = *nnz_ptr;
    if (i >= nnz) return;
    const int c = col_scan[i] - 1;
    col_of_entry[pos_sorted[i]] = c;
    if (head[i]) {
        vocab_keys[c] = keys_sorted[i];
        head_pos[c] = (int32_t)i;
    }
    if (i == nnz - 1) {
        *vocab_size = c + 1;
        head_pos[c + 1] = (int32_t)nnz;
    }
}

__global__ void tfidf64_df_kernel(const int32_t *__restrict__ vocab_size, const int32_t *__restrict__ head_pos,
                                  int32_t *__restrict__ df, int64_t cap) {
    const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (c < cap && c < *vocab_size) df[c] = head_pos[c + 1] - head_pos[c];
}

template <typename T>
struct IdfMath64;
template <>
struct IdfMath64<double> {
    static __device__ __forceinline__ double idf(int64_t n1, int32_t dfk) {
        return log(__ddiv_rn((double)n1, (double)(dfk + 1))) + 1.0;
    }
    static __device__ __forceinline__ double sq(double x) { return __dmul_rn(x, x); }
    static __device__ __forceinline__ double scale(double x, double norm) { return __ddiv_rn(x, norm); }
};
template <>
struct IdfMath64<float> {
    static __device__ __forceinline__ float idf(int64_t n1, int32_t dfk) {
        return __fadd_rn(logf(__fdiv_rn((float)n1, (float)(dfk + 1))), 1.0f);
    }
    static __device__ __forceinline__ double sq(float x) { return (double)__fmul_rn(x, x); }
    static __device__ __forceinline__ float scale(float x, double norm) { return (float)__ddiv_rn((double)x, norm); }
};

// same arithmetic as tfidf_finalize_kernel (sklearn: idf in T, x = tf*idf in T, squares summed in double in column
// order, x / sqrt(sum)); the column and df of an entry come from the sorted vocabulary
template <typename T>
__global__ void __launch_bounds__(K64_WARPS * 32)
tfidf64_finalize_kernel(const int64_t *__restrict__ offsets, int64_t n_docs, int64_t n_docs_fit,
                        const int32_t *__restrict__ df, const int32_t *__restrict__ col_of_entry,
                        const uint32_t *__restrict__ scratch_tf, const int64_t *__restrict__ indptr,
                        int32_t *__restrict__ indices, double *__restrict__ val64, float *__restrict__ val32) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t n1 = n_docs_fit + 1;
    for (int64_t doc = (int64_t)blockIdx.x * K64_WARPS + warp; doc < n_docs; doc += (int64_t)gridDim.x * K64_WARPS) {
        const int64_t s = offsets[doc], o = indptr[doc];
        const int nnz = (int)(indptr[doc + 1] - o);
        if (nnz == 0) continue;
        double sum = 0.0;
        for (int base = 0; base < nnz; base += 32) {
            const int i = base + lane;
            double sq = 0.0;
            if (i < nnz) {
                const T x = (T)scratch_tf[s + i] * IdfMath64<T>::idf(n1, df[col_of_entry[o + i]]);
                sq = IdfMath64<T>::sq(x);
            }
            const int m = nnz - base < 32 ? nnz - base : 32;
            for (int l = 0; l < m; ++l) sum = __dadd_rn(sum, __shfl_sync(FULL, sq, l));
        }
        const double norm = __dsqrt_rn(sum);
        for (int i = lane; i < nnz; i += 32) {
            const int c = col_of_entry[o + i];
            T x = (T)scratch_tf[s + i] * IdfMath64<T>::idf(n1, df[c]);
            if (sum != 0.0) x = IdfMath64<T>::scale(x, norm);
            indices[o + i] = c;
            if (val64) val64[o + i] = (double)x;
            val32[o + i] = (float)x;
        }
    }
}

__global__ void tfidf64_tail_kernel(int64_t n_docs, const int64_t *__restrict__ indptr, int64_t *__restrict__ nnz_total,
                                    int32_t *__restrict__ vocab_size) {
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        *nnz_total = indptr[n_docs];
        if (indptr[n_docs] == 0) *vocab_size = 0;
    }
}

}  // namespace sg

using namespace sg;

extern "C" {

int sg_tfidf64_count(const void *symbols, int sym_width, const int64_t *offsets, int64_t n_docs, int ngram, int bits,
                     const uint8_t *lut, uint32_t *scratch_clean, uint64_t *scratch_sort, uint64_t *scratch_key,
                     uint32_t *scratch_tf, int32_t *row_nnz, void *stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (ngram < 1 || bits < 1 || (int64_t)ngram * bits > 64)
        return fail(SG_ERR_UNSUPPORTED, "ngram_size %d over %d-bit symbols needs %lld-bit keys (limit 64)", ngram, bits,
                    (long long)ngram * bits);
    if (sym_width != 1 && sym_width != 4) return fail(SG_ERR_INVALID, "sym_width must be 1 or 4");
    if (sym_width == 1 && !lut) return fail(SG_ERR_INVALID, "1-byte symbols need the 256-entry table");
    if (n_docs <= 0) return SG_OK;
    int dev = 0, n_sm = 0;
    SG_CUDA_TRY(cudaGetDevice(&dev));
    SG_CUDA_TRY(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
    int64_t grid = (n_docs + K64_WARPS - 1) / K64_WARPS;
    const int64_t cap = (int64_t)n_sm * 6;
    if (grid > cap) grid = cap;
    if (sym_width == 1)
        tfidf64_count_kernel<uint8_t><<<(unsigned)grid, K64_WARPS * 32, 0, st>>>(
            (const uint8_t *)symbols, offsets, n_docs, ngram, bits, lut, scratch_clean, scratch_sort, scratch_key,
            scratch_tf, row_nnz);
    else
        tfidf64_count_kernel<uint32_t><<<(unsigned)grid, K64_WARPS * 32, 0, st>>>(
            (const uint32_t *)symbols, offsets, n_docs, ngram, bits, lut, scratch_clean, scratch_sort, scratch_key,
            scratch_tf, row_nnz);
    SG_LAUNCH_CHECK();
    return SG_OK;
}

size_t sg_tfidf64_finalize_workspace_bytes(int64_t n_docs, int64_t total_symbols) {
    const int64_t n = total_symbols < 1 ? 1 : total_symbols;
    size_t b1 = 0, b2 = 0, b3 = 0;
    cub::DeviceScan::ExclusiveScan(nullptr, b1, (int32_t *)nullptr, (int64_t *)nullptr, cub::Sum(), (int64_t)0,
                                   n_docs + 1);
    cub::DeviceRadixSort::SortPairs(nullptr, b2, (uint64_t *)nullptr, (uint64_t *)nullptr, (uint32_t *)nullptr,
                                    (uint32_t *)nullptr, n);
    cub::DeviceScan::InclusiveSum(nullptr, b3, (int32_t *)nullptr, (int32_t *)nullptr, n);
    size_t cubb = b1 > b2 ? b1 : b2;
    cubb = cubb > b3 ? cubb : b3;
    return 2 * align_up((size_t)n * 8, 256) + 5 * align_up((size_t)(n + 2) * 4, 256) + align_up(cubb, 256) + 4096;
}

/*
 * indptr, vocabulary (sorted distinct keys -> column ids, df), values.  `bits` bounds the sort.  Outputs: indptr,
 * indices, val64 (NULL for f32), val32, vocab_keys [total_symbols] (first V entries valid), df [total_symbols]
 * (first V valid), vocab_size, nnz_total.
 */
int sg_tfidf64_finalize(const int64_t *offsets, int64_t n_docs, int64_t n_docs_fit, int64_t total_symbols, int ngram,
                        int bits, int dtype, const uint64_t *scratch_key, const uint32_t *scratch_tf, int32_t *row_nnz,
                        int64_t *indptr, int32_t *indices, double *val64, float *val32, uint64_t *vocab_keys,
                        int32_t *df, int32_t *vocab_size, int64_t *nnz_total, void *ws, size_t ws_bytes,
                        void *stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (dtype != SG_DTYPE_F32 && dtype != SG_DTYPE_F64) return fail(SG_ERR_INVALID, "bad dtype");
    if (dtype == SG_DTYPE_F64 && !val64) return fail(SG_ERR_INVALID, "val64 is required for float64");
    if (n_docs < 0 || n_docs_fit < n_docs) return fail(SG_ERR_INVALID, "need 0 <= n_docs <= n_docs_fit");
    if (total_symbols >= (int64_t)0x7fffffff) return fail(SG_ERR_OVERFLOW, "corpus too large for int32 positions");
    const int64_t n = total_symbols < 1 ? 1 : total_symbols;
    Arena ar(ws, ws_bytes);
    uint64_t *keys = ar.take<uint64_t>((size_t)n);
    uint64_t *keys_sorted = ar.take<uint64_t>((size_t)n);
    uint32_t *pos = ar.take<uint32_t>((size_t)n + 2);
    uint32_t *pos_sorted = ar.take<uint32_t>((size_t)n + 2);
    int32_t *head = ar.take<int32_t>((size_t)n + 2);
    int32_t *col_scan = ar.take<int32_t>((size_t)n + 2);
    int32_t *col_of_entry = ar.take<int32_t>((size_t)n + 2);
    size_t b1 = 0, b2 = 0, b3 = 0;
    cub::DeviceScan::ExclusiveScan(nullptr, b1, (int32_t *)nullptr, (int64_t *)nullptr, cub::Sum(), (int64_t)0,
                                   n_docs + 1);
    cub::DeviceRadixSort::SortPairs(nullptr, b2, keys, keys_sorted, pos, pos_sorted, n);
    cub::DeviceScan::InclusiveSum(nullptr, b3, head, col_scan, n);
    size_t cubb = b1 > b2 ? b1 : b2;
    cubb = cubb > b3 ? cubb : b3;
    char *tmp = ar.take<char>(cubb);
    if (!ar.ok()) return fail(SG_ERR_INVALID, "tfidf64 workspace too small (%zu < %zu)", ws_bytes, ar.off);
    // head_pos re-uses `head`'s neighbour: V + 1 <= n + 1 entries are needed after the heads were consumed
    int32_t *head_pos = reinterpret_cast<int32_t *>(pos);      // `pos` is dead once it has been sorted

    SG_CUDA_TRY(cudaMemsetAsync(row_nnz + n_docs, 0, sizeof(int32_t), st));
    SG_CUDA_TRY(cudaMemsetAsync(vocab_size, 0, sizeof(int32_t), st));
    SG_CUDA_TRY(cudaMemsetAsync(keys, 0xff, (size_t)n * 8, st));
    SG_CUDA_TRY(cudaMemsetAsync(pos, 0, (size_t)n * 4, st));
    SG_CUDA_TRY(cub::DeviceScan::ExclusiveScan(tmp, cubb, row_nnz, indptr, cub::Sum(), (int64_t)0, n_docs + 1, st));
    if (n_docs > 0) {
        tfidf64_compact_kernel<<<(unsigned)((n_docs + 7) / 8), 256, 0, st>>>(n_docs, offsets, indptr, scratch_key, keys,
                                                                           pos);
        SG_LAUNCH_CHECK();
    }
    // nnz is not known on the host (no hidden synchronisation): the sort runs over the upper bound `n`, the tail
    // beyond indptr[n_docs] holds all-ones keys (stable sort: real entries come first), the kernels read nnz on the
    // device
    tfidf64_tail_kernel<<<1, 32, 0, st>>>(n_docs, indptr, nnz_total, vocab_size);
    SG_LAUNCH_CHECK();
    if (total_symbols > 0 && n_docs > 0) {
        const int key_bits = ngram * bits > 64 ? 64 : ngram * bits;
        SG_CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp, cubb, keys, keys_sorted, pos, pos_sorted, n, 0, key_bits, st));
        const unsigned g = (unsigned)((n + 255) / 256);
        tfidf64_heads_kernel<<<g, 256, 0, st>>>(n, indptr + n_docs, keys_sorted, head);
        SG_LAUNCH_CHECK();
        SG_CUDA_TRY(cub::DeviceScan::InclusiveSum(tmp, cubb, head, col_scan, n, st));
        tfidf64_columns_kernel<<<g, 256, 0, st>>>(indptr + n_docs, keys_sorted, pos_sorted, head, col_scan, col_of_entry,
                                                  vocab_keys, head_pos, vocab_size);
        SG_LAUNCH_CHECK();
        tfidf64_df_kernel<<<g, 256, 0, st>>>(vocab_size, head_pos, df, n);
        SG_LAUNCH_CHECK();
        int dev = 0, n_sm = 0;
        SG_CUDA_TRY(cudaGetDevice(&dev));
        SG_CUDA_TRY(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
        int64_t grid = (n_docs + K64_WARPS - 1) / K64_WARPS;
        const int64_t cap = (int64_t)n_sm * 8;
        if (grid > cap) grid = cap;
        if (dtype == SG_DTYPE_F64)
            tfidf64_finalize_kernel<double><<<(unsigned)grid, K64_WARPS * 32, 0, st>>>(
                offsets, n_docs, n_docs_fit, df, col_of_entry, scratch_tf, indptr, indices, val64, val32);
        else
            tfidf64_finalize_kernel<float><<<(unsigned)grid, K64_WARPS * 32, 0, st>>>(
                offsets, n_docs, n_docs_fit, df, col_of_entry, scratch_tf, indptr, indices, nullptr, val32);
        SG_LAUNCH_CHECK();
    }
    return SG_OK;
}

}  // extern "C"
