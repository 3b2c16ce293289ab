// Exact threshold pruning of the left operand of K2, for sm_90a (SURVEY.md §8f row 4).
//
// No reference counterpart: sp_matmul_topn (call sites string_grouper/string_grouper.py:725-743)
// walks every posting of every feature of a left row.  With x = x_P + x_S (P = a set of the row's features)
//
//     x . y  =  x_P . y + x_S . y  <=  |x_P| |y| + x_S . y            (Cauchy-Schwarz)
//
// so a pair can only exceed `threshold` if its partial score over the kept features S exceeds
// threshold - |x_P| * max|y|.  Per left row the features are ranked by cost / weight^2 (cost = document
// frequency of the feature in the RIGHT matrix = postings walked for it) and the most expensive ones are
// moved into P while |x_P| * max|y| stays within `budget`: the frequent n-grams, which carry most of the
// postings and (low idf) little of the norm.  The candidate list stays a superset of the true matches; every
// candidate is re-scored exactly over ALL features (sg_rescore), so results do not change.
//
// Tighter, per column tile: when P only holds features of a fixed set H (the 64 most frequent features of the
// right matrix, sg_heavy_features),  x_P . y = x_P . y_H <= |x_P| |y_H|,  and |y_H| (sg_heavy_norms) is well
// below |y| for most rows.  The right rows are ordered by quantised |y_H| first (sg_row_order), so the
// largest |y_H| inside a column tile (sg_tile_bounds) is close to that of each of its columns and the
// candidate threshold of (row i, tile t) becomes  threshold - |x_P(i)| * bound(t).
//
// Tighter again, per candidate: H is split into 16 groups by rank — the 14 most frequent features one group each
// (what gets pruned is almost always among them, and for a group of one the bound is the product itself), ranks
// 14..38 and 39..63 one group each.  With x_P,g / y_H,g the parts of x_P / y_H in group g,
// x_P . y = sum_g x_P,g . y_H,g <= sum_g |x_P,g| |y_H,g|.  sg_prune_rows and sg_heavy_norms store the group norms
// (fp16, rounded up, 32 bytes = one sector per row); sg_rescore_refined re-tests every candidate (row i, column j)
// with  partial score > threshold(i) - sum_g |x_P,g(i)| |y_H,g(j)|  before it reads the right row.  Candidates per
// left row on the 663k benchmark (sample): tile-wide bound 501, 8 groups of 8 ranks 85, this grouping 45, pairs
// above the threshold 42 (tests/gpu_bound_stats.py).
#include <cuda_fp16.h>

#include "sg_common.cuh"

namespace sg {

constexpr int HEAVY_GROUPS = 16;
__device__ __forceinline__ int heavy_group(int rank) { return rank < 14 ? rank : (rank < 39 ? 14 : 15); }

// fp32 norm from a sum of squares, rounded up: relative and absolute slack cover the fp32 arithmetic
__device__ __forceinline__ float norm_up(float s2) { return s2 > 0.f ? sqrtf(s2) * (1.f + 1e-5f) + 1e-6f : 0.f; }

__global__ void feature_df_kernel(int64_t n_rows, const int64_t *__restrict__ indptr,
                                  const int32_t *__restrict__ indices, int32_t *__restrict__ df) {
    const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= n_rows) return;
    const int64_t p1 = indptr[row + 1];
    for (int64_t p = indptr[row] + lane_id(); p < p1; p += 32) atomicAdd(df + indices[p], 1);
}

// one warp per left row
__global__ void prune_rows_kernel(int64_t row_begin, int64_t n_rows, const int64_t *__restrict__ indptr,
                                  const int32_t *__restrict__ idx, const float *__restrict__ val,
                                  const int32_t *__restrict__ df_right, const int8_t *__restrict__ prunable,
                                  float right_norm, float budget,
                                  float threshold, float margin, float margin_per_feature,
                                  const float *__restrict__ row_floor, float frac,
                                  int32_t *__restrict__ out_idx, float *__restrict__ out_val,
                                  int32_t *__restrict__ out_len, float *__restrict__ out_thr,
                                  float *__restrict__ out_xp, __half *__restrict__ out_xg) {
    const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (r >= n_rows) return;
    const int lane = lane_id();
    const int64_t row = row_begin + r;
    const int64_t p0 = indptr[row];
    const int nf = (int)(indptr[row + 1] - p0);
    if (row_floor) {        // per-row threshold: score > max(threshold, floor - FLOOR_EPS) covers score >= floor
        threshold = fmaxf(threshold, row_floor[row] - FLOOR_EPS);
        budget = fmaxf(frac * (threshold - margin), 0.f);
    }
    // |x_P| <= budget / max|y|
    const float lim = right_norm > 0.f ? budget / right_norm : 0.f;
    const float lim2 = lim * lim;
    int kept = 0;
    float norm_p2 = 0.f;
    float group_p2 = 0.f;      // lanes 0..15: squared norm of the pruned features of group `lane`
    for (int base = 0; base < nf; base += 32) {
        const int k = base + lane;
        float my_key = -1.f, my_w2 = 0.f, my_v = 0.f;
        int my_f = 0;
        if (k < nf) {
            my_f = idx[p0 + k];
            my_v = val[p0 + k];
            my_w2 = my_v * my_v;
            // cost per unit of squared norm; features nobody on the right holds cost nothing and stay,
            // and so do features outside the prunable set (key 0 = never pruned)
            my_key = (my_w2 > 0.f && (!prunable || prunable[my_f] >= 0)) ? (float)df_right[my_f] / my_w2 : 0.f;
        }
        // squared norm of everything ranked before feature k (larger key first, ties by position)
        float before = 0.f;
        for (int jb = 0; jb < nf; jb += 32) {
            const int j = jb + lane;
            float o_key = -1.f, o_w2 = 0.f;
            if (jb == base) {
                o_key = my_key;
                o_w2 = my_w2;
            } else if (j < nf) {
                const float v = val[p0 + j];
                const int f = idx[p0 + j];
                o_w2 = v * v;
                o_key = (o_w2 > 0.f && (!prunable || prunable[f] >= 0)) ? (float)df_right[f] / o_w2 : 0.f;
            }
            const int lim_s = nf - jb < 32 ? nf - jb : 32;
            for (int s = 0; s < lim_s; ++s) {
                const float kk = __shfl_sync(FULL, o_key, s);
                const float ww = __shfl_sync(FULL, o_w2, s);
                if (kk > my_key || (kk == my_key && jb + s < k)) before += ww;
            }
        }
        const bool in_p = k < nf && my_key > 0.f && before + my_w2 <= lim2;
        const bool keep = k < nf && !in_p;
        const unsigned km = __ballot_sync(FULL, keep);
        if (keep) {
            const int64_t w = p0 + kept + __popc(km & ((1u << lane) - 1u));
            out_idx[w] = my_f;
            out_val[w] = my_v;
        }
        kept += __popc(km);
        if (out_xg) {          // pruned features are few: one at a time, the lane of its group adds it
            const int my_g = in_p ? heavy_group((int)prunable[my_f]) : 0;
            unsigned pm = __ballot_sync(FULL, in_p);
            while (pm) {
                const int j = __ffs(pm) - 1;
                pm &= pm - 1;
                const float w2 = __shfl_sync(FULL, my_w2, j);
                if (lane == __shfl_sync(FULL, my_g, j)) group_p2 += w2;
            }
        }
        float s = in_p ? my_w2 : 0.f;
#pragma unroll
        for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(FULL, s, o);
        norm_p2 += s;
    }
    if (lane == 0) {
        out_len[row] = kept;
        // the rounding of the fp32 norm arithmetic is covered by the relative and absolute slack
        const float xp = norm_up(norm_p2);
        const float thr = threshold - margin - margin_per_feature * (float)kept;
        out_thr[row] = thr > 0.f ? thr : 0.f;
        out_xp[row] = xp;
    }
    if (out_xg && lane < HEAVY_GROUPS) out_xg[row * HEAVY_GROUPS + lane] = __float2half_ru(norm_up(group_p2));
}

// norm of every row restricted to the heavy features (hrank >= 0), rounded up; one warp per row
__global__ void heavy_norms_kernel(int64_t row_begin, int64_t n_rows, const int64_t *__restrict__ indptr,
                                   const int32_t *__restrict__ idx, const float *__restrict__ val,
                                   const int8_t *__restrict__ hrank, float *__restrict__ out,
                                   __half *__restrict__ out_g) {
    const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (r >= n_rows) return;
    const int lane = lane_id();
    const int64_t row = row_begin + r;
    const int64_t p1 = indptr[row + 1];
    float s = 0.f;
    float group2 = 0.f;        // lanes 0..15: squared norm over the heavy features of group `lane`
    for (int64_t base = indptr[row]; base < p1; base += 32) {
        const int64_t p = base + lane;
        int h = -1;
        float w2 = 0.f;
        if (p < p1) {
            h = hrank[idx[p]];
            if (h >= 0) {
                w2 = val[p] * val[p];
                s = fmaf(val[p], val[p], s);
            }
        }
        if (out_g) {
            unsigned hm = __ballot_sync(FULL, h >= 0);
            while (hm) {
                const int j = __ffs(hm) - 1;
                hm &= hm - 1;
                const float o2 = __shfl_sync(FULL, w2, j);
                if (lane == heavy_group(__shfl_sync(FULL, h, j))) group2 += o2;
            }
        }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(FULL, s, o);
    if (lane == 0) out[r] = norm_up(s);
    if (out_g && lane < HEAVY_GROUPS) out_g[r * HEAVY_GROUPS + lane] = __float2half_ru(norm_up(group2));
}

// bound[t] = largest heavy norm among the right rows at positions [t*W, (t+1)*W) of the processing order
__global__ void tile_bounds_kernel(int64_t n_right, const int32_t *__restrict__ perm,
                                   const float *__restrict__ row_norm, int W, float *__restrict__ bound) {
    const int64_t t = blockIdx.x;
    const int64_t p0 = t * W;
    const int64_t p1 = p0 + W < n_right ? p0 + W : n_right;
    float m = 0.f;
    for (int64_t p = p0 + threadIdx.x; p < p1; p += blockDim.x) m = fmaxf(m, row_norm[perm ? perm[p] : p]);
    __shared__ float part[32];
#pragma unroll
    for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(FULL, m, o));
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x < 32) {
        m = threadIdx.x < (blockDim.x >> 5) ? part[threadIdx.x] : 0.f;
#pragma unroll
        for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(FULL, m, o));
        if (threadIdx.x == 0) bound[t] = m;
    }
}

}  // namespace sg

using namespace sg;

extern "C" {

int sg_feature_df(int64_t n_rows, int64_t n_cols, const int64_t *indptr, const int32_t *indices, int32_t *df,
                  void *stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (n_cols <= 0) return SG_OK;
    SG_CUDA_TRY(cudaMemsetAsync(df, 0, (size_t)n_cols * sizeof(int32_t), st));
    if (n_rows > 0) {
        feature_df_kernel<<<(unsigned)((n_rows + 7) / 8), 256, 0, st>>>(n_rows, indptr, indices, df);
        SG_LAUNCH_CHECK();
    }
    return SG_OK;
}

int sg_prune_rows(int64_t row_begin, int64_t row_end, const int64_t *indptr, const int32_t *indices,
                  const float *val32, const int32_t *df_right, const int8_t *prunable, float right_norm,
                  float budget, float threshold, float margin, float margin_per_feature, int32_t *out_indices,
                  float *out_val32, int32_t *out_len, float *out_threshold, float *out_pruned_norm,
                  void *out_group_norms, void *stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    const int64_t n = row_end - row_begin;
    if (n <= 0) return SG_OK;
    if (!(budget >= 0.f) || !(right_norm >= 0.f)) return fail(SG_ERR_INVALID, "budget and right_norm must be >= 0");
    if (out_group_norms && !prunable) return fail(SG_ERR_INVALID, "group norms need the heavy-feature ranks");
    prune_rows_kernel<<<(unsigned)((n + 7) / 8), 256, 0, st>>>(row_begin, n, indptr, indices, val32, df_right,
                                                              prunable, right_norm, budget, threshold, margin,
                                                              margin_per_feature, nullptr, 0.f, out_indices,
                                                              out_val32, out_len, out_threshold, out_pruned_norm,
                                                              (__half *)out_group_norms);
    SG_LAUNCH_CHECK();
    return SG_OK;
}

int sg_prune_rows_floor(int64_t row_begin, int64_t row_end, const int64_t *indptr, const int32_t *indices,
                        const float *val32, const int32_t *df_right, const int8_t *prunable, float right_norm,
                        float frac, float threshold, const float *row_floor, float margin, float margin_per_feature,
                        int32_t *out_indices, float *out_val32, int32_t *out_len, float *out_threshold,
                        float *out_pruned_norm, void *out_group_norms, void *stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    const int64_t n = row_end - row_begin;
    if (n <= 0) return SG_OK;
    if (!row_floor) return fail(SG_ERR_INVALID, "row_floor is required");
    if (!(frac >= 0.f) || !(frac < 1.f) || !(right_norm >= 0.f))
        return fail(SG_ERR_INVALID, "frac must lie in [0, 1) and right_norm be >= 0");
    if (out_group_norms && !prunable) return fail(SG_ERR_INVALID, "group norms need the heavy-feature ranks");
    prune_rows_kernel<<<(unsigned)((n + 7) / 8), 256, 0, st>>>(row_begin, n, indptr, indices, val32, df_right,
                                                              prunable, right_norm, 0.f, threshold, margin,
                                                              margin_per_feature, row_floor, frac, out_indices,
                                                              out_val32, out_len, out_threshold, out_pruned_norm,
                                                              (__half *)out_group_norms);
    SG_LAUNCH_CHECK();
    return SG_OK;
}

int sg_heavy_norms(int64_t row_begin, int64_t row_end, const int64_t *indptr, const int32_t *indices,
                   const float *val32, const int8_t *hrank, float *out_norm, void *out_group_norms, void *stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    const int64_t n = row_end - row_begin;
    if (n <= 0) return SG_OK;
    heavy_norms_kernel<<<(unsigned)((n + 7) / 8), 256, 0, st>>>(row_begin, n, indptr, indices, val32, hrank,
                                                               out_norm, (__half *)out_group_norms);
    SG_LAUNCH_CHECK();
    return SG_OK;
}

int sg_tile_bounds(int64_t n_right, const int32_t *perm, const float *row_norm, int tile_w, float *bound,
                   void *stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (n_right <= 0) return SG_OK;
    if (tile_w <= 0) return fail(SG_ERR_INVALID, "tile_w must be positive");
    const int64_t T = (n_right + tile_w - 1) / tile_w;
    tile_bounds_kernel<<<(unsigned)T, 256, 0, st>>>(n_right, perm, row_norm, tile_w, bound);
    SG_LAUNCH_CHECK();
    return SG_OK;
}

}  // extern "C"
