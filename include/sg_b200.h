/*
 * sg_b200.h — C ABI of libsg_b200.so, the H100 (sm_90a) implementation of the
 * string_grouper hot path.  Plain pointers and sizes only; no torch types.
 *
 * The reference (Bergvca/string_grouper @ 270044e9, pure Python) has no FFI of
 * its own: its hot path calls scikit-learn and sparse_dot_topn.  Every entry
 * point below names the reference interface it replaces as
 * string_grouper/string_grouper.py:<line> ("sg.py:<line>").
 *
 * Conventions
 *   - every pointer marked [dev] is device memory owned by the caller
 *     (allocated through torch in the Python host side);
 *   - every call is asynchronous on `stream` (a cudaStream_t passed as void*),
 *     there are no hidden synchronisations; counters the host needs are left in
 *     device memory and the host reads them back when it chooses to;
 *   - return value: SG_OK or a negative SG_ERR_*; sg_last_error() gives the
 *     text for the calling thread; nothing throws across the ABI;
 *   - two-phase sizing: *_workspace_bytes() then the call with `ws`.
 */
#ifndef SG_B200_H
#define SG_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SG_OK 0
#define SG_ERR_INVALID (-1)     /* -> ValueError   */
#define SG_ERR_CUDA (-2)        /* -> RuntimeError */
#define SG_ERR_OVERFLOW (-3)    /* -> OverflowError (caught by fit(), sg.py:400) */
#define SG_ERR_UNSUPPORTED (-4) /* -> NotImplementedError */

#define SG_DTYPE_F32 0
#define SG_DTYPE_F64 1

/* analyzer flags for sg_tfidf_* (sg.py:365-378) */
#define SG_FLAG_IGNORE_CASE 1u   /* fold A-Z to a-z                                  */
#define SG_FLAG_STRIP_DEFAULT 2u /* delete the default regex class  [,-./]|\s         */

const char *sg_last_error(void);
int sg_abi_version(void);
/* SM count, opt-in shared memory per block, L2 bytes of the current device. */
int sg_device_info(int *sm_count, int *smem_optin_bytes, int *l2_bytes);

/* ------------------------------------------------------------------------- *
 * K1 — character n-gram TF-IDF, CSR emitted in HBM.
 * Replaces: StringGrouper.n_grams (sg.py:365-378) + TfidfVectorizer fit /
 * transform (sg.py:305-308, :685-707; sklearn text.py:_count_vocab, idf,
 * l2 normalise).  Input is the concatenation master ++ duplicates as UTF-8
 * bytes that are already pure ASCII (the Python host has run lower()/NFKD on
 * the rare non-ASCII rows, exactly sg.py:372-375), with n_docs+1 offsets.
 *
 * Phase 1 (sg_tfidf_count): per document (one warp): strip / fold bytes, pack
 * n-grams into order-preserving keys (7 bits per char, big endian), sort the
 * keys in the warp, run-length encode to (key, tf) stored at the document's
 * byte offset in scratch_key / scratch_tf, row_nnz[doc] = number of runs,
 * df_table[key] += 1 per run.  `df_table` has sg_tfidf_table_slots(ngram)
 * = 2^(7*ngram) int32 slots (1 <= ngram <= 4) and must be zeroed by the
 * caller; the four scratch arrays have total_bytes elements each
 * (scratch_clean / scratch_sort are only touched by documents longer than 256
 * characters).  row_nnz has n_docs + 1 slots.
 * ------------------------------------------------------------------------- */
int64_t sg_tfidf_table_slots(int ngram);
int sg_tfidf_count(const uint8_t *bytes /*[dev]*/, const int64_t *offsets /*[dev] n_docs+1*/,
                   int64_t n_docs, int ngram, unsigned flags, int32_t *df_table /*[dev] slots, zeroed*/,
                   uint8_t *scratch_clean /*[dev]*/, uint32_t *scratch_sort /*[dev]*/,
                   uint32_t *scratch_key /*[dev]*/, uint32_t *scratch_tf /*[dev]*/,
                   int32_t *row_nnz /*[dev] n_docs+1*/, void *stream);

/*
 * Phase 2 (sg_tfidf_vocab): exclusive scan of row_nnz -> indptr (int64);
 * exclusive scan of (df > 0) over the key table -> rank_table[key] = column id
 * = rank of the n-gram in sorted order (sklearn _sort_features).
 * `vocab_size` [dev] receives V, `nnz_total` [dev] receives indptr[n_docs].
 * The host then reads V and df in column order (sg_tfidf_vocab_df) back and
 * computes idf[V] in the matrix dtype exactly as TfidfTransformer.fit does on
 * the host (numpy's log: its result is not the device's log).
 *
 * Phase 3 (sg_tfidf_values): x = tf*idf[column] in the matrix dtype; row L2
 * norm accumulated in double in column order, IEEE sqrt and divide (sklearn
 * _inplace_csr_row_normalize_l2); writes indices, values in the matrix dtype
 * (val64 for f64, may be NULL for f32) and an fp32 copy for K2.
 * The caller sizes indices/val64/val32 with total_bytes entries (an upper
 * bound of nnz).
 */
size_t sg_tfidf_vocab_workspace_bytes(int64_t n_docs, int ngram);
int sg_tfidf_vocab(int64_t n_docs, int ngram, const int32_t *df_table /*[dev]*/, int32_t *rank_table /*[dev] slots*/,
                   int32_t *row_nnz /*[dev] n_docs+1*/, int64_t *indptr /*[dev] n_docs+1*/,
                   int32_t *vocab_size /*[dev] 1*/, int64_t *nnz_total /*[dev] 1*/, void *ws /*[dev]*/,
                   size_t ws_bytes, void *stream);
int sg_tfidf_values(const int64_t *offsets /*[dev]*/, int64_t n_docs, int dtype,
                    const void *idf /*[dev] V, matrix dtype*/, const int32_t *rank_table /*[dev]*/,
                    const uint32_t *scratch_key, const uint32_t *scratch_tf, const int32_t *row_nnz,
                    const int64_t *indptr /*[dev] n_docs+1*/, int32_t *indices /*[dev]*/,
                    double *val64 /*[dev]*/, float *val32 /*[dev]*/, void *stream);

/* keys_out[c] = packed n-gram of column c (sorted vocabulary), V entries. */
int sg_tfidf_vocab_keys(const int32_t *df_table /*[dev]*/, const int32_t *rank_table /*[dev]*/, int ngram,
                        uint32_t *keys_out /*[dev] V*/, void *stream);
/* df_out[c] = document frequency of column c over the fitted rows (TfidfVectorizer's df; equals sg_feature_df of
 * the matrix when it holds exactly the fitted rows). */
int sg_tfidf_vocab_df(const int32_t *df_table /*[dev]*/, const int32_t *rank_table /*[dev]*/, int ngram,
                      int32_t *df_out /*[dev] V*/, void *stream);

/* ------------------------------------------------------------------------- *
 * K1, general form (csrc/sg_tfidf64.cu): 64-bit n-gram keys and a sort-based vocabulary — ngram_size >= 4 and text
 * that keeps non-ASCII code points (normalize_to_ascii=False).  Same reference functions as above.
 * The host supplies an order-preserving dense alphabet: `bits` = ceil(log2(#symbols)), ngram*bits <= 64.
 *   sym_width 1: `symbols` are bytes, lut[256] maps a byte to its symbol id after case folding / stripping
 *                (0xff = deleted by the default regex);
 *   sym_width 4: `symbols` are uint32 symbol ids (the host ran lower() / regex on the code points), lut unused.
 * `offsets` count symbols.  Phase 1 writes, per document, its sorted distinct keys and term counts at the document's
 * offset in scratch_key / scratch_tf and row_nnz[doc]; scratch_clean / scratch_sort serve documents longer than 256
 * symbols.  Phase 2: indptr; ONE radix sort of all (document, key) runs -> vocabulary (vocab_keys[c] = key of column c,
 * df[c]), column ids by a scan, written to indices (sg_tfidf64_vocab).  The host reads V and df[:V] back and computes
 * idf[V] (as for sg_tfidf_vocab); sg_tfidf64_values then writes the values as sg_tfidf_values does.  No device-to-host
 * read-back inside any call.
 * ------------------------------------------------------------------------- */
int sg_tfidf64_count(const void *symbols /*[dev]*/, int sym_width, const int64_t *offsets /*[dev] n_docs+1*/,
                     int64_t n_docs, int ngram, int bits, const uint8_t *lut /*[dev] 256 or NULL*/,
                     uint32_t *scratch_clean /*[dev] total*/, uint64_t *scratch_sort /*[dev] total*/,
                     uint64_t *scratch_key /*[dev] total*/, uint32_t *scratch_tf /*[dev] total*/,
                     int32_t *row_nnz /*[dev] n_docs+1*/, void *stream);
size_t sg_tfidf64_vocab_workspace_bytes(int64_t n_docs, int64_t total_symbols);
int sg_tfidf64_vocab(const int64_t *offsets /*[dev]*/, int64_t n_docs, int64_t total_symbols, int ngram, int bits,
                     const uint64_t *scratch_key, int32_t *row_nnz, int64_t *indptr /*[dev] n_docs+1*/,
                     int32_t *indices /*[dev] total*/, uint64_t *vocab_keys /*[dev] total*/,
                     int32_t *df /*[dev] total*/, int32_t *vocab_size /*[dev] 1*/, int64_t *nnz_total /*[dev] 1*/,
                     void *ws /*[dev]*/, size_t ws_bytes, void *stream);
int sg_tfidf64_values(const int64_t *offsets /*[dev]*/, int64_t n_docs, int dtype,
                      const void *idf /*[dev] V, matrix dtype*/, const uint32_t *scratch_tf,
                      const int64_t *indptr /*[dev] n_docs+1*/, const int32_t *indices /*[dev] total*/,
                      double *val64 /*[dev] total or NULL*/, float *val32 /*[dev] total*/, void *stream);

/* ------------------------------------------------------------------------- *
 * K1 transform: new documents through a FITTED vocabulary (TfidfVectorizer.transform).  N-grams outside the
 * vocabulary are dropped, tf counts the known ones, idf and columns are the fitted ones, the L2 norm is taken after
 * the drop; a row without a known n-gram is empty.  The fitted vocabulary is only read.
 *
 * Dense form (ASCII, ngram <= 3 vocabulary of sg_tfidf_vocab):
 *   sg_tfidf_transform_count  = sg_tfidf_count without the df update;
 *   sg_tfidf_known            keeps the runs whose key has df_table[key] > 0 (compacted in place, row_nnz := kept),
 *                             indptr = exclusive scan;
 *   sg_tfidf_values           with the fitted rank_table and idf.
 * Sorted form (vocabulary of sg_tfidf64_vocab, or any vocabulary given as its sorted keys):
 *   sg_tfidf64_transform_count = sg_tfidf64_count over symbols mapped through the FITTED alphabet; a symbol outside
 *                             it is SG_SYMBOL_UNKNOWN (sym_width 4) or SG_LUT_UNKNOWN in the byte table, and no
 *                             n-gram containing it is emitted (no neighbouring id can alias a real key);
 *   sg_tfidf64_known          binary search of every run's key in vocab_keys[V] (sorted ascending), unknown runs
 *                             dropped, indptr, indices; scratch_col has total entries;
 *   sg_tfidf64_values         with the fitted idf.
 * Workspace of both *_known: sg_tfidf_transform_workspace_bytes(n_docs).
 * ------------------------------------------------------------------------- */
#define SG_SYMBOL_UNKNOWN 0xffffffffu
#define SG_LUT_UNKNOWN 0xfeu
int sg_tfidf_transform_count(const uint8_t *bytes /*[dev]*/, const int64_t *offsets /*[dev] n_docs+1*/,
                             int64_t n_docs, int ngram, unsigned flags, uint8_t *scratch_clean /*[dev]*/,
                             uint32_t *scratch_sort /*[dev]*/, uint32_t *scratch_key /*[dev]*/,
                             uint32_t *scratch_tf /*[dev]*/, int32_t *row_nnz /*[dev] n_docs+1*/, void *stream);
size_t sg_tfidf_transform_workspace_bytes(int64_t n_docs);
int sg_tfidf_known(const int64_t *offsets /*[dev]*/, int64_t n_docs, const int32_t *df_table /*[dev] slots*/,
                   uint32_t *scratch_key /*[dev]*/, uint32_t *scratch_tf /*[dev]*/, int32_t *row_nnz /*[dev] n_docs+1*/,
                   int64_t *indptr /*[dev] n_docs+1*/, void *ws /*[dev]*/, size_t ws_bytes, void *stream);
int sg_tfidf64_transform_count(const void *symbols /*[dev]*/, int sym_width, const int64_t *offsets /*[dev]*/,
                               int64_t n_docs, int ngram, int bits, const uint8_t *lut /*[dev] 256 or NULL*/,
                               uint32_t *scratch_clean, uint64_t *scratch_sort, uint64_t *scratch_key,
                               uint32_t *scratch_tf, int32_t *row_nnz /*[dev] n_docs+1*/, void *stream);
int sg_tfidf64_known(const int64_t *offsets /*[dev]*/, int64_t n_docs, const uint64_t *vocab_keys /*[dev] V*/,
                     int32_t vocab_size, const uint64_t *scratch_key /*[dev]*/, uint32_t *scratch_tf /*[dev]*/,
                     int32_t *scratch_col /*[dev] total*/, int32_t *row_nnz /*[dev] n_docs+1*/,
                     int64_t *indptr /*[dev] n_docs+1*/, int32_t *indices /*[dev] total*/, void *ws /*[dev]*/,
                     size_t ws_bytes, void *stream);

/* ------------------------------------------------------------------------- *
 * K2 — blocked CSR x CSR^T, thresholded, top-n per left row.
 * Replaces: StringGrouper._build_matches (sg.py:709-752), i.e. the
 * sp_matmul_topn block products (:737-743), the zip over right blocks (:746)
 * and the vstack over left blocks (:750).
 * ------------------------------------------------------------------------- */

/* number of column tiles for `n_right` rows at `tile_w` columns per tile; _padded: rounded up to a multiple of 64
 * (row length of bucket_maxw, length of tile_bound) */
int64_t sg_num_tiles(int64_t n_right, int tile_w);
int64_t sg_num_tiles_padded(int64_t n_right, int tile_w);

/*
 * Right matrix -> tile-major postings (the transpose that sp_matmul_topn performs on
 * `Bi.T`, sg.py:727/:738, done once and laid out for the kernel).  The right rows are taken in the
 * order `perm` (row at every position of the heavy-feature signature order, sg_row_order; NULL = input
 * order): column tile t holds positions [t*tile_w, (t+1)*tile_w), T = sg_num_tiles.  The postings of tile t lie
 * contiguously, sorted by feature; bucket (f, t) = the docs of feature f inside tile t (in no particular order).
 * A posting is 4 bytes: position - t*tile_w in the low 16 bits, the weight rounded to fp16 in the high 16 bits
 * (candidate scores only need to be within the caller's margin; every candidate is re-scored exactly).
 * `bucket_dir` receives the directory as aligned 8-byte entries {int32 start, u16 length, fp16 largest |weight| of
 * the bucket} at f*T + t (feature-major), T*(n_cols+1) of them, the form sg_cossim_candidates reads; empty buckets
 * are all zero.  `bucket_maxw` receives the largest weights again as fp16 rows, one row of sg_num_tiles_padded()
 * entries per feature (zero padded), which sg_cossim_candidates streams to skip every (left row, column tile) pair
 * whose score bound sum_f |a_f| * max|w_(f,t)| cannot reach the candidate threshold.  tile_w <= 32768.
 * A tile is sorted in shared memory by one CTA; a tile of more postings than fit there (long rows, wide tiles) is
 * sorted in global memory instead, and `n_spilled` (optional, zeroed by the caller) counts those tiles.
 * `indptr` may be a row-range view (indptr_base = indptr[0]).
 */
size_t sg_postings_workspace_bytes(int64_t nnz, int64_t n_cols, int64_t n_tiles);
int sg_postings_build(int64_t n_rows, int64_t n_cols, int64_t nnz, const int64_t *indptr /*[dev]*/,
                      const int32_t *indices /*[dev]*/, const float *val32 /*[dev]*/,
                      const int32_t *perm /*[dev] or NULL*/, int tile_w, int64_t indptr_base,
                      float w_scale /* weights are multiplied by this before the fp16 rounding (1 / largest row
                                       norm from 1 up, below it the largest power of two at most that, so that every
                                       weight lies in [-1, 1]); a nonzero weight that rounds to zero keeps the smallest
                                       fp16 subnormal instead */,
                      void *bucket_dir /*[dev] T*(n_cols+1)*8 B*/, void *bucket_maxw /*[dev] (n_cols+1)*Tp*2 B*/,
                      void *postings /*[dev] nnz*4 B*/, int32_t *n_spilled /*[dev] or NULL*/,
                      void *ws /*[dev]*/, size_t ws_bytes, void *stream);

/*
 * Exact threshold pruning of the left operand (SURVEY.md §8f row 4; no reference counterpart: sp_matmul_topn,
 * sg.py:725-743, walks every posting).  For a left row x split into a pruned part x_P and a kept part x_S,
 * x.y <= |x_P|*|y_P| + x_S.y, so only pairs whose partial score over the kept features exceeds
 * threshold - |x_P|*|y_P| can be matches.  sg_feature_df counts the document frequency of every feature
 * in the right matrix (= postings walked per use of the feature); sg_prune_rows ranks each row's prunable
 * features (`prunable[f] >= 0`, NULL = all) by df / weight^2 and prunes the most expensive ones while
 * |x_P|*right_norm <= budget.  Outputs, indexed like the inputs (absolute positions / row ids): the kept
 * features first inside the row's segment of out_indices/out_val32, out_len[row] = how many were kept,
 * out_threshold[row] = threshold - margin - margin_per_feature*kept (clamped at 0), out_pruned_norm[row] = |x_P|
 * rounded up.  With the prunable set = the heavy features of sg_heavy_features, |y_P| <= |y_H|:
 * sg_heavy_norms gives |y_H| per right row (rounded up), sg_row_order sorts the right rows by its quantisation
 * first, and sg_tile_bounds the largest |y_H| per column tile of that order; sg_cossim_candidates reports
 * (row i, column j of tile t) when the partial score exceeds out_threshold[i] - out_pruned_norm[i]*bound[t].
 * The candidate list stays a superset of the matches; sg_rescore scores every candidate over all features.
 */
int sg_feature_df(int64_t n_rows, int64_t n_cols, const int64_t *indptr /*[dev]*/, const int32_t *indices /*[dev]*/,
                  int32_t *df /*[dev] n_cols*/, void *stream);
int sg_prune_rows(int64_t row_begin, int64_t row_end, const int64_t *indptr /*[dev]*/,
                  const int32_t *indices /*[dev]*/, const float *val32 /*[dev]*/,
                  const int32_t *df_right /*[dev] n_cols*/, const int8_t *prunable /*[dev] n_cols or NULL*/,
                  float right_norm /* >= largest row norm on the right */,
                  float budget, float threshold, float margin, float margin_per_feature,
                  int32_t *out_indices /*[dev]*/, float *out_val32 /*[dev]*/, int32_t *out_len /*[dev] per row id*/,
                  float *out_threshold /*[dev] per row id*/, float *out_pruned_norm /*[dev] per row id*/,
                  void *out_group_norms /*[dev] fp16[16] per row id (32-byte aligned) or NULL: |x_P| per group of
                                          heavy ranks (csrc/sg_prune.cu: ranks 0..13 alone, 14..38, 39..63), rounded
                                          up; needs `prunable` = sg_heavy_features ranks*/,
                  void *stream);
/* sg_prune_rows with a per-row threshold: row i is pruned for t_i = max(threshold, row_floor[i] - 1e-6) (the
 * pairs that can still reach a top-n floor, sg_cossim_candidates_floor) with budget frac * (t_i - margin), and
 * out_threshold[i] = t_i - margin - margin_per_feature * kept. */
int sg_prune_rows_floor(int64_t row_begin, int64_t row_end, const int64_t *indptr /*[dev]*/,
                        const int32_t *indices /*[dev]*/, const float *val32 /*[dev]*/,
                        const int32_t *df_right /*[dev] n_cols*/, const int8_t *prunable /*[dev] n_cols or NULL*/,
                        float right_norm, float frac /* in [0, 1) */, float threshold,
                        const float *row_floor /*[dev] per row id*/, float margin, float margin_per_feature,
                        int32_t *out_indices /*[dev]*/, float *out_val32 /*[dev]*/, int32_t *out_len /*[dev]*/,
                        float *out_threshold /*[dev]*/, float *out_pruned_norm /*[dev]*/,
                        void *out_group_norms /*[dev] or NULL*/, void *stream);
int sg_heavy_norms(int64_t row_begin, int64_t row_end, const int64_t *indptr /*[dev]*/,
                   const int32_t *indices /*[dev]*/, const float *val32 /*[dev]*/, const int8_t *hrank /*[dev]*/,
                   float *out_norm /*[dev] row_end-row_begin*/,
                   void *out_group_norms /*[dev] fp16[16] per row of the range or NULL: |y_H| per group, rounded up*/,
                   void *stream);
int sg_tile_bounds(int64_t n_right, const int32_t *perm /*[dev] position -> row, or NULL*/,
                   const float *row_norm /*[dev] per row*/, int tile_w, float *bound /*[dev] n_tiles*/, void *stream);

/*
 * Candidate generation: for left rows [row_begin,row_end) stream the posting
 * buckets of the row's features into a per-warp shared-memory accumulator tile
 * (fp32 or 16-bit fixed point, `acc_dtype`), sweep each column tile and append every (row, col) whose score
 * exceeds the candidate threshold (`cand_threshold` = min_similarity - margin, clamped at 0, or the
 * row's own `cand_threshold_row[row]` when that array is given, lowered by pruned_norm_row[row] *
 * tile_bound[tile] when those are given) to the candidate list.  `a_len`
 * (optional, per row id) limits a row to its first a_len[row] stored features (sg_prune_rows).
 * `cand_count` [dev] (zeroed by the caller) ends up holding
 * the number of candidates FOUND, which may exceed `cand_cap` (then only the
 * first cand_cap were stored and the caller re-runs with a larger buffer).
 * `row_queue` [dev] (zeroed) is the dynamic work queue over (column-tile group, left row) items,
 * groups outermost, `tiles_per_group` column tiles per group (a multiple of 64, sized by the caller so that one
 * group's posting buckets stay L2-resident).
 * Triangle of a self-match: with `diag_rank` (per left row id: the row's position in the processing order of the
 * right rows, which must be the same matrix) row i only reports the columns at positions >= diag_rank[i], so every
 * unordered pair {i, j} is reported once (the pair (i, i) too); sg_rescore's `mirror_count` restores the other half.
 * `group_items` [dev] sg_num_tiles()/tiles_per_group + 1 entries (rounded up) is scratch for the work items of the
 * triangle, required with diag_rank.
 * Block-max test: a (row, column tile) pair is walked only if sum_f |a_f| * max|w_(f,t)| over ALL the row's kept
 * features (bucket_maxw, fp16, rounded up) can reach the pair's threshold.  The bound and the thresholds it is
 * tested against are both multiplied by `b_scale` (a power of two in (0, 1]: 1 / a power of two at or above
 * left norm * right norm, 1 for rows of norm <= 1), so that the bound's fp16 arithmetic works on values below 2.
 */
#define SG_ACC_F32 0
#define SG_ACC_U16 1 /* 1/32768 fixed point: caller adds 2e-5 per kept feature to the margin; weights >= 0, scores < 2 */
int sg_cossim_candidates(const int64_t *a_indptr /*[dev]*/, const int32_t *a_len /*[dev] or NULL*/,
                         const int32_t *a_indices /*[dev]*/,
                         const float *a_val32 /*[dev]*/, int64_t row_begin, int64_t row_end,
                         const int32_t *perm_a /*[dev] processing order of the left rows, or NULL*/,
                         int64_t n_right, int64_t n_cols, const void *bucket_dir /*[dev] directory entries*/,
                         const void *bucket_maxw /*[dev] fp16 rows of largest weights*/,
                         const void *postings /*[dev]*/,
                         const int32_t *perm_b /*[dev] position -> right row id, or NULL*/, int tile_w,
                         int acc_dtype,
                         float a_scale /* left weights are multiplied by this: the inverse of w_scale */,
                         float b_scale /* units of the block-max bound, see above */,
                         float cand_threshold, const float *cand_threshold_row /*[dev] per row id, or NULL*/,
                         const float *pruned_norm_row /*[dev] per row id, or NULL*/,
                         const float *tile_bound /*[dev] sg_num_tiles_padded() entries, zero padded*/,
                         int64_t tiles_per_group, const int32_t *diag_rank /*[dev] per left row id, or NULL*/,
                         unsigned long long *group_items /*[dev] scratch, with diag_rank*/,
                         int32_t *cand_row /*[dev] cap*/,
                         int32_t *cand_col /*[dev] cap*/,
                         float *cand_partial /*[dev] cap or NULL: the candidate's partial score over the kept features
                                               as accumulated (input of sg_rescore_refined)*/,
                         int64_t cand_cap,
                         unsigned long long *cand_count /*[dev] 1*/,
                         unsigned long long *row_queue /*[dev] 1*/, int warps_per_cta, void *stream);
/*
 * sg_cossim_candidates with a top-n floor (1 <= top_n <= 32, non-negative weights, warps_per_cta = 8, no triangle).
 * `row_floor` [dev, per left row id, float, zeroed before the first launch of a product] holds a proven lower bound
 * of the exact score of each row's top_n-th best pair and only rises.  A pair is reported when its partial score
 * exceeds max(threshold of the row, row_floor[row] - 1e-6 - E_r) - pruned_norm_row[row] * tile_bound[tile], with
 * E_r = floor_margin + floor_margin_per_feature * (kept features): the same margins the caller subtracted from the
 * row thresholds, which also bound how far a partial score can EXCEED the kept-feature product.  Every work item
 * keeps the best 32 values (partial - E_r, rounded down) of the pairs it reported and, once it holds top_n of them,
 * raises row_floor[row] to the top_n-th with atomicMax; the floor is read again at every batch of 64 column tiles.
 * Self-match (`self_rank` [dev] per row id: the row's position in the common processing order, perm_a the same
 * order): `flags` & SG_FLOOR_SEED walks only the column-tile group holding the row, starting at the 64-tile batch that
 * holds it; without it every other group.  self_rank = NULL: every group (two matrices).
 * `flags` & SG_FLOOR_LONG_ROWS is accepted and changes nothing: every candidates kernel bounds rows of more than 32
 * kept features by the block-max test over all their features.
 */
#define SG_FLOOR_SEED 1
#define SG_FLOOR_LONG_ROWS 2
int sg_cossim_candidates_floor(const int64_t *a_indptr /*[dev]*/, const int32_t *a_len /*[dev] or NULL*/,
                               const int32_t *a_indices /*[dev]*/, const float *a_val32 /*[dev]*/,
                               int64_t row_begin, int64_t row_end, const int32_t *perm_a /*[dev] or NULL*/,
                               int64_t n_right, int64_t n_cols, const void *bucket_dir /*[dev]*/,
                               const void *bucket_maxw /*[dev]*/, const void *postings /*[dev]*/,
                               const int32_t *perm_b /*[dev] or NULL*/, int tile_w, int acc_dtype, float a_scale,
                               float b_scale, float cand_threshold,
                               const float *cand_threshold_row /*[dev] per row id, or NULL*/,
                               const float *pruned_norm_row /*[dev] per row id, or NULL*/,
                               const float *tile_bound /*[dev]*/, int64_t tiles_per_group,
                               int32_t *cand_row /*[dev] cap*/, int32_t *cand_col /*[dev] cap*/,
                               float *cand_partial /*[dev] cap or NULL*/, int64_t cand_cap,
                               unsigned long long *cand_count /*[dev] 1*/, unsigned long long *row_queue /*[dev] 1*/,
                               int warps_per_cta, float *row_floor /*[dev] per left row id*/, int top_n,
                               float floor_margin, float floor_margin_per_feature,
                               const int32_t *self_rank /*[dev] per row id, or NULL*/, int flags, void *stream);
/*
 * sg_cossim_candidates over a position range per left row (warps_per_cta = 8): row i reports only the columns at
 * positions [lo_pos[i], hi_pos[i]) of the right processing order (`perm_b`), so a product restricted to pairs that
 * share a block id sorts both sides by (block id, row order) and passes the row's block as its range; in a
 * self-match lo_pos[i] is the row's own position (the triangle, as diag_rank).  Tiles wholly outside the range leave
 * the block-max test, the columns outside it are not reported, and no work item is handed out for a column-tile group
 * the range does not reach.  Work items are exact when lo_pos and hi_pos do not decrease along perm_a.
 * `group_items` [dev] scratch of 2 * (sg_num_tiles()/tiles_per_group, rounded up) + 1 entries.
 */
int sg_cossim_candidates_range(const int64_t *a_indptr /*[dev]*/, const int32_t *a_len /*[dev] or NULL*/,
                               const int32_t *a_indices /*[dev]*/, const float *a_val32 /*[dev]*/,
                               int64_t row_begin, int64_t row_end, const int32_t *perm_a /*[dev] or NULL*/,
                               int64_t n_right, int64_t n_cols, const void *bucket_dir /*[dev]*/,
                               const void *bucket_maxw /*[dev]*/, const void *postings /*[dev]*/,
                               const int32_t *perm_b /*[dev] or NULL*/, int tile_w, int acc_dtype, float a_scale,
                               float b_scale, float cand_threshold,
                               const float *cand_threshold_row /*[dev] per row id, or NULL*/,
                               const float *pruned_norm_row /*[dev] per row id, or NULL*/,
                               const float *tile_bound /*[dev]*/, int64_t tiles_per_group,
                               const int32_t *lo_pos /*[dev] per left row id*/,
                               const int32_t *hi_pos /*[dev] per left row id*/,
                               unsigned long long *group_items /*[dev] scratch*/, int32_t *cand_row /*[dev] cap*/,
                               int32_t *cand_col /*[dev] cap*/, float *cand_partial /*[dev] cap or NULL*/,
                               int64_t cand_cap, unsigned long long *cand_count /*[dev] 1*/,
                               unsigned long long *row_queue /*[dev] 1*/, int warps_per_cta, void *stream);
/*
 * sg_cossim_candidates_range with the top-n floor of sg_cossim_candidates_floor (the keyed arg-max: 1 <= top_n <= 32,
 * non-negative weights, warps_per_cta = 8, no triangle, so lo_pos is the start of the row's block).  Floors rise only
 * from the pairs inside each row's range.  Self-match (`self_rank` [dev] per row id: the row's position in the blocked
 * order of the right rows, which lies in [lo_pos, hi_pos) of the row): `flags` & SG_FLOOR_SEED walks only the
 * column-tile group holding that position, from the 128-tile pass holding it, and leaves `group_items` untouched;
 * without it every other group the range reaches.  self_rank = NULL: every group the range reaches.
 */
int sg_cossim_candidates_range_floor(const int64_t *a_indptr /*[dev]*/, const int32_t *a_len /*[dev] or NULL*/,
                                     const int32_t *a_indices /*[dev]*/, const float *a_val32 /*[dev]*/,
                                     int64_t row_begin, int64_t row_end, const int32_t *perm_a /*[dev] or NULL*/,
                                     int64_t n_right, int64_t n_cols, const void *bucket_dir /*[dev]*/,
                                     const void *bucket_maxw /*[dev]*/, const void *postings /*[dev]*/,
                                     const int32_t *perm_b /*[dev] or NULL*/, int tile_w, int acc_dtype,
                                     float a_scale, float b_scale, float cand_threshold,
                                     const float *cand_threshold_row /*[dev] per row id, or NULL*/,
                                     const float *pruned_norm_row /*[dev] per row id, or NULL*/,
                                     const float *tile_bound /*[dev]*/, int64_t tiles_per_group,
                                     const int32_t *lo_pos /*[dev] per left row id*/,
                                     const int32_t *hi_pos /*[dev] per left row id*/,
                                     unsigned long long *group_items /*[dev] scratch*/,
                                     int32_t *cand_row /*[dev] cap*/, int32_t *cand_col /*[dev] cap*/,
                                     float *cand_partial /*[dev] cap or NULL*/, int64_t cand_cap,
                                     unsigned long long *cand_count /*[dev] 1*/,
                                     unsigned long long *row_queue /*[dev] 1*/, int warps_per_cta,
                                     float *row_floor /*[dev] per left row id*/, int top_n, float floor_margin,
                                     float floor_margin_per_feature,
                                     const int32_t *self_rank /*[dev] per row id, or NULL*/, int flags, void *stream);

/* ------------------------------------------------------------------------- *
 * K2, tile-centric form (csrc/sg_tiles.cu) — the default for L2-normalised non-negative matrices (K1 output).
 * Replaces the same block loop (sg.py:734-750): the reference slices the right matrix into row blocks `Bs`
 * (:735) and runs one sp_matmul_topn per (left block, right block) pair (:737-743); here a right block is a
 * "column tile" of 256 rows in processing order whose inverted index (postings sorted by feature, a bitmap
 * directory over the features present, bucket offsets) is ONE contiguous blob that the candidates kernel
 * copies into shared memory with cp.async.bulk (TMA) and an mbarrier.  Products are integers
 * a_q*w_q (weights in 2^-15 units, rounded to nearest: the caller adds 2^-15 per kept feature to its margin).
 *
 *   sg_tiles_build       right matrix -> tile_desc[T] (16 B each), blob, bucket_maxw (fp16 block maxima, same
 *                        layout as sg_postings_build), maxima[2] = {largest blob bytes, largest posting count}
 *   sg_tiles_pack_left   pruned left rows (sg_prune_rows) in processing order `perm` -> lpack {feature, a_q}
 *                        at the rows' own CSR positions, rowinfo[rank] = {start, kept, threshold, pruned norm}
 *   sg_tiles_filter      block-max test of every (left rank, tile): mask[word*mask_stride + rank], the 64 tiles
 *                        [64b, 64b+64) in words 2b (even tiles) and 2b+1 (odd tiles), bit (tile & 63) >> 1
 *   sg_tiles_candidates  persistent CTAs over (tile, rank segment) items from `queue` [dev, zeroed]; reports
 *                        (row, col) in original ids; cand_count as in sg_cossim_candidates; `walk_stats`
 *                        [dev, 2 x u64, optional]: (row, tile) pairs taken and postings added
 * Triangle of a self-match as in sg_cossim_candidates: with `diag_rank` (per left row id; needs `perm`) the filter
 * sets no bit for a tile below the one holding diag_rank[row] and writes the smallest such tile of every 32 ranks
 * to `diag_tile_min` [dev, mask_stride / 32 entries]; sg_tiles_candidates (same diag_rank and diag_tile_min, which
 * it overwrites) skips the (tile, segment) items below all rows of the segment and drops the columns before
 * diag_rank[row].
 * Limits: n_cols <= sg_tiles_max_cols(); one tile's blob must fit shared memory (else SG_ERR_UNSUPPORTED and
 * the caller falls back to sg_cossim_candidates).
 * ------------------------------------------------------------------------- */
int sg_tiles_tile_w(void);
int64_t sg_tiles_max_cols(void);
int64_t sg_tiles_blob_bound(int64_t nnz, int64_t n_rows, int64_t n_cols);
size_t sg_tiles_workspace_bytes(int64_t nnz, int64_t n_rows, int64_t n_cols);
int sg_tiles_build(int64_t n_rows, int64_t n_cols, int64_t nnz, const int64_t *indptr /*[dev]*/,
                   const int32_t *indices /*[dev]*/, const float *val32 /*[dev]*/,
                   const int32_t *rank /*[dev] or NULL*/, int64_t indptr_base, float w_scale,
                   void *tile_desc /*[dev] T*16 B*/, void *blob /*[dev] blob_cap B*/, int64_t blob_cap,
                   void *bucket_maxw /*[dev] (n_cols+1)*Tp*2 B*/, int32_t *maxima /*[dev] 2*/, void *ws /*[dev]*/,
                   size_t ws_bytes, void *stream);
int sg_tiles_pack_left(int64_t n_ranks, const int32_t *perm /*[dev] or NULL*/, int64_t row_begin,
                       const int64_t *indptr /*[dev]*/, const int32_t *pruned_len /*[dev] per row id or NULL*/,
                       const int32_t *pruned_indices /*[dev]*/, const float *pruned_val32 /*[dev]*/,
                       const float *threshold_row /*[dev] per row id*/,
                       const float *pruned_norm_row /*[dev] per row id or NULL*/, float a_scale,
                       void *lpack /*[dev] 8 B per stored value*/, void *rowinfo /*[dev] 16 B per rank*/,
                       void *stream);
int64_t sg_tiles_mask_words(int64_t n_right);
int sg_tiles_filter(int64_t n_ranks, const void *rowinfo /*[dev]*/, const void *lpack /*[dev]*/,
                    const void *bucket_maxw /*[dev]*/, int64_t n_right, const float *tile_bound /*[dev]*/,
                    const int32_t *perm /*[dev] as given to sg_tiles_pack_left, or NULL*/,
                    const int32_t *diag_rank /*[dev] per row id, or NULL*/,
                    uint32_t *diag_tile_min /*[dev] mask_stride/32, with diag_rank*/,
                    uint32_t *mask /*[dev] words*mask_stride*/, int64_t mask_stride, void *stream);
size_t sg_tiles_smem_bytes(int stage_bytes, int warps_per_cta);
int sg_tiles_candidates(const int32_t *perm_a /*[dev] or NULL*/, int64_t n_ranks, int64_t row_begin,
                        const void *rowinfo /*[dev]*/, const void *lpack /*[dev]*/, const uint32_t *mask /*[dev]*/,
                        int64_t mask_stride, const void *tile_desc /*[dev]*/, const void *blob /*[dev]*/,
                        int64_t n_right, int64_t n_cols, const float *tile_bound /*[dev]*/,
                        const int32_t *perm_b /*[dev] or NULL*/, const int32_t *diag_rank /*[dev] or NULL*/,
                        uint32_t *diag_tile_min /*[dev] from sg_tiles_filter, with diag_rank*/,
                        int stage_bytes /* maxima[0] */,
                        int32_t *cand_row /*[dev] cap*/, int32_t *cand_col /*[dev] cap*/, int64_t cand_cap,
                        unsigned long long *cand_count /*[dev] 1*/, unsigned long long *queue /*[dev] 1*/,
                        unsigned long long *walk_stats /*[dev] 2 or NULL*/, int warps_per_cta, void *stream);

/*
 * Exact re-scoring of the candidates: sorted-merge dot product of left row i
 * and right row j in ascending feature order (the accumulation order of
 * sp_matmul_topn) in the matrix dtype (f64 default, sg.py:18), multiply and
 * add rounded separately (no FMA contraction) so that scores equal the CPU
 * path bit for bit.  With `keep_count` == NULL score_out[i] is the score of candidate i.  Otherwise only the
 * candidates scoring strictly above `keep_threshold` (sg.py:729/:740) are kept, compacted in no particular
 * order into (keep_row, keep_col, score_out), and *keep_count [dev] (zeroed by the caller) receives their number.
 * Mirror (`mirror_count` [dev, zeroed] or NULL; needs keep_count): the candidates are the triangle of a self-match
 * (sg_cossim_candidates with diag_rank, left = right matrix); every kept (r, c) with r != c is also written as (c, r)
 * with the same score (bit-equal: the merge adds the same products in the same order), counted in *keep_count
 * and in *mirror_count, and row_cnt counts it for row c.  The keep buffers then need 2 * n_cand entries.
 */
int sg_rescore(int64_t n_cand, const int32_t *cand_row, const int32_t *cand_col,
               const int64_t *a_indptr, const int32_t *a_indices, const void *a_val,
               const int64_t *b_indptr, const int32_t *b_indices, const void *b_val, int dtype,
               double *score_out /*[dev] n_cand*/, double keep_threshold, int32_t *keep_row /*[dev] n_cand or NULL*/,
               int32_t *keep_col /*[dev] n_cand or NULL*/, unsigned long long *keep_count /*[dev] 1 or NULL*/,
               unsigned long long *mirror_count /*[dev] 1 or NULL*/,
               int32_t *row_cnt /*[dev] per left row - row_begin, zeroed by the caller, or NULL: += kept per row*/,
               int64_t row_begin, void *stream);
/* sg_rescore behind the per-candidate grouped bound of csrc/sg_prune.cu: candidate i = (r, c) is only scored when
 *   cand_partial[i] + sum_g left_group_norms[r][g] * right_group_norms[c][g]  >  row_threshold[r]
 * (partial score from sg_cossim_candidates, group norms from sg_prune_rows / sg_heavy_norms, row_threshold =
 * sg_prune_rows' out_threshold): the others cannot reach the threshold and their right rows are never read.  Same
 * kept set and scores as sg_rescore on the same candidates.  *refined_count [dev] (zeroed, or NULL) += candidates that
 * were scored.  keep_count / keep_row / keep_col are required; `mirror_count` as in sg_rescore. */
int sg_rescore_refined(int64_t n_cand, const int32_t *cand_row, const int32_t *cand_col,
                       const float *cand_partial /*[dev] n_cand*/,
                       const void *left_group_norms /*[dev] fp16[16] per left row id*/,
                       const void *right_group_norms /*[dev] fp16[16] per right row id*/,
                       const float *row_threshold /*[dev] per left row id*/,
                       const int64_t *a_indptr, const int32_t *a_indices, const void *a_val,
                       const int64_t *b_indptr, const int32_t *b_indices, const void *b_val, int dtype,
                       double *score_out /*[dev] n_cand*/, double keep_threshold, int32_t *keep_row /*[dev] n_cand*/,
                       int32_t *keep_col /*[dev] n_cand*/, unsigned long long *keep_count /*[dev] 1*/,
                       unsigned long long *refined_count /*[dev] 1 or NULL*/,
                       unsigned long long *mirror_count /*[dev] 1 or NULL*/,
                       int32_t *row_cnt /*[dev] or NULL*/, int64_t row_begin, void *stream);
/* Top-n floor of the re-score (see sg_cossim_candidates_floor): a pair is kept only if its score is > keep_threshold
 * AND >= row_floor[r].  Every row keeps at least top_n pairs at or above its floor, so the selection that follows
 * returns the same output.  *floor_dropped [dev, zeroed, or NULL] += pairs above keep_threshold the floor removed.
 * sg_rescore_refined_floor also raises the grouped bound's threshold to
 * max(row_threshold[r], row_floor[r] - 1e-6 - (floor_margin + floor_margin_per_feature * row_len[r])), with the
 * margins and row_len (sg_prune_rows' out_len) the candidates were generated with.  No mirror. */
int sg_rescore_floor(int64_t n_cand, const int32_t *cand_row, const int32_t *cand_col,
                     const int64_t *a_indptr, const int32_t *a_indices, const void *a_val,
                     const int64_t *b_indptr, const int32_t *b_indices, const void *b_val, int dtype,
                     double *score_out /*[dev] n_cand*/, double keep_threshold, int32_t *keep_row /*[dev] n_cand*/,
                     int32_t *keep_col /*[dev] n_cand*/, unsigned long long *keep_count /*[dev] 1*/,
                     int32_t *row_cnt /*[dev] or NULL*/, int64_t row_begin,
                     const float *row_floor /*[dev] per left row id*/,
                     unsigned long long *floor_dropped /*[dev] 1 or NULL*/, void *stream);
int sg_rescore_refined_floor(int64_t n_cand, const int32_t *cand_row, const int32_t *cand_col,
                             const float *cand_partial /*[dev] n_cand*/,
                             const void *left_group_norms /*[dev] fp16[16] per left row id*/,
                             const void *right_group_norms /*[dev] fp16[16] per right row id*/,
                             const float *row_threshold /*[dev] per left row id*/,
                             const int64_t *a_indptr, const int32_t *a_indices, const void *a_val,
                             const int64_t *b_indptr, const int32_t *b_indices, const void *b_val, int dtype,
                             double *score_out /*[dev] n_cand*/, double keep_threshold,
                             int32_t *keep_row /*[dev] n_cand*/, int32_t *keep_col /*[dev] n_cand*/,
                             unsigned long long *keep_count /*[dev] 1*/,
                             unsigned long long *refined_count /*[dev] 1 or NULL*/,
                             int32_t *row_cnt /*[dev] or NULL*/, int64_t row_begin,
                             const float *row_floor /*[dev] per left row id*/,
                             const int32_t *row_len /*[dev] per left row id*/, float floor_margin,
                             float floor_margin_per_feature, unsigned long long *floor_dropped /*[dev] 1 or NULL*/,
                             void *stream);
/* Arg-max re-score (match_nearest): per left row the right row of the largest exact score, without a top-n
 * selection.  row_best[r - row_begin] [dev, zeroed by the caller before the first launch, kept across launches] holds
 * the order-preserving bits of the largest score > keep_threshold (and >= row_floor[r] when row_floor is set) row r
 * has met (atomicMax).  A pair is written to (keep_row, keep_col, score_out) only if its score is at least that
 * running best, so every pair equal to the row's final best is written (the best only rises) and
 * sg_nearest_master(nnz, keep_col, keep_row, score, n_rows, ...) over the written pairs gives the lowest column
 * among them.  *keep_count [dev] += pairs written.  The floor arguments are those of sg_rescore_floor /
 * sg_rescore_refined_floor (row_floor NULL: none); the refined form re-tests candidates as sg_rescore_refined.
 * No mirror, no row counts. */
int sg_rescore_nearest(int64_t n_cand, const int32_t *cand_row, const int32_t *cand_col,
                       const int64_t *a_indptr, const int32_t *a_indices, const void *a_val,
                       const int64_t *b_indptr, const int32_t *b_indices, const void *b_val, int dtype,
                       double *score_out /*[dev] n_cand*/, double keep_threshold, int32_t *keep_row /*[dev] n_cand*/,
                       int32_t *keep_col /*[dev] n_cand*/, unsigned long long *keep_count /*[dev] 1*/,
                       unsigned long long *row_best /*[dev] per left row - row_begin*/, int64_t row_begin,
                       const float *row_floor /*[dev] per left row id, or NULL*/,
                       unsigned long long *floor_dropped /*[dev] 1 or NULL*/, void *stream);
int sg_rescore_refined_nearest(int64_t n_cand, const int32_t *cand_row, const int32_t *cand_col,
                               const float *cand_partial /*[dev] n_cand*/,
                               const void *left_group_norms /*[dev] fp16[16] per left row id*/,
                               const void *right_group_norms /*[dev] fp16[16] per right row id*/,
                               const float *row_threshold /*[dev] per left row id*/,
                               const int64_t *a_indptr, const int32_t *a_indices, const void *a_val,
                               const int64_t *b_indptr, const int32_t *b_indices, const void *b_val, int dtype,
                               double *score_out /*[dev] n_cand*/, double keep_threshold,
                               int32_t *keep_row /*[dev] n_cand*/, int32_t *keep_col /*[dev] n_cand*/,
                               unsigned long long *keep_count /*[dev] 1*/,
                               unsigned long long *refined_count /*[dev] 1 or NULL*/,
                               unsigned long long *row_best /*[dev] per left row - row_begin*/, int64_t row_begin,
                               const float *row_floor /*[dev] per left row id, or NULL*/,
                               const int32_t *row_len /*[dev] per left row id, with row_floor*/, float floor_margin,
                               float floor_margin_per_feature, unsigned long long *floor_dropped /*[dev] 1 or NULL*/,
                               void *stream);

/*
 * Per-row selection: keep score > threshold (strict, sg.py:729/:740), at most
 * top_n per left row (largest first; ties: smaller column first), rows are
 * emitted in ascending order, entries inside a row by descending score
 * (sort=True, sg.py:730/:741).  Row ids are relative to `row_begin`.
 * Outputs: out_indptr (int64, n_rows+1), out_row/out_col/out_score with
 * capacity n_cand; `out_nnz` [dev] and `out_max_row` [dev] (= the value of
 * fit()'s _true_max_n_matches, sg.py:417).
 */
size_t sg_topn_select_workspace_bytes(int64_t n_cand, int64_t n_rows);
int sg_topn_select(int64_t n_cand, const int32_t *cand_row, const int32_t *cand_col,
                   const double *score, int64_t row_begin, int64_t n_rows, int top_n,
                   double threshold, int64_t *out_indptr, int32_t *out_row, int32_t *out_col,
                   double *out_score, int64_t *out_nnz /*[dev] 1*/, int32_t *out_max_row /*[dev] 1*/,
                   void *ws, size_t ws_bytes, void *stream);

/*
 * The same selection without global sorts (csrc/sg_select.cu): the survivors (already strictly above the threshold,
 * counted per row by sg_rescore's `row_cnt`) are bucketed by row; rows of up to 32 survivors are ranked by one warp
 * with a shuffle bitonic network, rows of up to 512 by one warp in shared memory, longer rows by one CTA in pieces of
 * sg_topn_rows_cap() with the best top_n carried along.  Valid when sg_row_count_max() <= sg_topn_rows_cap() or
 * top_n <= sg_topn_rows_cap() / 2; otherwise the caller uses sg_topn_select.  Same outputs and tie rule.
 */
int sg_topn_rows_cap(void);
int sg_row_count_max(int64_t n_rows, const int32_t *row_cnt /*[dev]*/, int32_t *out_max /*[dev] 1, zeroed*/,
                     void *stream);
size_t sg_topn_select_rows_workspace_bytes(int64_t n_cand, int64_t n_rows);
int sg_topn_select_rows(int64_t n_cand, const int32_t *cand_row, const int32_t *cand_col, const double *score,
                        int64_t row_begin, int64_t n_rows, int top_n, const int32_t *row_cnt /*[dev] n_rows*/,
                        int64_t *out_indptr, int32_t *out_row, int32_t *out_col, double *out_score,
                        int64_t *out_nnz /*[dev] 1*/, int32_t *out_max_row /*[dev] 1*/, void *ws, size_t ws_bytes,
                        void *stream);

/*
 * Self-match over groups of bit-identical rows (csrc/sg_dedup.cu, csrc/sg_select.cu; DESIGN.md §4 "Identical rows").
 * sg_row_dedup: uid[n_rows] = group of every row; groups numbered by their first member, which is the representative
 * rep[m]; members as a CSR over groups, mem_ptr[n_rows+1] (entries m..n_rows hold n_rows) and mem_rows[n_rows],
 * ascending inside a group; out_sizes = {m, stored values of the representatives}.  A group's members are verified
 * bit-identical (length, indices, value bits in `dtype`) to each other; the 64-bit row hash, masked by `hash_mask`
 * (all ones in production), only orders the rows.
 * sg_rows_gather: U = the rows rep[0..m) of a CSR matrix (out_indptr[m+1] from 0; out_val32 NULL: not copied).
 */
size_t sg_row_dedup_workspace_bytes(int64_t n_rows);
int sg_row_dedup(int64_t n_rows, const int64_t *indptr, const int32_t *indices, const void *val, int dtype,
                 uint64_t hash_mask, int32_t *uid, int32_t *mem_ptr, int32_t *mem_rows, int32_t *rep,
                 int64_t *out_sizes /*[dev] 2*/, void *ws, size_t ws_bytes, void *stream);
size_t sg_rows_gather_workspace_bytes(int64_t m);
int sg_rows_gather(int64_t m, const int32_t *rep, const int64_t *indptr, const int32_t *indices, const void *val,
                   const float *val32, int dtype, int64_t *out_indptr, int32_t *out_indices, void *out_val,
                   float *out_val32, void *ws, size_t ws_bytes, void *stream);
/*
 * Selection of the product of U with itself, expanded to the original rows.  Input: sg_rescore's kept pairs in group
 * space (u, v, score), mirrors included.  Every (u, v, s) stands for the pairs (u, c, s) of every member c of v; the
 * survivors of u are ranked like sg_topn_select_rows ranks a row (score descending, the larger column wins a tie at
 * the cut, ties written in ascending column order), and every row r gets a copy of the list of its group uid[r].
 * sg_topn_groups_count: grp_cnt[m] = expanded survivors per group, totals = {sum of grp_cnt, output pairs} (the
 * sizes the caller allocates).  Needs top_n <= sg_topn_rows_cap() / 2 when top_n > 32.
 */
int sg_topn_groups_count(int64_t n_cand, const int32_t *cand_row, const int32_t *cand_col, int64_t n_groups,
                         const int32_t *mem_ptr, int top_n, int32_t *grp_cnt /*[dev] n_groups*/,
                         int64_t *totals /*[dev] 2*/, void *stream);
size_t sg_topn_select_groups_workspace_bytes(int64_t n_cand, int64_t n_expanded, int64_t n_groups, int64_t n_rows,
                                             int top_n);
int sg_topn_select_groups(int64_t n_cand, const int32_t *cand_row, const int32_t *cand_col, const double *score,
                          int64_t n_groups, const int32_t *mem_ptr, const int32_t *mem_rows, const int32_t *grp_cnt,
                          int64_t n_expanded, int64_t n_rows, const int32_t *uid, int top_n, int64_t *out_indptr,
                          int32_t *out_row, int32_t *out_col, double *out_score, int64_t *out_nnz /*[dev] 1*/,
                          int32_t *out_max_row /*[dev] 1*/, void *ws, size_t ws_bytes, void *stream);

/*
 * K3 — per-row top-n merge of column-block results.  Replaces sparse_dot_topn.zip_sp_matmul_topn(top_n, C_mats)
 * (call site sg.py:746).  Input: the block results concatenated as COO (block column offsets already added, any
 * order); entries that are not strictly positive are dropped like the reference's heap does (its initial minimum
 * is the smallest positive normal of the value type `dtype`); outputs as sg_topn_select (value-descending rows).
 */
size_t sg_topn_merge_workspace_bytes(int64_t n_entries, int64_t n_rows);
int sg_topn_merge(int64_t n_entries, const int32_t *row, const int32_t *col, const double *score, int64_t n_rows,
                  int top_n, int dtype, int64_t *out_indptr, int32_t *out_row, int32_t *out_col, double *out_score,
                  int64_t *out_nnz /*[dev] 1*/, int32_t *out_max_row /*[dev] 1*/, void *ws, size_t ws_bytes,
                  void *stream);

/* ------------------------------------------------------------------------- *
 * Row ordering for K2 (csrc/sg_order.cu): both operands of C = A*B^T are processed in heavy-feature
 * signature order, so that the docs of a frequent n-gram are runs of consecutive column positions (the
 * lanes of a posting step hit distinct shared-memory banks) and neighbouring warps stream the same buckets.
 * No reference counterpart (the reference's block loop takes rows in input order, sg.py:734-750).
 * ------------------------------------------------------------------------- */
size_t sg_order_workspace_bytes(int64_t n_rows, int64_t n_cols);
/* hrank[n_cols] int8: rank among the n_heavy (<= 64) most frequent features of the matrix, else -1 */
int sg_heavy_features(int64_t n_rows, int64_t n_cols, const int64_t *indptr, const int32_t *indices,
                      const int32_t *df /*[dev] n_cols, optional: sg_feature_df of the matrix, else counted here*/,
                      int n_heavy, int8_t *hrank /*[dev]*/, void *ws, size_t ws_bytes, void *stream);
/* perm[i] = id of the i-th row of [row_begin,row_end) in signature order; rank = inverse (relative ids).
 * With `row_norm` (per row of the range, sg_heavy_norms) the 5-bit quantisation of row_norm*norm_scale leads the
 * sort key, so that rows of similar heavy norm share column tiles (see sg_tile_bounds). */
int sg_row_order(int64_t row_begin, int64_t row_end, const int64_t *indptr, const int32_t *indices,
                 const int8_t *hrank, const float *row_norm /*[dev] or NULL*/, float norm_scale,
                 int32_t *perm /*[dev]*/, int32_t *rank /*[dev] or NULL*/, void *ws,
                 size_t ws_bytes, void *stream);
/* keys[i] = the 64-bit key sg_row_order sorts row row_begin + i by, computed by the same kernel from the same
 * arguments (unsigned order).  A row of another matrix, keyed with the right matrix's hrank and norm scale, finds its
 * position in the right matrix's sorted order by a binary search over the right keys in that order. */
int sg_row_keys(int64_t row_begin, int64_t row_end, const int64_t *indptr, const int32_t *indices,
                const int8_t *hrank, const float *row_norm /*[dev] or NULL*/, float norm_scale,
                uint64_t *keys /*[dev] row_end - row_begin*/, void *stream);

/* ------------------------------------------------------------------------- *
 * K4 — self-match post-processing.
 * Replaces: _fix_diagonal + _symmetrize_matrix on LIL (sg.py:419-427,
 * :955-964): diagonal := 1 for every row, pattern := pattern U pattern^T,
 * output ordered by (row, col) ascending like tolil().tocsr().
 * Output capacity needed: 2*nnz_in + n.
 * ------------------------------------------------------------------------- */
#define SG_SYMM_FIX_DIAGONAL 1 /* _fix_diagonal,     sg.py:955-958 */
#define SG_SYMM_MIRROR 2       /* _symmetrize_matrix, sg.py:961-964 */
size_t sg_symmetrize_workspace_bytes(int64_t nnz_in, int64_t n);
int sg_symmetrize(int64_t n, int64_t nnz_in, int flags, const int32_t *in_row, const int32_t *in_col,
                  const double *in_score, int32_t *out_row, int32_t *out_col, double *out_score,
                  int64_t *out_nnz /*[dev] 1*/, void *ws, size_t ws_bytes, void *stream);

/* ------------------------------------------------------------------------- *
 * Group representatives (SURVEY.md §8f row 2).  Replaces the arithmetic of StringGrouper._deduplicate
 * (sg.py:851-904): weakly connected components of the match graph (:863), per-row similarity sums
 * (:875-881), representative = first member (group_rep='first') or first member with the largest sum
 * ('centroid', idxmax :885-886).  Input: the match list sorted by (row, col) as K4 leaves it.
 * This call synchronises the stream once per component-sweep round (a handful).
 * ------------------------------------------------------------------------- */
size_t sg_group_reps_workspace_bytes(int64_t n);
int sg_group_reps(int64_t n, int64_t nnz, const int32_t *row, const int32_t *col, const double *score,
                  int centroid, int32_t *rep /*[dev] n*/, void *ws, size_t ws_bytes, void *stream);

/* ------------------------------------------------------------------------- *
 * Star groups (group_similar_strings(linkage='star'), csrc/sg_star.cu): greedy star clustering of the match graph.
 * Strings are ranked by index (centroid = 0) or by the similarity sum of sg_group_reps descending, then index
 * (centroid = 1).  In rank order, a string not yet assigned becomes a pivot and takes every unassigned neighbour
 * (u ~ v when (u, v) or (v, u) is stored); rep[i] = the pivot of i's group, so rep[i] is i or one of i's matches.
 * Input: the match list sorted by row (any column order, symmetric or not).  Computed in rounds with the serial
 * rule's result, as many as needed (no cap); the stream is synchronised once every 8 rounds.
 * ------------------------------------------------------------------------- */
size_t sg_group_star_workspace_bytes(int64_t n);
int sg_group_star(int64_t n, int64_t nnz, const int32_t *row, const int32_t *col, const double *score,
                  int centroid, int32_t *rep /*[dev] n*/, void *ws, size_t ws_bytes, void *stream);

/* ------------------------------------------------------------------------- *
 * Nearest master per duplicate (SURVEY.md §8f row 3).  Replaces the reduction of StringGrouper._get_nearest_matches
 * (sg.py:783-849; the groupby / idxmax of :803-807): best[j] = left row with the highest similarity to right row j,
 * the smallest left index among equal scores, -1 when no match holds j.  Input: the match list in any order.
 * ------------------------------------------------------------------------- */
size_t sg_nearest_master_workspace_bytes(int64_t n_right);
int sg_nearest_master(int64_t nnz, const int32_t *row, const int32_t *col, const double *score, int64_t n_right,
                      int32_t *best /*[dev] n_right*/, void *ws, size_t ws_bytes, void *stream);

/* ------------------------------------------------------------------------- *
 * String gather for get_matches (SURVEY.md §8f row 1): replaces `Series.iloc[matches_list.master_side]` /
 * `.iloc[matches_list.dupe_side]` (sg.py:462, :467) for strings that are resident in HBM as packed UTF-8.
 * positions[i] is a row of the Series that starts at document `doc_base` of the packed buffer.
 * sg_gather_offsets: out_offsets[n_sel+1] (the last entry is the total byte count the caller must allocate);
 * sg_gather_bytes: the bytes.  The pair is a ready-made Arrow large_string array.
 * ------------------------------------------------------------------------- */
size_t sg_gather_workspace_bytes(int64_t n_sel);
int sg_gather_offsets(const int64_t *offsets /*[dev]*/, int64_t doc_base, int64_t n_sel,
                      const int32_t *positions /*[dev]*/, int64_t *out_offsets /*[dev] n_sel+1*/, void *ws,
                      size_t ws_bytes, void *stream);
int sg_gather_bytes(const uint8_t *bytes /*[dev]*/, const int64_t *offsets /*[dev]*/, int64_t doc_base,
                    int64_t n_sel, const int32_t *positions /*[dev]*/, const int64_t *out_offsets /*[dev]*/,
                    uint8_t *out_bytes /*[dev]*/, void *stream);

/* row-wise dot of two CSR matrices of equal shape (StringGrouper.dot, sg.py:433-440), summed in the reference's order:
 * master.multiply(dup).sum(axis=1) = p0 + numpy's pairwise sum of p1..pk-1 over the common features, in the matrix
 * dtype, no FMA */
int sg_rowwise_dot(int64_t n_rows, const int64_t *a_indptr, const int32_t *a_indices, const void *a_val,
                   const int64_t *b_indptr, const int32_t *b_indices, const void *b_val, int dtype,
                   double *out /*[dev] n_rows*/, void *stream);

/* ------------------------------------------------------------------------- *
 * Records: several string fields in one product (csrc/sg_fields.cu).  No reference counterpart: the reference
 * compares one Series.  Every field is vectorised by K1 on its own; sg_fields_stack lays the fields' rows side by
 * side into one CSR of n_rows rows:
 *   out_indptr = exclusive scan of the summed row lengths (out_indptr[0] = 0);
 *   row r holds field 0's entries of row r, then field 1's ..., field k's column ids + col_offset[k] and values
 *   val * scale[k] in the matrix dtype (one rounding, no FMA; for SG_DTYPE_F32 scale[k] is first rounded to float);
 *   out_val32 (or NULL for SG_DTYPE_F32, whose out_val is the fp32 array itself) = (float) of every value.
 * indptr[k] / indices[k] / val[k] are HOST arrays of n_fields device pointers; indptr[k] has n_rows+1 absolute
 * positions into indices[k] / val[k] (a row-range view need not start at 0).  scale[k] in (0, 1] and col_offset[k]
 * are host arrays too.  Output arrays hold sum of the fields' row lengths entries.  1 <= n_fields <= SG_FIELDS_MAX.
 * ------------------------------------------------------------------------- */
#define SG_FIELDS_MAX 32
size_t sg_fields_stack_workspace_bytes(int64_t n_rows);
int sg_fields_stack(int n_fields, int64_t n_rows, const int64_t *const *indptr, const int32_t *const *indices,
                    const void *const *val, const double *scale, const int32_t *col_offset, int dtype,
                    int64_t *out_indptr /*[dev] n_rows+1*/, int32_t *out_indices /*[dev]*/, void *out_val /*[dev]*/,
                    float *out_val32 /*[dev] or NULL*/, void *ws, size_t ws_bytes, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* SG_B200_H */
