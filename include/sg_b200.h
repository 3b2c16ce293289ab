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
 * Phase 2 (sg_tfidf_finalize): exclusive scan of row_nnz -> indptr (int64);
 * exclusive scan of (df > 0) over the key table -> rank_table[key] = column id
 * = rank of the n-gram in sorted order (sklearn _sort_features);
 * idf = ln((1+n)/(1+df)) + 1 and x = tf*idf in the matrix dtype; row L2 norm
 * accumulated in double in column order, IEEE sqrt and divide (sklearn
 * _inplace_csr_row_normalize_l2); writes indices, values in the matrix dtype
 * (val64 for f64, may be NULL for f32) and an fp32 copy for K2.
 * `vocab_size` [dev] receives V, `nnz_total` [dev] receives indptr[n_docs].
 * The caller sizes indices/val64/val32 with total_bytes entries (an upper
 * bound of nnz), so no host read-back is needed between the two phases.
 */
size_t sg_tfidf_finalize_workspace_bytes(int64_t n_docs, int ngram);
int sg_tfidf_finalize(const int64_t *offsets /*[dev]*/, int64_t n_docs,
                      int64_t n_docs_fit /* documents counted in df_table: n_docs, or the global count when the
                                            corpus is sharded over GPUs and df_table was all-reduced */,
                      int ngram, int dtype,
                      const int32_t *df_table /*[dev]*/, int32_t *rank_table /*[dev] slots*/,
                      const uint32_t *scratch_key, const uint32_t *scratch_tf, int32_t *row_nnz,
                      int64_t *indptr /*[dev] n_docs+1*/, int32_t *indices /*[dev]*/,
                      double *val64 /*[dev]*/, float *val32 /*[dev]*/,
                      int32_t *vocab_size /*[dev] 1*/, int64_t *nnz_total /*[dev] 1*/,
                      void *ws /*[dev]*/, size_t ws_bytes, void *stream);

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
 * df[c]), column ids by a scan; values as sg_tfidf_finalize.  No device-to-host read-back inside either call.
 * ------------------------------------------------------------------------- */
int sg_tfidf64_count(const void *symbols /*[dev]*/, int sym_width, const int64_t *offsets /*[dev] n_docs+1*/,
                     int64_t n_docs, int ngram, int bits, const uint8_t *lut /*[dev] 256 or NULL*/,
                     uint32_t *scratch_clean /*[dev] total*/, uint64_t *scratch_sort /*[dev] total*/,
                     uint64_t *scratch_key /*[dev] total*/, uint32_t *scratch_tf /*[dev] total*/,
                     int32_t *row_nnz /*[dev] n_docs+1*/, void *stream);
size_t sg_tfidf64_finalize_workspace_bytes(int64_t n_docs, int64_t total_symbols);
int sg_tfidf64_finalize(const int64_t *offsets /*[dev]*/, int64_t n_docs, int64_t n_docs_fit, int64_t total_symbols,
                        int ngram, int bits, int dtype, const uint64_t *scratch_key, const uint32_t *scratch_tf,
                        int32_t *row_nnz, int64_t *indptr /*[dev] n_docs+1*/, int32_t *indices /*[dev] total*/,
                        double *val64 /*[dev] total or NULL*/, float *val32 /*[dev] total*/,
                        uint64_t *vocab_keys /*[dev] total*/, int32_t *df /*[dev] total*/,
                        int32_t *vocab_size /*[dev] 1*/, int64_t *nnz_total /*[dev] 1*/, void *ws /*[dev]*/,
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
 * order `rank` (position of every row in heavy-feature signature order, sg_row_order; NULL = input
 * order): column tile t holds positions [t*tile_w, (t+1)*tile_w); bucket (f, t) = the docs of feature f
 * inside tile t (in no particular order), at bucket_ptr[f*T + t] (feature-major, T = sg_num_tiles); a posting is 4 bytes:
 * position - t*tile_w in the low 16 bits, the weight rounded to fp16 in the high 16 bits (candidate
 * scores only need to be within the caller's margin; every candidate is re-scored exactly).  `bucket_dir` (optional) receives the same directory as aligned
 * 8-byte entries {int32 start, u16 length, fp16 largest |weight| of the bucket}, T*(n_cols+1) of them, the form
 * sg_cossim_candidates reads.  `bucket_maxw` receives the largest weights again as fp16 rows, one row of
 * sg_num_tiles_padded() entries per feature (zero padded), which sg_cossim_candidates streams to skip every
 * (left row, column tile) pair whose score bound sum_f |a_f| * max|w_(f,t)| cannot reach the candidate
 * threshold.  tile_w <= 32768.
 * `indptr` may be a row-range view (indptr_base = indptr[0]).
 */
size_t sg_postings_workspace_bytes(int64_t nnz, int64_t n_cols, int64_t n_tiles);
int sg_postings_build(int64_t n_rows, int64_t n_cols, int64_t nnz, const int64_t *indptr /*[dev]*/,
                      const int32_t *indices /*[dev]*/, const float *val32 /*[dev]*/,
                      const int32_t *rank /*[dev] or NULL*/, int tile_w, int64_t indptr_base,
                      float w_scale /* weights are multiplied by this before the fp16 rounding: 1 / max|w| */,
                      int32_t *bucket_ptr /*[dev] T*(n_cols+1)+1*/,
                      void *bucket_dir /*[dev] T*(n_cols+1)*8 B or NULL*/,
                      void *bucket_maxw /*[dev] (n_cols+1)*Tp*2 B or NULL*/, void *postings /*[dev] nnz*4 B*/,
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
                         float cand_threshold, const float *cand_threshold_row /*[dev] per row id, or NULL*/,
                         const float *pruned_norm_row /*[dev] per row id, or NULL*/,
                         const float *tile_bound /*[dev] sg_num_tiles_padded() entries, zero padded*/,
                         int64_t tiles_per_group, int32_t *cand_row /*[dev] cap*/,
                         int32_t *cand_col /*[dev] cap*/,
                         float *cand_partial /*[dev] cap or NULL: the candidate's partial score over the kept features
                                               as accumulated (input of sg_rescore_refined)*/,
                         int64_t cand_cap,
                         unsigned long long *cand_count /*[dev] 1*/,
                         unsigned long long *row_queue /*[dev] 1*/, int warps_per_cta, void *stream);

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
                    uint32_t *mask /*[dev] words*mask_stride*/, int64_t mask_stride, void *stream);
size_t sg_tiles_smem_bytes(int stage_bytes, int warps_per_cta);
int sg_tiles_candidates(const int32_t *perm_a /*[dev] or NULL*/, int64_t n_ranks, int64_t row_begin,
                        const void *rowinfo /*[dev]*/, const void *lpack /*[dev]*/, const uint32_t *mask /*[dev]*/,
                        int64_t mask_stride, const void *tile_desc /*[dev]*/, const void *blob /*[dev]*/,
                        int64_t n_right, int64_t n_cols, const float *tile_bound /*[dev]*/,
                        const int32_t *perm_b /*[dev] or NULL*/, int stage_bytes /* maxima[0] */,
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
 */
int sg_rescore(int64_t n_cand, const int32_t *cand_row, const int32_t *cand_col,
               const int64_t *a_indptr, const int32_t *a_indices, const void *a_val,
               const int64_t *b_indptr, const int32_t *b_indices, const void *b_val, int dtype,
               double *score_out /*[dev] n_cand*/, double keep_threshold, int32_t *keep_row /*[dev] n_cand or NULL*/,
               int32_t *keep_col /*[dev] n_cand or NULL*/, unsigned long long *keep_count /*[dev] 1 or NULL*/,
               int32_t *row_cnt /*[dev] per left row - row_begin, zeroed by the caller, or NULL: += kept per row*/,
               int64_t row_begin, void *stream);
/* sg_rescore behind the per-candidate grouped bound of csrc/sg_prune.cu: candidate i = (r, c) is only scored when
 *   cand_partial[i] + sum_g left_group_norms[r][g] * right_group_norms[c][g]  >  row_threshold[r]
 * (partial score from sg_cossim_candidates, group norms from sg_prune_rows / sg_heavy_norms, row_threshold =
 * sg_prune_rows' out_threshold): the others cannot reach the threshold and their right rows are never read.  Same
 * kept set and scores as sg_rescore on the same candidates.  *refined_count [dev] (zeroed, or NULL) += candidates that
 * were scored.  keep_count / keep_row / keep_col are required. */
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
                       int32_t *row_cnt /*[dev] or NULL*/, int64_t row_begin, void *stream);

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

/* row-wise dot of two CSR matrices of equal shape (StringGrouper.dot, sg.py:433-440) */
int sg_rowwise_dot(int64_t n_rows, const int64_t *a_indptr, const int32_t *a_indices, const void *a_val,
                   const int64_t *b_indptr, const int32_t *b_indices, const void *b_val, int dtype,
                   double *out /*[dev] n_rows*/, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* SG_B200_H */
