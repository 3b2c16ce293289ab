"""ctypes binding of libsg_b200.so (the C ABI declared in include/sg_b200.h).

The product path has no CPU fallback: if the shared library is missing or a
CUDA device is absent, the callers raise.  Build with
`python -c "import __graft_entry__ as g; g.build()"` (nvcc, sm_90a).
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.path.join(_HERE, "libsg_b200.so")

SG_OK = 0
SG_ERR_INVALID = -1
SG_ERR_CUDA = -2
SG_ERR_OVERFLOW = -3
SG_ERR_UNSUPPORTED = -4
SG_DTYPE_F32 = 0
SG_DTYPE_F64 = 1
SG_FLAG_IGNORE_CASE = 1
SG_FLAG_STRIP_DEFAULT = 2
SG_SYMM_FIX_DIAGONAL = 1
SG_SYMM_MIRROR = 2
SG_ACC_F32 = 0
SG_ACC_U16 = 1
SG_FLOOR_SEED = 1
SG_FLOOR_LONG_ROWS = 2
SG_SYMBOL_UNKNOWN = 0xffffffff      # a query symbol outside the fitted alphabet (K1 transform)
SG_LUT_UNKNOWN = 0xfe
SG_FIELDS_MAX = 32                  # fields one sg_fields_stack call lays side by side

_i64 = ctypes.c_int64
_i32 = ctypes.c_int
_p = ctypes.c_void_p
_sz = ctypes.c_size_t
_f32 = ctypes.c_float
_f64 = ctypes.c_double
_u32 = ctypes.c_uint

# name -> (restype, argtypes); mirrors include/sg_b200.h one to one
SIGNATURES = {
    "sg_last_error": (ctypes.c_char_p, []),
    "sg_abi_version": (_i32, []),
    "sg_device_info": (_i32, [_p, _p, _p]),
    "sg_tfidf_table_slots": (_i64, [_i32]),
    "sg_tfidf_count": (_i32, [_p, _p, _i64, _i32, _u32, _p, _p, _p, _p, _p, _p, _p]),
    "sg_tfidf_vocab_workspace_bytes": (_sz, [_i64, _i32]),
    "sg_tfidf_vocab": (_i32, [_i64, _i32, _p, _p, _p, _p, _p, _p, _p, _sz, _p]),
    "sg_tfidf_values": (_i32, [_p, _i64, _i32, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p]),
    "sg_tfidf_vocab_keys": (_i32, [_p, _p, _i32, _p, _p]),
    "sg_tfidf_vocab_df": (_i32, [_p, _p, _i32, _p, _p]),
    "sg_tfidf64_count": (_i32, [_p, _i32, _p, _i64, _i32, _i32, _p, _p, _p, _p, _p, _p, _p]),
    "sg_tfidf64_vocab_workspace_bytes": (_sz, [_i64, _i64]),
    "sg_tfidf64_vocab": (_i32, [_p, _i64, _i64, _i32, _i32, _p, _p, _p, _p, _p, _p, _p, _p, _p, _sz, _p]),
    "sg_tfidf64_values": (_i32, [_p, _i64, _i32, _p, _p, _p, _p, _p, _p, _p]),
    "sg_tfidf_transform_count": (_i32, [_p, _p, _i64, _i32, _u32, _p, _p, _p, _p, _p, _p]),
    "sg_tfidf_transform_workspace_bytes": (_sz, [_i64]),
    "sg_tfidf_known": (_i32, [_p, _i64, _p, _p, _p, _p, _p, _p, _sz, _p]),
    "sg_tfidf64_transform_count": (_i32, [_p, _i32, _p, _i64, _i32, _i32, _p, _p, _p, _p, _p, _p, _p]),
    "sg_tfidf64_known": (_i32, [_p, _i64, _p, _i32, _p, _p, _p, _p, _p, _p, _p, _sz, _p]),
    "sg_num_tiles": (_i64, [_i64, _i32]),
    "sg_num_tiles_padded": (_i64, [_i64, _i32]),
    "sg_postings_workspace_bytes": (_sz, [_i64, _i64, _i64]),
    "sg_postings_build": (_i32, [_i64, _i64, _i64, _p, _p, _p, _p, _i32, _i64, _f32, _p, _p, _p, _p, _p, _sz, _p]),
    "sg_feature_df": (_i32, [_i64, _i64, _p, _p, _p, _p]),
    "sg_prune_rows": (_i32, [_i64, _i64, _p, _p, _p, _p, _p, _f32, _f32, _f32, _f32, _f32, _p, _p, _p, _p, _p, _p, _p]),
    "sg_prune_rows_floor": (_i32, [_i64, _i64, _p, _p, _p, _p, _p, _f32, _f32, _f32, _p, _f32, _f32, _p, _p, _p, _p,
                                   _p, _p, _p]),
    "sg_heavy_norms": (_i32, [_i64, _i64, _p, _p, _p, _p, _p, _p, _p]),
    "sg_tile_bounds": (_i32, [_i64, _p, _p, _i32, _p, _p]),
    "sg_cossim_candidates": (_i32, [_p, _p, _p, _p, _i64, _i64, _p, _i64, _i64, _p, _p, _p, _p, _i32, _i32, _f32,
                                    _f32, _f32, _p, _p, _p, _i64, _p, _p, _p, _p, _p, _i64, _p, _p, _i32, _p]),
    "sg_cossim_candidates_floor": (_i32, [_p, _p, _p, _p, _i64, _i64, _p, _i64, _i64, _p, _p, _p, _p, _i32, _i32,
                                          _f32, _f32, _f32, _p, _p, _p, _i64, _p, _p, _p, _i64, _p, _p, _i32, _p, _i32,
                                          _f32, _f32, _p, _i32, _p]),
    "sg_cossim_candidates_range": (_i32, [_p, _p, _p, _p, _i64, _i64, _p, _i64, _i64, _p, _p, _p, _p, _i32, _i32,
                                          _f32, _f32, _f32, _p, _p, _p, _i64, _p, _p, _p, _p, _p, _p, _i64, _p, _p, _i32,
                                          _p]),
    "sg_cossim_candidates_range_floor": (_i32, [_p, _p, _p, _p, _i64, _i64, _p, _i64, _i64, _p, _p, _p, _p, _i32,
                                                _i32, _f32, _f32, _f32, _p, _p, _p, _i64, _p, _p, _p, _p, _p, _p, _i64,
                                                _p, _p, _i32, _p, _i32, _f32, _f32, _p, _i32, _p]),
    "sg_tiles_tile_w": (_i32, []),
    "sg_tiles_max_cols": (_i64, []),
    "sg_tiles_blob_bound": (_i64, [_i64, _i64, _i64]),
    "sg_tiles_workspace_bytes": (_sz, [_i64, _i64, _i64]),
    "sg_tiles_build": (_i32, [_i64, _i64, _i64, _p, _p, _p, _p, _i64, _f32, _p, _p, _i64, _p, _p, _p, _sz, _p]),
    "sg_tiles_pack_left": (_i32, [_i64, _p, _i64, _p, _p, _p, _p, _p, _p, _f32, _p, _p, _p]),
    "sg_tiles_mask_words": (_i64, [_i64]),
    "sg_tiles_filter": (_i32, [_i64, _p, _p, _p, _i64, _p, _p, _p, _p, _p, _i64, _p]),
    "sg_tiles_smem_bytes": (_sz, [_i32, _i32]),
    "sg_tiles_candidates": (_i32, [_p, _i64, _i64, _p, _p, _p, _i64, _p, _p, _i64, _i64, _p, _p, _p, _p, _i32, _p, _p,
                                   _i64, _p, _p, _p, _i32, _p]),
    "sg_order_workspace_bytes": (_sz, [_i64, _i64]),
    "sg_heavy_features": (_i32, [_i64, _i64, _p, _p, _p, _i32, _p, _p, _sz, _p]),
    "sg_row_order": (_i32, [_i64, _i64, _p, _p, _p, _p, _f32, _p, _p, _p, _sz, _p]),
    "sg_row_keys": (_i32, [_i64, _i64, _p, _p, _p, _p, _f32, _p, _p]),
    "sg_rescore": (_i32, [_i64, _p, _p, _p, _p, _p, _p, _p, _p, _i32, _p, _f64, _p, _p, _p, _p, _p, _i64, _p]),
    "sg_rescore_refined": (_i32, [_i64, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _i32, _p, _f64, _p, _p, _p, _p,
                                  _p, _p, _i64, _p]),
    "sg_rescore_floor": (_i32, [_i64, _p, _p, _p, _p, _p, _p, _p, _p, _i32, _p, _f64, _p, _p, _p, _p, _i64, _p, _p,
                                _p]),
    "sg_rescore_refined_floor": (_i32, [_i64, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _i32, _p, _f64, _p, _p,
                                        _p, _p, _p, _i64, _p, _p, _f32, _f32, _p, _p]),
    "sg_rescore_nearest": (_i32, [_i64, _p, _p, _p, _p, _p, _p, _p, _p, _i32, _p, _f64, _p, _p, _p, _p, _i64, _p, _p,
                                  _p]),
    "sg_rescore_refined_nearest": (_i32, [_i64, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _i32, _p, _f64, _p,
                                          _p, _p, _p, _p, _i64, _p, _p, _f32, _f32, _p, _p]),
    "sg_topn_rows_cap": (_i32, []),
    "sg_row_count_max": (_i32, [_i64, _p, _p, _p]),
    "sg_topn_select_rows_workspace_bytes": (_sz, [_i64, _i64]),
    "sg_topn_select_rows": (_i32, [_i64, _p, _p, _p, _i64, _i64, _i32, _p, _p, _p, _p, _p, _p, _p, _p, _sz, _p]),
    "sg_row_dedup_workspace_bytes": (_sz, [_i64]),
    "sg_row_dedup": (_i32, [_i64, _p, _p, _p, _i32, ctypes.c_uint64, _p, _p, _p, _p, _p, _p, _sz, _p]),
    "sg_rows_gather_workspace_bytes": (_sz, [_i64]),
    "sg_rows_gather": (_i32, [_i64, _p, _p, _p, _p, _p, _i32, _p, _p, _p, _p, _p, _sz, _p]),
    "sg_topn_groups_count": (_i32, [_i64, _p, _p, _i64, _p, _i32, _p, _p, _p]),
    "sg_topn_select_groups_workspace_bytes": (_sz, [_i64, _i64, _i64, _i64, _i32]),
    "sg_topn_select_groups": (_i32, [_i64, _p, _p, _p, _i64, _p, _p, _p, _i64, _i64, _p, _i32, _p, _p, _p, _p, _p, _p,
                                     _p, _sz, _p]),
    "sg_topn_select_workspace_bytes": (_sz, [_i64, _i64]),
    "sg_topn_select": (_i32, [_i64, _p, _p, _p, _i64, _i64, _i32, _f64, _p, _p, _p, _p, _p, _p, _p, _sz, _p]),
    "sg_topn_merge_workspace_bytes": (_sz, [_i64, _i64]),
    "sg_topn_merge": (_i32, [_i64, _p, _p, _p, _i64, _i32, _i32, _p, _p, _p, _p, _p, _p, _p, _sz, _p]),
    "sg_symmetrize_workspace_bytes": (_sz, [_i64, _i64]),
    "sg_symmetrize": (_i32, [_i64, _i64, _i32, _p, _p, _p, _p, _p, _p, _p, _p, _sz, _p]),
    "sg_group_reps_workspace_bytes": (_sz, [_i64]),
    "sg_group_reps": (_i32, [_i64, _i64, _p, _p, _p, _i32, _p, _p, _sz, _p]),
    "sg_group_star_workspace_bytes": (_sz, [_i64]),
    "sg_group_star": (_i32, [_i64, _i64, _p, _p, _p, _i32, _p, _p, _sz, _p]),
    "sg_nearest_master_workspace_bytes": (_sz, [_i64]),
    "sg_nearest_master": (_i32, [_i64, _p, _p, _p, _i64, _p, _p, _sz, _p]),
    "sg_gather_workspace_bytes": (_sz, [_i64]),
    "sg_gather_offsets": (_i32, [_p, _i64, _i64, _p, _p, _p, _sz, _p]),
    "sg_gather_bytes": (_i32, [_p, _p, _i64, _i64, _p, _p, _p, _p]),
    "sg_rowwise_dot": (_i32, [_i64, _p, _p, _p, _p, _p, _p, _i32, _p, _p]),
    "sg_fields_stack_workspace_bytes": (_sz, [_i64]),
    "sg_fields_stack": (_i32, [_i32, _i64, _p, _p, _p, _p, _p, _i32, _p, _p, _p, _p, _p, _sz, _p]),
}

_LIB = None


class SgB200Error(RuntimeError):
    pass


def load():
    """Load libsg_b200.so and declare every exported symbol; raises if absent."""
    global _LIB
    if _LIB is None:
        if not os.path.exists(SO_PATH):
            raise SgB200Error(
                "libsg_b200.so is not built (%s). Run `python -c \"import __graft_entry__ as g; g.build()\"`; "
                "there is no CPU fallback for the hot path." % SO_PATH)
        lib = ctypes.CDLL(SO_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)   # AttributeError if the .so does not export it
            fn.restype = res
            fn.argtypes = args
        _LIB = lib
    return _LIB


def check(rc):
    """Translate a negative return code into the Python exception the reference would raise."""
    if rc == SG_OK:
        return
    msg = load().sg_last_error()
    msg = msg.decode("utf-8", "replace") if msg else "libsg_b200 error %d" % rc
    if rc == SG_ERR_INVALID:
        raise ValueError(msg)
    if rc == SG_ERR_OVERFLOW:
        raise OverflowError(msg)
    if rc == SG_ERR_UNSUPPORTED:
        raise NotImplementedError(msg)
    raise SgB200Error(msg)
