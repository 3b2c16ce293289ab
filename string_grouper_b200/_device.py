"""Device-side plumbing: HBM containers (torch tensors) and the calls into libsg_b200.so.

PyTorch is used for device memory, streams and (in _dist.py) torch.distributed
only; every kernel on the hot path lives in csrc/*.cu behind the C ABI.
"""
import ctypes
import os

import numpy as np

from . import _lib

_TORCH = None

# hand-written kernels launched so far (CUB scans / sorts and memsets are not counted); bench.py "gpu_launches"
LAUNCH_COUNTS = {"postings": 0, "candidates": 0, "rescore": 0, "select": 0, "symmetrize": 0, "tfidf": 0,
                 "rowdot": 0, "order": 0, "tiles": 0, "groups": 0, "gather": 0, "prune": 0}
# "tiles": the tile-centric K2 (csrc/sg_tiles.cu): build, pack_left, filter, candidates

TRANSFER_BYTES = {"d2h": 0, "h2d": 0}      # bytes moved by the bulk copies (bench.py e2e accounting)

DEFAULT_TILE_W = int(os.environ.get("SG_B200_TILE_W", "0"))         # 0: 256 (u16) columns per tile, 128 for large right matrices
DEFAULT_WARPS = int(os.environ.get("SG_B200_WARPS", "8"))           # 8 warps x 5 CTAs at 48 registers (no spills)
# posting bytes one column-tile group may hold: a group's buckets should stay resident in H100's 50 MB L2 next to the
# rest of the working set (663k rows on H100: 6 MB groups 43.4-44.0 ms for the candidates kernel, 12 MB 45.5-46.2, 24 MB 49.4)
GROUP_BYTES = int(os.environ.get("SG_B200_GROUP_MB", "6")) << 20
CAND_MARGIN = 1.5e-3   # candidates: fp16 posting weights (<= 4.9e-4) + fp32 accumulation; all are re-scored exactly
U16_MARGIN_PER_FEATURE = 2e-5   # 1/32768 fixed-point accumulator tile: one rounding of <= 2^-16 per added product
# Exact threshold pruning (csrc/sg_prune.cu): the most expensive heavy features of a left row are skipped while
# their norm times the largest right-row norm stays below PRUNE_FRAC * min_similarity.  0 switches it off.
PRUNE_FRAC = float(os.environ.get("SG_B200_PRUNE", "0.9"))
ACC_DTYPE = os.environ.get("SG_B200_ACC", "u16")                    # accumulator tile: u16 | f32
MAX_CAND_DENSITY = float(os.environ.get("SG_B200_MAX_CAND_DENSITY", "1.5e-3"))   # candidates per (row, column) pair
MAX_BUCKETS = int(os.environ.get("SG_B200_MAX_BUCKETS", str(400_000_000)))       # directory entries (22 B each)
CAND_CHUNK = int(os.environ.get("SG_B200_CAND_CHUNK", str(1 << 28)))            # candidates per chunk of left rows
# up to this many (left row, right row) pairs the candidates kernel is launched without a sizing pass (see cossim_topn)
OPTIMISTIC_PAIRS = float(os.environ.get("SG_B200_OPTIMISTIC_PAIRS", "5e11"))
REFINE = os.environ.get("SG_B200_REFINE", "1") != "0"      # grouped per-candidate bound before the exact re-score
# K2 formulation: "row" (the default) = one warp per left row over L2-resident posting buckets (csrc/sg_cossim.cu; also
# the general path: negative values, norms above 1, near-zero thresholds); "tiles" = right tiles staged through TMA into
# shared memory (csrc/sg_tiles.cu), for L2-normalised non-negative operands.  Measured on H100 at 663k rows the row kernel
# is the faster one (65 vs 80 ms per step, DESIGN.md §4).
K2_KERNEL = os.environ.get("SG_B200_KERNEL", "row").lower()
TILE_MARGIN = 2e-5               # fp32 arithmetic of thresholds / norms and the f64 -> f32 copy of the values
TILE_MARGIN_PER_FEATURE = 3.1e-5  # a_q * w_q / 2^30 vs a * w: both weights rounded to nearest 2^-15 (<= 2^-15 + 2^-32)
TILE_WARPS = int(os.environ.get("SG_B200_TILE_WARPS", "8"))
SELECT_MODE = os.environ.get("SG_B200_SELECT", "rows").lower()      # "rows" (per-row ranking) | "sort" (global sorts)


def torch():
    global _TORCH
    if _TORCH is None:
        import torch as _t
        _TORCH = _t
    return _TORCH


def require_cuda():
    t = torch()
    if not t.cuda.is_available():
        raise _lib.SgB200Error("string_grouper_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback "
                               "for the hot path")
    _lib.load()
    return t


def _ptr(x):
    return ctypes.c_void_p(0 if x is None else x.data_ptr())


def _stream():
    return ctypes.c_void_p(torch().cuda.current_stream().cuda_stream)


def _empty(n, dtype, device):
    return torch().empty(max(int(n), 1), dtype=dtype, device=device)


TIME_KERNELS = False      # bench.py: record CUDA events for the phases of every product (also through the public API)


def _timed(stats):
    return stats is not None and (stats.get("time_kernels") or TIME_KERNELS)


def mark(stats, name):
    """Phase boundary for bench.py `phases_ms`: a CUDA event on the current stream when stats["time_kernels"] is set."""
    if _timed(stats):
        ev = torch().cuda.Event(enable_timing=True)
        ev.record()
        stats.setdefault("marks", []).append((name, ev))


def phases_ms(stats):
    """{phase: milliseconds} from the marks of one step (the time between a mark and its predecessor is charged to
    the mark's name; the first mark only starts the clock)."""
    out = {}
    marks = stats.get("marks", [])
    for (_, e0), (name, e1) in zip(marks[:-1], marks[1:]):
        out[name] = out.get(name, 0.0) + e0.elapsed_time(e1)
    return out


def to_host(*tensors):
    """Device tensors -> numpy arrays through page-locked staging buffers (torch's caching host allocator
    re-uses them from call to call): all copies are queued on the current stream, one synchronisation.
    Pageable `.cpu()` copies run at a fraction of the PCIe rate and were the largest end-to-end cost."""
    t = torch()
    tensors = [x.contiguous() for x in tensors]
    TRANSFER_BYTES["d2h"] += sum(x.numel() * x.element_size() for x in tensors)
    try:
        outs = [t.empty(x.shape, dtype=x.dtype, pin_memory=bool(x.numel())) for x in tensors]
    except RuntimeError:          # page-locking refused (memlock limit): plain copies
        return [x.cpu().numpy() for x in tensors]
    for h, x in zip(outs, tensors):
        if x.numel():
            h.copy_(x, non_blocking=True)
    t.cuda.current_stream().synchronize()
    return [h.numpy() for h in outs]


class DeviceCSR:
    """CSR matrix resident in HBM: indptr int64, indices int32, val (matrix dtype), val32 (fp32 copy).

    Quacks like the scipy matrices StringGrouper._get_tf_idf_matrices returns
    (string_grouper/string_grouper.py:685-697): `.shape`,
    `.toarray()`, `.indptr` ... are served from a lazily materialised scipy
    copy, so reference-style tests and user code keep working.
    """

    def __init__(self, shape, indptr, indices, val, val32, nnz, dtype, norm_bound=1.0, base=0):
        self.shape = (int(shape[0]), int(shape[1]))
        # indptr holds ABSOLUTE positions into indices/val (a row-range view of a bigger matrix keeps
        # the parent's arrays and starts at `base`); the kernels never assume indptr[0] == 0.
        self.d_indptr, self.d_indices, self.d_val, self.d_val32 = indptr, indices, val, val32
        self.base = int(base)
        self.nnz = int(nnz)
        self.nnz_parent = int(nnz)     # stored values of the whole array a row-range view points into
        self.dtype = np.dtype(dtype)
        self.norm_bound = float(norm_bound)
        self._host = None
        self._order = None          # (hrank, perm, rank): rows ordered by (quantised heavy norm, heavy-feature signature)
        self._postings2 = {}
        self._tiles = None          # tile blobs of the tile-centric K2 (right_tiles)
        self.row_offset = None      # set when this matrix is one rank's block of rows of a sharded matrix
        self.global_rows = None
        self._df = None             # document frequency of every feature (sg_feature_df)
        self._heavy_norm = None     # per-row norm over the heavy features (sg_heavy_norms)
        self._heavy_groups = None   # the same per group of heavy ranks, fp16[16] (sg_rescore_refined)
        self.nonneg = True          # no negative stored value (K1 output; checked for uploaded matrices)

    @property
    def device(self):
        return self.d_indptr.device

    @classmethod
    def from_scipy(cls, m, device=None):
        t = require_cuda()
        from scipy.sparse import issparse
        if not issparse(m):
            raise TypeError("expected a scipy sparse matrix, got %r" % type(m))
        m = m.tocsr()
        if not m.has_sorted_indices:
            m = m.sorted_indices()
        if m.nnz >= 2**31 - 1:
            raise OverflowError("matrix has %d stored values; int32 indices overflow" % m.nnz)
        dtype = np.float32 if m.dtype == np.float32 else np.float64
        device = device or t.device("cuda", t.cuda.current_device())
        data = np.ascontiguousarray(m.data, dtype=dtype)
        indptr = t.from_numpy(np.ascontiguousarray(m.indptr, dtype=np.int64)).to(device)
        indices = t.from_numpy(np.ascontiguousarray(m.indices, dtype=np.int32)).to(device)
        val = t.from_numpy(data).to(device)
        val32 = val if dtype == np.float32 else val.to(t.float32)
        bound = float(np.sqrt(m.multiply(m).sum(axis=1).max())) if m.nnz else 1.0
        out = cls(m.shape, indptr, indices, val, val32, m.nnz, dtype, max(bound, 1e-30))
        out._host = m
        out.nonneg = bool(m.nnz == 0 or data.min() >= 0)
        return out

    def to_scipy(self):
        if self._host is None:
            from scipy.sparse import csr_matrix
            lo, hi = self.base, self.base + self.nnz
            indptr = self.d_indptr[:self.shape[0] + 1].cpu().numpy() - lo
            idx_dtype = np.int32 if max(self.shape) < 2**31 and self.nnz < 2**31 else np.int64
            self._host = csr_matrix((self.d_val[lo:hi].cpu().numpy(),
                                     self.d_indices[lo:hi].cpu().numpy().astype(idx_dtype),
                                     indptr.astype(idx_dtype)), shape=self.shape)
        return self._host

    def get_shape(self):
        return self.shape

    def toarray(self):
        return self.to_scipy().toarray()

    def __getitem__(self, key):
        return self.to_scipy()[key]

    def __matmul__(self, other):
        return self.to_scipy() @ (other.to_scipy() if hasattr(other, "to_scipy") else other)

    def __getattr__(self, name):
        # the scipy face: only the attributes below materialise the host copy (a typo or a probing hasattr() must not
        # trigger a device-to-host copy of the whole matrix)
        if name in _SCIPY_CSR_ATTRS:
            return getattr(self.to_scipy(), name)
        raise AttributeError("%s has no attribute %r" % (type(self).__name__, name))


# what callers of StringGrouper._get_tf_idf_matrices / _build_matches use on the returned scipy matrices
_SCIPY_CSR_ATTRS = frozenset([
    "indptr", "indices", "data", "T", "transpose", "multiply", "dot", "tocsr", "tocsc", "tocoo", "tolil", "todense",
    "nonzero", "sum", "max", "min", "mean", "getrow", "getcol", "diagonal", "astype", "copy", "getnnz", "has_sorted_indices",
    "sort_indices", "sorted_indices", "format", "ndim", "count_nonzero", "power", "maximum", "minimum", "A", "todok",
    "eliminate_zeros", "sum_duplicates", "asformat", "conj", "conjugate", "getH", "setdiag", "trace", "tobsr", "todia"])


def as_device_csr(m):
    return m if isinstance(m, DeviceCSR) else DeviceCSR.from_scipy(m)


def heavy_features(B):
    """int8 rank of every feature among the 64 most frequent ones of B (-1 otherwise)."""
    t = require_cuda()
    L = _lib.load()
    n_rows, n_cols = B.shape
    hrank = _empty(n_cols, t.int8, B.device)
    ws_bytes = int(L.sg_order_workspace_bytes(n_rows, n_cols))
    ws = _empty(ws_bytes, t.uint8, B.device)
    _lib.check(L.sg_heavy_features(n_rows, n_cols, _ptr(B.d_indptr), _ptr(B.d_indices), _ptr(feature_df(B)), 64,
                                   _ptr(hrank), _ptr(ws), ws_bytes, _stream()))
    LAUNCH_COUNTS["order"] += 3
    return hrank


def heavy_norms(M, hrank, row_begin=0, row_end=None, groups=False):
    """fp32 norm of rows [row_begin,row_end) of M over the heavy features, rounded up (sg_heavy_norms); with
    `groups` also the fp16 norms per group of heavy ranks (16 per row, csrc/sg_prune.cu): (norm, group_norms)."""
    t = require_cuda()
    L = _lib.load()
    row_end = M.shape[0] if row_end is None else row_end
    n = max(row_end - row_begin, 0)
    out = _empty(n, t.float32, M.device)
    grp = _empty(16 * n, t.float16, M.device) if groups else None
    _lib.check(L.sg_heavy_norms(row_begin, row_end, _ptr(M.d_indptr), _ptr(M.d_indices), _ptr(M.d_val32),
                                _ptr(hrank), _ptr(out), _ptr(grp), _stream()))
    LAUNCH_COUNTS["prune"] += 1
    return (out, grp) if groups else out


def row_order(M, hrank, row_begin=0, row_end=None, want_rank=True, row_norm=None, norm_scale=1.0):
    """(perm, rank) of rows [row_begin,row_end) of M sorted by (quantised heavy norm,) heavy-feature signature."""
    t = require_cuda()
    L = _lib.load()
    row_end = M.shape[0] if row_end is None else row_end
    n = max(row_end - row_begin, 0)
    perm = _empty(n, t.int32, M.device)
    rank = _empty(n, t.int32, M.device) if want_rank else None
    ws_bytes = int(L.sg_order_workspace_bytes(max(n, 1), M.shape[1]))
    ws = _empty(ws_bytes, t.uint8, M.device)
    _lib.check(L.sg_row_order(row_begin, row_end, _ptr(M.d_indptr), _ptr(M.d_indices), _ptr(hrank), _ptr(row_norm),
                              float(norm_scale), _ptr(perm), _ptr(rank), _ptr(ws), ws_bytes, _stream()))
    LAUNCH_COUNTS["order"] += 2
    return perm, rank


def right_order(B):
    """(hrank, perm, rank) of the right matrix: heavy features, rows sorted by (quantised heavy norm, signature)."""
    if B._order is None:
        hrank = heavy_features(B)
        B._heavy_norm, B._heavy_groups = heavy_norms(B, hrank, groups=True)
        perm, rank = row_order(B, hrank, row_norm=B._heavy_norm, norm_scale=1.0 / max(B.norm_bound, 1e-30))
        B._order = (hrank, perm, rank)
    return B._order


def right_tiles(B):
    """Tile blobs of the tile-centric K2 (csrc/sg_tiles.cu), cached on B: per 256-row tile of the processing order
    the postings sorted by feature, the bitmap directory and the bucket offsets as one blob (what the candidates
    kernel stages through TMA), the fp16 block maxima of every (feature, tile) and the per-tile pruning bound."""
    t = require_cuda()
    L = _lib.load()
    hrank, perm, rank = right_order(B)
    if B._tiles is None:
        n_rows, n_cols = B.shape
        W = int(L.sg_tiles_tile_w())
        T = int(L.sg_num_tiles(n_rows, W))
        Tp = int(L.sg_num_tiles_padded(n_rows, W))
        cap = int(L.sg_tiles_blob_bound(B.nnz, n_rows, n_cols))
        blob = _empty(cap, t.uint8, B.device)
        desc = _empty(2 * T, t.int64, B.device)
        maxw = _empty((n_cols + 1) * Tp, t.float16, B.device)
        maxima = t.zeros(2, dtype=t.int32, device=B.device)
        ws_bytes = int(L.sg_tiles_workspace_bytes(B.nnz, n_rows, n_cols))
        ws = _empty(ws_bytes, t.uint8, B.device)
        _lib.check(L.sg_tiles_build(n_rows, n_cols, B.nnz, _ptr(B.d_indptr), _ptr(B.d_indices), _ptr(B.d_val32),
                                    _ptr(rank), B.base, 1.0 / max(B.norm_bound, 1.0), _ptr(desc), _ptr(blob), cap,
                                    _ptr(maxw), _ptr(maxima), _ptr(ws), ws_bytes, _stream()))
        LAUNCH_COUNTS["tiles"] += 4
        bound = t.zeros(Tp, dtype=t.float32, device=B.device)
        _lib.check(L.sg_tile_bounds(n_rows, _ptr(perm), _ptr(B._heavy_norm), W, _ptr(bound), _stream()))
        LAUNCH_COUNTS["prune"] += 1
        B._tiles = {"desc": desc, "blob": blob, "maxw": maxw, "bound": bound, "maxima": maxima, "T": T, "W": W,
                    "stage_bytes": None}
    return B._tiles


def right_side(B, tile_w):
    """Row order (heavy norm, signature), feature-major bucketed postings, bucket directory with block maxima and
    per-tile pruning bounds of the right matrix, cached on B."""
    t = require_cuda()
    L = _lib.load()
    hrank, perm, rank = right_order(B)
    if tile_w not in B._postings2:
        n_rows, n_cols = B.shape
        T = int(L.sg_num_tiles(n_rows, tile_w))
        nb = T * (n_cols + 1) + 1
        if nb >= 2**31 - 1:
            raise OverflowError("posting bucket table too large: %d features x %d tiles" % (n_cols, T))
        Tp = int(L.sg_num_tiles_padded(n_rows, tile_w))
        bucket_ptr = _empty(nb, t.int32, B.device)
        bucket_dir = _empty(2 * nb, t.int32, B.device)
        bucket_maxw = _empty((n_cols + 1) * Tp, t.float16, B.device)
        post = _empty(max(B.nnz, 1), t.int32, B.device)
        ws_bytes = int(L.sg_postings_workspace_bytes(B.nnz, n_cols, T))
        ws = _empty(ws_bytes, t.uint8, B.device)
        _lib.check(L.sg_postings_build(n_rows, n_cols, B.nnz, _ptr(B.d_indptr), _ptr(B.d_indices), _ptr(B.d_val32),
                                       _ptr(rank), tile_w, B.base, 1.0 / max(B.norm_bound, 1.0), _ptr(bucket_ptr),
                                       _ptr(bucket_dir), _ptr(bucket_maxw), _ptr(post),
                                       _ptr(ws), ws_bytes, _stream()))
        LAUNCH_COUNTS["postings"] += 4
        bound = t.zeros(Tp, dtype=t.float32, device=B.device)
        _lib.check(L.sg_tile_bounds(n_rows, _ptr(perm), _ptr(B._heavy_norm), tile_w, _ptr(bound), _stream()))
        LAUNCH_COUNTS["prune"] += 1
        B._postings2[tile_w] = (bucket_dir, bucket_maxw, post, T, bound)     # bucket_ptr is only needed for the build
    return (hrank, perm, rank) + B._postings2[tile_w]


class DeviceMatches:
    """Result of the top-n product in HBM: COO triples ordered by (row asc, score desc)
    or, after symmetrize(), by (row asc, col asc).  Lazily materialises the scipy CSR that
    StringGrouper._build_matches returns in the reference (string_grouper.py:709-752)."""

    def __init__(self, shape, row, col, score, nnz, max_row, out_dtype=np.float64, indptr=None):
        self.shape = (int(shape[0]), int(shape[1]))
        self.d_row, self.d_col, self.d_score, self.d_indptr = row, col, score, indptr
        self.nnz = int(nnz)
        self.max_row = int(max_row)
        self.out_dtype = np.dtype(out_dtype)
        self._host = None
        self.pending_fix_diagonal = False
        self.pending_mirror = False

    def with_pending(self, fix_diagonal=False, mirror=False):
        """Record a post-processing step (StringGrouper._fix_diagonal / _symmetrize_matrix); the fused K4
        launch happens in apply_pending()."""
        self.pending_fix_diagonal |= bool(fix_diagonal)
        self.pending_mirror |= bool(mirror)
        return self

    def host_triples(self):
        """(row int64, col int64, score f64) on the host; the widening to the reference's int64 columns
        (string_grouper.py:759-763) happens on the device."""
        n = self.nnz
        t = torch()
        return tuple(to_host(self.d_row[:n].to(t.int64), self.d_col[:n].to(t.int64), self.d_score[:n]))

    def to_scipy(self):
        if self._host is None:
            from scipy.sparse import csr_matrix
            r, c, s = self.host_triples()
            indptr = np.zeros(self.shape[0] + 1, dtype=np.int64)
            np.cumsum(np.bincount(r, minlength=self.shape[0]), out=indptr[1:])
            idx_dtype = np.int32 if max(self.shape) < 2**31 and self.nnz < 2**31 else np.int64
            self._host = csr_matrix((s.astype(self.out_dtype, copy=False), c.astype(idx_dtype),
                                     indptr.astype(idx_dtype)), shape=self.shape)
        return self._host

    def get_shape(self):
        return self.shape

    def toarray(self):
        return self.to_scipy().toarray()

    def __getattr__(self, name):
        if name in _SCIPY_CSR_ATTRS:
            return getattr(self.to_scipy(), name)
        raise AttributeError("%s has no attribute %r" % (type(self).__name__, name))

    # operators scipy matrices answer; they materialise the host copy like the attributes above
    def __getitem__(self, key):
        return self.to_scipy()[key]

    def __matmul__(self, other):
        return self.to_scipy() @ other

    def __sub__(self, other):
        return self.to_scipy() - (other.to_scipy() if hasattr(other, "to_scipy") else other)

    def __ne__(self, other):
        return self.to_scipy() != (other.to_scipy() if hasattr(other, "to_scipy") else other)

    __hash__ = object.__hash__


def pick_tile(n_right, tile_w=None, warps=None, acc_bytes=4, n_left=None):
    """Column-tile width and warps per CTA.  Default: 512-byte accumulator tiles (256 columns of 16-bit fixed
    point): narrow tiles make the block-max test skip most (row, tile) pairs, and the test itself costs a
    fraction of an instruction per pair."""
    warps = int(warps or DEFAULT_WARPS)
    # 128-column tiles from a few 10^5 right rows on (the block-max test skips more; 663k on H100, 12 MB groups: 45.5-45.9 ms for the
    # candidates kernel vs 46.1-46.9 at 256 columns), 256-column tiles below (fewer directory entries to build, which
    # is not worth it for a small block of left rows, e.g. one of 8 shards)
    many_left = n_left is None or int(n_left) >= 150_000
    auto_w = 128 if (acc_bytes == 4 or (int(n_right) >= 400_000 and many_left)) else 256
    tile_w = int(tile_w or DEFAULT_TILE_W) or auto_w
    q = 256 // acc_bytes                               # tile bytes must be a multiple of 256
    need = ((max(int(n_right), 1) + q - 1) // q) * q
    tile_w = max(q, min(tile_w, 32768) // q * q)
    return min(tile_w, need), warps


def feature_df(B):
    """int32 document frequency of every feature of B (cached): the postings walked per use of the feature."""
    if B._df is None:
        t = require_cuda()
        L = _lib.load()
        df = _empty(B.shape[1], t.int32, B.device)
        _lib.check(L.sg_feature_df(B.shape[0], B.shape[1], _ptr(B.d_indptr), _ptr(B.d_indices), _ptr(df), _stream()))
        LAUNCH_COUNTS["prune"] += 1
        B._df = df
    return B._df


def prune_left(A, B, hrank, row_begin, row_end, threshold, margin, margin_per_feature, frac):
    """Exact threshold pruning of rows [row_begin,row_end) of A against B (sg_prune_rows); only B's heavy
    features (hrank >= 0) are prunable.  Returns (indices, val32, row_len, row_threshold, pruned_norm,
    pruned_group_norms) device arrays indexed like A's own."""
    t = require_cuda()
    L = _lib.load()
    df = feature_df(B)
    p_idx = t.empty_like(A.d_indices)
    p_val = t.empty_like(A.d_val32)
    p_len = _empty(A.shape[0], t.int32, A.device)
    p_thr = _empty(A.shape[0], t.float32, A.device)
    p_xp = _empty(A.shape[0], t.float32, A.device)
    p_xg = _empty(16 * A.shape[0], t.float16, A.device)     # |x_P| per group of heavy ranks
    budget = max(float(frac) * (float(threshold) - margin), 0.0)
    # the kernel works on left weights as stored and right rows of norm <= B.norm_bound
    _lib.check(L.sg_prune_rows(row_begin, row_end, _ptr(A.d_indptr), _ptr(A.d_indices), _ptr(A.d_val32), _ptr(df),
                               _ptr(hrank), float(B.norm_bound), budget, float(threshold), float(margin),
                               float(margin_per_feature), _ptr(p_idx), _ptr(p_val), _ptr(p_len), _ptr(p_thr),
                               _ptr(p_xp), _ptr(p_xg), _stream()))
    LAUNCH_COUNTS["prune"] += 1
    return p_idx, p_val, p_len, p_thr, p_xp, p_xg


def cossim_topn(A, B, top_n, threshold, row_begin=0, row_end=None, tile_w=None, warps=None, stats=None,
                prune=None, acc=None, kernel=None):
    """C[i,:] = top_n{ j : A_i . B_j > threshold } for rows [row_begin,row_end) of A.

    Device counterpart of the whole block loop of StringGrouper._build_matches
    (string_grouper.py:734-750).  Returns DeviceMatches with absolute row ids.
    """
    t = require_cuda()
    L = _lib.load()
    if A.shape[1] != B.shape[1]:
        raise ValueError("dimension mismatch: left has %d features, right has %d" % (A.shape[1], B.shape[1]))
    if A.dtype != B.dtype:
        raise TypeError("left and right matrices must have the same dtype")
    n_left, n_right = A.shape[0], B.shape[0]
    row_end = n_left if row_end is None else int(row_end)
    row_begin = int(row_begin)
    n_rows = max(row_end - row_begin, 0)
    dev = A.device
    top_n = int(min(int(top_n), n_right))
    dt = _lib.SG_DTYPE_F32 if A.dtype == np.float32 else _lib.SG_DTYPE_F64
    shape = (n_left, n_right)
    if n_rows == 0 or n_right == 0 or top_n <= 0 or A.nnz == 0 or B.nnz == 0:
        z32 = _empty(1, t.int32, dev)
        return DeviceMatches(shape, z32, z32, _empty(1, t.float64, dev), 0, 0)

    mark(stats, "k2_start")
    scale = A.norm_bound * B.norm_bound
    margin = CAND_MARGIN * max(scale, 1.0)
    thr_c = max(float(threshold) - margin, 0.0)
    # fixed-point accumulator tiles need non-negative weights and scores below 2 (K1's L2-normalised rows)
    acc = (acc or ACC_DTYPE).lower()
    if acc not in ("u16", "f32"):
        raise ValueError("accumulator dtype must be 'u16' or 'f32', got %r" % (acc,))
    if not (A.nonneg and B.nonneg and scale <= 1.0 + 1e-6) or thr_c < 0.05:
        acc = "f32"      # also near-zero thresholds: a tiny positive score must not round to a fixed-point zero
    acc_code = _lib.SG_ACC_U16 if acc == "u16" else _lib.SG_ACC_F32
    margin_pf = U16_MARGIN_PER_FEATURE if acc == "u16" else 0.0
    # tile-centric kernel: fixed-point products need what the u16 tiles need; the bitmap directory bounds the features
    kernel = (kernel or K2_KERNEL).lower()
    if kernel not in ("tiles", "row"):
        raise ValueError("kernel must be 'tiles' or 'row', got %r" % (kernel,))
    use_tiles = kernel == "tiles" and acc == "u16" and B.shape[1] <= int(L.sg_tiles_max_cols())
    tiles = None
    if use_tiles:
        tiles = right_tiles(B)
        if tiles["stage_bytes"] is None:
            tiles["stage_bytes"] = int(tiles["maxima"][0].item())       # one read-back per right matrix
        smem_optin = t.cuda.get_device_properties(dev).shared_memory_per_block_optin
        tile_warps = next((w for w in (TILE_WARPS, 8) if w in (8, 16) and
                           int(L.sg_tiles_smem_bytes(tiles["stage_bytes"], w)) <= smem_optin), None)
        if tile_warps is None:
            use_tiles, tiles = False, None          # a tile's index does not fit shared memory: row kernel
    if use_tiles:
        margin = TILE_MARGIN * max(scale, 1.0)
        margin_pf = TILE_MARGIN_PER_FEATURE
    prune_auto = prune is None          # the caller left the level open: it may be lowered, see below
    prune = PRUNE_FRAC if prune is None else float(prune)
    counters = t.zeros(4, dtype=t.int64, device=dev)       # [0] cand_count, [1] work queue
    # candidate buffer: clusters of identical names make this much larger than top_n * rows (37 M for the
    # 663k benchmark corpus); a second launch with the exact size happens only if this guess is too small
    cap = int(os.environ.get("SG_B200_CAND_CAP", 0)) or min(96 * n_rows + (1 << 22), 1 << 30)
    # both operands in the same processing order (quantised heavy norm, heavy-feature signature): neighbouring left
    # rows stream the same buckets, and the rows of a column tile have similar heavy norms (tight per-tile bound)
    if use_tiles:
        hrank, perm_b, _ = right_order(B)
        tile_w, warps, T, tile_bound = tiles["W"], tile_warps, tiles["T"], tiles["bound"]
        tiles_per_group = 0
        lpack = _empty(2 * A.d_indices.numel(), t.int32, dev)
        mask_words = int(L.sg_tiles_mask_words(n_right))
    else:
        tile_w, warps = pick_tile(n_right, tile_w, warps, 2 if acc == "u16" else 4, n_left=n_rows)
        # the bucket directory holds one entry per (feature, tile): widen the tiles until it stays below MAX_BUCKETS
        while (-(-n_right // tile_w)) * (B.shape[1] + 1) > MAX_BUCKETS and tile_w < 32768:
            tile_w *= 2
        hrank, perm_b, _, bucket_dir, bucket_maxw, post, T, tile_bound = right_side(B, tile_w)
        # column tiles per work group (a multiple of 64): the group's posting buckets should stay L2-resident
        tiles_per_group = max(64, int(GROUP_BYTES // max(4 * B.nnz / T, 1)) // 64 * 64)
    if A is B and row_begin == 0 and row_end == n_left:
        perm_a = perm_b
    else:
        perm_a, _ = row_order(A, hrank, row_begin, row_end, want_rank=False)
    mark(stats, "right_side")
    c_count = ctypes.c_void_p(counters.data_ptr())
    c_queue = ctypes.c_void_p(counters.data_ptr() + 8)
    c_walk = ctypes.c_void_p(counters.data_ptr() + 16)
    dummy = _empty(1, t.int32, dev)
    pruned = {}

    def launch_tiles(perm, n, row_buf, col_buf, capacity):
        """pack the pruned rows of `perm`, block-max filter -> survivor bits, tile kernel"""
        l_idx, l_val, l_len, l_thr, l_xp, _ = pruned["arrays"]
        stride = (n + 31) // 32 * 32
        rowinfo = _empty(4 * stride, t.int32, dev)
        mask = _empty(mask_words * stride, t.int32, dev)
        counters.zero_()
        _lib.check(L.sg_tiles_pack_left(n, _ptr(perm), 0, _ptr(A.d_indptr), _ptr(l_len), _ptr(l_idx), _ptr(l_val),
                                        _ptr(l_thr), _ptr(l_xp), max(B.norm_bound, 1.0), _ptr(lpack), _ptr(rowinfo),
                                        _stream()))
        _lib.check(L.sg_tiles_filter(n, _ptr(rowinfo), _ptr(lpack), _ptr(tiles["maxw"]), n_right, _ptr(tile_bound),
                                     _ptr(mask), stride, _stream()))
        _lib.check(L.sg_tiles_candidates(_ptr(perm), n, 0, _ptr(rowinfo), _ptr(lpack), _ptr(mask), stride,
                                         _ptr(tiles["desc"]), _ptr(tiles["blob"]), n_right, B.shape[1],
                                         _ptr(tile_bound), _ptr(perm_b), tiles["stage_bytes"], _ptr(row_buf),
                                         _ptr(col_buf), capacity, c_count, c_queue, c_walk, warps, _stream()))
        LAUNCH_COUNTS["tiles"] += 3

    def launch(perm, rb, re_, row_buf, col_buf, capacity, partial_buf=None):
        if use_tiles:
            return launch_tiles(perm, re_ - rb, row_buf, col_buf, capacity)
        l_idx, l_val, l_len, l_thr, l_xp, _ = pruned["arrays"]
        counters.zero_()
        _lib.check(L.sg_cossim_candidates(
            _ptr(A.d_indptr), _ptr(l_len), _ptr(l_idx), _ptr(l_val), rb, re_, _ptr(perm), n_right,
            A.shape[1], _ptr(bucket_dir), _ptr(bucket_maxw), _ptr(post), _ptr(perm_b), tile_w, acc_code,
            max(B.norm_bound, 1.0),
            thr_c, _ptr(l_thr), _ptr(l_xp), _ptr(tile_bound), tiles_per_group, _ptr(row_buf), _ptr(col_buf),
            _ptr(partial_buf), capacity, c_count, c_queue, warps, _stream()))
        LAUNCH_COUNTS["candidates"] += 1

    # Exact threshold pruning of the left rows (the fixed-point tile always takes per-row thresholds: its margin
    # grows with the number of features added).  A counting pass over a sample of the rows (in processing order,
    # so clusters of identical names are sampled in proportion) sizes the candidate buffers; when the caller left
    # the pruning level open and the sample reports more than MAX_CAND_DENSITY candidates per (row, column) pair,
    # the level is lowered: every candidate costs an exact re-score, every skipped posting saves one update.
    levels = [prune]
    if prune_auto and prune > 0.0 and thr_c > 0.0:
        levels = [prune, 0.75 * prune, 0.5 * prune, 0.25 * prune, 0.0]

    def prepare(level):
        if (level > 0.0 and thr_c > 0.0) or margin_pf > 0.0:
            pruned["arrays"] = prune_left(A, B, hrank, row_begin, row_end, float(threshold), margin, margin_pf,
                                          level if thr_c > 0.0 else 0.0)
        else:
            pruned["arrays"] = (A.d_indices, A.d_val32, None, None, None, None)

    def timed_launch(perm, rb, re_, row_buf, col_buf, capacity, partial_buf=None):
        if _timed(stats):
            ev0, ev1 = t.cuda.Event(enable_timing=True), t.cuda.Event(enable_timing=True)
            ev0.record()
        launch(perm, rb, re_, row_buf, col_buf, capacity, partial_buf)
        if _timed(stats):
            ev1.record()
            stats.setdefault("candidate_events", []).append((ev0, ev1))
        head = counters[:4].cpu().numpy()
        if use_tiles and stats is not None:
            stats["pairs_walked"] = stats.get("pairs_walked", 0) + int(head[2])
            stats["postings_walked"] = stats.get("postings_walked", 0) + int(head[3])
        return int(head[0])

    fixed_cap = bool(os.environ.get("SG_B200_CAND_CAP"))
    sample = None
    if not fixed_cap and n_rows >= 65536:
        stride = max(64, n_rows // 8192)
        sample = perm_a[:n_rows:stride].contiguous()
    est = None
    first = None          # (cand_row, cand_col, n_cand) of a whole-range launch that needed no sizing pass
    search = True
    dense = MAX_CAND_DENSITY * n_rows * n_right
    # The sizing pass is latency-bound (a few thousand rows against every column tile, cold: 2-3 ms whatever the
    # shard).  While a wasted launch costs no more than a few tens of ms, launch everything at once at the first
    # level into buffers of the density limit; only an overflow or a count above the limit falls back to the
    # sample / level search / row chunks below, and then the exact count of the first level is already known.
    # Candidates of the fixed-point row kernel carry their partial score: sg_rescore_refined re-tests each with the
    # grouped bound (csrc/sg_prune.cu) before its right row is read.
    refine = REFINE and not use_tiles and acc == "u16" and margin_pf > 0.0
    if not fixed_cap and float(n_rows) * float(n_right) <= OPTIMISTIC_PAIRS:
        prune = levels[0]
        prepare(prune)
        cap0 = int(min(int(dense) + (1 << 22), CAND_CHUNK))
        cand_row0 = _empty(cap0, t.int32, dev)
        cand_col0 = _empty(cap0, t.int32, dev)
        cand_part0 = _empty(cap0, t.float32, dev) if refine else None
        mark(stats, "prune_sample")
        n0 = timed_launch(perm_a, row_begin, row_end, cand_row0, cand_col0, cap0, cand_part0)
        mark(stats, "candidates")
        too_dense = len(levels) > 1 and sample is not None and n0 > dense
        if n0 <= cap0 and not too_dense:
            first = (cand_row0, cand_col0, cand_part0, n0)
            search = False
        else:
            del cand_row0, cand_col0, cand_part0
            if _timed(stats):
                stats["wasted_launch"] = True
            if too_dense:
                levels = levels[1:]
            else:
                est, search = n0, False          # stay at this level: chunks / buffers from the exact count
    if search:
        for level in levels:
            prepare(level)
            prune = level
            if sample is None:
                break
            launch(sample, row_begin, row_begin + int(sample.numel()), dummy, dummy, 0)
            est = int(counters[0].item()) * stride
            if est <= dense:
                break
    l_idx, l_val, l_len, l_thr, l_xp, l_xg = pruned["arrays"]
    mark(stats, "prune_sample")
    if stats is not None:
        stats["prune"], stats["acc"] = prune, acc
        stats["kernel"] = "tiles" if use_tiles else "row"
        stats["n_candidates_estimate"] = est
        if stats.get("count_macs") and l_len is not None:
            df = feature_df(B).long()
            pos = t.arange(A.d_indices.numel(), device=dev)
            rid = t.searchsorted(A.d_indptr[:n_left + 1].contiguous(), pos, right=True) - 1
            ok = (rid >= row_begin) & (rid < row_end)
            rid = rid.clamp(0, n_left - 1)
            live = ok & ((pos - A.d_indptr[rid]) < l_len[rid].long())
            stats["macs_walked"] = int(df[l_idx.long().clamp(0, A.shape[1] - 1)][live].sum().item())
            stats["features_kept"] = int(live.sum().item())

    # Left rows are taken in chunks (slices of the processing order) whose candidates fit CAND_CHUNK entries;
    # every chunk is re-scored exactly right away and only the pairs strictly above the threshold are kept.
    n_chunks = 1 if est is None else max(1, -(-int(1.3 * est) // CAND_CHUNK))
    rows_per_chunk = -(-n_rows // n_chunks)
    kept = []
    n_cand_total = 0
    max_row_cnt = 0
    row_cnt = t.zeros(n_rows + 1, dtype=t.int32, device=dev)      # survivors per left row (sg_rescore)
    for lo in range(0, n_rows, rows_per_chunk):
        hi = min(lo + rows_per_chunk, n_rows)
        perm_chunk = perm_a if (lo == 0 and hi == n_rows) else perm_a[lo:hi]
        if est is not None:
            cap = min(max(int(1.3 * est * (hi - lo) / n_rows) + (1 << 22), 1 << 22), 1 << 31)
        for attempt in range(3):
            if first is not None:
                cand_row, cand_col, cand_part, n_cand = first
                first = None
                break
            cand_row = _empty(cap, t.int32, dev)
            cand_col = _empty(cap, t.int32, dev)
            cand_part = _empty(cap, t.float32, dev) if refine else None
            n_cand = timed_launch(perm_chunk, row_begin, row_begin + (hi - lo), cand_row, cand_col, cap, cand_part)
            if n_cand <= cap:
                break
            if n_cand * 24 > t.cuda.get_device_properties(dev).total_memory // 2:
                raise OverflowError("%d candidate pairs above the threshold do not fit the candidate buffer; "
                                    "raise min_similarity or split the input" % n_cand)
            cap = n_cand
        else:
            raise OverflowError("candidate buffer overflow")
        n_cand_total += n_cand
        mark(stats, "candidates")
        # exact scores; only the candidates strictly above the threshold go on to the selection sorts
        score = _empty(n_cand, t.float64, dev)
        keep_row = _empty(n_cand, t.int32, dev)
        keep_col = _empty(n_cand, t.int32, dev)
        counters.zero_()
        if refine and cand_part is not None and l_xg is not None:
            _lib.check(L.sg_rescore_refined(n_cand, _ptr(cand_row), _ptr(cand_col), _ptr(cand_part), _ptr(l_xg),
                                            _ptr(B._heavy_groups), _ptr(l_thr), _ptr(A.d_indptr), _ptr(A.d_indices),
                                            _ptr(A.d_val), _ptr(B.d_indptr), _ptr(B.d_indices), _ptr(B.d_val), dt,
                                            _ptr(score), float(threshold), _ptr(keep_row), _ptr(keep_col), c_count,
                                            c_walk, _ptr(row_cnt), row_begin, _stream()))
        else:
            _lib.check(L.sg_rescore(n_cand, _ptr(cand_row), _ptr(cand_col), _ptr(A.d_indptr), _ptr(A.d_indices),
                                    _ptr(A.d_val), _ptr(B.d_indptr), _ptr(B.d_indices), _ptr(B.d_val), dt,
                                    _ptr(score), float(threshold), _ptr(keep_row), _ptr(keep_col), c_count,
                                    _ptr(row_cnt), row_begin, _stream()))
        LAUNCH_COUNTS["rescore"] += 1
        if lo + rows_per_chunk >= n_rows:      # last chunk: the largest row rides along with the read-back
            _lib.check(L.sg_row_count_max(n_rows, _ptr(row_cnt), c_queue, _stream()))      # counters[1], zeroed above
        head = counters[:3].cpu().numpy()
        n_keep, max_row_cnt = int(head[0]), int(head[1])
        if refine and stats is not None:
            stats["n_refined"] = stats.get("n_refined", 0) + int(head[2])
        mark(stats, "rescore")
        if n_chunks > 1:      # release the chunk-sized buffers, keep the survivors
            keep_row, keep_col, score = keep_row[:n_keep].clone(), keep_col[:n_keep].clone(), score[:n_keep].clone()
        kept.append((keep_row, keep_col, score, n_keep))
        del cand_row, cand_col, cand_part
    if len(kept) == 1:
        cand_row, cand_col, score, n_cand = kept[0]
    else:
        n_cand = sum(k[3] for k in kept)
        cand_row = t.cat([k[0][:k[3]] for k in kept]) if n_cand else _empty(1, t.int32, dev)
        cand_col = t.cat([k[1][:k[3]] for k in kept]) if n_cand else _empty(1, t.int32, dev)
        score = t.cat([k[2][:k[3]] for k in kept]) if n_cand else _empty(1, t.float64, dev)
    del kept
    if stats is not None:
        stats["n_candidates"] = n_cand_total
        stats["n_above_threshold"] = n_cand
        stats["n_row_chunks"] = n_chunks
        stats["tile_w"], stats["warps"], stats["n_tiles"] = tile_w, warps, T
        stats["tiles_per_group"] = tiles_per_group
        if use_tiles:
            stats["stage_bytes"] = tiles["stage_bytes"]

    out_indptr = _empty(n_rows + 1, t.int64, dev)
    out_row = _empty(n_cand, t.int32, dev)
    out_col = _empty(n_cand, t.int32, dev)
    out_score = _empty(n_cand, t.float64, dev)
    tail = t.zeros(2, dtype=t.int64, device=dev)            # [0] out_nnz, [1] max_row (int32 view)
    rows_cap = int(L.sg_topn_rows_cap())
    if (top_n <= 32 or max_row_cnt <= rows_cap or top_n <= rows_cap // 2) and SELECT_MODE != "sort":
        # survivors bucketed by row, every row ranked on its own (warp shuffle network / one CTA in shared memory)
        ws_bytes = int(L.sg_topn_select_rows_workspace_bytes(n_cand, n_rows))
        ws = _empty(ws_bytes, t.uint8, dev)
        _lib.check(L.sg_topn_select_rows(n_cand, _ptr(cand_row), _ptr(cand_col), _ptr(score), row_begin, n_rows, top_n,
                                         _ptr(row_cnt), _ptr(out_indptr), _ptr(out_row), _ptr(out_col),
                                         _ptr(out_score), ctypes.c_void_p(tail.data_ptr()),
                                         ctypes.c_void_p(tail.data_ptr() + 8), _ptr(ws), ws_bytes, _stream()))
        LAUNCH_COUNTS["select"] += 6
        if stats is not None:
            stats["select"] = "rows"
    else:
        # a row with more survivors than one CTA ranks in shared memory: three global radix sorts
        ws_bytes = int(L.sg_topn_select_workspace_bytes(n_cand, n_rows))
        ws = _empty(ws_bytes, t.uint8, dev)
        _lib.check(L.sg_topn_select(n_cand, _ptr(cand_row), _ptr(cand_col), _ptr(score), row_begin, n_rows, top_n,
                                    float(threshold), _ptr(out_indptr), _ptr(out_row), _ptr(out_col), _ptr(out_score),
                                    ctypes.c_void_p(tail.data_ptr()), ctypes.c_void_p(tail.data_ptr() + 8), _ptr(ws),
                                    ws_bytes, _stream()))
        LAUNCH_COUNTS["select"] += 7
        if stats is not None:
            stats["select"] = "sort"
    th = tail.cpu().numpy()
    mark(stats, "select")
    nnz = int(th[0])
    max_row = int(th[1:2].view(np.int32)[0])
    return DeviceMatches(shape, out_row, out_col, out_score, nnz, max_row, indptr=out_indptr)


def symmetrize(M, fix_diagonal=True, mirror=True):
    """diag := 1 (fix_diagonal), pattern := pattern U pattern^T (mirror), rows ordered by column
    (string_grouper.py:419-427, :955-964) on the device."""
    t = require_cuda()
    L = _lib.load()
    n = M.shape[0]
    dev = M.d_row.device
    flags = (_lib.SG_SYMM_FIX_DIAGONAL if fix_diagonal else 0) | (_lib.SG_SYMM_MIRROR if mirror else 0)
    cap = 2 * M.nnz + n
    out_row = _empty(cap, t.int32, dev)
    out_col = _empty(cap, t.int32, dev)
    out_score = _empty(cap, t.float64, dev)
    out_nnz = t.zeros(1, dtype=t.int64, device=dev)
    ws_bytes = int(L.sg_symmetrize_workspace_bytes(M.nnz, n))
    ws = _empty(ws_bytes, t.uint8, dev)
    _lib.check(L.sg_symmetrize(n, M.nnz, flags, _ptr(M.d_row), _ptr(M.d_col), _ptr(M.d_score), _ptr(out_row),
                               _ptr(out_col), _ptr(out_score), _ptr(out_nnz), _ptr(ws), ws_bytes, _stream()))
    LAUNCH_COUNTS["symmetrize"] += 3
    nnz = int(out_nnz.item())
    return DeviceMatches(M.shape, out_row, out_col, out_score, nnz, M.max_row, out_dtype=M.out_dtype)


def group_reps(M, n, centroid, keep_device=False):
    """Representative index of every string's group from the (row, col)-sorted device match list
    (StringGrouper._deduplicate, string_grouper.py:851-904).  keep_device: also return the int32 device tensor
    (positions for the device string gather)."""
    t = require_cuda()
    L = _lib.load()
    dev = M.d_row.device
    rep = _empty(n, t.int32, dev)
    ws_bytes = int(L.sg_group_reps_workspace_bytes(n))
    ws = _empty(ws_bytes, t.uint8, dev)
    _lib.check(L.sg_group_reps(n, M.nnz, _ptr(M.d_row), _ptr(M.d_col), _ptr(M.d_score), 1 if centroid else 0,
                               _ptr(rep), _ptr(ws), ws_bytes, _stream()))
    LAUNCH_COUNTS["groups"] += 6
    host = rep[:n].cpu().numpy().astype(np.int64)
    return (host, rep) if keep_device else host


def nearest_master(M, n_right):
    """int64 [n_right]: for every right row the left row of its best match (smallest index among equal scores),
    -1 without a match — the reduction of StringGrouper._get_nearest_matches (string_grouper.py:803-807)."""
    t = require_cuda()
    L = _lib.load()
    dev = M.d_row.device
    best = _empty(n_right, t.int32, dev)
    ws_bytes = int(L.sg_nearest_master_workspace_bytes(n_right))
    ws = _empty(ws_bytes, t.uint8, dev)
    _lib.check(L.sg_nearest_master(M.nnz, _ptr(M.d_row), _ptr(M.d_col), _ptr(M.d_score), n_right, _ptr(best), _ptr(ws),
                                   ws_bytes, _stream()))
    LAUNCH_COUNTS["groups"] += 3
    return best[:n_right].cpu().numpy().astype(np.int64)


class RawStrings:
    """Packed UTF-8 strings of master ++ duplicates as uploaded for K1, kept for the device string gather."""

    def __init__(self, d_bytes, d_off, n_master, n_docs):
        self.d_bytes, self.d_off, self.n_master, self.n_docs = d_bytes, d_off, int(n_master), int(n_docs)


def gather_strings(raw, sides):
    """For every (doc_base, positions, n_sel) in `sides`: (offsets int64 [n_sel+1], bytes uint8) on the host of the
    strings at `positions` (device int32) of the Series starting at document `doc_base` — the
    `Series.iloc[...]` of get_matches (string_grouper.py:462, :467).  Two synchronisations in total: the byte
    counts, then all offsets and bytes."""
    t = require_cuda()
    L = _lib.load()
    dev = raw.d_off.device
    offs = []
    for doc_base, positions, n_sel in sides:
        out_off = _empty(n_sel + 1, t.int64, dev)
        ws_bytes = int(L.sg_gather_workspace_bytes(n_sel))
        ws = _empty(ws_bytes, t.uint8, dev)
        _lib.check(L.sg_gather_offsets(_ptr(raw.d_off), int(doc_base), n_sel, _ptr(positions), _ptr(out_off),
                                       _ptr(ws), ws_bytes, _stream()))
        offs.append(out_off)
    totals = t.stack([o[n_sel] for o, (_, _, n_sel) in zip(offs, sides)]).cpu().numpy()
    datas = []
    for out_off, total, (doc_base, positions, n_sel) in zip(offs, totals, sides):
        out = _empty(int(total), t.uint8, dev)
        _lib.check(L.sg_gather_bytes(_ptr(raw.d_bytes), _ptr(raw.d_off), int(doc_base), n_sel, _ptr(positions),
                                     _ptr(out_off), _ptr(out), _stream()))
        LAUNCH_COUNTS["gather"] += 2
        datas.append(out[:int(total)])
    host = to_host(*([o[:n_sel + 1] for o, (_, _, n_sel) in zip(offs, sides)] + datas))
    k = len(sides)
    return [(host[i], host[k + i]) for i in range(k)]


def matches_from_scipy(m):
    """Upload a host CSR of matches (e.g. returned by a user-supplied _build_matches)."""
    t = require_cuda()
    m = m.tocsr()
    dev = t.device("cuda", t.cuda.current_device())
    # keep CSR storage order (value-descending inside a row for the reference's product)
    r2 = np.repeat(np.arange(m.shape[0], dtype=np.int32), np.diff(m.indptr))
    row = t.from_numpy(r2).to(dev)
    col = t.from_numpy(np.ascontiguousarray(m.indices, dtype=np.int32)).to(dev)
    score = t.from_numpy(np.ascontiguousarray(m.data, dtype=np.float64)).to(dev)
    max_row = int(np.diff(m.indptr).max()) if m.shape[0] else 0
    if row.numel() == 0:
        row = _empty(1, t.int32, dev)
        col = _empty(1, t.int32, dev)
        score = _empty(1, t.float64, dev)
    return DeviceMatches(m.shape, row, col, score, m.nnz, max_row, out_dtype=m.dtype)


def rowwise_dot(A, B):
    """StringGrouper.dot (string_grouper.py:433-440): row-wise similarity of two equal-shape matrices."""
    t = require_cuda()
    L = _lib.load()
    if A.shape != B.shape:
        raise ValueError("shape mismatch")
    out = _empty(A.shape[0], t.float64, A.device)
    dt = _lib.SG_DTYPE_F32 if A.dtype == np.float32 else _lib.SG_DTYPE_F64
    _lib.check(L.sg_rowwise_dot(A.shape[0], _ptr(A.d_indptr), _ptr(A.d_indices), _ptr(A.d_val), _ptr(B.d_indptr),
                                _ptr(B.d_indices), _ptr(B.d_val), dt, _ptr(out), _stream()))
    LAUNCH_COUNTS["rowdot"] += 1
    return out[:A.shape[0]].cpu().numpy().astype(A.dtype, copy=False)


class DeviceVocabulary:
    """df / rank tables of the fitted vectoriser (the device twin of TfidfVectorizer.vocabulary_ / idf_)."""

    def __init__(self, df_table, rank_table, ngram, n_docs, vocab_size):
        self.d_df, self.d_rank = df_table, rank_table
        self.ngram, self.n_docs, self.size = int(ngram), int(n_docs), int(vocab_size)

    def feature_names(self):
        """Sorted n-grams, column order of the TF-IDF matrices (sklearn get_feature_names_out)."""
        from ._ingest import decode_vocab_keys
        t = require_cuda()
        L = _lib.load()
        keys = _empty(self.size, t.int32, self.d_df.device)
        _lib.check(L.sg_tfidf_vocab_keys(_ptr(self.d_df), _ptr(self.d_rank), self.ngram, _ptr(keys), _stream()))
        return decode_vocab_keys(keys[:self.size].cpu().numpy().view(np.uint32), self.ngram)


def upload_strings(data, offsets, device=None):
    """H2D of the packed strings: (uint8 bytes, int64 offsets) -> device tensors."""
    t = require_cuda()
    device = device or t.device("cuda", t.cuda.current_device())
    total = int(offsets[-1])
    d_bytes = (t.from_numpy(np.ascontiguousarray(data)).to(device, non_blocking=True) if total
               else _empty(1, t.uint8, device))
    d_off = t.from_numpy(np.ascontiguousarray(offsets, dtype=np.int64)).to(device, non_blocking=True)
    return d_bytes, d_off, total


class DeviceVocabulary64:
    """Sorted vocabulary of the general vectoriser (csrc/sg_tfidf64.cu): 64-bit keys over a dense alphabet."""

    def __init__(self, keys, df, alphabet, bits, ngram, n_docs, vocab_size):
        self.d_keys, self.d_df, self.alphabet = keys, df, alphabet
        self.bits, self.ngram, self.n_docs, self.size = int(bits), int(ngram), int(n_docs), int(vocab_size)

    def feature_names(self):
        from ._ingest import decode_vocab_keys64
        keys = self.d_keys[:self.size].cpu().numpy().view(np.uint64)
        return decode_vocab_keys64(keys, self.ngram, self.bits, self.alphabet)


DENSE_KEY_BITS = 21      # the dense key table (2^(7n) slots) is used up to trigrams; beyond: sorted vocabulary


def tfidf_sorted(data, offsets, n_master, ngram, flags, dtype, device=None, stats=None):
    """K1, general form: 64-bit keys + sort-based vocabulary (ngram_size >= 4, or uint32 code points)."""
    from . import _ingest
    t = require_cuda()
    L = _lib.load()
    device = device or t.device("cuda", t.cuda.current_device())
    n_docs = len(offsets) - 1
    total = int(offsets[-1])
    raw_bytes = None
    if data.dtype == np.uint8:
        lut, alphabet = _ingest.byte_alphabet(data, flags)
        sym_width = 1
        d_sym = t.from_numpy(np.ascontiguousarray(data)).to(device) if total else _empty(1, t.uint8, device)
        d_lut = t.from_numpy(lut).to(device)
        raw_bytes = d_sym
    else:
        alphabet = np.unique(data)
        ids = np.searchsorted(alphabet, data).astype(np.uint32)
        sym_width = 4
        d_sym = t.from_numpy(ids.view(np.int32)).to(device) if total else _empty(1, t.int32, device)
        d_lut = None
    bits = _ingest.symbol_bits(len(alphabet))
    if int(ngram) * bits > 64:
        raise NotImplementedError(
            "ngram_size=%d over an alphabet of %d distinct characters needs %d-bit n-gram keys; the device vectoriser "
            "packs keys into 64 bits (ngram_size * ceil(log2(alphabet)) <= 64)" % (ngram, len(alphabet), ngram * bits))
    d_off = t.from_numpy(np.ascontiguousarray(offsets, dtype=np.int64)).to(device)
    TRANSFER_BYTES["h2d"] += int(total * sym_width + 8 * len(offsets))
    np_dtype = np.float32 if np.dtype(dtype) == np.float32 else np.float64
    s_clean = _empty(total, t.int32, device)
    s_sort = _empty(total, t.int64, device)
    s_key = _empty(total, t.int64, device)
    s_tf = _empty(total, t.int32, device)
    row_nnz = _empty(n_docs + 1, t.int32, device)
    _lib.check(L.sg_tfidf64_count(_ptr(d_sym), sym_width, _ptr(d_off), n_docs, int(ngram), bits, _ptr(d_lut),
                                  _ptr(s_clean), _ptr(s_sort), _ptr(s_key), _ptr(s_tf), _ptr(row_nnz), _stream()))
    indptr = _empty(n_docs + 1, t.int64, device)
    indices = _empty(total, t.int32, device)
    val32 = _empty(total, t.float32, device)
    val64 = _empty(total, t.float64, device) if np_dtype == np.float64 else None
    vocab_keys = _empty(total, t.int64, device)
    df = _empty(total, t.int32, device)
    tail = t.zeros(2, dtype=t.int64, device=device)         # [0] V (int32 view), [1] nnz
    ws_bytes = int(L.sg_tfidf64_finalize_workspace_bytes(n_docs, total))
    ws = _empty(ws_bytes, t.uint8, device)
    dt = _lib.SG_DTYPE_F32 if np_dtype == np.float32 else _lib.SG_DTYPE_F64
    _lib.check(L.sg_tfidf64_finalize(_ptr(d_off), n_docs, n_docs, total, int(ngram), bits, dt, _ptr(s_key), _ptr(s_tf),
                                     _ptr(row_nnz), _ptr(indptr), _ptr(indices), _ptr(val64), _ptr(val32),
                                     _ptr(vocab_keys), _ptr(df), ctypes.c_void_p(tail.data_ptr()),
                                     ctypes.c_void_p(tail.data_ptr() + 8), _ptr(ws), ws_bytes, _stream()))
    LAUNCH_COUNTS["tfidf"] += 7
    n_master = int(n_master)
    head = t.cat([tail, indptr[n_master:n_master + 1]]).cpu().numpy()
    V = int(head[0:1].view(np.int32)[0])
    nnz = int(head[1])
    split = int(head[2])
    val = val64 if np_dtype == np.float64 else val32
    vocab = DeviceVocabulary64(vocab_keys, df, alphabet, bits, ngram, n_docs, V)
    if stats is not None:
        stats.update(n_docs=n_docs, total_bytes=total, nnz=nnz, vocab=V, h2d_bytes=int(total * sym_width + 8 * len(offsets)),
                     vectoriser="sorted vocabulary, %d-bit keys" % (int(ngram) * bits))
        if raw_bytes is not None:
            stats["raw"] = RawStrings(raw_bytes, d_off, n_master, n_docs)
    master = DeviceCSR((n_master, V), indptr[:n_master + 1], indices, val, val32, split, np_dtype, 1.0, base=0)
    master.nnz_parent = nnz
    if n_master == n_docs:
        master._df = df[:max(V, 1)]       # fitted on exactly these rows: the vectoriser's df is sg_feature_df(master)
        return master, None, vocab
    dup = DeviceCSR((n_docs - n_master, V), indptr[n_master:], indices, val, val32, nnz - split, np_dtype, 1.0,
                    base=split)
    dup.nnz_parent = nnz
    return master, dup, vocab


def tfidf(data, offsets, n_master, ngram, flags, dtype, device=None, stats=None, df_allreduce=None, n_docs_fit=None):
    """K1 from host buffers: packed strings (master ++ duplicates) -> TF-IDF CSR in HBM.  uint8 `data` = ASCII bytes
    (dense key table up to trigrams), anything else goes through the sorted-vocabulary vectoriser."""
    if data.dtype != np.uint8 or 7 * int(ngram) > DENSE_KEY_BITS:
        if df_allreduce is not None:
            raise NotImplementedError("the sharded vectoriser (df all-reduce) needs ASCII text and ngram_size <= 3")
        return tfidf_sorted(data, offsets, n_master, ngram, flags, dtype, device=device, stats=stats)
    d_bytes, d_off, total = upload_strings(data, offsets, device)
    TRANSFER_BYTES["h2d"] += int(total + 8 * len(offsets))
    if stats is not None:
        stats["h2d_bytes"] = int(total + 8 * len(offsets))
        stats["raw"] = RawStrings(d_bytes, d_off, n_master, len(offsets) - 1)
    return tfidf_resident(d_bytes, d_off, len(offsets) - 1, total, n_master, ngram, flags, dtype, stats=stats,
                          df_allreduce=df_allreduce, n_docs_fit=n_docs_fit)


def tfidf_resident(d_bytes, d_off, n_docs, total, n_master, ngram, flags, dtype, stats=None, df_allreduce=None,
                   n_docs_fit=None):
    """K1 on strings already resident in HBM.

    Device counterpart of _fit_vectorizer + transform (string_grouper.py:685-707): the vocabulary /
    df / idf are fitted on ALL rows, then rows [0, n_master) form the master matrix and the rest the
    duplicate matrix (views of the same device arrays).  Returns (master, duplicates | None, vocab).
    """
    t = require_cuda()
    L = _lib.load()
    device = d_off.device
    slots = int(L.sg_tfidf_table_slots(int(ngram)))
    if slots < 0:
        raise NotImplementedError("ngram_size=%r: the device vectoriser supports 1 <= ngram_size <= 4" % (ngram,))
    np_dtype = np.float32 if np.dtype(dtype) == np.float32 else np.float64
    df = t.zeros(slots, dtype=t.int32, device=device)
    rank = _empty(slots, t.int32, device)
    s_clean = _empty(total, t.uint8, device)
    s_sort = _empty(total, t.int32, device)
    s_key = _empty(total, t.int32, device)
    s_tf = _empty(total, t.int32, device)
    row_nnz = _empty(n_docs + 1, t.int32, device)
    _lib.check(L.sg_tfidf_count(_ptr(d_bytes), _ptr(d_off), n_docs, int(ngram), int(flags), _ptr(df), _ptr(s_clean),
                                _ptr(s_sort), _ptr(s_key), _ptr(s_tf), _ptr(row_nnz), _stream()))
    if df_allreduce is not None:
        df_allreduce(df)          # corpus sharded over GPUs: document frequencies are summed over the ranks (NCCL)
    indptr = _empty(n_docs + 1, t.int64, device)
    indices = _empty(total, t.int32, device)
    val32 = _empty(total, t.float32, device)
    val64 = _empty(total, t.float64, device) if np_dtype == np.float64 else None
    tail = t.zeros(2, dtype=t.int64, device=device)         # [0] V (int32 view), [1] nnz
    ws_bytes = int(L.sg_tfidf_finalize_workspace_bytes(n_docs, int(ngram)))
    ws = _empty(ws_bytes, t.uint8, device)
    dt = _lib.SG_DTYPE_F32 if np_dtype == np.float32 else _lib.SG_DTYPE_F64
    _lib.check(L.sg_tfidf_finalize(_ptr(d_off), n_docs, int(n_docs if n_docs_fit is None else n_docs_fit), int(ngram),
                                   dt, _ptr(df), _ptr(rank), _ptr(s_key), _ptr(s_tf),
                                   _ptr(row_nnz), _ptr(indptr), _ptr(indices), _ptr(val64), _ptr(val32),
                                   ctypes.c_void_p(tail.data_ptr()), ctypes.c_void_p(tail.data_ptr() + 8), _ptr(ws),
                                   ws_bytes, _stream()))
    LAUNCH_COUNTS["tfidf"] += 4
    n_master = int(n_master)
    head = t.cat([tail, indptr[n_master:n_master + 1]]).cpu().numpy()     # one read-back: V, nnz, split point
    V = int(head[0:1].view(np.int32)[0])
    nnz = int(head[1])
    split = int(head[2])
    val = val64 if np_dtype == np.float64 else val32
    vocab = DeviceVocabulary(df, rank, ngram, n_docs if n_docs_fit is None else n_docs_fit, V)
    if stats is not None:
        stats.update(n_docs=n_docs, total_bytes=total, nnz=nnz, vocab=V)
    master = DeviceCSR((n_master, V), indptr[:n_master + 1], indices, val, val32, split, np_dtype, 1.0, base=0)
    master.nnz_parent = nnz
    if n_master == n_docs:
        if df_allreduce is None and n_docs_fit is None:
            # fitted on exactly these rows: the vectoriser's df, in column order, is sg_feature_df(master)
            col_df = _empty(max(V, 1), t.int32, device)
            _lib.check(L.sg_tfidf_vocab_df(_ptr(df), _ptr(rank), int(ngram), _ptr(col_df), _stream()))
            master._df = col_df
        return master, None, vocab
    dup = DeviceCSR((n_docs - n_master, V), indptr[n_master:], indices, val, val32, nnz - split, np_dtype, 1.0,
                    base=split)
    dup.nnz_parent = nnz
    return master, dup, vocab


def as_device_matches(m):
    return m if isinstance(m, DeviceMatches) else matches_from_scipy(m)


def empty_csr(like, n_rows):
    """A CSR block with `n_rows` empty rows on the device of `like` (ranks that own no rows of a sharded matrix)."""
    t = torch()
    dev = like.device
    val = _empty(1, t.float32 if like.dtype == np.float32 else t.float64, dev)
    val32 = val if like.dtype == np.float32 else _empty(1, t.float32, dev)
    return DeviceCSR((n_rows, like.shape[1]), t.zeros(n_rows + 1, dtype=t.int64, device=dev),
                     _empty(1, t.int32, dev), val, val32, 0, like.dtype, like.norm_bound)


def offset_rows(m, row_offset, n_rows_total):
    """Row ids of a per-rank block -> ids in the full left matrix."""
    if m.nnz:
        m.d_row[:m.nnz] += int(row_offset)
    return DeviceMatches((int(n_rows_total), m.shape[1]), m.d_row, m.d_col, m.d_score, m.nnz, m.max_row,
                         out_dtype=m.out_dtype)


def allgather_csr(M, n_rows_total):
    """Right matrix sharded by rows over the ranks (sharded K1) -> the full matrix on every rank (NCCL all-gather
    over NVLink of row lengths, indices and values)."""
    from . import _dist
    t = torch()
    n = M.shape[0]
    lo, hi = M.base, M.base + M.nnz
    row_len = (M.d_indptr[1:n + 1] - M.d_indptr[:n]).contiguous()
    vals = (M.d_val[lo:hi].contiguous(),) if M.d_val is M.d_val32 else (M.d_val[lo:hi].contiguous(),
                                                                         M.d_val32[lo:hi].contiguous())
    indptr, indices, gvals = _dist.allgather_csr_rows(row_len, M.d_indices[lo:hi].contiguous(), vals)
    nnz = int(indptr[-1].item())
    if nnz == 0:
        indices = _empty(1, t.int32, M.device)
        gvals = tuple(_empty(1, v.dtype, M.device) for v in vals)
    val = gvals[0]
    val32 = gvals[0] if len(gvals) == 1 else gvals[1]
    out = DeviceCSR((int(n_rows_total), M.shape[1]), indptr, indices, val, val32, nnz, M.dtype, M.norm_bound)
    return out


def gather_shards(m):
    """Multi-GPU: all-gather the per-rank top-n lists (each rank computed its own block of left rows) so that
    every rank holds the full result in row order; the `vstack` of string_grouper.py:750 over NVLink."""
    from . import _dist
    row, col, score, nnz, max_row = _dist.gather_matches(m.shape, m.d_row, m.d_col, m.d_score, m.nnz, m.max_row)
    t = torch()
    if nnz == 0:
        row, col, score = _empty(1, t.int32, row.device), _empty(1, t.int32, row.device), _empty(1, t.float64, row.device)
    return DeviceMatches(m.shape, row, col, score, nnz, max_row, out_dtype=m.out_dtype)


def apply_pending(m):
    """Run the recorded _fix_diagonal / _symmetrize_matrix steps as one K4 launch (string_grouper.py:419-427:
    the LIL round trip also re-orders every row by column, which K4 does even when only one step is set)."""
    m = as_device_matches(m)
    return symmetrize(m, fix_diagonal=m.pending_fix_diagonal, mirror=m.pending_mirror)
