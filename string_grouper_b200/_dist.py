"""Multi-GPU sharding of the hot path: one process per GPU (torchrun), torch.distributed for plumbing.

The block loop of StringGrouper._build_matches (string_grouper/string_grouper.py:734-750)
is data-parallel over LEFT row blocks (their results are only `vstack`ed, :750); right blocks need a
per-row merge (:746), so the right side is never split across GPUs.  Rank g owns the left rows
`define_chunks(n_left, world)[g]` (same ceil-sized chunking as :721-722), runs K2 on them against the
full right matrix, and the small per-rank top-n lists are all-gathered (variable length) so that every
rank holds the complete match list, in rank order == row order.  K1 runs redundantly on every rank
(the packed corpus is a few tens of MB); the only collective on the data path is the result gather.

Sharding is OPT-IN: an initialised default process group alone does not make fit() collective (the caller may be
inside somebody else's distributed job with rank-local data).  Set SG_B200_DISTRIBUTED=1 or call enable(); the
library then uses its own process group, checks that every rank was given the same input before it shards, and
exchanges an error flag before every collective so that a rank that failed locally takes the others down with a
clear exception instead of leaving them waiting.
"""
import contextlib
import os
import zlib

import numpy as np

_STATE = {"enabled": None, "group": None, "group_for": None}


def _dist():
    import torch.distributed as dist
    return dist


def enable(flag=True):
    """Switch the multi-GPU sharding of fit() on or off for this process (overrides SG_B200_DISTRIBUTED)."""
    _STATE["enabled"] = bool(flag)


def enabled():
    if _STATE["enabled"] is not None:
        return _STATE["enabled"]
    return os.environ.get("SG_B200_DISTRIBUTED", "0").lower() in ("1", "true", "yes", "on")


def group():
    """The library's own process group (all ranks of the default group), created on first use by every rank."""
    dist = _dist()
    default = dist.group.WORLD
    if _STATE["group"] is None or _STATE["group_for"] is not default:
        _STATE["group"] = dist.new_group(ranks=list(range(dist.get_world_size())))
        _STATE["group_for"] = default
    return _STATE["group"]


@contextlib.contextmanager
def local():
    """Inside the block world() is (0, 1): the work runs whole in this process, whatever the other ranks do."""
    saved = _STATE["enabled"]
    _STATE["enabled"] = False
    try:
        yield
    finally:
        _STATE["enabled"] = saved


def world():
    """(rank, world_size) to shard over; (0, 1) unless sharding was switched on and a process group exists."""
    try:
        dist = _dist()
        if enabled() and dist.is_available() and dist.is_initialized():
            return dist.get_rank(), dist.get_world_size()
    except Exception:
        pass
    return 0, 1


def result_on_all_ranks():
    """SG_B200_RESULT=all (default): every rank ends up with the full match list; =rank0: only rank 0 does (the
    others keep an empty list) — saves N-1 copies of the list over PCIe and N-1 DataFrame constructions."""
    return os.environ.get("SG_B200_RESULT", "all").lower() != "rank0"


def shard_range(n_rows, rank, world_size):
    """Rows of chunk `rank` when `n_rows` are split into `world_size` ceil-sized consecutive chunks
    (define_chunks, string_grouper.py:714-722); trailing chunks may be empty."""
    chunk = -(-int(n_rows) // int(world_size)) if n_rows > 0 else 0
    lo = min(rank * chunk, n_rows)
    hi = min(lo + chunk, n_rows)
    return lo, hi


def _device_for_collectives():
    import torch
    dist = _dist()
    if dist.get_backend(group()) == "nccl":
        return torch.device("cuda", torch.cuda.current_device())
    return torch.device("cpu")


def fingerprint(series_list):
    """A cheap fingerprint of the input Series (lengths, total characters, checksum of a sample of the strings)."""
    fp = []
    for s in series_list:
        n = len(s)
        take = s.iloc[np.unique(np.linspace(0, n - 1, num=min(n, 64)).astype(np.int64))] if n else s
        crc = zlib.crc32("\x00".join(take.tolist()).encode("utf-8", "surrogatepass"))
        fp += [n, int(crc)]
    return fp


def check_same_inputs(fp):
    """Raise ValueError on every rank when the ranks were not given the same input (sharding rank-local data would
    mix unrelated match lists)."""
    import torch
    dist = _dist()
    t = torch.tensor(fp, dtype=torch.int64, device=_device_for_collectives())
    hi, lo = t.clone(), t.clone()
    dist.all_reduce(hi, op=dist.ReduceOp.MAX, group=group())
    dist.all_reduce(lo, op=dist.ReduceOp.MIN, group=group())
    if not bool((hi == lo).all().item()):
        raise ValueError("string_grouper_b200: SG_B200_DISTRIBUTED is set but the ranks were given different input "
                         "Series; multi-GPU sharding needs the same master / duplicates on every rank")


def guarded(fn, *args, **kwargs):
    """Run the rank-local part `fn`; before anybody enters the next collective, all ranks learn whether one of them
    failed.  The failing rank re-raises its own exception, the others raise RuntimeError."""
    import torch
    dist = _dist()
    err, out = None, None
    try:
        out = fn(*args, **kwargs)
    except Exception as e:           # noqa: BLE001 — re-raised below, after the flag exchange
        err = e
    flag = torch.tensor([1 if err is not None else 0], dtype=torch.int32, device=_device_for_collectives())
    dist.all_reduce(flag, op=dist.ReduceOp.MAX, group=group())
    if err is not None:
        raise err
    if int(flag.item()):
        raise RuntimeError("string_grouper_b200: another rank failed in the rank-local part of fit(); see its traceback")
    return out


def allgather_varlen(tensors, extra=None):
    """All-gather a tuple of equally long 1-D tensors whose length differs per rank; `extra` (a small list of ints)
    rides along with the length exchange.

    Returns (tuple of concatenations in rank order, lengths, extras per rank).  One length exchange (the only host
    read-back), then ONE collective: the fields are packed into one byte buffer per rank; NCCL gathers the uneven
    buffers directly into pre-sized outputs, gloo (CPU tests) pads to the longest.
    """
    import torch
    dist = _dist()
    g = group()
    ws = dist.get_world_size(g)
    n = int(tensors[0].numel())
    dev = tensors[0].device
    extra = list(extra or [])
    head = torch.zeros(ws * (1 + len(extra)), dtype=torch.int64, device=dev)
    dist.all_gather_into_tensor(head, torch.tensor([n] + extra, dtype=torch.int64, device=dev), group=g)
    head = head.cpu().view(ws, 1 + len(extra))
    lens = head[:, 0].tolist()
    extras = head[:, 1:].tolist()
    # fields are packed widest first, so that every field of every rank starts on a multiple of its element size
    order = sorted(range(len(tensors)), key=lambda k: -tensors[k].element_size())
    widths = [tensors[k].element_size() for k in order]
    row_bytes = sum(widths)
    mine = torch.cat([tensors[k][:n].contiguous().view(torch.uint8) for k in order]) if n else \
        torch.empty(0, dtype=torch.uint8, device=dev)
    if dist.get_backend(g) == "nccl":
        bufs = [torch.empty(row_bytes * ln, dtype=torch.uint8, device=dev) for ln in lens]
        dist.all_gather(bufs, mine, group=g)
    else:
        cap = (max(max(lens), 1) * row_bytes + 15) // 16 * 16
        pad = torch.zeros(cap, dtype=torch.uint8, device=dev)
        pad[:mine.numel()] = mine
        flat = torch.empty(ws * cap, dtype=torch.uint8, device=dev)
        dist.all_gather_into_tensor(flat, pad, group=g)
        bufs = [flat[r * cap:r * cap + row_bytes * lens[r]] for r in range(ws)]
    out = [None] * len(tensors)
    for j, k in enumerate(order):
        off = sum(widths[:j])
        parts = [bufs[r][off * lens[r]:(off + widths[j]) * lens[r]].view(tensors[k].dtype) for r in range(ws) if lens[r]]
        out[k] = torch.cat(parts) if parts else torch.empty(0, dtype=tensors[k].dtype, device=dev)
    return tuple(out), lens, extras


def gather_matches(shape, row, col, score, nnz, max_row):
    """Combine the per-rank top-n lists of DeviceMatches into the global list (the `vstack` of :750 over NVLink)."""
    (g_row, g_col, g_score), lens, extras = allgather_varlen((row[:nnz], col[:nnz], score[:nnz]), extra=[int(max_row)])
    return g_row, g_col, g_score, int(sum(lens)), int(max(e[0] for e in extras))


def shard_vectorise(n_bytes_total):
    """Whether K1 should be sharded over the ranks (two-Series inputs only).  SG_B200_SHARD_VECTORISE = 0 / 1 /
    auto (default): auto shards once the packed corpus exceeds 256 MB — below that every rank vectorising
    everything costs a few milliseconds and needs no collective at all."""
    mode = os.environ.get("SG_B200_SHARD_VECTORISE", "auto").lower()
    if mode in ("1", "true", "yes", "on"):
        return True
    if mode in ("0", "false", "no", "off"):
        return False
    return n_bytes_total > (256 << 20)


def allreduce_sum_(tensor):
    """In-place sum over the ranks (the int32 document-frequency table of K1: ncclAllReduce over NVLink)."""
    dist = _dist()
    dist.all_reduce(tensor, op=dist.ReduceOp.SUM, group=group())
    return tensor


def allgather_csr_rows(row_len, indices, vals):
    """All-gather a row-sharded CSR (the right matrix after a sharded K1).

    row_len: int64 lengths of the local rows; indices: int32 [local nnz]; vals: tuple of value tensors
    [local nnz].  Returns (indptr int64 [n_total+1], indices, vals) of the concatenation in rank order.
    """
    import torch
    (all_len,), _, _ = allgather_varlen((row_len,))
    gathered, _, _ = allgather_varlen((indices,) + tuple(vals))
    indptr = torch.zeros(all_len.numel() + 1, dtype=torch.int64, device=row_len.device)
    torch.cumsum(all_len, 0, out=indptr[1:])
    return indptr, gathered[0], gathered[1:]


def shard_offsets(n_rows, world_size):
    return np.array([shard_range(n_rows, r, world_size)[0] for r in range(world_size)] + [n_rows], dtype=np.int64)
