"""Fused cosine top-k search over a MatrixTable: the nearest rows of a batch of query vectors.

``topk_cosine(table, queries, k)`` returns, for every query, the ``k`` table rows with the largest cosine,
sorted by score descending with ties broken by the smaller row id; a zero row scores 0 and missing slots
(fewer than ``k`` rows searched) hold id -1 and score -inf.

On the device the search is one pass over the table (``csrc/cuda/topk_cos.cu``): W tiles are streamed from
their owners' shards with TMA into tf32 wgmma, row norms are taken from the same shared-memory tiles, and a
top-k epilogue keeps k + 8 candidates per query, whose cosines are then recomputed in fp64. The score matrix
is never written, so 19,544 analogy questions against a 1M-word vocabulary need no 78 GB buffer. A call on
any rank searches the whole sharded table, with the consistency rule of ``get_gemm``: the caller orders it
after the Adds it wants to see (barrier / ``flush``).

Its cost is the per-query top-k bookkeeping, not the table stream: for a handful of queries ``get_gemm`` into a
score buffer followed by ``torch.topk`` is faster (1M x 300, one H100: 0.72 against 0.90 ms at M = 1); from a few
hundred queries up the fused search is faster and needs no score buffer (DESIGN.md section 6).

Without a GPU (CPU tensors, host-backend tables) the same call is a chunked fp32 matmul plus an exact
top-k with the same tie rule, :func:`topk_cosine_reference`.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch

from .. import _native as N

TOPK_MAX = 64             # MVB_TOPK_MAX (csrc/cuda/mvb200.h)
_Q_CHUNK = 4096           # queries per kernel call: bounds the scratch, 2 x M x ranges x (k + 8) x 8 bytes
                          # (1M rows, k = 10, 132 SMs: 4.9 MB at M = 1000, 5.9 MB at M = 4096)


def check_k(k, excluded: int = 0, what: str = "topk_cosine") -> int:
    """``k`` of a search that asks for ``k + excluded`` rows and drops ``excluded`` of them, as an int; raises
    with the caller's ``k`` when the search would exceed TOPK_MAX."""
    k = int(k)
    if not 1 <= k <= TOPK_MAX - excluded:
        raise ValueError(f"{what}: k must be in [1, {TOPK_MAX - excluded}], got {k}")
    return k


def _unit_rows(x: torch.Tensor) -> torch.Tensor:
    n = x.norm(dim=1, keepdim=True)
    return torch.where(n > 0, x / torch.where(n > 0, n, torch.ones_like(n)), torch.zeros_like(x))


def _sorted_topk(scores: torch.Tensor, ids: torch.Tensor, k: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """The k best (score desc, id asc) of each row of candidate (scores, ids)."""
    o = torch.argsort(ids, dim=1, stable=True)
    scores, ids = scores.gather(1, o), ids.gather(1, o)
    o = torch.argsort(-scores, dim=1, stable=True)[:, :k]
    return scores.gather(1, o), ids.gather(1, o)


def topk_cosine_reference(weights: torch.Tensor, queries: torch.Tensor, k: int,
                          rows: Optional[int] = None, row_chunk: int = 65536) -> Tuple[torch.Tensor, torch.Tensor]:
    """Host implementation: chunked fp32 matmul + exact top-k. ``weights``: [V, >= dim] fp32 (columns
    beyond the queries' width are ignored), ``queries``: [M, dim]. Returns (scores [M, k] fp32, ids [M, k]
    int64)."""
    k = check_k(k)
    q = torch.as_tensor(queries)
    if q.dtype != torch.float32 or q.dim() != 2:
        raise TypeError(f"topk_cosine: queries must be a 2-D float32 tensor, got {q.dtype} {tuple(q.shape)}")
    w = torch.as_tensor(weights)
    dim = q.shape[1]
    if w.dim() != 2 or dim > w.shape[1]:
        raise ValueError(f"topk_cosine: queries have {dim} columns, the table rows {tuple(w.shape)[1:]}")
    n = w.shape[0] if rows is None else int(rows)
    if not 0 <= n <= w.shape[0]:
        raise ValueError(f"topk_cosine: rows={n} outside [0, {w.shape[0]}]")
    q = _unit_rows(q)
    M = q.shape[0]
    best_s = torch.full((M, k), float("-inf"), dtype=torch.float32, device=q.device)
    best_i = torch.full((M, k), -1, dtype=torch.int64, device=q.device)
    for lo in range(0, n, row_chunk):
        hi = min(n, lo + row_chunk)
        wc = _unit_rows(w[lo:hi, :dim].to(device=q.device, dtype=torch.float32))
        best_s, best_i = merge_topk(best_s, best_i, q @ wc.t(), lo, k)
    return best_s, best_i


def merge_topk(best_s: torch.Tensor, best_i: torch.Tensor, s: torch.Tensor, lo: int,
               k: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """Fold the scores ``s`` [M, c] of rows [lo, lo + c) into a running top-k (``best_s``, ``best_i``) [M, k]
    under (score desc, id asc); empty slots hold -inf / -1."""
    kk = min(k, s.shape[1])
    v, _ = s.topk(kk, dim=1)
    # every row scoring at least the kk-th value is a candidate: ties at the boundary resolve by id
    cand = s >= v[:, -1:]
    width = int(cand.sum(1).max())
    cs = torch.where(cand, s, torch.full_like(s, float("-inf")))
    cv, ci = cs.topk(width, dim=1)
    ci = torch.where(cv > float("-inf"), ci + lo, torch.full_like(ci, torch.iinfo(torch.int64).max))
    best_s, best_i = _sorted_topk(torch.cat([best_s, cv], 1),
                                  torch.cat([torch.where(best_i < 0, torch.full_like(best_i, torch.iinfo(torch.int64).max), best_i), ci], 1), k)
    best_i = torch.where(best_i == torch.iinfo(torch.int64).max, torch.full_like(best_i, -1), best_i)
    return best_s, best_i


def _rowmap_of(table, what: str = "topk_cosine") -> Tuple[N.RowMap, int, int]:
    """(row map, rows, row width) of a MatrixDeviceTable or of a 2-D fp32 CUDA tensor (one local shard)."""
    rm = N.RowMap()
    if isinstance(table, torch.Tensor):
        if table.dtype != torch.float32 or table.dim() != 2 or not table.is_cuda:
            raise TypeError(f"{what}: a table tensor must be 2-D float32 on CUDA, got {table.dtype} "
                            f"{tuple(table.shape)} on {table.device}")
        if table.stride(1) != 1:
            raise ValueError(f"{what}: table rows must be contiguous")
        rm.num_row, rm.num_col = table.shape[0], table.stride(0) if table.shape[0] > 1 else table.shape[1]
        rm.nservers, rm.rows_per_server = 1, max(table.shape[0], 1)
        rm.shard_ptrs[0] = table.data_ptr()
        return rm, table.shape[0], table.shape[1]
    if getattr(table, "dtype", None) != torch.float32:
        raise TypeError(f"{what}: the table must be float32")
    src = table._rowmap
    rm.num_row, rm.num_col, rm.nservers, rm.rows_per_server = src.num_row, src.num_col, src.nservers, src.rows_per_server
    for s in range(src.nservers):
        rm.shard_ptrs[s] = src.shard_ptrs[s]
    return rm, table.num_row, table.num_col


def check_queries(rm: N.RowMap, width: int, queries: torch.Tensor, name: str,
                  what: str = "topk_cosine") -> None:
    """The kernel's demands on a query batch ``[M, dim]`` and on the table's row map."""
    if queries.dtype != torch.float32 or queries.dim() != 2:
        raise TypeError(f"{what}: {name} must be a 2-D float32 tensor, got {queries.dtype} {tuple(queries.shape)}")
    if not queries.is_cuda:
        raise ValueError(f"{what}: the table is on the GPU, the {name} must be too")
    dim = queries.shape[1]
    if dim < 1 or dim > width:
        raise ValueError(f"{what}: {name} have {dim} columns, the table rows {width}")
    if rm.num_col % 4 != 0:
        raise ValueError(f"{what}: the table's row pitch ({rm.num_col} floats) must be a multiple of 4 "
                         "(16-byte rows for TMA)")


def padded_queries(q: torch.Tensor) -> torch.Tensor:
    """``q`` [M, dim] in a fresh zero-padded [M, ldq] buffer, ldq = dim rounded up to 4 (16-byte TMA rows)."""
    M, dim = q.shape
    out = torch.zeros(M, (dim + 3) // 4 * 4, dtype=torch.float32, device=q.device)
    out[:, :dim] = q
    return out


def _topk_device(rm: N.RowMap, width: int, queries: torch.Tensor, k: int,
                 rows: Optional[int]) -> Tuple[torch.Tensor, torch.Tensor]:
    """Kernel path over an explicit row map (``width``: usable columns of a row)."""
    check_queries(rm, width, queries, "queries")
    M, dim = queries.shape
    n = rm.num_row if rows is None else int(rows)
    if not 0 <= n <= rm.num_row:
        raise ValueError(f"topk_cosine: rows={n} outside [0, {rm.num_row}]")
    dev = queries.device
    q = padded_queries(_unit_rows(queries))
    ldq = q.shape[1]
    scores = torch.empty(M, k, dtype=torch.float32, device=dev)
    ids = torch.empty(M, k, dtype=torch.int64, device=dev)
    lib = N.cuda_lib()
    # the kernel's need (queries x ranges per query tile) is not monotone in the query count: size the scratch
    # for every chunk size used, the full chunks and the last one
    chunks = {min(M, _Q_CHUNK), M % _Q_CHUNK or _Q_CHUNK} if M else {1}
    nbytes = max(lib.mvb_topk_cos_scratch_bytes(c, k, n) for c in chunks)
    scratch = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=dev)
    a = N.TopkCos()
    a.ldq, a.dim, a.n_rows, a.wmap, a.k = ldq, dim, n, rm, k
    a.scratch, a.scratch_bytes = scratch.data_ptr(), scratch.numel()
    for lo in range(0, M, _Q_CHUNK):
        hi = min(M, lo + _Q_CHUNK)
        a.q, a.M = q[lo].data_ptr(), hi - lo
        a.scores, a.ids = scores[lo].data_ptr(), ids[lo].data_ptr()
        lib.mvb_topk_cosine(a, N.stream_ptr())
    return scores, ids


def topk_cosine(table, queries, k: int, rows: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """Nearest rows by cosine. ``table``: MatrixDeviceTable or 2-D fp32 tensor; ``queries``: [M, dim] fp32
    with ``dim`` <= the row width (only the first ``dim`` columns of a row count); ``rows``: search rows
    [0, rows) only. Returns (scores [M, k] fp32, ids [M, k] int64)."""
    k = check_k(k)
    q = torch.as_tensor(queries)
    if isinstance(table, torch.Tensor) and not table.is_cuda:
        return topk_cosine_reference(table, q, k, rows)
    if not isinstance(table, torch.Tensor) and not hasattr(table, "_rowmap"):
        # a host-backend table: the CPU plane's implementation over its Get
        w = torch.as_tensor(table.get()).view(table.num_row, table.num_col)
        return topk_cosine_reference(w, q, k, rows)
    rm, _, width = _rowmap_of(table)
    return _topk_device(rm, width, q, k, rows)


def take_excluding(scores: torch.Tensor, ids: torch.Tensor, exclude: torch.Tensor,
                   k: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """The first ``k`` entries of each row whose id is not in the same row of ``exclude`` [M, e] (lists from
    :func:`topk_cosine` with ``k + e`` entries keep their order)."""
    ex = (ids[:, :, None] == exclude[:, None, :].to(ids.device)).any(2)
    o = torch.argsort(ex.to(torch.int8), dim=1, stable=True)[:, :k]
    return scores.gather(1, o), ids.gather(1, o)


def analogy_queries(ea: torch.Tensor, eb: torch.Tensor, ec: torch.Tensor) -> torch.Tensor:
    """3CosAdd query of word2vec's word-analogy: unit(b) - unit(a) + unit(c) (normalised by the search)."""
    return _unit_rows(eb) - _unit_rows(ea) + _unit_rows(ec)
