"""Random walks on a graph, the corpus of DeepWalk (Perozzi et al., KDD 2014) and node2vec (Grover and Leskovec,
KDD 2016)::

    g, labels = mv.ops.Graph.load("edges.txt")                 # SNAP edge list: "src dst [w]" lines, # comments
    walks = mv.ops.random_walks(g, starts, length=80, p=0.25, q=4, seed=1)   # int32 [n, 80], -1 after a dead end

A :class:`Graph` is a CSR: node v's out-list is ``indices[indptr[v]:indptr[v + 1]]``, sorted ascending, with repeated
entries for multi-edges; a weighted graph also holds ``cum``, the prefix sums of the arc weights within each list,
summed in list order in fp64. The whole CSR lives on one device: 8 bytes per node and 4 per arc, 8 more per arc
when weighted.

Walk i of a call is walk number ``g = first_walk + i``. It starts at ``starts[i]``; step s (s = 1 .. L - 1) moves from
v, reached from t (no t at s = 1), to a node x of v's list, and a node without out-arcs ends the walk, the rest of
the row being -1. Every random number is a 64-bit draw that is a pure function of (seed, g, s, j)::

    hash64(x)      = MurmurHash3's 64-bit finaliser (csrc/cuda/mvb_common.cuh), all arithmetic mod 2^64
    key(seed, g)   = hash64(hash64(seed ^ 0x9E3779B97F4A7C15) + g * 0xBF58476D1CE4E5B9)
    draw(g, s, j)  = hash64(key(seed, g) + ((s << 32) | j) * 0x94D049BB133111EB)

so a walk does not depend on the thread, grid, rank or call that produces it: the corpus is the same for any launch
shape, any split of the starts between calls (with matching ``first_walk``) and any number of GPUs.

* **Proposal** from draw r: unweighted, the list entry ``((r >> 32) * deg(v)) >> 32`` (integers only); weighted, the
  first entry j with ``cum[j] > u * total(v)``, ``u = (r >> 11) 2^-53`` and ``total(v)`` the last prefix sum (the
  last entry should the product round up to the total).
* **First order** (1/p and 1/q both 1 in fp32: DeepWalk), and the first step of every walk: the proposal of
  draw(g, s, 0) is the step.
* **Second order** (node2vec): alpha(t, x) = 1/p if x = t; 1 if x is in t's out-list (a binary search in it); 1/q
  otherwise. That is the paper's d(t, x), the distance from t to x. On an undirected graph it is the reference code's
  ``has_edge(x, t)``; on a directed graph the two differ, and this walker follows the paper (an arc t -> x, not
  x -> t, makes x a distance-1 node). Attempt a = 0 .. R - 1 proposes x from draw(g, s, 2a) and accepts it when
  ``u24 * amax < alpha(t, x)`` in fp32, with ``u24 = (draw(g, s, 2a + 1) >> 40) 2^-24`` and ``amax = max(1/p, 1,
  1/q)``, all fp32 values of ``1 / p`` and ``1 / q`` computed in fp64. Every product is exact or rounded the same way
  on the CPU.
* **Bounded fallback.** After R rejections (R = 256, ``REJECT_ROUNDS``) the step samples exactly by inversion: with
  w_j the arc weights (the differences of ``cum``, or 1), S = sum_j w_j alpha(t, x_j) over v's list in fp64 in list
  order (no fused multiply-adds), and the step takes the first entry whose running sum exceeds ``u * S``, u from
  draw(g, s, 2R). Each attempt accepts x with probability proportional to w_x alpha(t, x), so whether a step ends in
  an acceptance or in the fallback, its law is node2vec's (up to the fp32 rounding of alpha and of the acceptance
  product), and every loop is bounded by a function of deg(v) and deg(t): the walker never spins.

:func:`random_walks_reference` is this walker in numpy, bitwise equal to the kernel ``mvb_random_walk``
(``csrc/cuda/walk.cu``), and is what :func:`random_walks` runs for a graph on the CPU.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np
import torch

from .. import _native as N

REJECT_ROUNDS = 256         # WALK_REJECT_ROUNDS of csrc/cuda/walk.cu, which justifies the value
MAX_NODES = 2 ** 31 - 2     # node ids are int32 and N + 1 must fit as well

_K0, _K1, _K2 = np.uint64(0x9E3779B97F4A7C15), np.uint64(0xBF58476D1CE4E5B9), np.uint64(0x94D049BB133111EB)


def hash64(x: np.ndarray) -> np.ndarray:
    """MurmurHash3's 64-bit finaliser on uint64 values (``hash64`` of csrc/cuda/mvb_common.cuh)."""
    x = np.asarray(x, dtype=np.uint64)
    with np.errstate(over="ignore"):
        x = x ^ (x >> np.uint64(33))
        x = x * np.uint64(0xFF51AFD7ED558CCD)
        x = x ^ (x >> np.uint64(33))
        x = x * np.uint64(0xC4CEB9FE1A85EC53)
        return x ^ (x >> np.uint64(33))


def hash64_torch(x: torch.Tensor) -> torch.Tensor:
    """``hash64`` on an int64 tensor holding the uint64 bits (two's complement, products mod 2^64)."""
    def shr33(v):
        return (v >> 33) & ((1 << 31) - 1)
    x = x ^ shr33(x)
    x = x * -0xAE502812AA7333        # 0xFF51AFD7ED558CCD as int64
    x = x ^ shr33(x)
    x = x * -0x3B314601E57A13AD      # 0xC4CEB9FE1A85EC53 as int64
    return x ^ shr33(x)


def _walk_keys(seed: int, g: np.ndarray) -> np.ndarray:
    s = hash64(np.uint64(int(seed) & 0xFFFFFFFFFFFFFFFF) ^ _K0)
    with np.errstate(over="ignore"):
        return hash64(s + g.astype(np.uint64) * _K1)


def _draw(keys: np.ndarray, s: int, j: int) -> np.ndarray:
    with np.errstate(over="ignore"):
        return hash64(keys + np.uint64((s << 32) | j) * _K2)


def _device_default(device):
    if device is not None:
        return torch.device(device)
    return torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")


class Graph:
    """A graph in CSR form on one device (see the module docstring): ``num_nodes``, ``indptr`` int64 [N + 1],
    ``indices`` int32 [E] (each list sorted ascending), ``cum`` fp64 [E] or None."""

    def __init__(self, indptr: torch.Tensor, indices: torch.Tensor, cum: Optional[torch.Tensor] = None):
        self.indptr, self.indices, self.cum = indptr, indices, cum
        self.num_nodes = indptr.numel() - 1

    @property
    def device(self) -> torch.device:
        return self.indptr.device

    @property
    def num_arcs(self) -> int:
        return self.indices.numel()

    def degree(self) -> torch.Tensor:
        """Out-degree of every node (int64), or its weighted out-degree (fp64) for a weighted graph."""
        deg = self.indptr[1:] - self.indptr[:-1]
        if self.cum is None:
            return deg
        out = torch.zeros(self.num_nodes, dtype=torch.float64, device=self.device)
        has = deg > 0
        out[has] = self.cum[self.indptr[1:][has] - 1]
        return out

    @classmethod
    def from_edges(cls, src, dst, weights=None, num_nodes: Optional[int] = None, directed: bool = False,
                   device=None) -> "Graph":
        """The CSR of the edges ``src[k] -> dst[k]`` (node ids in [0, num_nodes); ``num_nodes=None``: one more than
        the largest id), on ``device`` (default: the current CUDA device, else the CPU). Undirected edges give both
        arcs, a self-loop one. Repeated edges and self-loops are kept. ``weights``: one finite weight > 0 per edge."""
        dev = _device_default(device)
        src = torch.as_tensor(src).to(dev).reshape(-1)
        dst = torch.as_tensor(dst).to(dev).reshape(-1)
        for name, t in (("src", src), ("dst", dst)):
            if t.is_floating_point() or t.is_complex() or t.dtype == torch.bool:
                raise TypeError(f"Graph.from_edges: {name} must be integers, got {t.dtype}")
        if src.shape != dst.shape:
            raise ValueError(f"Graph.from_edges: src and dst must have the same length, got {src.numel()} and "
                             f"{dst.numel()}")
        src, dst = src.to(torch.int64), dst.to(torch.int64)
        w = None
        if weights is not None:
            w = torch.as_tensor(weights).to(dev).reshape(-1).to(torch.float64)
            if w.shape != src.shape:
                raise ValueError(f"Graph.from_edges: weights must have one value per edge ({src.numel()}), got "
                                 f"{w.numel()}")
            if w.numel() and not bool(torch.all(torch.isfinite(w) & (w > 0))):
                raise ValueError("Graph.from_edges: weights must be finite and > 0")
        lo = int(torch.minimum(src.min(), dst.min())) if src.numel() else 0
        hi = int(torch.maximum(src.max(), dst.max())) if src.numel() else -1
        n = hi + 1 if num_nodes is None else int(num_nodes)
        if lo < 0 or hi >= n:
            raise ValueError(f"Graph.from_edges: node ids must be in [0, {n}), got min {lo} max {hi}")
        if n > MAX_NODES:
            raise ValueError(f"Graph.from_edges: at most {MAX_NODES} nodes, got {n}")
        if not directed:
            back = src != dst                                 # a self-loop is one arc
            src, dst = torch.cat([src, dst[back]]), torch.cat([dst, src[back]])
            if w is not None:
                w = torch.cat([w, w[back]])
        order = torch.sort(src * max(n, 1) + dst, stable=True).indices
        src, dst = src[order], dst[order]
        counts = torch.bincount(src, minlength=n) if src.numel() else torch.zeros(n, dtype=torch.int64, device=dev)
        if src.numel() >= 2 ** 32 and int(counts.max()) >= 2 ** 32:
            raise ValueError("Graph.from_edges: a node has 2^32 or more out-arcs")
        indptr = torch.zeros(n + 1, dtype=torch.int64, device=dev)
        torch.cumsum(counts, 0, out=indptr[1:])
        indices = dst.to(torch.int32).contiguous()
        cum = None
        if w is not None:
            cum = _segment_cumsum(indptr, w[order].contiguous())
        return cls(indptr, indices, cum)

    @classmethod
    def load(cls, path: str, directed: bool = False, weighted: bool = False, device=None):
        """Read a SNAP-style edge list: one ``src dst`` (``src dst w`` when ``weighted``) line per edge, labels
        non-negative integers up to 2^63 - 1, blank lines and ``#`` comments skipped. Returns ``(graph, labels)``:
        node i of the graph has the label ``labels[i]`` (int64 numpy), the labels in ascending order. A malformed
        line raises ValueError naming its line number."""
        src, dst, w = read_edge_list(path, weighted)
        labels = np.unique(np.concatenate([src, dst]))
        s, d = np.searchsorted(labels, src), np.searchsorted(labels, dst)
        g = cls.from_edges(torch.from_numpy(s), torch.from_numpy(d), None if w is None else torch.from_numpy(w),
                           num_nodes=labels.size, directed=directed, device=device)
        return g, labels


def read_edge_list(path: str, weighted: bool = False):
    """(src int64, dst int64, weights fp64 or None) of an edge-list file, parsed by the native reader
    (csrc/host/applib/graph_data.cpp)."""
    from ..apps._applib import lib
    L = lib()
    h = L.MVA_EdgeListOpen(str(path).encode(), int(bool(weighted)))
    if not h:
        raise OSError(f"cannot open the edge list {path}")
    try:
        err = L.MVA_EdgeListError(h)
        if err:
            raise ValueError(f"{path}: {err.decode(errors='replace')}")
        m = L.MVA_EdgeListSize(h)
        src, dst = np.empty(m, dtype=np.int64), np.empty(m, dtype=np.int64)
        w = np.empty(m, dtype=np.float64) if weighted else None
        L.MVA_EdgeListCopy(h, src.ctypes.data_as(C.c_void_p), dst.ctypes.data_as(C.c_void_p),
                           None if w is None else w.ctypes.data_as(C.c_void_p))
    finally:
        L.MVA_EdgeListClose(h)
    return src, dst, w


def _segment_cumsum(indptr: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """cum[j] = the weights of j's list up to j, summed in list order in fp64."""
    n = indptr.numel() - 1
    if w.is_cuda:
        cum = torch.empty_like(w)
        N.cuda_lib().mvb_csr_cumsum(indptr, w, n, cum, N.stream_ptr())
        return cum
    ip, wn = indptr.numpy(), w.numpy()
    deg = ip[1:] - ip[:-1]
    order = np.argsort(-deg, kind="stable")              # nodes by degree: the first cnt[k] have a k-th arc
    beg = ip[:-1][order]
    cnt = np.searchsorted(-deg[order], np.arange(int(deg.max()) if n else 0) * -1, side="left")
    cum = np.empty_like(wn)
    run = np.zeros(n, dtype=np.float64)
    for k, c in enumerate(cnt):
        j = beg[:c] + k
        run[:c] = run[:c] + wn[j]
        cum[j] = run[:c]
    return torch.from_numpy(cum)


def _check_walk_args(graph: Graph, starts, length: int, p: float, q: float, first_walk: int) -> torch.Tensor:
    starts = torch.as_tensor(starts)
    if starts.is_floating_point() or starts.is_complex() or starts.dtype == torch.bool:
        raise TypeError(f"random_walks: starts must be integers, got {starts.dtype}")
    starts = starts.reshape(-1).to(graph.device)
    if starts.numel():
        lo, hi = (int(v) for v in torch.aminmax(starts))
        if lo < 0 or hi >= graph.num_nodes:
            raise ValueError(f"random_walks: starts must be in [0, {graph.num_nodes}), got min {lo} max {hi}")
    if int(length) != length or length < 1:
        raise ValueError(f"random_walks: length must be a positive integer, got {length}")
    for name, v in (("p", p), ("q", q)):
        with np.errstate(over="ignore"):
            inv = np.float32(1.0 / v) if v != 0 else np.float32(np.inf)
        if not (np.isfinite(v) and v > 0 and np.isfinite(inv) and inv > 0):
            raise ValueError(f"random_walks: {name} must be finite and > 0 with 1/{name} finite and > 0 in fp32, "
                             f"got {v}")
    if int(first_walk) != first_walk or first_walk < 0:
        raise ValueError(f"random_walks: first_walk must be a non-negative integer, got {first_walk}")
    return starts.to(torch.int32).contiguous()


def launch_walks(graph: Graph, starts: torch.Tensor, out: torch.Tensor, length: int, p: float, q: float, seed: int,
                 first_walk: int, node_count: Optional[torch.Tensor] = None) -> None:
    """mvb_random_walk on the current stream: walks of int32 ``starts`` (in range) into the rows of the int32
    ``out`` [n, pitch >= length]; ``node_count`` (int64 [1]) += the nodes written."""
    a = N.RandomWalk()
    a.indptr, a.indices, a.cum, a.num_nodes = graph.indptr.data_ptr(), graph.indices.data_ptr(), N.ptr(graph.cum), \
        graph.num_nodes
    a.starts, a.n, a.length, a.pitch = starts.data_ptr(), starts.numel(), int(length), out.stride(0)
    a.p, a.q, a.seed, a.first_walk = float(p), float(q), int(seed) & 0xFFFFFFFFFFFFFFFF, int(first_walk)
    a.out, a.node_count = out.data_ptr(), N.ptr(node_count)
    N.cuda_lib().mvb_random_walk(a, N.stream_ptr())


def random_walks(graph: Graph, starts, length: int, p: float = 1.0, q: float = 1.0, seed: int = 0,
                 first_walk: int = 0) -> torch.Tensor:
    """Walks of ``length`` nodes from ``starts`` (see the module docstring): int32 [n, length] on the graph's device,
    -1 after a dead end. On the GPU the kernel ``mvb_random_walk``; on the CPU :func:`random_walks_reference`."""
    starts = _check_walk_args(graph, starts, length, p, q, first_walk)
    if not graph.device.type == "cuda":
        return torch.from_numpy(random_walks_reference(graph, starts, length, p, q, seed, first_walk))
    out = torch.empty(starts.numel(), int(length), dtype=torch.int32, device=graph.device)
    launch_walks(graph, starts, out, length, p, q, seed, first_walk)
    return out


# ------------------------------------------------------------------------------------------------------ reference
def _lower_bound(arr: np.ndarray, lo: np.ndarray, hi: np.ndarray, x: np.ndarray, upper: bool) -> np.ndarray:
    """Per element, the first j in [lo, hi) with arr[j] >= x (upper: arr[j] > x), or hi."""
    lo, hi = lo.copy(), hi.copy()
    while True:
        m = lo < hi
        if not m.any():
            return lo
        mid = np.where(m, lo + ((hi - lo) >> 1), 0)
        v = arr[mid]
        right = (v <= x) if upper else (v < x)
        lo = np.where(m & right, mid + 1, lo)
        hi = np.where(m & ~right, mid, hi)


def random_walks_reference(graph: Graph, starts, length: int, p: float = 1.0, q: float = 1.0, seed: int = 0,
                           first_walk: int = 0) -> np.ndarray:
    """The walker of the module docstring in numpy: int32 [n, length], bitwise the kernel's walks."""
    ip = graph.indptr.cpu().numpy()
    ind = graph.indices.cpu().numpy().astype(np.int64)
    cum = None if graph.cum is None else graph.cum.cpu().numpy()
    starts = torch.as_tensor(starts).cpu().numpy().astype(np.int64).reshape(-1)
    n, L, R = starts.size, int(length), REJECT_ROUNDS
    inv_p, inv_q = np.float32(1.0 / p), np.float32(1.0 / q)
    amax = max(inv_p, np.float32(1), inv_q)
    first_order = inv_p == 1 and inv_q == 1
    keys = _walk_keys(seed, int(first_walk) + np.arange(n, dtype=np.int64))
    out = np.full((n, L), -1, dtype=np.int32)
    out[:, 0] = starts
    v, t = starts.copy(), np.full(n, -1, dtype=np.int64)
    alive = np.ones(n, dtype=bool)

    def propose(beg, end, r):
        if cum is None:
            return beg + (((r >> np.uint64(32)) * (end - beg).astype(np.uint64)) >> np.uint64(32)).astype(np.int64)
        target = (r >> np.uint64(11)).astype(np.float64) * 2.0 ** -53 * cum[end - 1]
        return np.minimum(_lower_bound(cum, beg, end, target, upper=True), end - 1)

    def alpha(tt, tb, te, x):
        j = _lower_bound(ind, tb, te, x, upper=False)
        member = (j < te) & (ind[np.minimum(j, ind.size - 1)] == x)
        return np.where(x == tt, inv_p, np.where(member, np.float32(1), inv_q)).astype(np.float32)

    def weight_alpha(k, beg, deg, prev, tt, tb, te):
        m = k < deg
        j = np.where(m, beg + k, 0)
        if cum is None:
            w = np.ones(j.size)
        else:
            w = cum[j] - prev
            prev = np.where(m, cum[j], prev)
        return m, ind[j], w * alpha(tt, tb, te, ind[j]).astype(np.float64), prev

    for s in range(1, L):
        idx = np.nonzero(alive)[0]
        beg, end = ip[v[idx]], ip[v[idx] + 1]
        dead = end == beg
        alive[idx[dead]] = False
        idx, beg, end = idx[~dead], beg[~dead], end[~dead]
        if idx.size == 0:
            break
        kk = keys[idx]
        if first_order or s == 1:
            x = ind[propose(beg, end, _draw(kk, s, 0))]
        else:
            tt = t[idx]
            tb, te = ip[tt], ip[tt + 1]
            x = np.full(idx.size, -1, dtype=np.int64)
            todo = np.arange(idx.size)
            for r in range(R):
                if todo.size == 0:
                    break
                xr = ind[propose(beg[todo], end[todo], _draw(kk[todo], s, 2 * r))]
                u24 = (_draw(kk[todo], s, 2 * r + 1) >> np.uint64(40)).astype(np.float32) * np.float32(2.0 ** -24)
                ok = (u24 * amax).astype(np.float32) < alpha(tt[todo], tb[todo], te[todo], xr)
                x[todo[ok]] = xr[ok]
                todo = todo[~ok]
            if todo.size:                                   # the exact inversion of the rest
                b, d = beg[todo], end[todo] - beg[todo]
                ft, fb, fe = tt[todo], tb[todo], te[todo]
                total, prev = np.zeros(todo.size), np.zeros(todo.size)
                for k in range(int(d.max())):
                    m, _, wa, prev = weight_alpha(k, b, d, prev, ft, fb, fe)
                    total = np.where(m, total + wa, total)
                target = (_draw(kk[todo], s, 2 * R) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53 * total
                run, prev = np.zeros(todo.size), np.zeros(todo.size)
                pick = np.full(todo.size, -1, dtype=np.int64)
                for k in range(int(d.max())):
                    m, xk, wa, prev = weight_alpha(k, b, d, prev, ft, fb, fe)
                    m &= pick < 0
                    run = np.where(m, run + wa, run)
                    hit = m & (run > target)
                    pick[hit] = xk[hit]
                    if (pick >= 0).all():
                        break
                pick = np.where(pick < 0, ind[b + d - 1], pick)
                x[todo] = pick
        t[idx] = v[idx]
        v[idx] = x
        out[idx, s] = x
    return out
