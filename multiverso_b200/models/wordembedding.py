"""WordEmbedding (word2vec: skip-gram / CBOW x negative sampling / hierarchical softmax).

Reference application: Applications/WordEmbedding (SURVEY A1-A4).  The training maths is
WordEmbedding::TrainSample / FeedForward / BPOutputLayer (src/wordembedding.cpp:57-166), the
parameter-server glue is Communicator (src/communicator.cpp): two MatrixTables
(input rows U(-0.5/dim, 0.5/dim), output rows zero), optional AdaGrad G^2 tables, a KVTable
for the global word count, per data block RequestParameter -> train -> AddDeltaParameter
with delta = (trained - server_now) / num_workers.

Device mapping
--------------
* ``world == 1``: the shard *is* the table, so the block protocol degenerates exactly
  ((trained - cur)/1 added back == trained) and the K7 kernel trains in place on the HBM
  resident shards -- no gather, no scatter.
* ``world > 1`` (block mode = reference semantics): device-side PrepareData (``mvb_we_prepare``:
  bitmap-unique + prefix sum + negative pool, counts stay on the device), row pull of the needed
  rows over NVLink into a local block cache (``mvb_rows_pull``), K7 on the cache through id->slot
  maps, one-sided push of (new - old)/W into the owners' shards (``mvb_rows_push_delta``).  No
  host synchronisation and no eager PyTorch op anywhere in the step; pipelined, the pull of block
  i+1 and the push of block i-1 run on a side stream in one register-only CTA per SM, co-resident
  with block i's K7 on every SM.
* learning-rate decay follows UpdateLearningRate (wordembedding.cpp:38-47) from the global
  word count kept in the KV table (constant.h: kWordCountId).
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

from .. import _native as N
from ..runtime import Runtime
from ..tables.device import KVDeviceTable, MatrixDeviceTable
from ..utils import Log, monitor

K_WORD_COUNT_ID = 4  # constant.h:16-20
# Row pull / delta push CTAs per SM when nothing else runs (the non-pipelined step).  2 is the smallest
# grid at which both beat the former bulk-copy kernels at 32 CTAs: pull 1.21 vs 1.50 ms, push 0.90 vs 1.52 ms
# (both tables of a 1M-word Zipf block, dim 300, local shard; H100 80GB HBM3, 700 W power limit).
_BLOCKING_CTAS_PER_SM = 2


@dataclass
class WordEmbeddingOption:
    """The 21 CLI flags of the reference (util.cpp:31-56) with its defaults (util.cpp:6-29)."""
    train_file: Optional[str] = None
    read_vocab_file: Optional[str] = None
    output_file: Optional[str] = None
    sw_file: Optional[str] = None
    endpoints_file: Optional[str] = None
    hs: bool = False
    output_binary: bool = False
    cbow: bool = False
    stopwords: bool = False
    use_adagrad: bool = False
    is_pipeline: bool = True        # util.cpp:25 (reference default)
    sample: float = 0.0
    data_block_size: int = 1 << 20
    embeding_size: int = 100
    thread_cnt: int = 1
    window_size: int = 5
    negative_num: int = 5
    min_count: int = 5
    epoch: int = 1
    total_words: int = 0
    max_preload_data_size: int = 8 << 30
    init_learning_rate: float = 0.025


class HuffmanTables:
    """Device copy of the Huffman paths (HuffmanEncoder::BuildHuffmanTreeFromDict,
    huffman_encoder.cpp:87-196): per word the inner-node ids and branch codes, built by the
    native encoder (csrc/host/applib/wordembedding_data.cpp)."""

    MAX_CODE = 64
    FREQ_TOTAL_MAX = 1 << 62     # the encoder sums frequencies in int64: the root's weight is their total

    @classmethod
    def int_frequencies(cls, counts: np.ndarray) -> np.ndarray:
        """Integer encoder frequencies for `counts`: the counts themselves when they are whole numbers,
        fractional weights (the default Zipf 1/rank) scaled by 1e9; scaled down further while the
        total would overflow the encoder's int64 sums.  Every word gets at least 1."""
        c = np.asarray(counts, dtype=np.float64)
        if not np.all(c == np.floor(c)):
            c = c * 1e9
        total = float(np.maximum(c, 1.0).sum())
        if total >= cls.FREQ_TOTAL_MAX:
            c = c * (cls.FREQ_TOTAL_MAX / 4 / total)
        return np.ascontiguousarray(np.maximum(np.floor(c), 1.0).astype(np.int64))

    @classmethod
    def encode(cls, counts: np.ndarray):
        """The encoder's tree over `int_frequencies(counts)`: (points [V, MAX_CODE] int32, codes [V, MAX_CODE]
        int8, lens [V] int32, longest). `longest` is the longest code, or -1 when a code is longer than MAX_CODE."""
        from ..apps._applib import lib
        V = len(counts)
        freq = cls.int_frequencies(counts)
        P = np.zeros((V, cls.MAX_CODE), dtype=np.int32)
        Cd = np.zeros((V, cls.MAX_CODE), dtype=np.int8)
        lens = np.zeros(V, dtype=np.int32)
        longest = lib().MVA_HuffmanBuild(freq.ctypes.data_as(C.c_void_p), V, cls.MAX_CODE,
                                         P.ctypes.data_as(C.c_void_p), Cd.ctypes.data_as(C.c_void_p),
                                         lens.ctypes.data_as(C.c_void_p))
        return P, Cd, lens, int(longest)

    def __init__(self, counts: np.ndarray, device):
        P, Cd, lens, longest = self.encode(counts)
        if longest < 0:
            Log.fatal("Huffman code longer than %d", self.MAX_CODE)
        self.max_code = max(int(longest), 1)
        self.points = torch.from_numpy(np.ascontiguousarray(P[:, :self.max_code])).to(device)
        self.codes = torch.from_numpy(np.ascontiguousarray(Cd[:, :self.max_code])).to(device)
        self.lens = torch.from_numpy(lens).to(device)


class WordEmbedding:
    """Distributed word2vec trainer on HBM-resident tables."""

    def __init__(self, option: WordEmbeddingOption, vocab_size: int,
                 word_counts: Optional[np.ndarray] = None, seed: int = 1):
        rt = Runtime.get()
        if rt.backend != "device":
            Log.fatal("WordEmbedding needs the device backend (CUDA)")
        self.rt, self.opt, self.V = rt, option, int(vocab_size)
        self.D = int(option.embeding_size)
        self.dev = rt.device
        self.W = max(rt.num_workers(), 1)
        D = self.D
        # PrepareParameterTables (communicator.cpp:17-32)
        self.input_table = MatrixDeviceTable(self.V, D, "float32", updater="default",
                                             min_value=-0.5 / D, max_value=0.5 / D, seed=seed)
        self.output_table = MatrixDeviceTable(self.V, D, "float32", updater="default", init_value=0.0)
        self.g2_in = self.g2_out = None
        if option.use_adagrad:
            self.g2_in = MatrixDeviceTable(self.V, D, "float32", updater="default", init_value=0.0)
            self.g2_out = MatrixDeviceTable(self.V, D, "float32", updater="default", init_value=0.0)
        self.wordcount_table = KVDeviceTable("int64", "int64", capacity=1024)
        if word_counts is None:
            word_counts = 1.0 / np.arange(1, self.V + 1, dtype=np.float64)   # Zipf
        self.counts = np.asarray(word_counts, dtype=np.float64)
        # Sampler::SetNegativeSamplingDistribution (util.cpp:116-135): unigram^0.75
        if option.negative_num > 0 and not option.hs:
            prob = np.empty(self.V, dtype=np.float32)
            alias = np.empty(self.V, dtype=np.int32)
            w = np.power(self.counts, 0.75)
            N.cuda_lib().mvb_build_alias_table(w.ctypes.data, self.V, prob.ctypes.data, alias.ctypes.data)
            self.alias_prob = torch.from_numpy(prob).to(self.dev)
            self.alias_idx = torch.from_numpy(alias).to(self.dev)
        else:
            self.alias_prob = self.alias_idx = None
        self.huffman = HuffmanTables(self.counts, self.dev) if option.hs else None
        self.loss = torch.zeros(1, dtype=torch.float32, device=self.dev)
        self.pairs = torch.zeros(1, dtype=torch.int64, device=self.dev)
        self.word_count_actual = 0
        self.learning_rate = float(option.init_learning_rate)
        self._step = 0
        self._maps = [None, None]       # two (map_in, map_out) sets: block i trains while i+1 is prepared
        self._map_slot = 0
        self._side = None               # side stream of the pipelined mode
        self._prefetched = None
        self._pending_side = False
        self.kernel_launches = 0
        self.hogwild = False        # one GPU, skip-gram + NS: the Hogwild window kernel instead of the deterministic waves
        # world > 1 training mode: "block" (reference semantics: pull, train a block-local copy, push (new - old) / W)
        # or "direct": K7 trains IN the row-sharded tables, loading rows from and reducing deltas into their owners'
        # shards over NVLink (Hogwild across GPUs: no cache, no PrepareData, one kernel per block at any world size;
        # link bound: ~20 KB per word cross NVLink instead of ~2 KB in block mode)
        self.mode = os.environ.get("MVB_WE_MODE", "block")
        # direct mode runs only on the window kernel: dim <= 512, window <= 15
        if self.mode == "direct" and not (rt.size > 1 and self._dev_block_ok() and D <= 512
                                          and option.window_size <= 15):
            self.mode = "block"
        self._bufs = [None, None]   # device-side block protocol: two buffer sets (block i trains, i+1 is pulled)
        self.scale_in = self.scale_out = None
        self._build_hot_row_cap()

    # ------------------------------------------------------------------ hot-row step cap
    def _build_hot_row_cap(self) -> None:
        """Per-word step scales for the window-batched K7.

        The kernel keeps P centre positions in flight per device (one CTA per SM x 10 warps x 2 stages),
        i.e. ~P (W+1) (context, centre) samples whose rows were read before any of their updates
        landed.  The reference's Hogwild has <= `-threads` samples in flight; with ~18 000 the rows
        of the Zipf head collect hundreds of same-direction stale steps per staleness window and
        plain SGD overshoots (measured: loss diverges within 10 blocks on the raw Zipf corpus).
        A row expected to collect G > cap concurrent updates gets its step scaled by cap / G, i.e.
        its summed step per staleness window is what `cap` sequential samples would apply; every
        other row (all but the few dozen hottest words) trains exactly as before.  cap = 0 disables."""
        o = self.opt
        cap = float(os.environ.get("MVB_WE_HOT_CAP", "128"))
        if cap <= 0 or o.cbow or o.hs or o.use_adagrad or o.negative_num < 1:
            return
        pos = N.cuda_lib().mvb_sgns_win_inflight(self.D, o.negative_num, o.window_size)
        if pos <= 0:
            return
        f = self.counts / self.counts.sum()
        q = np.power(self.counts, 0.75)
        q /= q.sum()
        if getattr(self, "mode", "block") == "direct":
            pos *= self.rt.size                    # every GPU's in-flight positions hit the same shared rows
        pairs = pos * (o.window_size + 1.0)
        g_in = pairs * f
        g_out = pairs * (f + o.negative_num * q)
        s_in = np.minimum(1.0, cap / np.maximum(g_in, 1e-30)).astype(np.float32)
        s_out = np.minimum(1.0, cap / np.maximum(g_out, 1e-30)).astype(np.float32)
        self.hot_rows_capped = (int((s_in < 1).sum()), int((s_out < 1).sum()))
        self.scale_in = torch.from_numpy(s_in).to(self.dev)
        self.scale_out = torch.from_numpy(s_out).to(self.dev)

    # ------------------------------------------------------------------ lr schedule
    def update_learning_rate(self) -> float:
        o = self.opt
        if not o.use_adagrad and o.total_words > 0:
            lr = o.init_learning_rate * (1 - self.word_count_actual / (o.total_words * o.epoch + 1.0))
            self.learning_rate = max(lr, o.init_learning_rate * 1e-4)
        return self.learning_rate

    # ------------------------------------------------------------------ K7 launch
    def _launch(self, tokens: torch.Tensor, w_in, w_out, g2_in, g2_out, ld, map_in=None,
                map_out=None, neg_pool=None, compute_loss=True, neg_pool_size_ptr=None,
                direct: bool = False) -> None:
        o = self.opt
        a = N.Sgns()
        a.tokens, a.n_tokens = tokens.data_ptr(), tokens.numel()
        a.w_in, a.w_out = w_in.data_ptr(), w_out.data_ptr()
        a.g2_in = g2_in.data_ptr() if g2_in is not None else None
        a.g2_out = g2_out.data_ptr() if g2_out is not None else None
        a.dim, a.ld = self.D, ld
        a.window, a.negative = o.window_size, (0 if o.hs else o.negative_num)
        a.cbow, a.hs, a.use_adagrad = int(o.cbow), int(o.hs), int(o.use_adagrad)
        a.lr = self.learning_rate if not o.use_adagrad else o.init_learning_rate
        a.alias_prob = N.ptr(self.alias_prob)
        a.alias_idx = N.ptr(self.alias_idx)
        a.vocab = self.V
        a.neg_pool = N.ptr(neg_pool)
        a.neg_pool_size = neg_pool.numel() if neg_pool is not None else 0
        a.neg_pool_size_ptr = N.ptr(neg_pool_size_ptr)
        if self.huffman is not None:
            a.hs_points, a.hs_codes = self.huffman.points.data_ptr(), self.huffman.codes.data_ptr()
            a.hs_len, a.hs_max_code = self.huffman.lens.data_ptr(), self.huffman.max_code
        a.map_in, a.map_out = N.ptr(map_in), N.ptr(map_out)
        self._step += 1
        a.seed = ((0x5DEECE66D * (self.rt.rank + 1)) ^ (self._step * 0x9E3779B97F4A7C15)) & 0xFFFFFFFFFFFFFFFF
        a.loss_sum = self.loss.data_ptr() if compute_loss else None
        a.pair_count = self.pairs.data_ptr()
        a.hogwild = int(self.hogwild)
        if direct:
            ti, to = self.input_table, self.output_table
            a.nservers, a.rows_per_server = ti.S, ti.rps
            for s_ in range(ti.S):
                a.w_in_peers[s_], a.w_out_peers[s_] = ti.shard_ptrs[s_], to.shard_ptrs[s_]
        a.scale_in, a.scale_out = N.ptr(self.scale_in), N.ptr(self.scale_out)
        N.cuda_lib().mvb_sgns_train(a, N.stream_ptr())
        self.kernel_launches += N.cuda_lib().mvb_sgns_last_launches()

    # ------------------------------------------------------------------ one data block
    def train_block(self, tokens: torch.Tensor, compute_loss: bool = True,
                    next_tokens: Optional[torch.Tensor] = None, next_ready: Optional[torch.cuda.Event] = None) -> None:
        """Train on one block of token ids (int32 CUDA tensor, negative = sentence break).
        Asynchronous on the current stream; read ``loss`` / ``pairs`` after a sync.

        ``next_tokens`` (world > 1, ``-is_pipeline``): the following block.  Its PrepareData +
        RequestParameter run on a side stream while this block trains, and this block's
        AddDeltaParameter runs there while the next one trains -- the reference's pipeline
        (distributed_wordembedding.cpp:199-222: an extra thread prefetches the next block's
        parameters during TrainIteration), with streams instead of an OpenMP thread.
        ``next_ready``: event after which ``next_tokens`` is valid (e.g. recorded behind its H2D copy on a
        copy stream); without it the block must be valid on the current stream at the time of the call."""
        assert tokens.is_cuda and tokens.dtype == torch.int32
        if self.rt.size == 1:
            with monitor("WE_TRAIN_BLOCK", cuda=True):
                self._launch(tokens, self.input_table.shard, self.output_table.shard,
                             None if self.g2_in is None else self.g2_in.shard,
                             None if self.g2_out is None else self.g2_out.shard, self.D,
                             compute_loss=compute_loss)
            return
        if self.mode == "direct":
            with monitor("WE_TRAIN_BLOCK", cuda=True):
                self._launch(tokens, self.input_table.shard, self.output_table.shard, None, None, self.D,
                             compute_loss=compute_loss, direct=True)
            return
        if next_tokens is None and self._prefetched is None:
            st = self._prepare_block(tokens, wait=True)
            self._train_prepared(tokens, st, compute_loss)
            self._add_delta(st)
            return
        # ---- pipelined ------------------------------------------------------------------
        main = torch.cuda.current_stream()
        if self._side is None:
            self._side = torch.cuda.Stream(device=self.dev)
        side = self._side
        st = self._prefetched
        self._prefetched = None
        if st is None or st["tokens"].data_ptr() != tokens.data_ptr() or st["tokens"].numel() != tokens.numel():
            st = self._prepare_block(tokens, wait=False)          # first block: nothing to overlap with
            self._record_streams(st, side)                        # allocated here, last used over there
        else:
            main.wait_event(st["ready"])
            self._record_streams(st, main)
        inputs_ready = torch.cuda.Event()
        inputs_ready.record(main)                                 # next_tokens (e.g. an H2D copy) is complete here
        self._train_prepared(tokens, st, compute_loss)
        trained = torch.cuda.Event()
        trained.record(main)
        with torch.cuda.stream(side):
            if next_tokens is not None:
                side.wait_event(next_ready if next_ready is not None else inputs_ready)
                nxt = self._prepare_block(next_tokens, wait=False)
                nxt["tokens"] = next_tokens
                nxt["ready"] = torch.cuda.Event()
                nxt["ready"].record(side)
                self._prefetched = nxt
            side.wait_event(trained)
            self._add_delta(st, side=True)
        self._pending_side = True

    @staticmethod
    def _record_streams(st: dict, stream) -> None:
        if st.get("dev"):
            return                      # persistent buffers: never handed back to the caching allocator
        for v in st.values():
            if isinstance(v, torch.Tensor):
                v.record_stream(stream)

    def flush(self) -> None:
        """Make the current stream wait for the pipelined AddDeltaParameter work."""
        if self._side is not None and self._pending_side:
            torch.cuda.current_stream().wait_stream(self._side)
            self._pending_side = False

    # ------------------------------------------------------------------ device-side block protocol
    def _dev_block_ok(self) -> bool:
        o = self.opt
        # the pool size of a device-prepared block is only known on the device, and only the deterministic and
        # window kernels read it there (dim <= 512, window <= 15)
        return (not o.hs and not o.cbow and not o.use_adagrad and o.negative_num >= 1 and o.negative_num <= 7
                and self.D % 4 == 0 and self.D <= 512 and o.window_size <= 15)

    def _block_buffers(self, slot: int, n_tokens: int) -> dict:
        """Fixed-capacity buffers of one in-flight block: nothing is allocated or sized on the host per
        block (the counts only exist on the device)."""
        b = self._bufs[slot]
        cap_in = min(self.V, max(int(n_tokens), 1))
        if b is not None and b["cap_in"] >= cap_in:
            return b
        o, dev, V, D = self.opt, self.dev, self.V, self.D
        cap_out = min(V, cap_in * (1 + o.negative_num))
        words = (V + 31) // 32
        i32 = dict(dtype=torch.int32, device=dev)
        b = dict(cap_in=cap_in, cap_out=cap_out, dev=True,
                 bm_in=torch.empty(words, **i32), bm_out=torch.empty(words, **i32),
                 chunk_sums=torch.empty((words + 1023) // 1024 + 1, **i32),
                 map_in=torch.empty(V, **i32), map_out=torch.empty(V, **i32),
                 ids_in=torch.empty(cap_in, **i32), ids_out=torch.empty(cap_out, **i32),
                 neg_pool=torch.empty(max(cap_in * o.negative_num, 1), **i32), counts=torch.zeros(4, **i32),
                 cache_in=torch.empty(cap_in, D, device=dev), old_in=torch.empty(cap_in, D, device=dev),
                 cache_out=torch.empty(cap_out, D, device=dev), old_out=torch.empty(cap_out, D, device=dev))
        b["n_pool"] = b["counts"][2:]
        self._bufs[slot] = b
        return b

    def _prepare_block_dev(self, tokens: torch.Tensor, side: bool) -> dict:
        """PrepareData + RequestParameter, entirely enqueued on the current stream."""
        slot = self._map_slot
        self._map_slot ^= 1
        b = self._block_buffers(slot, tokens.numel())
        o, lib = self.opt, N.cuda_lib()
        st = N.stream_ptr()
        self._step += 1
        p = N.WePrep()
        p.tokens, p.n_tokens, p.vocab, p.negative = tokens.data_ptr(), tokens.numel(), self.V, o.negative_num
        p.alias_prob, p.alias_idx = N.ptr(self.alias_prob), N.ptr(self.alias_idx)
        p.seed = ((0xA24BAED4963EE407 * (self.rt.rank + 1)) ^ (self._step * 0x9FB21C651E98DF25)) & 0xFFFFFFFFFFFFFFFF
        p.bm_in, p.bm_out, p.chunk_sums = b["bm_in"].data_ptr(), b["bm_out"].data_ptr(), b["chunk_sums"].data_ptr()
        p.map_in, p.map_out = b["map_in"].data_ptr(), b["map_out"].data_ptr()
        p.ids_in, p.ids_out = b["ids_in"].data_ptr(), b["ids_out"].data_ptr()
        p.neg_pool, p.pool_cap, p.counts = b["neg_pool"].data_ptr(), b["neg_pool"].numel(), b["counts"].data_ptr()
        p.cap_in, p.cap_out = b["cap_in"], b["cap_out"]
        with monitor("WE_PREPARE_DATA", cuda=True):
            lib.mvb_we_prepare(p, st)
        self.kernel_launches += lib.mvb_we_prepare_launches(o.negative_num)
        ctas = 1 if side else _BLOCKING_CTAS_PER_SM      # side stream: one CTA per SM next to K7's
        cnt = b["counts"].data_ptr()
        with monitor("WE_REQUEST_PARAMETER", cuda=True):
            for tab, ids, ci, cache, old, cap in ((self.input_table, b["ids_in"], 0, b["cache_in"], b["old_in"], b["cap_in"]),
                                                  (self.output_table, b["ids_out"], 1, b["cache_out"], b["old_out"], b["cap_out"])):
                lib.mvb_rows_pull(tab._rowmap, 4, ids, cnt + 4 * ci, cap, cache, old, self.D, ctas, st)
        self.kernel_launches += 2
        return b

    def _add_delta_dev(self, b: dict, side: bool) -> None:
        """AddDeltaParameter (communicator.cpp:206-249): rows += (trained - pulled) / W, pushed one-sided."""
        lib, st = N.cuda_lib(), N.stream_ptr()
        cnt = b["counts"].data_ptr()
        ctas = 1 if side else _BLOCKING_CTAS_PER_SM
        with monitor("WE_ADD_DELTA", cuda=True):
            for tab, ids, ci, cache, old, cap in ((self.input_table, b["ids_in"], 0, b["cache_in"], b["old_in"], b["cap_in"]),
                                                  (self.output_table, b["ids_out"], 1, b["cache_out"], b["old_out"], b["cap_out"])):
                lib.mvb_rows_push_delta(tab._rowmap, ids, cnt + 4 * ci, cap, cache, old, self.D, 1.0 / self.W, ctas, st)
        self.kernel_launches += 2

    def _prepare_block(self, tokens: torch.Tensor, wait: bool) -> dict:
        """PrepareData (data_block / communicator.cpp:117-155) + RequestParameter on the current stream."""
        if self._dev_block_ok():
            return self._prepare_block_dev(tokens, side=not wait)
        o, dev, V = self.opt, self.dev, self.V
        slot = self._map_slot
        self._map_slot ^= 1
        with monitor("WE_PREPARE_DATA", cuda=True):
            valid = tokens[tokens >= 0].to(torch.int64)
            in_ids = torch.unique(valid)
            neg_pool = None
            if o.hs:
                # output nodes = inner nodes on the Huffman paths of the block's words
                pts = self.huffman.points[in_ids]
                ln = self.huffman.lens[in_ids].to(torch.int64)
                m = torch.arange(pts.shape[1], device=dev)[None, :] < ln[:, None]
                out_ids = torch.unique(pts[m].to(torch.int64))
            else:
                # PrepareData: negative_num * |input| draws form the block's negative pool
                n_draw = o.negative_num * in_ids.numel()
                idx = torch.randint(0, V, (n_draw,), device=dev)
                u = torch.rand(n_draw, device=dev)
                pool = torch.where(u < self.alias_prob[idx], idx, self.alias_idx[idx].to(torch.int64))
                neg_pool = pool.to(torch.int32)
                out_ids = torch.unique(torch.cat([in_ids, pool]))
            if self._maps[slot] is None:
                self._maps[slot] = (torch.full((V,), -1, dtype=torch.int32, device=dev),
                                    torch.full((V,), -1, dtype=torch.int32, device=dev))
            map_in, map_out = self._maps[slot]            # two sets: the next block is prepared while this one trains
            map_in[in_ids] = torch.arange(in_ids.numel(), dtype=torch.int32, device=dev)
            map_out[out_ids] = torch.arange(out_ids.numel(), dtype=torch.int32, device=dev)
        # RequestParameter (communicator.cpp:117-155): pull the block's rows
        get = (lambda t, ids: t.get_rows(ids)) if wait else (lambda t, ids: t.get_rows_async(ids)[1])
        cache_in = get(self.input_table, in_ids)
        cache_out = get(self.output_table, out_ids)
        self.kernel_launches += 2
        st = dict(in_ids=in_ids, out_ids=out_ids, neg_pool=neg_pool, map_in=map_in, map_out=map_out,
                  cache_in=cache_in, cache_out=cache_out, old_in=cache_in.clone(), old_out=cache_out.clone(),
                  g2i=None, g2o=None)
        if o.use_adagrad:
            st["g2i"] = get(self.g2_in, in_ids)
            st["g2o"] = get(self.g2_out, out_ids)
            st["old_g2i"], st["old_g2o"] = st["g2i"].clone(), st["g2o"].clone()
        return st

    def _train_prepared(self, tokens: torch.Tensor, st: dict, compute_loss: bool) -> None:
        tr = getattr(self, "trace", None)
        if tr is not None:                 # benchmark tracing: K7 start / end events of every block
            e0 = torch.cuda.Event(enable_timing=True)
            e0.record()
        self._train_prepared_inner(tokens, st, compute_loss)
        if tr is not None:
            e1 = torch.cuda.Event(enable_timing=True)
            e1.record()
            tr.append((e0, e1))

    def _train_prepared_inner(self, tokens: torch.Tensor, st: dict, compute_loss: bool) -> None:
        with monitor("WE_TRAIN_BLOCK", cuda=True):
            if st.get("dev"):
                self._launch(tokens, st["cache_in"], st["cache_out"], None, None, self.D, st["map_in"], st["map_out"],
                             st["neg_pool"], compute_loss, neg_pool_size_ptr=st["n_pool"])
            else:
                self._launch(tokens, st["cache_in"], st["cache_out"], st["g2i"], st["g2o"], self.D,
                             st["map_in"], st["map_out"], st["neg_pool"], compute_loss)

    def _add_delta(self, st: dict, side: bool = False) -> None:
        # AddDeltaParameter (communicator.cpp:206-249): delta = (trained - pulled) / W
        if st.get("dev"):
            self._add_delta_dev(st, side)
            return
        o, D = self.opt, self.D
        inv = 1.0 / self.W
        in_ids, out_ids = st["in_ids"], st["out_ids"]
        if D % 4 == 0:
            self.input_table.add_rows_delta(in_ids, st["cache_in"], st["old_in"], inv)
            self.output_table.add_rows_delta(out_ids, st["cache_out"], st["old_out"], inv)
            if o.use_adagrad:
                self.g2_in.add_rows_delta(in_ids, st["g2i"], st["old_g2i"], inv)
                self.g2_out.add_rows_delta(out_ids, st["g2o"], st["old_g2o"], inv)
            self.kernel_launches += 2
        else:
            self.input_table.add_rows(in_ids, (st["cache_in"] - st["old_in"]) * inv)
            self.output_table.add_rows(out_ids, (st["cache_out"] - st["old_out"]) * inv)
            if o.use_adagrad:
                self.g2_in.add_rows(in_ids, (st["g2i"] - st["old_g2i"]) * inv)
                self.g2_out.add_rows(out_ids, (st["g2o"] - st["old_g2o"]) * inv)

    # ------------------------------------------------------------------ word count (KV)
    def add_word_count(self, n: int) -> None:
        self.wordcount_table.add(K_WORD_COUNT_ID, int(n))

    def get_word_count(self) -> int:
        self.word_count_actual = int(self.wordcount_table.get(K_WORD_COUNT_ID))
        return self.word_count_actual

    # ------------------------------------------------------------------ results
    def embeddings(self) -> torch.Tensor:
        """Whole input-embedding matrix [V, D] (SaveEmbedding pulls it in 100k-row batches)."""
        self.flush()
        return self.input_table.get().view(self.V, self.D)

    def _input_rows(self, ids: torch.Tensor) -> torch.Tensor:
        return self.input_table.get_rows(ids)

    def most_similar(self, word_ids, k: int = 10, rows: Optional[int] = None):
        """Nearest input-embedding rows by cosine (word2vec's ``distance``) of each word in ``word_ids``,
        the word itself excluded; only rows [0, ``rows``) are searched. Returns (scores [n, k], ids [n, k]).
        Searches the live table through its shards (fused top-k kernel), nothing is pulled whole."""
        from ..ops.topk import check_k, take_excluding, topk_cosine
        k = check_k(k, 1, "most_similar")
        self.flush()
        ids = torch.as_tensor(word_ids, dtype=torch.int64).to(self.dev).view(-1)
        s, i = topk_cosine(self.input_table, self._input_rows(ids), k + 1, rows)
        return take_excluding(s, i, ids[:, None], k)

    def analogy(self, a, b, c, k: int = 1, rows: Optional[int] = None):
        """3CosAdd (word2vec's ``word-analogy``): the rows nearest to unit(b) - unit(a) + unit(c), with a, b
        and c excluded, for equally long id lists a, b, c. Returns (scores [n, k], ids [n, k])."""
        from ..ops.topk import analogy_queries, check_k, take_excluding, topk_cosine
        k = check_k(k, 3, "analogy")
        self.flush()
        abc = [torch.as_tensor(x, dtype=torch.int64).to(self.dev).view(-1) for x in (a, b, c)]
        q = analogy_queries(*(self._input_rows(x) for x in abc))
        s, i = topk_cosine(self.input_table, q, k + 3, rows)
        return take_excluding(s, i, torch.stack(abc, 1), k)

    def save_embedding(self, path: str, words=None, binary: bool = False) -> None:
        """word2vec text / binary format (distributed_wordembedding.cpp:263-325); rank 0 only."""
        self.flush()
        if self.rt.rank != 0:
            return
        batch = 100000
        with open(path, "wb") as f:
            f.write(f"{self.V} {self.D}\n".encode())
            for lo in range(0, self.V, batch):
                hi = min(self.V, lo + batch)
                rows = self.input_table.get_rows(torch.arange(lo, hi, device=self.dev)).cpu().numpy()
                for i in range(hi - lo):
                    w = words[lo + i] if words is not None else str(lo + i)
                    if binary:
                        f.write(w.encode() + b" " + rows[i].astype(np.float32).tobytes() + b"\n")
                    else:
                        f.write((w + " " + " ".join(f"{x:.6f}" for x in rows[i]) + "\n").encode())


def synthetic_zipf_corpus(n_tokens: int, vocab: int, sentence_len: int = 1000, seed: int = 0,
                          exponent: float = 1.0) -> np.ndarray:
    """Synthetic corpus of the benchmark shape: Zipf(``exponent``) word ids over ``vocab``
    words, sentences of ``sentence_len`` tokens (kMaxSentenceLength, constant.h:27) separated
    by -1.  There is no network, so no real corpus."""
    rng = np.random.default_rng(seed)
    ranks = np.arange(1, vocab + 1, dtype=np.float64)
    p = ranks ** (-exponent)
    cdf = np.cumsum(p / p.sum())
    ids = np.searchsorted(cdf, rng.random(n_tokens), side="right").astype(np.int32)
    np.minimum(ids, vocab - 1, out=ids)
    if sentence_len > 0:
        ids[sentence_len::sentence_len + 1] = -1
    return ids
