"""Row mailboxes (csrc/cuda/rowbox.cu) against a model of their protocol and the fp64 updater models.

S ranks are emulated on one device: each has its own ``RowBox`` (``me = r``) over its slab of a zero-filled mailbox
buffer, its own ack array and scratch, and the ranks share one error flag. Every launch goes on one stream in an
order the protocol model checked first: a push of epoch e > 2 only after every owner has applied that source's epoch
e - 2, a waiting poll only after the pushes it waits for. So no kernel waits on a later one, and a correct run never
spins (the short watchdog is a safety net).

After every push the owners' slots are read bitwise: header (seq, count, option bytes), ids and values
(``fp32(v * scale)`` or ``fp32(fp32(cur - old) * scale)``, bit-exact). After every event the counters (``applied``,
``ack``, ``done``, the error flag) match the model, and the shards and every source's state slabs match ServerModel,
RowwiseModel or AdamModel applied the way an owner drains: per drain, sources in rank order, one push each, the
source's rank as the worker id. The pushed option carries worker id 0, so an apply that takes the worker from the
header picks the wrong state slab. Rows never named, the padding between state slabs and the guard bands stay
bitwise unchanged.

The Python path sends ``add_rows`` through the mailbox of a one-process table (repeated ids in shuffled order, ids
that are negative, >= num_row or >= 2^31, more entries than a slot holds) and holds it and the owner-side row Add to
the same models.
"""

import numpy as np
import pytest
import torch

from test_adam_cpu import OPTS as ADAM_OPTS, AdamModel
from test_rowwise_adagrad_cpu import RowwiseModel
from test_table_numerics import _KSENT, _OPTS, _STATES, ServerModel, _assert_close, _delta, _start_values

UPDATERS = ["default", "sgd", "momentum_sgd", "adagrad", "dcasgd", "dcasgda", "rowwise_adagrad", "adam"]
GUARD = 16                     # floats of _KSENT around every region; a multiple of 4 keeps each region 16-byte aligned
HDR = 128
# (ranks, row map, columns): an even split, a remainder owner of 2 rps - 1 rows, and fewer rows than ranks
CONFIGS = [(1, "even", 68), (1, "rem", 1028), (2, "rem", 4), (2, "tiny", 388), (3, "even", 1028), (3, "tiny", 68),
           (8, "rem", 388), (8, "tiny", 4), (8, "even", 68)]
ROWS = {"even": lambda S: 56 * S, "rem": lambda S: 30 * S + 29, "tiny": lambda S: {2: 1, 3: 2, 8: 3}[S]}


def _split(num_row, S):
    """rows_per_server and each rank's [lo, hi), as tables/device.py partitions a table."""
    if num_row >= S:
        rps = num_row // S
        lo, hi = [s * rps for s in range(S)], [(s + 1) * rps for s in range(S)]
        hi[-1] = num_row
    else:
        rps, lo, hi = 1, [min(s, num_row) for s in range(S)], [min(s + 1, num_row) for s in range(S)]
    return rps, lo, hi


def _options(updater, k, worker):
    """The k-th AddOption for the model (worker id ``worker``) and its C struct with worker id 0."""
    from multiverso_b200.tables.device import _opt_struct
    from multiverso_b200.tables.options import AddOption
    if updater == "adam":
        b1, lr, rho = ADAM_OPTS[k % len(ADAM_OPTS)]
        o = AddOption(worker_id=worker, momentum=b1, learning_rate=lr, rho=rho)
    else:
        m, lr, rho, lam = _OPTS[k % len(_OPTS)]
        o = AddOption(worker_id=worker, momentum=m, learning_rate=lr, rho=rho, lambda_=lam)
    c = _opt_struct(o)
    c.worker_id = 0
    return o, c


def _model(updater, start, cols, S):
    if updater == "rowwise_adagrad":
        return RowwiseModel(start, cols, "float32", workers=S)
    if updater == "adam":
        return AdamModel(start, cols, "float32")
    return ServerModel(start, cols, updater, "float32", workers=S)


# ------------------------------------------------------------------------------------------ the protocol model
def check_schedule(S, events):
    """Replay a schedule against the protocol and assert that no launch would wait on a later one."""
    pushed, applied = [0] * S, [[0] * S for _ in range(S)]
    for ev in events:
        if ev[0] == "push":
            src = ev[1]
            e = pushed[src] + 1
            assert e <= 2 or all(applied[o][src] >= e - 2 for o in range(S)), f"push {ev} before its slot is free"
            pushed[src] = e
        else:
            _, o, wait = ev
            if wait:
                assert all(pushed[w] > applied[o][w] for w in range(S)), f"waiting drain {ev} before the push"
            for w in range(S):
                if pushed[w] > applied[o][w]:
                    applied[o][w] += 1
    return pushed, applied


def make_schedule(rng, S, n_events):
    """A random legal schedule: sources push different numbers of times (up to two outstanding each), owners drain
    with and without waiting, some drains find nothing; it ends with drains until every push is applied."""
    weights = np.array([1.0 + (w % 3) for w in range(S)])
    weights /= weights.sum()
    pushed, applied = [0] * S, [[0] * S for _ in range(S)]
    events = []
    while len(events) < n_events:
        if rng.random() < 0.5:
            src = int(rng.choice(S, p=weights))
            e = pushed[src] + 1
            if e > 2 and min(applied[o][src] for o in range(S)) < e - 2:
                continue
            events.append(("push", src))
            pushed[src] = e
        else:
            o = int(rng.integers(S))
            wait = int(all(pushed[w] > applied[o][w] for w in range(S)) and rng.random() < 0.5)
            events.append(("drain", o, wait))
            for w in range(S):
                if pushed[w] > applied[o][w]:
                    applied[o][w] += 1
    while any(pushed[w] > applied[o][w] for o in range(S) for w in range(S)):
        for o in range(S):
            events.append(("drain", o, 0))
            for w in range(S):
                if pushed[w] > applied[o][w]:
                    applied[o][w] += 1
    return events


# ------------------------------------------------------------------------------------------ id lists
KINDS = ["one_owner", "all", "none", "empty", "full_range", "edges", "runs"]


def make_ids(rng, kind, num_row, lo, hi, cap):
    """A sorted int64 id list of one kind, with at most ``cap`` entries per owner."""
    S = len(lo)
    owners = [o for o in range(S) if hi[o] > lo[o]]
    bad = [-(2 ** 31), -1, num_row, num_row + 1, 2 ** 31 - 1]
    if kind == "one_owner":
        o = owners[int(rng.integers(len(owners)))]
        ids = rng.integers(lo[o], hi[o], int(rng.integers(1, cap + 1)))
    elif kind == "all":
        ids = rng.choice(num_row, int(rng.integers(1, num_row + 1)), replace=False)
    elif kind == "none":
        ids = np.array(bad)
    elif kind == "empty":
        ids = np.array([], dtype=np.int64)
    elif kind == "full_range":
        o = owners[int(rng.integers(len(owners)))]
        ids = np.arange(lo[o], hi[o])
    elif kind == "edges":
        ids = np.array([x for o in owners for x in (lo[o], hi[o] - 1)] + bad[1:3])
    else:   # runs of a repeated row (one longer than 32) among other rows and out-of-range ids
        hot = rng.choice(num_row, min(2, num_row), replace=False)
        reps = [50, int(rng.integers(2, 33))][:len(hot)]
        ids = np.concatenate([np.repeat(hot, reps), rng.choice(num_row, min(10, num_row)), bad])
    ids = np.sort(np.asarray(ids, dtype=np.int64), kind="stable")
    keep, per = [], {}
    for x in ids.tolist():          # at most cap entries per owner
        if 0 <= x < num_row:
            o = min(x // (num_row // S if num_row >= S else 1), S - 1)
            if per.get(o, 0) == cap:
                continue
            per[o] = per.get(o, 0) + 1
        keep.append(x)
    return np.asarray(keep, dtype=np.int64)


# ------------------------------------------------------------------------------------------ the emulated world
class World:
    def __init__(self, S, num_row, cols, updater, rng):
        from multiverso_b200 import _native as N
        self.N, self.lib = N, N.cuda_lib()
        self.S, self.num_row, self.C, self.updater = S, num_row, cols, updater
        self.rps, self.lo, self.hi = _split(num_row, S)
        self.cap = max(h - l for l, h in zip(self.lo, self.hi))
        self.slot_bytes = (self.lib.mvb_rowbox_slot_bytes(self.cap, cols) + 255) // 256 * 256
        self.ids_bytes = (self.cap * 4 + 127) // 128 * 128
        self.nslots = self.lib.mvb_rowbox_slots()
        dev = "cuda"
        self.box = torch.zeros(S, S * self.nslots * self.slot_bytes, dtype=torch.uint8, device=dev)
        self.ack = torch.zeros(S, N.MAX_RANKS, dtype=torch.int64, device=dev)
        self.seg = torch.zeros(S, S + 4, dtype=torch.int32, device=dev)
        self.done = torch.zeros(S, 4, dtype=torch.int32, device=dev)
        self.applied = torch.zeros(S, S, dtype=torch.int64, device=dev)
        self.go = torch.zeros(S, S, dtype=torch.int32, device=dev)
        self.err = torch.zeros(4, dtype=torch.int32, device=dev)
        self.start = _start_values(rng, num_row * cols, np.float32).reshape(num_row, cols)
        self.model = _model(updater, self.start, cols, S)
        # per rank one float buffer: [G shard G st0 G st1 G]; a state region is one slab (shared state) or S slabs
        # (per-worker state) of `stride` elements whose tail past the slab's length keeps the sentinel
        nst, per_worker = _STATES.get(updater, (1, True) if updater == "rowwise_adagrad" else (2, False))
        self.nst, self.nslab = nst, (S if per_worker else 1)
        self.buf, self.ref, self.at = [], [], []
        for r in range(S):
            n = self.hi[r] - self.lo[r]
            ln = n if updater == "rowwise_adagrad" else n * cols
            stride = (ln + 3) // 4 * 4 + 8
            at = {"n": n, "len": ln, "stride": stride, "shard": GUARD}
            pos = GUARD + n * cols + GUARD
            for i in range(nst):
                at[f"st{i}"] = pos
                size = stride * self.nslab + ((n + 3) // 4 * 4 if updater == "adam" and i == 1 else 0)
                pos += size + GUARD
            init = np.full(pos, _KSENT, dtype=np.float32)
            init[GUARD:GUARD + n * cols] = self.start[self.lo[r]:self.hi[r]].reshape(-1)
            for i in range(nst):
                for w in range(self.nslab):
                    init[at[f"st{i}"] + w * stride:][:ln] = 0
                if updater == "adam" and i == 1:
                    init[at["st1"] + stride:][:n] = 0          # step counts after v's slab
            self.ref.append(init)
            self.buf.append(torch.from_numpy(init.copy()).cuda())
            self.at.append(at)
        self.boxes = []
        for r in range(S):
            b = N.RowBox()
            b.map.num_row, b.map.num_col, b.map.nservers, b.map.rows_per_server = num_row, cols, S, self.rps
            b.me, b.cap, b.slot_bytes = r, self.cap, self.slot_bytes
            for q in range(S):
                b.box[q] = self.box[q].data_ptr()
                b.ack[q] = self.ack[q].data_ptr()
            b.seg, b.done = self.seg[r].data_ptr(), self.done[r].data_ptr()
            b.applied, b.go = self.applied[r].data_ptr(), self.go[r].data_ptr()
            b.err_flag, b.timeout_s = self.err.data_ptr(), 5.0
            self.boxes.append(b)
        self.pushed = [0] * S
        self.log = [dict() for _ in range(S)]             # source -> epoch -> (ids, values, option) per owner
        self.applied_m = [[0] * S for _ in range(S)]
        self.nopt = 0
        self.keep = []

    def _ptr(self, r, name):
        a = self.at[r]
        if name == "shard":
            return self.buf[r].data_ptr() + 4 * a["shard"]
        i = int(name[2])
        return self.buf[r].data_ptr() + 4 * a[name] if i < self.nst else None

    def owner(self, x):
        return min(x // self.rps, self.S - 1)

    # ---- events
    def push(self, rng, src, kind, delta, padded):
        ids = make_ids(rng, kind, self.num_row, self.lo, self.hi, self.cap)
        n = ids.size
        extra = int(rng.integers(1, 4)) if padded else 0
        n_max, ld = n + extra, self.C + 4
        all_ids = np.concatenate([ids, rng.integers(0, self.num_row, extra)]).astype(np.int32)
        cur = np.full((n_max, ld), 3.0e4, dtype=np.float32)        # the padding and garbage rows must never be read
        cur[:, :self.C] = 0.5 * _delta(rng, (n_max, self.C), np.float32)
        old = np.full((n_max, ld), -3.0e4, dtype=np.float32)
        old[:, :self.C] = 0.5 * _delta(rng, (n_max, self.C), np.float32)
        scale = np.float32([1.0, 0.5, -0.75][int(rng.integers(3))])
        e = self.pushed[src] + 1
        opt, copt = _options(self.updater, self.nopt, src)
        self.nopt += 1
        ids_d = torch.from_numpy(all_ids).cuda()
        n_d = torch.tensor([n], dtype=torch.int32, device="cuda") if padded else None
        cur_d, old_d = torch.from_numpy(cur).cuda(), torch.from_numpy(old).cuda()
        self.keep.append((ids_d, n_d, cur_d, old_d))
        st = self.N.stream_ptr()
        if delta:
            self.lib.mvb_rowbox_push_delta(self.boxes[src], ids_d, n_d, n_max, cur_d, old_d, ld, float(scale), e,
                                           copt, 1, st)
            v = (cur[:n, :self.C] - old[:n, :self.C]) * scale
        else:
            self.lib.mvb_rowbox_push_vals(self.boxes[src], ids_d, n_d, n_max, cur_d, ld, float(scale), e, copt, 1, st)
            v = cur[:n, :self.C] * scale
        assert v.dtype == np.float32
        per = {}
        for o in range(self.S):
            sel = np.array([0 <= x < self.num_row and self.owner(x) == o for x in ids.tolist()], dtype=bool)
            per[o] = (ids[sel], v[sel], opt)
        self.pushed[src] = e
        self.log[src][e] = (per, bytes(copt))
        what = f"push {e} of source {src} ({kind}, {'delta' if delta else 'vals'}, n_ptr={padded})"
        torch.cuda.synchronize()
        self.check_slots(src, e, what)
        return what

    def drain(self, o, wait):
        st = self.N.stream_ptr()
        self.lib.mvb_rowbox_poll(self.boxes[o], -1, wait, st)
        upd = self.N.UPDATER_NAMES[self.updater]
        for w in range(self.S):
            self.lib.mvb_rowbox_apply(self.boxes[o], upd, self._ptr(o, "shard"), self._ptr(o, "st0"),
                                      self._ptr(o, "st1"), self.at[o]["stride"], self.lo[o], w, 1, st)
        for w in range(self.S):
            want = self.applied_m[o][w] + 1
            if self.pushed[w] >= want:
                ids, v, opt = self.log[w][want][0][o]
                self.model.add_rows(ids, v, opt)
                self.applied_m[o][w] = want
        torch.cuda.synchronize()
        return f"drain of owner {o} (wait={wait})"

    # ---- checks
    def check_slots(self, src, e, what):
        per, opt_bytes = self.log[src][e]
        box = self.box.cpu().numpy()
        for o in range(self.S):
            ids, v, _ = per[o]
            base = (src * self.nslots + (e & 1)) * self.slot_bytes
            slot = box[o, base:base + self.slot_bytes]
            hdr = slot[:HDR]
            assert int(hdr[:8].view(np.uint64)[0]) == e, f"{what}: owner {o} seq"
            assert int(hdr[8:12].view(np.int32)[0]) == ids.size, \
                f"{what}: owner {o} count {int(hdr[8:12].view(np.int32)[0])}, expected {ids.size}"
            assert bytes(hdr[16:16 + len(opt_bytes)]) == opt_bytes, f"{what}: owner {o} option bytes"
            got_ids = slot[HDR:HDR + 4 * ids.size].view(np.int32)
            assert np.array_equal(got_ids, ids.astype(np.int32)), f"{what}: owner {o} ids {got_ids} != {ids}"
            vb = HDR + self.ids_bytes
            got_v = slot[vb:vb + 4 * ids.size * self.C].view(np.uint32)
            assert np.array_equal(got_v, v.reshape(-1).view(np.uint32)), f"{what}: owner {o} values not bit-exact"

    def check(self, what):
        S = self.S
        assert int(self.err[0]) == 0, f"{what}: error flag {int(self.err[0])}"
        assert not self.done.any(), f"{what}: a completion counter was left non-zero"
        applied, ack = self.applied.cpu().numpy(), self.ack.cpu().numpy()
        for o in range(S):
            for w in range(S):
                assert applied[o, w] == self.applied_m[o][w], f"{what}: applied[{o}][{w}] = {applied[o, w]}"
                assert ack[w, o] == self.applied_m[o][w], f"{what}: ack[{w}][{o}] = {ack[w, o]}"
        bufs = [b.cpu().numpy() for b in self.buf]
        written = [np.zeros(b.size, dtype=bool) for b in bufs]
        shard = np.concatenate([bufs[r][self.at[r]["shard"]:][:self.at[r]["n"] * self.C] for r in range(S)])
        shard = shard.reshape(self.num_row, self.C)

        def slabs(i, w, ln):
            out = []
            for r in range(S):
                a = self.at[r]
                off = a[f"st{i}"] + w * a["stride"]
                n = a["len"] if ln is None else ln(a)
                written[r][off:off + n] = True
                out.append(bufs[r][off:off + n])
            return np.concatenate(out)

        for r in range(S):
            written[r][self.at[r]["shard"]:][:self.at[r]["n"] * self.C] = True
        m, u = self.model, self.updater
        if u == "rowwise_adagrad":
            m.check_values(shard, "float32", what)
            for w in range(S):
                m.check_state(slabs(0, w, None), w, "float32", what)
        elif u == "adam":
            m.check_values(shard, what)
            mm, vv = slabs(0, 0, None), slabs(1, 0, None)
            tt = np.concatenate([bufs[r][self.at[r]["st1"] + self.at[r]["stride"]:][:self.at[r]["n"]]
                                 for r in range(S)])
            for r in range(S):
                written[r][self.at[r]["st1"] + self.at[r]["stride"]:][:self.at[r]["n"]] = True
            m.check_state(mm, vv, tt, what)
        else:
            _assert_close(shard, m.data, np.abs(m.data) + m.mag, m.nupd, "float32", f"{what} values")
            for i in range(len(m.state)):
                for w in range(m.state[i].shape[0]):
                    _assert_close(slabs(i, w, None), m.state[i][w].reshape(-1), m.state_scale(i, w).reshape(-1),
                                  m.nupd.reshape(-1), "float32", f"{what} state{i}[worker {w}]")
        never = m.nupd[:, 0] == 0
        assert np.array_equal(shard[never].view(np.uint32), self.start[never].view(np.uint32)), \
            f"{what}: a row never named changed"
        for r in range(S):
            assert np.array_equal(bufs[r][~written[r]].view(np.uint32), self.ref[r][~written[r]].view(np.uint32)), \
                f"{what}: rank {r} memory outside the shard and the state slabs was written"


@pytest.mark.gpu
@pytest.mark.parametrize("S,rowmap,cols", CONFIGS)
@pytest.mark.parametrize("updater", UPDATERS)
def test_emulated_ranks(mv_device, updater, S, rowmap, cols):
    """A random legal schedule of pushes and drains over S emulated ranks, every push's id list of one kind in turn
    (one owner, every owner, no row, empty, one owner's full range, every owner's first and last row, runs of a
    repeated row up to 50 long), with negative and >= num_row ids, alternating value and delta pushes, half of them
    with a device count and garbage rows after it; slots, counters, values, state and untouched memory checked after
    every event."""
    num_row = ROWS[rowmap](S)
    seed = 1000 * S + 10 * cols + UPDATERS.index(updater) + len(rowmap)
    rng = np.random.default_rng(seed)
    events = make_schedule(rng, S, 24 + 12 * S)
    pushed, _ = check_schedule(S, events)
    world = World(S, num_row, cols, updater, rng)
    assert max(pushed) >= 3, "the schedule reuses no slot"
    j = 0
    for ev in events:
        if ev[0] == "push":
            what = world.push(rng, ev[1], KINDS[j % len(KINDS)], delta=j % 2 == 1, padded=(j // 2) % 2 == 1)
            j += 1
        else:
            what = world.drain(ev[1], ev[2])
        world.check(f"{updater} S={S} {rowmap} C={cols}: after {what}")
    from multiverso_b200.runtime import Runtime
    Runtime.get().check_watchdog()


# ------------------------------------------------------------------------------------------ the Python path
def _py_model(updater, start, cols):
    return _model(updater, start, cols, 1)


def _py_check(t, model, updater, what):
    got = t.get().cpu().numpy()
    if updater == "rowwise_adagrad":
        model.check_values(got, "float32", what)
        model.check_state(t.state[0][:t.num_row].cpu().numpy(), 0, "float32", what)
    elif updater == "adam":
        model.check_values(got, what)
        rows = t.my_len // t.num_col
        model.check_state(t.state[0][:t.my_len].cpu().numpy(), t.state[1][:t.my_len].cpu().numpy(),
                          t.state[1][t.state_stride:t.state_stride + rows].cpu().numpy(), what)
    else:
        got = got.reshape(model.data.shape)
        _assert_close(got, model.data, np.abs(model.data) + model.mag, model.nupd, "float32", f"{what} values")
        for i in range(len(model.state)):
            st = t.state[i][:t.my_len].cpu().numpy().reshape(model.data.shape)
            _assert_close(st, model.state[i][0], model.state_scale(i, 0), model.nupd, "float32", f"{what} state{i}")


@pytest.mark.gpu
@pytest.mark.parametrize("updater", UPDATERS[2:])
def test_python_add_rows(mv_device, updater):
    """``add_rows`` through the mailbox of a one-process table and through the owner-side row Add, against the
    model: hot rows repeated 50 and 33 times in shuffled order, ids -1, -2^33, num_row, 2^31 and 2^32 + 5, more
    entries than the slot's 40; row 5 is never named and stays bitwise unchanged."""
    from multiverso_b200.runtime import Runtime
    mv = mv_device
    rows, cols = 40, 68
    rng = np.random.default_rng(7 + UPDATERS.index(updater))
    tm = mv.MatrixTable(rows, cols, "float32", updater=updater, min_value=-1.0, max_value=1.0)
    to = mv.MatrixTable(rows, cols, "float32", updater=updater, min_value=-1.0, max_value=1.0)
    mb = tm.enable_row_mailbox()
    assert mb.cap == rows and to._mailbox is None
    push = mb.push_vals

    def checked_push(ids32, vals, option=None, **kw):
        # the push contract, checked before anything is launched: ascending ids in [-1, num_row), at most cap
        x = ids32.cpu().numpy()
        assert ids32.dtype == torch.int32 and x.size <= mb.cap, f"a push of {x.size} entries (slot: {mb.cap})"
        assert ((x >= -1) & (x < rows)).all(), f"pushed ids outside [-1, {rows}): {sorted(set(x[(x < -1) | (x >= rows)]))}"
        assert (np.diff(x) >= 0).all(), "pushed ids not ascending"
        return push(ids32, vals, option, **kw)

    mb.push_vals = checked_push
    models = [_py_model(updater, t.get().cpu().numpy(), cols) for t in (tm, to)]
    start5 = [t.get().cpu().numpy().reshape(rows, cols)[5].copy() for t in (tm, to)]
    others = np.setdiff1d(np.arange(rows), [5, 7, 19])
    bad = [-1, -(2 ** 33), rows, 2 ** 31, 2 ** 32 + 5]
    for k in range(3):
        ids = rng.permutation(np.concatenate([np.repeat([7, 19], [50, 33]), rng.choice(others, 15, replace=False),
                                              bad])).astype(np.int64)
        assert ids.size > mb.cap
        v = _delta(rng, (ids.size, cols), np.float32)
        opt, _ = _options(updater, k, 0)
        for t, model in zip((tm, to), models):
            t.add_rows(torch.from_numpy(ids).cuda(), torch.from_numpy(v).cuda(), opt)
            model.add_rows(ids, v, opt)
    torch.cuda.synchronize()
    assert mb.epoch >= 9, "the lists were not split into pushes of at most cap entries"
    for _ in range(mb.nslots):
        tm.drain_rows()
    mb.drain_stream.synchronize()
    Runtime.get().check_watchdog()
    for t, model, s5, path in zip((tm, to), models, start5, ("mailbox", "owner")):
        _py_check(t, model, updater, f"add_rows {updater} ({path})")
        got5 = t.get().cpu().numpy().reshape(rows, cols)[5]
        assert np.array_equal(got5.view(np.uint32), s5.view(np.uint32)), f"{path}: row 5 changed"


@pytest.mark.gpu
def test_overflowing_push_is_reported_and_clamped(mv_device):
    """A push that names more rows of one owner than a slot holds (allowed by no caller: ``add_rows`` splits such a
    list) sets the error flag to 3100 + owner, publishes a count of ``cap`` and keeps the first ``cap`` entries, so
    the apply never reads past the slot; those entries are applied and nothing else changes."""
    S, cols = 2, 68
    rng = np.random.default_rng(3)
    world = World(S, ROWS["rem"](S), cols, "adagrad", rng)
    o, cap = 1, world.cap
    ids = np.sort(rng.integers(world.lo[o], world.hi[o], cap + 5)).astype(np.int64)
    v = 0.5 * _delta(rng, (ids.size, cols), np.float32)
    opt, copt = _options("adagrad", 0, 0)
    lib, N = world.lib, world.N
    lib.mvb_rowbox_push_vals(world.boxes[0], torch.from_numpy(ids.astype(np.int32)).cuda(), None, ids.size,
                             torch.from_numpy(v).cuda(), cols, 1.0, 1, copt, 1, N.stream_ptr())
    torch.cuda.synchronize()
    assert int(world.err[0]) == 3100 + o, f"error flag {int(world.err[0])}"
    slot = world.box[o, (0 * world.nslots + 1) * world.slot_bytes:][:world.slot_bytes].cpu().numpy()
    assert int(slot[8:12].view(np.int32)[0]) == cap, "the published count exceeds the slot"
    assert np.array_equal(slot[HDR:HDR + 4 * cap].view(np.int32), ids[:cap].astype(np.int32))
    world.err.zero_()
    world.pushed[0] = 1
    world.log[0][1] = ({0: (ids[:0], v[:0], opt), 1: (ids[:cap], v[:cap], opt)}, bytes(copt))
    for q in range(S):
        world.drain(q, 0)
    world.check("overflowing push")
