"""The graph walker without a GPU: the numpy reference walker (the oracle of the GPU tests) against exactly enumerated
DeepWalk / node2vec transition probabilities, with the rejection and the fallback each on their own; its draws
against split calls; Graph.from_edges against scipy.sparse; the native edge-list reader against a numpy parse; the
app's arguments and its refusal to run without a GPU."""
import numpy as np
import pytest
import scipy.sparse as sp
import scipy.stats
import torch

from multiverso_b200.ops import Graph, random_walks, random_walks_reference
from multiverso_b200.ops import random_walk as rw

N_WALKS = 20000
GRAPHS = {
    "path": dict(src=[0, 1, 2, 3], dst=[1, 2, 3, 4], start=1),
    "star": dict(src=[0, 0, 0, 0, 0], dst=[1, 2, 3, 4, 5], start=0),
    "triangle_tail": dict(src=[0, 1, 2, 2], dst=[1, 2, 0, 3], start=2),
    "directed_dead_end": dict(src=[0, 1, 1, 2, 2], dst=[1, 2, 3, 0, 3], start=1, directed=True),
    "multi_edge": dict(src=[0, 0, 1, 1, 2], dst=[1, 1, 2, 3, 3], start=1),
    "self_loop": dict(src=[0, 0, 1, 1], dst=[0, 1, 2, 1], start=1),
    "weighted": dict(src=[0, 1, 2, 2, 1], dst=[1, 2, 0, 3, 3], weights=[1.0, 3.0, 0.5, 2.0, 1.5], start=1),
}
PQ = [(p, q) for p in (0.25, 1.0, 4.0) for q in (0.25, 1.0, 4.0)]
EXTREME = (1000.0, 1000.0)      # alpha 1e-3 off t's list: most steps there end in the fallback


def _graph(name):
    d = GRAPHS[name]
    return Graph.from_edges(d["src"], d["dst"], d.get("weights"), directed=d.get("directed", False),
                            device="cpu"), d["start"]


def _lists(g):
    ip, ind = g.indptr.numpy(), g.indices.numpy()
    w = np.ones(ind.size) if g.cum is None else np.diff(np.concatenate([[0.0], g.cum.numpy()]))
    if g.cum is not None:           # the first weight of each list is its prefix sum itself
        w[ip[:-1][ip[1:] > ip[:-1]]] = g.cum.numpy()[ip[:-1][ip[1:] > ip[:-1]]]
    return [(ind[ip[v]:ip[v + 1]], w[ip[v]:ip[v + 1]]) for v in range(g.num_nodes)]


def _step(lists, t, v, p, q):
    """{x: probability} of the step from v after t (t None: first order), by node2vec's formula in fp64."""
    xs, ws = lists[v]
    if len(xs) == 0:
        return {-1: 1.0}
    a = np.ones(len(xs))
    if t is not None:
        tl = set(lists[t][0].tolist())
        a = np.array([1 / p if x == t else (1.0 if x in tl else 1 / q) for x in xs])
    pr = ws * a / (ws * a).sum()
    out = {}
    for x, v_ in zip(xs.tolist(), pr):
        out[x] = out.get(x, 0.0) + v_
    return out


def _exact_two_steps(g, start, p, q):
    lists = _lists(g)
    out = {}
    for x1, p1 in _step(lists, None, start, p, q).items():
        for x2, p2 in (_step(lists, start, x1, p, q) if x1 >= 0 else {-1: 1.0}).items():
            out[(x1, x2)] = out.get((x1, x2), 0.0) + p1 * p2
    return out


def _chi2(g, start, p, q, seed):
    w = random_walks_reference(g, np.full(N_WALKS, start), 3, p, q, seed)
    assert (w[:, 0] == start).all()
    exact = _exact_two_steps(g, start, p, q)
    keys = sorted(exact)
    seen = {}
    for a, b in zip(w[:, 1].tolist(), w[:, 2].tolist()):
        seen[(a, b)] = seen.get((a, b), 0) + 1
    assert set(seen) <= set(keys), (set(seen) - set(keys))
    obs = np.array([seen.get(k, 0) for k in keys], dtype=np.float64)
    exp = np.array([exact[k] for k in keys]) * N_WALKS
    if len(keys) == 1:
        return 1.0
    return scipy.stats.chisquare(obs, exp).pvalue


@pytest.mark.parametrize("name", sorted(GRAPHS))
@pytest.mark.parametrize("pq", PQ + [EXTREME])
def test_reference_matches_exact_two_step_probabilities(name, pq):
    g, start = _graph(name)
    assert _chi2(g, start, *pq, seed=11) > 1e-4


@pytest.mark.parametrize("rounds", [0, 10 ** 6])
@pytest.mark.parametrize("name", ["triangle_tail", "directed_dead_end", "weighted", "self_loop"])
@pytest.mark.parametrize("pq", [(0.25, 4.0), (4.0, 0.25)])
def test_rejection_alone_and_fallback_alone_are_exact(monkeypatch, name, pq, rounds):
    """R = 0: every second-order step is the inversion; R huge: every step ends in an acceptance."""
    monkeypatch.setattr(rw, "REJECT_ROUNDS", rounds)
    g, start = _graph(name)
    assert _chi2(g, start, *pq, seed=5) > 1e-4


def test_first_order_is_deepwalk_and_one_step_law():
    g, start = _graph("weighted")
    w = random_walks_reference(g, np.full(N_WALKS, start), 2, seed=3)
    exact = _step(_lists(g), None, start, 1, 1)
    keys = sorted(exact)
    obs = np.array([(w[:, 1] == k).sum() for k in keys], dtype=np.float64)
    assert scipy.stats.chisquare(obs, np.array([exact[k] for k in keys]) * N_WALKS).pvalue > 1e-4


def _random_graph(n=300, m=2000, seed=0, weighted=False, directed=False):
    rng = np.random.default_rng(seed)
    src, dst = rng.integers(0, n, m), rng.integers(0, n, m)
    w = rng.uniform(0.1, 5.0, m) if weighted else None
    return Graph.from_edges(src, dst, w, num_nodes=n + 5, directed=directed, device="cpu")   # 5 isolated nodes


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("pq", [(1.0, 1.0), (0.25, 4.0), EXTREME])
def test_split_calls_equal_one_call(weighted, pq):
    g = _random_graph(weighted=weighted, directed=True)
    starts = np.arange(g.num_nodes).repeat(2)
    one = random_walks_reference(g, starts, 20, *pq, seed=9, first_walk=100)
    parts = [random_walks_reference(g, starts[a:b], 20, *pq, seed=9, first_walk=100 + a)
             for a, b in ((0, 1), (1, 257), (257, starts.size))]
    assert np.array_equal(one, np.concatenate(parts))
    assert np.array_equal(one, random_walks(g, torch.from_numpy(starts), 20, *pq, seed=9, first_walk=100).numpy())
    assert not np.array_equal(one, random_walks_reference(g, starts, 20, *pq, seed=10, first_walk=100))
    iso = np.arange(g.num_nodes - 5, g.num_nodes)
    assert (one[starts >= g.num_nodes - 5, 1:] == -1).all() and set(one[starts >= g.num_nodes - 5, 0]) == set(iso)
    ip = g.indptr.numpy()
    for row in one[:50]:                                   # every step follows an arc, -1 only after a dead end
        k = np.nonzero(row < 0)[0]
        end = k[0] if k.size else row.size
        assert (row[end:] == -1).all()
        for a, b in zip(row[:end - 1], row[1:end]):
            assert b in g.indices.numpy()[ip[a]:ip[a + 1]]
        if end < row.size:
            assert ip[row[end - 1] + 1] == ip[row[end - 1]]


def test_draws_match_the_stated_formula():
    """hash64 is MurmurHash3's finaliser, the torch version equals the numpy one, and the first step of an unweighted
    walk is the list entry ((draw >> 32) deg) >> 32 of draw(g, 1, 0)."""
    x = np.array([0, 1, 2, 2 ** 63, 2 ** 64 - 1], dtype=np.uint64)
    assert rw.hash64(np.array([0], dtype=np.uint64))[0] == 0
    assert np.array_equal(rw.hash64_torch(torch.from_numpy(x.view(np.int64))).numpy().view(np.uint64), rw.hash64(x))
    g = _random_graph()
    w = random_walks_reference(g, [7], 2, seed=4, first_walk=33)
    key = rw.hash64(rw.hash64(np.uint64(4) ^ np.uint64(0x9E3779B97F4A7C15)) + np.uint64(33) *
                    np.uint64(0xBF58476D1CE4E5B9))
    r = int(rw.hash64(key + np.uint64((1 << 32) | 0) * np.uint64(0x94D049BB133111EB)))
    ip = g.indptr.numpy()
    deg = int(ip[8] - ip[7])
    assert w[0, 1] == g.indices.numpy()[ip[7] + (((r >> 32) * deg) >> 32)]


def _scipy_counts(src, dst, n, w=None):
    data = np.ones(len(src)) if w is None else np.asarray(w, dtype=np.float64)
    m = sp.coo_matrix((data, (src, dst)), shape=(n, n)).tocsr()
    m.sort_indices()
    return m


@pytest.mark.parametrize("directed", [False, True])
def test_from_edges_matches_scipy(directed):
    rng = np.random.default_rng(1)
    n, m = 60, 400
    src, dst = rng.integers(0, n, m), rng.integers(0, n, m)
    src[:20], dst[:20] = src[20:40], dst[20:40]             # duplicates
    src[40:45] = dst[40:45]                                 # self-loops
    w = rng.uniform(0.5, 2.0, m)
    g = Graph.from_edges(src, dst, w, num_nodes=n, directed=directed, device="cpu")
    if directed:
        s2, d2, w2 = src, dst, w
    else:
        back = src != dst
        s2, d2, w2 = np.concatenate([src, dst[back]]), np.concatenate([dst, src[back]]), np.concatenate([w, w[back]])
    cnt = _scipy_counts(s2, d2, n)
    ip, ind = g.indptr.numpy(), g.indices.numpy()
    assert np.array_equal(ip, np.concatenate([[0], np.cumsum(np.asarray(cnt.sum(1)).ravel().astype(np.int64))]))
    for v in range(n):
        row = cnt[v]
        assert np.array_equal(ind[ip[v]:ip[v + 1]], np.repeat(row.indices, row.data.astype(np.int64)))
    wm = _scipy_counts(s2, d2, n, w2)
    assert np.allclose(g.degree().numpy(), np.asarray(wm.sum(1)).ravel(), rtol=1e-12)
    cum = g.cum.numpy()
    for v in range(n):                                     # per-list prefix sums, in list order (stable sort)
        o = np.lexsort((d2, s2))
        seg = w2[o][ip[v]:ip[v + 1]]
        assert np.array_equal(cum[ip[v]:ip[v + 1]], np.cumsum(seg))
    gu = Graph.from_edges(src, dst, num_nodes=n, directed=directed, device="cpu")
    assert gu.cum is None and np.array_equal(gu.indices.numpy(), ind)
    assert np.array_equal(gu.degree().numpy(), np.diff(ip))


@pytest.mark.parametrize("bad", [0.0, -1.0, float("nan"), float("inf")])
def test_from_edges_refuses_bad_weights(bad):
    with pytest.raises(ValueError, match="finite and > 0"):
        Graph.from_edges([0, 1], [1, 2], [1.0, bad], device="cpu")


def test_from_edges_refuses_bad_ids():
    with pytest.raises(ValueError, match=r"\[0, 3\)"):
        Graph.from_edges([0, 1], [1, 3], num_nodes=3, device="cpu")
    with pytest.raises(ValueError, match="got min -1"):
        Graph.from_edges([0, -1], [1, 2], device="cpu")
    with pytest.raises(TypeError, match="integers"):
        Graph.from_edges([0.0, 1.0], [1, 2], device="cpu")


def test_random_walks_refuses_bad_arguments():
    g = _random_graph()
    with pytest.raises(ValueError, match="starts must be in"):
        random_walks(g, [0, g.num_nodes], 5)
    with pytest.raises(ValueError, match="length"):
        random_walks(g, [0], 0)
    for bad in (0.0, -1.0, float("inf"), float("nan"), 1e-50):
        with pytest.raises(ValueError, match="finite and > 0"):
            random_walks(g, [0], 5, p=bad)
        with pytest.raises(ValueError, match="finite and > 0"):
            random_walks(g, [0], 5, q=bad)
    with pytest.raises(ValueError, match="first_walk"):
        random_walks(g, [0], 5, first_walk=-1)


def test_edge_list_reader_matches_numpy(tmp_path):
    rng = np.random.default_rng(2)
    src = rng.integers(0, 2 ** 40, 300)
    dst = rng.integers(0, 2 ** 40, 300)
    src[:3] = [2 ** 31, 2 ** 63 - 1, 0]
    w = rng.uniform(0.01, 10.0, 300)
    lines = ["# a SNAP header", "# FromNodeId\tToNodeId", ""]
    for i, (a, b, x) in enumerate(zip(src.tolist(), dst.tolist(), w.tolist())):
        lines.append(f"{a}\t{b}\t{x!r}" if i % 2 else f"  {a} {b}   {x!r} ")
        if i % 50 == 7:
            lines += ["", "   # comment after blank space", "\t"]
    path = tmp_path / "edges.txt"
    path.write_text("\n".join(lines) + "\n")
    ref = np.loadtxt(path, comments="#", dtype=str, ndmin=2)
    s, d, ww = rw.read_edge_list(str(path), weighted=True)
    assert np.array_equal(s, ref[:, 0].astype(np.int64)) and np.array_equal(d, ref[:, 1].astype(np.int64))
    assert np.array_equal(ww, ref[:, 2].astype(np.float64))
    g, labels = Graph.load(str(path), weighted=True, device="cpu")
    assert np.array_equal(labels, np.unique(np.concatenate([s, d])))
    ref_g = Graph.from_edges(np.searchsorted(labels, s), np.searchsorted(labels, d), ww, num_nodes=labels.size,
                             device="cpu")
    assert torch.equal(g.indptr, ref_g.indptr) and torch.equal(g.indices, ref_g.indices)
    assert torch.equal(g.cum, ref_g.cum)
    path2 = tmp_path / "unweighted.txt"
    path2.write_text("1 2\n# x\n3 1\n")
    s, d, ww = rw.read_edge_list(str(path2))
    assert s.tolist() == [1, 3] and d.tolist() == [2, 1] and ww is None


@pytest.mark.parametrize("text,line,weighted", [
    ("1 2\n3 4\n\n5 x\n", 4, False),
    ("# c\n1 2 3\n", 2, False),
    ("1 2\n-1 3\n", 2, False),
    ("1 9223372036854775808\n", 1, False),
    ("1 2 1.5\n2 3\n", 2, True),
    ("1 2 0\n", 1, True),
    ("1 2 0.5\n3 4 nan\n", 2, True),
])
def test_edge_list_reader_names_the_malformed_line(tmp_path, text, line, weighted):
    path = tmp_path / "bad.txt"
    path.write_text(text)
    with pytest.raises(ValueError, match=f"line {line}:"):
        Graph.load(str(path), weighted=weighted, device="cpu")
    with pytest.raises(OSError, match="cannot open"):
        Graph.load(str(tmp_path / "missing.txt"), device="cpu")


def test_app_arguments_and_no_gpu(monkeypatch, capsys):
    from multiverso_b200.apps import graph_embedding as app
    opt, g = app.parse_args([])
    assert (opt.embeding_size, opt.window_size, opt.negative_num, opt.cbow, opt.hs) == (128, 10, 5, False, False)
    assert g == dict(graph=None, directed=False, weighted=False, walk_length=80, walks_per_node=10, p=1.0, q=1.0,
                     seed=1)
    opt, g = app.parse_args("-graph e.txt -directed 1 -weighted 1 -walk_length 40 -walks_per_node 3 -p 0.25 -q 4 "
                            "-size 64 -window 5 -negative 7 -alpha 0.05 -epoch 2 -output v.txt -binary 1 -seed 9 "
                            "-cbow 1 -hs 1 -is_pipeline 0".split())
    assert g == dict(graph="e.txt", directed=True, weighted=True, walk_length=40, walks_per_node=3, p=0.25, q=4.0,
                     seed=9)
    assert (opt.embeding_size, opt.window_size, opt.negative_num, opt.init_learning_rate, opt.epoch) == \
        (64, 5, 7, 0.05, 2)
    assert opt.output_file == "v.txt" and opt.output_binary and opt.cbow and opt.hs and not opt.is_pipeline
    assert app.run([]) == {} and "usage" in capsys.readouterr().out
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(SystemExit, match="needs a CUDA GPU"):
        app.run(["-graph", "e.txt"])
