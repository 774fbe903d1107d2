"""Embedding bags without a GPU: the host reference against torch, PSEmbedding on the host backend (forward, the
coalesced push, the backward that runs when only ids go in) and the input checks."""
import pytest
import torch
import torch.nn.functional as F

from multiverso_b200.ops import PSEmbedding, embedding_bag, embedding_bag_reference


@pytest.fixture
def mv_host():
    if torch.cuda.is_available():
        pytest.skip("host-backend test (runs where there is no GPU)")
    import multiverso_b200 as mv
    mv.FLAGS.reset()
    mv.init()
    yield mv
    mv.shutdown(finalize_net=False)
    mv.FLAGS.reset()


def _case(V=50, D=8, seed=0):
    g = torch.Generator().manual_seed(seed)
    W = torch.randn(V, D, generator=g)
    ids = torch.randint(0, V, (40,), generator=g)
    ids[5:15] = 7                                              # duplicates
    offsets = torch.tensor([0, 0, 3, 4, 4, 20, 39])            # empty bags, length-1 bags, a long bag
    psw = torch.rand(40, generator=g)
    return W, ids, offsets, psw


@pytest.mark.parametrize("mode", ["sum", "mean"])
@pytest.mark.parametrize("idtype", [torch.int32, torch.int64])
def test_reference_equals_torch(mode, idtype):
    W, ids, offsets, psw = _case()
    ref = embedding_bag_reference(W, ids.to(idtype), offsets.to(idtype), mode=mode)
    exp = F.embedding_bag(ids, W, offsets, mode=mode)
    assert torch.allclose(ref, exp, atol=1e-6)
    assert (ref[0] == 0).all() and (ref[3] == 0).all()
    assert torch.allclose(ref[2], W[ids[3]])


def test_reference_weights_and_2d():
    W, ids, offsets, psw = _case()
    ref = embedding_bag_reference(W, ids, offsets, per_sample_weights=psw)
    assert torch.allclose(ref, F.embedding_bag(ids, W, offsets, mode="sum", per_sample_weights=psw), atol=1e-6)
    ids2 = ids[:36].view(6, 6).to(torch.int32)
    for mode in ("sum", "mean"):
        assert torch.allclose(embedding_bag_reference(W, ids2, mode=mode),
                              F.embedding_bag(ids2.long(), W, mode=mode), atol=1e-6)
    p2 = psw[:36].view(6, 6)
    assert torch.allclose(embedding_bag_reference(W, ids2, per_sample_weights=p2),
                          F.embedding_bag(ids2.long(), W, mode="sum", per_sample_weights=p2), atol=1e-6)
    assert torch.allclose(embedding_bag(W, ids2, mode="mean"), F.embedding_bag(ids2.long(), W, mode="mean"))


def _host_table(mv, W):
    t = mv.MatrixTable(W.shape[0], W.shape[1], "float32")
    t.add(W.numpy())
    return t


@pytest.mark.parametrize("mode", ["sum", "mean"])
def test_ps_embedding_host_step_equals_embeddingbag_sgd(mv_host, mode):
    W, ids, offsets, psw = _case()
    lr = 0.1
    t = _host_table(mv_host, W)
    layer = PSEmbedding(t, push_scale=-lr, mode=mode)          # default updater adds: push -lr * grad
    target = torch.randn(offsets.numel(), W.shape[1])
    weights = psw if mode == "sum" else None
    y = layer(ids, offsets, weights)
    assert torch.allclose(y, embedding_bag_reference(W, ids, offsets, weights, mode), atol=1e-6)
    ((y - target) ** 2).sum().backward()
    ref = torch.nn.EmbeddingBag(W.shape[0], W.shape[1], mode=mode, sparse=True)
    with torch.no_grad():
        ref.weight.copy_(W)
    opt = torch.optim.SGD(ref.parameters(), lr=lr)
    ((ref(ids, offsets, per_sample_weights=weights) - target) ** 2).sum().backward()
    opt.step()
    got = torch.from_numpy(t.get())
    assert torch.allclose(got, ref.weight.detach(), atol=1e-5)
    untouched = torch.ones(W.shape[0], dtype=torch.bool)
    untouched[ids] = False
    assert torch.equal(got[untouched], W[untouched])


def test_ps_embedding_backward_runs_on_ids_alone(mv_host):
    """Nothing but ids goes in: the anchor parameter still makes autograd run the backward, which pushes."""
    W, ids, offsets, _ = _case()
    t = _host_table(mv_host, W)
    layer = PSEmbedding(t, push_scale=1.0)
    assert not ids.requires_grad
    layer(ids, offsets).sum().backward()
    counts = torch.bincount(ids, minlength=W.shape[0]).float()
    assert torch.allclose(torch.from_numpy(t.get()), W + counts[:, None], atol=1e-6)
    assert layer.anchor.grad is not None and layer.anchor.grad.numel() == 0


def test_psw_grad_host(mv_host):
    W, ids, offsets, psw = _case()
    t = _host_table(mv_host, W)
    p = psw.clone().requires_grad_()
    dout = torch.randn(offsets.numel(), W.shape[1])
    (PSEmbedding(t, push_scale=None)(ids, offsets, p) * dout).sum().backward()
    p2 = psw.clone().requires_grad_()
    (F.embedding_bag(ids, W, offsets, mode="sum", per_sample_weights=p2) * dout).sum().backward()
    assert torch.allclose(p.grad, p2.grad, atol=1e-5)
    assert torch.equal(torch.from_numpy(t.get()), W)           # push_scale=None: nothing pushed


def test_validation_errors(mv_host):
    W, ids, offsets, psw = _case()
    t = _host_table(mv_host, W)
    bad = [
        (dict(ids=torch.tensor([0, 50]), offsets=torch.tensor([0])), ValueError, r"ids must be in \[0, 50\)"),
        (dict(ids=torch.tensor([-1, 3]), offsets=torch.tensor([0])), ValueError, r"ids must be in \[0, 50\)"),
        (dict(ids=ids, offsets=offsets.float()), TypeError, "offsets must be a 1-D int32 or int64"),
        (dict(ids=ids, offsets=torch.tensor([1, 5])), ValueError, "offsets must start at 0"),
        (dict(ids=ids, offsets=torch.tensor([0, 5, 3])), ValueError, "offsets must be non-decreasing"),
        (dict(ids=ids, offsets=torch.tensor([0, 41])), ValueError, "offsets exceed the number of ids"),
        (dict(ids=ids, offsets=offsets, per_sample_weights=psw, mode="mean"), ValueError,
         "per_sample_weights are only supported with mode='sum'"),
        (dict(ids=ids, offsets=offsets, per_sample_weights=psw[:10]), ValueError,
         "per_sample_weights must have the shape of ids"),
        (dict(ids=ids.float(), offsets=offsets), TypeError, "ids must be int32 or int64"),
        (dict(ids=ids, offsets=offsets, mode="max"), ValueError, "mode must be one of"),
        (dict(ids=ids.view(4, 10), offsets=offsets), ValueError, "offsets must be None when ids is 2-D"),
    ]
    for kw, exc, msg in bad:
        with pytest.raises(exc, match=msg):
            embedding_bag(t, **kw)
    t64 = mv_host.MatrixTable(10, 4, "float64")
    with pytest.raises(TypeError, match="the table must be float32"):
        embedding_bag(t64, torch.tensor([1]), torch.tensor([0]))
    with pytest.raises(TypeError, match="the table must be float32"):
        PSEmbedding(t64)(torch.tensor([1]), torch.tensor([0]))
    with pytest.raises(TypeError, match="must be a MatrixTable"):
        PSEmbedding(W)
