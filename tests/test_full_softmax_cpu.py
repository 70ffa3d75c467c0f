"""`parallax.nn.full_softmax_nll` and `parallax.nn.full_softmax_topk` without a GPU: the gather +
matmul compositions on the host fabric — the NLL bit for bit what `LM1B.full_softmax_loss`
computed before the op existed, the top-k against an fp64 oracle with its tie order — plus the
ops' argument checks and LM1B's `eval_top_k` outputs."""
import pytest
import torch
import torch.nn.functional as F

import parallax_b200 as parallax
import parallax_b200.nn as pnn
from parallax_b200.models.lm1b import LM1B, lm1b_graph

V = 301


def _batch(seed):
    x = torch.randint(0, V, (8, 4), generator=torch.Generator().manual_seed(seed))
    return {"x": [x], "y": [torch.roll(x, -1, dims=1)]}


def _session(eval_top_k=0, train=()):
    """A host-fabric LM1B session, trained on the batches `train` (to move the tables away from
    their initial values)."""
    torch.manual_seed(0)
    m = LM1B(vocab_size=V, emb_size=16, state_size=32, projected_size=16, num_sampled=0,
             num_steps=4, num_shards=3, keep_prob=1.0, eval_top_k=eval_top_k)
    sess, *_ = parallax.parallel_run(lm1b_graph(m, batch_size=8), "localhost",
                                     parallax_config=parallax.Config(
                                         sess_config={"fabric": "host"}))
    for feeds in train:
        sess.run(["loss", "train_op"], feeds)
    return sess, m


@pytest.fixture(scope="module")
def nll_lm1b():
    sess, m = _session(train=[_batch(1)] * 2)
    yield sess, m
    sess.close()


@pytest.fixture(scope="module")
def topk_lm1b():
    sess, m = _session(train=[_batch(0), _batch(1)])
    yield sess, m
    sess.close()


# ------------------------------------------------------------------ NLL
def _composition(inputs, targets, weight, bias, V):
    # the pre-op body of LM1B.full_softmax_loss, kept here as the oracle
    ids = torch.arange(V, device=inputs.device)
    w, b = parallax.nn.lookup_many([weight, bias], ids)
    w, b = w.to(inputs.dtype), b.squeeze(-1).float()
    logits = (inputs @ w.t()).float() + b
    return F.cross_entropy(logits, targets, reduction="none")


@pytest.mark.parametrize("grad", [False, True])
def test_host_fabric_matches_composition_bitwise(nll_lm1b, grad):
    sess, m = nll_lm1b
    gen = torch.Generator().manual_seed(2)
    inputs = torch.randn(37, 16, generator=gen, requires_grad=grad)
    targets = torch.randint(0, V, (37,), generator=gen)
    targets[0], targets[1] = 0, V - 1
    with torch.set_grad_enabled(grad):
        ref = _composition(inputs, targets, m.softmax_w, m.softmax_b, V)
        op = parallax.nn.full_softmax_nll(inputs, targets, m.softmax_w, m.softmax_b)
        via_model = m.full_softmax_loss(inputs, targets)
    assert op.shape == (37,) and op.dtype == torch.float32
    assert torch.equal(op, ref) and torch.equal(via_model, ref)
    if grad:
        op.sum().backward()             # the composition carries gradients to the inputs
        assert inputs.grad is not None and torch.isfinite(inputs.grad).all()


def test_eval_loss_through_session_is_finite(nll_lm1b):
    sess, m = nll_lm1b
    m.eval()
    try:
        x = torch.randint(0, V, (8, 4), generator=torch.Generator().manual_seed(3))
        loss = sess.run("loss", {"x": [x], "y": [torch.roll(x, -1, dims=1)]})[0]
    finally:
        m.train()
    assert loss == loss and 0.0 < float(loss) < 3 * torch.log(torch.tensor(float(V)))


def test_argument_validation(nll_lm1b):
    sess, m = nll_lm1b
    x, t = torch.randn(5, 16), torch.randint(0, V, (5,))
    fs = parallax.nn.full_softmax_nll
    with pytest.raises(ValueError, match="inputs must be"):
        fs(x.reshape(5, 4, 4), t, m.softmax_w, m.softmax_b)
    with pytest.raises(ValueError, match="targets must be \\[N\\]"):
        fs(x, t[:4], m.softmax_w, m.softmax_b)
    with pytest.raises(ValueError, match="targets must be \\[N\\]"):
        fs(x, t.reshape(5, 1), m.softmax_w, m.softmax_b)
    with pytest.raises(ValueError, match="integer ids"):
        fs(x, t.float(), m.softmax_w, m.softmax_b)
    with pytest.raises(ValueError, match="columns"):
        fs(torch.randn(5, 8), t, m.softmax_w, m.softmax_b)
    with pytest.raises(ValueError, match="bias must be"):
        fs(x, t, m.softmax_w, m.softmax_w)
    with pytest.raises(ValueError, match="bias must be"):
        fs(x, t, m.softmax_w, parallax.nn.Embedding(V + 1, 1))


# ------------------------------------------------------------------ top-k
def _oracle(inputs, m):
    """fp64 log-probabilities of every row, and each row's ids sorted by (logit desc, id asc)."""
    ids = torch.arange(V)
    w, b = pnn.lookup_many([m.softmax_w, m.softmax_b], ids)
    lp = torch.log_softmax(inputs.double() @ w.double().t() + b.double().t(), dim=-1)
    order = torch.sort(lp, dim=1, descending=True, stable=True).indices
    return lp, order


@pytest.mark.parametrize("k", [1, 5, 32, 40, V])
def test_topk_composition_matches_fp64(topk_lm1b, k):
    sess, m = topk_lm1b
    inputs = torch.randn(37, 16, generator=torch.Generator().manual_seed(k))
    with torch.no_grad():
        lp, ids = parallax.nn.full_softmax_topk(inputs, m.softmax_w, m.softmax_b, k)
    assert lp.shape == (37, k) and lp.dtype == torch.float32
    assert ids.shape == (37, k) and ids.dtype == torch.int64
    ref_lp, order = _oracle(inputs, m)
    assert ((ids >= 0) & (ids < V)).all()
    assert all(len(set(r.tolist())) == k for r in ids)
    torch.testing.assert_close(lp.double(), ref_lp.gather(1, ids), rtol=0, atol=1e-5)
    assert (lp[:, 1:] <= lp[:, :-1]).all()
    # ids agree with the oracle's order wherever its neighbouring log-probs are apart
    ref_sorted = ref_lp.gather(1, order)
    gap = torch.ones(37, k, dtype=torch.bool)
    gap[:, :-1] = (ref_sorted[:, :k - 1] - ref_sorted[:, 1:k]) > 1e-5
    gap[:, 1:] &= (ref_sorted[:, :k - 1] - ref_sorted[:, 1:k]) > 1e-5
    if k < V:
        gap[:, -1] &= (ref_sorted[:, k - 1] - ref_sorted[:, k]) > 1e-5
    assert gap.float().mean() > 0.5
    assert torch.equal(ids[gap], order[:, :k][gap])


def test_topk_gradients_flow_into_log_probs(topk_lm1b):
    sess, m = topk_lm1b
    inputs = torch.randn(5, 16, requires_grad=True)
    lp, _ = parallax.nn.full_softmax_topk(inputs, m.softmax_w, m.softmax_b, 3)
    lp.sum().backward()
    assert inputs.grad is not None and torch.isfinite(inputs.grad).all()
    assert inputs.grad.abs().sum() > 0


@pytest.mark.parametrize("k", [1, 4, 7])
def test_topk_exact_ties_come_back_in_ascending_id_order(k):
    """Rows 5, 17, 40 and 41 of the table are one row repeated, and so are rows 3 and 90:
    equal logits, ordered by ascending id."""
    n, K = 6, 8
    g = torch.Generator().manual_seed(3)
    weight, bias = torch.nn.Embedding(64 + 32, K), torch.nn.Embedding(64 + 32, 1)
    with torch.no_grad():
        weight.weight.copy_(torch.randn(96, K, generator=g) * 0.1)
        bias.weight.zero_()
        top = torch.randn(K, generator=g) * 3
        for r in (5, 17, 40, 41):
            weight.weight[r] = top
        for r in (3, 90):
            weight.weight[r] = top * 0.9
        inputs = top.repeat(n, 1) + torch.randn(n, K, generator=g) * 1e-3
        lp, ids = parallax.nn.full_softmax_topk(inputs, weight, bias, k)
    want = [5, 17, 40, 41, 3, 90][:k]
    for r in range(n):
        assert ids[r].tolist()[:min(k, 6)] == want[:min(k, 6)]
        assert len(set(lp[r, :min(k, 4)].tolist())) == 1


def test_topk_argument_validation(topk_lm1b):
    sess, m = topk_lm1b
    x = torch.randn(5, 16)
    ft = parallax.nn.full_softmax_topk
    for k in (0, -1, V + 1, True, False, 2.0, "3", None):
        with pytest.raises(ValueError, match="k must be"):
            ft(x, m.softmax_w, m.softmax_b, k)
    with pytest.raises(ValueError, match="inputs must be"):
        ft(x.reshape(5, 4, 4), m.softmax_w, m.softmax_b, 3)
    with pytest.raises(ValueError, match="inputs must be"):
        ft(x[0], m.softmax_w, m.softmax_b, 3)
    with pytest.raises(ValueError, match="columns"):
        ft(torch.randn(5, 8), m.softmax_w, m.softmax_b, 3)
    with pytest.raises(ValueError, match="bias must be"):
        ft(x, m.softmax_w, m.softmax_w, 3)
    with pytest.raises(ValueError, match="bias must be"):
        ft(x, m.softmax_w, parallax.nn.Embedding(V + 1, 1), 3)


def _eval(sess, m, fetches, seed=9):
    m.eval()
    try:
        return sess.run(fetches, _batch(seed))
    finally:
        m.train()


def test_lm1b_eval_top_k_outputs(monkeypatch):
    seen = {}
    orig_nll, orig_topk = pnn.full_softmax_nll, pnn.full_softmax_topk

    def nll(inputs, targets, w, b):
        seen["nll"] = inputs.detach().clone()
        return orig_nll(inputs, targets, w, b)

    def topk(inputs, w, b, k):
        seen["topk"] = inputs.detach().clone()
        seen["out"] = orig_topk(inputs, w, b, k)
        return seen["out"]
    monkeypatch.setattr(pnn, "full_softmax_nll", nll)
    monkeypatch.setattr(pnn, "full_softmax_topk", topk)
    sess, m = _session(eval_top_k=3)
    sess.run(["loss", "train_op"], _batch(0))
    assert "topk" not in seen                      # training: no top-k
    loss, top = _eval(sess, m, ["loss", "top_k_ids"])
    top = torch.as_tensor(top[0])                  # the session returns numpy arrays
    assert top.shape == (8, 4, 3) and top.dtype == torch.int64
    assert torch.equal(seen["topk"], seen["nll"])  # the same LSTM outputs as the loss
    # rows of the op are time-major (t, b); the output is batch-major like x and y
    assert torch.equal(top, seen["out"][1].reshape(4, 8, 3).transpose(0, 1))
    sess.close()


def test_eval_top_k_zero_leaves_the_outputs_unchanged():
    outs = []
    for k in (0, 2):
        sess, m = _session(eval_top_k=k)
        train = sess.run(["loss", "train_op"], _batch(0))[0][0]
        m.eval()
        try:
            out = sess.engine.forward({"x": _batch(5)["x"][0], "y": _batch(5)["y"][0]})
        finally:
            m.train()
        outs.append((train, out))
        sess.close()
    (t0, o0), (t2, o2) = outs
    assert float(t0) == float(t2)
    assert set(o0) == {"loss", "final_state_c", "final_state_h"}
    assert set(o2) == set(o0) | {"top_k_ids"}
    for key in o0:
        assert torch.equal(o0[key], o2[key]), key
