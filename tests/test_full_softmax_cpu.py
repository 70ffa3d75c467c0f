"""`parallax.nn.full_softmax_nll` on the host fabric: the gather + matmul + cross_entropy
composition, bit for bit what `LM1B.full_softmax_loss` computed before the op existed, plus
the op's argument checks."""
import pytest
import torch
import torch.nn.functional as F

import parallax_b200 as parallax
from parallax_b200.models.lm1b import LM1B, lm1b_graph


def _composition(inputs, targets, weight, bias, V):
    # the pre-op body of LM1B.full_softmax_loss, kept here as the oracle
    ids = torch.arange(V, device=inputs.device)
    w, b = parallax.nn.lookup_many([weight, bias], ids)
    w, b = w.to(inputs.dtype), b.squeeze(-1).float()
    logits = (inputs @ w.t()).float() + b
    return F.cross_entropy(logits, targets, reduction="none")


@pytest.fixture(scope="module")
def host_lm1b():
    torch.manual_seed(0)
    V = 301
    m = LM1B(vocab_size=V, emb_size=16, state_size=32, projected_size=16, num_sampled=0,
             num_steps=4, num_shards=3, keep_prob=1.0)
    sess, *_ = parallax.parallel_run(lm1b_graph(m, batch_size=8), "localhost",
                                     parallax_config=parallax.Config(
                                         sess_config={"fabric": "host"}))
    gen = torch.Generator().manual_seed(1)
    x = torch.randint(0, V, (8, 4), generator=gen)
    for _ in range(2):                   # move the tables away from their initial values
        sess.run(["loss", "train_op"], {"x": [x], "y": [torch.roll(x, -1, dims=1)]})
    yield sess, sess.engine.model, V
    sess.close()


@pytest.mark.parametrize("grad", [False, True])
def test_host_fabric_matches_composition_bitwise(host_lm1b, grad):
    sess, m, V = host_lm1b
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


def test_eval_loss_through_session_is_finite(host_lm1b):
    sess, m, V = host_lm1b
    m.eval()
    try:
        x = torch.randint(0, V, (8, 4), generator=torch.Generator().manual_seed(3))
        loss = sess.run("loss", {"x": [x], "y": [torch.roll(x, -1, dims=1)]})[0]
    finally:
        m.train()
    assert loss == loss and 0.0 < float(loss) < 3 * torch.log(torch.tensor(float(V)))


def test_argument_validation(host_lm1b):
    sess, m, V = host_lm1b
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
