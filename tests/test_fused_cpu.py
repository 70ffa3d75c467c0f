"""Host-side checks of the fused model nodes' algebra (their CUDA kernels are emulated by the
PyTorch fall-backs inside the nodes; the kernels themselves are checked on the device in
`tests/test_gpu_fused.py`)."""
import pytest
import torch


@pytest.mark.parametrize("weighted", [False, True])
def test_sampled_softmax_head_node_matches_autograd_of_the_reference(weighted):
    from parallax_b200.ops.fused import (_SampledSoftmaxHeadFn, sampled_softmax_head,
                                         sampled_softmax_reference)
    torch.manual_seed(0)
    N, S, P, V = 24, 40, 16, 200
    inputs = torch.randn(N, P, requires_grad=True)
    w_all = torch.randn(N + S, P, requires_grad=True)
    b_all = torch.randn(N + S, 1, requires_grad=True)
    logq = torch.randn(N + S)
    targets = torch.randint(0, V, (N,))
    sampled = torch.randperm(V)[:S]
    sampled[:3] = targets[:3]                       # accidental hits
    rw = torch.rand(N) if weighted else None
    adj = b_all.detach().reshape(-1) - logq
    out = _SampledSoftmaxHeadFn.apply(inputs, w_all, b_all, adj, targets, sampled, rw)
    (out * 3.0).backward()
    got = [t.grad.clone() for t in (inputs, w_all, b_all)]
    for t in (inputs, w_all, b_all):
        t.grad = None
    b = b_all.reshape(-1)
    ref = sampled_softmax_reference(inputs, w_all[:N], w_all[N:], b[:N], b[N:], logq[:N],
                                    logq[N:], targets, sampled)
    ref = (ref * rw if weighted else ref).mean()
    (ref * 3.0).backward()
    assert torch.allclose(out, ref, atol=1e-5)
    for a, t in zip(got, (inputs, w_all, b_all)):
        assert a.shape == t.grad.shape
        assert torch.allclose(a, t.grad, atol=1e-5)
    # the public wrapper on the host is the reference composition
    o2 = sampled_softmax_head(inputs, w_all, b_all, logq, targets, sampled, row_w=rw, adj=adj)
    assert torch.allclose(o2, ref, atol=1e-6)


def test_lstm_layer_reference_gradcheck_fp64():
    """The LSTM oracle every device test trusts: its autograd agrees with finite differences,
    which needs it to stay in fp64 end to end when given fp64."""
    from parallax_b200.ops.fused import lstm_layer_reference
    torch.manual_seed(0)
    T, B, E, S, P = 3, 2, 3, 4, 2
    mk = lambda *s: (torch.randn(*s, dtype=torch.float64) * 0.5).requires_grad_(True)
    args = (mk(T, B, E), mk(E, 4 * S), mk(P, 4 * S), mk(4 * S), mk(S, P), mk(B, S), mk(B, P))

    def f(*a):
        H, c, h = lstm_layer_reference(*a, forget_bias=0.7)
        assert H.dtype == c.dtype == h.dtype == torch.float64
        return H, c, h
    assert torch.autograd.gradcheck(f, args)


def test_sampled_softmax_reference_gradcheck_fp64_with_masked_hit():
    from parallax_b200.ops.fused import sampled_softmax_reference
    torch.manual_seed(1)
    N, S, P = 4, 6, 3
    mk = lambda *s: torch.randn(*s, dtype=torch.float64).requires_grad_(True)
    targets = torch.tensor([3, 7, 1, 9])
    sampled = torch.tensor([2, 7, 5, 3, 8, 0])          # rows 0 and 1 each have a hit
    lqt, lqs = torch.randn(N, dtype=torch.float64), torch.randn(S, dtype=torch.float64)
    args = (mk(N, P), mk(N, P), mk(S, P), mk(N), mk(S))

    def f(*a):
        out = sampled_softmax_reference(*a, lqt, lqs, targets, sampled)
        assert out.dtype == torch.float64
        return out
    assert torch.autograd.gradcheck(f, args)
    # the masked logit takes no part: moving the hit column's bias changes nothing in its row
    a = [t.detach() for t in args]
    base = f(*a)
    b2 = a[4].clone()
    b2[1] += 5.0
    moved = sampled_softmax_reference(a[0], a[1], a[2], a[3], b2, lqt, lqs, targets, sampled)
    assert moved[1] == base[1]
    assert moved[0] != base[0]


def test_lm1b_time_major_rows_give_the_batch_major_loss(monkeypatch):
    """The model orders its rows (t, b); the loss is the mean over all rows, so it must equal
    the batch-major formulation of `examples/lm1b/language_model.py:88-107`."""
    from parallax_b200.models import lm1b as L
    from parallax_b200.ops.fused import lstm_layer_reference, sampled_softmax_reference
    torch.manual_seed(3)
    B, T, V, E, S_, P = 6, 5, 300, 16, 32, 16
    m = L.LM1B(vocab_size=V, emb_size=E, state_size=S_, projected_size=P, num_sampled=24,
               num_steps=T, num_shards=1, keep_prob=1.0)
    x, y = torch.randint(0, V, (B, T)), torch.randint(0, V, (B, T))
    w = torch.rand(B, T)
    fixed = (torch.randperm(V)[:24], torch.tensor(30.0))
    monkeypatch.setattr(L, "log_uniform_sample_unique", lambda *a, **k: fixed)
    out = m(x, y, w)
    H, c, h = lstm_layer_reference(m.emb(x).transpose(0, 1), m.W[:E], m.W[E:], m.B, m.W_P,
                                   torch.zeros(B, S_), torch.zeros(B, P), 1.0)
    inputs = H.transpose(0, 1).reshape(B * T, -1)
    targets = y.reshape(-1)
    ids = torch.cat([targets, fixed[0]])
    wa, ba = m.softmax_w(ids), m.softmax_b(ids).squeeze(-1)
    lq = L.log_uniform_logq_unique(ids, fixed[1], V)
    N = B * T
    ref = (sampled_softmax_reference(inputs, wa[:N], wa[N:], ba[:N], ba[N:], lq[:N], lq[N:],
                                     targets, fixed[0]) * w.reshape(-1)).mean()
    assert abs(float(ref) - float(out["loss"])) < 1e-5
    assert torch.allclose(out["final_state_c"], c.detach(), atol=1e-6)
    assert torch.allclose(out["final_state_h"], h.detach(), atol=1e-6)
