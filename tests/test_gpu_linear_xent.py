"""The fused dense linear cross-entropy (`ops.fused.linear_cross_entropy`,
`kernels/linear_xent.cu`) against fp64 on the same bf16 operands, at the shapes
`tools/bench_linear_xent.py` measures and at edge shapes; chunking, reproducibility, CUDA-graph
replay, the scratch bound, the no-gradient path, the gate, and the NMT and skip-thoughts
training steps that now run through it.

Bounds against fp64: nll max abs error 2e-3 (fp32 logits of bf16 operands); loss 1e-4 relative
to Σ|w_i · nll_i| (the row weights may be negative, so the plain sum can cancel); dX, dW and db
1e-2 relative Frobenius error (the softmax gradient G is rounded to bf16)."""
import numpy as np
import pytest
import torch

from parallax_b200 import consts
from parallax_b200 import nn as pnn

pytestmark = pytest.mark.gpu

BENCH_SHAPES = [(6400, 512, 7709, None), (6400, 1024, 36548, None),
                (3968, 2400, 20000, torch.bfloat16), (1216, 1024, 30522, torch.bfloat16)]
EDGE_SHAPES = [(N, K, V, (None, torch.bfloat16, torch.float32)[i % 3])
               for i, (N, K, V) in enumerate((N, K, V) for N in (1, 127, 129)
                                             for V in (1, 7, 129) for K in (8, 72, 520, 4096))]


def _fused():
    from parallax_b200.ops import fused
    return fused


def _case(N, K, V, bias_dt, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = (torch.randn(N, K, device="cuda", generator=g) * 0.5).bfloat16()
    w = (torch.randn(V, K, device="cuda", generator=g) / K ** 0.5).bfloat16()
    b = None if bias_dt is None else torch.randn(V, device="cuda", generator=g).to(bias_dt)
    t = torch.randint(0, V, (N,), device="cuda", generator=g)
    t[0] = 0
    t[-1] = V - 1
    rw = torch.rand(N, device="cuda", generator=g) * 2 - 0.5    # negatives too
    rw[::5] = 0.0
    return x, w, b, t, rw


def _fp64(x, w, b, t, rw):
    x64, w64 = x.double().requires_grad_(True), w.double().requires_grad_(True)
    b64 = None if b is None else b.double().requires_grad_(True)
    s = x64 @ w64.t() + (0 if b64 is None else b64)
    nll = torch.nn.functional.cross_entropy(s, t, reduction="none")
    loss = (nll * rw.double()).sum()
    loss.backward()
    return (nll.detach(), loss.detach(), (nll * rw.double()).abs().sum().detach(), x64.grad,
            w64.grad, None if b64 is None else b64.grad)


def _run(x, w, b, t, rw, chunk=None):
    xs = x.clone().requires_grad_(True)
    ws = w.clone().requires_grad_(True)
    bs = None if b is None else b.clone().requires_grad_(True)
    fused = _fused()
    assert fused.linear_xent_applies(xs, ws, bs)
    loss, nll = fused.linear_cross_entropy(xs, t, ws, bs, rw, chunk=chunk)
    loss.backward()
    return nll.detach(), loss.detach(), xs.grad, ws.grad, None if bs is None else bs.grad


def _rel(a, ref):
    return float((a.double() - ref).norm() / max(float(ref.norm()), 1e-30)) \
        if float(ref.norm()) > 0 else float(a.double().norm())


def _check(got, ref):
    nll, loss, dx, dw, db = got
    r_nll, r_loss, r_abs, r_dx, r_dw, r_db = ref
    assert float((nll.double() - r_nll).abs().max()) <= 2e-3
    assert abs(float(loss) - float(r_loss)) <= 1e-4 * max(float(r_abs), 1e-30)
    assert _rel(dx, r_dx) <= 1e-2 and _rel(dw, r_dw) <= 1e-2
    if r_db is not None:
        assert _rel(db, r_db) <= 1e-2
    assert dx.dtype == torch.bfloat16 and dw.dtype == torch.bfloat16


@pytest.mark.parametrize("N,K,V,bias_dt", BENCH_SHAPES + EDGE_SHAPES)
def test_against_fp64(N, K, V, bias_dt):
    x, w, b, t, rw = _case(N, K, V, bias_dt)
    _check(_run(x, w, b, t, rw), _fp64(x, w, b, t, rw))


def test_forced_small_chunk_with_ragged_last_chunk():
    x, w, b, t, rw = _case(1000, 520, 3001, torch.float32, seed=3)
    ref = _fp64(x, w, b, t, rw)
    small = _run(x, w, b, t, rw, chunk=384)          # 384 + 384 + 232 rows
    whole = _run(x, w, b, t, rw)
    _check(small, ref)
    _check(whole, ref)
    assert torch.equal(small[0], whole[0])             # a row's logits do not depend on its chunk
    for a, c in zip(small[1:], whole[1:]):
        assert _rel(a, c.double()) <= 1e-2


def test_two_calls_are_bitwise_equal():
    x, w, b, t, rw = _case(3968, 2400, 20000, torch.bfloat16, seed=5)
    a, c = _run(x, w, b, t, rw), _run(x, w, b, t, rw)
    for u, v in zip(a, c):
        assert torch.equal(u, v)


def test_cuda_graph_replay_equals_eager():
    fused = _fused()
    x, w, b, t, rw = _case(1216, 1024, 30522, torch.bfloat16, seed=7)
    eager = _run(x, w, b, t, rw)
    sx = x.clone().requires_grad_(True)
    sw = w.clone().requires_grad_(True)
    sb = b.clone().requires_grad_(True)
    st_, srw = t.clone(), rw.clone()

    def step():
        for p in (sx, sw, sb):
            p.grad = None
        loss, nll = fused.linear_cross_entropy(sx, st_, sw, sb, srw)
        loss.backward()
        return nll, loss, sx.grad, sw.grad, sb.grad
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = step()
    with torch.no_grad():
        sx.copy_(torch.randn_like(sx))
    graph.replay()
    with torch.no_grad():
        sx.copy_(x)
    graph.replay()
    torch.cuda.synchronize()
    for a, c in zip(static, eager):
        assert torch.equal(a, c)


@pytest.mark.parametrize("N,K,V,bias_dt", BENCH_SHAPES)
def test_peak_allocation_is_bounded(N, K, V, bias_dt):
    fused = _fused()
    x, w, b, t, rw = _case(N, K, V, bias_dt)
    xs, ws = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    bs = None if b is None else b.clone().requires_grad_(True)
    fused.linear_cross_entropy(xs, t, ws, bs, rw)[0].backward()      # cuBLAS workspaces
    xs.grad = ws.grad = None
    if bs is not None:
        bs.grad = None
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fused.linear_cross_entropy(xs, t, ws, bs, rw)[0].backward()
    torch.cuda.synchronize()
    grown = torch.cuda.max_memory_allocated() - base
    vp = (V + 7) // 8 * 8
    n = fused.linear_xent_chunk_rows(N, V)
    nvt = (V + 255) // 256
    scratch = max(consts.LINEAR_XENT_WS_BYTES, 128 * vp * 6)
    # + dX (bf16), fp32 dW, the partials, and the returned bf16 dW / db and per-row vectors
    bound = scratch + N * K * 2 + V * K * 4 + n * nvt * 8 + V * K * 2 + 8 * V + 16 * N + (1 << 20)
    logits_fp32 = N * V * 4
    print("peak growth %.1f MB, bound %.1f MB, fp32 logits %.1f MB"
          % (grown / 2**20, bound / 2**20, logits_fp32 / 2**20))
    assert grown <= bound


def test_no_grad_allocates_no_gradient_and_runs_no_cublas(monkeypatch):
    fused = _fused()
    N, K, V = 1216, 1024, 30522
    x, w, b, t, rw = _case(N, K, V, torch.bfloat16)
    ref = _run(x, w, b, t, rw)
    calls = {"n": 0}
    for name in ("mm", "addmm", "matmul"):
        real = getattr(torch, name)

        def spy(*a, _real=real, **k):
            calls["n"] += 1
            return _real(*a, **k)
        monkeypatch.setattr(torch, name, spy)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    with torch.no_grad():
        loss, nll = pnn.linear_cross_entropy(x.requires_grad_(True), t, w, b, row_weights=rw)
    torch.cuda.synchronize()
    grown = torch.cuda.max_memory_allocated() - base
    n, vp = fused.linear_xent_chunk_rows(N, V), (V + 7) // 8 * 8
    assert calls["n"] == 0
    assert grown < n * vp * 4 + n * vp * 2           # fp32 logits, but no bf16 G
    assert torch.equal(nll, ref[0]) and torch.equal(loss, ref[1])


def test_gate_refuses_and_the_composition_runs(monkeypatch):
    fused = _fused()
    x, w, b, t, rw = _case(64, 72, 129, None)
    big = torch.empty(129 * 72 + 8, dtype=torch.bfloat16, device="cuda")
    w_off = big[1:1 + 129 * 72].view(129, 72)                       # 2-byte offset
    w_off.copy_(w)
    cases = [(x.float(), w.float()), (x, w_off), (x[:, :70].contiguous(), w[:, :70].contiguous())]
    calls = {"n": 0}
    real = fused.linear_cross_entropy

    def spy(*a, **k):
        calls["n"] += 1
        return real(*a, **k)
    monkeypatch.setattr(fused, "linear_cross_entropy", spy)
    for xi, wi in cases:
        assert not fused.linear_xent_applies(xi, wi, None)
        loss, nll = pnn.linear_cross_entropy(xi, t, wi, None, row_weights=rw)
        ref, ref_nll = fused.linear_cross_entropy_reference(xi, t, wi, None, rw)
        assert torch.equal(loss, ref) and torch.equal(nll, ref_nll)
    assert calls["n"] == 0
    pnn.linear_cross_entropy(x, t, w, None, row_weights=rw)
    assert calls["n"] == 1


# ===========================================================================
# the models on the NVLink fabric
# ===========================================================================
def _spy_or_compose(mp, composition, calls):
    fused = _fused()
    if composition:
        mp.setattr(fused, "linear_xent_applies", lambda *a, **k: False)
    else:
        real = fused.linear_cross_entropy

        def spy(*a, **k):
            calls["n"] += 1
            return real(*a, **k)
        mp.setattr(fused, "linear_cross_entropy", spy)


def _nmt_losses(option, arch, composition, monkeypatch, steps=6):
    import parallax_b200 as parallax
    import parallax_b200.models.nmt as nmt
    calls = {"n": 0}
    with monkeypatch.context() as mp:
        _spy_or_compose(mp, composition, calls)
        torch.manual_seed(0)
        hp = nmt.create_hparams(num_units=32, num_layers=2 if arch == "standard" else 3,
                                encoder_type="bi" if arch == "standard" else "gnmt",
                                attention=option, attention_architecture=arch, residual=True,
                                dropout=0.0, num_embeddings_partitions=2, learning_rate=0.5)
        nmt.extend_hparams(hp, 40, 40)
        m = nmt.create_model(hp)
        sess, *_ = parallax.parallel_run(
            nmt.nmt_graph(m, hp), "localhost:0",
            parallax_config=parallax.Config(search_partitions=False, sess_config={
                "fabric": "nvlink", "compute_dtype": "bf16"}))
        g = torch.Generator().manual_seed(1)
        B, S, T = 8, 7, 6
        feed = {"source": [torch.randint(3, 40, (B, S), generator=g)],
                "target_input": [torch.randint(3, 40, (B, T), generator=g)],
                "target_output": [torch.randint(3, 40, (B, T), generator=g)],
                "source_sequence_length": [torch.tensor([7, 5, 3, 6, 7, 2, 4, 7])],
                "target_sequence_length": [torch.tensor([6, 4, 6, 2, 5, 6, 3, 6])]}
        losses = [sess.run(["loss", "train_op"], feed)[0][0] for _ in range(steps)]
        sess.close()
    return np.array(losses, dtype=np.float64), calls["n"]


@pytest.mark.parametrize("option,arch", [("scaled_luong", "standard"),
                                         ("normed_bahdanau", "gnmt_v2")])
def test_nmt_trains_on_the_fused_head(option, arch, monkeypatch):
    fused_l, n_calls = _nmt_losses(option, arch, False, monkeypatch)
    comp_l, c_calls = _nmt_losses(option, arch, True, monkeypatch)
    print("losses fused", fused_l, "composition", comp_l)
    assert n_calls >= 6 and c_calls == 0
    assert np.isfinite(fused_l).all() and fused_l[-1] < fused_l[0]
    np.testing.assert_allclose(fused_l, comp_l, rtol=5e-2)


def _skip_thoughts_losses(bidirectional, composition, monkeypatch, steps=6):
    import parallax_b200 as parallax
    from parallax_b200.models import skip_thoughts as st
    from parallax_b200.models.skip_thoughts.input_ops import parse_example_batch
    calls = {"n": 0}
    with monkeypatch.context() as mp:
        _spy_or_compose(mp, composition, calls)
        torch.manual_seed(0)
        mc = st.model_config(vocab_size=48, word_embedding_dim=16, encoder_dim=32, batch_size=4,
                             num_embedding_partitions=2, bidirectional_encoder=bidirectional)
        tc = st.training_config(learning_rate=0.01)
        model = st.SkipThoughtsModel(mc)
        sess, *_ = parallax.parallel_run(
            st.skip_thoughts_graph(model, tc), "localhost:0",
            parallax_config=parallax.Config(search_partitions=False, sess_config={
                "fabric": "nvlink", "compute_dtype": "bf16"}))
        batch = parse_example_batch([([3, 4, 5, 0], [6, 7, 0], [8, 0]),
                                     ([9, 0], [3, 0], [4, 5, 6, 0]),
                                     ([10, 11, 0], [12, 0], [13, 14, 0]),
                                     ([5, 0], [6, 0], [7, 0])])
        losses = [sess.run(["loss", "train_op"], st.feed_from_batch(batch))[0][0]
                  for _ in range(steps)]
        sess.close()
    return np.array(losses, dtype=np.float64), calls["n"]


@pytest.mark.parametrize("bidirectional", [False, True])
def test_skip_thoughts_trains_on_the_fused_head(bidirectional, monkeypatch):
    fused_l, n_calls = _skip_thoughts_losses(bidirectional, False, monkeypatch)
    comp_l, c_calls = _skip_thoughts_losses(bidirectional, True, monkeypatch)
    print("losses fused", fused_l, "composition", comp_l)
    assert n_calls >= 6 * 2 and c_calls == 0          # both decoders of every step
    assert np.isfinite(fused_l).all() and fused_l[-1] < fused_l[0]
    np.testing.assert_allclose(fused_l, comp_l, rtol=5e-2)
