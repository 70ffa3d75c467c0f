"""The fused layer-normalised GRU (`ops.fused.ln_gru_layer`, `kernels/ln_gru.cu`) against the
fp64 composition (`LayerNormGRU._composition`).

Each kernel and the whole node are held to the calibrated bound of
`test_gpu_lm1b_numerics._assert_calibrated`: against fp64, the fused error stays within 2× the
error of the same composition run in the fused path's dtype (plus a small relative floor)."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.test_gpu_lm1b_numerics import _assert_calibrated

pytestmark = pytest.mark.gpu

_vp = ctypes.c_void_p
_DT = {torch.float32: 0, torch.bfloat16: 1}


def _p(t):
    return _vp(t.data_ptr()) if t is not None else None


def _stream():
    return _vp(torch.cuda.current_stream().cuda_stream)


def _lib():
    from parallax_b200 import ops
    from parallax_b200.ops import fused  # noqa: F401  (register the signatures)
    return ops.lib()


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _lengths(B, T, seed):
    """ragged lengths in [1, T] with 1 and T both present"""
    g = torch.Generator().manual_seed(seed)
    ln = torch.randint(1, T + 1, (B,), generator=g)
    ln[0] = T
    if B > 1:
        ln[1] = 1
    return ln.cuda()


# ===========================================================================
# the cell kernels, called directly on exact operands
# ===========================================================================
def _cell64(hh, gx, cx, h, prm, live, n):
    """one step of the composition from hh = h·w_hu (any dtype; fp64 is the oracle)"""
    g_wh, b_wh, g_u, b_u = prm
    zr = torch.sigmoid(F.layer_norm(hh[:, :2 * n], (2 * n,), g_wh, b_wh, 1e-5) + gx)
    z, r = zr[:, :n], zr[:, n:]
    cand = torch.tanh(r * F.layer_norm(hh[:, 2 * n:], (n,), g_u, b_u, 1e-5) + cx)
    h2 = (1.0 - z) * h + z * cand
    return torch.where(live, h2, h), torch.where(live, h2, torch.zeros_like(h2))


def _cell_operands(B, n, dt, seed):
    g = _gen(seed)
    hh = torch.randn(B, 3 * n, device="cuda", generator=g) * 3.0 + 0.5
    gx = torch.randn(B, 2 * n, device="cuda", generator=g).to(dt)
    cx = torch.randn(B, n, device="cuda", generator=g).to(dt)
    h = (torch.rand(B, n, device="cuda", generator=g) * 2 - 1).to(dt)
    prm = [(1.0 + 0.3 * torch.randn(k, device="cuda", generator=g)).to(dt) for k in (2 * n,)] + \
        [(0.2 * torch.randn(2 * n, device="cuda", generator=g)).to(dt)] + \
        [(1.0 + 0.3 * torch.randn(n, device="cuda", generator=g)).to(dt),
         (0.2 * torch.randn(n, device="cuda", generator=g)).to(dt)]
    dout = torch.randn(B, n, device="cuda", generator=g).to(dt)
    carry = torch.randn(B, n, device="cuda", generator=g)
    drec = torch.randn(B, n, device="cuda", generator=g)
    return hh, gx, cx, h, prm, dout, carry, drec


def _run_cells(B, n, dt, t, lengths, ops):
    hh, gx, cx, h, prm, dout, carry, drec = ops
    L = _lib()
    st = _stream()
    h_next = torch.empty(B, n, dtype=dt, device="cuda")
    out = torch.empty(B, n, dtype=dt, device="cuda")
    stats = torch.empty(B, 4, device="cuda")
    rc = L.px_ln_gru_fwd(_p(hh), _p(gx), 2 * n, _p(cx), n, _p(h), _p(h_next), _p(out), n,
                         _p(stats), *[_p(q) for q in prm], _p(lengths), t, B, n, 1e-5, 1e-5,
                         _DT[dt], st)
    assert rc == 0
    cy = carry.clone()
    dhh = torch.empty(B, 3 * n, dtype=dt, device="cuda")
    dgx = torch.empty(B, 2 * n, dtype=dt, device="cuda")
    dcx = torch.empty(B, n, dtype=dt, device="cuda")
    acc = torch.empty(B, 6 * n, device="cuda")
    rc = L.px_ln_gru_bwd(_p(hh), _p(stats), _p(gx), 2 * n, _p(cx), n, _p(h), _p(dout), n,
                         _p(drec), _p(cy), _p(dhh), _p(dgx), 2 * n, _p(dcx), n, _p(acc), 1,
                         *[_p(q) for q in prm], _p(lengths), t, B, n, _DT[dt], st)
    assert rc == 0
    torch.cuda.synchronize()
    return {"state": h_next, "out": out, "dhh": dhh, "dgx": dgx, "dcx": dcx, "carry": cy}


def _cell_grads(ops, n, live, dt):
    """the same step by autograd in `dt` (fp64 for the oracle)"""
    hh, gx, cx, h, prm, dout, carry, drec = ops
    leaves = [q.detach().to(dt).requires_grad_(True) for q in (hh, gx, cx, h)]
    state, out = _cell64(*leaves, [q.to(dt) for q in prm], live, n)
    dstate = (carry + drec).to(dt)
    torch.autograd.backward([out, state], [dout.to(dt), dstate])
    return {"state": state.detach(), "out": out.detach(), "dhh": leaves[0].grad,
            "dgx": leaves[1].grad, "dcx": leaves[2].grad, "carry": leaves[3].grad}


@pytest.mark.parametrize("B,n", [(128, 2400), (128, 1200), (3, 16), (4, 8), (4, 2048), (4, 2056),
                                 (4, 4096)])
@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float32])
def test_cell_kernels_vs_fp64(B, n, dt):
    ops = _cell_operands(B, n, dt, seed=B + n)
    lengths = _lengths(B, 9, seed=n)
    t = 4
    live = (lengths > t)[:, None]
    got = _run_cells(B, n, dt, t, lengths, ops)
    ref = _cell_grads(ops, n, live, torch.float64)
    low = _cell_grads(ops, n, live, dt)
    for k in got:
        _assert_calibrated("cell/%d/%d/%s" % (B, n, k), got[k], ref[k], low[k], dt)
    # dead rows pass the state and the carry through bit for bit and output zeros
    dead = ~live[:, 0]
    assert torch.equal(got["state"][dead], ops[3][dead])
    assert torch.equal(got["carry"][dead], (ops[6] + ops[7])[dead])
    assert not got["out"][dead].any() and not got["dhh"][dead].any()


# ===========================================================================
# the whole node
# ===========================================================================
def _module(I, n, seed):
    from parallax_b200.models.skip_thoughts.gru_cell import LayerNormGRU
    torch.manual_seed(seed)
    with torch.device("cuda"):      # the orthonormal init's SVDs, on the device at large n
        m = LayerNormGRU(I, n)
    with torch.no_grad():     # non-trivial LayerNorm parameters
        for ln in (m.ln_wx, m.ln_w, m.ln_wh, m.ln_u):
            ln.weight.add_(0.2 * torch.randn_like(ln.weight))
            ln.bias.add_(0.1 * torch.randn_like(ln.bias))
    return m


_PARAMS = ("w_x", "w", "w_hu", "ln_wh.weight", "ln_wh.bias", "ln_u.weight", "ln_u.bias")


def _run_layer(m, dt, data, composition):
    x, lengths, h0, rev, r_out, r_fin = data
    mm = __import__("copy").deepcopy(m).to(dt)
    xl = x.detach().to(dt).requires_grad_(True)
    hl = None if h0 is None else h0.detach().to(dt).requires_grad_(True)
    fn = mm._composition if composition else mm.forward
    out, fin = fn(xl, lengths, hl, reverse=rev)
    loss = (out.to(r_out.dtype) * r_out).sum() + (fin.to(r_fin.dtype) * r_fin).sum()
    loss.backward()
    prm = dict(mm.named_parameters())
    res = {"out": out.detach(), "final": fin.detach(), "dx": xl.grad}
    for k in _PARAMS:
        res["d_" + k] = prm[k].grad
    if hl is not None:
        res["dh0"] = hl.grad
    return res


def _layer_data(B, I, T, n, rev, with_h0, seed):
    g = _gen(seed)
    x = torch.randn(B, T, I, device="cuda", generator=g)
    h0 = torch.rand(B, n, device="cuda", generator=g) * 2 - 1 if with_h0 else None
    r_out = torch.randn(B, T, n, device="cuda", generator=g, dtype=torch.float64)
    r_fin = torch.randn(B, n, device="cuda", generator=g, dtype=torch.float64)
    return x, _lengths(B, T, seed), h0, rev, r_out, r_fin


_LAYER_CASES = [
    # bench shapes: B 128, I 620, T 31
    (128, 620, 31, 2400, False, False, torch.bfloat16),
    (128, 620, 31, 2400, False, True, torch.float32),
    (128, 620, 31, 1200, True, True, torch.bfloat16),
    (128, 620, 31, 1200, True, False, torch.float32),
] + [(5, 20, 7, 16, rev, h0, dt) for rev in (False, True) for h0 in (False, True)
     for dt in (torch.bfloat16, torch.float32)] + [(3, 12, 4, 40, True, True, torch.bfloat16)] + [
    # the largest n (two full groups per thread) and one thread with a second group
    (4, 24, 3, 4096, False, True, torch.bfloat16),
    (4, 24, 3, 4096, True, False, torch.float32),
    (4, 20, 4, 2056, True, True, torch.bfloat16),
    (3, 20, 1, 2056, False, False, torch.float32),
]


@pytest.mark.parametrize("B,I,T,n,rev,with_h0,dt", _LAYER_CASES)
def test_layer_vs_fp64(B, I, T, n, rev, with_h0, dt):
    from parallax_b200.parallel import nvops
    m = _module(I, n, seed=n + T)
    data = _layer_data(B, I, T, n, rev, with_h0, seed=B + n)
    l0 = nvops.launches["n"]
    got = _run_layer(m, dt, data, composition=False)
    assert nvops.launches["n"] - l0 == 2 * T + 1     # the fused node ran: T fwd, T + 1 bwd
    ref = _run_layer(m, torch.float64, data, composition=True)
    low = _run_layer(m, dt, data, composition=True)
    tag = "layer/%d/%d/%s/%s" % (n, T, "rev" if rev else "fwd", str(dt)[6:])
    for k in ref:
        _assert_calibrated("%s/%s" % (tag, k), got[k], ref[k], low[k], dt)


def test_layer_bit_identical_runs():
    m = _module(40, 64, seed=1)
    data = _layer_data(6, 40, 9, 64, True, True, seed=2)
    a = _run_layer(m, torch.bfloat16, data, composition=False)
    b = _run_layer(m, torch.bfloat16, data, composition=False)
    for k in a:
        assert torch.equal(a[k], b[k]), k


@pytest.mark.parametrize("n,dt", [(12, torch.bfloat16), (16, torch.float64)])
def test_other_shapes_take_the_composition(n, dt):
    from parallax_b200.parallel import nvops
    m = _module(10, n, seed=3)
    data = _layer_data(4, 10, 5, n, False, True, seed=4)
    l0 = nvops.launches["n"]
    a = _run_layer(m, dt, data, composition=False)
    assert nvops.launches["n"] == l0
    b = _run_layer(m, dt, data, composition=True)
    for k in a:
        assert torch.equal(a[k], b[k]), k


@pytest.mark.parametrize("bidirectional", [False, True])
def test_no_grad_encode_matches_training_forward(bidirectional):
    from parallax_b200.models import skip_thoughts as st
    torch.manual_seed(0)
    mc = st.model_config(vocab_size=50, word_embedding_dim=24, encoder_dim=64,
                         bidirectional_encoder=bidirectional)
    model = st.SkipThoughtsModel(mc).cuda().to(torch.bfloat16)
    emb = torch.randn(7, 6, 24, device="cuda").to(torch.bfloat16)
    mask = (torch.arange(6)[None, :] < torch.tensor([6, 1, 3, 6, 2, 5, 4])[:, None]).to(torch.int8)
    with torch.no_grad():
        a = model.encode_embeddings(emb, mask.cuda())
    b = model.encode_embeddings(emb.requires_grad_(True), mask.cuda())
    assert b.requires_grad
    assert torch.equal(a, b.detach())


def test_cuda_graph_replay_matches_eager():
    m = _module(32, 48, seed=5).to(torch.bfloat16)
    B, T, n = 8, 6, 48
    g = _gen(6)
    x = torch.randn(B, T, 32, device="cuda", generator=g).to(torch.bfloat16)
    h0 = torch.randn(B, n, device="cuda", generator=g).to(torch.bfloat16)
    lengths = _lengths(B, T, 7)
    r = torch.randn(B, T, n, device="cuda", generator=g).to(torch.bfloat16)
    params = [p for _, p in m.named_parameters()]

    def step(x_, h_):
        xl, hl = x_.detach().requires_grad_(True), h_.detach().requires_grad_(True)
        out, fin = m(xl, lengths, hl, reverse=True)
        loss = (out * r).float().sum() + fin.float().sum()
        return [out, fin] + list(torch.autograd.grad(loss, [xl, hl] + params))

    # warm-up and the eager reference on a side stream, as whole-step capture does: nothing of
    # the autograd graph may have been recorded on the legacy default stream
    sx, sh = x.clone(), h0.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step(sx, sh)
        eager = [t.clone() for t in step(x, h0)]
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = step(sx, sh)
    sx.zero_()
    graph.replay()      # on other inputs first, then on the eager ones
    sx.copy_(x)
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(static, eager):
        assert torch.equal(a, b)


# ===========================================================================
# the model on the NVLink fabric
# ===========================================================================
def _skip_thoughts_losses(bidirectional, composition, monkeypatch, steps=6, graph=False):
    import parallax_b200 as parallax
    from parallax_b200.models import skip_thoughts as st
    from parallax_b200.models.skip_thoughts import gru_cell
    from parallax_b200.models.skip_thoughts.input_ops import parse_example_batch
    from parallax_b200.ops import fused
    calls = {"n": 0}
    with monkeypatch.context() as mp:
        if composition:
            mp.setattr(gru_cell.LayerNormGRU, "forward", gru_cell.LayerNormGRU._composition)
        else:
            real = fused.ln_gru_layer

            def spy(*a, **k):
                calls["n"] += 1
                return real(*a, **k)
            mp.setattr(fused, "ln_gru_layer", spy)
        torch.manual_seed(0)
        mc = st.model_config(vocab_size=48, word_embedding_dim=16, encoder_dim=32, batch_size=4,
                             num_embedding_partitions=2, bidirectional_encoder=bidirectional)
        tc = st.training_config(learning_rate=0.01)
        model = st.SkipThoughtsModel(mc)
        sess, *_ = parallax.parallel_run(
            st.skip_thoughts_graph(model, tc), "localhost:0",
            parallax_config=parallax.Config(search_partitions=False, sess_config={
                "fabric": "nvlink", "compute_dtype": "bf16", "cuda_graph": graph}))
        batch = parse_example_batch([([3, 4, 5, 0], [6, 7, 0], [8, 0]),
                                     ([9, 0], [3, 0], [4, 5, 6, 0]),
                                     ([10, 11, 0], [12, 0], [13, 14, 0]),
                                     ([5, 0], [6, 0], [7, 0])])
        losses = [sess.run(["loss", "train_op"], st.feed_from_batch(batch))[0][0]
                  for _ in range(steps)]
        captured = bool(getattr(sess.engine, "graph_captured", False))
        sess.close()
    assert captured == graph
    return np.array(losses, dtype=np.float64), calls["n"]


@pytest.mark.parametrize("bidirectional", [False, True])
def test_skip_thoughts_trains_on_the_fused_layer(bidirectional, monkeypatch):
    fused_l, n_calls = _skip_thoughts_losses(bidirectional, False, monkeypatch)
    comp_l, _ = _skip_thoughts_losses(bidirectional, True, monkeypatch)
    print("losses fused", fused_l, "composition", comp_l)
    assert n_calls >= 6 * 3          # every GRU of every step took the fused node
    assert np.isfinite(fused_l).all() and fused_l[-1] < fused_l[0]
    # bf16 rounds differently in the two (the fused cell keeps hh, the statistics and the
    # state update in fp32); over six Adam steps the losses agree to 5 %
    np.testing.assert_allclose(fused_l, comp_l, rtol=5e-2)


def test_skip_thoughts_step_captured_in_a_cuda_graph(monkeypatch):
    """the session captures the whole training step, fused layers included, into a CUDA graph
    and replays it; the replayed losses equal the eager ones"""
    eager, _ = _skip_thoughts_losses(True, False, monkeypatch, steps=8)
    graphed, n_calls = _skip_thoughts_losses(True, False, monkeypatch, steps=8, graph=True)
    print("losses eager", eager, "graphed", graphed)
    assert n_calls > 0
    np.testing.assert_allclose(graphed, eager, rtol=1e-5)
