"""The fused layer-normalised LSTM (`ops.fused.ln_lstm_layer`, `kernels/ln_lstm.cu`) against
fp64: the cell kernels on exact operands, and the whole layer against the fp64 composition
(`LayerNormLSTM._composition`) under the calibrated bound of
`test_gpu_lm1b_numerics._assert_calibrated` (the fused error stays within 2× the error of the
same composition run in the fused path's dtype, plus a small relative floor)."""
import copy
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.test_gpu_lm1b_numerics import _assert_calibrated

pytestmark = pytest.mark.gpu

_vp = ctypes.c_void_p
_DT = {torch.float32: 0, torch.bfloat16: 1}
EPS = 1e-5


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
def _cell64(pre, c, gam, bet, fb):
    """one step of `LayerNormLSTM.cell` from the pre-LayerNorm gate terms"""
    U = c.shape[1]
    a = [F.layer_norm(g, (U,), gam[k], bet[k], EPS) for k, g in enumerate(pre.split(U, 1))]
    c2 = c * torch.sigmoid(a[2] + fb) + torch.sigmoid(a[0]) * torch.tanh(a[1])
    h2 = torch.tanh(F.layer_norm(c2, (U,), gam[4], bet[4], EPS)) * torch.sigmoid(a[3])
    return h2, c2


def _close(name, got, ref, dt):
    """fp32 math throughout; bf16 only where the kernel stores bf16"""
    tol = 2e-2 if dt == torch.bfloat16 else 2e-4
    scale = float(ref.abs().max())
    err = float((got.double() - ref).abs().max())
    print("%-28s max err %.2e (scale %.2e)" % (name, err, scale))
    assert torch.isfinite(got).all(), name
    assert err <= tol * max(scale, 1e-3), (name, err, scale)


@pytest.mark.parametrize("B,U", [(128, 512), (128, 1024), (3, 16), (4, 8), (4, 1032), (4, 2048)])
@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float32])
def test_cell_kernels_vs_fp64(B, U, dt):
    L = _lib()
    g = _gen(B + U)
    f32 = dict(device="cuda", dtype=torch.float32)
    P = torch.randn(B, 4 * U, generator=g, **f32) * 2.0 + 0.3
    gx = torch.randn(B, 4 * U, generator=g, **f32)
    c = torch.randn(B, U, generator=g, **f32)
    h = torch.randn(B, U, generator=g, **f32).to(dt)
    gam = [(1.0 + 0.3 * torch.randn(U, generator=g, **f32)).to(dt) for _ in range(5)]
    bet = [(0.2 * torch.randn(U, generator=g, **f32)).to(dt) for _ in range(5)]
    dout = torch.randn(B, U, generator=g, **f32).to(dt)
    carry_h0 = torch.randn(B, U, generator=g, **f32)
    carry_c0 = torch.randn(B, U, generator=g, **f32)
    drec = torch.randn(B, U, generator=g, **f32)
    fb, t = 1.0, 2
    lengths = torch.tensor([3 if b % 3 else 1 for b in range(B)], device="cuda")  # live: t < 3
    live = (lengths > t)[:, None]
    ln = (_vp * 10)(*[q.data_ptr() for q in gam + bet])
    ep = (ctypes.c_float * 5)(*[EPS] * 5)
    st = _stream()
    c_new = torch.empty(B, U, **f32)
    h_next = torch.empty(B, U, dtype=dt, device="cuda")
    out = torch.empty(B, U, dtype=dt, device="cuda")
    stats = torch.empty(B, 10, **f32)
    assert L.px_ln_lstm_fwd(_p(P), _p(gx), 4 * U, _p(c), _p(c_new), _p(h), U, _p(h_next), U,
                            _p(out), U, _p(stats), ln, ep, fb, _p(lengths), t, B, U, _DT[dt],
                            st) == 0
    carry_h, carry_c = carry_h0.clone(), carry_c0.clone()
    dpre = torch.empty(B, 4 * U, dtype=dt, device="cuda")
    acc = torch.empty(B, 10 * U, **f32)
    assert L.px_ln_lstm_bwd(_p(P), _p(gx), 4 * U, _p(stats), _p(c), _p(dout), U, _p(drec),
                            _p(carry_h), _p(carry_c), _p(dpre), 4 * U, _p(acc), 1, ln, ep, fb,
                            _p(lengths), t, B, U, _DT[dt], st) == 0
    dln = torch.empty(10, U, dtype=dt, device="cuda")
    assert L.px_ln_lstm_param_grad(_p(acc), B, U, _p(dln), _DT[dt], st) == 0
    torch.cuda.synchronize()

    # fp64 oracle on the same operands
    pre = (P.double() + gx.double()).requires_grad_(True)
    c64 = c.double().requires_grad_(True)
    g64 = [q.double().requires_grad_(True) for q in gam]
    b64 = [q.double().requires_grad_(True) for q in bet]
    h2, c2 = _cell64(pre, c64, g64, b64, fb)
    h64 = h.double()
    _close("h_next", h_next, torch.where(live, h2, h64), dt)
    _close("out", out, torch.where(live, h2, torch.zeros_like(h2)), dt)
    _close("c_new", c_new, torch.where(live, c2, c64), torch.float32)
    dh_t = carry_h0.double() + drec.double()
    dh = torch.where(live, dout.double() + dh_t, torch.zeros_like(dh_t))
    dc = torch.where(live, carry_c0.double(), torch.zeros_like(dh_t))
    grads = torch.autograd.grad((h2 * dh).sum() + (c2 * dc).sum(), [pre, c64] + g64 + b64)
    _close("dpre", dpre, grads[0], dt)
    _close("carry_c", carry_c, torch.where(live, grads[1], carry_c0.double()), torch.float32)
    _close("carry_h", carry_h, torch.where(live, torch.zeros_like(dh_t), dh_t), torch.float32)
    for k in range(10):
        _close("dln[%d]" % k, dln[k], grads[2 + k], dt)
    # the statistics of the live rows' LayerNorms
    mean = pre.detach().view(B, 4, U).mean(-1)
    var = pre.detach().view(B, 4, U).var(-1, correction=0)
    _close("mean", stats[:, 0:8:2], mean, torch.float32)
    _close("rstd", stats[:, 1:8:2], (var + EPS).rsqrt(), torch.float32)
    # bit-identical on a second launch
    again = torch.empty_like(dpre)
    ch, cc = carry_h0.clone(), carry_c0.clone()
    assert L.px_ln_lstm_bwd(_p(P), _p(gx), 4 * U, _p(stats), _p(c), _p(dout), U, _p(drec),
                            _p(ch), _p(cc), _p(again), 4 * U, _p(acc), 1, ln, ep, fb,
                            _p(lengths), t, B, U, _DT[dt], st) == 0
    assert torch.equal(again, dpre) and torch.equal(cc, carry_c) and torch.equal(ch, carry_h)


# ===========================================================================
# the whole layer
# ===========================================================================
def _module(I, U, seed):
    from parallax_b200.models.nmt.model import LayerNormLSTM
    torch.manual_seed(seed)
    m = LayerNormLSTM(I, U, forget_bias=1.0).cuda()
    with torch.no_grad():
        m.kernel.weight.uniform_(-0.1, 0.1)
        for ln in list(m.ln) + [m.ln_c]:        # non-trivial LayerNorm parameters
            ln.weight.add_(0.2 * torch.randn_like(ln.weight))
            ln.bias.add_(0.1 * torch.randn_like(ln.bias))
    return m


def _layer_data(B, T, I, U, with_state, seed):
    g = _gen(seed)
    x = torch.randn(B, T, I, device="cuda", generator=g)
    if with_state:
        h0 = torch.rand(B, U, device="cuda", generator=g) * 2 - 1
        c0 = torch.randn(B, U, device="cuda", generator=g)
    else:
        h0 = c0 = torch.zeros(B, U, device="cuda")
    r_out = torch.randn(B, T, U, device="cuda", generator=g, dtype=torch.float64)
    r_h = torch.randn(B, U, device="cuda", generator=g, dtype=torch.float64)
    r_c = torch.randn(B, U, device="cuda", generator=g, dtype=torch.float64)
    return x, _lengths(B, T, seed), h0, c0, r_out, r_h, r_c


def _run_layer(m, dt, data, composition):
    x, lengths, h0, c0, r_out, r_h, r_c = data
    mm = copy.deepcopy(m).to(dt)
    xl, hl, cl = (t.detach().to(dt).requires_grad_(True) for t in (x, h0, c0))
    fn = mm._composition if composition else mm.forward
    out, (h, c) = fn(xl, (hl, cl), lengths)
    loss = (out.to(r_out.dtype) * r_out).sum() + (h.to(r_h.dtype) * r_h).sum() + \
        (c.to(r_c.dtype) * r_c).sum()
    loss.backward()
    res = {"out": out.detach(), "h": h.detach(), "c": c.detach(), "dx": xl.grad,
           "dh0": hl.grad, "dc0": cl.grad}
    for k, p in mm.named_parameters():
        res["d_" + k] = p.grad
    return res


_LAYER_CASES = [
    # bench shapes: B 128, T 50, iwslt15 (U 512) and wmt16 (U 1024)
    (128, 50, 512, 512, True, torch.bfloat16),
    (128, 50, 1024, 1024, True, torch.bfloat16),
    (128, 50, 1024, 512, False, torch.float32),
] + [(5, 7, 20, 16, s, dt) for s in (False, True) for dt in (torch.bfloat16, torch.float32)] + \
    [(3, 4, 12, 40, True, torch.bfloat16)] + [
    # every thread on (U 2048), one thread past 1024, T 1, and odd I: W_h = w[:, I:] is then a
    # view at a 2-byte offset in bf16
    (4, 3, 24, 2048, True, torch.bfloat16),
    (4, 2, 16, 1032, False, torch.float32),
    (3, 1, 20, 1032, True, torch.bfloat16),
    (4, 3, 13, 40, True, torch.bfloat16),
    (4, 3, 1, 64, False, torch.bfloat16),
]


@pytest.mark.parametrize("B,T,I,U,with_state,dt", _LAYER_CASES)
def test_layer_vs_fp64(B, T, I, U, with_state, dt):
    from parallax_b200.parallel import nvops
    m = _module(I, U, seed=U + T)
    data = _layer_data(B, T, I, U, with_state, seed=B + U)
    l0 = nvops.launches["n"]
    got = _run_layer(m, dt, data, composition=False)
    assert nvops.launches["n"] - l0 == 2 * T + 1     # the fused node ran: T fwd, T + 1 bwd
    ref = _run_layer(m, torch.float64, data, composition=True)
    low = _run_layer(m, dt, data, composition=True)
    assert len(ref) == 6 + 11
    tag = "layer/%d/%d/%s" % (U, T, str(dt)[6:])
    for k in ref:
        _assert_calibrated("%s/%s" % (tag, k), got[k], ref[k], low[k], dt)


def test_layer_bit_identical_runs_and_no_grad():
    m = _module(40, 64, seed=1)
    data = _layer_data(6, 9, 40, 64, True, seed=2)
    a = _run_layer(m, torch.bfloat16, data, composition=False)
    b = _run_layer(m, torch.bfloat16, data, composition=False)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    x, lengths, h0, c0 = data[:4]
    mm = copy.deepcopy(m).to(torch.bfloat16)
    xb, hb, cb = (t.to(torch.bfloat16) for t in (x, h0, c0))
    with torch.no_grad():
        out, (h, c) = mm(xb, (hb, cb), lengths)
    assert torch.equal(out, a["out"]) and torch.equal(h, a["h"]) and torch.equal(c, a["c"])


def test_cuda_graph_replay_matches_eager():
    m = _module(32, 48, seed=5).to(torch.bfloat16)
    B, T, U = 8, 6, 48
    g = _gen(6)
    x = torch.randn(B, T, 32, device="cuda", generator=g).to(torch.bfloat16)
    h0 = torch.randn(B, U, device="cuda", generator=g).to(torch.bfloat16)
    c0 = torch.randn(B, U, device="cuda", generator=g).to(torch.bfloat16)
    lengths = _lengths(B, T, 7)
    r = torch.randn(B, T, U, device="cuda", generator=g).to(torch.bfloat16)
    params = list(m.parameters())

    def step(x_, h_, c_):
        xl, hl, cl = (t.detach().requires_grad_(True) for t in (x_, h_, c_))
        out, (h, c) = m(xl, (hl, cl), lengths)
        loss = (out * r).float().sum() + h.float().sum() + c.float().sum()
        return [out, h, c] + list(torch.autograd.grad(loss, [xl, hl, cl] + params))

    sx, sh, sc = x.clone(), h0.clone(), c0.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step(sx, sh, sc)
        eager = [t.clone() for t in step(x, h0, c0)]
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = step(sx, sh, sc)
    sx.zero_()
    graph.replay()      # on other inputs first, then on the eager ones
    sx.copy_(x)
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(static, eager):
        assert torch.equal(a, b)


@pytest.mark.parametrize("case", ["odd_units", "fp64", "cpu"])
def test_other_layers_take_the_composition(case, monkeypatch):
    from parallax_b200.ops import fused
    U, dt = {"odd_units": (12, torch.bfloat16), "fp64": (16, torch.float64),
             "cpu": (16, torch.float32)}[case]
    m = _module(10, U, seed=3)
    data = _layer_data(4, 5, 10, U, True, seed=4)
    if case == "cpu":
        m = m.cpu()
        data = tuple(t.cpu() for t in data)
    monkeypatch.setattr(fused, "ln_lstm_layer", lambda *a, **k: pytest.fail("the fused node ran"))
    a = _run_layer(m, dt, data, composition=False)
    b = _run_layer(m, dt, data, composition=True)
    for k in a:
        assert torch.equal(a[k], b[k]), k


# ===========================================================================
# the model on the NVLink fabric
# ===========================================================================
def _nmt_losses(composition, monkeypatch, steps=6):
    import parallax_b200 as parallax
    import parallax_b200.models.nmt as nmt
    from parallax_b200.models.nmt import model as nmt_model
    from parallax_b200.ops import fused
    calls = {"ln_lstm_layer": 0, "nmt_attention_decoder": 0}
    with monkeypatch.context() as mp:
        if composition:
            mp.setattr(nmt_model.LayerNormLSTM, "forward", nmt_model.LayerNormLSTM._composition)
            mp.setattr(nmt_model.Decoder, "forward", nmt_model.Decoder._composition)
        else:
            for name in calls:
                def spy(*a, _name=name, _real=getattr(fused, name), **k):
                    calls[_name] += 1
                    return _real(*a, **k)
                mp.setattr(fused, name, spy)
        torch.manual_seed(0)
        hp = nmt.create_hparams(num_units=32, num_layers=2, encoder_type="bi",
                                attention="scaled_luong", attention_architecture="standard",
                                residual=True, dropout=0.0, num_embeddings_partitions=2,
                                learning_rate=0.1, unit_type="layer_norm_lstm")
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
    return np.array(losses, dtype=np.float64), calls


def test_nmt_trains_on_the_fused_layer(monkeypatch):
    fused_l, calls = _nmt_losses(False, monkeypatch)
    comp_l, _ = _nmt_losses(True, monkeypatch)
    print("losses fused", fused_l, "composition", comp_l, calls)
    # per step: the two encoder directions on the layer node, the decoder on the decoder node
    assert calls["ln_lstm_layer"] >= 6 * 2 and calls["nmt_attention_decoder"] >= 6
    assert np.isfinite(fused_l).all() and fused_l[-1] < fused_l[0]
    # bf16 rounds differently in the two (the fused cell keeps the products, the statistics and
    # the cell state in fp32); at a learning rate where training is stable the losses of six
    # steps agree to 5 %
    np.testing.assert_allclose(fused_l, comp_l, rtol=5e-2)


# ===========================================================================
# the attention decoder node over LN-LSTM cells
# ===========================================================================
def _ln_node_inputs(B, T, S, U, M, L, option, arch, residual, dropout, seed):
    """`test_gpu_nmt_decoder._node_inputs` with each layer's weights as one bias-free kernel
    [4U, I + U] and the five LayerNorms' γ/β of each layer"""
    from tests.test_gpu_nmt_decoder import _node_inputs
    x, pad, masks, res, r = _node_inputs(B, T, S, U, M, L, option, arch, residual, dropout, seed)
    g = _gen(seed + 1)
    x["kernel"] = [torch.cat([a, b], 1) for a, b in zip(x.pop("w_ih"), x.pop("w_hh"))]
    del x["b_ih"], x["b_hh"]
    x["ln"] = [torch.cat([1.0 + 0.2 * torch.randn(5 * U, device="cuda", generator=g),
                          0.2 * torch.randn(5 * U, device="cuda", generator=g)])
               for _ in range(L)]
    return x, pad, masks, res, r


def _run_ln_node(x, pad, masks, residual, r, cdt, reference, step=False):
    from parallax_b200.ops import fused
    leaves = {k: ([t.to(cdt).detach().requires_grad_(True) for t in v] if isinstance(v, list)
                  else v.to(cdt).detach().requires_grad_(True)) for k, v in x.items()}
    kw = {k: leaves[k] for k in ("w_q", "g", "b", "w_a") if k in leaves}
    if "v" in leaves:
        kw["v"] = leaves["v"] if cdt == torch.float64 else leaves["v"].float()
    U = leaves["emb"].shape[2]
    I = [k.shape[1] - U for k in leaves["kernel"]]
    ln = [(list(p.view(10, U).unbind(0)), [EPS] * 5, 1.0) for p in leaves["ln"]]
    args = (leaves["emb"], leaves["h0"], leaves["c0"], leaves["att0"], leaves["keys"],
            leaves["values"], pad, [k[:, :i] for k, i in zip(leaves["kernel"], I)],
            [k[:, i:] for k, i in zip(leaves["kernel"], I)], None, None, residual)
    mk = None if masks is None else [m.to(cdt) for m in masks]
    fn = fused.nmt_attention_decoder_reference if reference else fused.nmt_attention_decoder
    out = fn(*args, masks=mk, ln=ln, **kw)
    outs = out if isinstance(out, tuple) else (out,)
    loss = sum((o.to(torch.float64) * rr.to(torch.float64)).sum() for o, rr in zip(outs, r))
    loss.backward()
    res = {"out%d" % i: o.detach() for i, o in enumerate(outs)}
    for k, v in leaves.items():
        for i, t in enumerate(v if isinstance(v, list) else [v]):
            res["d_%s%d" % (k, i)] = t.grad
    return res


_NODE_CASES = [
    # benchmark shapes: iwslt15's decoder and wmt16 gnmt's bottom layer, B 128, S = T = 50
    (128, 50, 50, 512, 1024, 2, "scaled_luong", "standard", False, torch.bfloat16),
    (128, 50, 50, 1024, 1024, 1, "normed_bahdanau", "gnmt_v2", False, torch.bfloat16),
] + [(5, 6, 7, 16, 24, 3, opt, "standard", True, dt)
     for opt in ("luong", "scaled_luong", "bahdanau", "normed_bahdanau")
     for dt in (torch.bfloat16, torch.float32)] + \
    [(5, 6, 7, 16, 16, 1, opt, "gnmt_v2", True, torch.float32)
     for opt in ("luong", "scaled_luong", "bahdanau", "normed_bahdanau")] + [
    # the largest shape the gate accepts, and S past one softmax pass of 256 threads
    (2, 2, 1024, 1024, 2048, 1, "scaled_luong", "standard", False, torch.float32),
    (3, 3, 300, 64, 128, 1, "normed_bahdanau", "gnmt_v2", True, torch.bfloat16),
]


@pytest.mark.parametrize("B,T,S,U,M,L,option,arch,residual,dt", _NODE_CASES)
def test_decoder_node_vs_fp64(B, T, S, U, M, L, option, arch, residual, dt):
    from parallax_b200.parallel import nvops
    x, pad, masks, res, r = _ln_node_inputs(B, T, S, U, M, L, option, arch, residual, 0.2,
                                            seed=U + L)
    l0 = nvops.launches["n"]
    got = _run_ln_node(x, pad, masks, res, r, dt, reference=False)
    assert nvops.launches["n"] - l0 >= 2 * T * (L + 1)       # the fused node ran both ways
    ref = _run_ln_node(x, pad, masks, res, r, torch.float64, reference=True)
    low = _run_ln_node(x, pad, masks, res, r, dt, reference=True)
    tag = "ln-node/%s/%s/%d/%s" % (arch, option, U, str(dt)[6:])
    for k in ref:
        # as in test_gpu_nmt_decoder: scaled_luong's d_g is one sum of B·T·S terms that largely
        # cancel, held to 4× the reference's error rather than 2×
        _assert_calibrated("%s/%s" % (tag, k), got[k].to(torch.float64), ref[k],
                           low[k].to(torch.float64), dt, factor=4.0 if ref[k].dim() == 0 else 2.0)


@pytest.mark.parametrize("option,arch,S", [
    pytest.param(o, a, 9, id="%s-%s" % (o, a))
    for o, a in (("luong", "standard"), ("normed_bahdanau", "standard"),
                 ("normed_bahdanau", "gnmt_v2"), ("scaled_luong", "gnmt"))] + [
    # a source of the longest accepted length: every softmax loop runs four passes per thread
    pytest.param("bahdanau", "standard", 1024, id="bahdanau-standard-S1024")])
def test_decode_step_reproduces_teacher_forced_logits(option, arch, S, monkeypatch):
    from parallax_b200.ops import fused
    from tests.test_gpu_nmt_decoder import _batch, _model
    m = _model(option, arch, unit_type="layer_norm_lstm", dt=torch.float32).eval()
    src, tgt, sl = _batch(S=S)
    calls = {"n": 0, "train": 0}
    real, real_train = fused.nmt_attention_decoder_step, fused.nmt_attention_decoder

    def spy(*a, **k):
        calls["n"] += 1
        return real(*a, **k)

    def spy_train(*a, **k):
        calls["train"] += 1
        return real_train(*a, **k)
    monkeypatch.setattr(fused, "nmt_attention_decoder_step", spy)
    monkeypatch.setattr(fused, "nmt_attention_decoder", spy_train)
    with torch.no_grad():
        full = m.logits(src, tgt, sl)
        memory, state = m.encode(src, sl)
        steps = []
        for t in range(tgt.shape[1]):
            lg, state = m.decode_step(tgt[:, t], state, memory)
            steps.append(lg)
    assert calls["n"] == tgt.shape[1] and calls["train"] == 1
    torch.testing.assert_close(torch.stack(steps, 1), full, rtol=1e-4, atol=1e-4)
