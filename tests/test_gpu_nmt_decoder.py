"""The fused NMT attention decoder (`ops.fused.nmt_attention_decoder`, `kernels/nmt_decoder.cu`)
against its fp64 reference (`nmt_attention_decoder_reference`) and the model's composition
(`Decoder._composition`).

Kernels and node are held to the calibrated bound of `test_gpu_lm1b_numerics._assert_calibrated`:
against fp64, the fused error stays within 2× the error of the same reference run in the fused
path's dtype (plus a small relative floor)."""
import ctypes

import numpy as np
import pytest
import torch

from tests.test_gpu_lm1b_numerics import _assert_calibrated

pytestmark = pytest.mark.gpu

_vp = ctypes.c_void_p
_DT = {torch.float32: 0, torch.bfloat16: 1}
OPTIONS = ("luong", "scaled_luong", "bahdanau", "normed_bahdanau")


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


def _pad(B, S, seed):
    """ragged source lengths in [1, S] with S and 1 present -> pad mask [B, S]"""
    g = torch.Generator().manual_seed(seed)
    ln = torch.randint(1, S + 1, (B,), generator=g)
    ln[0] = S
    if B > 1:
        ln[1] = 1
    return torch.arange(S)[None, :].cuda() >= ln.cuda()[:, None]


# ===========================================================================
# the kernels, called directly
# ===========================================================================
def _attn_params(option, U, seed):
    g = _gen(seed)
    prm = {"g": None, "v": None, "b": None, "w_q": None}
    if option == "scaled_luong":
        prm["g"] = torch.tensor(0.7, device="cuda")
    if option in ("bahdanau", "normed_bahdanau"):
        prm["v"] = torch.randn(U, device="cuda", generator=g) * 0.3
    if option == "normed_bahdanau":
        prm["b"] = torch.randn(U, device="cuda", generator=g) * 0.2
    return prm


def _attn64(q_or_pq, keys, values, pad, prm, bah):
    """one step of the attention from q (luong) or pq (bahdanau) in fp64 autograd"""
    if bah:
        h = keys + q_or_pq[:, None, :]
        if prm["b"] is not None:
            h = h + prm["b"]
        s = (torch.tanh(h) * prm["v"]).sum(-1)
    else:
        s = torch.bmm(q_or_pq[:, None, :], keys.transpose(1, 2))[:, 0]
        if prm["g"] is not None:
            s = s * prm["g"]
    a = torch.softmax(s.masked_fill(pad, float("-inf")), -1)
    return torch.bmm(a[:, None, :], values)[:, 0], a


@pytest.mark.parametrize("B,S,U,M", [(128, 50, 512, 1024), (128, 50, 1024, 2048),
                                     (128, 50, 1024, 1024), (3, 7, 16, 24),
                                     # the largest accepted shape; S around one pass of the
                                     # 256-thread softmax loops; one lane per score (U 8); M 8
                                     (2, 1024, 1024, 2048), (3, 255, 32, 48), (3, 256, 32, 48),
                                     (3, 257, 32, 48), (3, 1000, 64, 128), (3, 9, 8, 24),
                                     (3, 9, 16, 8)])
@pytest.mark.parametrize("option", OPTIONS)
@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float32])
def test_attention_kernels_vs_fp64(B, S, U, M, option, dt):
    L = _lib()
    bah = option in ("bahdanau", "normed_bahdanau")
    g = _gen(B + S + U)
    scale = 1.0 / np.sqrt(U) if not bah else 1.0
    q = (torch.randn(B, U, device="cuda", generator=g) * scale).to(dt)
    pq = torch.randn(B, U, device="cuda", generator=g) * 0.5
    keys = torch.randn(B, S, U, device="cuda", generator=g).to(dt)
    pad = _pad(B, S, S)
    values = torch.randn(B, S, M, device="cuda", generator=g).masked_fill(pad[..., None], 0).to(dt)
    dctx = torch.randn(B, M, device="cuda", generator=g)
    prm = _attn_params(option, U, seed=U)
    gt = None if prm["g"] is None else prm["g"].to(dt)
    bt = None if prm["b"] is None else prm["b"].to(dt)
    kind = 1 if bah else 0
    ctx = torch.empty(B, M, dtype=dt, device="cuda")
    align = torch.empty(B, S, device="cuda")
    st = _stream()
    assert L.px_nmt_attn_fwd(_p(q), U, _p(pq) if bah else None, _p(keys), _p(values), _p(pad),
                             _p(gt), _p(prm["v"]), _p(bt), _p(ctx), M, None, 0, None, 0,
                             _p(align), B, S, U, M, kind, _DT[dt], st) == 0
    dq = torch.empty(B, U, device="cuda")
    dpq = torch.empty(B, U, dtype=dt, device="cuda")
    dk = torch.zeros(B, S, U, device="cuda")
    dv = torch.zeros(B, S, M, device="cuda")
    part_g = torch.zeros(B, device="cuda")
    part_v = torch.zeros(B, U, device="cuda")
    part_b = torch.zeros(B, U, device="cuda")
    assert L.px_nmt_attn_bwd(_p(dctx), M, None, 0, None, 0, _p(align), _p(q), U,
                             _p(pq) if bah else None, _p(keys), _p(values), _p(gt),
                             _p(prm["v"]), _p(bt), None if bah else _p(dq),
                             _p(dpq) if bah else None, _p(dk), _p(dv), _p(part_g),
                             _p(part_v) if bah else None, _p(part_b) if bt is not None else None,
                             B, S, U, M, kind, _DT[dt], st) == 0
    torch.cuda.synchronize()
    got = {"ctx": ctx.float(), "align": align, "dk": dk, "dv": dv}
    got["dq"] = dpq.float() if bah else dq
    if bah:
        got["dvp"] = part_v.sum(0)
        if bt is not None:
            got["db"] = part_b.sum(0)
    elif gt is not None:
        got["dg"] = part_g.sum(0, keepdim=True)

    def run(cdt):
        lv = [(pq if bah else q).to(cdt), keys.to(cdt), values.to(cdt)]
        lv = [t.detach().requires_grad_(True) for t in lv]
        pr = {k: None if t is None else t.to(dt).to(cdt).detach().requires_grad_(True)
              for k, t in prm.items()}
        if bah:
            pr["v"] = prm["v"].to(cdt).detach().requires_grad_(True)
        c, a = _attn64(lv[0], lv[1], lv[2], pad, pr, bah)
        c.backward(dctx.to(cdt))
        out = {"ctx": c.detach(), "align": a.detach(), "dk": lv[1].grad, "dv": lv[2].grad,
               "dq": lv[0].grad}
        if bah:
            out["dvp"] = pr["v"].grad
            if pr["b"] is not None:
                out["db"] = pr["b"].grad
        elif pr["g"] is not None:
            out["dg"] = pr["g"].grad.reshape(1)
        return out
    ref, low = run(torch.float64), run(dt)
    for k in got:
        _assert_calibrated("attn/%s/%d/%d/%s/%s" % (option, S, U, str(dt)[6:], k),
                           got[k], ref[k], low[k].to(ref[k].dtype), dt)


@pytest.mark.parametrize("B,U", [(128, 512), (128, 1024), (3, 24), (4, 8), (4, 1032)])
@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float32])
def test_cell_kernels_vs_fp64(B, U, dt):
    L = _lib()
    g = _gen(B + U)
    P = torch.randn(B, 4 * U, device="cuda", generator=g) * 2
    gx = torch.randn(B, 4 * U, device="cuda", generator=g)
    b_ih = (torch.randn(4 * U, device="cuda", generator=g) * 0.3).to(dt)
    b_hh = (torch.randn(4 * U, device="cuda", generator=g) * 0.3).to(dt)
    cp = torch.randn(B, U, device="cuda", generator=g)
    resid = torch.randn(B, U, device="cuda", generator=g).to(dt)
    mask = (torch.rand(B, U, device="cuda", generator=g) > 0.2).to(dt) * 1.25
    dA = torch.randn(B, U, device="cuda", generator=g)
    dR = torch.randn(B, U, device="cuda", generator=g)
    drec = torch.randn(B, U, device="cuda", generator=g)
    dc0 = torch.randn(B, U, device="cuda", generator=g)
    cn = torch.empty(B, U, device="cuda")
    h = torch.empty(B, U, dtype=dt, device="cuda")
    y = torch.empty(B, U, dtype=dt, device="cuda")
    xn = torch.empty(B, U, dtype=dt, device="cuda")
    st = _stream()
    assert L.px_nmt_lstm_cell_fwd(_p(P), _p(gx), _p(b_ih), _p(b_hh), _p(cp), _p(cn), _p(h), U,
                                  _p(resid), U, _p(y), U, _p(mask), U, _p(xn), U, B, U, _DT[dt],
                                  st) == 0
    dc = dc0.clone()
    dG = torch.empty(B, 4 * U, dtype=dt, device="cuda")
    dY = torch.empty(B, U, device="cuda")
    assert L.px_nmt_lstm_cell_bwd(_p(P), _p(gx), _p(b_ih), _p(b_hh), _p(cp), _p(cn), _p(dA), U,
                                  _p(mask), U, _p(dR), None, 0, _p(drec), U, _p(dc), _p(dG),
                                  _p(dY), B, U, _DT[dt], st) == 0
    torch.cuda.synchronize()
    got = {"c": cn, "h": h.float(), "y": y.float(), "xn": xn.float(), "dG": dG.float(), "dc": dc}

    def run(cdt):
        pre = (P.to(cdt) + gx.to(cdt) + b_ih.to(cdt) + b_hh.to(cdt)).requires_grad_(True)
        c_prev = cp.to(cdt).requires_grad_(True)
        i, f, gg, o = pre.chunk(4, -1)
        c = torch.sigmoid(f) * c_prev + torch.sigmoid(i) * torch.tanh(gg)
        hh = torch.sigmoid(o) * torch.tanh(c)
        yy = hh + resid.to(cdt)
        dy = dA.to(cdt) * mask.to(cdt) + dR.to(cdt)
        torch.autograd.backward([hh, yy, c], [drec.to(cdt), dy, dc0.to(cdt)])
        return {"c": c.detach(), "h": hh.detach(), "y": yy.detach(),
                "xn": (yy * mask.to(cdt)).detach(), "dG": pre.grad, "dc": c_prev.grad}
    ref, low = run(torch.float64), run(dt)
    for k in got:
        _assert_calibrated("cell/%d/%s/%s" % (U, str(dt)[6:], k), got[k], ref[k],
                           low[k].to(torch.float64), dt)
    torch.testing.assert_close(dY, dA * mask.float() + dR, rtol=1e-6, atol=1e-6)


# ===========================================================================
# the whole node
# ===========================================================================
def _node_inputs(B, T, S, U, M, L, option, arch, residual, dropout, seed):
    g = _gen(seed)
    A = U if arch == "standard" else M
    I = [U + A] + [U] * (L - 1)

    def w(*shape, s=0.1):
        return torch.randn(*shape, device="cuda", generator=g) * s
    pad = _pad(B, S, seed)
    x = {"emb": w(B, T, U, s=1.0), "att0": w(B, A, s=0.5),
         "keys": w(B, S, U, s=1.0),
         "values": w(B, S, M, s=1.0).masked_fill(pad[..., None], 0)}
    x["h0"] = [w(B, U, s=0.5) for _ in range(L)]
    x["c0"] = [w(B, U, s=0.5) for _ in range(L)]
    x["w_ih"] = [w(4 * U, I[l], s=1.0 / np.sqrt(I[l])) for l in range(L)]
    x["w_hh"] = [w(4 * U, U, s=1.0 / np.sqrt(U)) for l in range(L)]
    x["b_ih"] = [w(4 * U, s=0.2) for _ in range(L)]
    x["b_hh"] = [w(4 * U, s=0.2) for _ in range(L)]
    if option in ("bahdanau", "normed_bahdanau"):
        x["w_q"] = w(U, U, s=1.0 / np.sqrt(U))
        x["v"] = w(U, s=0.3)
        if option == "normed_bahdanau":
            x["b"] = w(U, s=0.2)
    elif option == "scaled_luong":
        x["g"] = torch.tensor(0.5, device="cuda")
    if arch == "standard":
        x["w_a"] = w(U, U + M, s=1.0 / np.sqrt(U + M))
    masks = None
    if dropout:
        masks = [(torch.rand(T, B, I[l], device="cuda", generator=g) > dropout).float() /
                 (1 - dropout) for l in range(L)]
    r = [w(B, T, U, s=1.0, )] + ([w(B, T, M, s=1.0)] if arch != "standard" else [])
    return x, pad, masks, [residual and (l > 0 or L == 1) for l in range(L)], r


def _run_node(x, pad, masks, residual, r, cdt, reference, output_attention=True):
    from parallax_b200.ops import fused
    leaves = {}
    for k, v in x.items():
        if isinstance(v, list):
            leaves[k] = [t.to(cdt).detach().requires_grad_(True) for t in v]
        else:
            leaves[k] = v.to(cdt).detach().requires_grad_(True)
    kw = {k: leaves[k] for k in ("w_q", "g", "b", "w_a") if k in leaves}
    if "v" in leaves:
        kw["v"] = leaves["v"] if cdt == torch.float64 else leaves["v"].float()
    fn = fused.nmt_attention_decoder_reference if reference else fused.nmt_attention_decoder
    out = fn(leaves["emb"], leaves["h0"], leaves["c0"], leaves["att0"], leaves["keys"],
             leaves["values"], pad, leaves["w_ih"], leaves["w_hh"], leaves["b_ih"],
             leaves["b_hh"], residual,
             masks=None if masks is None else [m.to(cdt) for m in masks],
             output_attention=output_attention, **kw)
    outs = out if isinstance(out, tuple) else (out,)
    loss = sum((o.to(torch.float64) * rr.to(torch.float64)).sum() for o, rr in zip(outs, r))
    loss.backward()
    res = {"out%d" % i: o.detach() for i, o in enumerate(outs)}
    for k, v in leaves.items():
        if isinstance(v, list):
            for i, t in enumerate(v):
                res["d_%s%d" % (k, i)] = t.grad
        else:
            res["d_" + k] = v.grad
    return res


_NODE_CASES = [
    # the three benchmark shapes: B 128, S = T = 50
    (128, 50, 50, 512, 1024, 2, "scaled_luong", "standard", False, torch.bfloat16),
    (128, 50, 50, 1024, 2048, 4, "normed_bahdanau", "standard", True, torch.bfloat16),
    (128, 50, 50, 1024, 1024, 1, "normed_bahdanau", "gnmt_v2", False, torch.bfloat16),
] + [(5, 6, 7, 16, 24, 3, opt, "standard", True, dt) for opt in OPTIONS
     for dt in (torch.bfloat16, torch.float32)] + \
    [(5, 6, 7, 16, 16, 1, opt, "gnmt", opt in ("luong", "bahdanau"), torch.float32)
     for opt in OPTIONS] + [
    # the largest shape the gate accepts, and S past one softmax pass of 256 threads
    (2, 2, 1024, 1024, 2048, 1, "scaled_luong", "standard", False, torch.float32),
    (3, 3, 300, 64, 128, 1, "normed_bahdanau", "gnmt_v2", True, torch.bfloat16),
]


@pytest.mark.parametrize("B,T,S,U,M,L,option,arch,residual,dt", _NODE_CASES)
def test_node_vs_fp64(B, T, S, U, M, L, option, arch, residual, dt):
    from parallax_b200.parallel import nvops
    x, pad, masks, res, r = _node_inputs(B, T, S, U, M, L, option, arch, residual, 0.2,
                                         seed=U + L)
    l0 = nvops.launches["n"]
    got = _run_node(x, pad, masks, res, r, dt, reference=False)
    assert nvops.launches["n"] - l0 >= 2 * T * (L + 1)       # the fused node ran both ways
    ref = _run_node(x, pad, masks, res, r, torch.float64, reference=True)
    low = _run_node(x, pad, masks, res, r, dt, reference=True)
    tag = "node/%s/%s/%d/%s" % (arch, option, U, str(dt)[6:])
    for k in ref:
        # scaled_luong's d_g is one sum of B·T·S terms that largely cancel: its error is a
        # single draw, held to 4× the reference's rather than 2×
        _assert_calibrated("%s/%s" % (tag, k), got[k].to(torch.float64), ref[k],
                           low[k].to(torch.float64), dt, factor=4.0 if ref[k].dim() == 0 else 2.0)


def test_node_output_q_and_bit_identical_runs():
    x, pad, masks, res, r = _node_inputs(6, 5, 9, 32, 48, 2, "luong", "standard", True, 0.2, 3)
    a = _run_node(x, pad, masks, res, r, torch.bfloat16, False, output_attention=False)
    b = _run_node(x, pad, masks, res, r, torch.bfloat16, False, output_attention=False)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    ref = _run_node(x, pad, masks, res, r, torch.float64, True, output_attention=False)
    low = _run_node(x, pad, masks, res, r, torch.bfloat16, True, output_attention=False)
    for k in ref:
        _assert_calibrated("node/q/" + k, a[k].to(torch.float64), ref[k],
                           low[k].to(torch.float64), torch.bfloat16)


# ===========================================================================
# the model
# ===========================================================================
def _model(option, arch, unit_type="lstm", U=32, dt=torch.bfloat16, seed=0):
    import parallax_b200.models.nmt as nmt
    torch.manual_seed(seed)
    hp = nmt.create_hparams(num_units=U, num_layers=2 if arch == "standard" else 3,
                            encoder_type="bi" if arch == "standard" else "gnmt",
                            attention=option, attention_architecture=arch, residual=True,
                            dropout=0.0, unit_type=unit_type)
    nmt.extend_hparams(hp, 40, 40)
    return nmt.create_model(hp).cuda().to(dt)


def _batch(B=6, S=9, T=7, seed=1):
    g = torch.Generator().manual_seed(seed)
    src = torch.randint(3, 40, (B, S), generator=g).cuda()
    tgt = torch.randint(3, 40, (B, T), generator=g).cuda()
    sl = torch.randint(1, S + 1, (B,), generator=g)
    sl[0] = S
    return src, tgt, sl.cuda()


@pytest.mark.parametrize("option,arch", [("scaled_luong", "standard"),
                                         ("normed_bahdanau", "gnmt_v2"),
                                         ("bahdanau", "gnmt")])
def test_no_grad_forward_equals_training_forward(option, arch):
    m = _model(option, arch)
    src, tgt, sl = _batch()
    with torch.no_grad():
        a = m.logits(src, tgt, sl)
    b = m.logits(src, tgt, sl)
    assert b.requires_grad
    assert torch.equal(a, b.detach())


@pytest.mark.parametrize("option,arch,S", [
    pytest.param(o, a, 9, id="%s-%s" % (o, a))
    for o, a in (("luong", "standard"), ("normed_bahdanau", "standard"),
                 ("normed_bahdanau", "gnmt_v2"), ("scaled_luong", "gnmt"))] + [
    # a source of the longest accepted length: every softmax loop runs four passes per thread
    pytest.param("scaled_luong", "standard", 1024, id="scaled_luong-standard-S1024")])
def test_decode_step_reproduces_teacher_forced_logits(option, arch, S, monkeypatch):
    from parallax_b200.ops import fused
    m = _model(option, arch, dt=torch.float32).eval()
    src, tgt, sl = _batch(S=S)
    calls = {"n": 0}
    real = fused.nmt_attention_decoder_step

    def spy(*a, **k):
        calls["n"] += 1
        return real(*a, **k)
    monkeypatch.setattr(fused, "nmt_attention_decoder_step", spy)
    with torch.no_grad():
        full = m.logits(src, tgt, sl)
        memory, state = m.encode(src, sl)
        steps = []
        for t in range(tgt.shape[1]):
            lg, state = m.decode_step(tgt[:, t], state, memory)
            steps.append(lg)
    assert calls["n"] == tgt.shape[1]
    torch.testing.assert_close(torch.stack(steps, 1), full, rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("case", ["gru", "fp64", "odd_units"])
def test_other_decoders_take_the_composition(case, monkeypatch):
    from parallax_b200.ops import fused
    if case == "gru":
        m = _model("normed_bahdanau", "standard", unit_type="gru")
    elif case == "fp64":
        m = _model("normed_bahdanau", "gnmt_v2", dt=torch.float64)
    else:
        m = _model("scaled_luong", "standard", U=36)
    monkeypatch.setattr(fused, "nmt_attention_decoder",
                        lambda *a, **k: pytest.fail("the fused node ran"))
    src, tgt, sl = _batch()
    memory, state = m.encode(src, sl)
    emb = m.embedding_decoder(tgt).to(m.compute_dtype)
    a = m.decoder(emb, state, memory)
    b = m.decoder._composition(emb, state, memory)
    assert torch.equal(a, b)


def _nmt_losses(option, arch, composition, monkeypatch, steps=6):
    import parallax_b200 as parallax
    import parallax_b200.models.nmt as nmt
    from parallax_b200.models.nmt import model as nmt_model
    from parallax_b200.ops import fused
    calls = {"n": 0}
    with monkeypatch.context() as mp:
        if composition:
            mp.setattr(nmt_model.Decoder, "forward", nmt_model.Decoder._composition)
        else:
            real = fused.nmt_attention_decoder

            def spy(*a, **k):
                calls["n"] += 1
                return real(*a, **k)
            mp.setattr(fused, "nmt_attention_decoder", spy)
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
def test_nmt_trains_on_the_fused_decoder(option, arch, monkeypatch):
    fused_l, n_calls = _nmt_losses(option, arch, False, monkeypatch)
    comp_l, _ = _nmt_losses(option, arch, True, monkeypatch)
    print("losses fused", fused_l, "composition", comp_l)
    assert n_calls >= 6
    assert np.isfinite(fused_l).all() and fused_l[-1] < fused_l[0]
    np.testing.assert_allclose(fused_l, comp_l, rtol=5e-2)
