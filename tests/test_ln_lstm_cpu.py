"""`LayerNormLSTM` off the GPU: the fused layer's gate refuses CPU tensors, and the layer
computes what its Python time loop computed before the fused node existed, bit for bit."""
import copy

import pytest
import torch

from parallax_b200.models.nmt.model import LayerNormLSTM
from parallax_b200.ops import fused


def _loop(m, x, state, lengths=None):
    """`LayerNormLSTM.forward` as it was before the fused node: the reference for bit equality"""
    h, c = state
    outs = []
    for t in range(x.shape[1]):
        h2, c2 = m.cell(x[:, t], h, c)
        if lengths is not None:
            live = (lengths > t)[:, None]
            h2, c2 = torch.where(live, h2, h), torch.where(live, c2, c)
            outs.append(torch.where(live, h2, torch.zeros_like(h2)))
        else:
            outs.append(h2)
        h, c = h2, c2
    return torch.stack(outs, 1), (h, c)


def _module(I, U, dt, seed):
    torch.manual_seed(seed)
    m = LayerNormLSTM(I, U, forget_bias=1.0)
    with torch.no_grad():
        for ln in list(m.ln) + [m.ln_c]:
            ln.weight.add_(0.2 * torch.randn_like(ln.weight))
            ln.bias.add_(0.1 * torch.randn_like(ln.bias))
    return m.to(dt)


def _run(m, fn, x, h0, c0, lengths, r):
    xl, hl, cl = (t.detach().clone().requires_grad_(True) for t in (x, h0, c0))
    out, (h, c) = fn(m, xl, (hl, cl), lengths)
    loss = (out * r).sum() + h.sum() + 2 * c.sum()
    params = list(m.parameters())
    grads = torch.autograd.grad(loss, [xl, hl, cl] + params)
    return [out, h, c] + list(grads)


@pytest.mark.parametrize("dt", [torch.float32, torch.float64])
@pytest.mark.parametrize("ragged", [False, True])
def test_forward_on_the_cpu_equals_the_loop(dt, ragged):
    B, T, I, U = 5, 6, 12, 16
    m = _module(I, U, dt, seed=3)
    g = torch.Generator().manual_seed(4)
    x = torch.randn(B, T, I, generator=g).to(dt)
    h0 = torch.randn(B, U, generator=g).to(dt)
    c0 = torch.randn(B, U, generator=g).to(dt)
    r = torch.randn(B, T, U, generator=g).to(dt)
    lengths = torch.tensor([6, 1, 3, 6, 2]) if ragged else None
    assert not fused.ln_lstm_applies(x, m.kernel.weight, m.ln, m.ln_c, h0, c0)
    got = _run(m, LayerNormLSTM.forward, x, h0, c0, lengths, r)
    ref = _run(copy.deepcopy(m), _loop, x, h0, c0, lengths, r)
    for a, b in zip(got, ref):
        assert torch.equal(a, b)


def test_gate_refuses_cpu_tensors():
    m = _module(8, 16, torch.float32, seed=0)
    x = torch.randn(2, 3, 8)
    assert not fused.ln_lstm_applies(x, m.kernel.weight, m.ln, m.ln_c)
    assert not fused.ln_lstm_applies(x.bfloat16(), m.kernel.weight.bfloat16(), m.ln, m.ln_c)


# ---------------------------------------------------------------------------
# the attention decoder node's fp64 oracle with layer_norm_lstm cells
# ---------------------------------------------------------------------------
def _decoder_case(option, arch, residual, seed=0):
    import parallax_b200.models.nmt as nmt
    torch.manual_seed(seed)
    hp = nmt.create_hparams(num_units=16, num_encoder_layers=2 if arch == "standard" else 4,
                            num_decoder_layers=3 if arch == "standard" else 4,
                            encoder_type="gnmt" if arch != "standard" else "bi",
                            attention=option, attention_architecture=arch, residual=residual,
                            dropout=0.0, unit_type="layer_norm_lstm")
    nmt.extend_hparams(hp, 30, 30)
    m = nmt.create_model(hp).double()
    with torch.no_grad():      # non-trivial LayerNorm and attention parameters
        for n, p in m.named_parameters():
            if p.dim() < 2:
                p.add_(0.3 * torch.randn_like(p))
    B, S, T = 5, 7, 6
    memory, state = m.encode(torch.randint(3, 30, (B, S)), torch.tensor([7, 3, 5, 1, 6]))
    return m, torch.randn(B, T, 16, dtype=torch.float64), memory, state


def _leaves(emb, memory, state):
    keys, values, pad = memory
    keys, values = keys.detach().requires_grad_(True), values.detach().requires_grad_(True)
    cells = [tuple(x.detach().requires_grad_(True) for x in c) for c in state["cells"]]
    st = {"cells": cells, "attention": state["attention"].detach().requires_grad_(True)}
    return emb.detach().requires_grad_(True), (keys, values, pad), st


def _grads(m, out, emb, memory, state, r):
    layers, _, _ = m.decoder.node_arguments()
    ins = [emb, memory[0], memory[1], state["attention"]] + \
        [x for c in state["cells"][:len(layers)] for x in c]
    prm = [p for p in m.decoder.parameters() if p.requires_grad]
    g = torch.autograd.grad((out * r).sum(), ins + prm, allow_unused=True)
    return [torch.zeros_like(t) if x is None else x for x, t in zip(g, ins + prm)]


@pytest.mark.parametrize("option", ["luong", "scaled_luong", "bahdanau", "normed_bahdanau"])
@pytest.mark.parametrize("arch,residual", [("standard", False), ("standard", True),
                                           ("gnmt", True), ("gnmt_v2", True)])
def test_decoder_reference_equals_composition(option, arch, residual):
    """`nmt_attention_decoder_reference` with LN-LSTM cells equals `Decoder._composition` in
    fp64, outputs and every gradient (the composition's attention softmax is fp32)"""
    m, emb, memory, state = _decoder_case(option, arch, residual)
    dec = m.decoder
    r = torch.randn(emb.shape, dtype=torch.float64)
    e1, mem1, st1 = _leaves(emb, memory, state)
    comp = dec._composition(e1, st1, mem1)
    g_comp = _grads(m, comp, e1, mem1, st1, r)
    e2, mem2, st2 = _leaves(emb, memory, state)
    layers, kw, _ = dec.node_arguments()
    assert kw["ln"] is not None and kw["b_ih"] is None
    n = len(layers)
    T, B = emb.shape[1], emb.shape[0]
    masks = [torch.ones(T, B, l.input_size, dtype=torch.float64) for l in layers]
    out = fused.nmt_attention_decoder_reference(
        e2, [c[0] for c in st2["cells"][:n]], [c[1] for c in st2["cells"][:n]],
        st2["attention"], mem2[0], mem2[1], mem2[2], masks=masks,
        output_attention=dec.output_attention, **kw)
    if arch != "standard":
        out = dec._gnmt_upper(*out, st2)
    g_ref = _grads(m, out, e2, mem2, st2, r)
    torch.testing.assert_close(out, comp, rtol=1e-5, atol=1e-6)
    # the fp32 softmax's rounding reaches the gradients through five LayerNorm backwards per step
    for a, b in zip(g_ref, g_comp):
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-5)


def test_decoder_applies_refuses_cpu_and_gru():
    x = torch.zeros(2, 3, 8)
    assert not fused.nmt_decoder_applies(x, torch.zeros(2, 4, 8), torch.zeros(2, 4, 8), [], [],
                                         "layer_norm_lstm")
