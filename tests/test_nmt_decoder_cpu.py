"""`ops.fused.nmt_attention_decoder_reference` (the fp64 oracle of the fused NMT decoder node)
against `Decoder._composition`, on the CPU in fp64 with all-ones masks: outputs and gradients."""
import pytest
import torch

import parallax_b200.models.nmt as nmt
from parallax_b200.ops import fused


def _decoder_case(option, arch, residual, output_attention, seed=0):
    torch.manual_seed(seed)
    hp = nmt.create_hparams(num_units=16, num_encoder_layers=2 if arch == "standard" else 4,
                            num_decoder_layers=3 if arch == "standard" else 4,
                            encoder_type="gnmt" if arch != "standard" else "bi",
                            attention=option, attention_architecture=arch, residual=residual,
                            output_attention=output_attention, dropout=0.0)
    nmt.extend_hparams(hp, 30, 30)
    m = nmt.create_model(hp).double()
    with torch.no_grad():      # non-zero biases and attention parameters
        for n, p in m.named_parameters():
            if p.dim() < 2:
                p.add_(0.3 * torch.randn_like(p))
    B, S, T = 5, 7, 6
    src = torch.randint(3, 30, (B, S))
    src_len = torch.tensor([7, 3, 5, 1, 6])
    memory, state = m.encode(src, src_len)
    emb = torch.randn(B, T, 16, dtype=torch.float64)
    return m, emb, memory, state


def _leaves(m, emb, memory, state):
    """fresh leaves for the decoder's inputs (so both arms see the same graph roots)"""
    keys, values, pad = memory
    keys, values = keys.detach().requires_grad_(True), values.detach().requires_grad_(True)
    cells = [tuple(x.detach().requires_grad_(True) for x in c) for c in state["cells"]]
    st = {"cells": cells, "attention": state["attention"].detach().requires_grad_(True)}
    return emb.detach().requires_grad_(True), (keys, values, pad), st


def _grads(m, out, emb, memory, state, r):
    loss = (out * r).sum()
    layers, _, _ = m.decoder.node_arguments()
    n = len(layers)
    ins = [emb, memory[0], memory[1], state["attention"]] + \
        [x for c in state["cells"][:n] for x in c]
    prm = [p for p in m.decoder.parameters() if p.requires_grad]
    g = torch.autograd.grad(loss, ins + prm, allow_unused=True)
    return [torch.zeros_like(t) if x is None else x for x, t in zip(g, ins + prm)]


@pytest.mark.parametrize("option", ["luong", "scaled_luong", "bahdanau", "normed_bahdanau"])
@pytest.mark.parametrize("arch,residual,output_attention", [
    ("standard", False, True), ("standard", True, False),
    ("gnmt", True, True), ("gnmt_v2", True, True), ("gnmt_v2", False, True)])
def test_reference_equals_composition(option, arch, residual, output_attention):
    m, emb, memory, state = _decoder_case(option, arch, residual, output_attention)
    dec = m.decoder
    r = torch.randn(emb.shape, dtype=torch.float64)

    e1, mem1, st1 = _leaves(m, emb, memory, state)
    comp = dec._composition(e1, st1, mem1)
    g_comp = _grads(m, comp, e1, mem1, st1, r)

    e2, mem2, st2 = _leaves(m, emb, memory, state)
    layers, kw, _ = dec.node_arguments()
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

    # the composition takes its attention softmax in fp32 (`AttentionMechanism.forward` casts the
    # scores with .float()), the reference keeps fp64 throughout: they agree to fp32 rounding
    torch.testing.assert_close(out, comp, rtol=1e-5, atol=1e-6)
    for a, b in zip(g_ref, g_comp):
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)


def test_cpu_decoder_takes_the_composition():
    """on the CPU `forward` is the composition, bit for bit"""
    m, emb, memory, state = _decoder_case("normed_bahdanau", "gnmt_v2", True, True)
    with torch.no_grad():
        a = m.decoder(emb, state, memory)
        b = m.decoder._composition(emb, state, memory)
    assert torch.equal(a, b)
