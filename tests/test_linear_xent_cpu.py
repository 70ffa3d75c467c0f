"""`parallax.nn.linear_cross_entropy` off the fused path: on the CPU it is the composition
``(cross_entropy(linear(x, W, b).float(), t, reduction="none") * w).sum()`` bit for bit, the NMT
and skip-thoughts training losses built on it equal the formulas they replaced bit for bit, in
losses and every gradient, and each invalid argument raises `ValueError`."""
import pytest
import torch
import torch.nn.functional as F

import parallax_b200.models.nmt as nmt
import parallax_b200.models.skip_thoughts as st
from parallax_b200 import nn as pnn
from parallax_b200.models.skip_thoughts.input_ops import parse_example_batch
from parallax_b200.ops import fused


def _grads(params):
    return [None if p.grad is None else
            (p.grad.to_dense() if p.grad.is_sparse else p.grad).clone() for p in params]


def _assert_same_grads(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert (x is None) == (y is None)
        if x is not None:
            assert torch.equal(x, y)


@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("row_weights", [False, True])
@pytest.mark.parametrize("dt", [torch.float32, torch.float64])
def test_op_equals_the_composition(bias, row_weights, dt):
    torch.manual_seed(0)
    N, K, V = 37, 24, 53
    x = torch.randn(N, K, dtype=dt, requires_grad=True)
    w = torch.randn(V, K, dtype=dt, requires_grad=True)
    b = torch.randn(V, dtype=dt, requires_grad=True) if bias else None
    t = torch.randint(0, V, (N,))
    t[0], t[1] = 0, V - 1
    rw = torch.randn(N) if row_weights else None
    if rw is not None:
        rw[::3] = 0.0
    loss, nll = pnn.linear_cross_entropy(x, t, w, b, row_weights=rw)
    loss.backward()
    got = _grads([x, w] + ([b] if bias else []))
    for p in [x, w] + ([b] if bias else []):
        p.grad = None
    ref_nll = F.cross_entropy(F.linear(x, w, b).float(), t, reduction="none")
    ref = (ref_nll * rw).sum() if rw is not None else ref_nll.sum()
    ref.backward()
    assert torch.equal(loss, ref) and torch.equal(nll, ref_nll.detach())
    assert not nll.requires_grad
    _assert_same_grads(got, _grads([x, w] + ([b] if bias else [])))


def test_target_outside_the_vocabulary_gives_nan():
    torch.manual_seed(0)
    x, w = torch.randn(4, 8), torch.randn(5, 8)
    t = torch.tensor([0, 5, -1, 4])
    loss, nll = pnn.linear_cross_entropy(x, t, w)
    assert torch.isnan(nll[1]) and torch.isnan(nll[2]) and torch.isnan(loss)
    ok = F.cross_entropy(x @ w.t(), torch.tensor([0, 0, 0, 4]), reduction="none")
    assert torch.equal(nll[[0, 3]], ok[[0, 3]])


def test_cpu_and_fp32_take_the_composition(monkeypatch):
    calls = {"n": 0}

    def spy(*a, **k):
        calls["n"] += 1
        raise AssertionError("the fused op must not run here")
    monkeypatch.setattr(fused, "linear_cross_entropy", spy)
    x = torch.randn(3, 8, dtype=torch.bfloat16)
    pnn.linear_cross_entropy(x, torch.tensor([1, 2, 3]), torch.randn(4, 8, dtype=torch.bfloat16))
    assert calls["n"] == 0
    assert not fused.linear_xent_applies(x, torch.randn(4, 8, dtype=torch.bfloat16), None)


# ------------------------------------------------------------------------------------- models
def _nmt_case(option, arch, seed=0):
    torch.manual_seed(seed)
    hp = nmt.create_hparams(num_units=16, num_encoder_layers=2 if arch == "standard" else 4,
                            num_decoder_layers=2 if arch == "standard" else 4,
                            encoder_type="gnmt" if arch != "standard" else "bi",
                            attention=option, attention_architecture=arch, dropout=0.0)
    nmt.extend_hparams(hp, 30, 33)
    m = nmt.create_model(hp)
    m.train()
    B, S, T = 5, 7, 6
    feed = dict(source=torch.randint(3, 30, (B, S)), target_input=torch.randint(3, 33, (B, T)),
                target_output=torch.randint(3, 33, (B, T)),
                source_sequence_length=torch.tensor([7, 3, 5, 1, 6]),
                target_sequence_length=torch.tensor([6, 2, 4, 1, 5]))
    return m, feed


def _nmt_parent_loss(m, source, target_input, target_output, source_sequence_length,
                     target_sequence_length):
    """`Seq2Seq.forward`'s loss before it took `linear_cross_entropy`"""
    logits = m.logits(source, target_input, source_sequence_length)
    B, T, V = logits.shape
    xent = F.cross_entropy(logits.reshape(B * T, V), target_output.reshape(-1),
                           reduction="none").view(B, T)
    tl = target_sequence_length.to(xent.device)
    mask = (torch.arange(T, device=xent.device)[None, :] < tl[:, None]).to(xent.dtype)
    return (xent * mask).sum() / B


@pytest.mark.parametrize("option,arch", [("scaled_luong", "standard"),
                                         ("normed_bahdanau", "gnmt_v2")])
def test_nmt_loss_and_gradients_equal_the_parent_formula(option, arch):
    m, feed = _nmt_case(option, arch)
    params = list(m.parameters())
    ref = _nmt_parent_loss(m, **feed)
    ref.backward()
    ref_g = _grads(params)
    m.zero_grad(set_to_none=True)
    out = m(**feed)
    out["loss"].backward()
    assert torch.equal(out["loss"], ref)
    _assert_same_grads(_grads(params), ref_g)


def _skip_parent_loss(model, encode_ids, encode_mask, decode_pre_ids, decode_pre_mask,
                      decode_post_ids, decode_post_mask):
    """`SkipThoughtsModel.forward`'s losses before it took `linear_cross_entropy`"""
    thought = model.encode(encode_ids, encode_mask)

    def decode(gru, ids, mask):
        emb = model.word_embedding(ids).to(model.compute_dtype)
        inp = F.pad(emb[:, :-1, :], (0, 0, 1, 0))
        mask = mask.to(emb.device)
        out, _ = gru(inp, mask.sum(1), initial_state=thought)
        logits = model.logits(out).float()
        losses = F.cross_entropy(logits.view(-1, logits.shape[-1]), ids.reshape(-1),
                                 reduction="none")
        return losses, mask.reshape(-1).to(losses.dtype)
    l_pre, w_pre = decode(model.decoder_pre, decode_pre_ids, decode_pre_mask)
    l_post, w_post = decode(model.decoder_post, decode_post_ids, decode_post_mask)
    pre, post = (l_pre * w_pre).sum(), (l_post * w_post).sum()
    return pre + post, pre, post, w_pre.sum() + w_post.sum()


@pytest.mark.parametrize("bidirectional", [False, True])
def test_skip_thoughts_losses_and_gradients_equal_the_parent_formula(bidirectional):
    torch.manual_seed(0)
    m = st.SkipThoughtsModel(st.model_config(vocab_size=40, word_embedding_dim=12, encoder_dim=16,
                                             batch_size=16, bidirectional_encoder=bidirectional))
    with torch.no_grad():
        m.logits.bias.normal_()
    batch = parse_example_batch([([3, 4, 5, 0], [6, 7, 0], [8, 0]),
                                 ([9, 0], [3, 0], [4, 5, 6, 0]),
                                 ([10, 11, 0], [12, 0], [13, 14, 0])])
    feed = {k: v[0] for k, v in st.feed_from_batch(batch).items()}
    params = list(m.parameters())
    loss, pre, post, sw = _skip_parent_loss(m, **feed)
    loss.backward()
    ref_g = _grads(params)
    m.zero_grad(set_to_none=True)
    out = m(**feed)
    out["loss"].backward()
    assert torch.equal(out["loss"], loss)
    assert torch.equal(out["loss_pre"], pre.detach()) and torch.equal(out["loss_post"], post.detach())
    assert torch.equal(out["sum_weights"], sw.detach())
    _assert_same_grads(_grads(params), ref_g)


# ----------------------------------------------------------------------------- invalid calls
def _ok():
    return torch.randn(4, 8), torch.tensor([0, 1, 2, 3]), torch.randn(5, 8)


@pytest.mark.parametrize("case", ["inputs_1d", "weight_cols", "weight_1d", "dtype_mismatch",
                                  "int_inputs", "targets_len", "targets_2d", "targets_float",
                                  "targets_bool", "bias_shape", "bias_int", "rw_shape",
                                  "rw_bool", "devices"])
def test_invalid_arguments_raise_value_error(case):
    x, t, w = _ok()
    kw = {}
    if case == "inputs_1d":
        x = x[0]
    elif case == "weight_cols":
        w = torch.randn(5, 7)
    elif case == "weight_1d":
        w = torch.randn(8)
    elif case == "dtype_mismatch":
        w = w.double()
    elif case == "int_inputs":
        x, w = x.long(), w.long()
    elif case == "targets_len":
        t = t[:3]
    elif case == "targets_2d":
        t = t[:, None]
    elif case == "targets_float":
        t = t.float()
    elif case == "targets_bool":
        t = t > 1
    elif case == "bias_shape":
        kw["bias"] = torch.randn(4)
    elif case == "bias_int":
        kw["bias"] = torch.zeros(5, dtype=torch.long)
    elif case == "rw_shape":
        kw["row_weights"] = torch.ones(3)
    elif case == "rw_bool":
        kw["row_weights"] = torch.ones(4, dtype=torch.bool)
    elif case == "devices":
        t = t.to("meta")
    with pytest.raises(ValueError):
        pnn.linear_cross_entropy(x, t, w, **kw)
