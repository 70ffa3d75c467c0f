"""Fused full-softmax training (`NVSparseGroup.full_softmax_nll_lse` / `full_softmax_nll_grad`,
the GRAD instantiations of `ops/csrc/kernels/softmax_eval.cu`) against fp64 on worlds simulated
inside one GPU, and LM1B(num_sampled=0) sessions with ``full_softmax_train="fused"`` against the
composition."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import parallax_b200 as parallax
from parallax_b200 import consts
from tests.test_full_softmax_train_cpu import chunked_backward
from tests.test_gpu_full_softmax import CASES, _groups, _owners, _table

pytestmark = pytest.mark.gpu


def _rel(a, ref):
    return float((a.double() - ref).norm() / ref.norm().clamp_min(1e-300))


def _reference(x, Wt, Bt, targets, g):
    """fp64 (nll, lse, dx, dW, db) of the bf16-exact operands (the oracle's chunked schedule
    over the whole table)."""
    logits = x.double() @ Wt.double().t() + Bt.double().t()
    lse = torch.logsumexp(logits, dim=1)
    nll = lse - logits.gather(1, targets[:, None])[:, 0]
    gather = lambda ids: (Wt[ids].double(), Bt[ids, 0].double())
    dx, dW, db = chunked_backward(x, targets, lse, g, gather, Wt.shape[0], 4096)
    return nll, lse, dx, dW, db


def _composition(x, Wt, Bt, targets, g):
    """dx, dW, db of `engine.full_softmax_composition`'s arithmetic on the same bf16 operands:
    bf16 logits, fp32 bias add and cross entropy, bf16 lookup rows and their gradients."""
    xc = x.cuda().requires_grad_()
    w = Wt.cuda().bfloat16().requires_grad_()
    b = Bt.cuda().bfloat16().requires_grad_()
    logits = (xc @ w.t()).float() + b.squeeze(-1).float()
    F.cross_entropy(logits, targets.cuda(), reduction="none").backward(g.cuda())
    return xc.grad.cpu(), w.grad.cpu(), b.grad[:, 0].cpu()


def _check(grp, x, Wt, Bt, targets, g, chunk=None, bound=1e-2):
    nll_ref, lse_ref, dx_ref, dW_ref, db_ref = _reference(x, Wt, Bt, targets, g)
    comp = _composition(x, Wt, Bt, targets, g)
    nll, lse = grp.full_softmax_nll_lse(x.cuda(), targets.cuda())
    dx, dW, db = grp.full_softmax_nll_grad(x.cuda(), targets.cuda(), lse, g.cuda(), chunk=chunk)
    torch.cuda.synchronize()
    V, K = Wt.shape
    assert dx.shape == x.shape and dx.dtype == torch.bfloat16
    assert dW.shape == (V, K) and dW.dtype == torch.bfloat16
    assert db.shape == (V, 1) and db.dtype == torch.bfloat16
    torch.testing.assert_close(nll.cpu().double(), nll_ref, rtol=1e-5, atol=1e-3)
    torch.testing.assert_close(lse.cpu().double(), lse_ref, rtol=1e-5, atol=1e-3)
    for ours, c, ref in zip((dx, dW, db[:, 0]), comp, (dx_ref, dW_ref, db_ref)):
        ours = ours.cpu()
        assert torch.isfinite(ours).all()
        e, ec = _rel(ours, ref), _rel(c, ref)
        assert e <= bound and e <= 1.5 * ec, (e, ec)


def _inputs(N, K, V, seed, scale=1.0):
    gen = torch.Generator().manual_seed(seed)
    x = (torch.randn(N, K, generator=gen) * scale).bfloat16()
    targets = torch.randint(0, V, (N,), generator=gen)
    targets[0], targets[-1] = 0, V - 1
    g = torch.rand(N, generator=gen) * 2 - 0.5             # non-uniform, some negative
    g[N // 2] = 0.0
    return x, targets, g


@pytest.mark.parametrize("chunk", [None, 384])
@pytest.mark.parametrize("world,V,P,strategy,K,N,replicated", CASES)
def test_grad_matches_fp64(world, V, P, strategy, K, N, replicated, chunk):
    Wt, Bt = _table(V, K, 17)
    fabs, groups = _groups(world, Wt, Bt, P, strategy, replicated, _owners(world, P, replicated))
    x, targets, g = _inputs(N, K, V, world * 100 + K)
    for grp in groups:                    # every rank computes its batch alone
        _check(grp, x, Wt, Bt, targets, g, chunk)
    for f in fabs:
        f.close()


@pytest.mark.parametrize("world,P", [(1, 1), (2, 5), (4, 7)])
def test_grad_bf16_masters(world, P):
    V, K, N = 2999, 136, 300
    Wt, Bt = _table(V, K, 12)
    Bt = (Bt + 0.5).bfloat16().float()
    fabs, groups = _groups(world, Wt, Bt, P, weights="bf16")
    assert groups[0].tables[1].weight_dtype == torch.bfloat16
    x, targets, g = _inputs(N, K, V, 13)
    for grp in groups:
        _check(grp, x, Wt, Bt, targets, g, chunk=640)
    for f in fabs:
        f.close()


def test_large_logits_stay_finite():
    """Logits up to about ±80: exp(s − lse) never overflows."""
    V, K, N = 4097, 64, 300
    Wt, Bt = _table(V, K, 7, scale=8.0)
    fabs, groups = _groups(2, Wt, Bt, 4)
    x, targets, g = _inputs(N, K, V, 1, scale=2.0)
    logits = x.double() @ Wt.double().t() + Bt.double().t()
    assert 60 < float(logits.abs().max()) < 120
    for grp in groups:
        _check(grp, x, Wt, Bt, targets, g, chunk=1000)
    for f in fabs:
        f.close()


def test_bounded_memory():
    """V = 200 000, N = 2560, K = 512: forward plus backward grow the peak allocation by at most
    the gradient rows, the chunk scratch and 64 MB; the composition would need > 3 GB of
    logits."""
    V, K, N = 200000, 512, 2560
    Wt, Bt = _table(V, K, 7)
    fabs, groups = _groups(1, Wt, Bt, 1)
    grp = groups[0]
    x = torch.randn(N, K, device="cuda").bfloat16()
    targets = torch.randint(0, V, (N,), device="cuda")
    g = torch.rand(N, device="cuda")

    def step():
        nll, lse = grp.full_softmax_nll_lse(x, targets)
        return nll, grp.full_softmax_nll_grad(x, targets, lse, g)
    step()                                                   # warm-up (modules, cuBLAS)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    nll, (dx, dW, db) = step()
    torch.cuda.synchronize()
    growth = torch.cuda.max_memory_allocated() - base
    Dp = grp.tables[0].Dp
    assert growth <= V * Dp * 2 + consts.FULL_SOFTMAX_TRAIN_WS_BYTES + (64 << 20), growth
    assert N * V * 6 > 3e9
    assert grp.full_softmax_train_chunk(N) < V              # the backward ran in chunks
    # the first rows against fp64
    xs, ts, gs = x[:64].cpu(), targets[:64].cpu(), g[:64].cpu()
    logits = xs.double() @ Wt.double().t() + Bt.double().t()
    lse = torch.logsumexp(logits, 1)
    G = (torch.softmax(logits, 1) - F.one_hot(ts, V).double()) * gs[:, None].double()
    assert torch.isfinite(dx).all() and torch.isfinite(dW).all()
    assert _rel(dx[:64].cpu(), G @ Wt.double()) < 1e-2
    torch.testing.assert_close(nll[:64].cpu().double(), lse - logits.gather(1, ts[:, None])[:, 0],
                               rtol=1e-5, atol=1e-3)
    for f in fabs:
        f.close()


def test_argument_errors():
    Wt, Bt = _table(300, 32, 1)
    fabs, groups = _groups(1, Wt, Bt, 1)
    L = parallax.ops.lib()
    x = torch.randn(4, 32, device="cuda").bfloat16()
    z = torch.zeros(1024, device="cuda")
    p = z.data_ptr()
    # K not a multiple of 8; a G pitch below the chunk's 128-row blocks
    assert L.px_full_softmax_grad(x.data_ptr(), 4, 30, p, 32, p, 4, 0, 100, 0, p, p, p, p, 128,
                                  p, 132, None) == -1
    assert L.px_full_softmax_grad(x.data_ptr(), 4, 32, p, 32, p, 4, 0, 200, 0, p, p, p, p, 128,
                                  p, 132, None) == -2
    with pytest.raises(ValueError, match="bf16 inputs"):
        groups[0].full_softmax_nll_grad(x.float(), torch.zeros(4, dtype=torch.long),
                                        torch.zeros(4), torch.zeros(4))
    for f in fabs:
        f.close()


# ------------------------------------------------------------------ through the engine
def _session(train, **extra):
    from parallax_b200.models.lm1b import LM1B, lm1b_graph
    torch.manual_seed(0)
    m = LM1B(vocab_size=1003, emb_size=32, state_size=64, projected_size=32, num_sampled=0,
             num_steps=4, num_shards=3, keep_prob=1.0)
    sc = dict({"fabric": "nvlink", "compute_dtype": "bf16", "full_softmax_train": train}, **extra)
    sess, *_ = parallax.parallel_run(lm1b_graph(m, batch_size=128), "localhost:0",
                                     parallax_config=parallax.Config(sess_config=sc))
    return sess


def _batch(seed, V=1003):
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(0, V, (128, 4), generator=g)
    return {"x": [x], "y": [torch.roll(x, -1, dims=1)]}


_ROWS = torch.randperm(1003, generator=torch.Generator().manual_seed(5))[:64]


def _state(sess):
    m = sess.engine.model
    torch.cuda.synchronize()
    w = m.softmax_w.table.full_weight()[_ROWS].float().cpu()
    b = m.softmax_b.table.full_weight()[_ROWS].float().cpu()
    return [w, b] + [p.detach().float().cpu().clone() for p in (m.W, m.B, m.W_P)]


def _train(sess, steps, freeze_tables=False):
    m = sess.engine.model
    if freeze_tables:
        m.softmax_w._anchor.requires_grad_(False)
        m.softmax_b._anchor.requires_grad_(False)
    s0 = _state(sess)
    losses = [float(sess.run(["loss", "train_op"], _batch(i % 3))[0][0]) for i in range(steps)]
    return losses, s0, _state(sess)


def _counters(monkeypatch):
    from parallax_b200.parallel import engine
    from parallax_b200.parallel.nv_sparse import NVSparseGroup
    calls = {"fused": 0, "eval": 0, "composition": 0}

    def wrap(owner, name, key):
        orig = getattr(owner, name)

        def counted(*a, **k):
            calls[key] += 1
            return orig(*a, **k)
        monkeypatch.setattr(owner, name, counted)
    wrap(NVSparseGroup, "full_softmax_nll_lse", "fused")
    wrap(NVSparseGroup, "full_softmax_nll", "eval")
    wrap(engine, "full_softmax_composition", "composition")
    return calls


ENGINE = [
    # name, sess_config, steps, forward passes per step (before capture), frozen tables
    ("plain", {}, 3, 1, False),
    ("cuda_graph", {"cuda_graph": True, "graph_warmup": 2}, 5, 1, False),
    ("micro_batches", {"micro_batches": 2}, 3, 2, False),
    ("bf16_masters", {"sparse_weights": "bf16"}, 3, 1, False),
    ("inputs_only", {}, 3, 1, True),
]


@pytest.mark.parametrize("name,extra,steps,per_step,frozen", ENGINE, ids=[e[0] for e in ENGINE])
def test_engine_fused_training_matches_composition(monkeypatch, name, extra, steps, per_step,
                                                   frozen):
    comp = _session("composition", **extra)
    c_losses, c0, c1 = _train(comp, steps, frozen)
    comp.close()
    calls = _counters(monkeypatch)
    sess = _session("fused", **extra)
    grp = sess.engine.model.softmax_w.table.group
    f_losses, f0, f1 = _train(sess, steps, frozen)
    if extra.get("cuda_graph"):
        assert sess.engine.graph_captured
        # eager warm-up steps and the capture call the fused path; replays launch it
        assert calls["fused"] == extra["graph_warmup"] + 1
    else:
        assert calls["fused"] == steps * per_step
    assert calls["eval"] == 0 and calls["composition"] == 0
    assert grp.overflow_count() == 0
    sess.close()
    assert np.isfinite(f_losses).all() and f_losses[-1] < f_losses[0]
    np.testing.assert_allclose(f_losses, c_losses, rtol=0, atol=3e-2)
    for i, (a0, a1, b0, b1) in enumerate(zip(f0, f1, c0, c1)):
        assert torch.equal(a0, b0)                         # the same initial state
        du, dc = a1 - a0, b1 - b0
        if frozen and i < 2:
            assert not du.any() and not dc.any()           # the tables took no gradient
            continue
        assert dc.norm() > 0
        assert float((du - dc).norm() / dc.norm()) < 0.1
