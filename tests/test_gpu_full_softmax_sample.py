"""Fused full-softmax sampling (`parallax.nn.full_softmax_sample`, `px_full_softmax_sample` in
`ops/csrc/kernels/softmax_eval.cu`) against an fp64 Gumbel-top-k built from the same bf16 rows and
the same noise, on worlds simulated inside one GPU, and through the engine on the NVLink fabric."""
import numpy as np
import pytest
import torch
from scipy import stats

import parallax_b200 as parallax
from parallax_b200.parallel.engine import sample_uniform
from tests.test_gpu_full_softmax import (CASES, _batch, _groups, _lm1b_session, _owners,
                                         _table)

pytestmark = pytest.mark.gpu


def _inv(tau):
    return float(torch.tensor(1.0 / tau, dtype=torch.float32))


def _reference(x, Wt, Bt, tau, seed):
    """fp64 tempered log-probabilities [N, V], Gumbel keys [N, V] and each row's ids sorted by
    key (descending), with s = fp32(1/τ) · logit as the kernel scales"""
    N, V = x.shape[0], Wt.shape[0]
    s = (x.double() @ Wt.double().t() + Bt.double().t()) * _inv(tau)
    v = sample_uniform(seed, torch.arange(N), torch.arange(V)).double()
    keys = s - torch.log(-torch.log1p(-v))
    return torch.log_softmax(s, dim=-1), keys, torch.sort(keys, dim=1, descending=True).indices


def _check(lp, ids, ref, n, V, margin=2e-3):
    ref_lp, keys, order = ref
    lp, ids = lp.cpu(), ids.cpu()
    N = ref_lp.shape[0]
    assert lp.shape == (N, n) and lp.dtype == torch.float32
    assert ids.shape == (N, n) and ids.dtype == torch.int64
    assert ((ids >= 0) & (ids < V)).all()                    # never a padding row
    assert all(len(set(r)) == n for r in ids.tolist())
    torch.testing.assert_close(lp.double(), ref_lp.gather(1, ids), rtol=0, atol=1e-3)
    kk = keys.gather(1, ids)
    assert (kk[:, 1:] <= kk[:, :-1] + margin).all()          # draw order
    srt = keys.gather(1, order[:, :n + 1] if n < V else order)
    d = srt[:, :-1] - srt[:, 1:]
    ok = torch.ones(N, n, dtype=torch.bool)
    ok[:, 1:] &= d[:, :n - 1] > margin
    if n < V:
        ok &= d[:, :n] > margin
    assert ok.float().mean() > 0.3
    assert torch.equal(ids[ok], order[:, :n][ok])


@pytest.mark.parametrize("tau", [0.7, 1.0, 1.5])
@pytest.mark.parametrize("n", [1, 5, 12, 32])
@pytest.mark.parametrize("world,V,P,strategy,K,N,replicated", CASES)
def test_sample_kernel_matches_fp64_reference(world, V, P, strategy, K, N, replicated, n, tau):
    Wt, Bt = _table(V, K, world * 10 + P)
    fabs, groups = _groups(world, Wt, Bt, P, strategy, replicated, _owners(world, P, replicated))
    x = torch.randn(N, K, generator=torch.Generator().manual_seed(world * 100 + K)).bfloat16()
    seed = 1000 * n + world
    ref = _reference(x.float(), Wt, Bt, tau, seed)
    for grp in groups:                    # every rank evaluates its batch alone
        lp, ids = grp.full_softmax_sample(x.cuda(), n, _inv(tau), seed)
        torch.cuda.synchronize()
        _check(lp, ids, ref, n, V)
    for f in fabs:
        f.close()


def test_same_seed_same_draws_across_worlds_partitions_layouts_and_chunks(monkeypatch):
    from parallax_b200 import consts
    V, K, N, n = 3001, 64, 700, 8
    Wt, Bt = _table(V, K, 3)
    x = torch.randn(N, K, generator=torch.Generator().manual_seed(4)).bfloat16().cuda()
    draws = []
    for world, P, strategy, replicated in [(1, 1, "mod", False), (2, 5, "mod", False),
                                           (4, 7, "div", False), (3, 3, "div", False),
                                           (4, 1, "mod", True)]:
        fabs, groups = _groups(world, Wt, Bt, P, strategy, replicated,
                               _owners(world, P, replicated))
        for grp in groups:
            draws.append(grp.full_softmax_sample(x, n, 1.0, 42))
        if world == 2:                    # row chunks: 128 rows per launch
            monkeypatch.setattr(consts, "TOPK_WS_BYTES", 1 << 20)
            draws.append(groups[1].full_softmax_sample(x, n, 1.0, 42))
            monkeypatch.undo()
        for f in fabs:
            f.close()
    lp0, ids0 = draws[0]
    for lp, ids in draws[1:]:
        assert torch.equal(ids, ids0)
        torch.testing.assert_close(lp, lp0, rtol=0, atol=1e-5)


def test_n1_tau1_log_probs_are_minus_the_nll():
    V, K, N, P = 3001, 128, 700, 5
    Wt, Bt = _table(V, K, 8)
    fabs, groups = _groups(2, Wt, Bt, P)
    x = torch.randn(N, K, generator=torch.Generator().manual_seed(9)).bfloat16().cuda()
    for grp in groups:
        lp, ids = grp.full_softmax_sample(x, 1, 1.0, 7)
        nll = grp.full_softmax_nll(x, ids[:, 0])
        torch.testing.assert_close(-lp[:, 0].cpu(), nll.cpu(), rtol=0, atol=1e-4)
    for f in fabs:
        f.close()


def test_first_draws_follow_the_softmax():
    """V = 1000 over P = 7 partitions on W = 4 ranks: 200 000 copies of one input row."""
    V, K, N, tau = 1000, 32, 200000, 0.8
    Wt, Bt = _table(V, K, 21, scale=1.5)
    fabs, groups = _groups(4, Wt, Bt, 7, "div")
    xr = torch.randn(1, K, generator=torch.Generator().manual_seed(5)).bfloat16()
    x = xr.repeat(N, 1).cuda()
    p = torch.softmax((xr.double() @ Wt.double().t() + Bt.double().t())[0] * _inv(tau), 0).numpy()
    for grp in (groups[0], groups[3]):
        _, ids = grp.full_softmax_sample(x, 1, _inv(tau), 31 + grp.rank)
        cnt = np.bincount(ids[:, 0].cpu().numpy(), minlength=V)
        big = p * N >= 5
        obs = np.append(cnt[big], cnt[~big].sum())
        exp = np.append(p[big] * N, p[~big].sum() * N)
        assert stats.chisquare(obs, exp).pvalue > 1e-4
    for f in fabs:
        f.close()


@pytest.mark.parametrize("world,P,n", [(1, 1, 5), (2, 5, 32), (4, 7, 1)])
def test_sample_bf16_masters(world, P, n):
    """sparse_weights="bf16": bf16 bias master rows, widened to fp32 where they are added."""
    V, K, N, tau = 2999, 136, 300, 0.7
    Wt, Bt = _table(V, K, 12)
    fabs, groups = _groups(world, Wt, Bt + 0.5, P, weights="bf16")
    assert groups[0].tables[1].weight_dtype == torch.bfloat16
    x = torch.randn(N, K, generator=torch.Generator().manual_seed(13)).bfloat16()
    ref = _reference(x.float(), Wt, (Bt + 0.5).bfloat16().float(), tau, 3)
    for grp in groups:
        lp, ids = grp.full_softmax_sample(x.cuda(), n, _inv(tau), 3)
        _check(lp, ids, ref, n, V)
    for f in fabs:
        f.close()


def test_sample_no_logits_buffer():
    """V = 200 000, N = 2560, n = 32: peak allocation grows by less than 64 MB."""
    V, K, N, n = 200000, 512, 2560, 32
    Wt, Bt = _table(V, K, 14)
    fabs, groups = _groups(1, Wt, Bt, 1)
    x = torch.randn(N, K, device="cuda").bfloat16()
    groups[0].full_softmax_sample(x, n, 1.0, 1)           # warm-up (module load, maps)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    lp, ids = groups[0].full_softmax_sample(x, n, 1.0, 2)
    torch.cuda.synchronize()
    growth = torch.cuda.max_memory_allocated() - base
    assert growth < 64 << 20, growth
    ref = _reference(x[:64].float().cpu(), Wt, Bt, 1.0, 2)
    _check(lp[:64], ids[:64], ref, n, V)
    for f in fabs:
        f.close()


def test_sample_argument_errors():
    import ctypes
    from parallax_b200 import consts, ops
    Wt, Bt = _table(100, 32, 1)
    fabs, groups = _groups(1, Wt, Bt, 1)
    grp = groups[0]
    x = torch.randn(4, 32, device="cuda").bfloat16()
    for n in (0, 33, True):
        with pytest.raises(ValueError, match="num_samples must be"):
            grp.full_softmax_sample(x, n, 1.0, 0)
    with pytest.raises(ValueError, match="bf16 inputs"):
        grp.full_softmax_sample(x.float(), 3, 1.0, 0)
    # the entry point's own codes: -3 for n outside [1, 32], -4 for inv_tau not finite and > 0
    L = ops.lib()
    x, K, _, head, tail, stream = grp._eval_operands(x, "test")
    _, part = grp._slot_maps()
    ctas = consts.NUM_SMS
    ws = torch.empty(ctas * 4 * 2, dtype=torch.float32, device="cuda")
    tk = torch.empty(ctas * 4 * 32 * 2, dtype=torch.int32, device="cuda")
    lp = torch.empty(4, 32, device="cuda")
    ids = torch.empty(4, 32, dtype=torch.int64, device="cuda")

    def call(n, inv_tau):
        return L.px_full_softmax_sample(
            ctypes.c_void_p(x.data_ptr()), 4, K, *head, ctypes.c_void_p(part.data_ptr()), *tail,
            ctypes.c_void_p(ws.data_ptr()), ctas, n, ctypes.c_void_p(tk.data_ptr()),
            ctypes.c_void_p(lp.data_ptr()), ctypes.c_void_p(ids.data_ptr()), inv_tau, 5, 0,
            stream)
    for n in (0, 33, -1):
        assert call(n, 1.0) == -3
    for inv_tau in (0.0, -1.0, float("inf"), float("nan")):
        assert call(4, inv_tau) == -4
    assert call(4, 1.0) == 0
    torch.cuda.synchronize()
    for f in fabs:
        f.close()


# ------------------------------------------------------------------ through the engine
def _count_sample(monkeypatch):
    """n of every call of NVSparseGroup.full_softmax_sample"""
    from parallax_b200.parallel.nv_sparse import NVSparseGroup
    calls = []
    orig = NVSparseGroup.full_softmax_sample
    monkeypatch.setattr(NVSparseGroup, "full_softmax_sample",
                        lambda self, x, n, t, s: calls.append(n) or orig(self, x, n, t, s))
    return calls


def test_sample_engine_eval_between_training_steps(monkeypatch):
    from parallax_b200.parallel.engine import (_gathered_logits, full_softmax_sample_composition,
                                               sample_log_e)
    calls = _count_sample(monkeypatch)
    sess = _lm1b_session()
    m = sess.engine.model
    m.eval_sample = 3
    grp = m.softmax_w.table.group
    x = torch.randn(256, 32, device="cuda").bfloat16()
    tau = 0.9
    for step in range(3):
        sess.run(["loss", "train_op"], _batch(step))
        n0 = len(calls)
        ctl0 = grp.ctl.clone()
        m.eval()
        try:
            ids_s = sess.run("sample_ids", {"x": _batch(99)["x"], "sample_seed": [step]})[0]
        finally:
            m.train()
        assert np.asarray(ids_s).shape == (128, 4, 3)
        with torch.no_grad():
            lp, ids = parallax.nn.full_softmax_sample(x, m.softmax_w, m.softmax_b, 5, tau, step)
            clp, cids = full_softmax_sample_composition(x, m.softmax_w, m.softmax_b, 5,
                                                        _inv(tau), step)
            # the composition's keys: its logits are rounded to bf16
            ckeys = _gathered_logits(x, m.softmax_w, m.softmax_b) * _inv(tau) - sample_log_e(
                step, torch.arange(256, device="cuda"), torch.arange(1003, device="cuda"))
        torch.cuda.synchronize()
        assert calls[n0:] == [3, 5]               # the session's eval and ours were fused
        assert torch.equal(grp.ctl, ctl0)         # eval leaves the step flags alone
        srt = torch.sort(ckeys, dim=1, descending=True).values[:, :6].cpu()
        d = srt[:, :-1] - srt[:, 1:]
        ok = d > 0.1
        ok[:, 1:] &= d[:, :-1] > 0.1
        ids, cids, lp, clp = ids.cpu(), cids.cpu(), lp.cpu(), clp.cpu()
        assert ok.any() and torch.equal(ids[ok], cids[ok])
        torch.testing.assert_close(lp[ids == cids], clp[ids == cids], rtol=0, atol=3e-2)
    sess.close()


def test_sample_grad_or_large_n_takes_the_composition(monkeypatch):
    calls = _count_sample(monkeypatch)
    sess = _lm1b_session()
    m = sess.engine.model
    sess.run(["loss", "train_op"], _batch(0))
    x = torch.randn(64, 32, device="cuda").bfloat16()
    lp, ids = parallax.nn.full_softmax_sample(x.requires_grad_(), m.softmax_w, m.softmax_b, 4)
    assert lp.requires_grad and calls == []
    with torch.no_grad():
        lp, ids = parallax.nn.full_softmax_sample(x, m.softmax_w, m.softmax_b, 33, 1.0, 1)
        assert ids.shape == (64, 33) and calls == []
        parallax.nn.full_softmax_sample(x, m.softmax_w, m.softmax_b, 32, 1.0, 1)
    assert calls == [32]
    sess.close()
