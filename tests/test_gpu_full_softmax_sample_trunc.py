"""Truncated full-softmax sampling on the GPU (`parallax.nn.full_softmax_sample(..., top_k=,
top_p=)`; `px_full_softmax_sample_lse`, `px_full_softmax_radix` and
`px_full_softmax_sample_masked` in `ops/csrc/kernels/softmax_eval.cu`): the kernels' threshold θ*
against fp64 on worlds simulated inside one GPU, the draws against the composition and across
worlds, partitionings, layouts and row chunks, and the engine's dispatch on the NVLink fabric."""
import ctypes

import numpy as np
import pytest
import torch
from scipy import stats

import parallax_b200 as parallax
from parallax_b200 import consts, ops
from parallax_b200.parallel.engine import full_softmax_sample_composition
from tests.test_gpu_full_softmax import (CASES, _batch, _groups, _lm1b_session, _owners,
                                         _table)

pytestmark = pytest.mark.gpu


def _inv(tau):
    return float(torch.tensor(1.0 / tau, dtype=torch.float32))


def _vp(t):
    return ctypes.c_void_p(t.data_ptr())


def _key_to_float(key):
    """fp32 [N] of the order-preserving uint32 keys `key` (int32 [N] bits)"""
    u = key.to(torch.int64) & 0xffffffff
    bits = torch.where(u >= 1 << 31, u ^ (1 << 31), ~u & 0xffffffff)
    return bits.to(torch.int32).view(torch.float32)


def _threshold(grp, x, n, inv_tau, top_k=None, top_p=None):
    """(θ* fp32 [N], lse fp32 [N]) of the kernels: the log-sum-exp pass and every radix pass"""
    L = ops.lib()
    x, K, _, head, tail, stream = grp._eval_operands(x, "test")
    N, ctas, d = int(x.shape[0]), consts.NUM_SMS, consts.SAMPLE_RADIX_BITS
    ws = torch.empty(ctas * N * 2, dtype=torch.float32, device="cuda")
    hist = torch.empty(ctas * N * (1 << d) * 2, dtype=torch.int32, device="cuda")
    rows = torch.empty(N, 4, dtype=torch.int32, device="cuda")
    common = (_vp(x), N, K, *head, *tail)
    assert L.px_full_softmax_sample_lse(*common, _vp(ws), ctas, inv_tau, _vp(rows), stream) == 0
    for lo in range(32 - d, -1, -d):
        assert L.px_full_softmax_radix(*common, _vp(hist), ctas, inv_tau, _vp(rows), lo,
                                       top_k or 0, top_p or 0.0, n, stream) == 0
    torch.cuda.synchronize()
    rows = rows.cpu()
    return _key_to_float(rows[:, 0]), rows[:, 3].contiguous().view(torch.float32)


def _check_threshold(th, lse, s, n, top_k, top_p, min_checked=0.6):
    """θ* against the fp64 definition over fp64 scaled logits s [N, V].  Rows whose fp64 θ* has
    a neighbouring value within 1e-4 (relative), or whose cumulative mass at it or the value
    above lies within 1e-5 of p, are excluded and counted; on the others θ* is the fp64 θ*
    within 3e-5, top_k's chosen set has exactly the fp64 count, and top_p's chosen set reaches
    p − 1e-5 while the set without its lowest value does not.  (The band around p is 1e-5, not
    wider: at V ≈ 3000 the words at the nucleus' edge have masses near 1e-4 each, and the
    kernels' fp32 masses are within about 1e-6.)"""
    N, V = s.shape
    torch.testing.assert_close(lse.double(), torch.logsumexp(s, 1), rtol=0, atol=1e-4)
    vals, order = torch.sort(s, dim=1, descending=True)
    q = torch.softmax(s, 1).gather(1, order)
    cum = torch.cumsum(q, 1)
    cnt = torch.arange(1, V + 1).expand(N, V)
    ok = torch.zeros(N, V, dtype=torch.bool)
    if top_k is not None:
        ok |= cnt >= top_k
    if top_p is not None:
        ok |= (cum >= top_p) & (cnt >= n)
    j = torch.where(ok.any(1), ok.int().argmax(1), V - 1)
    th64 = vals.gather(1, j[:, None])[:, 0]
    tol = 1e-4 * (1 + th64.abs())
    pad = torch.full((N, 1), float("inf"), dtype=torch.float64)
    up = torch.cat([pad, vals], 1).gather(1, j[:, None])[:, 0] - th64
    down = th64 - torch.cat([vals, -pad], 1).gather(1, (j + 1)[:, None])[:, 0]
    clear = (up > tol) & (down > tol)
    if top_p is not None:
        near = (cum - top_p).abs() < 1e-5
        clear &= ~near.gather(1, j[:, None])[:, 0]
        clear &= ~near.gather(1, (j - 1).clamp(min=0)[:, None])[:, 0]
    assert clear.float().mean() >= min_checked, (int(clear.sum()), N)
    th = th.double()
    assert (th[clear] - th64[clear]).abs().le(0.3 * tol[clear]).all()
    chosen = s >= (th - 0.3 * tol)[:, None]
    size = chosen.sum(1)
    assert (size[clear] == (j + 1)[clear]).all()
    if top_k is not None and top_p is None:
        assert (size[clear] == top_k).all()
    if top_p is not None and top_k is None:
        mass = (torch.softmax(s, 1) * chosen).sum(1)
        low = torch.softmax(s, 1).gather(1, order).gather(1, j[:, None])[:, 0]
        big = size > n
        assert (mass[clear] >= top_p - 1e-5).all()
        assert (mass - low)[clear & big].lt(top_p + 1e-5).all()
    return int((~clear).sum())


MODES = [(1, 40, None), (1, None, 0.9), (3, None, 0.5), (2, 40, 0.9), (12, 40, 0.9)]


@pytest.mark.parametrize("n,top_k,top_p", MODES)
@pytest.mark.parametrize("world,V,P,strategy,K,N,replicated", CASES)
def test_threshold_matches_fp64(world, V, P, strategy, K, N, replicated, n, top_k, top_p):
    Wt, Bt = _table(V, K, world * 10 + P)
    fabs, groups = _groups(world, Wt, Bt, P, strategy, replicated, _owners(world, P, replicated))
    x = torch.randn(N, K, generator=torch.Generator().manual_seed(world * 100 + K)).bfloat16()
    inv = _inv(0.8)
    s = (x.double() @ Wt.double().t() + Bt.double().t()) * inv
    for grp in groups:                    # every rank evaluates its batch alone
        th, lse = _threshold(grp, x.cuda(), n, inv, top_k, top_p)
        _check_threshold(th, lse, s, n, top_k, top_p, min_checked=0.5 if N > 1 else 0.0)
    for f in fabs:
        f.close()


@pytest.mark.parametrize("n,top_k,top_p", MODES)
def test_threshold_large_logits_and_bf16_masters(n, top_k, top_p):
    """logits near ±80 (the masses of the tail underflow) with bf16 bias master rows"""
    V, K, N = 4097, 64, 300
    Wt, Bt = _table(V, K, 7, scale=8.0)
    fabs, groups = _groups(2, Wt, Bt + 0.5, 4, weights="bf16")
    x = (torch.randn(N, K, generator=torch.Generator().manual_seed(1)) * 2.0).bfloat16()
    s = x.double() @ Wt.double().t() + (Bt + 0.5).bfloat16().double().t()
    assert 60 < float(s.abs().max()) < 120
    for grp in groups:
        th, lse = _threshold(grp, x.cuda(), n, 1.0, top_k, top_p)
        _check_threshold(th, lse, s, n, top_k, top_p, min_checked=0.5)
    for f in fabs:
        f.close()


# ------------------------------------------------------------------ draws
def _embeddings(Wt, Bt):
    w, b = torch.nn.Embedding(*Wt.shape), torch.nn.Embedding(*Bt.shape)
    with torch.no_grad():
        w.weight.copy_(Wt)
        b.weight.copy_(Bt)
    return w, b


@pytest.mark.parametrize("top_k,top_p", [(50, None), (None, 0.9), (30, 0.8)])
def test_draws_match_the_composition_across_worlds_layouts_and_chunks(monkeypatch, top_k,
                                                                       top_p):
    V, K, N, n, tau = 3001, 64, 700, 4, 0.9
    Wt, Bt = _table(V, K, 3)
    x = torch.randn(N, K, generator=torch.Generator().manual_seed(4)).bfloat16()
    draws = []
    for world, P, strategy, replicated in [(1, 1, "mod", False), (2, 5, "mod", False),
                                           (4, 7, "div", False), (8, 32, "mod", False),
                                           (4, 1, "mod", True)]:
        fabs, groups = _groups(world, Wt, Bt, P, strategy, replicated,
                               _owners(world, P, replicated))
        for grp in groups:
            draws.append(grp.full_softmax_sample(x.cuda(), n, _inv(tau), 42, top_k=top_k,
                                                 top_p=top_p))
        if world == 2:                    # uneven row chunks: 128 rows per launch
            monkeypatch.setattr(consts, "TOPK_WS_BYTES", 1 << 20)
            draws.append(groups[1].full_softmax_sample(x.cuda(), n, _inv(tau), 42, top_k=top_k,
                                                       top_p=top_p))
            monkeypatch.undo()
        for f in fabs:
            f.close()
    lp0, ids0 = draws[0]
    for lp, ids in draws[1:]:
        assert torch.equal(ids, ids0)
        torch.testing.assert_close(lp, lp0, rtol=0, atol=1e-5)
    # the composition on the same fp32 logits: the same ids except where a key or the
    # threshold lies within a few ulp of another value
    w, b = _embeddings(Wt, Bt)
    clp, cids = full_softmax_sample_composition(x.float(), w, b, n, _inv(tau), 42, top_k, top_p)
    ids0, lp0 = ids0.cpu(), lp0.cpu()
    same = (ids0 == cids).all(1)
    assert same.float().mean() >= 0.98, int((~same).sum())
    torch.testing.assert_close(lp0[same], clp[same], rtol=0, atol=1e-4)


def test_top_k_v_is_the_untruncated_sample_bit_for_bit():
    V, K, N = 3001, 136, 640
    Wt, Bt = _table(V, K, 8)
    fabs, groups = _groups(4, Wt, Bt, 7, "div")
    x = torch.randn(N, K, generator=torch.Generator().manual_seed(9)).bfloat16().cuda()
    for grp in (groups[0], groups[3]):
        for n in (1, 12, 32):                # list capacities 8, 16 and 32
            lp, ids = grp.full_softmax_sample(x, n, _inv(0.7), 11, top_k=V)
            lp0, ids0 = grp.full_softmax_sample(x, n, _inv(0.7), 11)
            assert torch.equal(ids, ids0) and torch.equal(lp, lp0)
    for f in fabs:
        f.close()


def test_first_draws_follow_the_truncated_softmax():
    """V = 1000 over P = 7 partitions on W = 4 ranks: 200 000 copies of one input row, top_p =
    0.9 with the kernels' θ*."""
    V, K, N, tau, p = 1000, 32, 200000, 0.8, 0.9
    Wt, Bt = _table(V, K, 21, scale=1.5)
    fabs, groups = _groups(4, Wt, Bt, 7, "div")
    xr = torch.randn(1, K, generator=torch.Generator().manual_seed(5)).bfloat16()
    s = (xr.double() @ Wt.double().t() + Bt.double().t())[0] * _inv(tau)
    for grp in (groups[0], groups[3]):
        th, _ = _threshold(grp, xr.cuda(), 1, _inv(tau), top_p=p)
        keep = (s >= float(th[0]) - 1e-5 * (1 + abs(float(th[0])))).numpy()
        q = torch.softmax(s, 0).numpy() * keep
        assert 0.9 - 1e-5 <= q.sum() and keep.sum() < V
        q /= q.sum()
        _, ids = grp.full_softmax_sample(xr.repeat(N, 1).cuda(), 1, _inv(tau), 31 + grp.rank,
                                         top_p=p)
        cnt = np.bincount(ids[:, 0].cpu().numpy(), minlength=V)
        assert cnt[~keep].sum() == 0
        big = keep & (q * N >= 5)
        obs = np.append(cnt[big], cnt[keep & ~big].sum())
        exp = np.append(q[big] * N, q[keep & ~big].sum() * N)
        ok = exp > 0
        assert stats.chisquare(obs[ok], exp[ok]).pvalue > 1e-4
    for f in fabs:
        f.close()


def test_truncated_sample_no_logits_buffer():
    """V = 200 000, N = 2560, n = 32, top_k = 40 and top_p = 0.95: peak allocation grows by
    less than 64 MB (the digit bins reuse the lists' memory)."""
    V, K, N, n = 200000, 512, 2560, 32
    Wt, Bt = _table(V, K, 14)
    fabs, groups = _groups(1, Wt, Bt, 1)
    x = torch.randn(N, K, device="cuda").bfloat16()
    groups[0].full_softmax_sample(x, n, 1.0, 1, top_k=40, top_p=0.95)      # warm-up
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    lp, ids = groups[0].full_softmax_sample(x, n, 1.0, 2, top_k=40, top_p=0.95)
    torch.cuda.synchronize()
    growth = torch.cuda.max_memory_allocated() - base
    assert growth < 64 << 20, growth
    ids = ids.cpu()
    assert all(len(set(r)) == n for r in ids[:64].tolist())
    # every draw is among the row's 40 best logits (up to ties within the kernels' rounding)
    s = x[:64].float().cpu().double() @ Wt.double().t() + Bt.double().t()
    kth = torch.topk(s, 40, dim=1).values[:, -1:]
    assert (s.gather(1, ids[:64]) >= kth - 1e-3).all()
    for f in fabs:
        f.close()


# ------------------------------------------------------------------ codes and dispatch
def test_truncated_argument_errors():
    Wt, Bt = _table(100, 32, 1)
    fabs, groups = _groups(1, Wt, Bt, 1)
    grp = groups[0]
    x = torch.randn(4, 32, device="cuda").bfloat16()
    for k in (0, 101, True, 2.0):
        with pytest.raises(ValueError, match="top_k must be"):
            grp.full_softmax_sample(x, 1, 1.0, 0, top_k=k)
    with pytest.raises(ValueError, match="top_k must be"):
        grp.full_softmax_sample(x, 5, 1.0, 0, top_k=4)
    for p in (0.0, 1.5, True, "0.5"):
        with pytest.raises(ValueError, match="top_p must be"):
            grp.full_softmax_sample(x, 1, 1.0, 0, top_p=p)
    L = ops.lib()
    x, K, _, head, tail, stream = grp._eval_operands(x, "test")
    _, part = grp._slot_maps()
    ctas = consts.NUM_SMS
    ws = torch.empty(ctas * 4 * 2, dtype=torch.float32, device="cuda")
    hist = torch.empty(ctas * 4 * 32 * 2, dtype=torch.int32, device="cuda")
    rows = torch.empty(4, 4, dtype=torch.int32, device="cuda")
    lp = torch.empty(4, 32, device="cuda")
    ids = torch.empty(4, 32, dtype=torch.int64, device="cuda")
    common = (_vp(x), 4, K, *head, *tail)

    def lse(inv_tau):
        return L.px_full_softmax_sample_lse(*common, _vp(ws), ctas, inv_tau, _vp(rows), stream)

    def radix(lo=0, k=0, p=0.5, n=1, inv_tau=1.0):
        return L.px_full_softmax_radix(*common, _vp(hist), ctas, inv_tau, _vp(rows), lo, k, p, n,
                                       stream)

    def masked(n, inv_tau=1.0):
        return L.px_full_softmax_sample_masked(
            _vp(x), 4, K, *head, _vp(part), *tail, _vp(ws), ctas, n, _vp(hist), _vp(lp),
            _vp(ids), inv_tau, 5, 0, _vp(rows), stream)
    for inv_tau in (0.0, -1.0, float("inf"), float("nan")):
        assert lse(inv_tau) == -4 and radix(inv_tau=inv_tau) == -4 and masked(2, inv_tau) == -4
    for lo in (-4, 2, 32, 30):
        assert radix(lo=lo) == -2
    for n in (0, 33):
        assert radix(n=n) == -3 and masked(n) == -3
    for k in (-1, 3, 101):
        assert radix(k=k, n=4) == -5
    for p in (-0.1, 1.01, float("nan"), float("inf")):
        assert radix(p=p) == -6
    assert lse(1.0) == 0
    for lo in range(28, -1, -4):
        assert radix(lo=lo, k=10, p=0.5, n=4) == 0
    assert masked(4) == 0
    torch.cuda.synchronize()
    for f in fabs:
        f.close()


def _count_sample(monkeypatch):
    """(n, top_k, top_p) of every call of NVSparseGroup.full_softmax_sample"""
    from parallax_b200.parallel.nv_sparse import NVSparseGroup
    calls = []
    orig = NVSparseGroup.full_softmax_sample

    def rec(self, x, n, t, s, top_k=None, top_p=None):
        calls.append((n, top_k, top_p))
        return orig(self, x, n, t, s, top_k=top_k, top_p=top_p)
    monkeypatch.setattr(NVSparseGroup, "full_softmax_sample", rec)
    return calls


def test_truncated_engine_dispatch(monkeypatch):
    calls = _count_sample(monkeypatch)
    sess = _lm1b_session()
    m = sess.engine.model
    sess.run(["loss", "train_op"], _batch(0))
    w, b = m.softmax_w, m.softmax_b
    x = torch.randn(64, 32, device="cuda").bfloat16()
    with torch.no_grad():
        lp, ids = parallax.nn.full_softmax_sample(x, w, b, 4, 0.9, 3, top_k=20, top_p=0.8)
        parallax.nn.full_softmax_sample(x, w, b, 2, 1.0, 3, top_p=1.0)    # no nucleus
        parallax.nn.full_softmax_sample(x, w, b, 33, 1.0, 3, top_k=40)    # n > 32
        clp, cids = full_softmax_sample_composition(x.float(), w, b, 4, _inv(0.9), 3, 20, 0.8)
    assert calls == [(4, 20, 0.8), (2, None, None)]
    assert (ids.cpu() == cids.cpu()).all(1).float().mean() >= 0.9
    lp, _ = parallax.nn.full_softmax_sample(x.requires_grad_(), w, b, 4, 0.9, 3, top_k=20)
    assert lp.requires_grad and len(calls) == 2           # gradients: the composition
    sess.close()
