"""The full-softmax kernels (`ops/csrc/kernels/softmax_eval.cu`) at 512 < K <= 1024, where a work
item is a block of 64 table rows instead of 128: every pass against fp64 on exact operands
(`tests/full_softmax_ref.py`; at K <= 1024 every fine-row partial sum is a multiple of 2⁻⁸ below
2¹⁷, so the fp32 logits are still exact), LM1B's vocabulary at K = 1024, the choice between the
fused path and the composition at the width limit, and the engine's eval and training paths on an
LM1B output layer 1024 wide."""
import ctypes
import math

import numpy as np
import pytest
import torch

import parallax_b200 as parallax
from parallax_b200 import consts, ops
from parallax_b200.parallel.engine import sample_log_e
from parallax_b200.parallel.nv_sparse import full_softmax_block_rows
from tests import full_softmax_ref as R
from tests.test_gpu_full_softmax import _groups
from tests.test_gpu_full_softmax_lm1b import Problem, _bias_rows, _check_grad_chunk
from tests.test_gpu_full_softmax_sample_trunc import _threshold

pytestmark = pytest.mark.gpu

SEED = 77
WORST = {}


def _vp(t):
    return ctypes.c_void_p(t.data_ptr())


def _within(name, err, bound):
    """err <= 2·bound everywhere; records the worst err/(2·bound) under `name`"""
    r = float((err / (2 * bound)).max()) if err.numel() else 0.0
    WORST[name] = max(WORST.get(name, 0.0), r)
    assert r <= 1.0, (name, r)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst error/(2·bound):", {k: round(v, 4) for k, v in sorted(WORST.items())})


def _depth(grp):
    """(items per CTA, grid) of the kernels on `grp`: `R.lse_depth` with blocks of the height the
    kernels take at the group's K.  `R.lse_bound` counts 32 terms per lane; at 64-row blocks a lane
    sums 16, so the bound holds with room."""
    lay = grp.layout
    bv = full_softmax_block_rows(grp.tables[0].D)
    owners = 1 if lay.replicated else lay.world
    items = owners * -(-lay.parts_per_owner * lay.rows_per_part // bv)
    grid = min(items, consts.NUM_SMS)
    return -(-items // grid), grid


def _lse_b(grp, ref_lse, smax):
    per_cta, grid = _depth(grp)
    return R.lse_bound(ref_lse, smax, per_cta, grid)


def _grad_raw(x, Wc, bc, v0, lse, g, t, ctas, pad=64):
    """px_full_softmax_grad on one chunk with G and db guarded past what it may write: G
    [N, nblk·BV + pad] and db [rows + pad] start as NaN."""
    m, Kx = Wc.shape
    bv = full_softmax_block_rows(Kx)
    nblk = -(-m // bv)
    gp = nblk * bv + pad
    G = torch.full((x.shape[0], gp), float("nan"), dtype=torch.bfloat16, device="cuda")
    db = torch.full((m + pad,), float("nan"), dtype=torch.float32, device="cuda")
    rc = ops.lib().px_full_softmax_grad(
        _vp(x), x.shape[0], Kx, _vp(Wc), Wc.shape[1], _vp(bc), bc.shape[1],
        int(bc.dtype == torch.bfloat16), m, v0, _vp(lse), _vp(g), _vp(t), _vp(G), gp, _vp(db),
        ctas, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0
    torch.cuda.synchronize()
    assert G[:, nblk * bv:].isnan().all() and db[m:].isnan().all()     # the guards
    assert (G[:, m:nblk * bv] == 0).all()        # padding columns of the last block: zero
    return G[:, :m], db[:m]


def _check_nll_grad(grp, pr, x, t, g, chunk=None):
    """`full_softmax_nll_grad`'s dX, dW and db per element against fp64 (chunks of `chunk` rows,
    default `full_softmax_train_chunk`)"""
    N, K, V = x.shape[0], pr.K, pr.V
    nll, lse = grp.full_softmax_nll_lse(x, t)
    dx, dW, db = grp.full_softmax_nll_grad(x, t, lse, g, chunk=chunk)
    vc = chunk or grp.full_softmax_train_chunk(N)
    nch = -(-V // vc)
    xa = x.double().abs()
    smax = pr.ref["smax"]
    dx64 = torch.zeros(N, K, dtype=torch.float64, device="cuda")
    dxb = torch.zeros_like(dx64)
    for v0 in range(0, V, vc):
        m = min(vc, V - v0)
        s = x.double() @ pr.W[v0:v0 + m].double().t() + pr.b[v0:v0 + m, 0].double()[None, :]
        p = torch.exp(s - lse.double()[:, None])
        hot = (t[:, None] - v0) == torch.arange(m, device="cuda")[None, :]
        G64 = g.double()[:, None] * (p - hot.double())
        gb = R.grad_bound(p, g.double(), smax, lse.double())
        eG = gb + R.bf16_half_ulp(G64.abs() + gb)
        Wc = pr.W[v0:v0 + m].double()
        dx64 += G64 @ Wc
        dxb += eG @ Wc.abs() + (m + nch) * R.U * (G64.abs() @ Wc.abs())
        dW64 = G64.t() @ x.double()
        dWb = eG.t() @ xa + N * R.U * (G64.abs().t() @ xa)
        _within("dW", (dW[v0:v0 + m].double() - dW64).abs(),
                dWb + R.bf16_half_ulp(dW64.abs() + dWb))
        db64 = G64.sum(0)
        dbb = gb.sum(0) + (2 * -(-N // 128) + 11) * R.U * G64.abs().sum(0)
        _within("nll_grad db", (db[v0:v0 + m, 0].double() - db64).abs(),
                dbb + R.bf16_half_ulp(db64.abs() + dbb))
        del s, p, G64, gb, eG
    _within("dX", (dx.double() - dx64).abs(), dxb + R.bf16_half_ulp(dx64.abs() + dxb))


# ------------------------------------------------------------------ every pass against fp64
@pytest.fixture(scope="module", params=[520, 1000, 1024])
def wide(request):
    """K = 520 and 1000 leave a zero-filled tail in the last 64-column K-block"""
    pr = Problem(12007, request.param, 640, 31 + request.param)
    yield pr
    del pr
    torch.cuda.empty_cache()


# world, strategy, bias masters, replicated
WORLDS = [(1, "div", "fp32", False), (3, "mod", "bf16", False), (8, "div", "fp32", False),
          (8, "mod", "bf16", False), (3, "mod", "fp32", True)]


@pytest.mark.parametrize("W,strategy,weights,replicated", WORLDS,
                         ids=["W%d-%s-%s%s" % (w, s, b, "-repl" if r else "")
                              for w, s, b, r in WORLDS])
def test_every_pass_matches_fp64(wide, W, strategy, weights, replicated):
    pr, ref, x = wide, wide.ref, wide.xb()
    N = x.shape[0]
    assert full_softmax_block_rows(pr.K) == 64
    fabs, groups = _groups(W, pr.Wt, pr.Bt, 7, strategy, replicated, weights=weights)
    for grp in ([groups[0], groups[-1]] if W > 1 else groups):
        # NLL and lse
        nll, lse = grp.full_softmax_nll_lse(x, pr.t)
        b = _lse_b(grp, ref["lse"], ref["smax"])
        _within("lse", (lse.double() - ref["lse"]).abs(), b)
        nll_ref = ref["lse"] - pr.logit_t
        _within("nll", (nll.double() - nll_ref).abs(), b + R._ulp(nll_ref))
        # top-k: ids exactly, ties by ascending id
        for k in (1, 10, 32):
            lp, ids = grp.full_softmax_topk(x, k)
            assert torch.equal(ids, ref["top_i"][:, :k]), k
            lp_ref = ref["top_v"][:, :k] - ref["lse"][:, None]
            _within("topk log_probs", (lp.double() - lp_ref).abs(), b[:, None] + R._ulp(lp_ref))
        # sampling
        for tau in (0.5, 1.0):
            for n in (1, 10):
                lp, ids = grp.full_softmax_sample(x, n, R.inv_tau(tau), SEED)
                agree, ok = R.checked_draws(ids, ref["key_%g" % tau], ref["kid_%g" % tau],
                                            ref["loge_%g" % tau], n)
                assert agree and ok.float().mean() >= 0.99, (tau, n, float(ok.float().mean()))
                lp_ref = ref["ks_%g" % tau][:, :n] - ref["lse_%g" % tau][:, None]
                mg = R.draw_margin(ref["key_%g" % tau][:, :n], ref["loge_%g" % tau][:, :n])
                bt = _lse_b(grp, ref["lse_%g" % tau], ref["smax_%g" % tau])[:, None] + \
                    2 * mg + R._ulp(lp_ref)
                _within("sample log_probs", (lp.double() - lp_ref).abs()[ok], bt[ok])
        # truncated sampling: θ* of the count clause bit-exact, the nucleus outside its mass band
        for top_k in (40, 1000):
            th, tl = _threshold(grp, x, 1, 1.0, top_k=top_k)
            assert torch.equal(th.cuda().double(), ref["th_%d" % top_k]), top_k
            _within("trunc lse", (tl.cuda().double() - ref["lse"]).abs(), b)
        for n in (1, 10):
            lp, ids = grp.full_softmax_sample(x, n, 1.0, SEED, top_k=40)
            agree, ok = R.checked_draws(ids, ref["mkey_40"], ref["mkid_40"], ref["mloge_40"], n)
            assert agree and ok.float().mean() >= 0.99, n
        th, tl = _threshold(grp, x, 1, 1.0, top_p=0.9)
        dl = (tl.cuda().double() - ref["lse"]).abs()
        per_cta, grid = _depth(grp)
        depth = 32 + 4 + per_cta + math.ceil(grid / 2) + 1 + 4 + 8
        t = 4 * R.U + R.U * 3 * (ref["smax"] + ref["lse"].abs()) + \
            R.ETA * 2 * (ref["smax"] + ref["lse"].abs())
        mb = t + depth * R.U + 1.01 * dl
        band = ((ref["cum_p"] - 0.9).abs() <= 2 * mb) | ((ref["above_p"] - 0.9).abs() <= 2 * mb)
        assert band.float().mean() < 0.5
        assert torch.equal(th.cuda().double()[~band], ref["th_p"][~band])
        # nucleus draws (n = 1) against the fp64 keys restricted to s >= θ*, outside the band
        s = x.double() @ pr.W.double().t() + pr.b.double().t()
        loge = sample_log_e(SEED, torch.arange(N, device="cuda"),
                            torch.arange(pr.V, device="cuda")).double()
        keys = (s - loge).masked_fill(s < ref["th_p"][:, None], -math.inf)
        kv, ki = torch.sort(keys, dim=1, descending=True, stable=True)
        del s, keys
        lp, ids = grp.full_softmax_sample(x, 1, 1.0, SEED, top_p=0.9)
        agree, ok = R.checked_draws(ids[~band], kv[~band, :2], ki[~band, :2],
                                    loge.gather(1, ki[:, :2])[~band], 1)
        assert agree and ok.float().mean() >= 0.99
        del kv, ki, loge
    # the gradient: the group's chunked backward, and the raw kernel with guards
    grp = groups[-1]
    _check_nll_grad(grp, pr, x, pr.t, pr.g)
    _check_nll_grad(grp, pr, x, pr.t, pr.g, chunk=1000)    # chunks of 15 blocks and 40 rows
    bf = weights == "bf16"
    lse32 = ref["lse"].float()
    for v0, m in ((0, pr.V), (64 * 40, 64 * 33 + 5)):
        G, db = _grad_raw(x, pr.W[v0:v0 + m].contiguous(), _bias_rows(pr.b, v0, m, bf), v0,
                          lse32, pr.g, pr.t, consts.NUM_SMS)
        _check_grad_chunk("grad", G, db, x, pr.W, pr.b, v0, lse32, pr.g, pr.t, ref["smax"])
    for f in fabs:
        f.close()
    del groups, fabs
    torch.cuda.empty_cache()


# ------------------------------------------------------------------ LM1B's vocabulary at K = 1024
def test_lm1b_vocabulary_nll_and_gradient_chunks():
    """V = 793 470, K = 1024, 32 partitions, N = 2560: 12 398 blocks of 64 rows, so every CTA
    walks about 94 work items.  The NLL on one and on eight ranks, top-k ids where the coarse
    rows tie across the k-th position, and the gradient kernel over the default chunks of the
    backward (whole waves of 64-row blocks, the last one partial)."""
    V, K, P, N = R.V_LM1B, 1024, R.P_LM1B, 2560
    pr = Problem(V, K, N, 19, taus=(), trunc_k=())
    x = pr.xb()
    c = R.coarse_rows(N).cuda()
    for k in (10, 32):
        tie = pr.ref["top_v"][c, k - 1] == pr.ref["top_v"][c, k]
        assert tie.float().mean() >= 0.5, (k, float(tie.float().mean()))
    for W, strategy, weights in ((1, "div", "fp32"), (8, "mod", "bf16")):
        fabs, groups = _groups(W, pr.Wt, pr.Bt, P, strategy, weights=weights)
        for grp in ([groups[0], groups[-1]] if W > 1 else groups):
            per_cta, grid = _depth(grp)
            assert grid == consts.NUM_SMS and per_cta > 80
            for n in (N, 640):
                nll, lse = grp.full_softmax_nll_lse(pr.xb(n), pr.t[:n])
                b = _lse_b(grp, pr.ref["lse"][:n], pr.ref["smax"][:n])
                _within("lm1b lse", (lse.double() - pr.ref["lse"][:n]).abs(), b)
                nll_ref = pr.ref["lse"][:n] - pr.logit_t[:n]
                _within("lm1b nll", (nll.double() - nll_ref).abs(), b + R._ulp(nll_ref))
            for k in (10, 32):
                lp, ids = grp.full_softmax_topk(x, k)
                assert torch.equal(ids, pr.ref["top_i"][:, :k]), k
        if W == 1:
            vc = groups[0].full_softmax_train_chunk(N)
        for f in fabs:
            f.close()
        del groups, fabs
    assert vc % (64 * consts.NUM_SMS) == 0 and V % vc
    lse32 = pr.ref["lse"].float()
    for v0 in range(0, V, vc):
        m = min(vc, V - v0)
        G, db = _grad_raw(x, pr.W[v0:v0 + m].contiguous(), _bias_rows(pr.b, v0, m, True), v0,
                          lse32, pr.g, pr.t, consts.NUM_SMS)
        _check_grad_chunk("lm1b grad", G, db, x, pr.W, pr.b, v0, lse32, pr.g, pr.t,
                          pr.ref["smax"])
    del pr
    torch.cuda.empty_cache()


# ------------------------------------------------------------------ selection
def test_raw_entries_refuse_k_past_1024():
    L = ops.lib()
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    for K in (1032, 1028):
        assert L.px_full_softmax_nll(None, 4, K, None, K, None, 4, 0, None, 1, None, 0, None,
                                     None, 0, None, 1, None, None, None, None, None,
                                     stream) == -1, K
        assert L.px_full_softmax_topk(None, 4, K, None, K, None, 4, 0, None, None, 1, None, 0,
                                      None, None, 0, None, 1, 4, None, None, None,
                                      stream) == -1, K
        assert L.px_full_softmax_grad(None, 4, K, None, K, None, 4, 0, 64, 0, None, None, None,
                                      None, 64, None, 1, stream) == -1, K


def test_no_logits_buffer_at_1024():
    """V = 200 000, N = 2560, K = 1024: the fused call allocates only O(grid·N) scratch"""
    V, K, N = 200000, 1024, 2560
    g = torch.Generator().manual_seed(3)
    Wt = torch.randn(V, K, generator=g) * 0.03
    Bt = torch.randn(V, 1, generator=g) * 0.1
    fabs, groups = _groups(1, Wt, Bt, 1)
    x = torch.randn(N, K, device="cuda").bfloat16()
    targets = torch.randint(0, V, (N,), device="cuda")
    groups[0].full_softmax_nll(x, targets)             # warm-up (module load, row counts)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    nll = groups[0].full_softmax_nll(x, targets)
    torch.cuda.synchronize()
    growth = torch.cuda.max_memory_allocated() - base
    assert growth < 64 << 20, growth
    logits = x[:64].double() @ Wt.cuda().bfloat16().double().t() + Bt.cuda().double().t()
    ref = torch.nn.functional.cross_entropy(logits, targets[:64], reduction="none")
    torch.testing.assert_close(nll[:64].double(), ref, rtol=1e-5, atol=1e-3)
    for f in fabs:
        f.close()


# ------------------------------------------------------------------ through the engine
def _session(K, num_sampled=16, **sc):
    from parallax_b200.models.lm1b import LM1B, lm1b_graph
    torch.manual_seed(0)
    m = LM1B(vocab_size=1003, emb_size=K, state_size=64, projected_size=K,
             num_sampled=num_sampled, num_steps=4, num_shards=3, keep_prob=1.0)
    sc = dict({"fabric": "nvlink", "compute_dtype": "bf16"}, **sc)
    sess, *_ = parallax.parallel_run(lm1b_graph(m, batch_size=128), "localhost:0",
                                     parallax_config=parallax.Config(sess_config=sc))
    return sess


def _batch(seed, V=1003):
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(0, V, (128, 4), generator=g)
    return {"x": [x], "y": [torch.roll(x, -1, dims=1)]}


def _count(monkeypatch, method):
    from parallax_b200.parallel.nv_sparse import NVSparseGroup
    calls = []
    orig = getattr(NVSparseGroup, method)

    def counted(self, *a, **k):
        calls.append(a[1] if len(a) > 1 else None)
        return orig(self, *a, **k)
    monkeypatch.setattr(NVSparseGroup, method, counted)
    return calls


@pytest.mark.parametrize("K,fused", [(1024, True), (1032, False)])
def test_engine_eval_at_the_width_limit(monkeypatch, K, fused):
    """eval NLL, top-k and sampling through `parallax.nn` on an LM1B output layer K wide: fused
    at K = 1024 and in agreement with the composition; the composition at K = 1032"""
    from parallax_b200.parallel.engine import (_gathered_logits, full_softmax_composition,
                                               full_softmax_sample_composition,
                                               full_softmax_topk_composition)
    nll_calls = _count(monkeypatch, "full_softmax_nll")
    topk_calls = _count(monkeypatch, "full_softmax_topk")
    smp_calls = _count(monkeypatch, "full_softmax_sample")
    sess = _session(K)
    m = sess.engine.model
    w, b = m.softmax_w, m.softmax_b
    assert w.embedding_dim == K
    for step in range(2):
        sess.run(["loss", "train_op"], _batch(step))
    g = torch.Generator(device="cuda").manual_seed(K)
    x = torch.randn(256, K, device="cuda", generator=g).bfloat16()
    t = torch.randint(0, 1003, (256,), device="cuda", generator=g)
    with torch.no_grad():
        nll = parallax.nn.full_softmax_nll(x, t, w, b)
        cnll = full_softmax_composition(x, t, w, b)
        lp, ids = parallax.nn.full_softmax_topk(x, w, b, 5)
        clp, cids = full_softmax_topk_composition(x, w, b, 6)
        slp, sids = parallax.nn.full_softmax_sample(x, w, b, 5, 0.9, 7)
        sclp, scids = full_softmax_sample_composition(x, w, b, 5, R.inv_tau(0.9), 7)
        ckeys = _gathered_logits(x, w, b) * R.inv_tau(0.9) - sample_log_e(
            7, torch.arange(256, device="cuda"), torch.arange(1003, device="cuda"))
    torch.cuda.synchronize()
    n_fused = (len(nll_calls), len(topk_calls), len(smp_calls))
    assert n_fused == ((1, 1, 1) if fused else (0, 0, 0)), n_fused
    torch.testing.assert_close(nll.cpu(), cnll.cpu(), rtol=0, atol=3e-2)
    lp, ids, clp, cids = lp.cpu(), ids.cpu(), clp.cpu(), cids.cpu()
    torch.testing.assert_close(lp, clp[:, :5], rtol=0, atol=3e-2)
    d = clp[:, :-1] - clp[:, 1:]
    ok = d > 0.1
    ok[:, 1:] &= d[:, :-1] > 0.1
    assert ok.any() and torch.equal(ids[ok], cids[:, :5][ok])
    srt = torch.sort(ckeys, dim=1, descending=True).values[:, :6].cpu()
    d = srt[:, :-1] - srt[:, 1:]
    ok = d > 0.1
    ok[:, 1:] &= d[:, :-1] > 0.1
    sids, scids, slp, sclp = sids.cpu(), scids.cpu(), slp.cpu(), sclp.cpu()
    assert ok.any() and torch.equal(sids[ok], scids[ok])
    torch.testing.assert_close(slp[sids == scids], sclp[sids == scids], rtol=0, atol=3e-2)
    if fused:
        # the session's own eval outputs take the fused kernels as well
        m.eval_top_k, m.eval_sample = 5, 3
        m.eval()
        try:
            loss, top, smp = sess.run(["loss", "top_k_ids", "sample_ids"],
                                      dict(_batch(99), sample_seed=[1]))
        finally:
            m.train()
        assert np.isfinite(float(loss[0]))
        assert np.asarray(top[0]).shape == (128, 4, 5) and np.asarray(smp[0]).shape == (128, 4, 3)
        assert len(nll_calls) == 2 and topk_calls[-1] == 5 and smp_calls[-1] == 3
    sess.close()


_ROWS = torch.randperm(1003, generator=torch.Generator().manual_seed(5))[:64]


def _train(monkeypatch, setting, steps):
    from parallax_b200.parallel.nv_sparse import NVSparseGroup
    calls = {"fused": 0}
    orig = NVSparseGroup.full_softmax_nll_lse

    def counted(*a, **k):
        calls["fused"] += 1
        return orig(*a, **k)
    monkeypatch.setattr(NVSparseGroup, "full_softmax_nll_lse", counted)
    sess = _session(1024, 0, full_softmax_train=setting, cuda_graph=True, graph_warmup=2)
    m = sess.engine.model

    def state():
        torch.cuda.synchronize()
        w = m.softmax_w.table.full_weight()[_ROWS].float().cpu()
        b = m.softmax_b.table.full_weight()[_ROWS].float().cpu()
        return [w, b] + [p.detach().float().cpu().clone() for p in (m.W, m.B, m.W_P)]
    s0 = state()
    losses = [float(sess.run(["loss", "train_op"], _batch(i % 3))[0][0]) for i in range(steps)]
    s1 = state()
    captured = bool(sess.engine.graph_captured)
    sess.close()
    return losses, s0, s1, calls["fused"], captured


def test_engine_fused_training_at_1024_matches_composition(monkeypatch):
    """`full_softmax_train="fused"` steps under CUDA-graph capture against `"composition"` steps
    on the same seeded batches, LM1B's output layer 1024 wide"""
    c_losses, c0, c1, c_calls, _ = _train(monkeypatch, "composition", 5)
    f_losses, f0, f1, f_calls, captured = _train(monkeypatch, "fused", 5)
    assert c_calls == 0 and captured and f_calls == 2 + 1   # warm-up steps and the capture
    assert np.isfinite(f_losses).all() and f_losses[-1] < f_losses[0]
    np.testing.assert_allclose(f_losses, c_losses, rtol=0, atol=3e-2)
    for a0, a1, b0, b1 in zip(f0, f1, c0, c1):
        assert torch.equal(a0, b0)
        du, dc = a1 - a0, b1 - b0
        assert dc.norm() > 0
        assert float((du - dc).norm() / dc.norm()) < 0.1


# ------------------------------------------------------------------ the example scripts
_COUNTED = """
import runpy, sys
sys.path.insert(0, sys.argv[1])
from parallax_b200.parallel.nv_sparse import NVSparseGroup
n = [0]
for name in ("full_softmax_nll", "full_softmax_sample"):
    def wrap(self, *a, _o=getattr(NVSparseGroup, name), **k):
        n[0] += 1
        return _o(self, *a, **k)
    setattr(NVSparseGroup, name, wrap)
sys.argv = sys.argv[2:]
runpy.run_path(sys.argv[0], run_name="__main__")
print("fused calls %d" % n[0])
"""


def test_eval_and_generate_a_1024_wide_checkpoint(tmp_path):
    """the driver trains `--hpconfig projected_size=1024`; `lm1b_eval.py` and `lm1b_generate.py`
    restore the checkpoint with the same `--hpconfig` and run through the fused kernels"""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = {k: v for k, v in os.environ.items()
           if not k.startswith("PARALLAX_") and k not in ("RANK", "WORLD_SIZE", "LOCAL_RANK")}
    ck = str(tmp_path / "ck")
    hp = ["--use_synthetic", "--tiny", "--hpconfig", "projected_size=1024",
          "--compute_dtype", "bf16"]

    def run(script, args):
        r = subprocess.run([sys.executable, "-c", _COUNTED, root,
                            os.path.join(root, "examples/lm1b", script)] + hp + args,
                           env=env, cwd=str(tmp_path), capture_output=True, text=True,
                           timeout=600)
        assert r.returncode == 0, r.stderr[-2000:]
        return r.stdout
    run("lm1b_distributed_driver.py", ["--max_steps", "3", "--ckpt_dir", ck,
                                       "--save_ckpt_steps", "3", "--logdir",
                                       str(tmp_path / "log")])
    out = run("lm1b_eval.py", ["--ckpt_dir", ck, "--max_batches", "2"])
    assert "perplexity" in out and int(out.split("fused calls ")[1].split()[0]) == 2
    out = run("lm1b_generate.py", ["--ckpt_dir", ck, "--prefix", "5 17", "--num_words", "3",
                                   "--num_sequences", "2"])
    assert int(out.split("fused calls ")[1].split()[0]) == 3
    assert all(l.split()[:2] == ["5", "17"] for l in out.strip().splitlines()[-3:-1])
