"""The full-softmax kernels (`ops/csrc/kernels/softmax_eval.cu`) against fp64 at LM1B's geometry
(V = 793 470, K = 512, 32 partitions), where every CTA of the persistent grid walks dozens of
work items, and over launch grids, row counts and K at a moderate V.  The operands are exact
(`tests/full_softmax_ref.py`), so the logits are exact and every id the kernels return is
compared with the reference on every row, ties included; the floating-point results are held
to bounds derived from the kernels' operation order, with a factor 2 to spare.  The worst
error/(2·bound) of each quantity is printed."""
import ctypes
import math

import pytest
import torch

from parallax_b200 import consts, ops
from tests import full_softmax_ref as R
from tests.test_gpu_full_softmax import _groups
from tests.test_gpu_full_softmax_sample_trunc import _threshold

pytestmark = pytest.mark.gpu

V, K, P, N = R.V_LM1B, R.K_LM1B, R.P_LM1B, 2560
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
    print("peak allocated: %.1f GB" % (torch.cuda.max_memory_allocated() / 2 ** 30))


class Problem(object):
    """exact table (CPU, fp32) and inputs, targets, gradients and the fp64 reference (device)"""

    def __init__(self, V, K, N, seed, taus=(0.5, 1.0), trunc_k=(40, 1000)):
        self.V, self.K, self.N = V, K, N
        self.Wt, self.Bt = R.exact_table(V, K, seed)
        self.x = R.exact_inputs(N, K, seed + 1).cuda()
        g = torch.Generator().manual_seed(seed + 2)
        t = torch.randint(0, V, (N,), generator=g)
        t[0], t[-1] = 0, V - 1
        self.t = t.cuda()
        gr = torch.rand(N, generator=g) * 2 - 0.5
        gr[N // 2] = 0.0
        self.g = gr.cuda()
        W, b = self.Wt.cuda(), self.Bt.cuda()
        self.ref = R.reference(self.x, W, b, taus=taus, seed=SEED, trunc_k=trunc_k)
        self.logit_t = (self.x.double() * W[self.t].double()).sum(1) + b[self.t, 0].double()
        self.W, self.b = W.bfloat16(), b

    def xb(self, n=None):
        return self.x[:n].bfloat16()


@pytest.fixture(scope="module")
def lm1b():
    pr = Problem(V, K, N, 11)
    yield pr
    del pr
    torch.cuda.empty_cache()


GEOMS = [(1, "div", "fp32"), (3, "mod", "fp32"), (3, "div", "bf16"), (8, "mod", "bf16"),
         (8, "div", "fp32")]


@pytest.fixture(scope="module", params=GEOMS, ids=["W%d-%s-%s" % g for g in GEOMS])
def world(request, lm1b):
    W, strategy, weights = request.param
    fabs, groups = _groups(W, lm1b.Wt, lm1b.Bt, P, strategy, weights=weights)
    yield [groups[0], groups[-1]] if W > 1 else groups
    for f in fabs:
        f.close()
    del groups, fabs
    torch.cuda.empty_cache()


def _lse_b(grp, ref_lse, smax):
    """the log-sum-exp bound of rows with fp64 lse `ref_lse` and max |s| `smax` on `grp`'s grid"""
    per_cta, grid = R.lse_depth(grp)
    return R.lse_bound(ref_lse, smax, per_cta, grid)


def _lse_check(name, grp, lse, ref_lse, smax):
    b = _lse_b(grp, ref_lse, smax)
    _within(name, (lse.double() - ref_lse).abs(), b)
    return b


# ------------------------------------------------------------------ LM1B geometry
def test_lm1b_nll_and_lse(world, lm1b):
    ref = lm1b.ref
    for grp in world:
        per_cta, grid = R.lse_depth(grp)
        assert grid == consts.NUM_SMS and per_cta > 40      # every CTA walks many items
        for n in (N, 640):
            nll, lse = grp.full_softmax_nll_lse(lm1b.xb(n), lm1b.t[:n])
            b = _lse_check("lse", grp, lse, ref["lse"][:n], ref["smax"][:n])
            nll_ref = ref["lse"][:n] - lm1b.logit_t[:n]
            _within("nll", (nll.double() - nll_ref).abs(), b + R._ulp(nll_ref))


def test_lm1b_topk_ids_exact(world, lm1b):
    ref = lm1b.ref
    x = lm1b.xb()
    for grp in world:
        for k in (1, 8, 9, 16, 17, 32):
            lp, ids = grp.full_softmax_topk(x, k)
            assert torch.equal(ids, ref["top_i"][:, :k]), k
            lp_ref = ref["top_v"][:, :k] - ref["lse"][:, None]
            b = _lse_b(grp, ref["lse"], ref["smax"])[:, None] + R._ulp(lp_ref)
            _within("topk log_probs", (lp.double() - lp_ref).abs(), b)
    # the coarse rows put a tie across the k-th position in most rows
    c = R.coarse_rows(N).cuda()
    for k in (8, 16, 32):
        tie = ref["top_v"][c, k - 1] == ref["top_v"][c, k]
        assert tie.float().mean() >= 0.5, (k, float(tie.float().mean()))


def test_lm1b_sample_draws(world, lm1b):
    ref = lm1b.ref
    x = lm1b.xb()
    for grp in world:
        for tau in (0.5, 1.0):
            for n in (1, 12, 32):
                lp, ids = grp.full_softmax_sample(x, n, R.inv_tau(tau), SEED)
                agree, ok = R.checked_draws(ids, ref["key_%g" % tau], ref["kid_%g" % tau],
                                            ref["loge_%g" % tau], n)
                assert agree, (tau, n)
                assert ok.float().mean() >= 0.99, (tau, n, float(ok.float().mean()))
                lp_ref = ref["ks_%g" % tau][:, :n] - ref["lse_%g" % tau][:, None]
                mg = R.draw_margin(ref["key_%g" % tau][:, :n], ref["loge_%g" % tau][:, :n])
                b = _lse_b(grp, ref["lse_%g" % tau], ref["smax_%g" % tau])[:, None] + \
                    2 * mg + R._ulp(lp_ref)
                _within("sample log_probs", (lp.double() - lp_ref).abs()[ok], b[ok])


def test_lm1b_truncation_threshold(world, lm1b):
    ref = lm1b.ref
    x = lm1b.xb()
    for grp in world:
        for top_k in (40, 1000):
            th, lse = _threshold(grp, x, 1, 1.0, top_k=top_k)
            assert torch.equal(th.cuda().double(), ref["th_%d" % top_k]), top_k
            _lse_check("trunc lse", grp, lse.cuda(), ref["lse"], ref["smax"])
        # nucleus: the bins hold fp32 masses exp(s − lse) with the pass's own lse, which is
        # checked against its bound and whose measured error is carried; rows whose cumulative
        # mass at θ* or at the value above lies within 2·(mass bound) of p are not checked
        th, lse = _threshold(grp, x, 1, 1.0, top_p=0.9)
        _lse_check("trunc lse", grp, lse.cuda(), ref["lse"], ref["smax"])
        dl = (lse.cuda().double() - ref["lse"]).abs()
        per_cta, grid = R.lse_depth(grp)
        depth = 32 + 4 + per_cta + math.ceil(grid / 2) + 1 + 4 + 8
        t = 4 * R.U + R.U * 3 * (ref["smax"] + ref["lse"].abs()) + \
            R.ETA * 2 * (ref["smax"] + ref["lse"].abs())
        mb = t + depth * R.U + 1.01 * dl
        band = ((ref["cum_p"] - 0.9).abs() <= 2 * mb) | ((ref["above_p"] - 0.9).abs() <= 2 * mb)
        th = th.cuda().double()
        assert torch.equal(th[~band], ref["th_p"][~band])
        print("top_p = 0.9: %d of %d rows in the mass band" % (int(band.sum()), N))
        assert band.float().mean() < 0.5


def test_lm1b_masked_draws(world, lm1b):
    ref = lm1b.ref
    x = lm1b.xb()
    for grp in world:
        for n in (1, 12, 32):                     # list capacities 8, 16 and 32
            lp, ids = grp.full_softmax_sample(x, n, 1.0, SEED, top_k=40)
            agree, ok = R.checked_draws(ids, ref["mkey_40"], ref["mkid_40"], ref["mloge_40"], n)
            assert agree, n
            assert ok.float().mean() >= 0.99, (n, float(ok.float().mean()))


def _grad_raw(x, Wc, bc, v0, lse, g, t, ctas, pad=64):
    """px_full_softmax_grad on one chunk with G and db guarded past what it may write: G
    [N, nblk·128 + pad] and db [rows + pad] start as NaN."""
    m, Kx = Wc.shape
    nblk = -(-m // 128)
    gp = nblk * 128 + pad
    G = torch.full((x.shape[0], gp), float("nan"), dtype=torch.bfloat16, device="cuda")
    db = torch.full((m + pad,), float("nan"), dtype=torch.float32, device="cuda")
    b_bf16 = bc.dtype == torch.bfloat16
    bp = bc.shape[1]
    rc = ops.lib().px_full_softmax_grad(
        _vp(x), x.shape[0], Kx, _vp(Wc), Wc.shape[1], _vp(bc), bp, int(b_bf16), m, v0,
        _vp(lse), _vp(g), _vp(t), _vp(G), gp, _vp(db), ctas,
        ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0
    torch.cuda.synchronize()
    assert G[:, nblk * 128:].isnan().all() and db[m:].isnan().all()     # the guards
    assert (G[:, m:nblk * 128] == 0).all()       # padding columns of the last block: zero
    return G[:, :m], db[:m]


def _bias_rows(b, v0, m, bf16):
    """bias rows of a chunk at the 16-byte pitch the kernel reads (4 fp32 or 8 bf16)"""
    w = 8 if bf16 else 4
    out = torch.zeros(m, w, dtype=torch.bfloat16 if bf16 else torch.float32, device="cuda")
    out[:, 0] = b[v0:v0 + m, 0]
    return out


def _check_grad_chunk(name, G, db, x, W, b, v0, lse32, g, t, smax):
    """G and db of one chunk per element against fp64 with the kernel's lse; returns G64"""
    m = G.shape[1]
    s = x.double() @ W[v0:v0 + m].double().t() + b[v0:v0 + m, 0].double()[None, :]
    p = torch.exp(s - lse32.double()[:, None])
    hot = (t[:, None] - v0) == torch.arange(m, device="cuda")[None, :]
    G64 = g.double()[:, None] * (p - hot.double())
    gb = R.grad_bound(p, g.double(), smax, lse32.double())
    _within(name + " G", (G.double() - G64).abs(), gb + R.bf16_half_ulp(G64.abs() + gb))
    depth = 2 * -(-x.shape[0] // 128) + 3 + 8
    db_b = gb.sum(0) + depth * R.U * G64.abs().sum(0)
    _within(name + " db", (db.double() - G64.sum(0)).abs(), db_b)
    return G64, gb


# the default vocabulary chunk of the backward at N = 2560 (`full_softmax_train_chunk`, checked
# on every world below): two waves of 128-row blocks, so each CTA runs 2 blocks, and V is not a
# multiple of it, so the last chunk is partial
VC = 2 * 128 * consts.NUM_SMS


@pytest.mark.parametrize("bias", ["fp32", "bf16"])
def test_lm1b_grad_kernel_per_element(lm1b, bias):
    """px_full_softmax_grad over the default chunks: G and db per element, and nothing written
    past each chunk's blocks.  The kernel takes the gathered chunk, so no world is needed."""
    assert V % VC
    x = lm1b.xb()
    lse32 = lm1b.ref["lse"].float()
    for v0 in range(0, V, VC):
        m = min(VC, V - v0)
        G, db = _grad_raw(x, lm1b.W[v0:v0 + m].contiguous(), _bias_rows(lm1b.b, v0, m, bias == "bf16"),
                          v0, lse32, lm1b.g, lm1b.t, consts.NUM_SMS)
        _check_grad_chunk("grad", G, db, x, lm1b.W, lm1b.b, v0, lse32, lm1b.g, lm1b.t,
                          lm1b.ref["smax"])


def test_lm1b_nll_grad_per_element(world, lm1b):
    """`full_softmax_nll_grad`'s dX, dW and db per element against fp64 (default chunking)"""
    grp = world[-1]
    x = lm1b.xb()
    nll, lse = grp.full_softmax_nll_lse(x, lm1b.t)
    dx, dW, db = grp.full_softmax_nll_grad(x, lm1b.t, lse, lm1b.g)
    vc = grp.full_softmax_train_chunk(N)
    assert vc == VC
    nch = -(-V // vc)
    xa = x.double().abs()
    dx64 = torch.zeros(N, K, dtype=torch.float64, device="cuda")
    dxb = torch.zeros_like(dx64)
    for v0 in range(0, V, vc):
        m = min(vc, V - v0)
        s = x.double() @ lm1b.W[v0:v0 + m].double().t() + lm1b.b[v0:v0 + m, 0].double()[None, :]
        p = torch.exp(s - lse.double()[:, None])
        hot = (lm1b.t[:, None] - v0) == torch.arange(m, device="cuda")[None, :]
        G64 = lm1b.g.double()[:, None] * (p - hot.double())
        gb = R.grad_bound(p, lm1b.g.double(), lm1b.ref["smax"], lse.double())
        eG = gb + R.bf16_half_ulp(G64.abs() + gb)        # bf16 G against G64
        Wc = lm1b.W[v0:v0 + m].double()
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


# ------------------------------------------------------------------ grids and edges
@pytest.fixture(scope="module")
def moderate():
    pr = Problem(40009, 136, 3000, 5, trunc_k=(40,))
    fabs, groups = _groups(2, pr.Wt, pr.Bt, 5, "mod")
    lay = groups[0].layout                     # 2 owners · 188 blocks: more items than 256 CTAs
    assert lay.world * -(-lay.parts_per_owner * lay.rows_per_part // 128) > 256
    yield pr, groups
    for f in fabs:
        f.close()


@pytest.mark.parametrize("ctas", [1, 2, 33, 131, 132, 255, 256])
def test_grid_sweep(monkeypatch, moderate, ctas):
    """every eval path on a grid of exactly `ctas` CTAs (one CTA walks every item); 256 is the
    list kernels' limit, where the combine's lanes hold 8 lists each"""
    pr, groups = moderate
    grp = groups[1]
    ref, n = pr.ref, 640
    x = pr.xb(n)
    monkeypatch.setattr(consts, "NUM_SMS", ctas)
    assert R.lse_depth(grp)[1] == ctas
    nll, lse = grp.full_softmax_nll_lse(x, pr.t[:n])
    _lse_check("sweep lse", grp, lse, ref["lse"][:n], ref["smax"][:n])
    for k in (9, 32):
        lp, ids = grp.full_softmax_topk(x, k)
        assert torch.equal(ids, ref["top_i"][:n, :k])
    lp, ids = grp.full_softmax_sample(x, 12, R.inv_tau(0.5), SEED)
    agree, ok = R.checked_draws(ids, ref["key_0.5"][:n], ref["kid_0.5"][:n],
                                ref["loge_0.5"][:n], 12)
    assert agree and ok.float().mean() >= 0.99
    th, _ = _threshold(grp, x, 1, 1.0, top_k=40)
    assert torch.equal(th.cuda().double(), ref["th_40"][:n])
    lp, ids = grp.full_softmax_sample(x, 12, 1.0, SEED, top_k=40)
    agree, ok = R.checked_draws(ids, ref["mkey_40"][:n], ref["mkid_40"][:n],
                                ref["mloge_40"][:n], 12)
    assert agree and ok.float().mean() >= 0.99


def test_list_kernels_refuse_257_ctas(monkeypatch, moderate):
    pr, groups = moderate
    monkeypatch.setattr(consts, "NUM_SMS", 257)
    x = pr.xb(64)
    for call in (lambda: groups[0].full_softmax_topk(x, 4),
                 lambda: groups[0].full_softmax_sample(x, 4, 1.0, 1),
                 lambda: groups[0].full_softmax_sample(x, 4, 1.0, 1, top_k=40)):
        with pytest.raises(RuntimeError, match=r"rc=-2"):
            call()


@pytest.mark.parametrize("ctas", [1, 7, 132])
def test_grad_grid_sweep(moderate, ctas):
    pr, _ = moderate
    x = pr.xb()
    lse32 = pr.ref["lse"].float()
    for v0, m in ((0, pr.V), (128 * 40, 128 * 33 + 5)):
        G, db = _grad_raw(x, pr.W[v0:v0 + m].contiguous(), _bias_rows(pr.b, v0, m, False), v0,
                          lse32, pr.g, pr.t, ctas)
        _check_grad_chunk("sweep grad", G, db, x, pr.W, pr.b, v0, lse32, pr.g, pr.t,
                          pr.ref["smax"])


def test_truncated_draws_cross_the_row_chunk(moderate):
    """N = 3000 with n = 12: the truncated path runs its rows in chunks of 2944"""
    pr, groups = moderate
    d = consts.SAMPLE_RADIX_BITS
    assert consts.TOPK_WS_BYTES // (consts.NUM_SMS * (1 << d) * 8) // 128 * 128 < pr.N
    for grp in groups:
        lp, ids = grp.full_softmax_sample(pr.xb(), 12, 1.0, SEED, top_k=40)
        agree, ok = R.checked_draws(ids, pr.ref["mkey_40"], pr.ref["mkid_40"],
                                    pr.ref["mloge_40"], 12)
        assert agree and ok.float().mean() >= 0.99


@pytest.fixture(scope="module")
def tall():
    pr = Problem(3001, 64, 20000, 9, taus=(1.0,), trunc_k=(40,))
    fabs, groups = _groups(2, pr.Wt, pr.Bt, 3, "div")
    yield pr, groups
    for f in fabs:
        f.close()


@pytest.mark.parametrize("n", [1, 127, 129, 8448, 8449, 20000])
def test_nll_rows_past_one_combine_grid(tall, n):
    """the combine kernel's grid stops at 8448 rows: N = 8449 and 20000 take a second pass"""
    pr, groups = tall
    nll, lse = groups[0].full_softmax_nll_lse(pr.xb(n), pr.t[:n])
    b = _lse_check("edge lse", groups[0], lse, pr.ref["lse"][:n], pr.ref["smax"][:n])
    nll_ref = pr.ref["lse"][:n] - pr.logit_t[:n]
    _within("edge nll", (nll.double() - nll_ref).abs(), b + R._ulp(nll_ref))


@pytest.mark.parametrize("k", [1, 3])
def test_topk_rows_in_chunks(tall, k):
    """N = 20 000: one row chunk at k = 1 (47 616 rows), two at k = 3 (15 872)"""
    pr, groups = tall
    lp, ids = groups[1].full_softmax_topk(pr.xb(), k)
    assert torch.equal(ids, pr.ref["top_i"][:, :k])


@pytest.mark.parametrize("Kx", [8, 72, 504, 512])
def test_partial_k_blocks(Kx):
    """K = 8 and 72: a partial last K-block; kb from 1 to 8"""
    pr = Problem(4099, Kx, 300, 13 + Kx, taus=(1.0,), trunc_k=(40,))
    fabs, groups = _groups(2, pr.Wt, pr.Bt, 3, "mod")
    for grp in groups:
        nll, lse = grp.full_softmax_nll_lse(pr.xb(), pr.t)
        _lse_check("K lse", grp, lse, pr.ref["lse"], pr.ref["smax"])
        lp, ids = grp.full_softmax_topk(pr.xb(), 17)
        assert torch.equal(ids, pr.ref["top_i"][:, :17])
        th, _ = _threshold(grp, pr.xb(), 1, 1.0, top_k=40)
        assert torch.equal(th.cuda().double(), pr.ref["th_40"])
    G, db = _grad_raw(pr.xb(), pr.W.contiguous(), _bias_rows(pr.b, 0, pr.V, False), 0,
                      pr.ref["lse"].float(), pr.g, pr.t, consts.NUM_SMS)
    _check_grad_chunk("K grad", G, db, pr.xb(), pr.W, pr.b, 0, pr.ref["lse"].float(), pr.g,
                      pr.t, pr.ref["smax"])
    for f in fabs:
        f.close()
