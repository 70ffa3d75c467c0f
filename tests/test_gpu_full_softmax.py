"""Fused full-softmax NLL and top-k (`parallax.nn.full_softmax_nll` and `full_softmax_topk`,
`ops/csrc/kernels/softmax_eval.cu`) against fp64 references built from the same bf16 rows, on
worlds simulated inside one GPU, and through the engine on the NVLink fabric."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import parallax_b200 as parallax
from parallax_b200 import optim

pytestmark = pytest.mark.gpu


def _table(V, K, seed, scale=1.0):
    """weight [V, K] and bias [V, 1] with bf16-representable values, so the kernels' operands
    are exactly the reference's."""
    g = torch.Generator().manual_seed(seed)
    Wt = (torch.randn(V, K, generator=g) * scale / K ** 0.5).bfloat16().float()
    Bt = torch.randn(V, 1, generator=g).bfloat16().float()
    return Wt, Bt


def _groups(world, Wt, Bt, P, strategy="mod", replicated=False, owners=None, weights="fp32"):
    """One (weight, bias) bf16 co-lookup group per simulated rank holding Wt [V, K], Bt [V, 1]."""
    from tests.gpu_utils import make_world
    from parallax_b200.parallel import modes
    from parallax_b200.parallel.nvlink_backend import NVSparseTable, NVSparseGroup
    from parallax_b200.graph import Graph
    fabs = make_world(world)
    run_option = "MPI" if replicated else "HYBRID"
    route = modes.route_for(run_option, True)
    cfg = parallax.Config(run_option=run_option)
    opt = optim.Adagrad(0.2, 1.0)
    graph = Graph(torch.nn.Linear(1, 1), optimizer=opt)
    o = {"sparse_blocks": 4, "sparse_early_push": False, "sparse_weights": weights}
    groups = []
    for f in fabs:
        tw = NVSparseTable("w", Wt, P, strategy, opt, f, route, graph, cfg, options=o,
                           out_dtype=torch.bfloat16, owners=owners, auto_group=False)
        tb = NVSparseTable("b", Bt, P, strategy, opt, f, route, graph, cfg, options=o,
                           out_dtype=torch.bfloat16, owners=owners, auto_group=False)
        groups.append(NVSparseGroup([tw, tb]))
    torch.cuda.synchronize()
    return fabs, groups


def _nll_reference(x, Wt, Bt, targets):
    logits = x.double() @ Wt.double().t() + Bt.double().t()
    return F.cross_entropy(logits, targets.clamp(0, Wt.shape[0] - 1), reduction="none")


def _topk_reference(x, Wt, Bt):
    """fp64 log-probabilities [N, V] and each row's ids sorted by (logit desc, id asc)."""
    lp = torch.log_softmax(x.double() @ Wt.double().t() + Bt.double().t(), dim=-1)
    return lp, torch.sort(lp, dim=1, descending=True, stable=True).indices


def _check_topk(lp, ids, ref_lp, order, k, V, margin=2e-3):
    lp, ids = lp.cpu(), ids.cpu()
    n = ref_lp.shape[0]
    assert lp.shape == (n, k) and lp.dtype == torch.float32
    assert ids.shape == (n, k) and ids.dtype == torch.int64
    assert ((ids >= 0) & (ids < V)).all()
    assert all(len(set(r)) == k for r in ids.tolist())
    assert (lp[:, 1:] <= lp[:, :-1]).all()
    torch.testing.assert_close(lp.double(), ref_lp.gather(1, ids), rtol=0, atol=1e-3)
    # ids are the reference's top k wherever its consecutive logits differ by more than margin
    srt = ref_lp.gather(1, order[:, :k + 1] if k < V else order)
    d = srt[:, :-1] - srt[:, 1:]
    ok = torch.ones(n, k, dtype=torch.bool)
    ok[:, 1:] &= d[:, :k - 1] > margin
    if k < V:
        ok &= d[:, :k] > margin
    else:
        ok[:, :-1] &= d[:, :k - 1] > margin
    assert ok.float().mean() > 0.3
    assert torch.equal(ids[ok], order[:, :k][ok])


CASES = [
    # world, V, P, strategy, K, N, replicated
    (1, 1000, 1, "mod", 32, 1, False),
    (2, 1001, 5, "mod", 64, 7, False),
    (4, 3001, 7, "div", 136, 640, False),
    (8, 3001, 32, "mod", 512, 2560, False),
    (2, 2999, 3, "div", 512, 2560, False),
    (4, 777, 1, "mod", 64, 640, True),
]


def _owners(world, P, replicated):
    from parallax_b200.parallel.layout import assign_owners
    return None if replicated else assign_owners([("a", P, 7), ("b", P, 3)], world)["b"]


# ------------------------------------------------------------------ NLL
@pytest.mark.parametrize("world,V,P,strategy,K,N,replicated", CASES)
def test_kernel_matches_fp64_reference(world, V, P, strategy, K, N, replicated):
    Wt, Bt = _table(V, K, 7)
    fabs, groups = _groups(world, Wt, Bt, P, strategy, replicated, _owners(world, P, replicated))
    gen = torch.Generator().manual_seed(world * 100 + K)
    x = torch.randn(N, K, generator=gen).bfloat16()
    targets = torch.randint(0, V, (N,), generator=gen)
    targets[0] = 0
    targets[-1] = V - 1
    ref = _nll_reference(x.float(), Wt, Bt, targets).float()
    for grp in groups:                    # every rank evaluates its batch alone
        nll = grp.full_softmax_nll(x.cuda(), targets.cuda())
        torch.cuda.synchronize()
        assert nll.shape == (N,) and nll.dtype == torch.float32
        torch.testing.assert_close(nll.cpu(), ref, rtol=1e-5, atol=1e-3)
    for f in fabs:
        f.close()


def test_large_logits_stay_finite_and_exact():
    """Logits up to about ±80: the merged (max, Σexp) pairs never overflow."""
    V, K, N = 4097, 64, 300
    Wt, Bt = _table(V, K, 7, scale=8.0)
    fabs, groups = _groups(2, Wt, Bt, 4)
    gen = torch.Generator().manual_seed(1)
    x = (torch.randn(N, K, generator=gen) * 2.0).bfloat16()
    targets = torch.randint(0, V, (N,), generator=gen)
    logits = x.double() @ Wt.double().t() + Bt.double().t()
    assert 60 < float(logits.abs().max()) < 120
    ref = _nll_reference(x.float(), Wt, Bt, targets).float()
    for grp in groups:
        nll = grp.full_softmax_nll(x.cuda(), targets.cuda()).cpu()
        assert torch.isfinite(nll).all()
        torch.testing.assert_close(nll, ref, rtol=1e-5, atol=1e-3)
    for f in fabs:
        f.close()


def test_out_of_range_target_is_nan_in_its_row_only():
    V, K, N = 1000, 64, 50
    Wt, Bt = _table(V, K, 7)
    fabs, groups = _groups(2, Wt, Bt, 3)
    gen = torch.Generator().manual_seed(2)
    x = torch.randn(N, K, generator=gen).bfloat16()
    targets = torch.randint(0, V, (N,), generator=gen)
    targets[3], targets[9] = V + 5, -1
    ref = _nll_reference(x.float(), Wt, Bt, targets).float()
    nll = groups[0].full_softmax_nll(x.cuda(), targets.cuda()).cpu()
    bad = torch.zeros(N, dtype=torch.bool)
    bad[[3, 9]] = True
    assert torch.isnan(nll[bad]).all()
    torch.testing.assert_close(nll[~bad], ref[~bad], rtol=1e-5, atol=1e-3)
    for f in fabs:
        f.close()


def test_no_logits_buffer():
    """V = 200 000, N = 2560: the composition would need > 2 GB of [N, V] logits; the fused
    call allocates only O(N) scratch."""
    V, K, N = 200000, 512, 2560
    Wt, Bt = _table(V, K, 7)
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
    assert N * V * (2 + 4) > 2 << 30                   # what the bf16 + fp32 logits would take
    ref = _nll_reference(x[:64].float().cpu(), Wt, Bt, targets[:64].cpu()).float()
    torch.testing.assert_close(nll[:64].cpu(), ref, rtol=1e-5, atol=1e-3)
    for f in fabs:
        f.close()


# ------------------------------------------------------------------ top-k
@pytest.mark.parametrize("k", [1, 5, 9, 16, 17, 32])
@pytest.mark.parametrize("world,V,P,strategy,K,N,replicated", CASES)
def test_topk_kernel_matches_fp64_reference(world, V, P, strategy, K, N, replicated, k):
    Wt, Bt = _table(V, K, world * 10 + P)
    fabs, groups = _groups(world, Wt, Bt, P, strategy, replicated, _owners(world, P, replicated))
    x = torch.randn(N, K, generator=torch.Generator().manual_seed(world * 100 + K)).bfloat16()
    ref_lp, order = _topk_reference(x.float(), Wt, Bt)
    for grp in groups:                    # every rank evaluates its batch alone
        lp, ids = grp.full_softmax_topk(x.cuda(), k)
        torch.cuda.synchronize()
        _check_topk(lp, ids, ref_lp, order, k, V)
    for f in fabs:
        f.close()


@pytest.mark.parametrize("world", [1, 2, 4, 8])
def test_topk_exact_ties_in_ascending_id_order(world):
    """Duplicated table rows spread over partitions and owners: equal logits, ascending ids."""
    V, K, N, P, k = 2001, 64, 300, 7, 8
    Wt, Bt = _table(V, K, 5)
    Wt *= 0.1
    g = torch.Generator().manual_seed(6)
    top = (torch.randn(K, generator=g) * 2).bfloat16().float()
    dup = [1999, 3, 700, 701, 1200, 4]         # ids in several partitions, in no sorted order
    for r in dup:
        Wt[r], Bt[r] = top, 0.5
    for r in (11, 1500):                       # a second, lower tie group
        Wt[r], Bt[r] = top, 0.25
    fabs, groups = _groups(world, Wt, Bt, P, "mod" if world % 2 else "div")
    x = (top.repeat(N, 1) + torch.randn(N, K, generator=g) * 0.05).bfloat16()
    want = sorted(dup) + [11, 1500]
    for grp in groups:
        lp, ids = grp.full_softmax_topk(x.cuda(), k)
        lp, ids = lp.cpu(), ids.cpu()
        assert (ids == torch.tensor(want)).all(), ids[:3]
        assert (lp[:, :6] == lp[:, :1]).all() and (lp[:, 6:] == lp[:, 6:7]).all()
    for f in fabs:
        f.close()


def test_topk_k1_agrees_with_the_nll():
    V, K, N, P = 3001, 128, 700, 5
    Wt, Bt = _table(V, K, 8)
    fabs, groups = _groups(2, Wt, Bt, P)
    x = torch.randn(N, K, generator=torch.Generator().manual_seed(9)).bfloat16().cuda()
    for grp in groups:
        lp, ids = grp.full_softmax_topk(x, 1)
        nll = grp.full_softmax_nll(x, ids[:, 0])
        torch.testing.assert_close(-lp[:, 0].cpu(), nll.cpu(), rtol=0, atol=1e-3)
    for f in fabs:
        f.close()


@pytest.mark.parametrize("world,P,k", [(1, 1, 5), (2, 5, 32), (4, 7, 1)])
def test_topk_bf16_masters(world, P, k):
    """sparse_weights="bf16": bf16 bias master rows, widened to fp32 where they are added."""
    V, K, N = 2999, 136, 300
    Wt, Bt = _table(V, K, 12)
    fabs, groups = _groups(world, Wt, Bt + 0.5, P, weights="bf16")
    assert groups[0].tables[1].weight_dtype == torch.bfloat16
    x = torch.randn(N, K, generator=torch.Generator().manual_seed(13)).bfloat16()
    ref_lp, order = _topk_reference(x.float(), Wt, (Bt + 0.5).bfloat16().float())
    for grp in groups:
        lp, ids = grp.full_softmax_topk(x.cuda(), k)
        _check_topk(lp, ids, ref_lp, order, k, V)
    for f in fabs:
        f.close()


def test_topk_no_logits_buffer():
    """V = 200 000, N = 2560, k = 32: peak allocation grows by less than 64 MB."""
    V, K, N, k = 200000, 512, 2560, 32
    Wt, Bt = _table(V, K, 14)
    fabs, groups = _groups(1, Wt, Bt, 1)
    x = torch.randn(N, K, device="cuda").bfloat16()
    groups[0].full_softmax_topk(x, k)                  # warm-up (module load, maps)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    lp, ids = groups[0].full_softmax_topk(x, k)
    torch.cuda.synchronize()
    growth = torch.cuda.max_memory_allocated() - base
    assert growth < 64 << 20, growth
    ref_lp, order = _topk_reference(x[:64].float().cpu(), Wt, Bt)
    _check_topk(lp[:64], ids[:64], ref_lp, order, k, V)
    for f in fabs:
        f.close()


def test_topk_argument_errors():
    Wt, Bt = _table(100, 32, 1)
    fabs, groups = _groups(1, Wt, Bt, 1)
    x = torch.randn(4, 32, device="cuda").bfloat16()
    for k in (0, 33, True):
        with pytest.raises(ValueError, match="k must be"):
            groups[0].full_softmax_topk(x, k)
    with pytest.raises(ValueError, match="bf16 inputs"):
        groups[0].full_softmax_topk(x.float(), 3)
    for f in fabs:
        f.close()


# ------------------------------------------------------------------ through the engine
def _lm1b_session(fabric="nvlink", num_sampled=16, bf16=True, eval_top_k=0):
    from parallax_b200.models.lm1b import LM1B, lm1b_graph
    torch.manual_seed(0)
    m = LM1B(vocab_size=1003, emb_size=32, state_size=64, projected_size=32,
             num_sampled=num_sampled, num_steps=4, num_shards=3, keep_prob=1.0,
             eval_top_k=eval_top_k)
    sc = {"fabric": fabric}
    if bf16 and fabric == "nvlink":
        sc["compute_dtype"] = "bf16"
    sess, *_ = parallax.parallel_run(lm1b_graph(m, batch_size=128), "localhost:0",
                                     parallax_config=parallax.Config(sess_config=sc))
    return sess


def _batch(seed, V=1003):
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(0, V, (128, 4), generator=g)
    return {"x": [x], "y": [torch.roll(x, -1, dims=1)]}


def _count_fused(monkeypatch, method):
    """The second argument (targets or k) of every call of NVSparseGroup.`method`."""
    from parallax_b200.parallel.nv_sparse import NVSparseGroup
    calls = []
    orig = getattr(NVSparseGroup, method)
    monkeypatch.setattr(NVSparseGroup, method,
                        lambda self, x, a: calls.append(a) or orig(self, x, a))
    return calls


def _eval_loss(sess):
    m = sess.engine.model
    m.eval()
    try:
        return float(sess.run("loss", _batch(99))[0])
    finally:
        m.train()


def test_engine_eval_between_training_steps(monkeypatch):
    from parallax_b200.parallel.engine import full_softmax_composition
    calls = _count_fused(monkeypatch, "full_softmax_nll")
    sess = _lm1b_session()
    m = sess.engine.model
    grp = m.softmax_w.table.group
    x = torch.randn(256, 32, device="cuda").bfloat16()
    t = torch.randint(0, 1003, (256,), device="cuda")

    def fused_and_composition():
        with torch.no_grad():
            a = parallax.nn.full_softmax_nll(x, t, m.softmax_w, m.softmax_b)
            b = full_softmax_composition(x, t, m.softmax_w, m.softmax_b)
        return a.cpu(), b.cpu()

    losses, evals = [], []
    for step in range(4):
        losses.append(float(sess.run(["loss", "train_op"], _batch(step))[0][0]))
        n0 = len(calls)
        ctl0 = grp.ctl.clone()
        evals.append(_eval_loss(sess))
        fused, comp = fused_and_composition()
        torch.cuda.synchronize()
        assert len(calls) == n0 + 2                  # the session's eval and ours were fused
        assert torch.equal(grp.ctl, ctl0)            # eval leaves the step flags alone
        # the rows the lookup sees, i.e. fresh after the step; the fused logits are fp32,
        # the composition's are rounded to bf16
        torch.testing.assert_close(fused, comp, rtol=0, atol=3e-2)
    assert np.isfinite(evals).all() and len(set(evals)) == len(evals)
    assert np.isfinite(losses).all() and sess.engine.global_step == 4
    sd = sess.engine.state_dict()
    sess.close()
    # eval agrees with the host fabric restored from the same state (fp32 LSTM there)
    host = _lm1b_session("host")
    host.engine.load_state_dict(sd)
    np.testing.assert_allclose(_eval_loss(host), evals[-1], rtol=3e-2)
    host.close()


def test_training_with_full_softmax_takes_the_composition(monkeypatch):
    """num_sampled = 0 in training needs dense table gradients: the fused kernel never runs."""
    calls = _count_fused(monkeypatch, "full_softmax_nll")
    sess = _lm1b_session(num_sampled=0)
    losses = [float(sess.run(["loss", "train_op"], _batch(0))[0][0]) for _ in range(3)]
    assert calls == [] and np.isfinite(losses).all() and losses[-1] < losses[0]
    _eval_loss(sess)
    assert len(calls) == 1
    sess.close()


def test_topk_engine_eval_between_training_steps(monkeypatch):
    from parallax_b200.parallel.engine import full_softmax_topk_composition
    calls = _count_fused(monkeypatch, "full_softmax_topk")
    sess = _lm1b_session(eval_top_k=5)
    m = sess.engine.model
    grp = m.softmax_w.table.group
    x = torch.randn(256, 32, device="cuda").bfloat16()
    for step in range(3):
        sess.run(["loss", "train_op"], _batch(step))
        n0 = len(calls)
        ctl0 = grp.ctl.clone()
        m.eval()
        try:
            top = sess.run("top_k_ids", _batch(99))[0]
        finally:
            m.train()
        assert np.asarray(top).shape == (128, 4, 5)
        with torch.no_grad():
            lp, ids = parallax.nn.full_softmax_topk(x, m.softmax_w, m.softmax_b, 5)
            clp, cids = full_softmax_topk_composition(x, m.softmax_w, m.softmax_b, 6)
        torch.cuda.synchronize()
        assert calls[n0:] == [5, 5]               # the session's eval and ours were fused
        assert torch.equal(grp.ctl, ctl0)         # eval leaves the step flags alone
        # fp32 logits against the composition's bf16 logits: ids agree wherever the
        # composition's neighbours (the 6th included) are apart
        lp, ids, clp, cids = lp.cpu(), ids.cpu(), clp.cpu(), cids.cpu()
        torch.testing.assert_close(lp, clp[:, :5], rtol=0, atol=3e-2)
        d = clp[:, :-1] - clp[:, 1:]
        ok = d > 0.1
        ok[:, 1:] &= d[:, :-1] > 0.1
        assert ok.any() and torch.equal(ids[ok], cids[:, :5][ok])
    sess.close()


def test_topk_grad_or_large_k_takes_the_composition(monkeypatch):
    calls = _count_fused(monkeypatch, "full_softmax_topk")
    sess = _lm1b_session(eval_top_k=5)
    m = sess.engine.model
    sess.run(["loss", "train_op"], _batch(0))
    x = torch.randn(64, 32, device="cuda").bfloat16()
    lp, ids = parallax.nn.full_softmax_topk(x.requires_grad_(), m.softmax_w, m.softmax_b, 4)
    assert lp.requires_grad and calls == []
    with torch.no_grad():
        lp, ids = parallax.nn.full_softmax_topk(x, m.softmax_w, m.softmax_b, 33)
    assert ids.shape == (64, 33) and calls == []
    with torch.no_grad():
        parallax.nn.full_softmax_topk(x, m.softmax_w, m.softmax_b, 32)
    assert calls == [32]
    sess.close()
