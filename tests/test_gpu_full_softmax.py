"""Fused full-softmax NLL (`parallax.nn.full_softmax_nll`, `ops/csrc/kernels/softmax_eval.cu`)
against an fp64 reference built from the same bf16 rows, on worlds simulated inside one GPU,
and through the engine on the NVLink fabric."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import parallax_b200 as parallax
from parallax_b200 import optim

pytestmark = pytest.mark.gpu


def _groups(world, V, K, P, strategy="mod", replicated=False, owners=None, scale=1.0, seed=7):
    """One (weight [V, K], bias [V, 1]) bf16 co-lookup group per simulated rank; the initial
    values are bf16-representable, so the kernel's operands are exactly the reference's."""
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
    g = torch.Generator().manual_seed(seed)
    Wt = (torch.randn(V, K, generator=g) * scale / K ** 0.5).bfloat16().float()
    Bt = torch.randn(V, 1, generator=g).bfloat16().float()
    o = {"sparse_blocks": 4, "sparse_early_push": False}
    groups = []
    for f in fabs:
        tw = NVSparseTable("w", Wt, P, strategy, opt, f, route, graph, cfg, options=o,
                           out_dtype=torch.bfloat16, owners=owners, auto_group=False)
        tb = NVSparseTable("b", Bt, P, strategy, opt, f, route, graph, cfg, options=o,
                           out_dtype=torch.bfloat16, owners=owners, auto_group=False)
        groups.append(NVSparseGroup([tw, tb]))
    torch.cuda.synchronize()
    return fabs, groups, Wt, Bt


def _reference(x, Wt, Bt, targets):
    logits = x.double() @ Wt.double().t() + Bt.double().t()
    return F.cross_entropy(logits, targets.clamp(0, Wt.shape[0] - 1), reduction="none")


CASES = [
    # world, V, P, strategy, K, N, replicated
    (1, 1000, 1, "mod", 32, 1, False),
    (2, 1001, 5, "mod", 64, 7, False),
    (4, 3001, 7, "div", 136, 640, False),
    (8, 3001, 32, "mod", 512, 2560, False),
    (2, 2999, 3, "div", 512, 2560, False),
    (4, 777, 1, "mod", 64, 640, True),
]


@pytest.mark.parametrize("world,V,P,strategy,K,N,replicated", CASES)
def test_kernel_matches_fp64_reference(world, V, P, strategy, K, N, replicated):
    from parallax_b200.parallel.layout import assign_owners
    owners = None if replicated else assign_owners([("a", P, 7), ("b", P, 3)], world)["b"]
    fabs, groups, Wt, Bt = _groups(world, V, K, P, strategy, replicated, owners)
    gen = torch.Generator().manual_seed(world * 100 + K)
    x = torch.randn(N, K, generator=gen).bfloat16()
    targets = torch.randint(0, V, (N,), generator=gen)
    targets[0] = 0
    targets[-1] = V - 1
    ref = _reference(x.float(), Wt, Bt, targets).float()
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
    fabs, groups, Wt, Bt = _groups(2, V, K, 4, scale=8.0)
    gen = torch.Generator().manual_seed(1)
    x = (torch.randn(N, K, generator=gen) * 2.0).bfloat16()
    targets = torch.randint(0, V, (N,), generator=gen)
    logits = x.double() @ Wt.double().t() + Bt.double().t()
    assert 60 < float(logits.abs().max()) < 120
    ref = _reference(x.float(), Wt, Bt, targets).float()
    for grp in groups:
        nll = grp.full_softmax_nll(x.cuda(), targets.cuda()).cpu()
        assert torch.isfinite(nll).all()
        torch.testing.assert_close(nll, ref, rtol=1e-5, atol=1e-3)
    for f in fabs:
        f.close()


def test_out_of_range_target_is_nan_in_its_row_only():
    V, K, N = 1000, 64, 50
    fabs, groups, Wt, Bt = _groups(2, V, K, 3)
    gen = torch.Generator().manual_seed(2)
    x = torch.randn(N, K, generator=gen).bfloat16()
    targets = torch.randint(0, V, (N,), generator=gen)
    targets[3], targets[9] = V + 5, -1
    ref = _reference(x.float(), Wt, Bt, targets).float()
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
    fabs, groups, Wt, Bt = _groups(1, V, K, 1)
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
    ref = _reference(x[:64].float().cpu(), Wt, Bt, targets[:64].cpu()).float()
    torch.testing.assert_close(nll[:64].cpu(), ref, rtol=1e-5, atol=1e-3)
    for f in fabs:
        f.close()


# ------------------------------------------------------------------ through the engine
def _lm1b_session(fabric, num_sampled=16, bf16=True):
    from parallax_b200.models.lm1b import LM1B, lm1b_graph
    torch.manual_seed(0)
    m = LM1B(vocab_size=1003, emb_size=32, state_size=64, projected_size=32,
             num_sampled=num_sampled, num_steps=4, num_shards=3, keep_prob=1.0)
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


def _eval_loss(sess):
    m = sess.engine.model
    m.eval()
    try:
        return float(sess.run("loss", _batch(99))[0])
    finally:
        m.train()


def test_engine_eval_between_training_steps(monkeypatch):
    from parallax_b200.parallel.engine import full_softmax_composition
    from parallax_b200.parallel.nv_sparse import NVSparseGroup
    calls = []
    orig = NVSparseGroup.full_softmax_nll
    monkeypatch.setattr(NVSparseGroup, "full_softmax_nll",
                        lambda self, x, t: calls.append(1) or orig(self, x, t))
    sess = _lm1b_session("nvlink")
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
    from parallax_b200.parallel.nv_sparse import NVSparseGroup
    calls = []
    orig = NVSparseGroup.full_softmax_nll
    monkeypatch.setattr(NVSparseGroup, "full_softmax_nll",
                        lambda self, x, t: calls.append(1) or orig(self, x, t))
    sess = _lm1b_session("nvlink", num_sampled=0)
    losses = [float(sess.run(["loss", "train_op"], _batch(0))[0][0]) for _ in range(3)]
    assert calls == [] and np.isfinite(losses).all() and losses[-1] < losses[0]
    _eval_loss(sess)
    assert calls == [1]
    sess.close()
