"""`ClipByGlobalNorm(include_sparse=True)` on the NVLink fabric: the owner-side norm
kernel against an fp64 reference of the merged rows, the clipped apply through the
unchanged owner kernel, and the engine against the host-fabric oracle."""
import numpy as np
import pytest
import torch

import parallax_b200 as parallax
from parallax_b200 import optim
from parallax_b200.models.simple import MLPWithEmbedding

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------ kernel level
def _groups(world, V, Ds, P, opt, run_option, average, local_agg, out_dtype, scale):
    from tests.gpu_utils import make_world
    from parallax_b200.parallel import modes
    from parallax_b200.parallel.nvlink_backend import NVSparseTable, NVSparseGroup
    fabs = make_world(world)
    route = modes.route_for(run_option, True)
    cfg = parallax.Config(run_option=run_option, average_sparse=average)
    cfg.communication_config = parallax.CommunicationConfig(
        parallax.PSConfig(local_aggregation=local_agg))
    names = ["t%d" % k for k in range(len(Ds))]
    graph = parallax.Graph(torch.nn.Linear(1, 1), optimizer=opt,
                           grad_rules=[parallax.ScaleGradients(scale, params=names[:1])])
    g = torch.Generator().manual_seed(7)
    W0 = [torch.randn(V, D, generator=g) for D in Ds]
    o = {"sparse_blocks": 4, "sparse_early_push": False}
    groups = []
    for f in fabs:
        tabs = [NVSparseTable(n, w, P, "mod", opt, f, route, graph, cfg, options=o,
                              out_dtype=out_dtype, auto_group=False)
                for n, w in zip(names, W0)]
        grp = NVSparseGroup(tabs)
        grp.hp_clip = torch.zeros_like(grp.hp.dev)
        groups.append(grp)
    return fabs, groups


def _merged_reference(grp, avg_of):
    """fp64 merge of what sits in this owner's receive rings: {table k: (rows, merged ×
    the owner-side factor)} — the rows the owner kernel hands to the optimizer."""
    from parallax_b200 import ops
    W, cap = grp.world, grp.cap
    R = ops.sparse_abi()["hdr_words"] // 3
    hdr = grp.hdr_buf.tensor(torch.int32, 3 * R).cpu()
    cnt = hdr[2 * R:2 * R + W].tolist()
    ring_ids = grp.ids_buf.tensor(torch.int32, W * cap).view(W, cap).cpu()
    out = []
    for t in grp.tables:
        ring = t.ring_buf.tensor(grp.wire_dtype, W * cap * t.Dp).view(W, cap, t.Dp).cpu()
        ids = torch.cat([ring_ids[s, :cnt[s]] for s in range(W)]).long()
        vals = torch.cat([ring[s, :cnt[s]].double() for s in range(W)])
        keep = ids >= 0
        u, inv = torch.unique(ids[keep], return_inverse=True)
        m = torch.zeros(u.numel(), t.Dp, dtype=torch.float64).index_add_(0, inv, vals[keep])
        out.append((u, m * avg_of(t)))
    return out


def _avg_of(grp):
    def f(t):
        a = (1.0 / grp.world) if t.average else 1.0
        return a if grp.boundary else a * t.scale
    return f


def _clip_scale_all(fabs, sums, max_norm):
    """Phase 3 of a joint step on every simulated rank: the one-shot all-reduce of Σg²
    and clip_scale, as `NVDenseGroup._finish_clip` issues them."""
    from parallax_b200.parallel import nvops
    from parallax_b200.parallel.symmetric import CH_SMALL
    # allocated (and filled) before the first launch: nothing may run on the host between
    # the launches of the simulated ranks, and the fills must not race the comm streams
    scales = [torch.ones(1, device="cuda") for _ in fabs]
    norms = [torch.zeros(1, device="cuda") for _ in fabs]
    tots = [torch.zeros(4, device="cuda") for _ in fabs]
    torch.cuda.synchronize()
    if len(fabs) > 1:
        for f, loc, tot in zip(fabs, sums, tots):
            nvops.allreduce_oneshot(f.heap, loc, tot, f.small_stage, 4, torch.float32, 1.0,
                                    CH_SMALL, stream=f.comm_stream)
    else:
        tots = sums
    for f, loc, tot, sc, nm in zip(fabs, sums, tots, scales, norms):
        nvops.clip_scale(tot, max_norm, sc, nm, loc, stream=f.comm_stream)
    torch.cuda.synchronize()
    return scales, norms


@pytest.mark.parametrize("world", [1, 2, 4, 8])
@pytest.mark.parametrize("layout", ["HYBRID", "MPI"])
@pytest.mark.parametrize("wire", ["fp32", "bf16"])
@pytest.mark.parametrize("local_agg", [True, False])
def test_owner_norm_and_clipped_apply(world, layout, wire, local_agg):
    """Steps 1 and 3 joint-clipped, step 2 plain: Σ of the norm kernel vs fp64, tables
    and slots vs the optimizer applied to scale × merged rows; the plain step in between
    checks that the norm kernel left slotmap, step counters and the grid barrier clean."""
    V, P, n = 701, 8, 300
    Ds = (36, 1) if world in (2, 8) else (36,)             # a 2-table co-lookup group too
    opt = optim.Adagrad(0.2, 0.5)
    bf16 = wire == "bf16"
    fabs, groups = _groups(world, V, Ds, P, opt, layout, average=(world == 4),
                           local_agg=local_agg,
                           out_dtype=torch.bfloat16 if bf16 else torch.float32, scale=2.0)
    for grp in groups:
        grp._ensure_capacity(n)
    for grp in groups:
        grp.warm(n)
    torch.cuda.synchronize()
    owners = range(world)           # with MPI every replica applies every row
    ref = [[t.table.cpu().clone() for t in grp.tables] for grp in groups]
    ref_slots = [[tuple(s.cpu().clone() for s in t.slots) for t in grp.tables]
                 for grp in groups]
    gen = torch.Generator().manual_seed(11)
    max_norm = 0.5
    for step in (1, 2, 3):
        joint = step != 2
        toks, grads = [], []
        for grp in groups:
            ids = torch.randint(0, V, (n,), generator=gen)
            ids[:40] = ids[0]
            ids[40:60] = 17
            _, pend = grp.lookup(ids.cuda())
            toks.append(pend)
            gdt = torch.bfloat16 if bf16 else torch.float32
            grads.append([torch.randn(n, D, generator=gen).to(gdt).cuda() for D in Ds])
        torch.cuda.synchronize()
        for grp, tok, gs in zip(groups, toks, grads):
            grp.add_pending(tok, gs)
            grp.begin_step(step)
        torch.cuda.synchronize()
        for grp in groups:                                   # 1. every rank's push
            grp.stage_push(step)
        torch.cuda.synchronize()
        assert groups[0].wire_dtype == (torch.bfloat16 if bf16 else torch.float32)
        merged = [_merged_reference(grp, _avg_of(grp)) for grp in groups]
        scale = 1.0
        if joint:
            sums = [torch.zeros(4, device="cuda") for _ in groups]
            torch.cuda.synchronize()
            for grp, s in zip(groups, sums):                  # 2. every rank's norm
                grp.stage_norm(s if grp.norm_counts() else None)
            torch.cuda.synchronize()
            want = [sum(float((m ** 2).sum()) for _, m in mg) for mg in merged]
            for r, grp in enumerate(groups):
                got = float(sums[r][0])
                exp = want[r] if grp.norm_counts() else 0.0
                assert abs(got - exp) <= 1e-5 * max(exp, 1e-30), (r, got, exp)
            total = sum(want[r] for r, g_ in enumerate(groups) if g_.norm_counts())
            scales, norms = _clip_scale_all(fabs, sums, max_norm)   # 3. all-reduce + scale
            for nm in norms:
                assert abs(float(nm) - total ** 0.5) <= 1e-5 * total ** 0.5
            scale = float(scales[0])
            assert scale < 1.0
            for grp, sc in zip(groups, scales):              # 4. every rank's apply
                grp.stage_apply(step, hp=grp.clip_hp(sc))
        else:
            for grp in groups:
                grp.stage_apply(step)
        torch.cuda.synchronize()
        hp = opt.hyper(step)
        for r in owners:
            for k, (u, m) in enumerate(merged[r]):
                optim.apply_sparse_rows_(opt.kind, ref[r][k], u, (m * scale).float(),
                                         ref_slots[r][k], hp)
        for r in owners:
            grp = groups[r]
            assert int(grp.ctl[0]) == step                   # ctl->step
            assert bool((grp.slotmap == -1).all())
            for k, t in enumerate(grp.tables):
                D = t.D
                torch.testing.assert_close(t.table[:, :D].cpu(), ref[r][k][:, :D],
                                           rtol=1e-4, atol=1e-5)
                for s, rs in zip(t.slots, ref_slots[r][k]):
                    torch.testing.assert_close(s[:, :D].cpu(), rs[:, :D], rtol=1e-4, atol=1e-5)
                ref[r][k] = t.table.cpu().clone()            # track the device from here
                ref_slots[r][k] = tuple(s.cpu().clone() for s in t.slots)
    for f in fabs:
        f.close()


# ------------------------------------------------------------------ engine level
def _run(fabric, run_option, opt, steps, dense_update="sharded", graph=False,
         params=None, max_norm=0.05):
    model = MLPWithEmbedding(64, partitioner=parallax.get_partitioner(3))
    rules = [parallax.ScaleGradients(2.0, params=["emb.weight"]),
             parallax.ClipByGlobalNorm(max_norm, params=params, include_sparse=True)]
    g = parallax.Graph(model, optimizer=opt, grad_rules=rules,
                       ema=parallax.ExponentialMovingAverage(0.9, ["fc2.*"]))
    cfg = parallax.Config(run_option=run_option, sess_config={
        "fabric": fabric, "dense_update": dense_update, "cuda_graph": graph})
    sess, *_ = parallax.parallel_run(g, "localhost:0", sync=True, parallax_config=cfg)
    gen = torch.Generator().manual_seed(0)
    losses, norms = [], []
    for _ in range(steps):
        ids = torch.randint(0, 64, (8, 3), generator=gen)
        ids[:, 0] = 5
        labels = torch.randint(0, 4, (8,), generator=gen)
        loss, _ = sess.run(["loss", "train_op"], {"ids": [ids], "labels": [labels]})
        losses.append(loss[0])
        norms.append(sess.engine.grad_norm(0))
    sd = sess.engine.state_dict()
    sess.close()
    return losses, norms, sd


def _same(a, b, rtol):
    np.testing.assert_allclose(a[0], b[0], rtol=rtol, atol=rtol * 0.1)
    np.testing.assert_allclose(a[1], b[1], rtol=rtol)
    for n, w in b[2]["dense"]["master"].items():
        torch.testing.assert_close(a[2]["dense"]["master"][n], w, rtol=rtol, atol=rtol * 0.1)
    torch.testing.assert_close(a[2]["sparse"]["emb.weight"]["weight"],
                               b[2]["sparse"]["emb.weight"]["weight"], rtol=rtol,
                               atol=rtol * 0.1)
    torch.testing.assert_close(a[2]["sparse"]["emb.weight"]["slots"],
                               b[2]["sparse"]["emb.weight"]["slots"], rtol=rtol,
                               atol=rtol * 0.1)


@pytest.mark.parametrize("run_option", ["HYBRID", "MPI", "PS"])
@pytest.mark.parametrize("opt_name", ["sgd", "adagrad", "adam"])
@pytest.mark.parametrize("dense_update", ["sharded", "replicated"])
def test_engine_joint_clip_matches_host_oracle(run_option, opt_name, dense_update):
    mk = lambda: {"sgd": optim.GradientDescent(0.3), "adagrad": optim.Adagrad(0.2, 1.0),
                  "adam": optim.Adam(0.01)}[opt_name]
    ref = _run("host", run_option, mk(), 5)
    got = _run("nvlink", run_option, mk(), 5, dense_update=dense_update)
    assert all(n > 0.05 for n in ref[1])                     # the clip is active
    _same(got, ref, 1e-4)


def test_engine_sparse_only_rule_matches_host_oracle():
    ref = _run("host", "HYBRID", optim.Adagrad(0.2, 1.0), 4, params=["emb.*"], max_norm=0.02)
    got = _run("nvlink", "HYBRID", optim.Adagrad(0.2, 1.0), 4, params=["emb.*"],
               max_norm=0.02)
    _same(got, ref, 1e-4)


def test_engine_joint_clip_cuda_graph_matches_eager():
    eager = _run("nvlink", "HYBRID", optim.Adagrad(0.2, 1.0), 8)
    replay = _run("nvlink", "HYBRID", optim.Adagrad(0.2, 1.0), 8, graph=True)
    _same(replay, eager, 1e-5)


def test_engine_joint_clip_nccl_protocol_refused():
    model = MLPWithEmbedding(64)
    g = parallax.Graph(model, optimizer=optim.Adagrad(0.2, 1.0), grad_rules=[
        parallax.ClipByGlobalNorm(1.0, include_sparse=True)])
    cfg = parallax.Config(sess_config={"fabric": "nvlink"})
    cfg.communication_config = parallax.CommunicationConfig(
        parallax.PSConfig(protocol="nccl"))
    with pytest.raises(NotImplementedError, match="library"):
        parallax.parallel_run(g, "localhost:0", sync=True, parallax_config=cfg)
