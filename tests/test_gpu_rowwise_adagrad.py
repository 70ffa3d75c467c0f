"""Row-wise Adagrad on the NVLink fabric: the family-2 owner kernel against an fp64 merge of
the receive rings with the rule applied, the clipped apply, and the engine against the
host-fabric oracle (eager and under CUDA-graph replay), checkpoints and repartition."""
import numpy as np
import pytest
import torch

import parallax_b200 as parallax
from parallax_b200 import optim
from parallax_b200.models.simple import MLPWithEmbedding

pytestmark = pytest.mark.gpu

DIMS = {"narrow": (1, 3, 64), "wide": (500, 1024), "lm1b": (512, 1)}


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
    graph = parallax.Graph(torch.nn.Linear(1, 1), optimizer=optim.Adagrad(0.1),
                           sparse_optimizer=opt,
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


def _merged_reference(grp):
    """fp64 merge of this owner's receive rings × the owner-side factor: {table k: (local
    rows, merged rows [n, D])} — what the owner kernel hands to the optimizer."""
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
        a = (1.0 / grp.world) if t.average else 1.0
        a = a if grp.boundary else a * t.scale
        out.append((u, (m * a)[:, :t.D]))
    return out


def _rowwise_fp64(w, s, rows, g, hp):
    """The rule in fp64 on copies of the fp32 state: w [R, D], s [R, 1]."""
    w, s = w.double(), s.double()
    gs = g * hp[optim.HP_GSCALE]
    s[rows] += (gs * gs).mean(dim=1, keepdim=True)
    w[rows] -= hp[optim.HP_LR] * gs / (s[rows].sqrt() + hp[optim.HP_EPS])
    return w, s


@pytest.mark.parametrize("world", [1, 2, 4, 8])
@pytest.mark.parametrize("layout", ["HYBRID", "MPI"])
@pytest.mark.parametrize("wire", ["fp32", "bf16"])
@pytest.mark.parametrize("local_agg", [True, False])
@pytest.mark.parametrize("dims", sorted(DIMS))
def test_owner_kernel_rowwise(world, layout, wire, local_agg, dims):
    """Two steps per case; the second is a clipped apply (hp[HP_GSCALE] × 0.37 through
    `clip_hp`, as a joint ClipByGlobalNorm issues it) after the sparse norm kernel ran on
    the same rings.  Master rows, accumulators and the bf16 shadow against fp64; rows no
    source touched keep their exact bits."""
    V, P, n = 701, 8, 300
    Ds = DIMS[dims]
    opt = optim.RowWiseAdagrad(0.3, initial_accumulator_value=0.2, epsilon=1e-3)
    bf16 = wire == "bf16"
    fabs, groups = _groups(world, V, Ds, P, opt, layout, average=(world == 4),
                           local_agg=local_agg,
                           out_dtype=torch.bfloat16 if bf16 else torch.float32, scale=2.0)
    for grp in groups:
        grp._ensure_capacity(n)
    for grp in groups:
        grp.warm(n)
    torch.cuda.synchronize()
    for grp in groups:
        for t in grp.tables:
            assert tuple(t.slots[0].shape) == (t.layout.rows_local, 1)
    gen = torch.Generator().manual_seed(11)
    clip = torch.full((1,), 0.37, device="cuda")
    for step in (1, 2):
        before = [[(t.table.cpu().clone(), t.slots[0].cpu().clone()) for t in grp.tables]
                  for grp in groups]
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
        for grp in groups:
            grp.stage_push(step)
        torch.cuda.synchronize()
        merged = [_merged_reference(grp) for grp in groups]
        hp = opt.hyper(step)
        if step == 2:
            sums = [torch.zeros(4, device="cuda") for _ in groups]
            torch.cuda.synchronize()
            for grp, s in zip(groups, sums):
                grp.stage_norm(s)
            torch.cuda.synchronize()
            for r, grp in enumerate(groups):
                want = sum(float((m ** 2).sum()) for _, m in merged[r])
                assert abs(float(sums[r][0]) - want) <= 1e-5 * max(want, 1e-30)
            for grp in groups:
                grp.stage_apply(step, hp=grp.clip_hp(clip))
            hp = list(hp)
            hp[optim.HP_GSCALE] *= 0.37
        else:
            for grp in groups:
                grp.stage_apply(step)
        torch.cuda.synchronize()
        for r, grp in enumerate(groups):
            assert int(grp.ctl[0]) == step
            assert bool((grp.slotmap == -1).all())
            for k, t in enumerate(grp.tables):
                u, m = merged[r][k]
                w0, s0 = before[r][k]
                w_ref, s_ref = _rowwise_fp64(w0[:, :t.D], s0, u, m, hp)
                w, s = t.table.cpu(), t.slots[0].cpu()
                torch.testing.assert_close(s.double(), s_ref, rtol=1e-5, atol=1e-7)
                torch.testing.assert_close(w[:, :t.D].double(), w_ref, rtol=1e-5, atol=1e-6)
                assert bool((w[:, t.D:] == 0).all())                 # padding stays zero
                untouched = torch.ones(w.shape[0], dtype=torch.bool)
                untouched[u] = False
                assert torch.equal(w[untouched], w0[untouched])
                assert torch.equal(s[untouched], s0[untouched])
                if t.use_shadow:
                    torch.testing.assert_close(t.shadow[:, :t.D].cpu(),
                                               w[:, :t.D].to(torch.bfloat16), rtol=0, atol=0)
    for f in fabs:
        f.close()


# ------------------------------------------------------------------ engine level
def _run(fabric, run_option, steps, graph=False, clip=False, partitions=3, hook=None):
    torch.manual_seed(0)
    model = MLPWithEmbedding(64, partitioner=parallax.get_partitioner(partitions))
    rules = [parallax.ScaleGradients(2.0, params=["emb.weight"])]
    if clip:
        rules.append(parallax.ClipByGlobalNorm(0.05, include_sparse=True))
    g = parallax.Graph(model, optimizer=optim.Adagrad(0.2, 1.0),
                       sparse_optimizer=optim.RowWiseAdagrad(0.2, 0.5), grad_rules=rules)
    cfg = parallax.Config(run_option=run_option, sess_config={
        "fabric": fabric, "cuda_graph": graph})
    sess, *_ = parallax.parallel_run(g, "localhost:0", sync=True, parallax_config=cfg)
    gen = torch.Generator().manual_seed(0)
    losses = []
    for _ in range(steps):
        ids = torch.randint(0, 64, (8, 3), generator=gen)
        ids[:, 0] = 5
        labels = torch.randint(0, 4, (8,), generator=gen)
        loss, _ = sess.run(["loss", "train_op"], {"ids": [ids], "labels": [labels]})
        losses.append(loss[0])
    out = hook(sess.engine) if hook is not None else None
    sd = sess.engine.state_dict()
    sess.close()
    return losses, sd, out


def _same(a, b, rtol):
    np.testing.assert_allclose(a[0], b[0], rtol=rtol, atol=rtol * 0.1)
    for n, w in b[1]["dense"]["master"].items():
        torch.testing.assert_close(a[1]["dense"]["master"][n], w, rtol=rtol, atol=rtol * 0.1)
    for k in ("weight", "slots"):
        torch.testing.assert_close(a[1]["sparse"]["emb.weight"][k],
                                   b[1]["sparse"]["emb.weight"][k], rtol=rtol, atol=rtol * 0.1)


@pytest.mark.parametrize("run_option", ["HYBRID", "PS", "MPI"])
@pytest.mark.parametrize("clip", [False, True])
def test_engine_matches_host_oracle(run_option, clip):
    ref = _run("host", run_option, 6, clip=clip)
    got = _run("nvlink", run_option, 6, clip=clip)
    assert tuple(got[1]["sparse"]["emb.weight"]["slots"][0].shape) == (64, 1)
    _same(got, ref, 1e-4)


def test_engine_cuda_graph_matches_eager():
    eager = _run("nvlink", "HYBRID", 10)
    replay = _run("nvlink", "HYBRID", 10, graph=True)
    _same(replay, eager, 1e-6)


def test_checkpoint_round_trip_and_repartition(tmp_path):
    """Sharded save of a row-wise table, the offline reader's [V, 1] slot, a reload at
    another partition count, and `repartition` in place."""
    from parallax_b200 import checkpoint as ckpt

    def save(eng):
        d = str(tmp_path / ("model.ckpt-%d" % eng.global_step))
        ckpt.save_sharded(eng, d, True)
        return d

    losses, sd, d = _run("nvlink", "HYBRID", 4, hook=save)
    tab = ckpt.assemble_table(d, "emb.weight")
    assert tuple(tab["slots"][0].shape) == (64, 1)
    torch.testing.assert_close(tab["weight"], sd["sparse"]["emb.weight"]["weight"])
    torch.testing.assert_close(tab["slots"][0], sd["sparse"]["emb.weight"]["slots"][0])

    def reload(eng):
        ckpt.load_sharded(eng, d)
        return eng.state_dict()

    got = _run("nvlink", "HYBRID", 0, partitions=5, hook=reload)[2]
    for k in ("weight", "slots"):
        torch.testing.assert_close(got["sparse"]["emb.weight"][k], sd["sparse"]["emb.weight"][k])

    def repart(eng):
        before = eng.state_dict()
        eng.repartition(7)
        assert eng.tables["emb.weight"].layout.P == 7
        return before, eng.state_dict()

    before, after = _run("nvlink", "HYBRID", 3, hook=repart)[2]
    for k in ("weight", "slots"):
        torch.testing.assert_close(after["sparse"]["emb.weight"][k],
                                   before["sparse"]["emb.weight"][k])
