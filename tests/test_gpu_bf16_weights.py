"""bf16 master rows (sess_config["sparse_weights"] = "bf16") on the NVLink fabric: the owner
kernel against `optim.apply_sparse_rows_` with the same stochastic rounding (bit for bit on
exact SGD updates), layout invariance, storage, drift, the engine against the host oracle,
CUDA-graph replay, sharded checkpoints and the fused full-softmax evaluation."""
import pytest
import torch
import torch.nn.functional as F

import parallax_b200 as parallax
from parallax_b200 import optim
from parallax_b200.models.simple import MLPWithEmbedding
from tests import sparse_plane_ref

pytestmark = pytest.mark.gpu

DS = (1, 64, 500, 512)
BF = {"sparse_weights": "bf16", "sparse_blocks": 4, "sparse_early_push": False}


def _groups(world, V, Ds, P, opt, run_option, local_agg, W0, opts=None):
    from tests.gpu_utils import make_world
    from parallax_b200.parallel import modes
    from parallax_b200.parallel.nvlink_backend import NVSparseTable, NVSparseGroup
    fabs = make_world(world)
    route = modes.route_for(run_option, True)
    cfg = parallax.Config(run_option=run_option)
    cfg.communication_config = parallax.CommunicationConfig(
        parallax.PSConfig(local_aggregation=local_agg))
    graph = parallax.Graph(torch.nn.Linear(1, 1), optimizer=optim.Adagrad(0.1),
                           sparse_optimizer=opt)
    groups = []
    for f in fabs:
        tabs = [NVSparseTable("t%d" % k, w, P, "mod", opt, f, route, graph, cfg,
                              options=dict(BF, **(opts or {})), out_dtype=torch.bfloat16,
                              auto_group=False) for k, w in enumerate(W0)]
        groups.append(NVSparseGroup(tabs))
    return fabs, groups


def _gids(t):
    lay = t.layout
    gid = torch.full((lay.rows_local,), -1, dtype=torch.int64)
    g, l = lay.global_ids_of_owner(0 if t.replicated else t.rank)
    gid[l] = g
    return gid


def _step(groups, ids_per_rank, grads_per_rank, step):
    for grp, ids, gs in zip(groups, ids_per_rank, grads_per_rank):
        _, pend = grp.lookup(ids.cuda())
        grp.add_pending(pend, [g.cuda() for g in gs])
        grp.begin_step(step)
    torch.cuda.synchronize()
    for grp in groups:
        grp.stage_push(step)
    torch.cuda.synchronize()
    # each owner's receive rings merged per row (fp32 of the fp64 sum): [(local rows, rows)]
    merged = [[(r.rows, r.sum.float()) for r in sparse_plane_ref.merged(grp)] for grp in groups]
    for grp in groups:
        grp.stage_apply(step)
    torch.cuda.synchronize()
    return merged


RULES = {
    "sgd": lambda: optim.GradientDescent(2.0 ** -3),
    "adagrad": lambda: optim.Adagrad(0.05, 0.1),
    "adam": lambda: optim.Adam(0.01),
    "ftrl": lambda: optim.Ftrl(0.05, l1_regularization_strength=0.001),
    "rowwise_adagrad": lambda: optim.RowWiseAdagrad(0.05, 0.1, epsilon=1e-3),
}


@pytest.mark.parametrize("kind", sorted(RULES))
@pytest.mark.parametrize("world", [1, 2, 4, 8])
@pytest.mark.parametrize("layout", ["HYBRID", "MPI"])
@pytest.mark.parametrize("wire", ["fp32", "bf16"])
@pytest.mark.parametrize("local_agg", [True, False])
def test_owner_kernel_matches_oracle(kind, world, layout, wire, local_agg):
    """A group of four tables (D = 1, 64, 500, 512), two steps.  Weights k·2^-8 and gradients
    k·2^-4 (|k| small): with SGD at lr = 2^-3 every fp32 value is exact, so the rounded
    tables must equal the oracle's bit for bit; with the other rules fewer than 0.1 % of the
    elements differ from the oracle (see below for how far)."""
    V, P, n = 701, 8, 300
    opt = RULES[kind]()
    gen = torch.Generator().manual_seed(world * 7 + len(kind))
    W0 = [torch.randint(-256, 257, (V, D), generator=gen).float() * 2.0 ** -8 for D in DS]
    fabs, groups = _groups(world, V, DS, P, opt, layout, local_agg, W0)
    for grp in groups:
        grp._ensure_capacity(n)
    for grp in groups:
        grp.warm(n)
    torch.cuda.synchronize()
    for grp in groups:
        for t, w in zip(grp.tables, W0):
            assert t.table.dtype == torch.bfloat16 and tuple(t.table.shape) == \
                (t.layout.rows_local, t.Dps)
    gdt = torch.bfloat16 if wire == "bf16" else torch.float32
    oracle = [[(t.table[:, :t.D].cpu().clone(),
                [s.cpu()[:, :t.slot_dim].clone() for s in t.slots]) for t in grp.tables]
              for grp in groups]
    for step in (1, 2):
        ids = [torch.randint(0, V, (n,), generator=gen) for _ in groups]
        for i in ids:
            i[:30] = i[0]
        grads = [[(torch.randint(-4, 5, (n, D), generator=gen).float() * 2.0 ** -4).to(gdt)
                  for D in DS] for _ in groups]
        merged = _step(groups, ids, grads, step)
        hp = opt.hyper(step)
        for r, grp in enumerate(groups):
            for k, t in enumerate(grp.tables):
                u, m = merged[r][k]
                w, slots = oracle[r][k]
                optim.apply_sparse_rows_(opt.kind, w, u, m, slots, hp, t.sr_seed, _gids(t)[u])
                got = t.table.cpu()
                assert bool((got[:, t.D:] == 0).all())                  # padding stays zero
                got = got[:, :t.D]
                if kind == "sgd":
                    assert torch.equal(got.view(torch.int16), w.view(torch.int16)), (r, k)
                else:
                    # fewer than 0.1 % of the elements differ.  Adam and FTRL leave a few
                    # elements (at most 4 per table seen, not the same ones on every run) more
                    # than one bf16 ulp off where an update cancels the weight; those, and
                    # their slots, stay within the bf16-boundary tolerance of the fp32-master
                    # tests.  Adagrad and row-wise Adagrad stay within one ulp.
                    a, b = got.double(), w.double()
                    ulp = 2.0 ** (torch.floor(torch.log2(b.abs().clamp_min(1e-30))) - 7)
                    far = (a - b).abs() > ulp
                    assert int(far.sum()) <= (8 if kind in ("adam", "ftrl") else 0), \
                        (r, k, int(far.sum()))
                    torch.testing.assert_close(a, b, rtol=2e-2, atol=2e-3)
                    assert float((a != b).double().mean()) < 1e-3, (r, k)
                    for s_got, s_want in zip(t.slots, slots):
                        torch.testing.assert_close(s_got.cpu()[:, :s_want.shape[1]], s_want,
                                                   rtol=2e-2, atol=2e-3)
    for f in fabs:
        f.close()


def _logical(groups):
    """The logical table of every member, assembled from the owners' local rows."""
    out = []
    for k in range(len(groups[0].tables)):
        t0 = groups[0].tables[k]
        full = torch.zeros(t0.V, t0.D, dtype=torch.bfloat16)
        for grp in (groups[:1] if t0.replicated else groups):
            g, rows = grp.tables[k].local_rows("weight")
            full[g] = rows
        out.append(full)
    return out


def _exact_run(world, P, layout="HYBRID", steps=3):
    V, n_total = 997, 512
    opt = optim.GradientDescent(2.0 ** -3)
    gen = torch.Generator().manual_seed(5)
    W0 = [torch.randint(-256, 257, (V, D), generator=gen).float() * 2.0 ** -8 for D in (64, 8)]
    fabs, groups = _groups(world, V, (64, 8), P, opt, layout, True, W0)
    n = n_total // world
    for grp in groups:
        grp._ensure_capacity(n)
    for grp in groups:
        grp.warm(n)
    for step in range(1, steps + 1):
        ids = torch.randint(0, V, (n_total,), generator=gen)
        grads = [torch.randint(-4, 5, (n_total, D), generator=gen).float() * 2.0 ** -4
                 for D in (64, 8)]
        _step(groups, [ids[r * n:(r + 1) * n] for r in range(world)],
              [[g[r * n:(r + 1) * n] for g in grads] for r in range(world)], step)
    res = _logical(groups)
    replicas = [[t.table.cpu().clone() for t in grp.tables] for grp in groups]
    for f in fabs:
        f.close()
    return res, replicas


def test_layout_invariance():
    """Exact updates: the same batches at W = 1, 2, 4 and P = 3, 5 give bit-identical logical
    tables (the rounding is keyed by global ids only); AR replicas are bit-identical."""
    ref, _ = _exact_run(1, 3)
    for world, P in ((1, 5), (2, 3), (2, 5), (4, 3), (4, 5)):
        got, _ = _exact_run(world, P)
        for a, b in zip(got, ref):
            assert torch.equal(a.view(torch.int16), b.view(torch.int16)), (world, P)
    got, replicas = _exact_run(4, 3, layout="MPI")
    for a, b in zip(got, ref):
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))
    for rep in replicas[1:]:
        for a, b in zip(rep, replicas[0]):
            assert torch.equal(a.view(torch.int16), b.view(torch.int16))


@pytest.mark.parametrize("kind", ["adagrad", "adam", "rowwise_adagrad"])
@pytest.mark.parametrize("D", [1, 64, 500])
def test_storage(kind, D):
    """No fp32 table: the bf16 master and the fp32 slots take exactly `table_row_bytes` per
    local row on the symmetric heap; lookups return the master's values."""
    from parallax_b200 import ops
    V, P = 1000, 4
    opt = RULES[kind]()
    W0 = [torch.randn(V, D, generator=torch.Generator().manual_seed(D))]
    heap0 = ops.lib().px_symm_live_bytes()
    fabs, groups = _groups(1, V, (D,), P, opt, "HYBRID", True, W0)
    t = groups[0].tables[0]
    nbytes = t.table.numel() * 2 + sum(s.numel() * 4 for s in t.slots)
    assert nbytes == t.layout.rows_local * optim.table_row_bytes(kind, D, torch.bfloat16)
    assert t.shadow_buf is t.tab_buf and t.table.dtype == torch.bfloat16
    assert ops.lib().px_symm_live_bytes() - heap0 >= nbytes
    ids = torch.arange(V).cuda()
    rows, _ = t.lookup(ids, record=False)
    assert rows.dtype == torch.bfloat16
    assert torch.equal(rows.cpu().float(), W0[0].to(torch.bfloat16).float())
    assert torch.equal(t.full_weight(), W0[0].to(torch.bfloat16).float())
    for f in fabs:
        f.close()


def test_drift_on_device():
    """1000 SGD updates of 2^-12 on 64 Ki weights of 1.0 through the owner kernel: the mean
    reaches 1 - 1000·2^-12 within 4 sigma (round-to-nearest would leave every weight at 1)."""
    import math
    V, D, steps = 1024, 64, 1000
    opt = optim.GradientDescent(2.0 ** -12)
    fabs, groups = _groups(1, V, (D,), 1, opt, "HYBRID", True, [torch.ones(V, D)])
    grp = groups[0]
    ids = torch.arange(V).cuda()
    g = torch.ones(V, D, device="cuda")
    grp._ensure_capacity(V)
    grp.warm(V)
    for s in range(1, steps + 1):
        _, pend = grp.lookup(ids)
        grp.add_pending(pend, [g])
        grp.begin_step(s)
        grp.stage_push(s)
        grp.stage_apply(s)
    torch.cuda.synchronize()
    w = grp.tables[0].table[:, :D].double()
    want = 1.0 - steps * 2.0 ** -12
    sigma = math.sqrt(steps * (2.0 ** -8) ** 2 / 4 / (V * D))
    assert abs(float(w.mean()) - want) <= 4 * sigma
    for f in fabs:
        f.close()


# ------------------------------------------------------------------ engine level
def _batch(gen, unique):
    if unique:
        ids = torch.randperm(64, generator=gen)[:24].view(8, 3)
    else:
        ids = torch.randint(0, 64, (8, 3), generator=gen)
        ids[:, 0] = 5
    return ids, torch.randint(0, 4, (8,), generator=gen)


def _run(fabric, run_option, steps, graph=False, clip=False, partitions=3, weights="bf16",
         unique=False, hook=None, ckpt=None, protocol="nvlink", first_step=0):
    torch.manual_seed(0)
    model = MLPWithEmbedding(64, partitioner=parallax.get_partitioner(partitions))
    rules = [parallax.ClipByGlobalNorm(0.05, include_sparse=True)] if clip else []
    g = parallax.Graph(model, optimizer=optim.Adagrad(0.2, 1.0),
                       sparse_optimizer=optim.Adagrad(0.2, 0.5), grad_rules=rules)
    sc = {"fabric": fabric, "cuda_graph": graph, "sparse_weights": weights}
    if fabric == "nvlink":
        sc["compute_dtype"] = "bf16"
    cfg = parallax.Config(run_option=run_option, sess_config=sc, search_partitions=False)
    cfg.communication_config = parallax.CommunicationConfig(parallax.PSConfig(protocol=protocol))
    sess, *_ = parallax.parallel_run(g, "localhost:0", sync=True, parallax_config=cfg)
    if ckpt is not None:
        from parallax_b200 import checkpoint as ck
        ck.load_sharded(sess.engine, ckpt)
    gen = torch.Generator().manual_seed(0)
    for _ in range(first_step):
        _batch(gen, unique)
    losses = []
    for _ in range(steps):
        ids, labels = _batch(gen, unique)
        loss, _ = sess.run(["loss", "train_op"], {"ids": [ids], "labels": [labels]})
        losses.append(float(loss[0]))
    out = hook(sess.engine) if hook is not None else None
    sd = sess.engine.state_dict()
    sess.close()
    return losses, sd, out


@pytest.mark.parametrize("run_option", ["HYBRID", "PS", "MPI"])
@pytest.mark.parametrize("clip", [False, True])
def test_engine_matches_host_oracle(run_option, clip):
    """The NVLink run computes in bf16, the host oracle in fp32: both keep bf16 masters."""
    ref = _run("host", run_option, 6, clip=clip)
    got = _run("nvlink", run_option, 6, clip=clip)
    w_got = got[1]["sparse"]["emb.weight"]["weight"]
    assert torch.equal(w_got, w_got.to(torch.bfloat16).float())
    torch.testing.assert_close(got[0], ref[0], rtol=2e-2, atol=2e-2)
    torch.testing.assert_close(w_got, ref[1]["sparse"]["emb.weight"]["weight"],
                               rtol=2e-2, atol=2e-3)


def test_engine_nccl_protocol_arm():
    got = _run("nvlink", "HYBRID", 4, protocol="nccl")
    ref = _run("nvlink", "HYBRID", 4)
    torch.testing.assert_close(got[0], ref[0], rtol=0, atol=0)


def test_cuda_graph_replay_matches_eager():
    eager = _run("nvlink", "HYBRID", 10, unique=True)
    replay = _run("nvlink", "HYBRID", 10, graph=True, unique=True)
    assert eager[0] == replay[0]
    for k in ("weight", "slots"):
        a, b = replay[1]["sparse"]["emb.weight"][k], eager[1]["sparse"]["emb.weight"][k]
        assert all(torch.equal(x, y) for x, y in zip(a if k == "slots" else [a],
                                                      b if k == "slots" else [b]))


def test_checkpoint_restore_continues_bit_identically(tmp_path):
    """Save after 3 steps, restore at P = 5, run 3 more: the same as 6 uninterrupted steps
    (unique ids: the push has no fp32 atomics to reorder)."""
    from parallax_b200 import checkpoint as ck
    d = str(tmp_path / "model.ckpt-3")
    _run("nvlink", "HYBRID", 3, unique=True, hook=lambda e: ck.save_sharded(e, d, True))
    man = ck.read_manifest(d)
    assert man["sparse"]["emb.weight"]["weight_dtype"] == "bfloat16"
    sh = torch.load(d + "/" + man["sparse"]["emb.weight"]["files"][0], weights_only=False)
    assert sh["weight"].dtype == torch.bfloat16
    full = _run("nvlink", "HYBRID", 6, unique=True)
    resumed = _run("nvlink", "HYBRID", 3, unique=True, partitions=5, ckpt=d, first_step=3)
    assert resumed[0] == full[0][3:]
    assert torch.equal(resumed[1]["sparse"]["emb.weight"]["weight"],
                       full[1]["sparse"]["emb.weight"]["weight"])
    # cross-dtype restores: bf16 -> fp32 exact, fp32 -> bf16 round to nearest even
    as32 = _run("nvlink", "HYBRID", 0, weights="fp32", ckpt=d)[1]["sparse"]["emb.weight"]
    tab = ck.assemble_table(d, "emb.weight")
    assert tab["weight"].dtype == torch.float32
    assert torch.equal(as32["weight"], tab["weight"])
    d32 = str(tmp_path / "model.ckpt-2")
    w32 = _run("nvlink", "HYBRID", 2, weights="fp32",
               hook=lambda e: ck.save_sharded(e, d32, True))[1]["sparse"]["emb.weight"]
    assert "weight_dtype" in ck.read_manifest(d32)["sparse"]["emb.weight"]
    as16 = _run("nvlink", "HYBRID", 0, ckpt=d32)[1]["sparse"]["emb.weight"]
    assert torch.equal(as16["weight"], w32["weight"].to(torch.bfloat16).float())
    torch.testing.assert_close(as16["slots"][0], w32["slots"][0], rtol=0, atol=0)


# ------------------------------------------------------------- full softmax
@pytest.mark.parametrize("world,V,P,K,N", [(1, 1000, 1, 32, 5), (2, 3001, 5, 512, 640),
                                           (4, 2999, 7, 136, 300)])
def test_full_softmax_bf16_master(world, V, P, K, N):
    """The fused evaluation reads the bf16 weight master through its shadow descriptor and the
    bf16 bias master (non-zero, width 1) widened to fp32: it matches fp64 on the same rows."""
    from tests.gpu_utils import make_world
    from parallax_b200.parallel import modes
    from parallax_b200.parallel.nvlink_backend import NVSparseTable, NVSparseGroup
    fabs = make_world(world)
    route = modes.route_for("HYBRID", True)
    cfg = parallax.Config(run_option="HYBRID")
    opt = optim.Adagrad(0.2, 1.0)
    graph = parallax.Graph(torch.nn.Linear(1, 1), optimizer=opt)
    g = torch.Generator().manual_seed(K)
    Wt = torch.randn(V, K, generator=g) / K ** 0.5
    Bt = torch.randn(V, 1, generator=g) + 0.5
    groups = []
    for f in fabs:
        tw = NVSparseTable("w", Wt, P, "mod", opt, f, route, graph, cfg, options=BF,
                           out_dtype=torch.bfloat16, auto_group=False)
        tb = NVSparseTable("b", Bt, P, "mod", opt, f, route, graph, cfg, options=BF,
                           out_dtype=torch.bfloat16, auto_group=False)
        groups.append(NVSparseGroup([tw, tb]))
    torch.cuda.synchronize()
    x = torch.randn(N, K, generator=g).bfloat16()
    targets = torch.randint(0, V, (N,), generator=g)
    w16, b16 = Wt.bfloat16().double(), Bt.bfloat16().double()
    ref = F.cross_entropy(x.double() @ w16.t() + b16.t(), targets, reduction="none").float()
    for grp in groups:
        nll = grp.full_softmax_nll(x.cuda(), targets.cuda())
        torch.cuda.synchronize()
        torch.testing.assert_close(nll.cpu(), ref, rtol=1e-5, atol=1e-3)
    for f in fabs:
        f.close()


def test_engine_full_softmax_takes_the_fused_path(monkeypatch):
    """LM1B with bf16 masters: the engine's gate picks the fused kernel (no table gather) after
    training steps, and it agrees with the gather + matmul composition."""
    from parallax_b200.models.lm1b import LM1B, lm1b_graph
    from parallax_b200.parallel.engine import full_softmax_composition
    from parallax_b200.parallel.nv_sparse import NVSparseGroup
    calls = []
    orig = NVSparseGroup.full_softmax_nll
    monkeypatch.setattr(NVSparseGroup, "full_softmax_nll",
                        lambda self, x, t: calls.append(1) or orig(self, x, t))
    torch.manual_seed(0)
    V = 1003
    m = LM1B(vocab_size=V, emb_size=32, state_size=64, projected_size=32, num_sampled=16,
             num_steps=4, num_shards=3, keep_prob=1.0)
    sc = {"fabric": "nvlink", "compute_dtype": "bf16", "sparse_weights": "bf16"}
    sess, *_ = parallax.parallel_run(lm1b_graph(m, batch_size=128), "localhost:0",
                                     parallax_config=parallax.Config(sess_config=sc))
    m = sess.engine.model
    assert m.softmax_b.table.weight_dtype == torch.bfloat16
    gen = torch.Generator().manual_seed(1)
    for _ in range(3):
        x = torch.randint(0, V, (128, 4), generator=gen)
        sess.run(["loss", "train_op"], {"x": [x], "y": [torch.roll(x, -1, dims=1)]})
    b = m.softmax_b.table.full_weight()
    assert bool((b != 0).any())
    x = torch.randn(256, 32, device="cuda").bfloat16()
    t = torch.randint(0, V, (256,), device="cuda")
    with torch.no_grad():
        fused = parallax.nn.full_softmax_nll(x, t, m.softmax_w, m.softmax_b)
        comp = full_softmax_composition(x, t, m.softmax_w, m.softmax_b)
    torch.cuda.synchronize()
    assert calls == [1]
    torch.testing.assert_close(fused.cpu(), comp.cpu(), rtol=0, atol=3e-2)
    sess.close()
