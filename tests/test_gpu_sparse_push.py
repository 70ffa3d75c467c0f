"""What the sparse push kernel writes, read back from the owners' receive rings before any
owner kernel runs, on a world simulated inside one GPU.

Every gradient value is k·2^-4 with |k| <= 4 and no row of one sender sums more than 60 of
them, so every fp32 sum is exact, and so is one rounding of it to bf16: whatever order the
kernel adds duplicates in, the rows must match the reference bit for bit."""
import pytest
import torch

import parallax_b200 as parallax
from parallax_b200 import ops, optim
from parallax_b200.graph import Graph, ScaleGradients

pytestmark = pytest.mark.gpu


def _groups(world, widths, opt, run_option="HYBRID", sync=True, scale=1.0, boundary=True,
            local_agg=True, V=503, P=8, cap=4096, blocks=4):
    from tests.gpu_utils import make_world
    from parallax_b200.parallel import modes
    from parallax_b200.parallel.nvlink_backend import NVSparseTable, NVSparseGroup
    fabs = make_world(world)
    route = modes.route_for(run_option, sync)
    cfg = parallax.Config(run_option=run_option)
    cfg.communication_config = parallax.CommunicationConfig(
        parallax.PSConfig(local_aggregation=local_agg,
                          boundary_between_workers_and_servers=boundary))
    g = torch.Generator().manual_seed(7)
    W0 = [torch.randn(V, D, generator=g) for D in widths]
    graph = Graph(torch.nn.Linear(1, 1), optimizer=opt, grad_rules=[ScaleGradients(scale)])
    names = ["t%d" % i for i in range(len(widths))]
    o = {"sparse_capacity": {nm: cap for nm in names}, "sparse_early_push": False,
         "sparse_blocks": blocks}
    groups = [NVSparseGroup([NVSparseTable(nm, w, P, "mod", opt, f, route, graph, cfg,
                                           options=o, auto_group=False)
                             for nm, w in zip(names, W0)]) for f in fabs]
    return fabs, groups, W0


def _warm(groups, n):
    """Every rank allocates its rings before any rank reads its peers' pointers."""
    for grp in groups:
        grp._ensure_capacity(n)
    for grp in groups:
        grp.warm(n)
    torch.cuda.synchronize()


def _exact_grads(gen, n, D, dtype):
    return (torch.randint(-4, 5, (n, D), generator=gen).float() / 16).to(dtype)


def _step_inputs(gen, groups, V, n, dtype, r):
    ids = torch.randint(0, V, (n,), generator=gen)
    ids[:40] = 5 + r                   # duplicates inside a rank
    ids[40:60] = 17                    # and across ranks
    ids[70] = V + 5                    # out of range: pend carries -1
    grads = [_exact_grads(gen, n, t.D, dtype) for t in groups[r].tables]
    return ids, grads


def _lookup_and_stage(groups, step, inputs):
    toks = []
    for grp, (ids, _) in zip(groups, inputs):
        _, pend = grp.lookup(ids.cuda())
        toks.append(pend)
    torch.cuda.synchronize()
    for grp, tok, (_, grads) in zip(groups, toks, inputs):
        grp.begin_step(step)
        grp.add_pending(tok, [g.cuda() for g in grads])
    torch.cuda.synchronize()


def _check_push_stamps(grp):
    d = grp.device_times()
    ph = [d["push_start"]] + d["push_phases"][:6]
    assert all(a <= b for a, b in zip(ph, ph[1:])), ph
    assert d["pushed"] >= d["push_start"] > 0


def _check_rings(groups, inputs, V, scale, overflow=False):
    """Every (owner, source) ring against the source's positions routed to that owner."""
    g0 = groups[0]
    L, W, cap = g0.layout, g0.world, g0.cap
    R = ops.sparse_abi()["hdr_words"] // 3
    wire = g0.wire_dtype
    rows_local = L.rows_local
    for o, grp in enumerate(groups):
        assert grp.wire_dtype == wire
        counts = grp.hdr_buf.tensor(torch.int32)[2 * R:2 * R + W].cpu()
        ring_ids = grp.ids_buf.tensor(torch.int32, W * cap).view(W, cap).cpu()
        for s, (ids, grads) in enumerate(inputs):
            cnt = int(counts[s])
            rows = ring_ids[s, :cnt].long()
            sel = (ids >= 0) & (ids < V)
            if not L.replicated:
                sel &= L.owner_of(ids.clamp(0, V - 1)) == o
            local = L.local_row_of(ids[sel])
            # 1. every entry is a row this source pushed and this owner owns
            assert bool(torch.isin(rows, local).all()), (o, s)
            if grp.local_aggregation and not overflow:
                assert rows.unique().numel() == cnt, (o, s)      # one entry per row
            if not grp.local_aggregation:
                assert cnt == local.numel(), (o, s)              # one entry per position
            for t, g in zip(grp.tables, grads):
                ring = t.ring_buf.tensor(wire, W * cap * t.Dp).view(W, cap, t.Dp)[s, :cnt]
                ring = ring.float().cpu()
                # 3. padding columns stay zero
                assert not ring[:, t.D:].any(), (o, s, t.name)
                # 2. grouped by row, the entries sum to the (sender-scaled) reference exactly
                ref = g[sel].float()
                if grp.boundary:
                    ref = ref * scale
                want = torch.zeros(rows_local, t.D).index_add_(0, local, ref)
                got = torch.zeros(rows_local, t.D).index_add_(0, rows, ring[:, :t.D])
                assert torch.equal(got, want), (o, s, t.name)
    for grp in groups:
        # 5. the flush pass leaves every staging row zero
        for t in grp.tables:
            assert not t.staging.any(), t.name
        _check_push_stamps(grp)


def _push_check_apply(groups, inputs, step, V, scale, overflow=False):
    _lookup_and_stage(groups, step, inputs)
    for grp in groups:
        grp.stage_push(step)
    torch.cuda.synchronize()
    _check_rings(groups, inputs, V, scale, overflow)
    for grp in groups:
        grp.stage_apply(step)
    torch.cuda.synchronize()


@pytest.mark.parametrize("world,run_option", [(2, "HYBRID"), (3, "HYBRID"), (4, "HYBRID"),
                                              (6, "HYBRID"), (2, "MPI"), (4, "MPI")])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("boundary", [True, False])
@pytest.mark.parametrize("local_agg", [True, False])
@pytest.mark.parametrize("D,scale", [(36, 0.5), (64, 1.0), (64, 0.5)])
def test_push_rings_exact(world, run_option, dtype, boundary, local_agg, D, scale):
    """D = 36 ships through the generic float4 path, D = 64 (bf16 wire, partitioned) through
    16-byte copies; fp32 wire unless bf16 gradients cross with the boundary optimisation.
    W = 3 and 6 place the P = 8 partitions unevenly over the owners."""
    V, n = 503, 300
    fabs, groups, _ = _groups(world, [D], optim.Adagrad(0.2, 1.0), run_option=run_option,
                              scale=scale, boundary=boundary, local_agg=local_agg, V=V)
    _warm(groups, n)
    gen = torch.Generator().manual_seed(11)
    for step in (1, 2):
        inputs = [_step_inputs(gen, groups, V, n, dtype, r) for r in range(world)]
        _push_check_apply(groups, inputs, step, V, scale)
    want = torch.bfloat16 if (dtype == torch.bfloat16 and boundary) else torch.float32
    assert groups[0].wire_dtype == want
    for f in fabs:
        f.close()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_push_rings_exact_co_lookup_group(dtype):
    """Two tables (D 48 and D 1) in one push: both rings carry the same entries."""
    V, n, world = 811, 500, 2
    fabs, groups, _ = _groups(world, [48, 1], optim.Adagrad(0.2, 1.0), scale=0.5, V=V)
    _warm(groups, n)
    gen = torch.Generator().manual_seed(13)
    for step in (1, 2):
        inputs = [_step_inputs(gen, groups, V, n, dtype, r) for r in range(world)]
        _push_check_apply(groups, inputs, step, V, 0.5)
    for f in fabs:
        f.close()


def test_push_rings_exact_smem_overflow():
    """One CTA and ~36k distinct ids per rank: the ids its shared-memory table cannot hold
    travel as raw entries after the deduplicated ones."""
    V, n, world = 60013, 40000, 2
    fabs, groups, _ = _groups(world, [8], optim.GradientDescent(0.5), V=V, P=4, cap=50000)
    for grp in groups:
        grp.max_blocks = 1
    _warm(groups, n)
    gen = torch.Generator().manual_seed(9)
    inputs = [_step_inputs(gen, groups, V, n, torch.float32, r) for r in range(world)]
    _push_check_apply(groups, inputs, 1, V, 1.0, overflow=True)
    assert all(grp.overflow_count() > 0 for grp in groups)
    for f in fabs:
        f.close()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("kind", ["adagrad", "ftrl"])
def test_async_push_apply_exact_inputs(dtype, kind):
    """Hogwild push (the optimizer runs in the push kernel), one writer at a time."""
    V, D, n, world = 301, 36, 200, 2
    opt = {"adagrad": optim.Adagrad(0.3, 1.0),
           "ftrl": optim.Ftrl(0.3, l1_regularization_strength=0.01)}[kind]
    fabs, groups, W0 = _groups(world, [D], opt, run_option="PS", sync=False, scale=0.5, V=V,
                               P=4)
    ref_w = W0[0].clone()
    ref_slots = tuple(torch.full_like(ref_w, v) for v in opt.slot_init())
    for grp in groups:
        grp.warm(n)
    gen = torch.Generator().manual_seed(5)
    for step in (1, 2):
        for r, grp in enumerate(groups):
            ids, grads = _step_inputs(gen, groups, V, n, dtype, r)
            _, pend = grp.lookup(ids.cuda())
            grp.add_pending(pend, [grads[0].cuda()])
            grp.begin_step(step)
            grp.finish_step(step)
            torch.cuda.synchronize()
            assert not grp.tables[0].staging.any()
            _check_push_stamps(grp)
            ok = ids < V
            u, inv = torch.unique(ids[ok], return_inverse=True)
            gsum = torch.zeros(u.numel(), D).index_add_(0, inv, grads[0][ok].float() * 0.5)
            optim.apply_sparse_rows_(kind, ref_w, u, gsum, ref_slots, opt.hyper(step))
    L = groups[0].layout
    got = torch.zeros(V, D)
    for o in range(world):
        g, l = L.global_ids_of_owner(o)
        got[g] = groups[o].tables[0].table[:, :D].cpu()[l]
    torch.testing.assert_close(got, ref_w, rtol=5e-4, atol=5e-5)
    for f in fabs:
        f.close()
