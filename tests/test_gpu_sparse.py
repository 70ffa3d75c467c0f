"""Sparse-path kernels (lookup / dedup / push / claim / apply / async) vs a
plain PyTorch fp32 reference, on a world simulated inside one GPU."""
import pytest
import torch

import parallax_b200 as parallax
from parallax_b200 import optim

pytestmark = pytest.mark.gpu


def _tables(world, V, D, P, opt, run_option="HYBRID", sync=True, average=False,
            local_agg=True, out_dtype=torch.float32, strategy="mod", cap=None, owners=None,
            boundary=True, blocks=4):
    from tests.gpu_utils import make_world
    from parallax_b200.parallel import modes
    from parallax_b200.parallel.nvlink_backend import NVSparseTable
    from parallax_b200.graph import Graph
    fabs = make_world(world)
    route = modes.route_for(run_option, sync)
    cfg = parallax.Config(run_option=run_option, average_sparse=average)
    cfg.communication_config = parallax.CommunicationConfig(
        parallax.PSConfig(local_aggregation=local_agg,
                          boundary_between_workers_and_servers=boundary))
    g = torch.Generator().manual_seed(7)
    W0 = torch.randn(V, D, generator=g)
    graph = Graph(torch.nn.Linear(1, 1), optimizer=opt)
    options = {"sparse_capacity": {"emb.weight": cap or 4096}, "sparse_early_push": False}
    if blocks is not None:                  # None: the default, sized from the row count
        options["sparse_blocks"] = blocks
    tabs = [NVSparseTable("emb.weight", W0, P, strategy, opt, f, route, graph, cfg,
                          out_dtype=out_dtype, owners=owners, options=options)
            for f in fabs]
    return fabs, tabs, W0


def _finish_all(tabs, step):
    """Every simulated rank's sender stage is enqueued before any rank's owner
    stage: the ranks' streams live in one process and may share a hardware
    queue, so a spinning owner kernel must never sit in front of a peer's push."""
    for t in tabs:
        t.stage_push(step)
    for t in tabs:
        t.stage_apply(step)
    torch.cuda.synchronize()


def _full(tabs, V, D):
    out = torch.zeros(V, D)
    L = tabs[0].layout
    owners = [0] if L.replicated else range(len(tabs))
    for o in owners:
        g, l = L.global_ids_of_owner(o)
        out[g] = tabs[o].table[:, :D].cpu()[l]
    return out


@pytest.mark.parametrize("world,P,strategy", [(1, 1, "mod"), (2, 5, "mod"), (3, 8, "mod"),
                                              (4, 8, "div"), (5, 8, "div"), (8, 32, "mod")])
@pytest.mark.parametrize("D", [1, 4, 64, 130])
@pytest.mark.parametrize("out_dtype", [torch.float32, torch.bfloat16])
def test_lookup_matches_index_select(world, P, strategy, D, out_dtype):
    V = 1000
    from parallax_b200.parallel.layout import assign_owners
    owners = assign_owners([("a", P, 7), ("b", P, 3)], world)["b"]      # not round-robin
    fabs, tabs, W0 = _tables(world, V, D, P, optim.GradientDescent(0.1),
                             strategy=strategy, out_dtype=out_dtype, owners=owners)
    torch.cuda.synchronize()
    for r, t in enumerate(tabs):
        assert t.use_shadow == (out_dtype == torch.bfloat16)
        ids = torch.randint(0, V, (257,), device="cuda")
        ids[3] = V + 5                               # out of range -> zeros, pend -1
        rows, pend = t.lookup(ids)
        torch.cuda.synchronize()
        ref = W0[ids.cpu().clamp(max=V - 1)].to(out_dtype)
        ref[3] = 0
        assert rows.dtype == out_dtype and rows.shape == (257, D)
        torch.testing.assert_close(rows.cpu(), ref)
        exp = ids.cpu().long()
        exp[3] = -1
        assert torch.equal(pend.cpu().long(), exp)
    for f in fabs:
        f.close()


@pytest.mark.parametrize("world,run_option", [(1, "HYBRID"), (2, "HYBRID"), (3, "HYBRID"),
                                              (4, "PS"), (4, "MPI"), (6, "HYBRID"),
                                              (8, "HYBRID")])
@pytest.mark.parametrize("kind", ["sgd", "adagrad", "adam"])
@pytest.mark.parametrize("local_agg", [True, False])
def test_push_claim_apply(world, run_option, kind, local_agg):
    V, D, P = 503, 36, 8
    opt = {"sgd": optim.GradientDescent(0.5), "adagrad": optim.Adagrad(0.2, 1.0),
           "adam": optim.Adam(0.05)}[kind]
    fabs, tabs, W0 = _tables(world, V, D, P, opt, run_option=run_option,
                             average=(kind == "adam"), local_agg=local_agg)
    ref_w = W0.clone()
    ref_slots = tuple(torch.full_like(W0, v) for v in opt.slot_init())
    gen = torch.Generator().manual_seed(11)
    n = 300
    for t in tabs:
        t._ensure_capacity(n)
    for t in tabs:
        t.warm(n)
    torch.cuda.synchronize()
    for step in (1, 2, 3):
        all_ids, all_g = [], []
        toks = []
        for r, t in enumerate(tabs):
            ids = torch.randint(0, V, (n,), generator=gen)
            ids[:40] = ids[0]                     # duplicates inside a rank
            ids[40:60] = 17                       # and across ranks
            gr = torch.randn(n, D, generator=gen)
            rows, pend = t.lookup(ids.cuda())
            toks.append(pend)
            all_ids.append(ids)
            all_g.append(gr)
        torch.cuda.synchronize()
        # lookups observe the previous step's update
        for r, t in enumerate(tabs):
            rows, _ = t.lookup(all_ids[r].cuda(), record=False)
            torch.cuda.synchronize()
            torch.testing.assert_close(rows.cpu(), ref_w[all_ids[r]], rtol=1e-4, atol=1e-5)
        for r, t in enumerate(tabs):
            t.add_pending(toks[r], all_g[r].cuda())
            t.begin_step(step)
        torch.cuda.synchronize()
        _finish_all(tabs, step)
        ids_c, g_c = torch.cat(all_ids), torch.cat(all_g)
        u, inv = torch.unique(ids_c, return_inverse=True)
        gsum = torch.zeros(u.numel(), D).index_add_(0, inv, g_c)
        if kind == "adam":
            gsum /= world
        optim.apply_sparse_rows_(kind, ref_w, u, gsum, ref_slots, opt.hyper(step))
        if run_option == "MPI":
            for t in tabs:        # every replica applied the same update
                torch.testing.assert_close(t.table[:, :D].cpu(), ref_w, rtol=2e-4, atol=2e-5)
        else:
            torch.testing.assert_close(_full(tabs, V, D), ref_w, rtol=2e-4, atol=2e-5)
    for f in fabs:
        f.close()


@pytest.mark.parametrize("kind", ["ftrl", "centered_rmsprop"])
def test_bf16_wire_family1_merge_at_default_grid(kind):
    """bf16 wire, a family-1 rule and the merge path, with `sparse_blocks` at its default:
    6 000 rows per rank make the owner ask for more CTAs than its bf16 family-1 kernel keeps
    resident (2 per SM), so the cooperative launch must be capped by that kernel's residency."""
    from parallax_b200 import consts
    V, D, P, world, n = 20011, 32, 4, 2, 6000
    # epsilon keeps the centered RMSProp step a smooth function of g: near eps = 0 it is
    # lr·sign(g), which a bf16 rounding of a merged row that nearly cancels could flip
    opt = {"ftrl": optim.Ftrl(0.3, l1_regularization_strength=0.01),
           "centered_rmsprop": optim.CenteredRMSProp(0.05, momentum=0.5, epsilon=1e-2)}[kind]
    fabs, tabs, W0 = _tables(world, V, D, P, opt, out_dtype=torch.bfloat16, cap=2 * n,
                             blocks=None)
    for t in tabs:
        t._ensure_capacity(n)
    for t in tabs:
        t.warm(n)
    gen = torch.Generator().manual_seed(13)
    all_ids, all_g, toks = [], [], []
    for r, t in enumerate(tabs):
        ids = torch.randint(0, V, (n,), generator=gen)
        gr = torch.randn(n, D, generator=gen).bfloat16()
        rows, pend = t.lookup(ids.cuda())
        toks.append(pend)
        all_ids.append(ids)
        all_g.append(gr)
    torch.cuda.synchronize()
    for r, t in enumerate(tabs):
        t.add_pending(toks[r], all_g[r].cuda())
        t.begin_step(1)
    torch.cuda.synchronize()
    _finish_all(tabs, 1)
    for t in tabs:
        assert t.group.wire_dtype == torch.bfloat16 and t.group._use_merge()
        assert t.group._owner_blocks() > 2 * consts.NUM_SMS
    ids_c, g_c = torch.cat(all_ids), torch.cat(all_g).float()
    u, inv = torch.unique(ids_c, return_inverse=True)
    gsum = torch.zeros(u.numel(), D).index_add_(0, inv, g_c)
    ref_w = W0.clone()
    ref_slots = tuple(torch.full_like(W0, v) for v in opt.slot_init())
    optim.apply_sparse_rows_(kind, ref_w, u, gsum, ref_slots, opt.hyper(1))
    # duplicated ids are summed in fp32 and rounded to bf16 once when they cross the wire
    torch.testing.assert_close(_full(tabs, V, D), ref_w, rtol=2e-2, atol=2e-2)
    for t in tabs:
        torch.testing.assert_close(t.shadow[:, :D].float(), t.table[:, :D].bfloat16().float())
    for f in fabs:
        f.close()


@pytest.mark.parametrize("boundary", [True, False])
def test_large_n_bf16_grads_and_wire(boundary):
    """20 000 rows per rank through 4 CTAs (5 000 ids per CTA's SMEM table), bf16
    gradients: bf16 on the wire with the boundary optimisation, fp32 without; the
    lookups read the bf16 shadow rows, which the owner kernel keeps in sync."""
    V, D, P, world = 20011, 32, 4, 2
    opt = optim.Adagrad(0.1, 1.0)
    fabs, tabs, W0 = _tables(world, V, D, P, opt, out_dtype=torch.bfloat16,
                             cap=40000, boundary=boundary)
    n = 20000
    for t in tabs:
        t._ensure_capacity(n)
    for t in tabs:
        t.warm(n)
    gen = torch.Generator().manual_seed(3)
    all_ids, all_g, toks = [], [], []
    for r, t in enumerate(tabs):
        ids = torch.randint(0, V, (n,), generator=gen)
        gr = torch.randn(n, D, generator=gen).bfloat16()
        rows, pend = t.lookup(ids.cuda())
        assert rows.dtype == torch.bfloat16
        toks.append(pend)
        all_ids.append(ids)
        all_g.append(gr)
    torch.cuda.synchronize()
    for r, t in enumerate(tabs):
        t.add_pending(toks[r], all_g[r].cuda())
        t.begin_step(1)
    torch.cuda.synchronize()
    _finish_all(tabs, 1)
    ids_c, g_c = torch.cat(all_ids), torch.cat(all_g).float()
    u, inv = torch.unique(ids_c, return_inverse=True)
    gsum = torch.zeros(u.numel(), D).index_add_(0, inv, g_c)
    ref_w = W0.clone()
    optim.apply_sparse_rows_("adagrad", ref_w, u, gsum,
                             (torch.full_like(W0, 1.0),), opt.hyper(1))
    # duplicated ids are summed in fp32 and rounded to bf16 once when they cross the wire
    tol = dict(rtol=2e-2, atol=2e-2) if boundary else dict(rtol=1e-3, atol=1e-4)
    torch.testing.assert_close(_full(tabs, V, D), ref_w, **tol)
    for t in tabs:
        assert t.group.wire_dtype == (torch.bfloat16 if boundary else torch.float32)
        assert t.group.overflow_count() == 0
        torch.testing.assert_close(t.shadow[:, :D].float(), t.table[:, :D].bfloat16().float())
    for f in fabs:
        f.close()


def test_smem_overflow_falls_back_to_raw_entries():
    """More distinct ids in one CTA than its shared-memory table holds: the surplus
    positions travel un-aggregated and the owner merges them — still exact."""
    V, D, P, world = 60013, 8, 4, 2
    opt = optim.GradientDescent(0.5)
    fabs, tabs, W0 = _tables(world, V, D, P, opt, cap=50000)
    for t in tabs:
        t.group.max_blocks = 1                     # one CTA: 8192 slots for ~36k distinct ids
    n = 40000
    for t in tabs:
        t._ensure_capacity(n)
    for t in tabs:
        t.warm(n)
    gen = torch.Generator().manual_seed(9)
    all_ids, all_g, toks = [], [], []
    for r, t in enumerate(tabs):
        ids = torch.randint(0, V, (n,), generator=gen)
        gr = torch.randn(n, D, generator=gen)
        rows, pend = t.lookup(ids.cuda())
        toks.append(pend)
        all_ids.append(ids)
        all_g.append(gr)
    for r, t in enumerate(tabs):
        t.add_pending(toks[r], all_g[r].cuda())
        t.begin_step(1)
    torch.cuda.synchronize()
    _finish_all(tabs, 1)
    assert all(t.group.overflow_count() > 0 for t in tabs)
    ids_c, g_c = torch.cat(all_ids), torch.cat(all_g)
    u, inv = torch.unique(ids_c, return_inverse=True)
    gsum = torch.zeros(u.numel(), D).index_add_(0, inv, g_c)
    ref_w = W0.clone()
    optim.apply_sparse_rows_("sgd", ref_w, u, gsum, (), opt.hyper(1))
    torch.testing.assert_close(_full(tabs, V, D), ref_w, rtol=2e-4, atol=2e-4)
    for f in fabs:
        f.close()


@pytest.mark.parametrize("world", [1, 4])
def test_co_lookup_group_shares_one_push_and_owner_kernel(world):
    """Two tables (D=48 and D=1) looked up with the same ids: one lookup, one push and
    one owner launch serve both; every extended optimizer rule runs on the owner."""
    from tests.gpu_utils import make_world
    from parallax_b200.parallel import modes, nvops
    from parallax_b200.parallel.nvlink_backend import NVSparseTable, NVSparseGroup
    from parallax_b200.graph import Graph
    V, P, n = 811, 8, 500
    for opt in (optim.Adagrad(0.2, 1.0), optim.Ftrl(0.3, l1_regularization_strength=0.01),
                optim.CenteredRMSProp(0.05, momentum=0.5), optim.Adadelta(0.5),
                optim.ProximalAdagrad(0.2, l1_regularization_strength=0.01),
                optim.AdagradDA(0.2, l1_regularization_strength=0.001)):
        fabs = make_world(world)
        route = modes.route_for("HYBRID", True)
        cfg = parallax.Config(run_option="HYBRID")
        g = torch.Generator().manual_seed(7)
        Wa, Wb = torch.randn(V, 48, generator=g), torch.randn(V, 1, generator=g)
        graph = Graph(torch.nn.Linear(1, 1), optimizer=opt)
        o = {"sparse_blocks": 4, "sparse_early_push": False}
        groups = []
        for f in fabs:
            ta = NVSparseTable("a", Wa, P, "mod", opt, f, route, graph, cfg, options=o,
                               auto_group=False)
            tb = NVSparseTable("b", Wb, P, "mod", opt, f, route, graph, cfg, options=o,
                               auto_group=False)
            groups.append(NVSparseGroup([ta, tb]))
        for grp in groups:
            grp._ensure_capacity(n)
        for grp in groups:
            grp.warm(n)
        torch.cuda.synchronize()
        ref = [Wa.clone(), Wb.clone()]
        ref_slots = [tuple(torch.full_like(w, v) for v in opt.slot_init()) for w in ref]
        gen = torch.Generator().manual_seed(11)
        for step in (1, 2):
            ids_l, ga_l, gb_l, toks = [], [], [], []
            l0 = nvops.launches["n"]
            for grp in groups:
                ids = torch.randint(0, V, (n,), generator=gen)
                ids[:50] = ids[0]
                (ra, rb), pend = grp.lookup(ids.cuda())
                torch.cuda.synchronize()
                torch.testing.assert_close(ra.cpu(), ref[0][ids], rtol=1e-4, atol=1e-5)
                torch.testing.assert_close(rb.cpu(), ref[1][ids], rtol=1e-4, atol=1e-5)
                toks.append(pend)
                ids_l.append(ids)
                ga_l.append(torch.randn(n, 48, generator=gen))
                gb_l.append(torch.randn(n, 1, generator=gen))
            for grp, tok, ga, gb in zip(groups, toks, ga_l, gb_l):
                grp.begin_step(step)
                grp.add_pending(tok, [ga.cuda(), gb.cuda()])
            torch.cuda.synchronize()
            for grp in groups:
                grp.stage_push(step)
            for grp in groups:
                grp.stage_apply(step)
            torch.cuda.synchronize()
            assert nvops.launches["n"] - l0 == 3 * world       # lookup + push + owner
            ids_c = torch.cat(ids_l)
            u, inv = torch.unique(ids_c, return_inverse=True)
            for k, (gl, D) in enumerate(((ga_l, 48), (gb_l, 1))):
                gsum = torch.zeros(u.numel(), D).index_add_(0, inv, torch.cat(gl))
                optim.apply_sparse_rows_(opt.kind, ref[k], u, gsum, ref_slots[k], opt.hyper(step))
        for k, D in ((0, 48), (1, 1)):
            got = torch.zeros(V, D)
            L = groups[0].layout
            for o_ in range(world):
                gi, li = L.global_ids_of_owner(o_)
                got[gi] = groups[o_].tables[k].table[:, :D].cpu()[li]
            torch.testing.assert_close(got, ref[k], rtol=5e-4, atol=5e-5)
        for f in fabs:
            f.close()


def test_async_apply_single_writer_matches_reference():
    """Hogwild path, exercised without races (one rank pushes at a time)."""
    V, D, P, world = 301, 16, 4, 2
    opt = optim.Adagrad(0.3, 1.0)
    fabs, tabs, W0 = _tables(world, V, D, P, opt, run_option="PS", sync=False)
    ref_w, ref_acc = W0.clone(), torch.full_like(W0, 1.0)
    gen = torch.Generator().manual_seed(5)
    for t in tabs:
        t.warm(64)
    for step in (1, 2):
        for r, t in enumerate(tabs):
            ids = torch.randint(0, V, (64,), generator=gen)
            gr = torch.randn(64, D, generator=gen)
            rows, pend = t.lookup(ids.cuda())
            t.add_pending(pend, gr.cuda())
            t.begin_step(step)
            t.finish_step(step)
            torch.cuda.synchronize()
            u, inv = torch.unique(ids, return_inverse=True)
            gsum = torch.zeros(u.numel(), D).index_add_(0, inv, gr)
            optim.apply_sparse_rows_("adagrad", ref_w, u, gsum, (ref_acc,),
                                     opt.hyper(step))
    torch.testing.assert_close(_full(tabs, V, D), ref_w, rtol=2e-4, atol=2e-5)
    for f in fabs:
        f.close()
