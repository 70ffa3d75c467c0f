"""The LM1B optimizer step against fp64, at the benchmark's shapes and launch grids.

Dense: the clipped LSTM bucket (W [1024, 8192], B [8192], W_P [2048, 512], 9,445,376 bf16
elements) through the kernel sequence `NVDenseGroup` issues for a clipped bucket: `dense_step`
mode 1 with Σg², the one-shot all-reduce of the partials (W > 1), `clip_scale`, mode 2, with
Adagrad(0.2, 1.0) and EMA 0.999.  Sparse: `emb` (V = 793,470, D = 512, ScaleGradients(128))
and the `softmax_w` + `softmax_b` co-lookup group, 32 `mod` partitions, bf16 gradients, bf16
lookups and a bf16 wire, at the default `sparse_blocks`.

Every reference is fp64 (`tests/lm1b_opt_ref.py`); the bounds are derived from the kernels'
fp32 arithmetic and carried step by step.  `pytest -s` prints the worst error / bound ratio of
every check.  A world of W ranks is simulated on one GPU (`tests/gpu_utils.py`); a rank's dense
grid is capped so that every rank's CTAs are resident at once (the kernel's start barrier spins
in each of them)."""
import time

import pytest
import torch

import parallax_b200 as parallax
from parallax_b200 import consts, optim
from tests import lm1b_opt_ref as R

pytestmark = pytest.mark.gpu


def _report(name, ratios):
    print("  %-44s %s" % (name, "  ".join("%s %.3g" % kv for kv in ratios.items())))


def _worst(acc, key, r):
    acc[key] = max(acc.get(key, 0.0), r)


def _bits(t):
    return t.contiguous().view(torch.int16) if t.dtype == torch.bfloat16 else \
        t.contiguous().view(torch.int32)


# ------------------------------------------------------------------------------------- dense
def _dense_params(gen, layout, n):
    """bf16 bucket with the model's initialisation (uniform ±sqrt(3/fan_in), B = 0)."""
    p = torch.zeros(n, device="cuda")
    fan = {"W": 1024, "W_P": 2048}
    for name, off, numel in layout:
        if name in fan:
            a = (3.0 / fan[name]) ** 0.5
            p[off:off + numel] = (torch.rand(numel, device="cuda", generator=gen) * 2 - 1) * a
    return p.bfloat16()


@pytest.mark.parametrize("world,exact,clip", [(1, True, True), (1, False, True),
                                              (2, True, True), (2, False, True),
                                              (8, True, True), (8, False, True),
                                              (1, True, False)])
def test_dense_lstm_bucket(world, exact, clip):
    """Three steps of the LSTM bucket.  W = 1 launches at the benchmark's grid (4·NUM_SMS CTAs
    of the 2-CTA/SM kernel); W > 1 with NUM_SMS / W CTAs per rank.  `exact`: gradients k·2^-6,
    |k| <= 64 (the W-way sum and 1/W are exact); otherwise randn, with the fp32 sum's error in
    the bound.  clip=False: the fused mode 0 at W = 1, the path of an unclipped bucket."""
    from tests.gpu_utils import make_world
    from parallax_b200.parallel import nvops
    from parallax_b200.parallel.symmetric import CH_COMM, CH_SMALL
    t0 = time.time()
    fabs = make_world(world)
    layout, n = R.dense_layout(world)
    pad = R.padding_mask(layout, n, "cuda")
    sl = n // world
    mb = consts.NUM_SMS if world == 1 else consts.NUM_SMS // world
    assert world * mb <= consts.NUM_SMS
    ctas, iters = R.dense_grid(n, world, mb, consts.NUM_SMS)
    opt = optim.Adagrad(R.LR, R.ACC0)
    dt = torch.bfloat16
    gen = torch.Generator(device="cuda").manual_seed(21 + world)
    p0 = _dense_params(gen, layout, n)
    gb = [f.heap.alloc(n * 2, "g") for f in fabs]
    pb = [f.heap.alloc(n * 2, "p") for f in fabs]
    for b in pb:
        b.tensor(dt, n).copy_(p0)
    master = [p0[r * sl:(r + 1) * sl].float() for r in range(world)]
    acc = [torch.full((sl,), R.ACC0, device="cuda") for _ in range(world)]
    ema = [m.clone() for m in master]
    red = [torch.empty(sl, device="cuda") for _ in range(world)]
    loc = [torch.zeros(4, device="cuda") for _ in range(world)]
    tot = [torch.zeros(4, device="cuda") for _ in range(world)]
    scale = [torch.ones(1, device="cuda") for _ in range(world)]
    norm = [torch.zeros(1, device="cuda") for _ in range(world)]
    ref = R.DenseRef(p0.float(), world, exact)
    worst, used = {}, 0.0
    for step in (1, 2, 3):
        grads = R.dense_grads(gen, world, n, exact, device="cuda")
        for r in range(world):
            grads[r][pad] = 0
            gb[r].tensor(dt, n).copy_(grads[r])
        hp = torch.tensor(opt.hyper(step), device="cuda")
        torch.cuda.synchronize()
        if clip:
            # phase-interleaved launches, as in `NVDenseGroup.contributed` / `_finish_clip`: no
            # simulated rank may enqueue a later phase in front of a peer's earlier one
            for r, f in enumerate(fabs):
                nvops.dense_step(f.heap, gb[r].c_ptrs(), pb[r].c_ptrs(), master[r], acc[r],
                                 None, ema[r], red[r], hp, None, loc[r], n, 1.0 / world,
                                 R.EMA_DECAY, "adagrad", 1, dt, CH_COMM, max_blocks=mb,
                                 stream=f.comm_stream)
            if world > 1:
                for r, f in enumerate(fabs):
                    nvops.allreduce_oneshot(f.heap, loc[r], tot[r], f.small_stage, 4,
                                            torch.float32, 1.0, CH_SMALL, stream=f.comm_stream)
            for r, f in enumerate(fabs):
                nvops.clip_scale(tot[r] if world > 1 else loc[r], R.MAX_NORM, scale[r], norm[r],
                                 loc[r], stream=f.comm_stream)
                nvops.dense_step(f.heap, gb[r].c_ptrs(), pb[r].c_ptrs(), master[r], acc[r],
                                 None, ema[r], red[r], hp, scale[r], None, n, 1.0 / world,
                                 R.EMA_DECAY, "adagrad", 2, dt, CH_COMM, max_blocks=mb,
                                 stream=f.comm_stream)
        else:
            for r, f in enumerate(fabs):
                nvops.dense_step(f.heap, gb[r].c_ptrs(), pb[r].c_ptrs(), master[r], acc[r],
                                 None, ema[r], None, hp, None, None, n, 1.0 / world,
                                 R.EMA_DECAY, "adagrad", 0, dt, CH_COMM, max_blocks=mb,
                                 stream=f.comm_stream)
        torch.cuda.synchronize()
        scale_k = None
        if clip:
            for r in range(world):
                assert torch.equal(_bits(scale[r]), _bits(scale[0]))
                assert torch.equal(_bits(norm[r]), _bits(norm[0]))
                assert float(loc[r].abs().sum()) == 0.0          # re-armed for the next step
            scale_k = float(scale[0])
            assert scale_k < 1.0                                # the bucket is clipped
            rn, rs = ref.check_norm(grads, float(norm[0]), scale_k, 8, iters, ctas)
            _worst(worst, "norm", rn)
            _worst(worst, "clip scale", rs)
        ref.step(grads, scale_k)
        w_k, s_k, m_k = torch.cat(master), torch.cat(acc), torch.cat(ema)
        rw, rs_, rm = ref.check(w_k, s_k, m_k, "step %d " % step)
        _worst(worst, "master", rw)
        _worst(worst, "accumulator", rs_)
        _worst(worst, "ema", rm)
        # the pushed parameters: RNE bf16 of the master, identical on every replica
        want = _bits(w_k.bfloat16())
        for r in range(world):
            assert torch.equal(_bits(pb[r].tensor(dt, n)), want), (step, r)
        # padding (none in the LM1B bucket at W <= 8, see test_lm1b_layout) stays untouched
        assert torch.equal(_bits(pb[0].tensor(dt, n)[pad]), _bits(p0[pad]))
        assert not w_k[pad].any() and not m_k[pad].any() and bool((s_k[pad] == R.ACC0).all())
        used = max(used, _device_used_gb())
    torch.cuda.synchronize()
    _report("dense W=%d %s %s (%d CTAs x %d iters, %d pad)"
            % (world, "exact" if exact else "randn", "clip" if clip else "mode 0", ctas, iters,
               int(pad.sum())), worst)
    print("    %.1f s, device memory in use %.2f GB" % (time.time() - t0, used))
    for f in fabs:
        f.close()


# ------------------------------------------------------------------------------------ sparse
EMB_N, N_TARGETS, N_SAMPLED = 2560, 2560, 8192


def _sparse_world(world, blocks, early, weights):
    from tests.gpu_utils import make_world
    from parallax_b200.graph import Graph, ScaleGradients
    from parallax_b200.parallel import modes
    from parallax_b200.parallel.nvlink_backend import NVSparseTable, NVSparseGroup
    fabs = make_world(world)
    route = modes.route_for("HYBRID", True)
    cfg = parallax.Config(run_option="HYBRID", average_sparse=False)
    cfg.communication_config = parallax.CommunicationConfig(
        parallax.PSConfig(local_aggregation=True, boundary_between_workers_and_servers=True))
    opt = optim.Adagrad(R.LR, R.ACC0)
    graph = Graph(torch.nn.Linear(1, 1), optimizer=opt,
                  grad_rules=[ScaleGradients(R.EMB_SCALE, params=["emb.weight"])])
    n_sm = N_TARGETS + N_SAMPLED
    options = {"sparse_capacity": {"emb.weight": EMB_N, "softmax_w.weight": n_sm,
                                   "softmax_b.weight": n_sm},
               "sparse_early_push": early, "sparse_weights": weights}
    if blocks is not None:
        options["sparse_blocks"] = blocks
    V, D, P = R.LM1B_V, R.LM1B_D, R.LM1B_P
    meta = torch.empty(V, D, device="meta")
    emb, smx = [], []
    for f in fabs:
        kw = dict(out_dtype=torch.bfloat16, options=options)
        emb.append(NVSparseTable("emb.weight", meta, P, "mod", opt, f, route, graph, cfg,
                                 init={"seed": 1, "scale": 0.05}, **kw).group)
        tw = NVSparseTable("softmax_w.weight", meta, P, "mod", opt, f, route, graph, cfg,
                           init={"seed": 2, "scale": 0.05}, auto_group=False, **kw)
        tb = NVSparseTable("softmax_b.weight", torch.empty(V, 1, device="meta"), P, "mod", opt,
                           f, route, graph, cfg, init={"seed": 3, "scale": 0.05},
                           auto_group=False, **kw)
        smx.append(NVSparseGroup([tw, tb]))
    for groups, nn in ((emb, EMB_N), (smx, n_sm)):
        for g in groups:
            g._ensure_capacity(nn)
        for g in groups:
            g.warm(nn)
    torch.cuda.synchronize()
    return fabs, emb, smx


def _gather(groups, k, what, gids):
    """Rows `gids` (global ids, all < V) of member table k, read where their owners keep them:
    "table", "slot0" or "shadow", [len, D]."""
    L = groups[0].layout
    t0 = groups[0].tables[k]
    owner = L.owner_of(gids)
    local = L.local_row_of(gids)
    dt = torch.bfloat16 if what == "shadow" else t0.table.dtype if what == "table" \
        else torch.float32
    out = torch.empty(gids.numel(), t0.D, dtype=dt, device="cuda")
    for o, grp in enumerate(groups):
        t = grp.tables[k]
        src = {"table": t.table, "slot0": t.slots[0], "shadow": t.shadow}[what]
        m = owner == o
        out[m] = src[local[m], :t.D]
    return out


def _ids_all_steps(world, steps, gen):
    """Per step, per rank: (emb ids, softmax ids).  The samples come from the benchmark's
    unique log-uniform sampler (seeded through the global CUDA generator)."""
    from parallax_b200.models.lm1b import log_uniform_sample_unique
    V = R.LM1B_V
    out = []
    for _ in range(steps):
        per = []
        for r in range(world):
            e = R.sparse_ids(gen, V, EMB_N, r, device="cuda")
            sampled, _ = log_uniform_sample_unique(N_SAMPLED, V, "cuda")
            per.append((e, R.softmax_ids(gen, V, N_TARGETS, sampled, r, device="cuda")))
        out.append(per)
    return out


def _untouched_sample(touched, gen):
    """A seeded sample of >= 100k untouched rows outside partitions 0 and 31, plus every
    untouched row of those two (0 holds one of the extra rows, 31 does not)."""
    V, P = R.LM1B_V, R.LM1B_P
    s = torch.unique(torch.randint(0, V, (150000,), generator=gen, device="cuda"))
    s = s[(s % P != 0) & (s % P != 31) & ~torch.isin(s, touched)]
    assert s.numel() >= 100000
    parts = torch.cat([torch.arange(p, V, P, device="cuda") for p in (0, 31)])
    assert parts.numel() == 24796 + 24795
    parts = parts[~torch.isin(parts, touched)]
    return torch.cat([s, parts])


def _device_used_gb():
    """Device memory in use, symmetric-heap segments included (they bypass torch's
    allocator): total - free."""
    free, total = torch.cuda.mem_get_info()
    return (total - free) / 2**30


def _sparse_grads(gen, n, D, exact):
    if exact:
        return R.exact_grads(gen, (n, D), 4, 4, device="cuda")
    return torch.randn(n, D, generator=gen, device="cuda").bfloat16()


def _check_lookup(groups, ids_per_rank, outs_per_rank, prev):
    """Each rank's lookup returned the owners' shadow rows of the previous step, bit for bit;
    zeros for the id past the end."""
    V = R.LM1B_V
    for ids, outs in zip(ids_per_rank, outs_per_rank):
        ok = ids < V
        for k, got in enumerate(outs):
            want = torch.zeros_like(got)
            want[ok] = prev[k](ids[ok])
            assert torch.equal(_bits(got), _bits(want)), k


def _run_sparse(world, blocks, early, exact, weights="fp32", steps=3):
    t0 = time.time()
    fabs, emb, smx = _sparse_world(world, blocks, early, weights)
    V = R.LM1B_V
    bf16_master = weights == "bf16"
    gen = torch.Generator(device="cuda").manual_seed(31 + world)
    torch.manual_seed(41 + world)
    ids = _ids_all_steps(world, steps, gen)
    spec = [("emb", emb, 0, R.EMB_SCALE), ("softmax_w", smx, 0, 1.0), ("softmax_b", smx, 1, 1.0)]
    touched, refs, snaps = {}, {}, {}
    for name, groups, k, _ in spec:
        j = 0 if name == "emb" else 1
        rows = torch.unique(torch.cat([ids[s][r][j] for s in range(steps) for r in range(world)]))
        rows = rows[rows < V]
        touched[name] = rows
        w0 = _gather(groups, k, "table", rows)
        refs[name] = R.SparseRef(rows, w0.float())
        un = _untouched_sample(rows, gen)
        snaps[name] = (un, [_gather(groups, k, w, un) for w in ("table", "slot0", "shadow")])
    worst, used = {}, _device_used_gb()
    sr_sum = sr_sq = 0.0
    sr_n = 0
    for step in range(1, steps + 1):
        for j, groups in enumerate((emb, smx)):
            names = ["emb"] if j == 0 else ["softmax_w", "softmax_b"]
            sid = [ids[step - 1][r][j] for r in range(world)]
            n = sid[0].numel()
            # the state this step starts from (lookups must return its shadow)
            prev = [(lambda g, kk=kk, grp=groups: _gather(grp, kk, "shadow", g))
                    for kk in range(len(names))]
            before = {nm: (_gather(groups, kk, "table", touched[nm]).double(),
                           _gather(groups, kk, "slot0", touched[nm]).double())
                      for kk, nm in enumerate(names)} if bf16_master else None
            grads = [[_sparse_grads(gen, n, t.D, exact) for t in groups[0].tables]
                     for _ in range(world)]
            outs, toks = [], []
            for grp, i in zip(groups, sid):
                grp.begin_step(step)
                o, pend = grp.lookup(i)
                outs.append(o)
                toks.append(pend)
            torch.cuda.synchronize()
            _check_lookup(groups, sid, outs, prev)
            for grp, tok, g in zip(groups, toks, grads):
                grp.add_pending(tok, g)      # with the early push: the step runs from here
            if early:
                for grp in groups:
                    grp.finish_step(step)
            else:
                # every rank's push is enqueued before any rank's (spinning) owner kernel
                for grp in groups:
                    grp.stage_push(step)
                for grp in groups:
                    grp.stage_apply(step)
            torch.cuda.synchronize()
            used = max(used, _device_used_gb())
            for grp in groups:
                assert grp.overflow_count() == 0
                assert grp.wire_dtype == torch.bfloat16
            for kk, nm in enumerate(names):
                scale = [s for x, _, _, s in spec if x == nm][0]
                u, g64, gerr = R.sparse_row_grads(sid, [g[kk] for g in grads], V, scale, exact)
                w_k = _gather(groups, kk, "table", touched[nm])
                s_k = _gather(groups, kk, "slot0", touched[nm])
                ref = refs[nm]
                if not bf16_master:
                    ref.step(u, g64, gerr)
                    rw, rs = ref.check(w_k, s_k, "%s step %d " % (nm, step))
                    _worst(worst, nm + " rows", rw)
                    _worst(worst, nm + " acc", rs)
                    for grp in groups:                    # the shadow is RNE of the master
                        t = grp.tables[kk]
                        assert torch.equal(_bits(t.shadow[:, :t.D]),
                                           _bits(t.table[:, :t.D].bfloat16()))
                    continue
                # bf16 master: one step from the kernel's own previous state, then one
                # stochastic rounding to bf16
                w_prev, s_prev = before[nm]
                i = torch.searchsorted(ref.rows, u)
                zero = torch.zeros_like(g64)
                ew, es = R.adagrad_bound(w_prev[i], s_prev[i], g64, ref.lr, zero, zero, gerr)
                w64, s64 = R.adagrad_fp64(w_prev[i], s_prev[i], g64, ref.lr)
                lo, hi = R.bf16_bracket(w64 - R.MARGIN * ew, w64 + R.MARGIN * ew)
                wk = w_k[i].double()
                assert bool(((wk >= lo) & (wk <= hi)).all()), (nm, step)
                _worst(worst, nm + " acc",
                       R.check_bound(nm + " acc", (s_k[i].double() - s64).abs(), es))
                # rows not touched in this step kept their bits
                idle = torch.ones(ref.rows.numel(), dtype=torch.bool, device="cuda")
                idle[i] = False
                assert torch.equal(_bits(w_k[idle]), _bits(w_prev[idle].to(w_k.dtype)))
                d = R.sr_ulps(wk, w64)
                sr_sum += float(d.sum())
                sr_sq += float((d * d).sum())
                sr_n += d.numel()
    # rows no step touched: table, accumulator and shadow keep their bits
    for name, groups, k, _ in spec:
        un, before = snaps[name]
        for what, b in zip(("table", "slot0", "shadow"), before):
            assert torch.equal(_bits(_gather(groups, k, what, un)), _bits(b)), (name, what)
    if bf16_master:
        mean = sr_sum / sr_n
        sd = max(sr_sq / sr_n - mean * mean, 0.0) ** 0.5
        worst.update({"sr draws": sr_n, "sr mean (ulp)": mean, "sr sd (ulp)": sd,
                      "|mean|/(5sd/sqrtN)": abs(mean) / (5 * sd / sr_n ** 0.5)})
        assert abs(mean) <= 5 * sd / sr_n ** 0.5, (mean, sd, sr_n)
    torch.cuda.synchronize()
    _report("sparse W=%d blocks=%s %s %s%s" % (world, blocks, "exact" if exact else "randn",
                                               weights, " early" if early else ""), worst)
    print("    %.1f s, device memory in use %.2f GB, %d emb / %d softmax rows touched"
          % (time.time() - t0, used, touched["emb"].numel(), touched["softmax_w"].numel()))
    for f in fabs:
        f.close()


@pytest.mark.parametrize("world,blocks,early", [(1, None, True), (2, None, False),
                                                (8, 2 * consts.NUM_SMS // 8, False)])
def test_sparse_tables_exact(world, blocks, early):
    """Exact gradients (k·2^-4, |k| <= 4, at most 60 per row and sender): the wire carries the
    exact sums, so only the rule's arithmetic is left.  The early push (the benchmark's
    default) only at W = 1: at W > 1 it would enqueue one simulated rank's owner kernel ahead
    of a peer's push."""
    _run_sparse(world, blocks, early, True)


def test_sparse_tables_randn():
    """randn bf16 gradients: a row duplicated within one sender may be off by its fp32 sum's
    error and one bf16 rounding on the wire, carried into the bound."""
    _run_sparse(2, None, False, False)


def test_sparse_tables_bf16_masters():
    """sparse_weights="bf16": every stored element lies in the bf16 bracket of the fp64 step
    from the previous stored state, and the stochastic rounding is unbiased."""
    _run_sparse(2, None, False, True, weights="bf16")
