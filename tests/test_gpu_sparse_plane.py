"""The sparse owner kernel and the async (Hogwild) push apply against fp64 at every world size
1..8 (`px_sparse_owner_kernel`, `px_sparse_push_kernel<.., ASYNC>` in `ops/csrc/kernels/sparse.cu`),
on a world simulated inside one GPU (`tests/gpu_utils.py`).

Every owner starts from a random per-row state (`dense_plane_ref.random_state`, or a 2^-10 grid
for the exact cases) in its master rows, slots and bf16 shadow, so a kernel that reads another
row's slots, or the slots' initial values, computes different numbers.  Two steps run, and the
second step's ids overlap the first's, so that a stale list head or `slotmap` entry would show.
Every rank's `stage_push` is enqueued before any rank's `stage_apply`; between the two the
receive rings are read back (`sparse_plane_ref.merged`), and each owner's step is checked
against the fp64 step of the same rows from the state it stored before the step
(`tests/sparse_plane_ref.py`):
  * exact -- sgd, momentum and Nesterov momentum on exact operands, bit for bit;
  * random -- every elementwise rule within `STEP_C` (`ASYNC_C` for the async apply); bf16
    master rows within the bf16 bracket of that bound.
After every step: rows no entry touched keep their bits (master, slots, shadow), the shadow is
the master rounded to nearest even, padding columns are zero, `slotmap` is all -1, replicas are
bitwise identical, and lookups (int64 and int32 ids) return the new shadow bit for bit."""
import time

import pytest
import torch

import parallax_b200 as parallax
from parallax_b200 import consts
from parallax_b200.graph import Graph, ScaleGradients
from tests import dense_plane_ref as DR
from tests import sparse_plane_ref as S

pytestmark = pytest.mark.gpu

P = 8
EXACT_WORLDS = [(w, "HYBRID") for w in range(1, 9)] + [(2, "MPI"), (4, "MPI"), (3, "PS")]
RANDOM_WORLDS = [(w, "HYBRID") for w in (1, 2, 3, 5, 7, 8)] + [(4, "MPI"), (8, "MPI")]
GDTS = [torch.float32, torch.bfloat16]
# (ScaleGradients factor, boundary optimisation): scaled on the sender, or on the owner
SCALES = [(1.0, True), (0.5, True), (0.5, False)]


def _bits(t):
    return t.view(torch.int32) if t.element_size() == 4 else t.view(torch.int16)


def _same_bits(a, b):
    return torch.equal(_bits(a.contiguous()), _bits(b.contiguous()))


class Case(object):
    """One group per rank, built on the shared world `fabs`, with its settings."""

    def __init__(self, fabs, tag, kind, opt, Ds, run_option="HYBRID", sync=True, average=False,
                 scale=1.0, boundary=True, local_agg=True, blocks=4, weights="fp32", V=331):
        from parallax_b200.parallel import modes
        from parallax_b200.parallel.nvlink_backend import NVSparseTable, NVSparseGroup
        self.tag, self.kind, self.opt, self.V = tag, kind, opt, V
        self.world = len(fabs)
        self.scale, self.boundary, self.average = scale, boundary, average
        route = modes.route_for(run_option, sync)
        cfg = parallax.Config(run_option=run_option, average_sparse=average)
        cfg.communication_config = parallax.CommunicationConfig(
            parallax.PSConfig(local_aggregation=local_agg,
                              boundary_between_workers_and_servers=boundary))
        graph = Graph(torch.nn.Linear(1, 1), optimizer=opt,
                      grad_rules=[ScaleGradients(scale)] if scale != 1.0 else [])
        o = {"sparse_early_push": False, "sparse_weights": weights}
        if blocks is not None:
            o["sparse_blocks"] = blocks
        W0 = [torch.zeros(V, D) for D in Ds]
        self.groups = [NVSparseGroup([
            NVSparseTable("%s.t%d" % (tag, k), w, P, "mod", opt, f, route, graph, cfg,
                          options=o, out_dtype=torch.bfloat16, auto_group=False)
            for k, w in enumerate(W0)]) for f in fabs]
        self.g_mul = S.gmul(S.owner_avg(self.world, average, scale, boundary))

    def release(self):
        for grp in self.groups:
            for t in grp.tables:
                t.release()

    @property
    def replicated(self):
        return self.groups[0].replicated

    def warm(self, n):
        for grp in self.groups:
            grp._ensure_capacity(n)
        for grp in self.groups:
            grp.warm(n)
        torch.cuda.synchronize()

    def seed_state(self, gen, exact):
        """Random (or 2^-10 grid) master rows and slots on every owner, shadow = RNE(master);
        the replicas of a replicated layout get the same state."""
        for k in range(len(self.groups[0].tables)):
            state = None
            for grp in self.groups:
                t = grp.tables[k]
                if state is None or not t.replicated:
                    n = t.layout.rows_local
                    if exact:
                        state = S.grid_state(gen, self.kind, (n, t.D))
                    else:
                        w, s = DR.random_state(gen, self.kind, n * t.D)
                        state = (w.view(n, t.D), tuple(x.view(n, t.D) for x in s))
                w, s = state
                t.table[:, :t.D] = w.to(t.table.dtype).cuda()
                for dst, src in zip(t.slots, s):
                    dst[:, :t.D] = src.cuda()
                if t.shadow is not None and t.shadow is not t.table:
                    t.shadow.zero_()
                    t.shadow[:, :t.Dp] = t.table
        torch.cuda.synchronize()

    def snapshot(self):
        """[rank][table] -> (master, slots, shadow or None), on the host."""
        out = []
        for grp in self.groups:
            out.append([(t.table.cpu().clone(), [s.cpu().clone() for s in t.slots],
                         t.shadow.cpu().clone() if t.shadow is not None and
                         t.shadow is not t.table else None) for t in grp.tables])
        return out

    def lookup_shadow(self, snap, k, rank):
        """The logical bf16 rows [V, D] lookups of table k on `rank` must return, from `snap`
        (a replicated layout reads the rank's own replica)."""
        t0 = self.groups[0].tables[k]
        L = t0.layout
        full = torch.zeros(self.V, t0.D, dtype=torch.bfloat16)
        for o in ([rank] if t0.replicated else range(self.world)):
            tab, _, sh = snap[o][k]
            src = sh if sh is not None else tab
            g, l = L.global_ids_of_owner(0 if t0.replicated else o)
            full[g] = src[l, :t0.D]
        return full

    def check_lookups(self, ids, snap, outs=None):
        """Lookups of `ids` against the shadow rows in `snap`, bit for bit; ids outside [0, V)
        give zero rows.  `outs`: lookups made with int64 ids while `snap` was current; without
        them, lookups with int64 and with int32 ids are made now."""
        torch.cuda.synchronize()
        for r, grp in enumerate(self.groups):
            if outs is None:
                made = [(grp.lookup(ids[r].to(dt).cuda(), record=False)[0], str(dt))
                        for dt in (torch.int64, torch.int32)]
            else:
                made = [(outs[r], "int64, step start")]
            torch.cuda.synchronize()
            ok = (ids[r] >= 0) & (ids[r] < self.V)
            for k in range(len(grp.tables)):
                want = self.lookup_shadow(snap, k, r)[ids[r].clamp(0, self.V - 1)]
                want[~ok] = 0
                for got, how in made:
                    assert _same_bits(got[k].cpu(), want), "%s: lookup (%s ids) of table %d " \
                        "on rank %d is not the shadow" % (self.tag, how, k, r)

    def step(self, step, ids, grads):
        """One synchronous step: lookups, push, rings read back, apply.  Returns (lookup
        outputs, merged rings) per rank."""
        outs = []
        for grp, i in zip(self.groups, ids):
            o, pend = grp.lookup(i.cuda())
            outs.append((o, pend))
        for grp, (_, pend), g in zip(self.groups, outs, grads):
            grp.begin_step(step)
            grp.add_pending(pend, [x.cuda() for x in g])
        torch.cuda.synchronize()
        for grp in self.groups:
            grp.stage_push(step)
        torch.cuda.synchronize()
        rings = [S.merged(grp) for grp in self.groups]
        for grp in self.groups:
            grp.stage_apply(step)
        torch.cuda.synchronize()
        return [o for o, _ in outs], rings

    def check_step(self, before, after, rings, step, exact):
        """Every owner's touched rows against fp64 (or the exact prediction) and every
        invariant of the module docstring.  Returns the worst err/bound."""
        hp = self.opt.hyper(step)
        worst = 0.0
        for r, grp in enumerate(self.groups):
            assert bool((grp.slotmap == -1).all()), "%s: slotmap not reset on rank %d" % (
                self.tag, r)
            for k, t in enumerate(grp.tables):
                D, ring = t.D, rings[r][k]
                tag = "%s rank %d table %d (D %d) step %d" % (self.tag, r, k, D, step)
                (w_b, s_b, sh_b), (w_a, s_a, sh_a) = before[r][k], after[r][k]
                rows = ring.rows
                w0 = w_b[rows, :D].float()
                s0 = tuple(s[rows, :D] for s in s_b)
                w_k, s_k = w_a[rows, :D], tuple(s[rows, :D] for s in s_a)
                bf16 = t.weight_dtype == torch.bfloat16
                if exact:
                    w_p, s_p = S.predict_owner_exact(self.kind, w0, s0, ring, self.g_mul)
                    assert _same_bits(w_k, w_p), "%s: master, %d of %d differ" % (
                        tag, int((w_k != w_p).sum()), w_p.numel())
                    for x, y in zip(s_k, s_p):
                        assert _same_bits(x, y), "%s: slot differs" % tag
                elif bf16:
                    worst = max(worst, S.check_owner_bf16(tag, self.kind, w_k.float(), s_k, w0,
                                                          s0, ring, self.g_mul, hp))
                else:
                    worst = max(worst, S.check_owner(tag, self.kind, w_k, s_k, w0, s0, ring,
                                                     self.g_mul, hp))
                # untouched rows keep their bits: master, slots, shadow
                idle = torch.ones(w_a.shape[0], dtype=torch.bool)
                idle[rows] = False
                pairs = [(w_a, w_b)] + list(zip(s_a, s_b)) + \
                    ([(sh_a, sh_b)] if sh_a is not None else [])
                for a, b in pairs:
                    assert _same_bits(a[idle], b[idle]), "%s: an untouched row changed" % tag
                # padding columns stay zero; the shadow is the master rounded to nearest even
                assert not bool(w_a[:, D:].float().any()), "%s: master padding" % tag
                if sh_a is not None:
                    assert not bool(sh_a[:, D:].float().any()), "%s: shadow padding" % tag
                    assert _same_bits(sh_a[:, :t.Dp], w_a.bfloat16()), \
                        "%s: shadow != RNE(master)" % tag
        if self.replicated:
            # every replica merges every row, summing its entries in ring-entry order: the
            # replicas stay bitwise identical, random operands included
            for r in range(1, self.world):
                for (a, sa, ha), (b, sb, hb) in zip(after[r], after[0]):
                    assert _same_bits(a, b) and all(_same_bits(x, y) for x, y in zip(sa, sb))
                    assert ha is None or _same_bits(ha, hb), "%s: replicas differ" % self.tag
        return worst

    def run(self, gen, steps, make_ids, make_grads, exact):
        """Seed the state, run `steps` steps, check each; the worst err/bound."""
        self.seed_state(gen, exact)
        worst = 0.0
        before = self.snapshot()
        for step in range(1, steps + 1):
            ids = [make_ids(gen, r) for r in range(self.world)]
            grads = [[make_grads(gen, ids[r].numel(), t.D) for t in grp.tables]
                     for r, grp in enumerate(self.groups)]
            outs, rings = self.step(step, ids, grads)
            self.check_lookups(ids, before, outs)
            after = self.snapshot()
            worst = max(worst, self.check_step(before, after, rings, step, exact))
            # the step's result, through the lookup kernel, at the next step's ids
            self.check_lookups([make_ids(gen, r) for r in range(self.world)], after)
            before = after
        self.release()
        return worst


@pytest.fixture
def make_world():
    """Simulated worlds that are closed when the test ends, whether it passed or not (closing
    a fabric frees every segment of its heap, the tables of a failed case included)."""
    from tests.gpu_utils import make_world as _make
    made = []

    def make(world):
        made.append(_make(world))
        return made[-1]
    yield make
    torch.cuda.synchronize()
    for fabs in made:
        for f in fabs:
            f.close()


def _dup_ids(V, n):
    """Ids with duplicates inside a rank (20 copies of one id), across ranks (id 17) and one
    id past the end."""
    def make(gen, r):
        ids = torch.randint(0, V, (n,), generator=gen)
        ids[:20] = ids[0]
        ids[20:30] = 17
        ids[30] = V + 3
        return ids
    return make


def _unique_ids(V, n):
    """n - 1 distinct ids and one past the end: at most one ring entry per (row, sender)."""
    def make(gen, r):
        ids = torch.randperm(V, generator=gen)[:n]
        ids[-1] = V + 3
        return ids
    return make


def _exact_grads(gdt):
    return lambda gen, n, D: DR.exact_grads(gen, (n, D), 64, 6).to(gdt)


def _random_grads(gdt):
    return lambda gen, n, D: torch.randn(n, D, generator=gen).to(gdt)


def _report(label, worst):
    print("%s: worst err/bound %.3f" % (label, worst))


# ----------------------------------------------------------------------------------- exact
@pytest.mark.parametrize("local_agg", [True, False])
@pytest.mark.parametrize("gdt", GDTS)
@pytest.mark.parametrize("world,layout", EXACT_WORLDS)
def test_owner_exact(world, layout, gdt, local_agg, make_world):
    """sgd, momentum and Nesterov momentum, with and without `average_sparse`, ScaleGradients
    1 and 0.5 on the sender or on the owner: bit for bit.  Tables of D 1, 36 and 64 (odd and
    even D4: the 4- and 8-wide apply paths of a bf16 wire)."""
    V, n = 331, 160
    fabs = make_world(world)
    gen = torch.Generator().manual_seed(world * 100 + local_agg)
    for kind in S.EXACT_KINDS:
        for average in (False, True):
            for scale, boundary in SCALES:
                tag = "%s.%s.%s.%s.%d" % (kind, layout, average, scale, boundary)
                c = Case(fabs, tag, kind, S.make_exact_opt(kind), (1, 36, 64),
                         run_option=layout, average=average, scale=scale, boundary=boundary,
                         local_agg=local_agg, V=V)
                c.warm(n)
                c.run(gen, 2, _dup_ids(V, n), _exact_grads(gdt), exact=True)
                assert c.groups[0].wire_dtype == (
                    torch.bfloat16 if gdt == torch.bfloat16 and boundary else torch.float32)


# ---------------------------------------------------------------------------------- random
@pytest.mark.parametrize("local_agg", [True, False])
@pytest.mark.parametrize("gdt", GDTS)
@pytest.mark.parametrize("world,layout", RANDOM_WORLDS)
def test_owner_random(world, layout, gdt, local_agg, make_world):
    """Every elementwise rule on random operands, averaged: a group of D 1, 36 and 64 and a
    group of D 130 and 512, within `STEP_C`."""
    V, n = 331, 96
    fabs = make_world(world)
    gen = torch.Generator().manual_seed(world * 10 + local_agg + 2 * (gdt == torch.bfloat16))
    t0 = time.time()
    for kind in DR.ELEMENTWISE_VARIANTS:
        worst = 0.0
        for j, Ds in enumerate(((1, 36, 64), (130, 512))):
            c = Case(fabs, "%s.%d" % (kind, j), kind, DR.make_opt(kind), Ds,
                     run_option=layout, average=True, local_agg=local_agg, V=V)
            c.warm(n)
            worst = max(worst, c.run(gen, 2, _unique_ids(V, n), _random_grads(gdt), False))
        _report("owner W=%d %s %s agg=%s %s" % (world, layout, gdt, local_agg, kind), worst)
    print("test time %.1f s" % (time.time() - t0))


@pytest.mark.parametrize("kind", ["adam", "ftrl"])
@pytest.mark.parametrize("blocks", [1, 3, None])
def test_owner_grids(kind, blocks, make_world):
    """`sparse_blocks` 1, 3 and the default, with 6 000 rows per rank: at the default the owner
    asks for more CTAs than its bf16 family-1 kernel keeps resident, so the cooperative launch
    is capped by that kernel's residency."""
    V, n, world = 20011, 6000, 2
    fabs = make_world(world)
    gen = torch.Generator().manual_seed(23)
    c = Case(fabs, "%s.%s" % (kind, blocks), kind, DR.make_opt(kind), (32,), average=True,
             blocks=blocks, V=V)
    c.warm(n)
    worst = c.run(gen, 2, _unique_ids(V, n), _random_grads(torch.bfloat16), False)
    for grp in c.groups:
        assert grp.wire_dtype == torch.bfloat16 and grp._use_merge()
        if blocks is None:
            assert grp._owner_blocks() > 2 * consts.NUM_SMS
    _report("grid %s %s" % (kind, blocks), worst)


@pytest.mark.parametrize("kind", ["adagrad", "ftrl"])
def test_owner_smem_overflow(kind, make_world):
    """One push CTA and ~40k distinct ids per rank: the ids its shared-memory table cannot
    hold travel as raw entries, and the owner merges them with the rest."""
    V, n, world = 60013, 40000, 2
    fabs = make_world(world)
    gen = torch.Generator().manual_seed(29)
    c = Case(fabs, kind, kind, DR.make_opt(kind), (8,), average=True, blocks=1, V=V)
    c.warm(n)
    worst = c.run(gen, 2, _unique_ids(V, n), _random_grads(torch.float32), False)
    assert all(grp.overflow_count() > 0 for grp in c.groups)
    _report("overflow %s" % kind, worst)


@pytest.mark.parametrize("world", [2, 5])
def test_owner_bf16_master(world, make_world):
    """bf16 master rows (`sparse_weights="bf16"`), every elementwise rule: the stored value in
    the bf16 bracket of the fp64 step from the stored state, the slots within their bounds."""
    V, n = 331, 96
    fabs = make_world(world)
    gen = torch.Generator().manual_seed(31 + world)
    for kind in DR.ELEMENTWISE_VARIANTS:
        c = Case(fabs, "bf16.%s" % kind, kind, DR.make_opt(kind), (1, 36, 64, 130),
                 average=True, weights="bf16", V=V)
        c.warm(n)
        worst = c.run(gen, 2, _unique_ids(V, n), _random_grads(torch.bfloat16), False)
        _report("bf16 master W=%d %s (slots)" % (world, kind), worst)


# ----------------------------------------------------------------------------------- async
def _logical(c, k):
    """(master [V, D] fp32, slots, shadow [V, D] bf16) of table k, from its owners."""
    t0 = c.groups[0].tables[k]
    L, D = t0.layout, t0.D
    w = torch.zeros(c.V, D)
    s = [torch.zeros(c.V, D) for _ in t0.slots]
    sh = torch.zeros(c.V, D, dtype=torch.bfloat16)
    for o, grp in enumerate(c.groups):
        t = grp.tables[k]
        g, l = L.global_ids_of_owner(o)
        w[g] = t.table[:, :D].cpu()[l]
        for x, y in zip(s, t.slots):
            x[g] = y[:, :D].cpu()[l]
        sh[g] = t.shadow[:, :D].cpu()[l]
    return w, s, sh


def _async_step(c, step, gen, make_ids, make_grads):
    """Senders one at a time (no races); returns [(ids, grads per table)] in sender order."""
    sent = []
    for r, grp in enumerate(c.groups):
        ids = make_ids(gen, r)
        grads = [make_grads(gen, ids.numel(), t.D) for t in grp.tables]
        _, pend = grp.lookup(ids.cuda())
        grp.add_pending(pend, [g.cuda() for g in grads])
        grp.begin_step(step)
        grp.finish_step(step)
        torch.cuda.synchronize()
        sent.append((ids, grads))
    return sent


def _async_check_invariants(c, k, w0, s0, sh0, w, s, sh, touched):
    idle = torch.ones(c.V, dtype=torch.bool)
    idle[touched] = False
    for a, b in [(w, w0), (sh, sh0)] + list(zip(s, s0)):
        assert _same_bits(a[idle], b[idle]), "%s: an untouched row changed" % c.tag
    assert _same_bits(sh, w.bfloat16()), "%s: shadow != RNE(master)" % c.tag
    for grp in c.groups:
        t = grp.tables[k]
        assert not bool(t.table[:, t.D:].any()) and not bool(t.shadow[:, t.D:].float().any())
        assert not bool(t.staging.any())


@pytest.mark.parametrize("gdt", GDTS)
@pytest.mark.parametrize("world", [2, 5])
def test_async_random(world, gdt, make_world):
    """The Hogwild push applies every elementwise rule on the owners' rows, one sender at a
    time, ids unique within a sender: within `ASYNC_C` of the fp64 chain over the senders."""
    V, n = 331, 96
    fabs = make_world(world)
    gen = torch.Generator().manual_seed(41 + world)
    for kind in DR.ELEMENTWISE_VARIANTS:
        c = Case(fabs, "async.%s" % kind, kind, DR.make_opt(kind), (1, 36, 64), run_option="PS",
                 sync=False, V=V)
        c.warm(n)
        c.seed_state(gen, exact=False)
        worst = 0.0
        for step in (1, 2):
            before = [_logical(c, k) for k in range(3)]
            sent = _async_step(c, step, gen, _unique_ids(V, n), _random_grads(gdt))
            hp = c.opt.hyper(step)
            for k in range(3):
                w0, s0, sh0 = before[k]
                w, s, sh = _logical(c, k)
                senders = []
                for ids, grads in sent:
                    ok = ids < V
                    senders.append((ids[ok], grads[k][ok].float()))
                touched = torch.unique(torch.cat([i for i, _ in senders]))
                worst = max(worst, S.check_async("%s table %d step %d" % (c.tag, k, step), kind,
                                                 w, s, w0, s0, senders, hp, touched))
                _async_check_invariants(c, k, w0, s0, sh0, w, s, sh, touched)
        _report("async W=%d %s %s" % (world, gdt, kind), worst)


def test_async_exact_sgd_with_duplicates(make_world):
    """SGD at lr 2^-3, ScaleGradients 0.5, exact gradients with duplicates inside and across
    senders: each sender's rows, summed and scaled, are applied in turn, bit for bit."""
    V, n, world = 331, 160, 2
    fabs = make_world(world)
    gen = torch.Generator().manual_seed(43)
    c = Case(fabs, "async.sgd.exact", "sgd", S.make_exact_opt("sgd"), (1, 36, 64),
             run_option="PS", sync=False, scale=0.5, V=V)
    c.warm(n)
    c.seed_state(gen, exact=True)
    for step in (1, 2):
        before = [_logical(c, k) for k in range(3)]
        sent = _async_step(c, step, gen, _dup_ids(V, n), _exact_grads(torch.bfloat16))
        for k in range(3):
            w = before[k][0].double()
            for ids, grads in sent:
                ok = ids < V
                u, inv = torch.unique(ids[ok], return_inverse=True)
                g = torch.zeros(u.numel(), w.shape[1], dtype=torch.float64).index_add_(
                    0, inv, grads[k][ok].double())
                w[u] = S.predict_exact("sgd", w[u], (), S.mul32(g, S.f32(0.5)))[0].double()
            got, _, _ = _logical(c, k)
            assert _same_bits(got, w.float()), "table %d step %d: %d elements differ" % (
                k, step, int((got != w.float()).sum()))
