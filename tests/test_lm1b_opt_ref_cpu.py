"""The fp64 references and bounds of `tests/lm1b_opt_ref.py`, without a GPU: an emulation of
the kernels' fp32 arithmetic, in kernel order and with rsqrtf off by up to 2 ulp either way,
stays inside them over the inputs `test_gpu_lm1b_optimizer.py` draws (at a shorter bucket and
one table), and each of the slips a kernel could make does not."""
import math

import pytest
import torch

from tests import lm1b_opt_ref as R

N_CPU = 2048 * 24          # bucket length of the emulated dense step (a multiple of W·vn·32)


def fma32(a, b, c):
    """fmaf on fp32 tensors: the fp64 product of two floats is exact, one rounding to fp32."""
    return (a.double() * b.double() + c.double()).float()


def rsqrt32(s, direction):
    """rsqrtf off by 1..2 ulp of the true value, upwards (direction > 0) or downwards."""
    r64 = 1.0 / s.double().sqrt()
    r = r64.float()
    if direction > 0:
        r = torch.where(r.double() > r64, torch.nextafter(r, torch.full_like(r, -math.inf)), r)
        up = torch.full_like(r, math.inf)
        return torch.nextafter(torch.nextafter(r, up), up)
    r = torch.where(r.double() < r64, torch.nextafter(r, torch.full_like(r, math.inf)), r)
    dn = torch.full_like(r, -math.inf)
    return torch.nextafter(torch.nextafter(r, dn), dn)


def _tree32(x):
    """fp32 pairwise sum over the last dimension (a power of two)."""
    while x.shape[-1] > 1:
        h = x.shape[-1] // 2
        x = x[..., :h] + x[..., h:]
    return x[..., 0]


def sumsq32(g, world, ctas, iters, vn=8, threads=512):
    """Σg² as `px_dense_step` mode 1 adds it: per thread over its grid-stride vectors, a warp
    tree, a tree over the block's warps, one atomic per CTA, then the ranks' partials."""
    sl = g.numel() // world
    stride = ctas * threads
    total = torch.zeros((), dtype=torch.float32)
    for r in range(world):
        x = torch.zeros(iters * stride * vn, dtype=torch.float32)
        x[:sl] = g[r * sl:(r + 1) * sl]
        x = x.view(iters, stride, vn)
        acc = torch.zeros(stride, dtype=torch.float32)
        for it in range(iters):
            for i in range(vn):
                acc = fma32(x[it, :, i], x[it, :, i], acc)
        warps = _tree32(acc.view(ctas, threads // 32, 32))
        blocks = _tree32(torch.nn.functional.pad(warps, (0, 32 - threads // 32)))
        part = torch.zeros((), dtype=torch.float32)
        for b in blocks:
            part = part + b
        total = total + part
    return total


def _run(fails, name, fn):
    try:
        return fn()
    except AssertionError:
        fails.add(name)
        return None


DENSE_MUTANTS = ("old_acc", "avg_twice", "clip_twice", "clip_none", "bf16_master", "ema_decay")


def dense_emulation(world, exact, direction, mutant=None, steps=3):
    """Three clipped steps of the bucket; returns the names of the checks that failed."""
    gen = torch.Generator().manual_seed(100 + world)
    n = N_CPU
    w = ((torch.rand(n, generator=gen) - 0.5) * 0.1).bfloat16().float()
    ref = R.DenseRef(w, world, exact)
    s = torch.full_like(w, R.ACC0)
    m = w.clone()
    lr = torch.tensor(R.f32(R.LR))
    avg = torch.tensor(1.0 / world, dtype=torch.float32)
    c = torch.tensor(R.ema_coef(R.EMA_DECAY) if mutant != "ema_decay" else R.f32(R.EMA_DECAY))
    mb = 132 if world == 1 else 132 // world
    ctas, iters = R.dense_grid(n, world, mb)
    fails = set()
    for _ in range(steps):
        grads = R.dense_grads(gen, world, n, exact)
        g = torch.zeros(n, dtype=torch.float32)
        for x in grads:
            g = g + x.float()
        g = g * avg
        if mutant == "avg_twice":
            g = g * avg
        norm = sumsq32(g, world, ctas, iters).sqrt()
        scale = torch.tensor(R.MAX_NORM, dtype=torch.float32) / \
            torch.clamp_min(norm, R.MAX_NORM)
        _run(fails, "norm", lambda: ref.check_norm(grads, float(norm), float(scale), 8, iters,
                                                   ctas))
        g2 = g if mutant == "clip_none" else g * scale
        if mutant == "clip_twice":
            g2 = g2 * scale
        s_old, s = s, fma32(g2, g2, s)
        r = rsqrt32(s_old if mutant == "old_acc" else s, direction)
        w = fma32(-lr * g2, r, w)
        if mutant == "bf16_master":
            w = w.bfloat16().float()
        m = fma32(-c, m - w, m)
        ref.step(grads, float(scale))
        _run(fails, "master", lambda: R.check_bound("master", (w.double() - ref.w).abs(),
                                                     ref.ew))
        _run(fails, "accumulator", lambda: R.check_bound("acc", (s.double() - ref.s).abs(),
                                                          ref.es))
        _run(fails, "ema", lambda: R.check_bound("ema", (m.double() - ref.m).abs(), ref.em))
    return fails


SPARSE_MUTANTS = ("old_acc", "drop_dup")


def sparse_emulation(world, exact, direction, mutant=None, steps=3, n=2560, D=512):
    """Three steps of the `emb` table (ScaleGradients(128), bf16 wire) over the touched rows;
    returns the names of the checks that failed."""
    V = R.LM1B_V
    gen = torch.Generator().manual_seed(200 + world)
    ids = [[R.sparse_ids(gen, V, n, r) for r in range(world)] for _ in range(steps)]
    rows = torch.unique(torch.cat([i for st in ids for i in st]))
    rows = rows[rows < V]
    w = torch.randn(rows.numel(), D, generator=gen) * 0.05
    ref = R.SparseRef(rows, w)
    s = torch.full_like(w, R.ACC0)
    lr = torch.tensor(R.f32(R.LR))
    fails = set()
    for st in range(steps):
        if exact:
            grads = [R.exact_grads(gen, (n, D), 4, 4) for _ in range(world)]
        else:
            grads = [torch.randn(n, D, generator=gen).bfloat16() for _ in range(world)]
        merged = torch.zeros(rows.numel(), D, dtype=torch.float32)
        for r, (i, g) in enumerate(zip(ids[st], grads)):
            ok = i < V
            i, g = i[ok], g[ok].float()
            if mutant == "drop_dup" and r == 0:
                drop = int((i == 1000).nonzero()[-1])        # one copy of a duplicated row
                keep = torch.arange(i.numel()) != drop
                i, g = i[keep], g[keep]
            us, inv = torch.unique(i, return_inverse=True)
            wire = torch.zeros(us.numel(), D).index_add_(0, inv, g) * R.EMB_SCALE
            wire = wire.bfloat16().float()
            merged.index_add_(0, torch.searchsorted(rows, us), wire)
        u, g64, gerr = R.sparse_row_grads(ids[st], grads, V, R.EMB_SCALE, exact)
        t = torch.searchsorted(rows, u)
        g = merged[t]
        s_old = s[t]
        s_new = fma32(g, g, s_old)
        r_ = rsqrt32(s_old if mutant == "old_acc" else s_new, direction)
        w[t] = fma32(-lr * g, r_, w[t])
        s[t] = s_new
        ref.step(u, g64, gerr)
        _run(fails, "rows", lambda: ref.check(w, s))
    return fails


# ------------------------------------------------------------------------------------- tests
@pytest.mark.parametrize("world", [1, 2, 8])
@pytest.mark.parametrize("exact", [True, False])
@pytest.mark.parametrize("direction", [1, -1])
def test_dense_emulation_inside_bounds(world, exact, direction):
    assert dense_emulation(world, exact, direction) == set()


@pytest.mark.parametrize("world", [2, 8])
@pytest.mark.parametrize("mutant", DENSE_MUTANTS)
def test_dense_mutant_exceeds_bounds(world, mutant):
    """Every slip fails at least one check.  1/W applied twice only shows in the norm: the clip
    scale absorbs it as long as the bucket is clipped."""
    fails = dense_emulation(world, True, 1, mutant)
    assert fails, mutant
    if mutant == "avg_twice":
        assert "norm" in fails
    if mutant == "ema_decay":
        assert fails == {"ema"}


@pytest.mark.parametrize("world", [1, 2])
@pytest.mark.parametrize("exact", [True, False])
@pytest.mark.parametrize("direction", [1, -1])
def test_sparse_emulation_inside_bounds(world, exact, direction):
    assert sparse_emulation(world, exact, direction) == set()


@pytest.mark.parametrize("mutant", SPARSE_MUTANTS)
def test_sparse_mutant_exceeds_bounds(mutant):
    assert sparse_emulation(2, True, 1, mutant) == {"rows"}


def test_lm1b_layout():
    """The bucket the tests lay out is the one the backend builds for LM1B's LSTM variables:
    W_P, B, W at offsets 0, 2048·512 and 2048·512 + 8192, no padding at W = 1, 2, 8."""
    from parallax_b200.models.lm1b import LM1B
    m = LM1B(vocab_size=64, num_shards=2, lazy=True)
    dense = [(k, tuple(p.shape)) for k, p in m.named_parameters() if k in ("W", "B", "W_P")]
    assert tuple(dense) == R.LSTM_ITEMS
    for world in (1, 2, 8):
        layout, n = R.dense_layout(world)
        assert [(k, o) for k, o, _ in layout] == [("W_P", 0), ("B", 1048576), ("W", 1056768)]
        assert n == 9445376 and not R.padding_mask(layout, n).any()
    assert R.dense_layout(8, items=(("a", (3,)), ("b", (10,))))[1] == 2048
    layout, n = R.dense_layout(1, items=(("a", (3,)), ("b", (10,))))
    assert layout == [("b", 0, 10), ("a", 16, 3)] and int(R.padding_mask(layout, n).sum()) == 243


def test_lm1b_row_geometry():
    """793,470 = 32·24,795 + 30: the ids V-30 .. V-1 are the extra rows of partitions 0..29."""
    from parallax_b200.parallel.layout import TableLayout
    L = TableLayout(R.LM1B_V, R.LM1B_P, 8, "mod")
    last = torch.arange(R.LM1B_V - 30, R.LM1B_V)
    assert torch.equal(L.partition_of(last), torch.arange(30))
    assert bool((L.index_in_partition(last) == 24795).all())
    assert [L.partition_rows(p) for p in (0, 29, 30, 31)] == [24796, 24796, 24795, 24795]


def test_bf16_helpers():
    x = torch.tensor([1.0, 1.5, -3.0, 2.0 ** -130, 0.0, 255.0], dtype=torch.float64)
    assert R.ulp_bf16(x).tolist() == [2.0 ** -7, 2.0 ** -7, 2.0 ** -6, 2.0 ** -133,
                                      2.0 ** -133, 1.0]
    lo, hi = R.bf16_bracket(torch.tensor([1.0 + 2.0 ** -10, -1.0 - 2.0 ** -10, 1.0]),
                            torch.tensor([1.0 + 2.0 ** -9, -1.0 + 2.0 ** -12, 1.0]))
    assert lo.tolist() == [1.0, -1.0 - 2.0 ** -7, 1.0]
    assert hi.tolist() == [1.0 + 2.0 ** -7, -1.0 + 2.0 ** -8, 1.0]
    # every bf16 value of a random sample lies in its own bracket, and nothing else does
    v = (torch.randn(10000, generator=torch.Generator().manual_seed(1)) * 10).bfloat16().double()
    lo, hi = R.bf16_bracket(v, v)
    assert torch.equal(lo, v) and torch.equal(hi, v)
    lo, hi = R.bf16_bracket(v + R.ulp_bf16(v) / 4, v + R.ulp_bf16(v) / 4)
    assert torch.equal(lo, v) and bool((hi > v).all())


def test_ema_coef_is_the_fp32_difference():
    c = R.ema_coef(0.999)
    assert c != 0.001 and c == 1.0 - float(torch.tensor(0.999, dtype=torch.float32))


def test_norm_bound_covers_fp32_sums():
    """The serial-sum part of `norm_bound` against plain fp32 accumulation of positive terms."""
    x = torch.rand(4096, generator=torch.Generator().manual_seed(3)).float()
    acc = torch.zeros((), dtype=torch.float32)
    for v in x:
        acc = acc + v * v
    exact = float((x.double() ** 2).sum())
    assert abs(float(acc) - exact) <= R.norm_bound(4096, 1, 1) * exact
