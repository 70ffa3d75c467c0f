"""The sparse-plane references of `tests/sparse_plane_ref.py` (used by
`test_gpu_sparse_plane.py`) on the CPU: an fp32 emulation of the owner kernel and of the async
apply stays inside the bounds for every elementwise rule, the exact prediction rounds like
fmaf, and the slips a sparse data path is likely to make fail: the neighbouring row's slots,
the slots' initial values instead of the row's own, 1/W dropped or applied twice,
ScaleGradients applied on both sides, a dropped ring entry, and the async senders' rows applied
as one averaged update."""
from fractions import Fraction

import pytest
import torch

from parallax_b200 import optim
from tests import dense_plane_ref as DR
from tests import sparse_plane_ref as S
from tests.lm1b_opt_ref import bf16_floor

M, D = 2048, 8
WITH_SLOTS = tuple(k for k in DR.ELEMENTWISE_VARIANTS if k not in ("sgd", "proximal_sgd"))


def _entries(gen, world, m=M):
    """Ring entries of m rows: each row carries 1..W entries of randn (zero past its last)."""
    count = torch.randint(1, world + 1, (m,), generator=gen)
    e = torch.randn(m, world, D, generator=gen)
    e = e * (torch.arange(world)[None, :] < count[:, None])[:, :, None]
    return e, count


def _case(kind, world, seed, avg=None, m=M):
    gen = torch.Generator().manual_seed(seed)
    hp = DR.make_opt(kind).hyper(2)
    w0, s0 = DR.random_state(gen, kind, m * D)
    w0, s0 = w0.view(m, D), tuple(s.view(m, D) for s in s0)
    e, count = _entries(gen, world, m)
    g_mul = S.gmul(S.owner_avg(world, True) if avg is None else avg)
    return gen, hp, w0, s0, e, count, g_mul


def _check(kind, world, hp, w_k, s_k, w0, s0, ring, g_mul):
    return S.check_owner("emulation", kind, w_k, s_k, w0, s0, ring, g_mul, hp)


@pytest.mark.parametrize("kind", DR.ELEMENTWISE_VARIANTS)
@pytest.mark.parametrize("world", [1, 3, 5, 8])
def test_owner_emulation_within_bound(kind, world):
    """Shuffled fp32 merge of 1..W entries per row, × fp32(1/W), the rule in fp32: inside
    `STEP_C` on a seed the calibration never saw."""
    gen, hp, w0, s0, e, count, g_mul = _case(kind, world, 200 + world)
    w_k, s_k = S.emulate_owner(kind, w0, s0, e, g_mul, hp, gen)
    assert _check(kind, world, hp, w_k, s_k, w0, s0, S.ring_of(e, count), g_mul) <= 1.0


@pytest.mark.parametrize("kind", DR.ELEMENTWISE_VARIANTS)
def test_owner_emulation_second_step_within_bound(kind):
    """A step from the state the rule itself produced, as the GPU tests' second step (FTRL's
    master is then small and tied to its linear slot)."""
    gen, hp, w0, s0, e, count, g_mul = _case(kind, 3, 400, m=1 << 16)
    w1, s1 = S.emulate_owner(kind, w0, s0, e, g_mul, hp, gen)
    e, count = _entries(gen, 3, 1 << 16)
    w_k, s_k = S.emulate_owner(kind, w1, s1, e, g_mul, hp, gen)
    assert _check(kind, 3, hp, w_k, s_k, w1, s1, S.ring_of(e, count), g_mul) <= 1.0


@pytest.mark.parametrize("kind", DR.ELEMENTWISE_VARIANTS)
def test_owner_emulation_bf16_master_within_bracket(kind):
    """bf16 master: the emulated fp32 step from the bf16 state, rounded down or up to bf16,
    lands in the bracket."""
    gen, hp, w0, s0, e, count, g_mul = _case(kind, 5, 300)
    w0 = w0.bfloat16().float()
    w_k, s_k = S.emulate_owner(kind, w0, s0, e, g_mul, hp, gen)
    ring = S.ring_of(e, count)
    down = bf16_floor(w_k.double())
    for w_r in (down, -bf16_floor(-w_k.double())):       # a stochastic rounding's two outcomes
        S.check_owner_bf16("emulation", kind, w_r.float(), s_k, w0, s0, ring, g_mul, hp)


@pytest.mark.parametrize("kind", DR.ELEMENTWISE_VARIANTS)
def test_async_emulation_within_bound(kind):
    """W = 5 senders with unique rows each, applied in turn in fp32: inside `ASYNC_C`."""
    gen = torch.Generator().manual_seed(17)
    hp = DR.make_opt(kind).hyper(2)
    w0, s0 = DR.random_state(gen, kind, M * D)
    w0, s0 = w0.view(M, D), tuple(s.view(M, D) for s in s0)
    senders = [(torch.randperm(M, generator=gen)[:M // 2], None) for _ in range(5)]
    senders = [(r, torch.randn(r.numel(), D, generator=gen)) for r, _ in senders]
    w, s = w0.clone(), tuple(x.clone() for x in s0)
    for rows, g in senders:
        wr, sr = w[rows], tuple(x[rows] for x in s)
        optim.apply_dense_(DR._kind(kind), wr, g, sr, hp)
        w[rows] = wr
        for x, y in zip(s, sr):
            x[rows] = y
    rows = torch.unique(torch.cat([r for r, _ in senders]))
    assert S.check_async("emulation", kind, w, s, w0, s0, senders, hp, rows) <= 1.0


# ---------------------------------------------------------------------------------- exactness
def test_fma32_rounds_once():
    """`fma32` against exact rational arithmetic, on operands where fp64 a·b + c rounds (the
    exponents of a·b and c far apart) and on ties of the fp32 rounding."""
    gen = torch.Generator().manual_seed(3)
    a = torch.randn(4000, generator=gen).float().double()
    b = torch.randn(4000, generator=gen).float().double()
    c = (torch.randn(4000, generator=gen) * 2.0 ** torch.randint(-60, 30, (4000,),
                                                                  generator=gen)).float().double()
    got = S.fma32(a, b, c).tolist()
    for x, y, z, r in zip(a.tolist(), b.tolist(), c.tolist(), got):
        exact = Fraction(x) * Fraction(y) + Fraction(z)
        f = float(torch.tensor(float(exact), dtype=torch.float64).float())
        # float(exact) is RNE in fp64, then fp32: wrong only at a double rounding; check the
        # neighbours of f and keep the nearest (ties to even)
        cands = [f, float(torch.nextafter(torch.tensor(f).float(), torch.tensor(1e38))),
                 float(torch.nextafter(torch.tensor(f).float(), torch.tensor(-1e38)))]
        best = min(cands, key=lambda v: (abs(Fraction(v) - exact),
                                         int(torch.tensor(v).float().view(torch.int32)) & 1))
        assert r == best, (x, y, z, r, best)


@pytest.mark.parametrize("kind", S.EXACT_KINDS)
def test_exact_prediction_matches_fp32_rule(kind):
    """On exact operands the prediction is the fp32 rule itself: `apply_dense_` in fp32 agrees
    wherever its separate multiply and add round like one fmaf (their products are exact)."""
    gen = torch.Generator().manual_seed(5)
    w0, s0 = S.grid_state(gen, kind, (M, D))
    g = S.mul32(DR.exact_operands(gen, 3, M * D)[0].view(M, D).double(), S.gmul(1.0 / 3))
    w_p, s_p = S.predict_exact(kind, w0, s0, g)
    opt = S.make_exact_opt(kind)
    w, s = w0.clone(), tuple(x.clone() for x in s0)
    optim.apply_dense_("momentum" if kind == "nesterov" else kind, w, g.float(), s, opt.hyper(1))
    # lr = 2^-3 and momentum = 0.5 scale exactly: every product is exact, so the fp32 rule
    # rounds only at its additions, as the fmas do
    assert torch.equal(w_p, w)
    for x, y in zip(s_p, s):
        assert torch.equal(x, y)


# ---------------------------------------------------------------------------------- the slips
def _slip(kind, world=4, seed=11, **kw):
    gen, hp, w0, s0, e, count, g_mul = _case(kind, world, seed)
    ring = S.ring_of(e, count)
    w_k, s_k = S.emulate_owner(kind, kw.get("w0", lambda w: w)(w0),
                               kw.get("s0", lambda s: s)(s0),
                               kw.get("e", lambda x: x)(e), kw.get("g_mul", g_mul), hp, gen)
    with pytest.raises(AssertionError):
        _check(kind, world, hp, w_k, s_k, w0, s0, ring, g_mul)


@pytest.mark.parametrize("kind", WITH_SLOTS)
def test_neighbouring_row_slots_fail(kind):
    _slip(kind, s0=lambda s: tuple(x.roll(1, 0) for x in s))


@pytest.mark.parametrize("kind", WITH_SLOTS)
def test_initial_slots_instead_of_row_state_fail(kind):
    init = DR.make_opt(kind).slot_init()
    _slip(kind, s0=lambda s: tuple(torch.full_like(x, v) for x, v in zip(s, init)))


@pytest.mark.parametrize("kind", DR.ELEMENTWISE_VARIANTS)
def test_dropped_average_fails(kind):
    _slip(kind, g_mul=1.0)


@pytest.mark.parametrize("kind", DR.ELEMENTWISE_VARIANTS)
def test_average_applied_twice_fails(kind):
    _slip(kind, g_mul=S.gmul(1.0 / 16))


@pytest.mark.parametrize("kind", DR.ELEMENTWISE_VARIANTS)
def test_scale_on_sender_and_owner_fails(kind):
    """ScaleGradients 0.5 on the wire (entries halved) and again in the owner's avg."""
    gen, hp, w0, s0, e, count, _ = _case(kind, 4, 12)
    g_mul = S.gmul(S.owner_avg(4, True, 0.5, boundary=False))
    ring = S.ring_of(e, count)
    w_k, s_k = S.emulate_owner(kind, w0, s0, e * 0.5, g_mul, hp, gen)
    with pytest.raises(AssertionError):
        _check(kind, 4, hp, w_k, s_k, w0, s0, ring, g_mul)


@pytest.mark.parametrize("kind", DR.ELEMENTWISE_VARIANTS)
def test_dropped_ring_entry_fails(kind):
    """The last entry of every row that merges two or more is lost."""
    def drop(e):
        e = e.clone()
        n = (e != 0).any(2).sum(1)
        rows = torch.nonzero(n >= 2).squeeze(1)
        e[rows, n[rows] - 1] = 0
        return e
    _slip(kind, e=drop)


@pytest.mark.parametrize("kind", DR.ELEMENTWISE_VARIANTS)
def test_async_averaged_update_fails(kind):
    """The W = 4 senders' rows (every row from each) applied once, averaged, instead of in turn."""
    gen = torch.Generator().manual_seed(19)
    hp = DR.make_opt(kind).hyper(2)
    w0, s0 = DR.random_state(gen, kind, M * D)
    w0, s0 = w0.view(M, D), tuple(s.view(M, D) for s in s0)
    rows = torch.arange(M)
    senders = [(rows, torch.randn(M, D, generator=gen)) for _ in range(4)]
    w, s = w0.clone(), tuple(x.clone() for x in s0)
    optim.apply_dense_(DR._kind(kind), w, sum(g for _, g in senders) / 4, s, hp)
    with pytest.raises(AssertionError):
        S.check_async("slip", kind, w, s, w0, s0, senders, hp, rows)
