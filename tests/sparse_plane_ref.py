"""fp64 references and error bounds for the sparse owner kernel (`px_sparse_owner_kernel`) and
the asynchronous (Hogwild) apply of the sparse push kernel, `ops/csrc/kernels/sparse.cu`.

The owner starts from its receive rings.  The push is tested bit for bit on its own
(`test_gpu_sparse_push.py`), so the references here read what it wrote (`merged`, after every
rank's `stage_push` and before any `stage_apply`) and model only the owner: for each touched
row it sums the row's n_e ring entries in fp32 (in the order its list happens to hold them),
multiplies the sum once by

    gmul = fp32(fp32(avg) · fp32(hp[HP_GSCALE]))                         (`gmul`)

where avg = 1/W with `average_sparse` (else 1), times the ScaleGradients factor when the
sender did not apply it (boundary optimisation off), and then runs the rule of
`optim_rules.cuh` on the row's own state.  That is the dense step's model
(`tests/dense_plane_ref.py`) with world := n_e per row, scale := gmul and
G = |gmul|·Σ|entries|, so its bounds `rule_bounds` / `check_rule` and constants `STEP_C` apply
as they stand (`apply_dense_` multiplies by hp[HP_GSCALE] itself, so the reference runs with
GSCALE 1 once gscale is folded into gmul).  The constants were calibrated for up to 8 summed
terms; the random-operand GPU cases keep every row at no more than W <= 8 entries (ids are
unique within a sender), so they need no calibration beyond that.  FTRL's master bound gained
its linear slot's term (`rule_bounds`), and `STEP_C` / `ASYNC_C` for ftrl and ftrl_p were
recalibrated with it (the ratios are recorded in `dense_plane_ref`).  Rows with more entries
(duplicates without local aggregation) run only with exact operands.

Exact operands (`predict_exact`): lr 2^-3, momentum 0.5, weights and slots on a 2^-10 grid and
gradients k·2^-6.  Every ring entry is then a multiple of 2^-7 and every partial sum of a row
stays below 2^17, so the owner's fp32 sum is exact in any order; g·gmul rounds once, and each
`fmaf` of sgd, momentum and Nesterov momentum rounds once.  `fma32` rounds a·b + c correctly
to fp32 (round to odd in fp64, then to nearest in fp32), so the prediction is the kernel's
value bit for bit, at every W, including 3, 5, 6 and 7 where 1/W is inexact.

The async apply runs each sender's rows through the rule in turn: each row of sender p is
g_p = fp32(x_p · fp32(scale · gscale)) applied to the state sender p - 1 left.  The reference
chains `apply64` over the senders from the step's start and is held to `ASYNC_C`, with
world := the number of senders that touched the row.

bf16 master rows (`sparse_weights="bf16"`): the rule runs in fp32 on the widened bf16 master,
then the result is rounded stochastically.  The stored value must lie in `bf16_bracket` of
[ref - bound, ref + bound], with ref the fp64 step from the previous *stored* state.

`tests/test_sparse_plane_ref_cpu.py` shows that an fp32 emulation of the owner passes and
that the slips a sparse data path is likely to make fail."""
import collections

import torch

from parallax_b200 import optim
from tests.dense_plane_ref import ASYNC_C, apply64, check_rule, f32, rule_bounds, worst_ratio
from tests.lm1b_opt_ref import bf16_bracket

# the variants the exact (bit-for-bit) tests predict, and their optimizers
EXACT_KINDS = ("sgd", "momentum", "nesterov")
EXACT_LR = 2.0 ** -3
EXACT_MOMENTUM = 0.5


def make_exact_opt(kind):
    return {"sgd": lambda: optim.GradientDescent(EXACT_LR),
            "momentum": lambda: optim.Momentum(EXACT_LR, EXACT_MOMENTUM, False),
            "nesterov": lambda: optim.Momentum(EXACT_LR, EXACT_MOMENTUM, True)}[kind]()


def grid_state(gen, kind, shape, device=None):
    """(master, slots) on the 2^-10 grid, |x| <= 1: the exact tests' starting state."""
    def r():
        return (torch.randint(-1024, 1025, shape, generator=gen).float() * 2.0 ** -10).to(device)
    return r(), tuple(r() for _ in range(optim.NUM_SLOTS["momentum" if kind == "nesterov"
                                                        else kind]))


# -------------------------------------------------------------------------------- owner side
def owner_avg(world, average, scale=1.0, boundary=True, micro_batches=1):
    """The fp32 `avg` of the owner's descriptor (`NVSparseGroup._owner_tables`): 1/W with
    `average_sparse`, / micro-batches, × the ScaleGradients factor when the sender did not
    apply it."""
    avg = (1.0 / world) if average else 1.0
    avg /= micro_batches
    return f32(avg if boundary else avg * scale)


def gmul(avg, gscale=1.0):
    """The owner's gradient multiplier: fp32(fp32(avg) · fp32(gscale))."""
    return f32(f32(avg) * f32(gscale))


def hp_folded(hp):
    """hp with GSCALE 1: the reference multiplies by gmul, which already holds it."""
    hp = list(hp)
    hp[optim.HP_GSCALE] = 1.0
    return hp


Ring = collections.namedtuple("Ring", "rows sum abs_sum count")


def merged(grp):
    """This owner's receive rings, merged per row in fp64, one `Ring` per member table: the
    local rows it touched (sorted), their sums [m, D], Σ|entry| [m, D] and entry counts [m, 1].
    Read after every rank's `stage_push` and before `stage_apply`."""
    from parallax_b200 import ops
    W, cap = grp.world, grp.cap
    R = ops.sparse_abi()["hdr_words"] // 3
    cnt = grp.hdr_buf.tensor(torch.int32, 3 * R).cpu()[2 * R:2 * R + W].tolist()
    ring_ids = grp.ids_buf.tensor(torch.int32, W * cap).view(W, cap).cpu()
    ids = torch.cat([ring_ids[s, :cnt[s]] for s in range(W)]).long()
    keep = ids >= 0
    u, inv, n = torch.unique(ids[keep], return_inverse=True, return_counts=True)
    out = []
    for t in grp.tables:
        ring = t.ring_buf.tensor(grp.wire_dtype, W * cap * t.Dp).view(W, cap, t.Dp).cpu()
        vals = torch.cat([ring[s, :cnt[s]].double() for s in range(W)])[keep]
        m = torch.zeros(u.numel(), t.Dp, dtype=torch.float64).index_add_(0, inv, vals)
        a = torch.zeros_like(m).index_add_(0, inv, vals.abs())
        out.append(Ring(u, m[:, :t.D], a[:, :t.D], n[:, None].double()))
    return out


def owner_ref(variant, w0, s0, ring, g_mul, hp):
    """fp64 (w', slots', G, n_e) of the owner's step on rows `ring.rows` from the fp32 state
    (w0, s0) of those rows."""
    w, s = apply64(variant, w0, s0, ring.sum * g_mul, hp_folded(hp))
    return w, s, ring.abs_sum * abs(g_mul), ring.count


def check_owner(tag, variant, w_got, s_got, w0, s0, ring, g_mul, hp):
    """Master and slots of the touched rows within `rule_bounds` (`STEP_C`); the worst ratio."""
    w_ref, s_ref, G, n_e = owner_ref(variant, w0, s0, ring, g_mul, hp)
    return check_rule(tag, variant, w_got, s_got, w0, s0, w_ref, s_ref, G, n_e, hp)


def check_owner_bf16(tag, variant, w_got, s_got, w0, s0, ring, g_mul, hp):
    """bf16 master: the stored bf16 value in `bf16_bracket` of [ref - bound, ref + bound] (the
    rule's fp32 error, then one stochastic rounding); the fp32 slots within their bounds.
    Returns the worst slot ratio."""
    w_ref, s_ref, G, n_e = owner_ref(variant, w0, s0, ring, g_mul, hp)
    bw, bs = rule_bounds(variant, w0, s0, w_ref, s_ref, G, n_e, hp)
    lo, hi = bf16_bracket(w_ref - bw, w_ref + bw)
    got = w_got.double()
    bad = (got < lo) | (got > hi)
    if bool(bad.any()):
        i = int(torch.argmax(bad.to(torch.int8).reshape(-1)))
        raise AssertionError("%s %s bf16 master: %d of %d outside the bracket; first at %d: "
                             "got %r ref %r bound %r" % (
                                 tag, variant, int(bad.sum()), bad.numel(), i,
                                 float(got.reshape(-1)[i]), float(w_ref.reshape(-1)[i]),
                                 float(bw.reshape(-1)[i])))
    worst = 0.0
    for k, (g, r, b) in enumerate(zip(s_got, s_ref, bs)):
        err = (g.double() - r).abs()
        if not bool((err <= b).all()):
            raise AssertionError("%s %s bf16 master slot%d: %d of %d out of bound, worst "
                                 "err/bound %g" % (tag, variant, k, int((err > b).sum()),
                                                   err.numel(), worst_ratio(err, b)))
        worst = max(worst, worst_ratio(err, b))
    return worst


# ------------------------------------------------------------------------- exact prediction
def _round_to_odd_sum(p, c):
    """fp64 p + c rounded to odd (p, c fp64): the two-sum's error decides the sticky bit."""
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    even = (s.view(torch.int64) & 1) == 0
    toward = torch.where(e > 0, torch.full_like(s, float("inf")), torch.full_like(s, -float("inf")))
    return torch.where((e != 0) & even, torch.nextafter(s, toward), s)


def fma32(a, b, c):
    """fp32 fmaf(a, b, c), correctly rounded, for fp32 values held in fp64 tensors (or floats):
    a·b is exact in fp64, the sum is rounded to odd in fp64 (53 >= 24 + 2 bits), then to
    nearest in fp32.  Returns fp64 holding the fp32 result."""
    a, b, c = (torch.as_tensor(x, dtype=torch.float64) for x in (a, b, c))
    return _round_to_odd_sum(a * b, c).float().double()


def mul32(a, b):
    """fp32 a·b (one rounding: the product of two fp32 values is exact in fp64)."""
    return (torch.as_tensor(a, dtype=torch.float64) * b).float().double()


def predict_exact(kind, w0, s0, g):
    """The kernel's fp32 result of sgd / momentum / Nesterov momentum at `EXACT_LR` and
    `EXACT_MOMENTUM` on fp32 state (w0, s0) with the fp32 gradient g (fp64 in, fp32 out)."""
    lr, a = f32(EXACT_LR), f32(EXACT_MOMENTUM)
    w = w0.double()
    g = g.double()
    if kind == "sgd":
        return fma32(-lr, g, w).float(), ()
    s = fma32(a, s0[0].double(), g)
    d = fma32(a, s, g) if kind == "nesterov" else s
    return fma32(-lr, d, w).float(), (s.float(),)


def predict_owner_exact(kind, w0, s0, ring, g_mul):
    """`predict_exact` for the owner's rows: the exact ring sum times gmul, rounded once."""
    assert ring.abs_sum.numel() == 0 or float(ring.abs_sum.max()) < 2.0 ** 17
    assert bool((ring.sum * 2 ** 7 == (ring.sum * 2 ** 7).round()).all()), \
        "ring entries are not exact operands"
    return predict_exact(kind, w0, s0, mul32(ring.sum, g_mul))


# -------------------------------------------------------------------------------- async apply
def async_ref(variant, w0, s0, senders, hp):
    """fp64 chain of the async apply over `senders` = [(rows, g [m, D] fp32 as applied)], in
    order, from (w0, s0) of the whole table: (w, slots, G, touched count) over every row."""
    w = w0.double().clone()
    s = tuple(x.double().clone() for x in s0)
    G = torch.zeros_like(w)
    n = torch.zeros(w.shape[0], 1, dtype=torch.float64)
    for rows, g in senders:
        wr, sr = apply64(variant, w[rows], tuple(x[rows] for x in s), g.double(),
                         hp_folded(hp))
        w[rows] = wr
        for x, y in zip(s, sr):
            x[rows] = y
        G[rows] += g.double().abs()
        n[rows] += 1
    return w, s, G, n


def check_async(tag, variant, w_got, s_got, w0, s0, senders, hp, rows):
    """The async result on `rows` (every row some sender touched) within `ASYNC_C`."""
    w, s, G, n = async_ref(variant, w0, s0, senders, hp)
    return check_rule(tag, variant, w_got[rows], tuple(x[rows] for x in s_got), w0[rows],
                      tuple(x[rows] for x in s0), w[rows], tuple(x[rows] for x in s),
                      G[rows], n[rows], hp, ASYNC_C)


# ------------------------------------------------------------------------------ fp32 emulation
def emulate_owner(variant, w0, s0, entries, g_mul, hp, gen):
    """What the owner computes for rows whose ring entries are `entries` ([m, n_max, D] fp32,
    zero past a row's last entry): each row's entries summed in fp32 in its own shuffled
    order, × gmul in fp32, the rule in fp32."""
    m, nmax, D = entries.shape
    perm = torch.rand(m, nmax, generator=gen).argsort(1)
    e = entries.float().gather(1, perm[:, :, None].expand(-1, -1, D))
    g = torch.zeros(m, D, dtype=torch.float32)
    for k in range(nmax):
        g = g + e[:, k]
    g = g * torch.tensor(g_mul, dtype=torch.float32)
    w = w0.float().clone()
    s = tuple(x.float().clone() for x in s0)
    optim.apply_dense_(variant if variant != "ftrl_p" else "ftrl", w, g, s, hp_folded(hp))
    return w, s


def ring_of(entries, count):
    """The `Ring` of rows whose (zero-padded) entries are `entries` [m, n_max, D]."""
    e = entries.double()
    return Ring(torch.arange(e.shape[0]), e.sum(1), e.abs().sum(1), count.double()[:, None])
