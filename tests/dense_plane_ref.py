"""fp64 references and error bounds for the dense NVLink data plane (`collectives.cu`,
`dense_step.cu`): the two-shot, TMA two-shot and one-shot all-reduces, the fused dense step and
the asynchronous (Hogwild) dense apply.

Reductions.  Every kernel sums the W ranks' vectors in fp32 (in the rank rotation of the
launcher) and multiplies the sum once by the fp32 scale.  With *exact operands* -- values
k·2^-6, |k| <= 64 (`lm1b_opt_ref.exact_grads`) -- every partial sum is exact in fp32, so the
output is the exact sum times fp32(scale), rounded once to fp32 (`reduce_exact`), then RNE to
bf16 for a bf16 buffer.  With random operands the recursive fp32 sum of W terms is within
(W - 1)·u·Σ|x_p| of the exact one (first order, u = 2^-24), the scale multiply adds one rounding
of the result, and a bf16 store adds half a bf16 ulp (`reduce_bound`).

Optimizer rules.  The rules of `optim_rules.cuh` on random operands are compared with
`optim.apply_dense_` on fp64 copies of the same fp32 state, elementwise:

    |got - ref| <= C_kind · u · M

    M (master) = |w0| + |w_ref| + |w_ref - w0| + W·G·(lr + |w0|)
    M (slot)   = |s0| + |s_ref| + |s_ref - s0| + W·G·(1 + G)
                 (+ |w0|·(p(acc') + p(acc))/lr for FTRL's linear slot, p(a) = a^-lr_power:
                  the rule subtracts (p(acc') - p(acc))/lr·w, a difference of close values)
    FTRL's master also carries M (linear slot)·lr/p(acc'): the rule computes w' from linear'
    divided by quad >= p(acc')/lr.  Random states (|w0| ~ 1) hide that term; states an FTRL
    step produced (small w0, |linear| near l1) do not.

G = |scale|·Σ_p|x_p| bounds the gradient and W·u·G its fp32 error; the G terms carry that error
through the rule.  C_kind is calibrated, not derived: `calibrate` runs the same rule in fp32
(`emulate_fp32`: the rotated fp32 sum, one rounding by the scale, `apply_dense_` in fp32) at
the step the GPU tests run (`hyper(2)`) and in fp64, over 2^18 random states per world size
1..8 from `random_state`, for each of four independent seeds.  C_kind is the smallest power of
two, at least 4, that is at least twice the worst err / (u·M) of all four seeds.  So each
constant sits at least 2x above the worst of about 8.4 million draws; that is a margin over
independent draws, not a proof: the tail is heavy, one seed's worst can be 1.5x another's.
The states keep every denominator of the rules away from zero (accumulators >= 0.1, Adam's
v >= 0.01, centered RMSProp's ms - mg² >= 0.5), so the rules stay well conditioned and a
random draw cannot land on a singularity the calibration never saw.
`tests/test_dense_plane_ref_cpu.py` shows that a fresh fp32 emulation passes and that a dropped
1/W, a neighbouring slice and a clip applied twice fail."""
import torch

from parallax_b200 import optim
from tests.lm1b_opt_ref import U, exact_grads, ulp_bf16

# the kinds of the random-operand dense-step test, and every elementwise kind (async apply)
DENSE_KINDS = ("momentum", "adagrad", "adam", "ftrl", "centered_rmsprop")
ELEMENTWISE_KINDS = optim.KINDS + optim.EXT_KINDS
# every kind, and FTRL at a learning-rate power other than -0.5 (its powf branch)
ELEMENTWISE_VARIANTS = ELEMENTWISE_KINDS + ("ftrl_p",)

# C_kind of the module docstring: (master, slots) for one fused step (`STEP_C`) and for W
# sequential applies of un-averaged gradients (`ASYNC_C`).  `python -m tests.dense_plane_ref`
# prints the worst ratios of the four seeds and these constants.  The worst master ratios were
# 0.57 (sgd) to 1.99 (rmsprop) for the step and up to 2.86 (adadelta) for the async apply; the
# worst slot ratio was 1.43 (ftrl).  FTRL's master bound carries its linear slot's error (see
# `rule_bounds`); with that term its worst master ratios on these random states are 0.64 (ftrl)
# and 0.57 (ftrl_p), step and async alike, so C stays at the floor of 4, about 6x above them.
# States an FTRL step produced need the term: the sparse tests' second step exceeded the bound
# without it.
STEP_C = {k: (4, 4) for k in ELEMENTWISE_VARIANTS}
ASYNC_C = dict(STEP_C)
ASYNC_C.update({"adadelta": (8, 4), "proximal_sgd": (8, 4), "proximal_adagrad": (8, 4)})


def make_opt(kind, wd=0.0):
    """The optimizer of `kind` the random-operand tests run, with hyper-parameters that make
    every term of its rule matter."""
    return {"sgd": lambda: optim.GradientDescent(0.1, weight_decay=wd),
            "momentum": lambda: optim.Momentum(0.1, 0.9, True, weight_decay=wd),
            "adagrad": lambda: optim.Adagrad(0.1, 0.5, weight_decay=wd),
            "adam": lambda: optim.Adam(0.01, weight_decay=wd),
            "rmsprop": lambda: optim.RMSProp(0.01, momentum=0.9, weight_decay=wd),
            "adadelta": lambda: optim.Adadelta(0.5, rho=0.9, epsilon=1e-4, weight_decay=wd),
            "ftrl": lambda: optim.Ftrl(0.1, l1_regularization_strength=0.01,
                                       l2_regularization_strength=0.02, weight_decay=wd),
            "ftrl_p": lambda: optim.Ftrl(0.1, learning_rate_power=-0.3,
                                         l1_regularization_strength=0.01, weight_decay=wd),
            "proximal_sgd": lambda: optim.ProximalGradientDescent(0.1, 0.05, 0.1,
                                                                  weight_decay=wd),
            "proximal_adagrad": lambda: optim.ProximalAdagrad(
                0.1, 0.5, l1_regularization_strength=0.05, l2_regularization_strength=0.1,
                weight_decay=wd),
            "adagrad_da": lambda: optim.AdagradDA(0.1, l1_regularization_strength=0.01,
                                                  l2_regularization_strength=0.1,
                                                  weight_decay=wd),
            "centered_rmsprop": lambda: optim.CenteredRMSProp(0.01, momentum=0.9,
                                                              epsilon=1e-3, weight_decay=wd),
            }[kind]()


# ------------------------------------------------------------------------------- reductions
def f32(x):
    """fp32 value of the Python float x, as a Python float."""
    return float(torch.tensor(x, dtype=torch.float32))


def exact_operands(gen, world, n, device=None):
    """Per-rank fp32 vectors of k·2^-6, |k| <= 64: exact in bf16, every W-way sum exact."""
    return [exact_grads(gen, (n,), 64, 6, device).float() for _ in range(world)]


def random_operands(gen, world, n, dtype, device=None):
    """Per-rank randn vectors, already rounded to `dtype` (returned as fp32)."""
    return [torch.randn(n, generator=gen, device=device).to(dtype).float()
            for _ in range(world)]


def reduce_exact(xs, scale):
    """The kernels' fp32 result of Σ_p x_p · fp32(scale) for exact operands: the exact sum
    times fp32(scale), rounded once (fp64 holds the product exactly)."""
    s = torch.zeros_like(xs[0], dtype=torch.float64)
    for x in xs:
        s += x.double()
    return (s * f32(scale)).float()


def reduce_ref(xs, scale):
    """(fp64 Σ_p x_p · fp32(scale), fp64 |fp32(scale)|·Σ_p |x_p|)."""
    s = torch.zeros_like(xs[0], dtype=torch.float64)
    a = torch.zeros_like(s)
    for x in xs:
        s += x.double()
        a += x.double().abs()
    sc = f32(scale)
    return s * sc, a * abs(sc)


def reduce_bound(ref, G, world, dtype):
    """Per-element bound on |kernel - ref| for random operands: the recursive fp32 sum's
    (W - 1)·u·|scale|·Σ|x_p|, one rounding of the scaled result u·|ref| (the reference already
    uses fp32(scale)), and half a bf16 ulp of the rounded value for a bf16 output."""
    e = (world - 1) * U * G + U * (ref.abs() + (world - 1) * U * G)
    if dtype == torch.bfloat16:
        e = e + 0.5 * ulp_bf16(ref.abs() + e)
    return e


# -------------------------------------------------------------------------- optimizer rules
def _kind(variant):
    return "ftrl" if variant == "ftrl_p" else variant


def random_state(gen, variant, n, device=None):
    """fp32 (master, slots) of one step's start, well conditioned for every rule (see the
    module docstring)."""
    kind = _kind(variant)
    def r(s=1.0):
        return torch.randn(n, generator=gen, device=device) * s

    def pos(lo, s):
        return lo + r(s).abs()
    w = r()
    slots = {
        "sgd": (), "proximal_sgd": (),
        "momentum": (r(0.1),),
        "adagrad": (pos(0.1, 1.0),), "proximal_adagrad": (pos(0.1, 1.0),),
        "adam": (r(0.1), pos(0.01, 0.1)),
        "rmsprop": (pos(0.1, 1.0), r(0.01)),
        "adadelta": (pos(0.1, 1.0), pos(0.1, 1.0)),
        "ftrl": (pos(0.1, 1.0), r(0.1)),
        "adagrad_da": (r(1.0), pos(0.1, 1.0)),
    }.get(kind)
    if kind == "centered_rmsprop":
        mg = r(0.1)
        slots = (mg * mg + pos(0.5, 0.5), mg, r(0.01))
    return w, tuple(s.float() for s in slots)


def hp32(hp):
    """The hyper-parameters as the kernels read them: fp32.  The reference must start from
    these: 1 - β2 of the fp32 β2 = 0.999 is 1.3e-5 (relative) away from 0.001, far more than
    any rounding the bounds allow."""
    return [f32(v) for v in hp]


def apply64(variant, w, slots, g, hp):
    """`optim.apply_dense_` on fp64 copies with the fp32 hyper-parameters: (w', slots').
    (It rounds g to fp32 first.)"""
    w = w.double().clone()
    slots = tuple(s.double().clone() for s in slots)
    optim.apply_dense_(_kind(variant), w, g.double(), slots, hp32(hp))
    return w, slots


def emulate_fp32(variant, w, slots, xs, scale, hp, rank=0):
    """What the fused step computes, in fp32: the ranks' vectors summed in the launcher's
    rotation (rank, rank + 1, ...), one rounding by fp32(scale), the rule in fp32."""
    W = len(xs)
    g = torch.zeros_like(xs[0], dtype=torch.float32)
    for p in range(W):
        g = g + xs[(rank + p) % W].float()
    g = g * torch.tensor(scale, dtype=torch.float32)
    w = w.float().clone()
    slots = tuple(s.float().clone() for s in slots)
    optim.apply_dense_(_kind(variant), w, g, slots, hp32(hp))
    return w, slots


def rule_bounds(kind, w0, s0, w_ref, s_ref, G, world, hp, consts=STEP_C):
    """(master bound, [slot bounds]) of the module docstring."""
    cw, cs = consts[kind]
    lr = hp[optim.HP_LR]
    mw = w0.double().abs() + w_ref.abs() + (w_ref - w0.double()).abs() + \
        world * G * (abs(lr) + w0.double().abs())
    bs = []
    for a, b in zip(s0, s_ref):
        ms = a.double().abs() + b.abs() + (b - a.double()).abs() + world * G * (1 + G)
        if _kind(kind) == "ftrl" and len(bs) == 1:
            pw = -hp[optim.HP_A]
            ms = ms + w0.double().abs() * (s_ref[0].pow(pw) + s0[0].double().pow(pw)) / lr
            # w' = (l1·sign(linear') - linear') / quad, quad >= acc'^-lr_power / lr: the linear
            # slot's error reaches the master divided by quad (it dominates once w0 is itself
            # an FTRL result, small and tied to linear)
            mw = mw + ms * lr / s_ref[0].pow(pw)
        bs.append(cs * U * ms)
    return cw * U * mw, bs


def worst_ratio(err, bound):
    """max err / bound (0 for empty)."""
    if err.numel() == 0:
        return 0.0
    return float((err / bound.clamp_min(1e-300)).max())


def check_rule(tag, kind, w_got, s_got, w0, s0, w_ref, s_ref, G, world, hp, consts=STEP_C):
    """Assert the master and every slot within `rule_bounds`; returns the worst ratio."""
    bw, bs = rule_bounds(kind, w0, s0, w_ref, s_ref, G, world, hp, consts)
    worst = 0.0
    pairs = [("master", w_got, w_ref, bw)] + \
        [("slot%d" % i, g, r, b) for i, (g, r, b) in enumerate(zip(s_got, s_ref, bs))]
    for name, got, ref, b in pairs:
        err = (got.double() - ref).abs()
        bad = ~(err <= b)
        if bool(bad.any()):
            i = int(torch.argmax(bad.to(torch.int8)))
            raise AssertionError("%s %s %s: %d of %d out of bound; first at %d: got %r ref %r "
                                 "bound %r" % (tag, kind, name, int(bad.sum()), bad.numel(), i,
                                               float(got.reshape(-1)[i]),
                                               float(ref.reshape(-1)[i]),
                                               float(b.reshape(-1)[i])))
        worst = max(worst, worst_ratio(err, b))
    return worst


def calibrate(kind, n=1 << 18, worlds=range(1, 9), seed=0, sequential=False):
    """Worst err / (u·M) of `emulate_fp32` against fp64 (both C = 1), over `worlds`.
    `sequential`: the async apply -- each rank's un-averaged gradient applied in turn."""
    gen = torch.Generator().manual_seed(seed)
    opt = make_opt(kind)
    hp = opt.hyper(2)           # the step the GPU tests run
    unit = {kind: (1, 1)}
    worst_w = worst_s = 0.0
    for W in worlds:
        w0, s0 = random_state(gen, kind, n)
        xs = random_operands(gen, W, n, torch.float32)
        if sequential:
            w32, s32 = w0, s0
            w64, s64 = w0.double(), tuple(s.double() for s in s0)
            for x in xs:
                w32, s32 = emulate_fp32(kind, w32, s32, [x], 1.0, hp)
                w64, s64 = apply64(kind, w64, s64, x.double(), hp)
            G = sum(x.double().abs() for x in xs)
        else:
            w32, s32 = emulate_fp32(kind, w0, s0, xs, 1.0 / W, hp)
            g64, G = reduce_ref(xs, 1.0 / W)
            w64, s64 = apply64(kind, w0, s0, g64, hp)
        bw, bs = rule_bounds(kind, w0, s0, w64, s64, G, W, hp, unit)
        worst_w = max(worst_w, worst_ratio((w32.double() - w64).abs(), bw))
        for got, ref, b in zip(s32, s64, bs):
            worst_s = max(worst_s, worst_ratio((got.double() - ref).abs(), b))
    return worst_w, worst_s


def suggested(worst):
    """The smallest power of two, at least 4, that is at least 2x the worst ratio."""
    c = 4
    while c < 2 * worst:
        c *= 2
    return c


CALIBRATION_SEEDS = (0, 1, 2, 3)


if __name__ == "__main__":
    for seq in (False, True):
        for k in ELEMENTWISE_VARIANTS:
            rs = [calibrate(k, seed=sd, sequential=seq) for sd in CALIBRATION_SEEDS]
            ww, ws = max(r[0] for r in rs), max(r[1] for r in rs)
            print("async" if seq else "step", k, (ww, ws), (suggested(ww), suggested(ws)))
