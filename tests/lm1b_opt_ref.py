"""fp64 references and derived error bounds for the LM1B optimizer step: Adagrad(0.2, 1.0) on
the clipped LSTM bucket (`dense_step.cu`, modes 1 and 2, EMA 0.999) and on the embedding and
softmax tables (`sparse.cu`, owner kernel).

The bounds follow the kernels' fp32 arithmetic operation by operation (`optim_rules.cuh`):

    s = fmaf(g, g, s)                    one rounding of the accumulator
    w = fmaf(-lr * g, rsqrtf(s), w)      the rounding of lr·g, rsqrtf's 2 ulp, one final rounding
    m -= (1.f - decay) * (m - w)         EMA (dense only)

and are carried elementwise along the fp64 trajectory, first order in u = 2^-24.  A kernel result
is accepted when its error is at most MARGIN times the bound; MARGIN covers the second-order
terms and nothing else.  `tests/test_lm1b_opt_ref_cpu.py` shows that an emulation of the kernel
arithmetic stays inside and that the kernels' likely slips do not."""
import math

import torch

U = 2.0 ** -24            # fp32 unit roundoff (round to nearest)
RSQRT_REL = 2.0 ** -22    # rsqrtf: at most 2 ulp, and an fp32 ulp is <= 2^-23 of the value
MARGIN = 2.0

LR = 0.2
ACC0 = 1.0
MAX_NORM = 10.0
EMA_DECAY = 0.999
EMB_SCALE = 128.0         # ScaleGradients(batch_size) on `emb`

# LM1B's LSTM variables at the benchmark's shapes, in module order (`models/lm1b.py`)
LSTM_ITEMS = (("W", (1024, 8192)), ("B", (8192,)), ("W_P", (2048, 512)))
LM1B_V, LM1B_D, LM1B_P = 793470, 512, 32


def f32(x):
    """The fp32 value of the Python float x, as a Python float."""
    return float(torch.tensor(x, dtype=torch.float32))


def ema_coef(decay):
    """What the kernel subtracts with: (1.f - decay) with decay already an fp32 (exact, Sterbenz)."""
    return float(torch.tensor(1.0, dtype=torch.float32) - torch.tensor(decay, dtype=torch.float32))


# ------------------------------------------------------------------------------- dense layout
def dense_layout(world, items=LSTM_ITEMS, es=2):
    """[(name, offset, numel)] and the bucket length n, as `NVDenseGroup._build_buckets` lays a
    bucket out: tensors in reverse module order, each padded to a whole 16-byte vector, the
    total padded to a multiple of W·vn·32."""
    vn = 16 // es
    out, off = [], 0
    for name, shape in reversed(items):
        numel = math.prod(shape)
        out.append((name, off, numel))
        off += (numel + vn - 1) // vn * vn
    q = world * vn * 32
    return out, (off + q - 1) // q * q


def dense_grid(n, world, max_blocks, num_sms=132, vn=8, threads=512):
    """(CTAs, grid-stride iterations per thread) of one rank's `px_dense_step` launch: one
    thread per 16-byte vector of the slice, capped at 4·NUM_SMS CTAs at W = 1 and at
    `max_blocks` otherwise."""
    nvec = n // world // vn
    b = (nvec + threads - 1) // threads
    cap = num_sms * 4 if world == 1 else (max_blocks if max_blocks > 0 else num_sms)
    ctas = max(1, min(b, cap))
    return ctas, -(-nvec // (ctas * threads))


def padding_mask(layout, n, device=None):
    """bool [n]: True on the elements that belong to no tensor."""
    m = torch.ones(n, dtype=torch.bool, device=device)
    for _, off, numel in layout:
        m[off:off + numel] = False
    return m


# ----------------------------------------------------------------------------------- inputs
def exact_grads(gen, shape, lim, frac_bits, device=None):
    """bf16 values k·2^-frac_bits, |k| <= lim: sums of a few of them are exact in fp32 and,
    while they need at most 8 significant bits, in bf16."""
    k = torch.randint(-lim, lim + 1, shape, generator=gen, device=device)
    return (k.float() * 2.0 ** -frac_bits).bfloat16()


def dense_grads(gen, world, n, exact, device=None):
    """Per-rank bf16 gradient buckets of one step: k·2^-6, |k| <= 64 (the W-way fp32 sum and
    the 1/W scale are then exact), or randn."""
    if exact:
        return [exact_grads(gen, (n,), 64, 6, device) for _ in range(world)]
    return [torch.randn(n, generator=gen, device=device).bfloat16() for _ in range(world)]


def sparse_ids(gen, V, n, rank, device=None):
    """`n` int64 ids of one rank with the forced cases: 40 copies of a rank-specific id, 20 of an
    id every rank carries, the last 32 rows of the table (V-30 .. V-1 are the extra rows of the
    partitions that hold one), one id past the end; the rest uniform."""
    ids = torch.randint(0, V, (n,), generator=gen, device=device)
    ids[:40] = 1000 + 7 * rank
    ids[40:60] = 123457 % V
    ids[60:92] = torch.arange(V - 32, V, device=device)
    ids[100] = V
    return ids


def softmax_ids(gen, V, n_targets, sampled, rank, device=None):
    """The softmax group's ids of one rank: `n_targets` targets (the forced cases of
    `sparse_ids`, 200 of the sampled ids and the 40 most frequent ids, so targets and samples
    collide), followed by the unique log-uniform samples `sampled`."""
    t = sparse_ids(gen, V, n_targets, rank, device)
    t[200:400] = sampled[:200]
    t[400:440] = torch.arange(40, device=device)
    return torch.cat([t, sampled.to(t.device)])


# ---------------------------------------------------------------------- Adagrad, fp64 + bound
def adagrad_fp64(w, acc, g, lr):
    """One Adagrad step in fp64: (w', acc')."""
    s = acc + g * g
    return w - lr * g / s.sqrt(), s


def adagrad_bound(w, acc, g, lr, ew, es, g_err=0.0, g_rel=0.0):
    """Carry the elementwise error bounds (ew on w, es on acc) over one kernel step.

    w, acc, g: the fp64 state before the step and the fp64 gradient of the reference; the
    kernel's gradient may differ from g by g_err (absolute, e.g. an fp32 W-way sum or a bf16
    wire rounding) and then by one relative rounding g_rel (the mode-2 multiply by the clip
    scale: 2^-24).  Returns (ew', es') for the state after the step."""
    ag = g.abs()
    eg = g_err + g_rel * (ag + g_err)
    s = acc + g * g
    # fmaf(g, g, s): the carried error, the gradient's, one rounding of the result
    es_n = es + 2 * ag * eg + eg * eg
    es_n = es_n + U * (s + es_n)
    # δ = lr·g·rsqrt(s): rounding of lr·g, rsqrtf, the accumulator's relative error halved by
    # the square root, the gradient's error
    s_lo = (s - es_n).clamp_min(s * 0.5)
    delta = lr * ag / s.sqrt()
    ed = delta * (U + RSQRT_REL + es_n / (2 * s_lo)) + lr * eg / s_lo.sqrt()
    # the final fma rounds once, relative to its result
    w_n = w - lr * g / s.sqrt()
    ew_n = ew + ed + U * (w_n.abs() + ew + ed)
    return ew_n, es_n


# -------------------------------------------------------------------------------------- EMA
def ema_fp64(m, w, c):
    """m' = m - c·(m - w) in fp64, c = `ema_coef(decay)`."""
    return m - c * (m - w)


def ema_bound(m, w_new, c, em, ew_new):
    """Error bound on the kernel's EMA after one step: m̂ - ŵ (one rounding), its product with c
    (one rounding, or none when fused into an fma), the subtraction (one rounding)."""
    d = (m - w_new).abs() + em + ew_new
    m_n = ema_fp64(m, w_new, c)
    return (1 - c) * em + c * ew_new + c * U * d + c * d * U + U * (m_n.abs() + em + c * d)


# ------------------------------------------------------------------------------------- norm
def norm_bound(vn, iters, ctas, threads=512, ranks=1):
    """Relative error bound of the fp32 Σg² of the mode-1 reduction (every term >= 0): each
    thread adds vn·iters squares in sequence, the block sums its threads in a two-level warp
    tree (log2 32 + log2 32 levels), the CTAs add into one float with one atomic each, and the
    one-shot all-reduce adds the ranks' partials.  One more rounding for each square."""
    depth = 1 + vn * iters + 2 * 5 + ctas + (ranks - 1)
    assert threads <= 1024
    return depth * U / (1 - depth * U)


# ------------------------------------------------------------------------------------- bf16
def ulp_bf16(x):
    """Spacing of bf16 at |x| (x fp64): 2^(e-8) for |x| in [2^(e-1), 2^e); 2^-133 below the
    normal range."""
    _, e = torch.frexp(x.abs().clamp_min(2.0 ** -126))
    return torch.ldexp(torch.ones_like(x), (e - 8).to(torch.int32))


def _f32_down(x):
    y = x.float()
    return torch.where(y.double() > x, torch.nextafter(y, torch.full_like(y, -math.inf)), y)


def bf16_floor(x):
    """Largest bf16 value <= x (fp64 in, fp64 out)."""
    u = _f32_down(x).view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    t = u & 0xFFFF0000
    t = torch.where(((u >> 31) == 1) & ((u & 0xFFFF) != 0), t + 0x10000, t)
    t = torch.where(t >= 2 ** 31, t - 2 ** 32, t).to(torch.int32)
    return t.view(torch.float32).double()


def bf16_bracket(lo, hi):
    """(largest bf16 <= lo, smallest bf16 >= hi): where any bf16 rounding of a value in [lo, hi]
    that moves by at most one bf16 step lands."""
    return bf16_floor(lo), -bf16_floor(-hi)


def sr_ulps(got, ref):
    """(got - ref) / ulp_bf16(ref) over the elements whose fp64 value is not a bf16 value: the
    draws of a stochastic rounding to bf16, in units of the spacing."""
    m = bf16_floor(ref) != ref
    return ((got - ref) / ulp_bf16(ref))[m]


# ------------------------------------------------------------------- the dense bucket, 3 steps
class DenseRef(object):
    """fp64 trajectory and carried bounds of one bucket (full length n, every owner's slice
    concatenated) under Adagrad + EMA.  `exact`: the per-rank gradients are k·2^-6, |k| <= 64,
    so the fp32 W-way sum and its 1/W are exact; otherwise the fp32 sum's error is carried."""

    def __init__(self, w0, world, exact, lr=LR, decay=EMA_DECAY):
        self.w = w0.double().clone()
        self.s = torch.full_like(self.w, ACC0)
        self.m = self.w.clone()
        self.ew = torch.zeros_like(self.w)
        self.es = torch.zeros_like(self.w)
        self.em = torch.zeros_like(self.w)
        self.world, self.exact = world, exact
        self.lr, self.c = f32(lr), ema_coef(decay)

    def mean_grad(self, grads):
        """(ḡ in fp64, bound on |fp32 ḡ - ḡ|) of the per-rank bf16 buckets."""
        W = self.world
        g = torch.zeros_like(self.w)
        a = torch.zeros_like(self.w)
        for x in grads:
            g += x.double()
            a += x.double().abs()
        err = torch.zeros_like(g) if self.exact else (W - 1) * U * a / W
        return g / W, err

    def check_norm(self, grads, norm_k, scale_k, vn, iters, ctas):
        """The kernel's global norm and clip scale against fp64 -> (norm ratio, scale ratio)."""
        g, err = self.mean_grad(grads)
        ss = float((g * g).sum())
        rel = norm_bound(vn, iters, ctas, ranks=self.world) + \
            float((2 * g.abs() * err + err * err).sum()) / ss
        n64 = math.sqrt(ss)
        r_norm = check_bound("global norm", torch.tensor([abs(norm_k - n64)]),
                             torch.tensor([(rel / 2 + U) * n64]))
        want = MAX_NORM / max(n64, MAX_NORM)
        r_scale = check_bound("clip scale", torch.tensor([abs(scale_k - want)]),
                              torch.tensor([(rel / 2 + 2 * U) * want]))
        return r_norm, r_scale

    def step(self, grads, scale_k=None):
        """One update with the mean gradient times the kernel's own clip scale (mode 2: one
        fp32 multiply) or, without one, as it is (mode 0)."""
        g, err = self.mean_grad(grads)
        g_rel = 0.0
        if scale_k is not None:
            g, err, g_rel = g * scale_k, err * scale_k, U
        ew, es = adagrad_bound(self.w, self.s, g, self.lr, self.ew, self.es, err, g_rel)
        w, s = adagrad_fp64(self.w, self.s, g, self.lr)
        self.em = ema_bound(self.m, w, self.c, self.em, ew)
        self.m = ema_fp64(self.m, w, self.c)
        self.w, self.s, self.ew, self.es = w, s, ew, es

    def check(self, w_k, s_k, m_k, tag=""):
        """Master, accumulator and EMA against fp64 -> their worst ratios."""
        return (check_bound(tag + "master", (w_k.double() - self.w).abs(), self.ew),
                check_bound(tag + "accumulator", (s_k.double() - self.s).abs(), self.es),
                check_bound(tag + "ema", (m_k.double() - self.m).abs(), self.em))


# ------------------------------------------------------------------------ sparse rows, 3 steps
def sparse_row_grads(ids, grads, V, scale, exact):
    """The gradient the owner applies to each touched row: (unique ids, fp64 sums [u, D],
    bound [u, D] on the kernel's deviation).  Each sender sums its duplicates in fp32, scales
    and rounds to bf16 once (the wire); the owner adds the senders' rows in fp32.  `exact`: the
    inputs make every one of these sums and roundings exact."""
    D = grads[0].shape[1]
    dev = grads[0].device
    keep = [(i >= 0) & (i < V) for i in ids]
    all_ids = torch.cat([i[k] for i, k in zip(ids, keep)])
    u, inv = torch.unique(all_ids, return_inverse=True)
    g64 = torch.zeros(u.numel(), D, dtype=torch.float64, device=dev)
    g64.index_add_(0, inv, torch.cat([g[k].double() for g, k in zip(grads, keep)]) * scale)
    if exact:
        return u, g64, torch.zeros_like(g64)
    err = torch.zeros_like(g64)
    wabs = torch.zeros_like(g64)
    nsrc = torch.zeros(u.numel(), 1, dtype=torch.float64, device=dev)
    for i, g, k in zip(ids, grads, keep):
        us, invs, cnt = torch.unique(i[k], return_inverse=True, return_counts=True)
        x = g[k].double()
        S = torch.zeros(us.numel(), D, dtype=torch.float64, device=dev).index_add_(0, invs, x)
        A = torch.zeros_like(S).index_add_(0, invs, x.abs())
        A = (cnt[:, None] - 1).double() * U * A
        # unique rows leave as scaled bf16 values (exact); duplicated ones as one RNE rounding
        # of their scaled fp32 sum
        e = torch.where(cnt[:, None] > 1, scale * A + 0.5 * ulp_bf16(scale * (S.abs() + A)),
                        torch.zeros_like(S))
        pos = torch.searchsorted(u, us)
        err.index_add_(0, pos, e)
        wabs.index_add_(0, pos, scale * S.abs() + e)
        nsrc.index_add_(0, pos, torch.ones_like(nsrc[:us.numel()]))
    return u, g64, err + (nsrc - 1).clamp_min(0) * U * wabs


class SparseRef(object):
    """fp64 rows and carried bounds of every row a run touches (`rows`, sorted global ids)."""

    def __init__(self, rows, w0, lr=LR):
        self.rows = rows
        self.w = w0.double().clone()
        self.s = torch.full_like(self.w, ACC0)
        self.ew = torch.zeros_like(self.w)
        self.es = torch.zeros_like(self.w)
        self.lr = f32(lr)

    def step(self, u, g64, gerr):
        i = torch.searchsorted(self.rows, u)
        assert bool((self.rows[i] == u).all())
        w, s, ew, es = self.w[i], self.s[i], self.ew[i], self.es[i]
        self.ew[i], self.es[i] = adagrad_bound(w, s, g64, self.lr, ew, es, gerr)
        self.w[i], self.s[i] = adagrad_fp64(w, s, g64, self.lr)

    def check(self, w_k, s_k, tag=""):
        return (check_bound(tag + "rows", (w_k.double() - self.w).abs(), self.ew),
                check_bound(tag + "accumulators", (s_k.double() - self.s).abs(), self.es))


def check_bound(name, err, bound, margin=MARGIN):
    """Assert err <= margin·bound elementwise; returns the worst err / (margin·bound)."""
    lim = margin * bound
    ok = err <= lim
    ratio = float((err / lim.clamp_min(1e-300)).max()) if err.numel() else 0.0
    if not bool(ok.all()):
        i = int(torch.argmax((err - lim).reshape(-1)))
        raise AssertionError("%s: %d of %d elements out of bound; worst at %d: err %r bound %r"
                             % (name, int((~ok).sum()), ok.numel(), i,
                                float(err.reshape(-1)[i]), float(lim.reshape(-1)[i])))
    return ratio
