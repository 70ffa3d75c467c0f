"""Exact operands, an fp64 reference and error bounds for the full-softmax kernels
(`ops/csrc/kernels/softmax_eval.cu`): log-sum-exp and NLL, top-k, Gumbel-top-k sampling, the
truncation threshold θ* and masked sampling, and the training gradient.

**Exact operands.**  Table rows, bias and inputs are small integers times powers of two:

- fine rows:   x ∈ {−8..8}·2⁻³, w ∈ {−8..8}·2⁻⁵, b ∈ {−16..16}·2⁻⁴.  Every product x·w is a
  multiple of 2⁻⁸ of magnitude ≤ 2⁻², and at K ≤ 512 every partial sum of x·w (plus b) is a
  multiple of 2⁻⁸ of magnitude < 2⁷ + 1, i.e. an integer times 2⁻⁸ below 2¹⁶ ≤ 2²⁴.  Such a
  number is exact in fp32 (24-bit significand), so every fp32 partial sum is exact in any order
  and the kernels' fp32 logits equal the fp64 ones bit for bit.  The logits have a standard
  deviation of about 2, a realistic softmax over 793 470 words.
- coarse rows: x = ±e_j ± e_l·2⁻³ ± e_m·2⁻⁶ (three distinct columns), so the logit b_v ± w_vj ±
  w_vl/8 ± w_vm/64 is a multiple of 2⁻¹¹ of magnitude < 2, exact in fp32 likewise.  It takes
  about 2·10⁴ distinct values, so the best words of a row share values and most rows have a tie
  across the k-th position: the (logit descending, id ascending) rule decides them.

Every operand has at most 5 significant bits, so it is exact in bf16 (the shadow rows, the bf16
bias masters and X).  With τ ∈ {½, 1, 2}, s = logit · fp32(1/τ) is exact too.

**Reference.**  `reference` computes, in fp64 on the device and in blocks of rows (the [N, V]
logits at V = 793 470 do not fit), each row's lse, its 1001 best words by (s desc, id asc), the
count- and mass-clause θ* of truncated sampling from the exactly sorted row (ties kept
together), and the Gumbel-top-k draws from the keys s − log E in fp64, with log E from
`engine.sample_log_e`: its uniform v is bit-exact, its log E is torch's fp32 value widened to
fp64, which `draw_margin` allows for.

**Bounds** (u = 2⁻²⁴, the fp32 unit roundoff; CUDA's exp2f, logf and log1pf are within 2, 1 and 1
ulp).  Each is an upper bound on |kernel − fp64| derived from the kernels' operation order; the
tests allow 2× the bound and report the worst error/(2·bound).

An absolute error δ in a base-2 exponent x·L2E is a relative error ln2·δ of exp2f's result;
a rounding of x·L2E (δ ≤ u·|x|·L2E) therefore costs at most u·|x|, since ln2·L2E = 1.

- `lse_bound`: a term exp2f(fmaf(v, L2E, −m·L2E)) is within 4u (exp2f) + u·(|v − m| + |m|) (the
  rounded m·L2E and the fma's rounding) of exp((v − m)·(1 + η)), η the relative error of the
  fp32 L2E, which scales every exponent alike and moves lse by at most η·2·max|s|.  A lane
  sums 32 such terms (31 roundings), the quad 2 shuffles; each lse_merge of a (max, Σ) pair
  into the CTA's running pair costs 2 exp2f, their rounded arguments and 2 roundings, and a
  row sees one merge per work item of the CTA and ceil(grid/32) + 5 in the grid merge.  The
  relative error of Σ becomes an absolute error of lse, plus logf (1 ulp of log Σ) and the
  final add (½ ulp of lse).
- `draw_margin`: the fp32 key s − log E is within ½ ulp of key + |Δ log E| of the exact key, and
  log E = logf(−log1pf(−v)) is within 1 ulp + 2·2u relative of E carried through the log, in
  the kernel and in torch alike.
- `grad_bound`: G = bf16(g·(exp2f(fmaf(l, L2E, −lse·L2E)) − [v = t])) is within ½ bf16 ulp
  (2⁻⁹ relative) of the fp32 value, which is within |g|·p·ε_p of the exact one (ε_p as a
  term above, with the lse the kernel is given); db sums the fp32 values (not the bf16 ones)
  over N rows, 2·ceil(N/128) per lane, 3 shuffles and 8 warps; dX = Σ_v G·w and dW = Σ_i G·x
  multiply the bf16 G in fp32 (depth ≤ the chunk's rows or N) and round to bf16."""
import math

import torch

U = 2.0 ** -24
L2E_ERR = abs(float(torch.tensor(math.log2(math.e), dtype=torch.float32)) - math.log2(math.e))
V_LM1B, K_LM1B, P_LM1B = 793470, 512, 32


# ------------------------------------------------------------------ operands
def exact_table(V, K, seed):
    """(W [V, K], b [V, 1]) fp32 on the CPU: w ∈ {−8..8}·2⁻⁵, b ∈ {−16..16}·2⁻⁴."""
    g = torch.Generator().manual_seed(seed)
    W = torch.randint(-8, 9, (V, K), generator=g, dtype=torch.int8).float().mul_(2.0 ** -5)
    b = torch.randint(-16, 17, (V, 1), generator=g, dtype=torch.int8).float().mul_(2.0 ** -4)
    return W, b


def exact_inputs(N, K, seed, coarse_every=4):
    """x [N, K] fp32 (bf16-exact) on the CPU: fine rows x ∈ {−8..8}·2⁻³, and every
    `coarse_every`-th row (row % coarse_every == coarse_every − 1; 0: none) a coarse row ±e_j ±
    e_l/8 ± e_m/64."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(-8, 9, (N, K), generator=g, dtype=torch.int8).float().mul_(2.0 ** -3)
    if coarse_every and K >= 3:
        for r in range(coarse_every - 1, N, coarse_every):
            cols = torch.randperm(K, generator=g)[:3]
            sign = torch.randint(0, 2, (3,), generator=g).float() * 2 - 1
            x[r] = 0.0
            x[r, cols] = sign * torch.tensor([1.0, 2.0 ** -3, 2.0 ** -6])
    return x


def inv_tau(tau):
    """fp32(1/τ) as a Python float, the factor the kernels scale by"""
    return float(torch.tensor(1.0 / tau, dtype=torch.float32))


def coarse_rows(N, coarse_every=4):
    return torch.arange(coarse_every - 1, N, coarse_every) if coarse_every else torch.arange(0)


# ------------------------------------------------------------------ bounds
def _ulp(x):
    """fp32 ulp of |x| (a tensor), at least the smallest normal's"""
    x = x.abs().double().clamp_min(2.0 ** -126)
    return torch.pow(2.0, torch.floor(torch.log2(x)) - 23)


ETA = L2E_ERR / math.log2(math.e)                     # relative error of the fp32 L2E


def lse_bound(lse, smax, items_per_cta, grid):
    """|lse_kernel − lse| for rows with log-sum-exp `lse` and max |s| `smax` (fp64 tensors) when
    a CTA merges `items_per_cta` work items and the grid has `grid` CTAs.

    The fp32 L2E scales every exponent v − max by the same 1 + η, which moves lse by at most
    η·2·max|s|.  A block's own Σ carries exp2f (4u), its 31 lane and 2 quad additions, the
    rounded max·L2E and fma arguments (u·(|v − m| + |m|) ≤ 3u·max|s|), and its rescale
    into the running pair (exp2f and an argument of at most 2·max|s|).  Each merge adds two
    roundings and at most one rescale of the running Σ (exp2f, 4u); the arguments of those
    rescales sum to the rise of the running max, at most 2·max|s|, in the CTA and in the grid."""
    depth = items_per_cta + math.ceil(grid / 32) + 5
    block = 4 * U + 33 * U + U * 3 * smax + 4 * U + 2 * U * 2 * smax
    rel = block + depth * 6 * U + 2 * 2 * U * 2 * smax
    log_s = (lse.abs() + smax).clamp_min(1.0)             # |log Σ| <= |lse| + max |s|
    return rel * 1.01 + ETA * 2 * smax + _ulp(log_s) + _ulp(lse)


def lse_depth(grp):
    """(items per CTA, grid) of the log-sum-exp kernels on group `grp` with NUM_SMS CTAs"""
    from parallax_b200 import consts
    lay = grp.layout
    owners = 1 if lay.replicated else lay.world
    nblk = -(-lay.parts_per_owner * lay.rows_per_part // 128)
    items = owners * nblk
    grid = min(items, consts.NUM_SMS)
    return -(-items // grid), grid


def draw_margin(key, log_e):
    """bound on |fp32 key − exact key| for exact s, keys `key` and log E `log_e` (fp64 tensors)"""
    return 0.5 * _ulp(key) + _ulp(log_e) + 4 * U * 1.01 + U


def grad_bound(p, g, smax, lse):
    """bound on |g·(p32 − [v = t]) − g·(p − [v = t])| per element, the fp32 value of G before
    its bf16 rounding, where p = exp(s − lse) in fp64 with the lse the kernel is given [N] and
    smax = max |s| [N]: exp2f (4u), the rounded −lse·L2E and fma argument, the fp32 L2E over
    |s − lse| ≤ max|s| + |lse|, then p − 1 and g·(·) (2u)."""
    lse, smax, g = lse[:, None], smax[:, None], g.abs()[:, None]
    t = 4 * U + U * (lse.abs() + 2 * (smax + lse.abs())) + ETA * (smax + lse.abs())
    return g * (p * (t + 2 * U) + 2 * U)


def bf16_half_ulp(x):
    x = x.abs().double().clamp_min(2.0 ** -126)
    return torch.pow(2.0, torch.floor(torch.log2(x)) - 8)


# ------------------------------------------------------------------ reference
def logits64(x, W, b):
    return x.double() @ W.double().t() + b.double().t()


def truncation_theta(vals, n, top_k=None, top_p=None):
    """θ* over rows of values sorted descending `vals` [R, V] (fp64): the largest θ with
    count(θ) >= top_k or (mass(θ) >= top_p and count(θ) >= n), ties counted together.
    Returns (θ* [R], cum mass at θ* [R], cum mass at the next value above θ* [R], count [R])."""
    R, V = vals.shape
    q = torch.softmax(vals, 1)
    mass = torch.cumsum(q, 1)
    neg = (-vals).contiguous()
    end = torch.searchsorted(neg, neg, right=True) - 1     # last position of each run
    cnt, m = end + 1, mass.gather(1, end)
    ok = torch.zeros_like(cnt, dtype=torch.bool)
    if top_k is not None:
        ok |= cnt >= top_k
    if top_p is not None:
        ok |= (m >= top_p) & (cnt >= n)
    j = torch.where(ok.any(1), ok.int().argmax(1), torch.full_like(ok[:, 0], V - 1, dtype=torch.long))
    th = vals.gather(1, j[:, None])[:, 0]
    start = torch.searchsorted(neg, neg, right=False).gather(1, j[:, None])[:, 0]
    above = torch.where(start > 0, mass.gather(1, (start - 1).clamp_min(0)[:, None])[:, 0],
                        torch.zeros_like(th))
    return th, m.gather(1, j[:, None])[:, 0], above, cnt.gather(1, j[:, None])[:, 0]


def _draws(s, keys, nmax):
    kv, ki = torch.sort(keys, dim=1, descending=True, stable=True)
    return kv[:, :nmax], ki[:, :nmax]


def reference(x, W, b, *, ktop=1001, nmax=33, taus=(0.5, 1.0), seed=0, trunc_k=(40, 1000),
              top_p=0.9, rows=128):
    """The fp64 reference of rows x [N, K] against (W [V, K], b [V, 1]), all on one device:
    a dict of per-row tensors on that device (`lse`, `smax`, `top_v`, `top_i`: the `ktop` best
    (s desc, id asc) at τ = 1; per τ in `taus`: `key_<τ>`, `kid_<τ>`, `loge_<τ>` of the `nmax`
    best Gumbel keys, `ks_<τ>` their s, `lse_<τ>` and `smax_<τ>` of s; at τ = 1, `th_<k>` for each top_k, `mkey_<k>` / `mkid_<k>` / `mloge_<k>`
    the draws among s >= θ*(k), and `th_p`, `cum_p`, `above_p` for top_p with n = 1)."""
    from parallax_b200.parallel.engine import sample_log_e
    N, V = x.shape[0], W.shape[0]
    dev = x.device
    Wd, bd = W.double(), b.double().t()
    gids = torch.arange(V, device=dev)
    out = {}

    def put(name, t, r0):
        if name not in out:
            out[name] = torch.empty((N,) + t.shape[1:], dtype=t.dtype, device=dev)
        out[name][r0:r0 + t.shape[0]] = t

    for r0 in range(0, N, rows):
        xs = x[r0:r0 + rows].double()
        s = xs @ Wd.t() + bd
        R = s.shape[0]
        put("lse", torch.logsumexp(s, 1), r0)
        put("smax", s.abs().amax(1), r0)
        vals, order = torch.sort(s, dim=1, descending=True, stable=True)
        put("top_v", vals[:, :ktop], r0)
        put("top_i", order[:, :ktop], r0)
        for k in trunc_k:
            th = vals[:, k - 1]
            put("th_%d" % k, th, r0)
        th_p, cum_p, above_p, _ = truncation_theta(vals, 1, top_p=top_p)
        put("th_p", th_p, r0)
        put("cum_p", cum_p, r0)
        put("above_p", above_p, r0)
        del vals, order
        for tau in taus:
            st = s * inv_tau(tau)
            loge = sample_log_e(seed, torch.arange(r0, r0 + R, device=dev), gids).double()
            keys = st - loge
            kv, ki = _draws(st, keys, nmax)
            put("key_%g" % tau, kv, r0)
            put("kid_%g" % tau, ki, r0)
            put("loge_%g" % tau, loge.gather(1, ki), r0)
            put("ks_%g" % tau, st.gather(1, ki), r0)
            put("lse_%g" % tau, torch.logsumexp(st, 1), r0)
            put("smax_%g" % tau, st.abs().amax(1), r0)
            if tau == 1.0:
                for k in trunc_k[:1]:
                    th = out["th_%d" % k][r0:r0 + R]
                    mk = keys.masked_fill(s < th[:, None], -math.inf)
                    kv, ki = _draws(st, mk, nmax)
                    put("mkey_%d" % k, kv, r0)
                    put("mkid_%d" % k, ki, r0)
                    put("mloge_%d" % k, loge.gather(1, ki), r0)
                    put("mks_%d" % k, st.gather(1, ki), r0)
            del keys, loge, st
        del s
    return out


def checked_draws(ids, key, kid, loge, n):
    """(agree, checked): kernel draws `ids` [N, n] against the reference's keys (fp64 `key`,
    ids `kid`, log E `loge`, fp64 [N, ≥ n + 1], descending): position j is checked where the
    reference key j is apart from keys j − 1 and j + 1 by more than twice the sum of their
    draw margins."""
    key, kid, loge = key[:, :n + 1], kid[:, :n + 1], loge[:, :n + 1]
    fin = torch.isfinite(key)
    mg = torch.where(fin, draw_margin(key.nan_to_num(0, 0, 0), loge), torch.zeros_like(key))
    gap = (key[:, :-1] - key[:, 1:]).nan_to_num(math.inf, math.inf)
    sep = gap > 2 * (mg[:, :-1] + mg[:, 1:])             # key j vs key j + 1
    ok = sep[:, :n].clone()
    ok[:, 1:] &= sep[:, :n - 1]
    agree = ids[ok] == kid[:, :n][ok]
    return bool(agree.all()), ok
