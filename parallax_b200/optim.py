"""Optimizer specifications with TensorFlow-1.x update semantics.

The reference does not implement optimizers; it recognises TF's update ops in
the user graph (`graph_transform_lib.py:56-75`: ApplyGradientDescent,
ApplyMomentum, ApplyAdagrad, ApplyAdam, ApplyRMSProp … and, for sparse
variables, SparseApplyAdagrad / Scatter*) and runs TF's kernels
(`tensorflow/core/kernels/training_ops_gpu.cu.cc:28-283`, CPU sparse
`training_ops.cc:1276-1382`).  Here an optimizer is a *spec* (kind +
hyper-parameters); the math is executed by

* the fused sm_90a kernels (`ops/csrc/kernels/dense_step.cu`,
  `sparse_apply.cu`) on the NVLink fabric, or
* the pure-torch fp32 functions in this file on the host fabric — which are
  also the numerics oracle for the kernel tests.

Update rules (g = aggregated gradient):

* sgd      : w -= lr·g
* momentum : a = μ·a + g ; w -= lr·a            (nesterov: w -= lr·(g + μ·a))
* adagrad  : a += g² ; w -= lr·g / sqrt(a)       (a₀ = initial_accumulator_value)
* adam     : m = β₁m+(1-β₁)g ; v = β₂v+(1-β₂)g² ;
             w -= lr·sqrt(1-β₂ᵗ)/(1-β₁ᵗ) · m/(sqrt(v)+ε)
* rmsprop  : ms = ρ·ms+(1-ρ)g² ; mom = μ·mom + lr·g/sqrt(ms+ε) ; w -= mom
* rowwise_adagrad (sparse variables only): one accumulator per row,
             s += mean_j(g_j²) ; w -= lr·g / (sqrt(s) + ε)
* lars     (dense only, layer-wise): trust = η‖w‖/(‖g‖ + λ‖w‖ + ε) per tensor ;
             mom = μ·mom + g ; w -= lr·trust·mom
* lamb     (dense only, layer-wise): m, v as Adam ; r = m̂/(sqrt(v̂)+ε) + λw ;
             w -= lr·(‖w‖/‖r‖)·r, the norms over the whole tensor

Sparse variants touch only the rows present in the aggregated gradient
("lazy" Adam/momentum, exactly like TF's sparse apply ops).
"""
import math

import torch

# Every kind has a fused sm_90a rule (`ops/csrc/kernels/optim_rules.cuh`), split in two
# template families so the five hot rules keep their register budget: KINDS (family 0)
# and EXT_KINDS (family 1: the rest of the reference's recognised update ops,
# `graph_transform_lib.py:56-75` — ApplyAdadelta, ApplyFtrl, ApplyProximalGradientDescent,
# ApplyProximalAdagrad, ApplyAdagradDA, ApplyCenteredRMSProp; up to three slots).
KINDS = ("sgd", "momentum", "adagrad", "adam", "rmsprop")
EXT_KINDS = ("adadelta", "ftrl", "proximal_sgd", "proximal_adagrad", "adagrad_da",
             "centered_rmsprop")
HOST_KINDS = EXT_KINDS            # historical name
# family 2: rules that keep one fp32 slot value per table ROW (sparse variables only; the
# sparse owner kernel merges a whole row before it applies it)
ROWWISE_KINDS = ("rowwise_adagrad",)
# family 3: layer-wise rules, whose step is scaled by a trust ratio of norms over each whole
# dense tensor (dense variables only; `dense_step.cu` runs them as a norm pass, an all-reduce
# of the per-tensor sums and an update pass)
LAYERWISE_KINDS = ("lars", "lamb")
KIND_ID = {k: i for i, k in enumerate(KINDS + EXT_KINDS + ROWWISE_KINDS + LAYERWISE_KINDS)}
# number of fp32 state slots per kind
NUM_SLOTS = {"sgd": 0, "momentum": 1, "adagrad": 1, "adam": 2, "rmsprop": 2,
             "adadelta": 2, "ftrl": 2, "proximal_sgd": 0, "proximal_adagrad": 1,
             "adagrad_da": 2, "centered_rmsprop": 3, "rowwise_adagrad": 1,
             "lars": 1, "lamb": 2}
SLOT_NAMES = {
    "sgd": (), "momentum": ("momentum",), "adagrad": ("accumulator",),
    "adam": ("m", "v"), "rmsprop": ("ms", "mom"),
    "adadelta": ("accum", "accum_update"), "ftrl": ("accum", "linear"), "proximal_sgd": (),
    "proximal_adagrad": ("accumulator",),
    "adagrad_da": ("gradient_accumulator", "gradient_squared_accumulator"),
    "centered_rmsprop": ("ms", "mg", "mom"), "rowwise_adagrad": ("accumulator",),
    "lars": ("momentum",), "lamb": ("m", "v"),
}


def kind_family(kind):
    """Kernel template family of `kind` (`optim_rules.cuh`): 0, 1, 2 (row-wise) or 3
    (layer-wise)."""
    if kind in LAYERWISE_KINDS:
        return 3
    return 0 if kind in KINDS else 1 if kind in EXT_KINDS else 2


def slot_width(kind, D):
    """Columns of each state slot of a [V, D] variable: 1 for row-wise rules, else D."""
    return 1 if kind in ROWWISE_KINDS else D


def table_row_bytes(kind, D, weight_dtype=torch.float32):
    """Bytes one row of a sparse variable of width D takes on its owner: the master row and
    the fp32 slots, every D-wide row padded to a multiple of 4 columns.  A bf16 master row
    (``sess_config["sparse_weights"] = "bf16"``) is padded to a multiple of 8 columns."""
    Dp = (D + 3) // 4 * 4
    w = 4 * Dp if weight_dtype == torch.float32 else 2 * ((Dp // 4 + 1) // 2 * 8)
    return w + 4 * NUM_SLOTS[kind] * slot_width(kind, Dp)


# ---------------------------------------------------------------------------
# bf16 master rows: stochastic rounding (`ops/csrc/kernels/sparse.cu` holds the same hash and
# rounding; the two agree bit for bit)
# ---------------------------------------------------------------------------
SPARSE_WEIGHTS = {"fp32": torch.float32, "bf16": torch.bfloat16}
_M32 = 0xffffffff


def sparse_weight_dtype(value):
    """torch dtype of ``sess_config["sparse_weights"]``: "fp32" (default) or "bf16"."""
    if value not in SPARSE_WEIGHTS:
        raise ValueError("sess_config['sparse_weights'] must be 'fp32' or 'bf16', not %r"
                         % (value,))
    return SPARSE_WEIGHTS[value]


def sr_seed(name):
    """The stochastic-rounding seed of sparse variable `name` (a 32-bit constant)."""
    import zlib
    return zlib.crc32(name.encode("utf-8")) & _M32


def _mul32(x, c):
    """(x · c) mod 2^32 for x in [0, 2^32) (int64 tensors or ints) without int64 overflow."""
    return ((x & 0xffff) * c + ((((x >> 16) * (c & 0xffff)) & 0xffff) << 16)) & _M32


def sr_mix(x):
    """32-bit integer hash (a 32-bit finaliser: xor-shift, multiply, twice)."""
    x = x ^ (x >> 16)
    x = _mul32(x, 0x7feb352d)
    x = x ^ (x >> 15)
    x = _mul32(x, 0x846ca68b)
    return x ^ (x >> 16)


def round_bf16_stochastic(x, seed, step, gids):
    """bf16 [n, D] of fp32 rows `x` [n, D] of global ids `gids` [n], rounded stochastically at
    global step `step`: element (i, j) takes the top 16 bits of ``bits(x) + r`` with
    ``r = sr_mix(sr_mix(sr_mix(seed ^ step) ^ gid) ^ j) >> 16``, so it rounds away from zero
    with probability equal to its fraction of a bf16 ulp.  Inf and NaN pass through."""
    x = x.to(torch.float32).contiguous()
    n, D = x.shape
    u = x.view(torch.int32).to(torch.int64) & _M32
    key = sr_mix(sr_mix(int(seed) ^ int(step)) ^ (gids.to(x.device, torch.int64) & _M32))
    r = sr_mix(key[:, None] ^ torch.arange(D, dtype=torch.int64, device=x.device)[None, :]) >> 16
    finite = (u & 0x7f800000) != 0x7f800000
    special = (u >> 16) | torch.where((u & 0x7fffff) != 0, 0x40, 0)
    b = torch.where(finite, (u + r) >> 16, special) & 0xffff
    return ((b ^ 0x8000) - 0x8000).to(torch.int16).view(torch.bfloat16)


def check_table_slots(name, kind, V, D, slots):
    """Raise ValueError unless every tensor of `slots` has the logical shape of a slot of
    sparse variable `name` ([V, D], trained with `kind`): [V, D], or [V, 1] for a row-wise
    rule — so that a checkpoint of another optimizer cannot be broadcast into the slots."""
    want = (V, slot_width(kind, D))
    for i, s in enumerate(slots):
        if tuple(s.shape) != want:
            raise ValueError("sparse variable %r: slot %d has shape %s, but its %s optimizer "
                             "keeps slots of shape %s" % (name, i, tuple(s.shape), kind, want))


def require_fused(kind, where):
    if kind not in KIND_ID:
        raise NotImplementedError(
            "optimizer kind %r has no fused kernel (%s).  Fused kinds: %s"
            % (kind, where, ", ".join(KIND_ID)))

# layout of the device-side hyper-parameter vector read by the kernels; HP_BC1 / HP_BC2 are
# LAMB's bias corrections 1/(1-β1ᵗ) and 1/(1-β2ᵗ), folded on the host in double
HP_LR, HP_A, HP_B, HP_EPS, HP_WD, HP_STEP, HP_GSCALE, HP_FLAGS, HP_BC1, HP_BC2 = range(10)
HP_SIZE = 10
# bits of hp[HP_FLAGS] for the layer-wise rules (the same bits as their per-tensor flags in
# the dense step's segment map): nesterov (LARS), weight decay applies (LAMB), trust ratio
# applies (both)
LW_NESTEROV, LW_DECAY, LW_ADAPT = 1, 2, 4


class Optimizer(object):
    kind = None

    def __init__(self, learning_rate, weight_decay=0.0, name=None):
        # weight_decay: L2 term added to the gradient of DENSE variables (g + wd·w)
        self.learning_rate = learning_rate
        self.weight_decay = float(weight_decay)
        self.name = name or type(self).__name__

    # -- hyper-parameters ----------------------------------------------------
    def lr_at(self, step):
        lr = self.learning_rate
        return float(lr(step)) if callable(lr) else float(lr)

    def slot_init(self):
        """Initial value of each state slot."""
        return tuple(0.0 for _ in range(NUM_SLOTS[self.kind]))

    def hyper(self, step):
        """Vector [lr, a, b, eps, wd, step, gscale, flags, bc1, bc2] for step `step`
        (1-based count of the update being applied)."""
        hp = [0.0] * HP_SIZE
        hp[HP_LR] = self.lr_at(step)
        hp[HP_WD] = self.weight_decay
        hp[HP_STEP] = float(step)
        hp[HP_GSCALE] = 1.0
        self._fill(hp, step)
        return hp

    def _fill(self, hp, step):
        pass

    def hyper_for(self, name, step):
        """`hyper(step)` for the dense parameter `name`: a layer-wise rule clears the
        weight-decay and trust-ratio bits of hp[HP_FLAGS] that its exclude lists remove
        (`layer_flags`); every other rule has no per-name setting."""
        return self.hyper(step)

    def describe(self):
        d = {k: v for k, v in vars(self).items() if not callable(v)}
        d["kind"] = self.kind
        return d


class GradientDescent(Optimizer):
    kind = "sgd"


class Momentum(Optimizer):
    kind = "momentum"

    def __init__(self, learning_rate, momentum=0.9, use_nesterov=False, **kw):
        super().__init__(learning_rate, **kw)
        self.momentum = float(momentum)
        self.use_nesterov = bool(use_nesterov)

    def _fill(self, hp, step):
        hp[HP_A] = self.momentum
        hp[HP_FLAGS] = 1.0 if self.use_nesterov else 0.0


class Adagrad(Optimizer):
    kind = "adagrad"

    def __init__(self, learning_rate, initial_accumulator_value=0.1, **kw):
        super().__init__(learning_rate, **kw)
        self.initial_accumulator_value = float(initial_accumulator_value)

    def slot_init(self):
        return (self.initial_accumulator_value,)


class Adam(Optimizer):
    kind = "adam"

    def __init__(self, learning_rate=0.001, beta1=0.9, beta2=0.999,
                 epsilon=1e-8, **kw):
        super().__init__(learning_rate, **kw)
        self.beta1, self.beta2, self.epsilon = \
            float(beta1), float(beta2), float(epsilon)

    def _fill(self, hp, step):
        hp[HP_A], hp[HP_B], hp[HP_EPS] = self.beta1, self.beta2, self.epsilon
        # bias-corrected step size, folded on the host (TF does the same in
        # `_prepare`/`_finish`)
        t = max(int(step), 1)
        hp[HP_LR] = self.lr_at(step) * math.sqrt(1.0 - self.beta2 ** t) / \
            (1.0 - self.beta1 ** t)


class RMSProp(Optimizer):
    kind = "rmsprop"

    def __init__(self, learning_rate, decay=0.9, momentum=0.0,
                 epsilon=1e-10, **kw):
        super().__init__(learning_rate, **kw)
        self.decay, self.momentum, self.epsilon = \
            float(decay), float(momentum), float(epsilon)

    def _fill(self, hp, step):
        hp[HP_A], hp[HP_B], hp[HP_EPS] = self.decay, self.momentum, self.epsilon


class Adadelta(Optimizer):
    """`tf.train.AdadeltaOptimizer` (ApplyAdadelta)"""
    kind = "adadelta"

    def __init__(self, learning_rate=0.001, rho=0.95, epsilon=1e-8, **kw):
        super().__init__(learning_rate, **kw)
        self.rho, self.epsilon = float(rho), float(epsilon)

    def _fill(self, hp, step):
        hp[HP_A], hp[HP_EPS] = self.rho, self.epsilon


class Ftrl(Optimizer):
    """`tf.train.FtrlOptimizer` (ApplyFtrl): FTRL-proximal with L1/L2"""
    kind = "ftrl"

    def __init__(self, learning_rate, learning_rate_power=-0.5, initial_accumulator_value=0.1,
                 l1_regularization_strength=0.0, l2_regularization_strength=0.0, **kw):
        super().__init__(learning_rate, **kw)
        if learning_rate_power > 0:
            raise ValueError("learning_rate_power must be <= 0")
        self.learning_rate_power = float(learning_rate_power)
        self.initial_accumulator_value = float(initial_accumulator_value)
        self.l1, self.l2 = float(l1_regularization_strength), float(l2_regularization_strength)

    def slot_init(self):
        return (self.initial_accumulator_value, 0.0)

    def _fill(self, hp, step):
        hp[HP_A], hp[HP_B], hp[HP_EPS] = self.learning_rate_power, self.l1, self.l2


class ProximalGradientDescent(Optimizer):
    """`tf.train.ProximalGradientDescentOptimizer` (ApplyProximalGradientDescent)"""
    kind = "proximal_sgd"

    def __init__(self, learning_rate, l1_regularization_strength=0.0,
                 l2_regularization_strength=0.0, **kw):
        super().__init__(learning_rate, **kw)
        self.l1, self.l2 = float(l1_regularization_strength), float(l2_regularization_strength)

    def _fill(self, hp, step):
        hp[HP_A], hp[HP_B] = self.l1, self.l2


class ProximalAdagrad(ProximalGradientDescent):
    """`tf.train.ProximalAdagradOptimizer` (ApplyProximalAdagrad)"""
    kind = "proximal_adagrad"

    def __init__(self, learning_rate, initial_accumulator_value=0.1, **kw):
        super().__init__(learning_rate, **kw)
        self.initial_accumulator_value = float(initial_accumulator_value)

    def slot_init(self):
        return (self.initial_accumulator_value,)


class AdagradDA(ProximalGradientDescent):
    """`tf.train.AdagradDAOptimizer` (ApplyAdagradDA): dual averaging, needs the step"""
    kind = "adagrad_da"

    def __init__(self, learning_rate, initial_gradient_squared_accumulator_value=0.1, **kw):
        super().__init__(learning_rate, **kw)
        self.initial_gradient_squared_accumulator_value = \
            float(initial_gradient_squared_accumulator_value)

    def slot_init(self):
        return (0.0, self.initial_gradient_squared_accumulator_value)


class CenteredRMSProp(RMSProp):
    """`tf.train.RMSPropOptimizer(centered=True)` (ApplyCenteredRMSProp)"""
    kind = "centered_rmsprop"


class RowWiseAdagrad(Optimizer):
    """Row-wise Adagrad for embedding tables (FBGEMM's ``EXACT_ROWWISE_ADAGRAD``): one fp32
    accumulator per row instead of one per element.  For a row with aggregated gradient g
    of the table's D columns::

        s   += (1/D) · Σ_j g_j²
        w_j -= lr · g_j / (sqrt(s) + epsilon)

    Lazy like every sparse rule: rows without a gradient this step, and their accumulators,
    are untouched.  With D = 1 it is Adagrad.  A *sparse-variable* optimizer: pass it as
    ``Graph(..., sparse_optimizer=RowWiseAdagrad(...))``; the engine refuses it for dense
    variables and with ``sync=False``."""
    kind = "rowwise_adagrad"

    def __init__(self, learning_rate, initial_accumulator_value=0.1, epsilon=0.0, **kw):
        super().__init__(learning_rate, **kw)
        self.initial_accumulator_value = float(initial_accumulator_value)
        self.epsilon = float(epsilon)

    def slot_init(self):
        return (self.initial_accumulator_value,)

    def _fill(self, hp, step):
        hp[HP_EPS] = self.epsilon


class Lars(Optimizer):
    """`tf.contrib.opt.LARSOptimizer`: momentum with a layer-wise learning rate (You et al.,
    2017).  For each dense parameter tensor, with g its gradient (after averaging,
    `ScaleGradients` and clipping) and w its fp32 master before the update::

        trust = eeta·‖w‖ / (‖g‖ + weight_decay·‖w‖ + epsilon)   if ‖w‖ > 0 and ‖g‖ > 0, else 1
        mom   = momentum·mom + g
        w    -= learning_rate·trust·mom       (nesterov: learning_rate·trust·(g + momentum·mom))

    The norms are over the whole tensor.  `weight_decay` enters only the trust ratio, as in
    the reference: no λw term is added to the gradient.  A parameter whose name contains an
    entry of `skip_list` as a substring takes trust = 1.  A *dense-variable* optimizer, for
    sync training only; the engine refuses it for sparse variables."""
    kind = "lars"

    def __init__(self, learning_rate, momentum=0.9, weight_decay=1e-4, eeta=0.001,
                 epsilon=0.0, skip_list=None, use_nesterov=False, name=None):
        super().__init__(learning_rate, weight_decay=weight_decay, name=name)
        self.momentum, self.eeta, self.epsilon = float(momentum), float(eeta), float(epsilon)
        self.skip_list = list(skip_list) if skip_list is not None else None
        self.use_nesterov = bool(use_nesterov)

    def _fill(self, hp, step):
        hp[HP_A], hp[HP_B], hp[HP_EPS] = self.momentum, self.eeta, self.epsilon
        hp[HP_FLAGS] = float((LW_NESTEROV if self.use_nesterov else 0) | LW_ADAPT)

    def layer_flags(self, name):
        """The per-tensor flags of `name`: LW_NESTEROV with `use_nesterov`, and LW_ADAPT
        unless an entry of `skip_list` is a substring of `name`.  The dense step reads every
        flag of the rule from these (its segment map), not from hp[HP_FLAGS]."""
        skip = self.skip_list is not None and any(s in name for s in self.skip_list)
        return (LW_NESTEROV if self.use_nesterov else 0) | (0 if skip else LW_ADAPT)

    def hyper_for(self, name, step):
        hp = self.hyper(step)
        hp[HP_FLAGS] = float(self.layer_flags(name))
        return hp


class Lamb(Optimizer):
    """LAMB (You et al., 2019; `tfa.optimizers.LAMB`): Adam moments with a layer-wise trust
    ratio.  For each dense parameter tensor::

        m = β1·m + (1−β1)·g ;  v = β2·v + (1−β2)·g²
        r = (m/(1−β1ᵗ)) / (sqrt(v/(1−β2ᵗ)) + epsilon)  [+ weight_decay·w]
        trust = ‖w‖/‖r‖  if ‖w‖ > 0 and ‖r‖ > 0, else 1
        w -= learning_rate·trust·r

    Weight decay is decoupled (added to r, not to g).  `exclude_from_weight_decay` and
    `exclude_from_layer_adaptation` are lists of regexes, matched with `re.search` against
    the dotted parameter name, that turn off the decay term and the trust ratio (trust = 1)
    of the parameters they match; `exclude_from_layer_adaptation=None` means "the same as
    `exclude_from_weight_decay`".  A *dense-variable* optimizer, for sync training only."""
    kind = "lamb"

    def __init__(self, learning_rate=0.001, beta1=0.9, beta2=0.999, epsilon=1e-6,
                 weight_decay=0.0, exclude_from_weight_decay=None,
                 exclude_from_layer_adaptation=None, name=None):
        super().__init__(learning_rate, weight_decay=weight_decay, name=name)
        self.beta1, self.beta2, self.epsilon = float(beta1), float(beta2), float(epsilon)
        self.exclude_from_weight_decay = list(exclude_from_weight_decay or [])
        self.exclude_from_layer_adaptation = list(
            exclude_from_layer_adaptation if exclude_from_layer_adaptation is not None
            else self.exclude_from_weight_decay)

    def _fill(self, hp, step):
        hp[HP_A], hp[HP_B], hp[HP_EPS] = self.beta1, self.beta2, self.epsilon
        t = max(int(step), 1)
        hp[HP_BC1] = 1.0 / (1.0 - self.beta1 ** t)
        hp[HP_BC2] = 1.0 / (1.0 - self.beta2 ** t)
        hp[HP_FLAGS] = float(LW_DECAY | LW_ADAPT)

    def layer_flags(self, name):
        """LW_DECAY and LW_ADAPT, each unless one of its exclude patterns matches `name`."""
        import re
        f = 0
        if self.weight_decay != 0.0 and \
                not any(re.search(p, name) for p in self.exclude_from_weight_decay):
            f |= LW_DECAY
        if not any(re.search(p, name) for p in self.exclude_from_layer_adaptation):
            f |= LW_ADAPT
        return f

    def hyper_for(self, name, step):
        hp = self.hyper(step)
        hp[HP_FLAGS] = float(self.layer_flags(name))
        return hp


# TF-style aliases
LARSOptimizer = Lars
AdadeltaOptimizer = Adadelta
FtrlOptimizer = Ftrl
ProximalGradientDescentOptimizer = ProximalGradientDescent
ProximalAdagradOptimizer = ProximalAdagrad
AdagradDAOptimizer = AdagradDA
GradientDescentOptimizer = GradientDescent
MomentumOptimizer = Momentum
AdagradOptimizer = Adagrad
AdamOptimizer = Adam
RMSPropOptimizer = RMSProp


# ---------------------------------------------------------------------------
# fp32 torch reference math (host fabric + test oracle)
# ---------------------------------------------------------------------------
def lamb_direction(g, w, m, v, hp):
    """LAMB's (new m, new v, r) for gradient g, master w and moments m, v, all fp32; r
    includes the decoupled weight-decay term when hp[HP_FLAGS] has LW_DECAY."""
    a, b, eps = hp[HP_A], hp[HP_B], hp[HP_EPS]
    m = m * a + g * (1.0 - a)
    v = v * b + g * g * (1.0 - b)
    r = (m * hp[HP_BC1]) / ((v * hp[HP_BC2]).sqrt() + eps)
    if int(hp[HP_FLAGS]) & LW_DECAY:
        r = r + hp[HP_WD] * w
    return m, v, r


def trust_ratio(kind, wn, xn, hp):
    """Layer-wise trust ratio from ‖w‖ and ‖x‖ (x = g for LARS, r for LAMB): 1 when the
    rule's LW_ADAPT bit is clear or either norm is 0."""
    if not int(hp[HP_FLAGS]) & LW_ADAPT or not (wn > 0.0 and xn > 0.0):
        return 1.0
    if kind == "lars":
        return hp[HP_B] * wn / (xn + hp[HP_WD] * wn + hp[HP_EPS])
    return wn / xn


def apply_dense_(kind, w, g, slots, hp):
    """In-place update of fp32 tensor `w` with gradient `g` (already
    aggregated); `slots` is a tuple of fp32 state tensors shaped like `w`.  A layer-wise rule
    (`LAYERWISE_KINDS`) treats `w` as one whole tensor: its norms are taken over all of it,
    and its per-tensor flags come from hp[HP_FLAGS] (`Optimizer.hyper_for`)."""
    lr, a, b, eps, wd = hp[HP_LR], hp[HP_A], hp[HP_B], hp[HP_EPS], hp[HP_WD]
    g = g.to(torch.float32) * hp[HP_GSCALE]
    if kind in LAYERWISE_KINDS:           # weight decay is the rule's own term
        return _apply_layerwise_(kind, w, g, slots, hp)
    if wd != 0.0:
        g = g + wd * w
    if kind == "sgd":
        w.add_(g, alpha=-lr)
    elif kind == "momentum":
        (acc,) = slots
        acc.mul_(a).add_(g)
        if hp[HP_FLAGS] >= 0.5:
            w.add_(g + a * acc, alpha=-lr)
        else:
            w.add_(acc, alpha=-lr)
    elif kind == "adagrad":
        (acc,) = slots
        acc.addcmul_(g, g)
        w.addcdiv_(g, acc.sqrt(), value=-lr)
    elif kind == "adam":
        m, v = slots
        m.mul_(a).add_(g, alpha=1.0 - a)
        v.mul_(b).addcmul_(g, g, value=1.0 - b)
        w.addcdiv_(m, v.sqrt().add_(eps), value=-lr)
    elif kind == "rmsprop":
        ms, mom = slots
        ms.mul_(a).addcmul_(g, g, value=1.0 - a)
        mom.mul_(b).add_(g / (ms + eps).sqrt(), alpha=lr)
        w.sub_(mom)
    elif kind == "centered_rmsprop":
        ms, mg, mom = slots
        ms.mul_(a).addcmul_(g, g, value=1.0 - a)
        mg.mul_(a).add_(g, alpha=1.0 - a)
        mom.mul_(b).add_(g / (ms - mg * mg + eps).sqrt(), alpha=lr)
        w.sub_(mom)
    elif kind == "adadelta":
        accum, accum_update = slots
        accum.mul_(a).addcmul_(g, g, value=1.0 - a)
        update = (accum_update + eps).sqrt() / (accum + eps).sqrt() * g
        accum_update.mul_(a).addcmul_(update, update, value=1.0 - a)
        w.add_(update, alpha=-lr)
    elif kind == "ftrl":                  # a = lr_power (<= 0), b = l1, eps = l2
        accum, linear = slots
        new_accum = accum + g * g
        p_new, p_old = new_accum.pow(-a), accum.pow(-a)
        linear.add_(g - (p_new - p_old) / lr * w)
        quadratic = p_new / lr + 2.0 * eps
        w.copy_(torch.where(linear.abs() > b,
                            (torch.sign(linear) * b - linear) / quadratic,
                            torch.zeros_like(w)))
        accum.copy_(new_accum)
    elif kind in ("proximal_sgd", "proximal_adagrad"):       # a = l1, b = l2
        if kind == "proximal_adagrad":
            (accum,) = slots
            accum.addcmul_(g, g)
            lr_t = lr / accum.sqrt()
        else:
            lr_t = torch.full_like(w, lr)
        prox = w - lr_t * g
        w.copy_(torch.sign(prox) * (prox.abs() - lr_t * a).clamp(min=0.0) / (1.0 + lr_t * b))
    elif kind == "adagrad_da":            # a = l1, b = l2, hp[HP_STEP] = global step
        g_acc, gg_acc = slots
        t = float(hp[HP_STEP])
        g_acc.add_(g)
        gg_acc.addcmul_(g, g)
        tmp = torch.sign(g_acc) * (g_acc.abs() - a * t).clamp(min=0.0) if a > 0 else g_acc
        w.copy_(-lr * tmp / (b * t * lr + gg_acc.sqrt()))
    elif kind == "rowwise_adagrad":       # rows of w (dim 0); acc is [rows, 1]
        (acc,) = slots
        acc.add_((g * g).mean(dim=-1, keepdim=True))
        w.addcdiv_(g, acc.sqrt().add_(eps), value=-lr)
    else:  # pragma: no cover
        raise ValueError(kind)
    return w


def _apply_layerwise_(kind, w, g, slots, hp):
    lr = hp[HP_LR]
    wn = float(w.double().norm())
    if kind == "lars":
        (mom,) = slots
        trust = trust_ratio(kind, wn, float(g.double().norm()), hp)
        mom.mul_(hp[HP_A]).add_(g)
        if int(hp[HP_FLAGS]) & LW_NESTEROV:
            w.add_(g + hp[HP_A] * mom, alpha=-lr * trust)
        else:
            w.add_(mom, alpha=-lr * trust)
    else:
        m, v = slots
        m_new, v_new, r = lamb_direction(g, w, m, v, hp)
        trust = trust_ratio(kind, wn, float(r.double().norm()), hp)
        m.copy_(m_new)
        v.copy_(v_new)
        w.add_(r, alpha=-lr * trust)
    return w


def apply_sparse_rows_(kind, w, rows, g, slots, hp, seed=None, gids=None):
    """Row-sparse update: `rows` (int64, unique) index dim 0 of `w`/`slots`;
    `g` is [len(rows), D] — the *summed* gradient of each row.  `weight_decay` is a
    dense-variable setting: sparse rows are not decayed (TF's SparseApply* ops have no
    L2 term either, and the fused `sparse_update4` kernel takes none).  A bf16 `w` is
    widened, updated in fp32 and stored with `round_bf16_stochastic` (the table's `seed`,
    hp[HP_STEP] and the rows' global ids `gids`)."""
    if rows.numel() == 0:
        return w
    if hp[HP_WD] != 0.0:
        hp = list(hp)
        hp[HP_WD] = 0.0
    w_r = w.index_select(0, rows).to(torch.float32)
    s_r = tuple(s.index_select(0, rows) for s in slots)
    apply_dense_(kind, w_r, g, s_r, hp)
    if w.dtype == torch.bfloat16:
        w_r = round_bf16_stochastic(w_r, seed, int(hp[HP_STEP]), gids)
    w.index_copy_(0, rows, w_r)
    for s, sr in zip(slots, s_r):
        s.index_copy_(0, rows, sr)
    return w


# ---------------------------------------------------------------------------
# learning-rate schedules (`tf.train.*_decay`) — callables for `learning_rate=`
# ---------------------------------------------------------------------------
class schedules(object):
    """Every function returns ``lr(step)``; `step` is the 1-based index of the update
    being applied, and — like TF, which evaluates a schedule with the number of
    *completed* steps — the formulas use ``global_step = step − 1``."""

    @staticmethod
    def _gs(step):
        return max(int(step) - 1, 0)

    @staticmethod
    def exponential_decay(learning_rate, decay_steps, decay_rate, staircase=False):
        def lr(step):
            p = schedules._gs(step) / float(decay_steps)
            return learning_rate * decay_rate ** (math.floor(p) if staircase else p)
        return lr

    @staticmethod
    def natural_exp_decay(learning_rate, decay_steps, decay_rate, staircase=False):
        def lr(step):
            p = schedules._gs(step) / float(decay_steps)
            return learning_rate * math.exp(-decay_rate * (math.floor(p) if staircase else p))
        return lr

    @staticmethod
    def inverse_time_decay(learning_rate, decay_steps, decay_rate, staircase=False):
        def lr(step):
            p = schedules._gs(step) / float(decay_steps)
            return learning_rate / (1.0 + decay_rate * (math.floor(p) if staircase else p))
        return lr

    @staticmethod
    def piecewise_constant(boundaries, values):
        """values[i] while global_step ≤ boundaries[i]; values[-1] afterwards"""
        if len(values) != len(boundaries) + 1:
            raise ValueError("The length of boundaries should be 1 less than the length of values")

        def lr(step):
            gs = schedules._gs(step)
            for b, v in zip(boundaries, values):
                if gs <= b:
                    return v
            return values[-1]
        return lr

    @staticmethod
    def polynomial_decay(learning_rate, decay_steps, end_learning_rate=0.0001, power=1.0,
                         cycle=False):
        def lr(step):
            gs, ds = schedules._gs(step), float(decay_steps)
            if cycle:
                ds *= max(1.0, math.ceil(gs / ds))
            else:
                gs = min(gs, decay_steps)
            return (learning_rate - end_learning_rate) * (1.0 - gs / ds) ** power + \
                end_learning_rate
        return lr

    @staticmethod
    def cosine_decay(learning_rate, decay_steps, alpha=0.0):
        def lr(step):
            gs = min(schedules._gs(step), decay_steps)
            cos = 0.5 * (1.0 + math.cos(math.pi * gs / float(decay_steps)))
            return learning_rate * ((1.0 - alpha) * cos + alpha)
        return lr

    @staticmethod
    def warmup(schedule, warmup_steps, start_factor=0.0):
        """linear ramp from start_factor·lr to the schedule's value over `warmup_steps`"""
        base = schedule if callable(schedule) else (lambda step: schedule)

        def lr(step):
            gs = schedules._gs(step)
            v = base(step)
            if gs >= warmup_steps:
                return v
            return v * (start_factor + (1.0 - start_factor) * gs / float(warmup_steps))
        return lr
