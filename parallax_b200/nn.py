"""User-facing modules for declaring sparse (row-indexed) variables.

In the reference a variable is *sparse* when its gradient is an
`IndexedSlices` (produced by `tf.gather`/`embedding_lookup`), recorded through
the `GRADIENTS_INFO` collection (`tensorflow/python/ops/gradients_impl.py:943-947`,
`common/runner.py:40-60`), and it is *partitioned* when created under a
`parallax.get_partitioner(...)` variable scope (`examples/lm1b/language_model.py:34-45`).
The torch analogue: an `nn.Embedding` with ``sparse=True`` produces row-sparse
gradients; `parallax.nn.Embedding` is that module plus an optional
partitioner and an optional *lazy* initialiser so a 100M-row table is never
materialised on the host.
"""
import math

import torch
import torch.nn as tnn


class Embedding(tnn.Embedding):
    """``nn.Embedding(sparse=True)`` + partitioner + lazy init.

    Args:
      partitioner: result of `parallax.get_partitioner(min_p)` (optional).
      lazy: if True the weight lives on the ``meta`` device; each owner
        initialises only its shard (uniform in ``[-init_scale, init_scale]``).
      init_scale: default ``sqrt(3/embedding_dim)`` — TF's
        `uniform_unit_scaling_initializer` used by LM1B.
    """

    def __init__(self, num_embeddings, embedding_dim, partitioner=None,
                 lazy=False, init_scale=None, seed=1234, **kw):
        kw["sparse"] = True
        if lazy:
            kw["device"] = "meta"
        super().__init__(num_embeddings, embedding_dim, **kw)
        self.partitioner = partitioner
        self.lazy = bool(lazy)
        self.init_scale = float(init_scale) if init_scale is not None \
            else math.sqrt(3.0 / embedding_dim)
        self.init_seed = int(seed)
        if not lazy:
            with torch.no_grad():
                self.weight.uniform_(-self.init_scale, self.init_scale)


class EmbeddingBag(tnn.Module):
    """``nn.EmbeddingBag`` semantics (sum / mean / max over bags of ids, optional
    per-sample weights) on top of a sparse `Embedding`, so the table is an ordinary
    sparse variable: partitionable, looked up over the fabric, updated by its row
    owners.  Accepts 2-D input (fixed-size bags) or 1-D input + `offsets`."""

    def __init__(self, num_embeddings, embedding_dim, mode="sum", partitioner=None,
                 lazy=False, init_scale=None, seed=1234, include_last_offset=False,
                 padding_idx=None):
        super().__init__()
        if mode not in ("sum", "mean", "max"):
            raise ValueError("mode must be sum, mean or max")
        self.mode, self.include_last_offset, self.padding_idx = mode, include_last_offset, \
            padding_idx
        self.table = Embedding(num_embeddings, embedding_dim, partitioner=partitioner, lazy=lazy,
                               init_scale=init_scale, seed=seed)

    @property
    def weight(self):
        return self.table.weight

    def forward(self, input, offsets=None, per_sample_weights=None):
        if per_sample_weights is not None and self.mode != "sum":
            raise NotImplementedError("per_sample_weights needs mode='sum'")
        if input.dim() == 2:
            if offsets is not None:
                raise ValueError("offsets must be None for 2-D input")
            B, L = input.shape
            flat = input.reshape(-1)
            bag = torch.arange(B, device=input.device).repeat_interleave(L)
            psw = per_sample_weights.reshape(-1) if per_sample_weights is not None else None
        else:
            if offsets is None:
                raise ValueError("offsets are required for 1-D input")
            flat, psw = input, per_sample_weights
            off = offsets.to(input.device)
            B = off.numel() - (1 if self.include_last_offset else 0)
            ends = off[1:] if self.include_last_offset else \
                torch.cat([off[1:], off.new_tensor([flat.numel()])])
            lens = ends - off[:B]
            bag = torch.arange(B, device=input.device).repeat_interleave(lens)
        rows = self.table(flat)                               # [N, D] — the sparse lookup
        keep = None
        if self.padding_idx is not None:
            keep = (flat != self.padding_idx)
            rows = rows * keep[:, None].to(rows.dtype)
        if psw is not None:
            rows = rows * psw[:, None].to(rows.dtype)
        bag = bag.to(rows.device)
        D = rows.shape[1]
        if self.mode == "max":
            out = torch.full((B, D), float("-inf"), dtype=rows.dtype, device=rows.device)
            out = out.scatter_reduce(0, bag[:, None].expand(-1, D), rows, "amax",
                                     include_self=True)
            return torch.where(torch.isinf(out), torch.zeros_like(out), out)   # empty bags → 0
        out = torch.zeros(B, D, dtype=rows.dtype, device=rows.device).index_add_(0, bag, rows)
        if self.mode == "mean":
            ones = torch.ones(flat.numel(), device=rows.device, dtype=rows.dtype) if keep is None \
                else keep.to(rows.dtype)
            cnt = torch.zeros(B, dtype=rows.dtype, device=rows.device).index_add_(0, bag, ones)
            out = out / cnt.clamp(min=1.0)[:, None]
        return out


def partition(module, partitioner):
    """Attach a partitioner to an existing ``nn.Embedding(sparse=True)``."""
    assert isinstance(module, tnn.Embedding), "only nn.Embedding is partitionable"
    module.sparse = True
    module.partitioner = partitioner
    return module


def lookup_many(modules, ids, defer=False):
    """Rows of several embedding modules for the SAME ids (e.g. a softmax weight table
    and its bias table).  Declare the modules as a group on the model
    (``co_lookup_groups = [("softmax_w", "softmax_b")]``) and the NVLink fabric serves
    them with one lookup kernel, one push kernel and one owner kernel per step.
    ``defer=True`` returns a handle whose ``.rows()`` yields the tensors: issue the lookup
    early (e.g. on a side stream) and call ``.rows()`` where the rows are consumed."""
    from .parallel.engine import lookup_many as _lm
    return _lm(list(modules), ids, defer=defer)


def full_softmax_nll(inputs, targets, weight, bias):
    """Full-softmax cross entropy of every row of `inputs` against every row of a partitioned
    output table: per-row NLL ``[N]`` fp32, i.e. ``reduction="none"`` of ::

        cross_entropy(inputs @ weight.weight.T + bias.weight.T, targets)

    `inputs` is ``[N, K]``, `targets` ``[N]`` integer ids, `weight` / `bias` are the two
    embedding modules (``[V, K]`` and ``[V, 1]``) — the arguments `lookup_many` takes.  When
    they form a co-lookup group on the NVLink fabric with a bf16 weight shadow, inputs are bf16
    with K % 8 == 0 and K <= 1024, and no gradient is wanted, one fused kernel evaluates the
    softmax where the rows live (no gathered table, no [N, V] logits, fp32 logits; a target
    outside [0, V) gives NaN in its row).  Under the same conditions in training, a session
    with ``sess_config["full_softmax_train"] = "fused"`` also runs the forward fused and a
    fused backward: the table is recomputed in vocabulary chunks of bounded scratch, the
    softmax gradient is bf16, and `inputs` and the tables get their gradients (the tables'
    as every row, through the same push and owner kernels as a lookup's).  Otherwise the
    table is gathered and the logits materialised, which also carries gradients to the
    tables."""
    if inputs.dim() != 2:
        raise ValueError("inputs must be [N, K], got shape %s" % (tuple(inputs.shape),))
    if targets.dim() != 1 or targets.shape[0] != inputs.shape[0]:
        raise ValueError("targets must be [N] = [%d], got shape %s"
                         % (inputs.shape[0], tuple(targets.shape)))
    if targets.dtype.is_floating_point or targets.dtype == torch.bool:
        raise ValueError("targets must be integer ids, got %s" % targets.dtype)
    _check_full_softmax(inputs, weight, bias)
    from .parallel.engine import full_softmax_nll as _fs
    return _fs(inputs, targets, weight, bias)


def full_softmax_topk(inputs, weight, bias, k):
    """The k most likely rows of a partitioned output table for every row of `inputs`:
    ``(log_probs, ids)``, both ``[N, k]``, where `log_probs` (fp32) is ::

        log_softmax(inputs @ weight.weight.T + bias.weight.T)

    at `ids` (int64 global row ids in [0, V), never a padding row, no duplicates in a row).
    Within a row the order is logit descending, equal logits by ascending id, so the result
    does not depend on the partitioning, the world size or the path taken.  `inputs`, `weight`
    and `bias` are those of `full_softmax_nll`; `k` is an int with 1 <= k <= V.  Under the
    conditions of `full_softmax_nll`'s fused path and with k <= 32, one fused kernel keeps each
    row's k best (logit, id) pairs where the rows live (no gathered table, no [N, V] logits);
    otherwise the table is gathered and the logits materialised, which also carries gradients
    into `log_probs`."""
    if inputs.dim() != 2:
        raise ValueError("inputs must be [N, K], got shape %s" % (tuple(inputs.shape),))
    _check_full_softmax(inputs, weight, bias)
    if isinstance(k, bool) or not isinstance(k, int) or not 1 <= k <= weight.num_embeddings:
        raise ValueError("k must be an int in [1, %d], got %r" % (weight.num_embeddings, k))
    from .parallel.engine import full_softmax_topk as _ft
    return _ft(inputs, weight, bias, k)


def full_softmax_sample(inputs, weight, bias, num_samples=1, temperature=1.0, seed=None,
                        top_k=None, top_p=None):
    """Next-word sampling from a partitioned output table: for every row of `inputs`,
    `num_samples` = n distinct rows of the table drawn without replacement from ::

        softmax((inputs @ weight.weight.T + bias.weight.T) / temperature)

    in draw order.  Returns ``(log_probs, ids)``, both ``[N, n]``: `ids` int64 global row ids
    (never a padding row), `log_probs` fp32 the tempered ``log_softmax(logits / temperature)``
    at each id — each id's own log-probability, not the probability of the sequence of draws
    without replacement.

    The draws are the n largest Gumbel keys ``s − log E`` of the row (Gumbel-top-k), s the fp32
    logit times fp32(1 / temperature) and E ~ Exp(1) a hash of (seed, row index in `inputs`,
    global id) (`parallax_b200.parallel.engine.sample_uniform`).  So a given seed draws the same
    ids whatever the world size, partitioning, layout or path, except where two keys are within
    a few ulp.  `seed=None` draws a seed from torch's default CPU generator, so successive calls
    differ, as `torch.multinomial`'s do.  `inputs`, `weight` and `bias` are those of
    `full_softmax_nll`.  Under the conditions of its fused path and with n <= 32, one fused
    kernel keeps each row's n best keys where the rows live (no gathered table, no [N, V]
    logits); otherwise the table is gathered and the logits materialised, which also carries
    gradients into `log_probs`.

    Truncation: `top_k` (an int in [num_samples, V]) and `top_p` (a real number in (0, 1]; 1
    means no nucleus) restrict each row's draws to T = {v : s_v >= θ*}, θ* the largest θ with ::

        count(θ) >= top_k   or   (mass(θ) >= top_p  and  count(θ) >= num_samples)

    where count(θ) and mass(θ) are the number and the softmax(s) mass of the row's s >= θ, and an
    absent argument makes its clause false.  So `top_k` alone keeps the k most likely words and
    every word tied with the k-th; `top_p` alone keeps the smallest nucleus of mass >= p, never
    fewer than num_samples words; both keep the smaller of the two sets.  The draws are the n
    best keys within T (the untruncated draw order filtered to T, same noise), and `log_probs`
    stay the log-probabilities under the untruncated softmax: the log-probability under the
    renormalised distribution is ``log_probs − log mass(T)``, with mass(T) = Σ_{v in T}
    exp(log_probs of v).  The fused path finds θ* with a radix search over the fp32 key, one
    histogram pass over the table per 4-bit digit, so a truncated call reads the table 10 times.
    With both None the call is exactly the untruncated one.

    `ValueError` for the shapes `full_softmax_nll` refuses, a `num_samples` that is not an int in
    [1, V], a `temperature` that is not a finite real number > 0, a `seed` that is neither None
    nor an int in [0, 2^32), a `top_k` that is not an int in [1, V] or is below `num_samples`,
    and a `top_p` that is not a finite real number in (0, 1]."""
    import math
    import numbers
    if inputs.dim() != 2:
        raise ValueError("inputs must be [N, K], got shape %s" % (tuple(inputs.shape),))
    _check_full_softmax(inputs, weight, bias)
    V = weight.num_embeddings
    if isinstance(num_samples, bool) or not isinstance(num_samples, int) or \
            not 1 <= num_samples <= V:
        raise ValueError("num_samples must be an int in [1, %d], got %r" % (V, num_samples))
    if isinstance(temperature, bool) or not isinstance(temperature, numbers.Real) or \
            not math.isfinite(temperature) or not temperature > 0:
        raise ValueError("temperature must be a finite real number > 0, got %r" % (temperature,))
    inv_tau = float(torch.tensor(1.0 / float(temperature), dtype=torch.float32))
    if not math.isfinite(inv_tau) or inv_tau <= 0.0:
        raise ValueError("temperature %r has no finite fp32 reciprocal > 0" % (temperature,))
    if seed is None:
        seed = int(torch.randint(0, 1 << 32, (), dtype=torch.int64))
    elif isinstance(seed, bool) or not isinstance(seed, numbers.Integral) or \
            not 0 <= seed < 1 << 32:
        raise ValueError("seed must be None or an int in [0, 2^32), got %r" % (seed,))
    if top_k is not None:
        if isinstance(top_k, bool) or not isinstance(top_k, numbers.Integral) or \
                not 1 <= top_k <= V:
            raise ValueError("top_k must be None or an int in [1, %d], got %r" % (V, top_k))
        if num_samples > top_k:
            raise ValueError("num_samples (%d) must not exceed top_k (%d)" % (num_samples, top_k))
        top_k = int(top_k)
    if top_p is not None:
        if isinstance(top_p, bool) or not isinstance(top_p, numbers.Real) or \
                not math.isfinite(top_p) or not 0 < top_p <= 1:
            raise ValueError("top_p must be None or a finite real number in (0, 1], got %r"
                             % (top_p,))
        top_p = None if top_p == 1 else float(top_p)
    from .parallel.engine import full_softmax_sample as _fsm
    return _fsm(inputs, weight, bias, num_samples, inv_tau, int(seed), top_k, top_p)


def _check_full_softmax(inputs, weight, bias):
    if weight.embedding_dim != inputs.shape[1]:
        raise ValueError("weight rows have %d columns, inputs have %d"
                         % (weight.embedding_dim, inputs.shape[1]))
    if bias.embedding_dim != 1 or bias.num_embeddings != weight.num_embeddings:
        raise ValueError("bias must be a [%d, 1] embedding, got [%d, %d]"
                         % (weight.num_embeddings, bias.num_embeddings, bias.embedding_dim))
