"""LM1B language model (the reference's headline sparse workload).

Parity: `parallax/parallax/examples/lm1b/language_model.py:18-110` (model) and
`language_model_graph.py:24-81` (training graph):

* vocab 793 470, embedding 512, one LSTM layer with 2048 cells projected to
  512, 20 unrolled steps, dropout keep 0.9 on inputs and outputs, batch 128
  per GPU;
* `emb` and `softmax_w` are partitioned variables
  (`parallax.get_partitioner(num_variable_shards)`, default 32); with
  `softmax_b` they are *sparse* (their gradients are IndexedSlices);
* LSTM math: ``i, j, f, o = split(xw_plus_b(cat(x, h), W, B))``,
  ``c = σ(f + 1)·c + σ(i)·tanh(j)``, ``h = (σ(o)·tanh(c)) @ W_P``;
* loss: `tf.nn.sampled_softmax_loss` with 8192 log-uniform negatives shared by
  the batch (accidental hits removed), mean over batch×steps, scaled by
  ``num_steps`` before differentiation;
* Adagrad(lr 0.2, initial accumulator 1.0); embedding grads × batch_size; LSTM
  grads clipped to global norm 10; EMA(0.999) over the LSTM variables.

Differences: TF's unique log-uniform sampler loops on the host until 8192
distinct ids were drawn; here the same distribution/semantics (first 8192
distinct values of the draw sequence, expected counts from `num_tries`) is
computed on the device with static shapes; the LSTM layer and the sampled
softmax run as fused autograd nodes (`ops/fused.py`).
"""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import nn as pnn
from .. import optim
from ..graph import (Graph, ClipByGlobalNorm, ScaleGradients,
                     ExponentialMovingAverage)
from ..partitions import get_partitioner


def log_uniform_sample(num_sampled, range_max, device, generator=None):
    """ids ~ P(k) = log((k+2)/(k+1)) / log(range_max+1), with replacement."""
    u = torch.rand(num_sampled, device=device, generator=generator)
    ids = (torch.exp(u * math.log(range_max + 1.0)) - 1.0).to(torch.int64)
    return ids.clamp_(0, range_max - 1)


def log_uniform_logq(ids, num_sampled, range_max):
    """log of the expected count of each id among `num_sampled` draws."""
    idf = ids.to(torch.float32)
    p = (torch.log(idf + 2.0) - torch.log(idf + 1.0)) / math.log(range_max + 1.0)
    return torch.log(p * num_sampled)


def log_uniform_sample_unique(num_sampled, range_max, device, oversample=3):
    """TF's `log_uniform_candidate_sampler(unique=True)`: keep drawing until
    `num_sampled` distinct ids were seen; returns (ids [num_sampled] in draw
    order, num_tries) — with static shapes and no host round-trip (TF loops on
    the host): draw `oversample·num_sampled` candidates at once, keep the first
    occurrence of each value, take the first `num_sampled` of those."""
    M = int(oversample * num_sampled)
    d = log_uniform_sample(M, range_max, device)
    # first occurrence of each value = the draw whose position is the minimum over
    # all draws of that value: one scatter-min into a [range_max] table (3 small
    # kernels) instead of a 64-bit radix sort of the candidates
    pos = torch.arange(M, device=device, dtype=torch.int32)
    first_pos = torch.full((range_max,), M, dtype=torch.int32, device=device)
    first_pos.scatter_reduce_(0, d, pos, reduce="amin", include_self=True)
    first = first_pos[d] == pos
    cum = torch.cumsum(first.to(torch.int32), 0)
    sel = first & (cum <= num_sampled)
    slot = torch.where(sel, cum - 1, torch.full_like(cum, num_sampled)).to(torch.int64)
    out = torch.zeros(num_sampled + 1, dtype=torch.int64, device=device)
    out.scatter_(0, slot, d)
    num_tries = ((cum < num_sampled).sum() + 1).clamp(max=M).to(torch.float32)
    return out[:num_sampled], num_tries


def log_uniform_logq_unique(ids, num_tries, range_max):
    """log expected count under unique sampling: Q = -expm1(tries·log1p(-p))."""
    idf = ids.to(torch.float32)
    p = (torch.log(idf + 2.0) - torch.log(idf + 1.0)) / math.log(range_max + 1.0)
    return torch.log(-torch.expm1(num_tries * torch.log1p(-p)))


class LM1B(nn.Module):
    # softmax_w and softmax_b are always looked up with the same ids: one lookup / push /
    # owner kernel serves both on the NVLink fabric (`parallax.nn.lookup_many`)
    co_lookup_groups = [("softmax_w", "softmax_b")]

    def __init__(self, vocab_size=793470, emb_size=512, state_size=2048,
                 projected_size=512, num_sampled=8192, num_steps=20,
                 num_shards=32, keep_prob=0.9, lazy=False, eval_top_k=0, eval_sample=0,
                 sample_temperature=1.0, sample_top_k=None, sample_top_p=None):
        """`eval_top_k` = k > 0: in eval mode `forward` also returns ``"top_k_ids"``, the k
        most likely next words of every position (`parallax.nn.full_softmax_topk`).
        `eval_sample` = n > 0: in eval mode `forward` also returns ``"sample_ids"`` and
        ``"sample_log_probs"`` [B, T, n], n next words of every position drawn without
        replacement at temperature `sample_temperature` (`parallax.nn.full_softmax_sample`,
        seeded by the `sample_seed` feed), truncated to the `sample_top_k` most likely words
        and to the nucleus of mass `sample_top_p` when those are given (None: no truncation)."""
        super().__init__()
        self.eval_top_k = int(eval_top_k)
        self.eval_sample = int(eval_sample)
        self.sample_temperature = float(sample_temperature)
        self.sample_top_k, self.sample_top_p = sample_top_k, sample_top_p
        self.vocab_size, self.emb_size = vocab_size, emb_size
        self.state_size, self.projected_size = state_size, projected_size
        self.num_sampled, self.num_steps = num_sampled, num_steps
        self.keep_prob = keep_prob
        part = get_partitioner(num_shards)
        self.emb = pnn.Embedding(vocab_size, emb_size, partitioner=part, lazy=lazy)
        self.softmax_w = pnn.Embedding(vocab_size, projected_size,
                                       partitioner=part, lazy=lazy, seed=4321)
        self.softmax_b = pnn.Embedding(vocab_size, 1, partitioner=part, lazy=lazy,
                                       init_scale=0.0, seed=99)
        k = emb_size + projected_size
        self.W = nn.Parameter(torch.empty(k, 4 * state_size).uniform_(
            -math.sqrt(3.0 / k), math.sqrt(3.0 / k)))
        self.B = nn.Parameter(torch.zeros(4 * state_size))
        self.W_P = nn.Parameter(torch.empty(state_size, projected_size).uniform_(
            -math.sqrt(3.0 / state_size), math.sqrt(3.0 / state_size)))

    def lstm(self, x, c, h):
        """x: [T, B, E] (time-major) -> outputs [T*B, P] (rows ordered (t, b), a view of
        the layer's output), final c, h.  One fused autograd node
        (`ops.fused.lstm_layer`)."""
        from ..ops.fused import lstm_layer_stacked
        T, Bsz, E = x.shape
        out, c, h = lstm_layer_stacked(x, self.W, self.B, self.W_P, c, h, forget_bias=1.0)
        if self.training and self.keep_prob < 1.0:
            out = F.dropout(out, 1.0 - self.keep_prob)
        return out.reshape(T * Bsz, -1), c, h

    def forward(self, x, y=None, w=None, initial_state_c=None, initial_state_h=None,
                sample_seed=None):
        """`y` may be None in eval mode: no loss (and no pass over the softmax table for it),
        e.g. to generate text with `eval_sample`.  `sample_seed`: the int seed of the eval-mode
        samples (None: drawn from torch's default generator)."""
        Bsz, T = x.shape
        dev = self.W.device
        dt = self.W.dtype
        if y is None and self.training:
            raise ValueError("LM1B needs targets y in training")
        # Everything below is time-major (rows ordered (t, b)): the LSTM node consumes and
        # produces [T, B, ·] and the loss is a mean over all rows, so transposing the
        # [B, T] *ids* once replaces transposed copies of the [B, T, 512] activations and
        # of their gradients.
        e = self.emb(x.t())
        if e.dtype != dt:
            e = e.to(dt)
        if self.training and self.keep_prob < 1.0:
            e = F.dropout(e, 1.0 - self.keep_prob)
        c = initial_state_c.float() if initial_state_c is not None else \
            torch.zeros(Bsz, self.state_size, device=dev, dtype=torch.float32)
        h = initial_state_h.to(dt) if initial_state_h is not None else \
            torch.zeros(Bsz, self.projected_size, device=dev, dtype=dt)
        sampled_mode = self.training and self.num_sampled > 0
        # the sampler and the softmax-table lookups do not depend on the LSTM: issue them
        # on a side stream so they run underneath the (latency-bound) recurrent chain
        pre = self.prefetch_softmax(y) if sampled_mode else None
        inputs, c, h = self.lstm(e, c, h)
        row_w = None if w is None else w.t().reshape(-1)
        out = {}
        if sampled_mode:
            out["loss"] = self.sampled_softmax_loss(inputs, pre, row_w)
        elif y is not None:
            loss = self.full_softmax_loss(inputs, y.t().reshape(-1))
            if row_w is not None:
                loss = loss * row_w.to(loss.dtype)
            out["loss"] = loss.mean()
        out.update(final_state_c=c.detach(), final_state_h=h.detach())
        if self.eval_top_k > 0 and not self.training:
            _, ids = pnn.full_softmax_topk(inputs, self.softmax_w, self.softmax_b,
                                           self.eval_top_k)
            out["top_k_ids"] = ids.reshape(T, Bsz, -1).transpose(0, 1).contiguous()
        if self.eval_sample > 0 and not self.training:
            seed = None if sample_seed is None else int(sample_seed)
            trunc = {k: v for k, v in (("top_k", self.sample_top_k),
                                       ("top_p", self.sample_top_p)) if v is not None}
            lp, ids = pnn.full_softmax_sample(inputs, self.softmax_w, self.softmax_b,
                                              self.eval_sample, self.sample_temperature, seed,
                                              **trunc)
            out["sample_ids"] = ids.reshape(T, Bsz, -1).transpose(0, 1).contiguous()
            out["sample_log_probs"] = lp.reshape(T, Bsz, -1).transpose(0, 1).contiguous()
        return out

    def prefetch_softmax(self, y):
        """Time-major targets, negative sampling, one fused lookup of (softmax_w, softmax_b)
        rows for targets ∪ samples and the ``bias - log Q`` correction; on CUDA all of it
        runs on the side stream."""
        S, V = self.num_sampled, self.vocab_size
        dev = self.W.device

        def work():
            targets = y.t().reshape(-1).to(torch.int64)
            sampled, tries = log_uniform_sample_unique(S, V, dev)
            ids = torch.cat([targets, sampled])
            rows = pnn.lookup_many([self.softmax_w, self.softmax_b], ids, defer=True)
            logq = log_uniform_logq_unique(ids, tries, V)
            with torch.no_grad():
                adj = rows._rows[1].detach().reshape(-1).float() - logq
            return targets, sampled, rows, logq, adj
        if dev.type != "cuda":
            return work() + (None,)
        from ..ops import sinks
        cur = torch.cuda.current_stream(dev)
        side = sinks.side_stream(dev)
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            out = work()
        return out + (side,)

    def sampled_softmax_loss(self, inputs, pre, row_w=None):
        """mean sampled-softmax loss of `inputs` [T*B, P] (one fused node,
        `ops.fused.sampled_softmax_head`)."""
        from ..ops.fused import sampled_softmax_head
        targets, sampled, rows, logq, adj, side = pre
        if side is not None:
            cur = torch.cuda.current_stream(inputs.device)
            cur.wait_stream(side)
            for t in [targets, sampled, logq, adj] + list(rows._rows):
                t.record_stream(cur)
        # the rows enter the autograd graph HERE (late), so their gradients are handed to
        # the sparse group first thing in the backward pass, underneath the LSTM backward
        w_all, b_all = rows.rows()
        return sampled_softmax_head(inputs, w_all, b_all, logq, targets, sampled,
                                    row_w=row_w, adj=adj)

    def full_softmax_loss(self, inputs, targets):
        """per-row full-softmax NLL of `inputs` [T*B, P] (`parallax.nn.full_softmax_nll`)."""
        return pnn.full_softmax_nll(inputs, targets, self.softmax_w, self.softmax_b)


def lm1b_graph(model, batch_size=128, learning_rate=0.2, max_grad_norm=10.0):
    """The training graph of `language_model_graph.py:24-81`."""
    lstm_vars = ["W", "B", "W_P"]
    return Graph(
        model,
        optimizer=optim.Adagrad(learning_rate, initial_accumulator_value=1.0),
        loss="loss", loss_scale=float(model.num_steps),
        grad_rules=[ScaleGradients(float(batch_size), params=["emb.weight"]),
                    ClipByGlobalNorm(max_grad_norm, params=lstm_vars)],
        ema=ExponentialMovingAverage(0.999, params=lstm_vars),
        name="lm1b")


# the LM1B keyword arguments `--hpconfig` sets in the example scripts, and their types
HPCONFIG_MODEL_KEYS = {"keep_prob": float, "num_sampled": int, "emb_size": int,
                       "state_size": int, "projected_size": int}


def parse_hpconfig(spec, flags):
    """`--hpconfig name=value,...` of the LM1B example scripts (the reference's `hps.parse`):
    returns the model's keys (`HPCONFIG_MODEL_KEYS`) as `LM1B` keyword arguments, and sets any
    other name that is an attribute of `flags` (an argparse namespace) to the value, converted
    to the attribute's current type.  The training, evaluation and generation scripts share it,
    so the same flags build the same model and a checkpoint restores into it.  `ValueError` for
    any other name."""
    model_kw = {}
    for item in filter(None, (x.strip() for x in spec.split(","))):
        k, _, v = item.partition("=")
        if k in HPCONFIG_MODEL_KEYS:
            model_kw[k] = HPCONFIG_MODEL_KEYS[k](v)
        elif hasattr(flags, k):
            cur = getattr(flags, k)
            setattr(flags, k, type(cur)(v) if cur is not None else v)
        else:
            raise ValueError("unknown hyper-parameter %r in --hpconfig" % k)
    return model_kw
