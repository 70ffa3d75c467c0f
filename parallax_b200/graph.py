"""`Graph` — the single-device program handed to `parallel_run`.

The reference takes a complete single-GPU `tf.Graph` (model + gradients +
optimizer + global_step, `doc/parallax_api.md:4-21`) and rewrites it.  The
torch analogue is a `Graph`: an ordinary single-device ``nn.Module`` whose
``forward(**placeholders)`` returns named tensors (one of them the loss), an
optimizer spec, and declarative gradient post-processing that in the reference
lives in the user graph between `tf.gradients` and `apply_gradients`
(e.g. LM1B: `examples/lm1b/language_model_graph.py:44-62`):

* `ClipByGlobalNorm(max_norm, params, include_sparse)` — `tf.clip_by_global_norm`
* `ScaleGradients(factor, params)`      — e.g. embedding grads × batch_size
* `ClipByValue(clip, params)`            — `tf.clip_by_value`
* `ExponentialMovingAverage(decay, params)` — `ema.apply(lstm_vars)`

Fetch/feed names: placeholders are the forward argument names; fetchable
names are the keys of the forward result plus ``global_step`` and
``train_op`` (fetching ``train_op`` performs the update), mirroring
`session.run(fetches, feed_dict)` in `common/session_context.py:35-92`.
"""
import fnmatch
import inspect

import torch.nn as tnn

from . import optim as _optim

GLOBAL_STEP = "global_step"
TRAIN_OP = "train_op"


def _match(patterns, name):
    if patterns is None:
        return True
    if callable(patterns):
        return bool(patterns(name))
    if isinstance(patterns, str):
        patterns = [patterns]
    return any(fnmatch.fnmatchcase(name, p) for p in patterns)


class GradRule(object):
    def __init__(self, params=None):
        self.params = params

    def applies_to(self, name):
        return _match(self.params, name)


class ClipByGlobalNorm(GradRule):
    """Scale the aggregated gradients of `params` so that their joint L2 norm is
    at most `max_norm` (`tf.clip_by_global_norm`).

    With ``include_sparse=False`` (the default) only dense variables are matched:
    their gradient is the mean over workers after `ScaleGradients`.

    With ``include_sparse=True`` every sparse variable (embedding table) matched by
    `params` joins the norm too.  Its gradient is the one the optimizer applies
    this step: after `ScaleGradients`, duplicate ids merged, summed over workers
    (÷ num_workers with ``average_sparse``); rows not touched contribute 0.  Then::

        norm  = sqrt(Σ_dense ‖g_v‖² + Σ_sparse Σ_rows ‖g_v[row]‖²)
        scale = max_norm / max(norm, max_norm)

    and every matched gradient, dense and sparse, is multiplied by `scale`
    before its update; sparse optimizers still touch only the rows that received
    gradient.  This equals ``torch.nn.utils.clip_grad_norm_`` over the matched
    parameters of a single-device model whose embeddings have dense gradients.
    A variable belongs to the first clip rule that matches it.  Needs
    ``sync=True``."""

    def __init__(self, max_norm, params=None, include_sparse=False):
        super().__init__(params)
        self.max_norm = float(max_norm)
        self.include_sparse = bool(include_sparse)


class ScaleGradients(GradRule):
    """Multiply the gradients of `params` by `factor` before aggregation."""

    def __init__(self, factor, params=None):
        super().__init__(params)
        self.factor = float(factor)


class ClipByValue(GradRule):
    """Clamp every element of the dense gradients of `params` to
    ``[-clip_value, clip_value]`` (`tf.clip_by_value`, e.g. tf_cnn_benchmarks'
    `--gradient_clip`, `benchmark_cnn.py:797-802`).  Applied to each worker's
    gradient as it is produced (a tensor hook), i.e. before aggregation — with one
    process per GPU there is no per-worker aggregated tensor to clamp afterwards."""

    def __init__(self, clip_value, params=None):
        super().__init__(params)
        self.clip_value = float(clip_value)
        assert self.clip_value > 0


class ExponentialMovingAverage(GradRule):
    """Maintain ``shadow -= (1-decay)·(shadow - var)`` after every update for
    dense `params` (`tf.train.ExponentialMovingAverage.apply`)."""

    def __init__(self, decay, params=None):
        super().__init__(params)
        self.decay = float(decay)


class Graph(object):
    """A complete single-device training program.

    Args:
      model: ``nn.Module``; ``forward`` takes the placeholders as keyword (or
        positional) arguments and returns a dict ``name -> tensor`` (or a
        single tensor, taken to be the loss).
      optimizer: a `parallax.optim` spec applied to every trainable variable.
      sparse_optimizer: optional different spec for sparse variables.
      loss: key of the scalar to differentiate.
      grad_rules: list of `ClipByGlobalNorm` / `ClipByValue` / `ScaleGradients`.
      ema: optional `ExponentialMovingAverage`.
      loss_scale: the backward pass differentiates ``loss * loss_scale``
        (LM1B uses ``loss * num_steps``).
    """

    def __init__(self, model, optimizer=None, sparse_optimizer=None,
                 loss="loss", grad_rules=(), ema=None, loss_scale=1.0,
                 name="graph"):
        assert isinstance(model, tnn.Module)
        self.model = model
        self.optimizer = optimizer
        self.sparse_optimizer = sparse_optimizer or optimizer
        assert optimizer is None or isinstance(optimizer, _optim.Optimizer)
        self.loss = loss
        self.grad_rules = list(grad_rules)
        self.ema = ema
        self.loss_scale = float(loss_scale)
        self.name = name
        sig = inspect.signature(model.forward)
        self.placeholders = [
            p.name for p in sig.parameters.values()
            if p.kind in (p.POSITIONAL_OR_KEYWORD, p.KEYWORD_ONLY)]
        self._install_value_clips()

    def _install_value_clips(self):
        for rule in self.grad_rules:
            if not isinstance(rule, ClipByValue):
                continue
            c = rule.clip_value
            for name, p in self.model.named_parameters():
                if p.requires_grad and rule.applies_to(name):
                    p.register_hook(lambda g, c=c: g if g.is_sparse else g.clamp(-c, c))

    # -- helpers used by the engine -------------------------------------------
    def clip_rules(self):
        return [r for r in self.grad_rules if isinstance(r, ClipByGlobalNorm)]

    def joint_clip_index(self, name):
        """Index in `clip_rules()` of the rule that clips sparse variable `name`
        jointly with its dense variables (the first rule matching `name`, when it
        has ``include_sparse``), else -1."""
        for i, r in enumerate(self.clip_rules()):
            if r.applies_to(name):
                return i if r.include_sparse else -1
        return -1

    def scale_for(self, name):
        f = 1.0
        for r in self.grad_rules:
            if isinstance(r, ScaleGradients) and r.applies_to(name):
                f *= r.factor
        return f

    def trainable(self):
        return self.optimizer is not None
