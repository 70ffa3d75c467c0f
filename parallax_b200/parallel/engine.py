"""`TrainEngine` — turns a single-device `Graph` into a sparsity-aware
data-parallel trainer.

This is the counterpart of the reference's graph transforms
(`mpi/graph_transform.py:64-101`, `ps/graph_transform.py:21-60`,
`hybrid/graph_transform.py:280-377`) — but instead of rewriting a MetaGraph it
performs *module surgery* once, at wrap time:

1. analyse: tag each variable dense/sparse (`analyzer.py`);
2. choose the effective run option (degeneration rules) and the route;
3. sparse variables: replace each ``nn.Embedding(sparse=True)`` by a
   `ShardedEmbedding` backed by a row-partitioned table on the fabric;
4. dense variables: hand them to a dense group (bucketed, fused
   aggregation + optimizer);
5. static schedule: the order in which buckets/tables are processed is fixed
   here, identically on every rank (replaces Horovod's per-step negotiation,
   `horovod/common/operations.cc:1274-1590`); a debug cross-rank check
   reproduces its mismatch errors (`operations.cc:213-415`).
"""
import hashlib
import json
import os
import time

import torch
import torch.nn as tnn

from .. import consts, optim as _optim
from ..analyzer import analyze
from ..log import parallax_log
from . import modes


class _LookupFn(torch.autograd.Function):
    """rows = table[ids]; backward records (ids, grad_rows) on the table —
    the engine ships them after backward (push → owner apply)."""

    @staticmethod
    def forward(ctx, anchor, ids, table):
        ctx.table = table
        ctx.ids_shape = tuple(ids.shape)
        flat = ids.reshape(-1)
        rows, token = table.lookup(flat)
        ctx.token = token
        return rows.reshape(*ids.shape, table.D)

    @staticmethod
    def backward(ctx, grad_out):
        ctx.table.add_pending(ctx.token, grad_out.reshape(-1, ctx.table.D))
        return None, None, None


class _GroupLookupFn(torch.autograd.Function):
    """One fused lookup of several co-indexed tables (`parallax.nn.lookup_many`):
    rows_k = table_k[ids] for every member; backward hands all gradients to the group,
    which ships them with one push kernel."""

    @staticmethod
    def forward(ctx, anchor, ids, group):
        ctx.group = group
        outs, token = group.lookup(ids.reshape(-1))
        ctx.token = token
        return tuple(o.reshape(*ids.shape, t.D) for o, t in zip(outs, group.tables))

    @staticmethod
    def backward(ctx, *grads):
        ctx.group.add_pending(ctx.token, list(grads))
        return None, None, None


class _AttachFn(torch.autograd.Function):
    """Gives the rows of an already-executed lookup their place in the autograd graph
    *now*.  Autograd runs backward nodes in reverse creation order, so a lookup that was
    prefetched at the top of the forward pass would hand its gradients over last; attaching
    where the rows are consumed keeps the push of that group early in the backward pass
    (underneath whatever was computed between the prefetch and the use)."""

    @staticmethod
    def forward(ctx, anchor, pending, *rows):
        ctx.pending = pending
        return tuple(r.view_as(r) for r in rows)

    @staticmethod
    def backward(ctx, *grads):
        p = ctx.pending
        p.group.add_pending(p.token, list(grads))
        return (None, None) + (None,) * len(grads)


class PendingLookup(object):
    """Result of `lookup_many(..., defer=True)`: the lookup kernel has been issued (on the
    current stream); `rows()` returns the tensors and, when gradients are enabled, attaches
    them to the autograd graph at that point."""

    def __init__(self, rows, group=None, token=None, anchor=None):
        self._rows, self.group, self.token, self._anchor = rows, group, token, anchor

    def rows(self):
        if self.group is None or self.token is None:
            return self._rows
        return list(_AttachFn.apply(self._anchor, self, *self._rows))


def lookup_many(modules, ids, defer=False):
    """rows of several embedding modules for the SAME ids.  On the NVLink fabric, when
    the modules form a co-lookup group (`Model.co_lookup_groups`), this is one lookup
    kernel forward and one push / one owner kernel backward for all of them; anywhere
    else it is the plain sequence of lookups.  `defer=True` returns a `PendingLookup`
    (prefetch now, attach to autograd where the rows are used)."""
    tabs = [getattr(m, "table", None) for m in modules]
    grp = getattr(tabs[0], "group", None) if tabs[0] is not None else None
    if grp is not None and len(modules) > 1 and list(grp.tables) == tabs:
        if torch.is_grad_enabled():
            if defer:
                outs, token = grp.lookup(ids.reshape(-1))
                outs = [o.reshape(*ids.shape, t.D) for o, t in zip(outs, grp.tables)]
                return PendingLookup(outs, grp, token, modules[0]._anchor)
            return list(_GroupLookupFn.apply(modules[0]._anchor, ids, grp))
        outs, _ = grp.lookup(ids.reshape(-1), record=False)
        outs = [o.reshape(*ids.shape, t.D) for o, t in zip(outs, grp.tables)]
        return PendingLookup(outs) if defer else outs
    outs = [m(ids) for m in modules]
    return PendingLookup(outs) if defer else outs


def _fused_group(inputs, weight, bias):
    """The co-lookup group whose fused full-softmax kernels can take `inputs` against the
    (weight, bias) embedding modules, else None: the modules form a group on the NVLink fabric
    (protocol nvlink) whose weight table keeps a bf16 shadow, and `inputs` is bf16 on the group's
    device with K % 8 == 0 and K <= 512."""
    tabs = [getattr(m, "table", None) for m in (weight, bias)]
    grp = getattr(tabs[0], "group", None) if tabs[0] is not None else None
    K = int(inputs.shape[-1])
    if grp is not None and list(grp.tables) == tabs and grp.protocol == "nvlink" and \
            tabs[0].use_shadow and inputs.dtype == torch.bfloat16 and \
            inputs.device == grp.device and K % 8 == 0 and K <= 512:
        return grp
    return None


def _wants_grad(inputs, weight, bias):
    return torch.is_grad_enabled() and (inputs.requires_grad or weight._anchor.requires_grad or
                                        bias._anchor.requires_grad)


def _fused_eval_group(inputs, weight, bias):
    """`_fused_group` where no gradient is wanted, else None."""
    grp = _fused_group(inputs, weight, bias)
    return None if grp is None or _wants_grad(inputs, weight, bias) else grp


class _FullSoftmaxNLLFn(torch.autograd.Function):
    """Fused full-softmax NLL in training (sess_config["full_softmax_train"] = "fused"):
    forward `NVSparseGroup.full_softmax_nll_lse`, backward `full_softmax_nll_grad`.  When the
    tables want gradients the forward counts one pending call of every row of the group
    (`record_all_rows`) and the backward hands the rows to `add_pending`, so the unchanged
    push and owner kernels apply them like a lookup's."""

    @staticmethod
    def forward(ctx, anchor_w, anchor_b, inputs, targets, group):
        nll, lse = group.full_softmax_nll_lse(inputs, targets)
        ctx.group = group
        ctx.tables = ctx.needs_input_grad[0] or ctx.needs_input_grad[1]
        ctx.token = group.record_all_rows() if ctx.tables else None
        ctx.save_for_backward(inputs, targets, lse)
        return nll

    @staticmethod
    def backward(ctx, g):
        inputs, targets, lse = ctx.saved_tensors
        want_x = ctx.needs_input_grad[2]
        dx, dW, db = ctx.group.full_softmax_nll_grad(inputs, targets, lse, g, want_x=want_x,
                                                     want_tables=ctx.tables)
        if ctx.tables:
            ctx.group.add_pending(ctx.token, [dW, db])
        return None, None, dx if want_x else None, None, None


def full_softmax_nll(inputs, targets, weight, bias):
    """Per-row ``cross_entropy(inputs @ W.T + b, targets, reduction="none")`` over every row
    of the (weight, bias) embedding modules.  Where `_fused_group` finds a group, its fused
    kernel computes it where the rows live when no gradient is wanted, and also in training
    when the session sets ``full_softmax_train="fused"`` (`_FullSoftmaxNLLFn`); everything else
    runs the gather + matmul + cross_entropy composition (which also gives the tables their
    gradients in training)."""
    grp = _fused_group(inputs, weight, bias)
    if grp is not None:
        if not _wants_grad(inputs, weight, bias):
            return grp.full_softmax_nll(inputs, targets)
        if grp.full_softmax_train == "fused":
            return _FullSoftmaxNLLFn.apply(weight._anchor, bias._anchor, inputs, targets, grp)
    return full_softmax_composition(inputs, targets, weight, bias)


# largest k of the fused top-k kernel (its per-row list capacity)
FUSED_TOPK_MAX = 32


def full_softmax_topk(inputs, weight, bias, k):
    """``(log_probs [N, k], ids [N, k])`` of the k largest full-softmax logits of each row,
    logit descending and equal logits by ascending id.  Fused where `_fused_eval_group` finds a
    group and k <= 32; everything else (and training) runs `full_softmax_topk_composition`."""
    grp = _fused_eval_group(inputs, weight, bias)
    if grp is not None and k <= FUSED_TOPK_MAX:
        return grp.full_softmax_topk(inputs, k)
    return full_softmax_topk_composition(inputs, weight, bias, k)


def _gathered_logits(inputs, weight, bias):
    """fp32 [N, V] logits of the unfused compositions, from every row of the tables gathered."""
    ids = torch.arange(weight.num_embeddings, device=inputs.device)
    w, b = lookup_many([weight, bias], ids)
    w, b = w.to(inputs.dtype), b.squeeze(-1).float()
    return (inputs @ w.t()).float() + b


def full_softmax_composition(inputs, targets, weight, bias):
    """The unfused full softmax: gather every row, materialise the [N, V] logits."""
    logits = _gathered_logits(inputs, weight, bias)
    return torch.nn.functional.cross_entropy(logits, targets, reduction="none")


def full_softmax_topk_composition(inputs, weight, bias, k):
    """The unfused top-k: gather every row, materialise the [N, V] logits, `log_softmax`, then
    the k best of each row by (logit descending, id ascending) (`_ordered_top`).  Gradients
    flow into `log_probs`."""
    lp = torch.log_softmax(_gathered_logits(inputs, weight, bias), dim=-1)
    top = _ordered_top(lp.detach(), k)
    return lp.gather(1, top), top


def _ordered_top(keys, k):
    """int64 [N, k]: the columns of each row's k largest `keys` [N, V], ordered by (key
    descending, column ascending).  `torch.topk` leaves the order of equal values open, so it
    only finds each row's k-th value; the rows' candidates at or above it are then sorted
    stably (ascending column within equal values)."""
    n = keys.shape[0]
    with torch.no_grad():
        kth = torch.topk(keys, k, dim=1).values[:, -1:]
        r, c = (keys >= kth).nonzero(as_tuple=True)   # row-major: ids ascend within a row
        o = torch.sort(keys[r, c], descending=True, stable=True).indices
        o = o[torch.sort(r[o], stable=True).indices]
        r, c = r[o], c[o]
        cnt = torch.bincount(r, minlength=n)
        rank = torch.arange(r.numel(), device=r.device) - (torch.cumsum(cnt, 0) - cnt)[r]
        keep = rank < k
        top = torch.empty(n, k, dtype=torch.int64, device=keys.device)
        top[r[keep], rank[keep]] = c[keep]
    return top


def full_softmax_sample(inputs, weight, bias, n, inv_tau, seed, top_k=None, top_p=None):
    """``(log_probs [N, n], ids [N, n])``: n draws without replacement from the tempered full
    softmax of each row, in draw order (the n largest Gumbel keys), truncated to each row's top
    `top_k` / nucleus `top_p` when given (`truncation_threshold`).  Fused where
    `_fused_eval_group` finds a group and n <= 32; everything else (and training) runs
    `full_softmax_sample_composition`.  Both take the same keys, so they draw the same ids
    except where two keys are within a few ulp."""
    grp = _fused_eval_group(inputs, weight, bias)
    if grp is not None and n <= FUSED_TOPK_MAX:
        if top_k is None and top_p is None:
            return grp.full_softmax_sample(inputs, n, inv_tau, seed)
        return grp.full_softmax_sample(inputs, n, inv_tau, seed, top_k=top_k, top_p=top_p)
    return full_softmax_sample_composition(inputs, weight, bias, n, inv_tau, seed, top_k, top_p)


def sample_uniform(seed, rows, gids):
    """fp32 [len(rows), len(gids)]: the sampling noise's uniform v of (seed, row, global id),
    bit for bit the kernels' (`sample_log_e` in `kernels/sparse_group.cuh`)::

        h = sr_mix(sr_mix(sr_mix(seed) ^ row) ^ gid)
        v = min(fp32(h) · 2^-32 + 2^-33, 1 − 2^-24)

    `rows` and `gids` are int64 tensors of values in [0, 2^32)."""
    sr_mix, m32 = _optim.sr_mix, _optim._M32
    rk = sr_mix(sr_mix(int(seed) & m32) ^ (rows & m32))
    h = sr_mix(rk[:, None] ^ (gids & m32)[None, :])
    v = h.to(torch.float32) * 2.0 ** -32 + 2.0 ** -33
    return v.clamp_(max=1.0 - 2.0 ** -24)


def sample_log_e(seed, rows, gids):
    """fp32 [len(rows), len(gids)]: log E with E = −log1p(−v) ~ Exp(1) (`sample_uniform`); the
    Gumbel key of a scaled logit s is s − log E."""
    return torch.log(-torch.log1p(-sample_uniform(seed, rows, gids)))


# elements of the int64 temporaries of the composition's noise, per row chunk
_NOISE_CHUNK = 1 << 24


def truncation_threshold(s, n, top_k=None, top_p=None):
    """fp32 [N]: each row's θ* of truncated sampling over the scaled logits `s` [N, V] (fp32):
    the largest θ with ``count(θ) >= top_k`` or ``(mass(θ) >= top_p and count(θ) >= n)``, where
    count(θ) and mass(θ) are the number and the softmax(s) mass of the row's s >= θ (an absent
    argument makes its clause false; −0 equals +0, as in fp32 comparison).  A row keeps T = {v :
    s_v >= θ*}.  Sort-based in row chunks: s is sorted per row, the masses are fp64, and every
    position of a run of equal values takes the run's count and mass, so ties are kept together.
    −inf where the predicate never holds (every word kept)."""
    N, V = s.shape
    out = torch.empty(N, dtype=torch.float32, device=s.device)
    step = max(1, _NOISE_CHUNK // max(V, 1))
    with torch.no_grad():
        for r0 in range(0, N, step):
            vals = torch.sort(s[r0:r0 + step].detach().float(), dim=1, descending=True).values
            q = torch.softmax(vals.double(), dim=1)
            mass = torch.cumsum(q, dim=1)
            neg = (-vals).contiguous()                       # ascending
            end = torch.searchsorted(neg, neg, right=True) - 1   # last position of each run
            cnt, m = end + 1, mass.gather(1, end)
            ok = torch.zeros_like(cnt, dtype=torch.bool)
            if top_k is not None:
                ok |= cnt >= top_k
            if top_p is not None:
                ok |= (m >= top_p) & (cnt >= n)
            th = vals.gather(1, ok.int().argmax(1, keepdim=True))[:, 0]   # the first that holds
            out[r0:r0 + step] = torch.where(ok.any(1), th, -float("inf"))
    return out


def full_softmax_sample_composition(inputs, weight, bias, n, inv_tau, seed, top_k=None,
                                    top_p=None):
    """The unfused sampler: gather every row, materialise the [N, V] logits, scale them by
    `inv_tau` and take `log_softmax`; the keys s − log E come from the torch noise in row chunks,
    and the ids are each row's n best keys by (key descending, id ascending) (`_ordered_top`).
    With `top_k` / `top_p` the keys of s below the row's `truncation_threshold` are −inf first;
    `log_probs` stay those of the untruncated softmax.  Gradients flow into `log_probs`."""
    s = _gathered_logits(inputs, weight, bias) * inv_tau
    lp = torch.log_softmax(s, dim=-1)
    N, V = s.shape
    with torch.no_grad():
        keys = s.detach().clone()
        gids = torch.arange(V, device=s.device)
        step = max(1, _NOISE_CHUNK // max(V, 1))
        for r0 in range(0, N, step):
            rows = torch.arange(r0, min(N, r0 + step), device=s.device)
            keys[r0:r0 + step] -= sample_log_e(seed, rows, gids)
        if top_k is not None or top_p is not None:
            th = truncation_threshold(s, n, top_k, top_p)
            keys.masked_fill_(s.detach() < th[:, None], -float("inf"))
        top = _ordered_top(keys, n)
    return lp.gather(1, top), top


class ShardedEmbedding(tnn.Module):
    """Drop-in replacement for ``nn.Embedding(sparse=True)`` whose storage is
    a partitioned table on the fabric."""

    def __init__(self, table, padding_idx=None):
        super().__init__()
        self.table = table
        self.num_embeddings, self.embedding_dim = table.V, table.D
        # gives autograd a reason to call backward; never updated
        self._anchor = tnn.Parameter(torch.zeros((), device=table.anchor_device),
                                     requires_grad=True)
        self._anchor._parallax_skip = True

    def forward(self, ids):
        if torch.is_grad_enabled():
            return _LookupFn.apply(self._anchor, ids, self.table)
        rows, _ = self.table.lookup(ids.reshape(-1), record=False)
        return rows.reshape(*ids.shape, self.table.D)

    def extra_repr(self):
        return "V=%d, D=%d, P=%d, replicated=%s" % (
            self.table.V, self.table.D, self.table.layout.P,
            self.table.layout.replicated)


class _HostTableAdapter(object):
    """Gives `HostSparseTable` the lookup/add_pending(token) protocol."""

    def __init__(self, t):
        self.t = t
        self.V, self.D, self.layout = t.V, t.D, t.layout
        self.anchor_device = t.device
        self.name = t.name

    def lookup(self, flat_ids, record=True):
        ids = flat_ids.to(torch.int64).to(self.t.device)
        return self.t.gather_rows(ids).to(self.t.out_dtype), ids

    def add_pending(self, token, grad_rows):
        self.t.add_pending(token, grad_rows)

    def __getattr__(self, k):
        return getattr(self.t, k)


def _set_submodule(root, path, new):
    """Replace the module at `path` — and every other attribute that refers to the
    same module object (tied embeddings, e.g. NMT `share_vocab`) — by `new`."""
    parts = path.split(".")
    parent = root
    for p in parts[:-1]:
        parent = getattr(parent, p)
    old = getattr(parent, parts[-1])
    setattr(parent, parts[-1], new)
    if isinstance(old, tnn.Module):
        for m in root.modules():
            for name, child in list(m._modules.items()):
                if child is old:
                    m._modules[name] = new


class TrainEngine(object):
    def __init__(self, graph, comm, config, sync=True, backend=None):
        self.graph = graph
        self.comm = comm
        self.config = config
        self.model = graph.model
        requested = config.normalized_run_option()
        modes.validate(requested, sync, config.communication_config.ps_config)
        self.analysis = analyze(self.model, comm.world)
        self.run_option = self.analysis.effective_run_option(requested)
        if self.run_option != requested:
            parallax_log.info("run_option %s degenerates to %s (dense=%d sparse=%d)",
                              requested, self.run_option,
                              len(self.analysis.dense), len(self.analysis.sparse))
        self.route = modes.route_for(self.run_option, sync)
        self.backend = backend or self._pick_backend()
        self.global_step = 0
        self.tables = {}
        self.dense = None
        self.step_times = []
        self._check_joint_clip(sync)
        self._check_rowwise(sync)
        self._check_layerwise(sync)
        self._check_sparse_weights(sync)
        self._check_micro_batches(sync)
        self._check_full_softmax_train()
        self._build()
        self._consistency_check()
        self._start_aux()
        if config.export_graph_path:
            self.export_report(config.export_graph_path)

    # ------------------------------------------------------------------ build
    def _pick_backend(self):
        forced = os.environ.get(consts.PARALLAX_FABRIC) or \
            self.config.sess_option("fabric")
        if forced:
            return forced
        return "nvlink" if self.comm.is_cuda else "host"

    def _build(self):
        g, comm, cfg = self.graph, self.comm, self.config
        if self.backend in ("host", "library"):
            from .host_backend import HostDenseGroup, HostSparseTable
            # "host": everything on the CPU over gloo (tests, oracle);
            # "library": same code, tensors on this worker's device, collectives on
            # NCCL — for jobs spanning several NVLink domains
            dev = torch.device("cpu") if self.backend == "host" else comm.device
            self._lib_device = dev
            # byte-greedy placement of every sparse variable's partitions on the owners — the
            # same rule as the NVLink fabric (`ps/between_graph_parallel.py:49-70`)
            from .layout import assign_owners
            kind = g.sparse_optimizer.kind if g.sparse_optimizer else "sgd"
            items = []
            for path, mod in sorted(self.analysis.sparse_modules.items()):
                info = self.analysis.variables[path + ".weight" if path else "weight"]
                rows = (int(mod.weight.shape[0]) + info.partitions - 1) // info.partitions
                items.append((path, info.partitions,
                              rows * _optim.table_row_bytes(kind, int(mod.weight.shape[1]),
                                                            self.sparse_weight_dtype)))
            placed = assign_owners(items, comm.world) \
                if bool(cfg.communication_config.ps_config.boundary_among_servers) else {}
            for path, mod in self.analysis.sparse_modules.items():
                pname = path + ".weight" if path else "weight"
                info = self.analysis.variables[pname]
                part = getattr(mod, "partitioner", None)
                t = HostSparseTable(
                    pname, mod.weight, info.partitions,
                    part.strategy if part is not None else "mod",
                    g.sparse_optimizer, comm, self.route, g, cfg,
                    init={"seed": getattr(mod, "init_seed", 1234),
                          "scale": getattr(mod, "init_scale", 0.05)}, device=dev,
                    owners=placed.get(path), weight_dtype=self.sparse_weight_dtype)
                adapter = _HostTableAdapter(t)
                self.tables[pname] = adapter
                _set_submodule(self.model, path, ShardedEmbedding(adapter))
            self.model.to(dev)
            dense_named = [(n, p) for n, p in self.model.named_parameters()
                           if p.requires_grad and
                           not getattr(p, "_parallax_skip", False)]
            if g.trainable():
                self.dense = HostDenseGroup(dense_named, g.optimizer, comm,
                                            self.route, g,
                                            micro_batches=self.micro_batches)
                self._link_joint_tables()
        elif self.backend == "nvlink":
            from .nvlink_backend import build_nvlink
            build_nvlink(self)
        else:
            raise ValueError("unknown fabric %r" % self.backend)

    def _link_joint_tables(self):
        """Host / library fabric: hand the tables of `include_sparse` clip rules to the
        dense group, which applies them once the rule's norm is known."""
        self.dense.joint_tables = [t.t for t in self._table_order() if t.clip_rule >= 0]

    def _check_joint_clip(self, sync):
        """Refuse at build what a `ClipByGlobalNorm(include_sparse=True)` cannot mean."""
        g = self.graph
        if not any(r.include_sparse for r in g.clip_rules()):
            return
        if not sync:
            raise ValueError(
                "ClipByGlobalNorm(include_sparse=True) needs sync=True: an asynchronous "
                "PS has no aggregated sparse gradient to take the norm of")
        if self.backend == "nvlink" and \
                self.config.communication_config.ps_config.protocol == "nccl":
            raise NotImplementedError(
                "ClipByGlobalNorm(include_sparse=True) is not implemented for "
                "PSConfig(protocol='nccl') on the NVLink fabric; use "
                "sess_config={'fabric': 'library'} (or 'host') for a joint clip over "
                "library collectives")
        opts = self.config.sess_config if isinstance(self.config.sess_config, dict) else {}
        declared = list(opts.get("sparse_groups") or
                        getattr(self.model, "co_lookup_groups", None) or [])
        known = set(self.analysis.sparse_modules)
        for paths in declared:
            paths = [p for p in paths if p in known]
            rules = {g.joint_clip_index(p + ".weight" if p else "weight") for p in paths}
            if len(rules) > 1:
                raise ValueError(
                    "co-lookup group %s: its tables must all be clipped by the same "
                    "ClipByGlobalNorm(include_sparse=True) rule or all by none" % paths)

    def _check_sparse_weights(self, sync):
        """``sess_config["sparse_weights"]``: "fp32" (default) or "bf16" master rows for every
        sparse variable.  Refuses at build, before anything is allocated, what bf16 masters
        cannot do; sets `self.sparse_weight_dtype`."""
        value = self.config.sess_option("sparse_weights", "fp32")
        self.sparse_weight_dtype = _optim.sparse_weight_dtype(value)
        if value != "bf16":
            return
        if not sync:
            raise ValueError(
                "sparse_weights='bf16' needs sync=True: the asynchronous push applies rows "
                "into fp32 master tables on their owners")
        if self.backend == "nvlink":
            cdt = self.config.sess_option("compute_dtype")
            if cdt not in ("bf16", "bfloat16", torch.bfloat16):
                raise ValueError(
                    "sparse_weights='bf16' on the NVLink fabric needs compute_dtype='bf16' "
                    "(got %r): lookups read bf16 master rows into bf16 outputs only" % (cdt,))

    def _check_micro_batches(self, sync):
        """``sess_config["micro_batches"]``: forward/backward passes per optimizer step
        (default 1).  Refuses at build, before anything is allocated, what cannot
        accumulate; sets `self.micro_batches`."""
        k = self.config.sess_option("micro_batches", 1)
        if isinstance(k, bool) or not isinstance(k, int) or k < 1:
            raise ValueError("sess_config['micro_batches'] must be a positive int, got %r "
                             "(1 runs one forward/backward pass per step)" % (k,))
        self.micro_batches = k
        if k == 1:
            return
        if not sync:
            raise ValueError(
                "micro_batches=%d needs sync=True: an asynchronous PS applies every "
                "gradient as it arrives and has no step to accumulate into; use "
                "micro_batches=1" % k)
        if self.backend == "nvlink":
            if self.config.sess_option("dense_update", "sharded") == "replicated" or \
                    self.config.communication_config.ps_config.protocol == "nccl":
                raise ValueError(
                    "micro_batches=%d is not implemented on the NVLink fabric with "
                    "dense_update='replicated' or PSConfig(protocol='nccl'): those reduce in "
                    "place with an all-reduce per step.  Use the default sharded update, or "
                    "sess_config={'fabric': 'library'} to accumulate over library "
                    "collectives" % k)

    def _check_full_softmax_train(self):
        """``sess_config["full_softmax_train"]``: "composition" (default) or "fused", how
        `parallax.nn.full_softmax_nll` trains.  Refuses at build, before anything is
        allocated, where the fused kernels cannot run."""
        value = self.config.sess_option("full_softmax_train", "composition")
        if value not in ("composition", "fused"):
            raise ValueError("sess_config['full_softmax_train'] must be 'composition' or "
                             "'fused', got %r" % (value,))
        if value == "composition":
            return
        if self.backend != "nvlink":
            raise ValueError(
                "full_softmax_train='fused' needs the NVLink fabric (got fabric %r): the fused "
                "kernels read the table rows where their owners store them" % (self.backend,))
        if self.config.communication_config.ps_config.protocol == "nccl":
            raise ValueError(
                "full_softmax_train='fused' is not implemented for PSConfig(protocol='nccl'): "
                "the fused kernels read peers' rows over NVLink, not through library "
                "collectives")
        cdt = self.config.sess_option("compute_dtype")
        if cdt not in ("bf16", "bfloat16", torch.bfloat16):
            raise ValueError(
                "full_softmax_train='fused' needs compute_dtype='bf16' (got %r): the fused "
                "kernels take bf16 inputs and bf16 table rows" % (cdt,))

    def _split_feeds(self, feeds):
        """The `micro_batches` parts of a step's feeds: every tensor feed with a dim 0 as
        K equal views along it, everything else unchanged in every part."""
        K = self.micro_batches
        parts = [dict() for _ in range(K)]
        for name, v in feeds.items():
            if torch.is_tensor(v) and v.dim() > 0:
                if v.shape[0] % K:
                    raise ValueError(
                        "feed %r: dim 0 (%d) is not divisible by micro_batches=%d"
                        % (name, v.shape[0], K))
                n = v.shape[0] // K
                for k in range(K):
                    parts[k][name] = v[k * n:(k + 1) * n]
            else:
                for k in range(K):
                    parts[k][name] = v
        return parts

    @staticmethod
    def _combine_outputs(outs):
        """One step's outputs from its micro-batches': floating-point 0-dim tensors (the loss)
        averaged, integer 0-dim tensors (counts, e.g. NMT's `word_count`) summed, other tensors
        with a dim 0 concatenated along it, anything else (0-dim booleans included) from the
        last micro-batch."""
        res = {}
        for k, v in outs[-1].items():
            vals = [o[k] for o in outs]
            if not torch.is_tensor(v) or v.dtype == torch.bool and v.dim() == 0:
                res[k] = v
            elif v.dim() == 0 and (v.is_floating_point() or v.is_complex()):
                res[k] = torch.stack(vals).mean()
            elif v.dim() == 0:
                res[k] = torch.stack(vals).sum().to(v.dtype)
            else:
                res[k] = torch.cat(vals)
        return res

    def _check_rowwise(self, sync):
        """Refuse at build, before anything is allocated, what a row-wise optimizer
        (`optim.ROWWISE_KINDS`: one accumulator per embedding row) cannot do."""
        g = self.graph
        opt, sparse_opt = g.optimizer, g.sparse_optimizer
        if opt is not None and opt.kind in _optim.ROWWISE_KINDS and self.analysis.dense:
            raise ValueError(
                "%s keeps one accumulator per embedding row and trains sparse variables "
                "only, but the model has trainable dense variables: pass it as "
                "Graph(..., sparse_optimizer=%s(...)) and give optimizer= a dense rule"
                % (type(opt).__name__, type(opt).__name__))
        if sparse_opt is not None and sparse_opt.kind in _optim.ROWWISE_KINDS and not sync:
            raise ValueError(
                "%s needs sync=True: the asynchronous push applies every worker's rows "
                "element by element on the owner, without the merged row a row-wise rule "
                "needs" % type(sparse_opt).__name__)

    def _check_layerwise(self, sync):
        """Refuse at build, before anything is allocated, what a layer-wise optimizer
        (`optim.LAYERWISE_KINDS`: LARS, LAMB — a trust ratio per dense tensor) cannot do."""
        g = self.graph
        opt, sparse_opt = g.optimizer, g.sparse_optimizer
        if sparse_opt is not None and sparse_opt.kind in _optim.LAYERWISE_KINDS and \
                self.analysis.sparse:
            raise ValueError(
                "%s scales each dense tensor's step by a trust ratio over the whole tensor and "
                "has no rule for the rows of sparse variables, but the model has sparse "
                "variables: give them their own optimizer, e.g. "
                "Graph(..., sparse_optimizer=Momentum(...)) (the reference LARS's own sparse "
                "fallback) or Adam(...)" % type(sparse_opt).__name__)
        if opt is None or opt.kind not in _optim.LAYERWISE_KINDS:
            return
        name = type(opt).__name__
        if not sync:
            raise ValueError(
                "%s needs sync=True: its trust ratio is a norm over the whole aggregated "
                "gradient of a tensor, which an asynchronous PS never forms" % name)
        if self.backend == "nvlink" and (
                self.config.sess_option("dense_update", "sharded") == "replicated" or
                self.config.communication_config.ps_config.protocol == "nccl"):
            raise ValueError(
                "%s is not implemented on the NVLink fabric with dense_update='replicated' or "
                "PSConfig(protocol='nccl'): use the default sharded update, or "
                "sess_config={'fabric': 'library'} to run it over library collectives" % name)

    def grad_norm(self, i):
        """Pre-clip global norm of clip rule `i` (index in the graph's
        `ClipByGlobalNorm` rules) from the last completed step, as a float."""
        rule = self.graph.clip_rules()[i]
        if self.backend in ("host", "library"):
            return float(self.dense.last_grad_norm.get(id(rule), 0.0))
        st = self.dense.clip_state.get(i) if self.dense is not None else None
        return float(st.norm.item()) if st is not None else 0.0

    def _start_aux(self):
        """Timeline, stall watchdog and autotuner (SURVEY §5.1, §5.3)."""
        from ..utils import timeline
        self.timeline = timeline
        self.watchdog = None
        self.autotuner = None
        if self.comm.rank == 0:
            for name, why in consts.inert_horovod_env().items():
                parallax_log.info("%s is set but has no effect: %s", name, why)
        try:
            timeline.start_from_env(self.comm.rank)
        except Exception as e:  # pragma: no cover
            parallax_log.warning("timeline disabled: %s", e)
        if self.backend == "nvlink":
            from ..utils.watchdog import Watchdog
            from ..utils.autotune import EngineAutotuner
            if self.comm.world > 1 or os.environ.get(
                    consts.PARALLAX_STALL_CHECK_TIME_SECONDS):
                self.watchdog = Watchdog(self.comm.rank, self.comm.world,
                                         self.fabric.heap)
            if EngineAutotuner.wanted():
                self.autotuner = EngineAutotuner(self)

    def _consistency_check(self):
        """Cross-rank check of the static schedule — reproduces Horovod's
        coordinator validation (mismatched name/shape/dtype ⇒ error on all
        ranks, `horovod/common/operations.cc:213-415`)."""
        if not self.comm.distributed:
            return
        desc = [(v.name, v.shape, str(v.dtype), v.sparse, v.partitions)
                for v in self.analysis.variables.values()]
        digest = hashlib.sha1(json.dumps(desc).encode()).hexdigest()
        all_d = self.comm.all_gather_object((digest, self.run_option,
                                             self.route.sync))
        if len(set(all_d)) != 1:
            bad = [i for i, d in enumerate(all_d) if d != all_d[0]]
            raise RuntimeError(
                "Mismatched model/config across ranks (ranks %s differ from "
                "rank 0): every worker must build the same single-device "
                "graph" % bad)

    # ------------------------------------------------------------------- run
    def _prepare_feeds(self, feeds):
        dev = getattr(self, "_lib_device", None) or self.comm.device
        return {k: (v.to(dev, non_blocking=True)
                    if torch.is_tensor(v) and v.device != dev else v)
                for k, v in feeds.items()}

    def forward(self, feeds):
        feeds = self._prepare_feeds(feeds)
        out = self.model(**feeds)
        if not isinstance(out, dict):
            out = {self.graph.loss: out}
        return out

    def _table_order(self):
        return [self.tables[k] for k in sorted(self.tables)]

    def _begin_step(self, step):
        if self.dense is not None and hasattr(self.dense, "begin_step"):
            self.dense.begin_step(step)
        for t in self._table_order():
            if hasattr(t, "begin_step"):
                t.begin_step(step)

    def _step_body(self, feeds, step):
        """forward + backward + aggregation + update.  The order in which
        peer-synchronising work is issued is static: dense buckets (from
        autograd hooks, in bucket order) then sparse tables in name order."""
        ev = getattr(self, "_comm_events", None)
        if ev is not None:
            ev["start"].record()
        st = getattr(self, "_stamps", None)        # device timestamps (graph-capturable)
        if st is not None:
            from . import nvops
            nvops.stamp(st.data_ptr() + 0)
            if self.dense is not None:
                self.dense.stamp_before = st.data_ptr() + 40
        if self.micro_batches == 1:
            out = self.forward(feeds)
            self._backward(out)
        else:
            out = self._accumulate(feeds)
        if ev is not None:
            ev["bwd"].record()
        if st is not None:
            nvops.stamp(st.data_ptr() + 8)
        # sparse groups not yet pushed from inside backward, then the held-back last dense
        # bucket: the embedding push/apply is what the next step's lookup waits for
        for t in self._table_order():
            t.finish_step(step)
        if ev is not None:
            ev["sparse"].record(self.fabric.comm_stream)
        if st is not None:
            nvops.stamp(st.data_ptr() + 16, self.fabric.comm_stream)
        if self.dense is not None:
            self.dense.finish_step(step)
        if ev is not None:
            ev["dense"].record(self.fabric.comm_stream)
        if st is not None:
            nvops.stamp(st.data_ptr() + 24, self.fabric.comm_stream)
        if self.backend == "nvlink":
            torch.cuda.current_stream(self.comm.device).wait_stream(
                self.fabric.comm_stream)
        if ev is not None:
            ev["end"].record()
        if st is not None:
            nvops.stamp(st.data_ptr() + 32)
        return {k: (v.detach() if torch.is_tensor(v) else v)
                for k, v in out.items()}

    def _backward(self, out):
        loss = out[self.graph.loss]
        if self.graph.loss_scale != 1.0:
            (loss * self.graph.loss_scale).backward()
        else:
            loss.backward()

    def _accumulate(self, feeds):
        """Forward and backward of every micro-batch of the step.  The fabric reduces each
        micro-batch's gradients into the owners' fp32 accumulators; only the last one's
        are followed by the optimizer (`finish_step`)."""
        K, outs = self.micro_batches, []
        groups = [g for g in [self.dense] + list(getattr(self, "sparse_groups", ()))
                  if hasattr(g, "micro_batch")]
        for k, part in enumerate(self._split_feeds(feeds)):
            for grp in groups:
                grp.micro_batch(k, K)
            out = self.forward(part)
            if k > 0 and self.backend == "nvlink":
                # the gradient buckets are rewritten from here on: the previous micro-batch's
                # reductions, which read them (on this rank and, through the kernel's end
                # barrier, on every peer), must be complete.  The forward pass overlaps them.
                torch.cuda.current_stream(self.comm.device).wait_stream(
                    self.fabric.comm_stream)
            self._backward(out)
            if k < K - 1 and self.dense is not None:
                self.dense.end_micro_batch()
            outs.append(out)
        return self._combine_outputs(outs)

    def train_step(self, feeds):
        """One synchronous (or async-PS) training step.

        On the NVLink fabric with ``sess_config['cuda_graph']`` the whole step
        (forward, backward, every bucket/table kernel on the comm stream) is
        captured once into a CUDA graph after a few eager warm-up steps and
        replayed afterwards: the step is launch-bound otherwise (an unrolled
        20-step LSTM is ~1.5k tiny kernels).  All cross-rank state the kernels
        need (barrier epochs, step counters, hyper-parameters) lives in device
        memory, so a replay is exactly a re-execution."""
        t0 = time.perf_counter()
        if self.micro_batches > 1:
            self._split_feeds(feeds)        # a feed that cannot be split fails before the step
        step = self.global_step + 1
        tl = self.timeline.enabled()
        tuning = self.autotuner is not None and not self.autotuner.done
        if tuning:
            self.autotuner.step_begin()
        if tl:
            # a training step is this design's "cycle" (HOROVOD_TIMELINE_MARK_CYCLES,
            # `horovod/common/operations.cc:1286-1289`); marks are on unless set to 0
            if os.environ.get("PARALLAX_TIMELINE_MARK_CYCLES", "1") != "0":
                self.timeline.instant("CYCLE_START", args="step %d" % step)
            self.timeline.begin("step", "STEP", "global_step %d" % step)
        self._begin_step(step)
        # traced steps run eagerly (CUDA-event ranges cannot live inside a captured graph);
        # the autotuner re-captures the graph for every candidate setting
        if self._use_graph() and not tl:
            out = self._graph_step(feeds, step)
        else:
            out = self._step_body(feeds, step)
        self.global_step = step
        if tl:
            self.timeline.end("step", "STEP")
        if tuning:
            self.autotuner.step_end()
        if self.watchdog is not None:
            self.watchdog.step_enqueued(step)
        self.step_times.append(time.perf_counter() - t0)
        return out

    def comm_breakdown(self, feeds, steps=5):
        """Exposed (non-overlapped) communication time per step, dense vs sparse
        (BASELINE.json metric), measured with CUDA events on eager steps:
        dense kernels are launched from autograd hooks and overlap backward; what
        is *exposed* is whatever finishes after backward does."""
        assert self.backend == "nvlink"
        mk = lambda: torch.cuda.Event(enable_timing=True)
        acc = {"step_ms": 0.0, "fwd_bwd_ms": 0.0, "exposed_dense_ms": 0.0,
               "exposed_sparse_ms": 0.0}
        for _ in range(steps):
            self._comm_events = {k: mk() for k in ("start", "bwd", "dense", "sparse", "end")}
            step = self.global_step + 1
            self._begin_step(step)
            self._step_body(feeds, step)
            self.global_step = step
            torch.cuda.synchronize(self.comm.device)
            e = self._comm_events
            t_b = e["start"].elapsed_time(e["bwd"])
            t_d = e["start"].elapsed_time(e["dense"])
            t_s = e["start"].elapsed_time(e["sparse"])
            acc["step_ms"] += e["start"].elapsed_time(e["end"])
            acc["fwd_bwd_ms"] += t_b
            acc["exposed_dense_ms"] += max(0.0, t_d - t_b)
            acc["exposed_sparse_ms"] += max(0.0, t_s - max(t_d, t_b))
        self._comm_events = None
        return {k: v / steps for k, v in acc.items()}

    def comm_breakdown_replayed(self, feeds, steps=20):
        """Exposed (non-overlapped) communication per step measured INSIDE the CUDA-graph
        replay (BASELINE.json metric): `%globaltimer` probes are captured into the step
        graph — at the step start / after backward / before the first kernel of the last
        dense bucket (on the comm stream, after its inputs are complete) / after the last
        sparse group / after the last dense bucket / at the step end — and the push / owner
        kernels stamp themselves.  Returns per-step averages in ms:

        * ``exposed_sparse_ms``  comm-stream sparse work still running after backward ended
        * ``exposed_dense_ms``   the held-back dense bucket(s): fused reduce + optimizer +
          parameter all-gather, from "inputs complete" to done (at N=1 this is the fused
          optimizer alone — the N>1 minus N=1 difference is the communication)
        * ``owner_wait_ms``      time the owner kernels spent waiting for other ranks' rows
        * ``tail_ms``            backward end → step end (everything that is not overlapped)
        """
        assert self.backend == "nvlink"
        dev = self.comm.device
        self._stamps = torch.zeros(8, dtype=torch.int64, device=dev)
        self._graph_state = None
        warm = int(self.config.sess_option("graph_warmup", 3))
        self._graph_not_before = self.global_step + warm
        for _ in range(warm + 2):
            self.train_step(feeds)
        acc = {"step_ms": 0.0, "fwd_bwd_ms": 0.0, "exposed_sparse_ms": 0.0,
               "exposed_dense_ms": 0.0, "owner_wait_ms": 0.0, "tail_ms": 0.0}
        for _ in range(steps):
            self.train_step(feeds)
            torch.cuda.synchronize(dev)
            t = self._stamps.tolist()
            t0, t_bwd, t_sp, t_de, t_end, t_db = t[0], t[1], t[2], t[3], t[4], t[5]
            acc["step_ms"] += (t_end - t0) / 1e6
            acc["fwd_bwd_ms"] += (t_bwd - t0) / 1e6
            acc["exposed_sparse_ms"] += max(0, t_sp - t_bwd) / 1e6
            if self.dense is not None and t_db:
                acc["exposed_dense_ms"] += max(0, t_de - max(t_db, t_bwd)) / 1e6
            acc["tail_ms"] += max(0, t_end - t_bwd) / 1e6
            for grp in getattr(self, "sparse_groups", ()):
                if self.route.sync:
                    d = grp.device_times()
                    acc["owner_wait_ms"] += max(0, d["arrived"] - d["owner_start"]) / 1e6
        self._stamps = None
        if self.dense is not None:
            self.dense.stamp_before = None
        self._graph_state = None
        self._graph_not_before = self.global_step + warm
        out = {k: v / steps for k, v in acc.items()}
        out["graph_replay"] = bool(self._use_graph_possible())
        return out

    def _use_graph_possible(self):
        return self.backend == "nvlink" and bool(self.config.sess_option("cuda_graph", False))

    # ------------------------------------------------------------ CUDA graph
    def _use_graph(self):
        if self.backend != "nvlink" or not self.config.sess_option("cuda_graph", False):
            return False
        warm = int(self.config.sess_option("graph_warmup", 3))
        return self.global_step >= max(warm, getattr(self, "_graph_not_before", 0))

    @staticmethod
    def _feed_sig(feeds):
        return tuple((k, tuple(v.shape), v.dtype) for k, v in sorted(feeds.items()))

    def _graph_step(self, feeds, step):
        sig = self._feed_sig(feeds)
        st = getattr(self, "_graph_state", None)
        if st is None or st["sig"] != sig:
            if st is not None:
                parallax_log.warning("feed signature changed; re-capturing the step graph")
            dev = self.comm.device
            static = {k: torch.empty_like(v, device=dev) for k, v in feeds.items()}
            for k, v in feeds.items():
                static[k].copy_(v, non_blocking=True)
            torch.cuda.synchronize(dev)
            if self.comm.distributed:
                self.comm.barrier()
            from . import nvops
            g = torch.cuda.CUDAGraph()
            l0 = nvops.launches["n"]
            with torch.cuda.graph(g, capture_error_mode="thread_local"):
                out = self._step_body(static, step)
            # our own kernels recorded in the graph: each replay launches them again
            st = {"sig": sig, "graph": g, "in": static, "out": out,
                  "launches": nvops.launches["n"] - l0}
            nvops.launches["n"] = l0
            self._graph_state = st
            self.graph_captured = True
            parallax_log.info("captured the training step into a CUDA graph")
        else:
            for k, v in feeds.items():
                st["in"][k].copy_(v, non_blocking=True)
        st["graph"].replay()
        from . import nvops
        nvops.launches["n"] += st["launches"]
        return st["out"]

    def eval_step(self, feeds):
        with torch.no_grad():
            return self.forward(feeds)

    # ----------------------------------------------------------- checkpoints
    def state_dict(self):
        """Layout-independent state: full logical tensors keyed by the
        single-device variable names (so a checkpoint can be resumed with a
        different world size / run option / partition count)."""
        sd = {"global_step": self.global_step, "dense": None, "sparse": {},
              "buffers": {}}
        if self.dense is not None:
            sd["dense"] = self.dense.state_dict()
        for name, t in self.tables.items():
            sd["sparse"][name] = {"weight": t.full_weight(),
                                  "slots": t.full_slots()}
        for n, b in self.model.named_buffers():
            sd["buffers"][n] = b.detach().cpu().clone()
        return sd

    def load_state_dict(self, sd):
        self.global_step = int(sd["global_step"])
        if self.dense is not None and sd.get("dense") is not None:
            self.dense.load_state_dict(sd["dense"])
        for name, t in self.tables.items():
            if name in sd["sparse"]:
                t.load_full(sd["sparse"][name]["weight"],
                            sd["sparse"][name]["slots"])
        bufs = dict(self.model.named_buffers())
        for n, v in sd.get("buffers", {}).items():
            if n in bufs:
                with torch.no_grad():
                    bufs[n].copy_(v)

    # ---------------------------------------------------------- re-partition
    def repartition(self, num_partitions, names=None):
        """Re-shard sparse tables to `num_partitions` partitions IN PLACE
        (collective).  The reference's search relaunches the whole job for every
        candidate P (`common/partitions.py:74-138`); on one box the tables are
        re-laid out between timing windows instead, keeping weights and optimizer
        slots (SURVEY §7.4)."""
        names = sorted(self.tables) if names is None else names
        if self.backend == "nvlink":
            self._repartition_nvlink(num_partitions, names)
        else:
            from .host_backend import HostSparseTable
            for name in names:
                old = self.tables[name]
                if old.layout.P == num_partitions or old.layout.replicated:
                    continue
                weight, slots = old.full_weight(), old.full_slots()
                holder = None
                for p_, m_ in self.model.named_modules():
                    if isinstance(m_, ShardedEmbedding) and m_.table is old:
                        holder = m_
                new = _HostTableAdapter(HostSparseTable(
                    name, weight, num_partitions, old.layout.strategy,
                    self.graph.sparse_optimizer, self.comm, self.route, self.graph,
                    self.config, device=old.t.device, weight_dtype=old.t.weight_dtype))
                new.load_full(weight, slots)
                self.tables[name] = new
                if holder is not None:
                    holder.table = new
            if self.dense is not None:
                self._link_joint_tables()
        # captured graphs hold the old tables; the new ones allocate their rings
        # lazily, so run a few eager steps before capturing again
        self._graph_state = None
        self._graph_not_before = self.global_step + \
            int(self.config.sess_option("graph_warmup", 3))

    def _repartition_nvlink(self, num_partitions, names):
        from .nvlink_backend import NVSparseTable, NVSparseGroup
        from .layout import assign_owners
        opts = dict(self.config.sess_config) \
            if isinstance(self.config.sess_config, dict) else {}
        ps_cfg = self.config.communication_config.ps_config
        new_groups = []
        for grp in list(self.sparse_groups):
            olds = list(grp.tables)
            if not any(t.name in names for t in olds) or grp.layout.replicated or \
                    grp.layout.P == num_partitions:
                new_groups.append(grp)
                continue
            state = [(t.full_weight(), t.full_slots()) for t in olds]
            nbytes = sum(((t.V + num_partitions - 1) // num_partitions) *
                         _optim.table_row_bytes(t.kind, t.D, t.weight_dtype) for t in olds)
            owners = assign_owners([("g", num_partitions, nbytes)], self.comm.world)["g"] \
                if bool(ps_cfg.boundary_among_servers) else None
            cap = grp.cap
            for t in olds:
                t.release()
            news = []
            for t, (w, sl) in zip(olds, state):
                nt = NVSparseTable(t.name, w, num_partitions, t.layout.strategy,
                                   self.graph.sparse_optimizer, self.fabric, self.route,
                                   self.graph, self.config, out_dtype=t.out_dtype,
                                   options=opts, owners=owners, auto_group=False)
                nt.load_full(w, sl)
                news.append(nt)
                self.tables[t.name] = nt
                for m_ in self.model.modules():
                    if isinstance(m_, ShardedEmbedding) and m_.table is t:
                        m_.table = nt
            ng = NVSparseGroup(news)
            if cap:
                ng.capacity_hint = ng.capacity_hint or cap
            new_groups.append(ng)
        self.sparse_groups = new_groups
        if self.dense is not None:
            self.dense.link_groups(new_groups)

    # ------------------------------------------------------------ reporting
    def export_report(self, path):
        rep = self.analysis.report()
        rep.update({"run_option": self.run_option, "route": repr(self.route),
                    "backend": self.backend, "world": self.comm.world,
                    "rank": self.comm.rank})
        for name, t in self.tables.items():
            rep.setdefault("tables", {})[name] = {
                "V": t.V, "D": t.D, "P": t.layout.P,
                "strategy": t.layout.strategy,
                "rows_local": t.layout.rows_local,
                "replicated": t.layout.replicated}
        os.makedirs(path, exist_ok=True)
        fn = os.path.join(path, "analysis_worker_%d.json" % self.comm.rank)
        with open(fn, "w") as f:
            json.dump(rep, f, indent=1, default=str)
        return fn

    def close(self):
        if self.dense is not None and hasattr(self.dense, "close"):
            self.dense.close()
        for t in self.tables.values():
            if hasattr(t, "close"):
                t.close()
        if getattr(self, "watchdog", None) is not None:
            self.watchdog.stop()
            self.watchdog = None
        fab = getattr(self, "fabric", None)
        if fab is not None:
            fab.close()
            self.fabric = None
