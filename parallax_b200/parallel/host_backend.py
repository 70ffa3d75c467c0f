"""Host / library fabric: the whole engine expressed with plain torch ops and
`torch.distributed` library collectives (gloo on CPU; with ``fabric="library"``
the same code keeps every tensor on the worker's GPU and the collectives run on
NCCL — the path for jobs that span several NVLink domains, where peer memory
cannot be addressed).

Purpose: (1) BASELINE config 1 — plumbing and dense/sparse routing tests with
``world_size=2`` and no GPU; (2) the semantic oracle the sm_90a kernels are
checked against.  It is *not* a second production path: on a GPU box the
engine refuses to fall back to it unless explicitly asked (tests, baseline).

Aggregation semantics reproduced (SURVEY §8.1, reference
`graph_transform_lib.py:1056-1065,1095-1118,358-390`,
`horovod/tensorflow/__init__.py:62-82`): dense = mean over workers; sparse =
duplicates merged, **sum** over workers, or ÷ num_workers when
``average_sparse`` (accumulator average option 1); exactly one optimizer
application per variable/row per step.
"""
import torch

from .. import optim as _optim
from . import modes
from .layout import TableLayout


def _slots_like(t, optimizer):
    if optimizer.kind in _optim.ROWWISE_KINDS:      # one value per row of a sparse table
        t = t[:, :1]
    return tuple(torch.full_like(t, v, dtype=torch.float32)
                 for v in optimizer.slot_init())


class HostDenseGroup(object):
    """All dense variables of the graph on the host fabric."""

    def __init__(self, named_params, optimizer, comm, route, graph,
                 options=None, micro_batches=1):
        self.comm = comm
        self.route = route
        self.optimizer = optimizer
        self.graph = graph
        self.names = [n for n, _ in named_params]
        self.params = [p for _, p in named_params]
        # fp32 master copies (identity when the model is fp32)
        self.master = [p.detach().to(torch.float32).clone() for p in self.params]
        self.slots = [_slots_like(m, optimizer) for m in self.master]
        self.scales = [graph.scale_for(n) for n in self.names]
        self.ema_rule = graph.ema
        self.ema = {}
        if self.ema_rule is not None:
            for i, n in enumerate(self.names):
                if self.ema_rule.applies_to(n):
                    self.ema[i] = self.master[i].clone()
        self.last_grad_norm = {}
        # sparse tables clipped jointly with dense variables (`HostSparseTable.clip_rule`):
        # aggregated before this group's step, applied by `_clip` with the rule's scale
        self.joint_tables = []
        # micro_batches > 1: every micro-batch's gradient is widened and summed in fp32
        # (`end_micro_batch`); the step applies the sum × 1/K
        self.micro_batches = micro_batches
        self.acc = None
        # make every replica start from rank 0's values
        # (reference `mpi/runner.py:134-139` broadcast of global variables)
        for m, p in zip(self.master, self.params):
            comm.broadcast_(m, 0)
            with torch.no_grad():
                p.copy_(m.to(p.dtype))

    def zero_grad(self):
        for p in self.params:
            p.grad = None

    def end_micro_batch(self):
        """Add this micro-batch's gradients, widened to fp32, into the step's
        accumulators and clear them."""
        if self.acc is None:
            self.acc = [torch.zeros_like(p, dtype=torch.float32) for p in self.params]
        for a, p in zip(self.acc, self.params):
            if p.grad is not None:
                a.add_(p.grad.detach().to(torch.float32))
        self.zero_grad()

    def finish_step(self, step):
        W = self.comm.world
        acc = None
        if self.micro_batches > 1:
            self.end_micro_batch()
            acc, self.acc = self.acc, None
        grads = []
        for i, (p, s) in enumerate(zip(self.params, self.scales)):
            if acc is not None:
                g = acc[i] * (1.0 / self.micro_batches)
            else:
                g = p.grad
                if g is None:
                    g = torch.zeros_like(p)
                g = g.detach().to(torch.float32)
            if s != 1.0:
                g = g * s
            grads.append(g)
        hp = self.optimizer.hyper(step)
        kind = self.optimizer.kind
        if self.route.sync:
            # mean over workers; one fused buffer, one library all-reduce
            if W > 1:
                flat = torch.cat([g.reshape(-1) for g in grads]) if grads \
                    else torch.zeros(0, device=self.params[0].device if self.params else "cpu")
                self.comm.all_reduce_sum_(flat)
                flat.div_(W)
                off = 0
                for i, g in enumerate(grads):
                    n = g.numel()
                    grads[i] = flat[off:off + n].view_as(g)
                    off += n
            self._clip(grads, step)
            per_name = kind in _optim.LAYERWISE_KINDS     # exclude lists act per tensor
            for i, g in enumerate(grads):
                hp_i = self.optimizer.hyper_for(self.names[i], step) if per_name else hp
                _optim.apply_dense_(kind, self.master[i], g, self.slots[i], hp_i)
        else:
            # asynchronous PS: every worker's gradient is applied on its own,
            # un-averaged.  The host fabric serialises them in rank order.
            self._clip(grads)
            all_g = [self.comm.all_gather_tensors(g) for g in grads] \
                if W > 1 else [[g] for g in grads]
            for i, per_rank in enumerate(all_g):
                for g in per_rank:
                    _optim.apply_dense_(kind, self.master[i], g,
                                        self.slots[i], hp)
        if self.ema:
            d = self.ema_rule.decay
            for i, sh in self.ema.items():
                sh.sub_((sh - self.master[i]) * (1.0 - d))
        with torch.no_grad():
            for m, p in zip(self.master, self.params):
                p.copy_(m.to(p.dtype))
        self.zero_grad()

    def _clip(self, grads, step=None):
        for ri, rule in enumerate(self.graph.clip_rules()):
            idx = [i for i, n in enumerate(self.names) if rule.applies_to(n)]
            tabs = [t for t in self.joint_tables if t.clip_rule == ri]
            if not idx and not tabs:
                continue
            sq = sum(float((grads[i] ** 2).sum()) for i in idx)
            if tabs:
                sq += self._sparse_sumsq(tabs)
            norm = sq ** 0.5
            self.last_grad_norm[id(rule)] = norm
            scale = rule.max_norm / max(norm, rule.max_norm)
            if scale < 1.0:
                for i in idx:
                    grads[i] = grads[i] * scale
            for t in tabs:
                t.apply(step, scale)

    def _sparse_sumsq(self, tabs):
        """Σg² of the merged rows of `tabs` over the whole job.  The dense Σ is taken
        from the all-reduced gradients, identical on every rank, so only the sparse
        part is summed: the owners' shares of partitioned tables with one
        all-reduce; a replicated table was merged in full on every rank and counts
        once."""
        part = sum(t.sumsq() for t in tabs if not t.replicated)
        rep = sum(t.sumsq() for t in tabs if t.replicated)
        if self.comm.world > 1 and any(not t.replicated for t in tabs):
            buf = torch.tensor([part], dtype=torch.float64, device=tabs[0].device)
            self.comm.all_reduce_sum_(buf)
            part = float(buf[0])
        return part + rep

    # -- checkpoint -----------------------------------------------------------
    def state_dict(self):
        sd = {"master": {}, "slots": {}, "ema": {}}
        for i, n in enumerate(self.names):
            sd["master"][n] = self.master[i].detach().cpu().clone()
            sd["slots"][n] = [s.detach().cpu().clone() for s in self.slots[i]]
            if i in self.ema:
                sd["ema"][n] = self.ema[i].detach().cpu().clone()
        return sd

    def load_state_dict(self, sd):
        for i, n in enumerate(self.names):
            if n in sd["master"]:
                self.master[i].copy_(sd["master"][n])
                for s, v in zip(self.slots[i], sd["slots"].get(n, [])):
                    s.copy_(v)
                if i in self.ema and n in sd.get("ema", {}):
                    self.ema[i].copy_(sd["ema"][n])
        with torch.no_grad():
            for m, p in zip(self.master, self.params):
                p.copy_(m.to(p.dtype))

    def ema_value(self, name):
        return self.ema[self.names.index(name)]


class HostSparseTable(object):
    """One sparse variable (embedding table) on the host fabric."""

    def __init__(self, name, weight, num_partitions, strategy, optimizer, comm,
                 route, graph, config, init=None, device=None, owners=None,
                 weight_dtype=torch.float32):
        self.name = name
        self.device = torch.device("cpu") if device is None else torch.device(device)
        self.comm = comm
        self.route = route
        self.optimizer = optimizer
        self.V, self.D = int(weight.shape[0]), int(weight.shape[1])
        self.replicated = route.sparse == modes.SPARSE_ALLGATHER
        self.layout = TableLayout(self.V, num_partitions, comm.world, strategy,
                                  replicated=self.replicated, owners=owners)
        self.average = bool(config.average_sparse)
        # the rows of every micro-batch of a step are pending together and weighted 1/K
        self.micro_batches = int(config.sess_option("micro_batches", 1))
        self.local_aggregation = bool(
            config.communication_config.ps_config.local_aggregation)
        self.scale = graph.scale_for(name)
        self.clip_rule = graph.joint_clip_index(name)
        self.merged = []
        L = self.layout
        # bf16 master rows (sparse_weights="bf16"): every update is applied in fp32 on the
        # widened rows and rounded stochastically (`optim.round_bf16_stochastic`), keyed by
        # the rows' global ids
        self.weight_dtype = weight_dtype
        self.sr_seed = _optim.sr_seed(name)
        shard = torch.zeros(L.rows_local, self.D, dtype=torch.float32)
        g, l = L.global_ids_of_owner(comm.rank)
        self._gid = torch.zeros(L.rows_local, dtype=torch.int64)
        self._gid[l] = g
        if weight.device.type == "meta":
            gen = torch.Generator().manual_seed(init["seed"])
            full = torch.empty(self.V, self.D).uniform_(
                -init["scale"], init["scale"], generator=gen)
            shard[l] = full[g]
        else:
            shard[l] = weight.detach().to(torch.float32).cpu()[g]
        self.shard = shard.to(self.device, weight_dtype)
        self.slots = _slots_like(self.shard, optimizer)
        self.nslots = len(self.slots)
        self.slot_dim = _optim.slot_width(optimizer.kind, self.D)
        self.pending = []
        self.out_dtype = weight.dtype if weight.device.type != "meta" \
            else torch.float32
        self.stats = {"pushed_rows": 0, "unique_rows": 0}

    # -- forward --------------------------------------------------------------
    def gather_rows(self, ids):
        """rows = table[ids] for arbitrary global ids (ids: 1-D int64)."""
        L, W, me = self.layout, self.comm.world, self.comm.rank
        if self.replicated or W == 1:
            return self.shard[L.local_row_of(ids)].float()
        # PS-style request/response all-to-all: ids travel to their owners, rows
        # travel back; O(n) traffic per rank instead of an all-gather of every id
        owners = L.owner_of(ids)
        order = torch.argsort(owners, stable=True)
        counts = torch.bincount(owners, minlength=W).tolist()
        req, req_counts = self.comm.all_to_all_varlen(ids[order], counts)
        rows = self.shard[L.local_row_of(req)].float()
        resp, _ = self.comm.all_to_all_varlen(rows, req_counts)
        out = torch.empty(ids.numel(), self.D, dtype=torch.float32, device=self.device)
        out[order] = resp
        return out

    def add_pending(self, ids, grad_rows):
        self.pending.append((ids.reshape(-1).to(torch.int64),
                             grad_rows.reshape(-1, self.D).to(torch.float32)))

    # -- backward / update ------------------------------------------------------
    def finish_step(self, step):
        """Aggregate and apply; a table clipped jointly with other variables
        (`clip_rule` >= 0) only aggregates here and is applied by the dense group
        once the rule's norm is known."""
        self.aggregate(step)
        if self.clip_rule < 0:
            self.apply(step)

    def aggregate(self, step):
        """All-to-all (or all-gather) of this step's rows and the duplicate merge on
        the owner.  Keeps the owner's (local rows, merged gradient) segments for
        `apply`."""
        L, W, me = self.layout, self.comm.world, self.comm.rank
        if self.pending:
            ids = torch.cat([p[0] for p in self.pending])
            rows = torch.cat([p[1] for p in self.pending])
        else:
            ids = torch.zeros(0, dtype=torch.int64, device=self.device)
            rows = torch.zeros(0, self.D, device=self.device)
        self.pending = []
        if self.scale != 1.0:
            rows = rows * self.scale
        self.stats["pushed_rows"] += int(ids.numel())
        if self.local_aggregation and ids.numel():
            ids, inv = torch.unique(ids, return_inverse=True)
            agg = torch.zeros(ids.numel(), self.D, device=self.device)
            agg.index_add_(0, inv, rows)
            rows = agg
        self.stats["unique_rows"] += int(ids.numel())
        if self.replicated:
            # AR run option (Horovod semantics): all-gather of indices and values,
            # every replica applies the full update
            ids_c = torch.cat(self.comm.all_gather_varlen(ids))
            rows_c = torch.cat(self.comm.all_gather_varlen(rows))
            segs = [(ids_c, rows_c)]
        else:
            # PS / HYBRID: all-to-all of (index, row) pairs to the owning rank
            owners = L.owner_of(ids)
            order = torch.argsort(owners, stable=True)
            counts = torch.bincount(owners, minlength=W).tolist()
            ids_c, rc = self.comm.all_to_all_varlen(ids[order], counts)
            rows_c, _ = self.comm.all_to_all_varlen(rows[order], counts)
            if self.route.sync:
                segs = [(ids_c, rows_c)]
            else:
                # async PS: each worker's rows are applied on their own (rank order)
                segs, off = [], 0
                for n in rc:
                    segs.append((ids_c[off:off + n], rows_c[off:off + n]))
                    off += n
        self.merged = []
        for seg_ids, seg_rows in segs:
            u, inv = torch.unique(seg_ids, return_inverse=True)
            g = torch.zeros(u.numel(), self.D, device=self.device)
            g.index_add_(0, inv, seg_rows)
            if self.average and self.route.sync:
                g.div_(W)
            if self.micro_batches > 1:
                g.mul_(1.0 / self.micro_batches)
            self.merged.append((L.local_row_of(u), g))

    def sumsq(self):
        """Σg² (float64) over the merged rows of the last `aggregate` held here."""
        return sum(float((g.double() ** 2).sum()) for _, g in self.merged)

    def apply(self, step, scale=1.0):
        """The optimizer on the segments of the last `aggregate`, gradient × `scale`."""
        hp = self.optimizer.hyper(step)
        for rows, g in self.merged:
            if scale != 1.0:
                g = g * scale
            _optim.apply_sparse_rows_(self.optimizer.kind, self.shard, rows, g,
                                      self.slots, hp, self.sr_seed,
                                      self._gid[rows.cpu()])
        self.merged = []

    # -- checkpoint / inspection -------------------------------------------------
    def _gather_full(self, local):
        L, W = self.layout, self.comm.world
        if self.replicated or W == 1:
            g, l = L.global_ids_of_owner(0 if self.replicated else self.comm.rank)
            out = torch.zeros(self.V, local.shape[1])
            out[g] = local.cpu()[l].float()
            return out
        shards = self.comm.all_gather_tensors(local.float())
        out = torch.zeros(self.V, local.shape[1])
        for o in range(W):
            g, l = L.global_ids_of_owner(o)
            out[g] = shards[o].cpu()[l]
        return out

    def full_weight(self):
        return self._gather_full(self.shard)

    def full_slots(self):
        return [self._gather_full(s) for s in self.slots]

    def load_full(self, weight, slots=None):
        if slots is not None:
            _optim.check_table_slots(self.name, self.optimizer.kind, self.V, self.D, slots)
        g, l = self.layout.global_ids_of_owner(
            0 if self.replicated else self.comm.rank)
        l = l.to(self.device)
        self.shard[l] = weight.to(torch.float32)[g].to(self.device, self.shard.dtype)
        if slots is not None:
            for s, full in zip(self.slots, slots):
                s[l] = full.to(torch.float32)[g].to(self.device)
