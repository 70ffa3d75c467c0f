"""Sparse variables on the NVLink fabric.

`NVSparseTable` is the storage of one row-partitioned variable (fp32 master rows,
optimizer slots and — for bf16 models — a bf16 *shadow* copy that lookups read, all
in symmetric memory; with ``sess_config["sparse_weights"] = "bf16"`` the master rows
themselves are bf16, in the shadow's layout, and there is no second copy).  `NVSparseGroup` is the machinery of one *group* of tables
that are looked up with the same ids (LM1B: ``softmax_w`` + ``softmax_b``; every
other table is a group of one): per step ONE remote-gather lookup kernel per
lookup call, ONE push kernel (SMEM local aggregation + P2P stores + flag) and ONE
owner kernel (cross-source merge + sparse optimizer + flag) — see
`ops/csrc/kernels/sparse.cu`.

Reference semantics kept (file:line in /root/reference/parallax/parallax):
* sparse sync across workers — `core/python/common/graph_transform_lib.py:1558-1946`
  (accumulate every worker's IndexedSlices on the variable's server, apply once,
  workers read the result);
* local aggregation — `:1372-1556` (`PSConfig.local_aggregation`);
* average_option — SUM vs ÷num_workers (`:101-102,385-387`);
* boundary between workers and servers — `:1315-1370`: size-increasing casts run
  on the consumer (owner) side, so bf16 gradients cross the wire as bf16 and are
  widened/accumulated in fp32 by the owner (`boundary_between_workers_and_servers
  =False` widens on the sender instead, fp32 on the wire);
* variable-size receive negotiation — `horovod/common/ops/collective_operations.cc
  :80-90`: ring capacity follows the largest per-rank row count; in eager mode the
  counts are agreed on every step (one small host all-reduce), under CUDA-graph
  replay shapes are static.
"""
import ctypes
import numbers

import torch

from .. import consts, ops, optim as _optim
from ..log import parallax_log
from . import modes
from .layout import TableLayout

_vp = ctypes.c_void_p
_DT = {torch.float32: 0, torch.bfloat16: 1}


def _lookup_table(t, src, out):
    """LookupTable descriptor: table `t`'s rows, read from every rank's `src` ("shadow":
    the bf16 copy, "table": the fp32 master), into `out`."""
    return ops.LookupTable(t.dev_ptrs(src).data_ptr(), out.data_ptr(), t.D4,
                           int(src == "shadow"), int(out.dtype == torch.bfloat16))


def _count(k=1):
    from . import nvops
    nvops.launches["n"] += k


def _sp(stream):
    return _vp(stream.cuda_stream)


def full_softmax_block_rows(K):
    """Table rows per work item of the fused full-softmax kernels at input width K (`ev_bv` in
    `ops/csrc/kernels/softmax_eval.cu`): 128 up to K = 512, 64 up to K = 1024."""
    return 128 if K <= 512 else 64


class HPStage(object):
    """Device copy of an optimizer's hyper-parameter vector, refreshed once per step
    through a ring of pinned buffers (the host may run several CUDA-graph replays ahead
    of the device, so one re-used pinned buffer could be overwritten before its H2D copy
    has executed)."""
    DEPTH = 8

    def __init__(self, optimizer, device):
        self.optimizer = optimizer
        self.dev = torch.zeros(_optim.HP_SIZE, dtype=torch.float32, device=device)
        self.host = [torch.zeros(_optim.HP_SIZE, dtype=torch.float32).pin_memory()
                     for _ in range(self.DEPTH)]
        self.events = [None] * self.DEPTH
        self.i = 0
        self.step = None

    def upload(self, step):
        if self.step == step:
            return self.dev
        i = self.i
        self.i = (i + 1) % self.DEPTH
        if self.events[i] is not None:
            self.events[i].synchronize()
        h = self.host[i]
        for j, v in enumerate(self.optimizer.hyper(step)):
            h[j] = v
        self.dev.copy_(h, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self.events[i] = ev
        self.step = step
        return self.dev


def hp_stage(fabric, optimizer):
    cache = fabric.__dict__.setdefault("_hp_stages", {})
    st = cache.get(id(optimizer))
    if st is None:
        st = cache[id(optimizer)] = HPStage(optimizer, fabric.device)
    return st


class NVSparseTable(object):
    """Storage + per-table facade.  Kernels run through `self.group`."""

    def __init__(self, name, weight, num_partitions, strategy, optimizer, fabric,
                 route, graph, config, init=None, out_dtype=None, options=None,
                 owners=None, auto_group=True):
        self.name = name
        self.fabric, self.heap = fabric, fabric.heap
        self.comm = fabric.comm
        self.rank, self.world, self.device = fabric.rank, fabric.world, fabric.device
        self.route, self.optimizer, self.graph, self.config = route, optimizer, graph, config
        self.kind = optimizer.kind
        self.nslots = _optim.NUM_SLOTS[self.kind]
        self.V, self.D = int(weight.shape[0]), int(weight.shape[1])
        self.Dp = (self.D + 3) // 4 * 4
        self.D4 = self.Dp // 4
        self.replicated = route.sparse == modes.SPARSE_ALLGATHER
        self.layout = TableLayout(self.V, num_partitions, self.world, strategy,
                                  replicated=self.replicated, owners=owners)
        self.average = bool(config.average_sparse)
        ps = config.communication_config.ps_config
        self.local_aggregation = bool(ps.local_aggregation)
        self.scale = graph.scale_for(name)
        # PSConfig.boundary_between_workers_and_servers (graph_transform_lib.py:1315-1370):
        # True  — post-processing that does not grow the data (ScaleGradients) runs on the
        #         sender, the widening bf16→fp32 cast on the owner: bf16 on the wire;
        # False — nothing is moved: rows are widened to fp32 by the sender and the scale
        #         runs on the owner.
        self.boundary = bool(ps.boundary_between_workers_and_servers)
        opts = options or {}
        self.options = opts
        self.out_dtype = out_dtype or torch.float32
        self.anchor_device = self.device
        self.capacity_hint = (opts.get("sparse_capacity") or {}).get(name)
        self.weight_dtype = _optim.sparse_weight_dtype(opts.get("sparse_weights", "fp32"))
        if self.weight_dtype == torch.bfloat16 and self.out_dtype != torch.bfloat16:
            raise ValueError(
                "sparse variable %r: sparse_weights='bf16' needs bf16 lookups "
                "(compute_dtype='bf16'): the lookup kernel copies bf16 rows into bf16 outputs"
                % name)
        self.sr_seed = _optim.sr_seed(name)
        L = self.layout
        rows = L.rows_local
        heap = self.heap
        self.Dps = (self.D4 + 1) // 2 * 8          # shadow row length (16-byte vectors)
        if self.weight_dtype == torch.bfloat16:
            # bf16 master rows in the shadow's layout: lookups and the full-softmax evaluation
            # read them through the shadow descriptors; the owner kernel rounds every update
            # stochastically.  No fp32 copy exists.
            self.tab_buf = heap.alloc(rows * self.Dps * 2, "table:" + name)
            self.table = self.tab_buf.tensor(torch.bfloat16, rows * self.Dps) \
                .view(rows, self.Dps)
            self.table.zero_()
            self.shadow = None
            self._init_weights(weight, init)
        else:
            self.tab_buf = heap.alloc(rows * self.Dp * 4, "table:" + name)
            self.table = self.tab_buf.tensor(torch.float32, rows * self.Dp).view(rows, self.Dp)
        # a row-wise rule keeps one fp32 per row: a dense [rows_local] array (the kernels
        # address it with a 4-byte pitch); every other rule keeps padded rows like the table
        self.slot_dim = _optim.slot_width(self.kind, self.D)
        slot_cols = _optim.slot_width(self.kind, self.Dp)
        self.slot_bufs, self.slots = [], []
        for v in optimizer.slot_init():
            sb = heap.alloc(rows * slot_cols * 4, "slot:" + name)
            t = sb.tensor(torch.float32, rows * slot_cols).view(rows, slot_cols)
            t.fill_(v)
            self.slot_bufs.append(sb)
            self.slots.append(t)
        # bf16 shadow rows for bf16 models: lookups move half the bytes over NVLink / HBM;
        # the owner kernel refreshes the shadow row together with the fp32 master row.  A
        # bf16 master is its own shadow (`sparse_shadow` has no effect).
        want = opts.get("sparse_shadow", "auto")
        if self.weight_dtype == torch.bfloat16:
            self.use_shadow = True
            self.shadow_buf, self.shadow = self.tab_buf, self.table
        else:
            self.shadow_buf = self.shadow = None
            self.use_shadow = (self.out_dtype == torch.bfloat16 and bool(want) and
                               (want is True or rows * self.Dps * 2 <= (16 << 30)))
            if self.use_shadow:
                self.shadow_buf = heap.alloc(rows * self.Dps * 2, "shadow:" + name)
                self.shadow = self.shadow_buf.tensor(torch.bfloat16, rows * self.Dps) \
                    .view(rows, self.Dps)
            self._init_weights(weight, init)
        self._ptrs = {}
        self.ring_buf = None
        self.staging = None
        self.group = None
        self.stats = {"pushed_rows": 0, "steps": 0}
        if auto_group:
            NVSparseGroup([self])

    # ------------------------------------------------------------- storage
    def _init_weights(self, weight, init):
        L = self.layout
        if weight.device.type == "meta":
            # lazy: initialise only this owner's rows on the device
            gen = torch.Generator(device=self.device)
            gen.manual_seed(int(init["seed"]) * 1000003 + (0 if self.replicated
                                                           else self.rank))
            if self.weight_dtype == torch.bfloat16:
                # the fp32 initialisation, rounded to nearest even (runs before the slots
                # are allocated, and returns its fp32 scratch to the device)
                w = torch.empty(self.table.shape[0], self.Dp, device=self.device)
                w[:, :self.D].uniform_(-init["scale"], init["scale"], generator=gen)
                self.table[:, :self.D] = w[:, :self.D]
                del w
                torch.cuda.empty_cache()
                return
            self.table[:, :self.D].uniform_(-init["scale"], init["scale"], generator=gen)
            if self.Dp != self.D:
                self.table[:, self.D:].zero_()
        else:
            w = weight.detach().to(torch.float32)
            for g, l in L.owner_chunks(0 if self.replicated else self.rank):
                self.table[l.to(self.device), :self.D] = w[g].to(self.device, self.table.dtype)
        self.refresh_shadow()

    def refresh_shadow(self):
        if self.shadow is not None and self.shadow is not self.table:
            self.shadow.zero_()
            self.shadow[:, :self.Dp].copy_(self.table)

    def dev_ptrs(self, what):
        """Device array of every rank's pointer for `what` (built lazily: in a simulated
        world the peers allocate after us)."""
        t = self._ptrs.get(what)
        if t is None:
            if what == "table":
                buf = self.tab_buf
            elif what == "shadow":
                buf = self.shadow_buf
            elif what == "ring":
                buf = self.ring_buf
            else:
                buf = self.slot_bufs[int(what[4:])]
            if self.replicated and what != "ring":
                # every replica reads and updates its own full copy
                t = torch.tensor([buf.local_ptr] * self.world, dtype=torch.int64,
                                 device=self.device)
            else:
                t = buf.dev_ptrs()
            self._ptrs[what] = t
        return t

    # ------------------------------------------------- per-table facade (group of 1..)
    def lookup(self, flat_ids, record=True):
        if record and len(self.group.tables) > 1:
            raise RuntimeError(
                "table %r belongs to the co-lookup group %s: training lookups must go "
                "through parallax.nn.lookup_many()" % (self.name, self.group.name))
        outs, pend = self.group.lookup(flat_ids, record=record,
                                       members=[self] if not record else None)
        return outs[0], pend

    def add_pending(self, token, grad_rows):
        self.group.add_pending(token, [grad_rows])

    def begin_step(self, step):
        self.group.begin_step(step)

    def finish_step(self, step, stream=None):
        self.group.finish_step(step, stream)

    def stage_push(self, step, stream=None):
        self.group.stage_push(step, stream)

    def stage_apply(self, step, stream=None):
        self.group.stage_apply(step, stream)

    def warm(self, n):
        self.group.warm(n)

    def _ensure_capacity(self, n):
        self.group._ensure_capacity(n)

    @property
    def cap(self):
        return self.group.cap

    # -------------------------------------------------------------- checkpoint
    def _width(self, what):
        """Logical columns of "weight" (D) or of slot `what` (D, or 1 for a row-wise rule)."""
        return self.D if what == "weight" else self.slot_dim

    def local_rows(self, what="weight"):
        """(global ids, rows [n, D] — [n, 1] for a row-wise slot) of the real rows this rank
        owns — the unit of a sharded checkpoint (no cross-rank traffic)."""
        src = self.table if what == "weight" else self.slots[int(what)]
        d = self._width(what)
        gs, rows = [], []
        for g, l in self.layout.owner_chunks(0 if self.replicated else self.rank):
            gs.append(g)
            rows.append(src[l.to(self.device), :d].cpu())
        if not gs:
            return torch.zeros(0, dtype=torch.int64), torch.zeros(0, d, dtype=src.dtype)
        return torch.cat(gs), torch.cat(rows)

    def _gather_full(self, local, d):
        L, W = self.layout, self.world
        local = local[:, :d].contiguous()
        out = torch.zeros(self.V, d)
        if self.replicated or W == 1:
            g, l = L.global_ids_of_owner(0 if self.replicated else self.rank)
            out[g] = local.cpu()[l].float()
            return out
        shards = self.comm.all_gather_tensors(local)
        for o in range(W):
            g, l = L.global_ids_of_owner(o)
            out[g] = shards[o].cpu()[l].float()
        return out

    def full_weight(self):
        torch.cuda.synchronize(self.device)
        return self._gather_full(self.table, self.D)

    def full_slots(self):
        torch.cuda.synchronize(self.device)
        return [self._gather_full(s, self.slot_dim) for s in self.slots]

    def load_full(self, weight, slots=None):
        if slots is not None:
            _optim.check_table_slots(self.name, self.kind, self.V, self.D, slots)
        for g, l in self.layout.owner_chunks(0 if self.replicated else self.rank):
            l = l.to(self.device)
            self.table[l, :self.D] = weight.float()[g].to(self.device, self.table.dtype)
            if slots is not None:
                for s, full in zip(self.slots, slots):
                    s[l, :self.slot_dim] = full.float()[g].to(self.device)
        self.refresh_shadow()
        torch.cuda.synchronize(self.device)

    def load_rows(self, ids, rows, what="weight"):
        """Scatter (global id, row) pairs into this rank's shard; ids owned by other
        ranks are ignored (sharded-checkpoint restore, any source layout)."""
        d = self._width(what)
        if rows.dim() != 2 or int(rows.shape[1]) != d:
            raise ValueError("sparse variable %r: %s rows of shape %s, want [n, %d]"
                             % (self.name, what, tuple(rows.shape), d))
        L = self.layout
        ids = ids.to(torch.int64)
        own = torch.ones_like(ids, dtype=torch.bool) if self.replicated else \
            (L.owner_of(ids) == self.rank)
        if own.any():
            l = L.local_row_of(ids[own]).to(self.device)
            dst = self.table if what == "weight" else self.slots[int(what)]
            dst[l, :d] = rows[own].float().to(self.device, dst.dtype)

    def release(self):
        """Free this table's symmetric segments (collective)."""
        torch.cuda.synchronize(self.device)
        if self.comm.distributed:
            self.comm.barrier()
        if self.group is not None:
            self.group.release_shared()
        shadow = self.shadow_buf if self.shadow_buf is not self.tab_buf else None
        for b in [self.tab_buf, shadow, self.ring_buf] + list(self.slot_bufs):
            if b is not None:
                self.heap.free(b)
        self.table = self.shadow = None
        self.slots = []


class NVSparseGroup(object):
    """Tables with one placement that are looked up with the same ids."""
    _seq = 0

    def __init__(self, tables, name=None):
        abi = ops.sparse_abi()
        gmax = abi["group_max"]
        if not 1 <= len(tables) <= gmax:
            raise ValueError("a co-lookup group holds 1..%d tables" % gmax)
        t0 = tables[0]
        for t in tables[1:]:
            if not t.layout.same_placement(t0.layout):
                raise ValueError(
                    "co-lookup group: %r and %r differ in rows / partitions / strategy / "
                    "owner placement" % (t0.name, t.name))
            if _optim.kind_family(t.kind) != _optim.kind_family(t0.kind):
                raise ValueError("co-lookup group mixes optimizer families")
        self.tables = list(tables)
        self.name = name or "+".join(t.name for t in tables)
        for t in tables:
            t.group = self
        self.fabric, self.heap, self.comm = t0.fabric, t0.heap, t0.comm
        self.rank, self.world, self.device = t0.rank, t0.world, t0.device
        self.route, self.layout = t0.route, t0.layout
        self.replicated = t0.replicated
        self.local_aggregation = t0.local_aggregation
        self.boundary = t0.boundary
        opts = t0.options
        # PSConfig.protocol == "nccl": the in-engine library baseline — same engine, same
        # kernels for the optimizer, but every byte that crosses GPUs goes through NCCL
        # collectives (Horovod's IndexedSlices path: all-gather of ids and rows)
        self.protocol = opts.get("_protocol", "nvlink")
        self.max_blocks = int(opts.get("sparse_blocks", consts.NUM_SMS * 2))
        self.early_push = bool(opts.get("sparse_early_push", True))
        # sess_config["micro_batches"] = K: the rows of all K micro-batches of a step are
        # pushed together, after the last one's backward, and weighted 1/K on the owner
        self.micro_batches = int(opts.get("micro_batches", 1))
        self._last_mb = True
        # sess_config["full_softmax_train"]: "fused" trains `parallax.nn.full_softmax_nll` over
        # this (weight, bias) group with `full_softmax_nll_lse` / `full_softmax_nll_grad`
        self.full_softmax_train = opts.get("full_softmax_train", "composition")
        self._all_ids = None
        hints = [t.capacity_hint for t in tables if t.capacity_hint]
        self.capacity_hint = max(hints) if hints else None
        self.hp = hp_stage(self.fabric, t0.optimizer)
        lay = self.layout
        self._owners_dev = torch.tensor(lay.owners, dtype=torch.int32, device=self.device)
        self._slots_dev = torch.tensor(lay.slots, dtype=torch.int32, device=self.device)
        g = ops.GroupGeom()
        g.V, g.P, g.W, g.rows_per_part = lay.V, lay.P, lay.world, lay.rows_per_part
        g.strategy = 0 if lay.strategy == "mod" else 1
        g.replicated = 1 if lay.replicated else 0
        g.extras, g.base = getattr(lay, "_extras", 0), getattr(lay, "_base", 0)
        g.part_owner = self._owners_dev.data_ptr()
        g.part_slot = self._slots_dev.data_ptr()
        self.geom = g
        # the partition held in each of my slots (-1: none): a bf16 master's owner kernel keys
        # its stochastic rounding by global row ids
        slot_part = [-1] * max(lay.parts_per_owner, 1)
        for p_ in range(lay.P):
            if not lay.replicated and lay.owners[p_] == self.rank:
                slot_part[lay.slots[p_]] = p_
        self._slot_part_dev = torch.tensor(slot_part, dtype=torch.int32, device=self.device)
        if len({t.weight_dtype for t in tables}) != 1:
            raise ValueError("co-lookup group %s mixes fp32 and bf16 master rows" % self.name)
        self.ctl = torch.zeros(abi["ctl_bytes"] // 4, dtype=torch.int32, device=self.device)
        self.hdr_buf = self.heap.alloc(abi["hdr_words"] * 4, "hdr:" + self.name)
        self.ids_buf = None
        self.slotmap = torch.full((lay.rows_local,), -1, dtype=torch.int32,
                                  device=self.device)
        self.next = None
        self.cap = 0
        self.scratch_n = 0
        self.wire_dtype = None
        self._hdrs_dev = self._ids_dev = None
        self.calls = []            # (pend ids, [grad rows per table]) per lookup this step
        self._fwd_calls = self._bwd_calls = 0
        self._cur_step = 0
        self._done_step = -1
        self._last_n = 1
        self._slots = None
        # ClipByGlobalNorm(include_sparse=True): (dense group, clip state) of the rule this
        # group contributes to, and the group's private hyper-parameters for the clipped apply
        self.joint_clip = None
        self.hp_clip = None
        NVSparseGroup._seq += 1

    # ---------------------------------------------------------------- forward
    # ------------------------------------------------- library-collective (NCCL) arm
    def _nccl(self):
        return (self.protocol == "nccl" and self.world > 1 and self.comm.distributed and
                self.route.sync)

    def _place(self, ids):
        """(valid, owner, local row) of global ids from the device-resident maps (`owner_of` /
        `local_row_of` of TableLayout copy host maps over: illegal in a CUDA-graph capture)."""
        lay = self.layout
        valid = (ids >= 0) & (ids < lay.V)
        idc = ids.clamp(0, lay.V - 1).to(torch.int64)
        if lay.replicated:
            return valid, torch.zeros_like(idc), idc
        p = lay.partition_of(idc)
        owner = self._owners_dev[p].to(torch.int64)
        local = self._slots_dev[p].to(torch.int64) * lay.rows_per_part + \
            lay.index_in_partition(idc)
        return valid, owner, local

    def _lookup_nccl(self, members, ids, n, record):
        import torch.distributed as dist
        W, grp = self.world, self.comm.group
        ids64 = ids.to(torch.int64)
        all_ids = torch.empty(W * n, dtype=torch.int64, device=self.device)
        dist.all_gather_into_tensor(all_ids, ids64, group=grp)
        valid, owner, local = self._place(all_ids)
        mine = valid & (owner == self.rank)
        rows = torch.where(mine, local, torch.zeros_like(local))
        outs = []
        for t in members:
            src = t.shadow[:, :t.Dp] if t.use_shadow else t.table
            part = src.index_select(0, rows).to(t.out_dtype) * mine[:, None].to(t.out_dtype)
            out = torch.empty(n, t.Dp, dtype=t.out_dtype, device=self.device)
            dist.reduce_scatter_tensor(out, part, group=grp)
            outs.append(out if t.Dp == t.D else out[:, :t.D])
        pend = None
        if record:
            v0, _, _ = self._place(ids64)
            pend = torch.where(v0, ids64, torch.full_like(ids64, -1)).to(torch.int32)
            self._fwd_calls += 1
        _count()
        return outs, pend

    def _push_apply_nccl(self, pend_ids, grads, n, cs):
        """all-gather (ids, rows) from every rank, then the owner kernel applies the rows
        this rank owns (entries of other owners are marked -1)."""
        import torch.distributed as dist
        W, grp = self.world, self.comm.group
        with torch.cuda.stream(cs):
            all_ids = torch.empty(W * n, dtype=torch.int32, device=self.device)
            dist.all_gather_into_tensor(all_ids, pend_ids, group=grp)
            valid, owner, local = self._place(all_ids.to(torch.int64))
            mine = valid if self.replicated else (valid & (owner == self.rank))
            ring_ids = torch.where(mine, local, torch.full_like(local, -1)).to(torch.int32)
            nxt = torch.empty(W * n, dtype=torch.int32, device=self.device)
            all_gs = []
            for t, g in zip(self.tables, grads):
                all_g = torch.empty(W * n, t.Dp, dtype=g.dtype, device=self.device)
                dist.all_gather_into_tensor(all_g, g, group=grp)
                all_gs.append(all_g)
            # the rows travel unscaled through all_gather: the owner applies the scale
            descs = self._owner_tables([g.data_ptr() for g in all_gs], sender_scaled=False)
            keep = [all_ids, ring_ids, nxt] + all_gs
            if not torch.cuda.is_current_stream_capturing():
                for k_ in keep:
                    k_.record_stream(cs)
            self._keep_n = (keep, descs)
            blocks = max(1, min(self.max_blocks, (n * W + 7) // 8))
            _count()
            ops.check(ops.lib().px_sparse_owner(
                descs, len(self.tables), _DT[grads[0].dtype], _vp(ring_ids.data_ptr()),
                _vp(self.hdr_buf.local_ptr), _vp(self.hdrs_dev.data_ptr()),
                _vp(self.slotmap.data_ptr()), _vp(nxt.data_ptr()), n,
                ctypes.byref(self.geom), _vp(self.ctl.data_ptr()), self.rank, 1, blocks, n,
                _sp(cs)), "sparse_owner(nccl)")

    @property
    def _wait(self):
        """1: lookups and the eval first wait for every owner's `applied` flag (sync NVLink)."""
        return 1 if (self.route.sync and self.world > 1 and not self._nccl()) else 0

    def lookup(self, flat_ids, record=True, members=None):
        members = self.tables if members is None else members
        n = int(flat_ids.numel())
        ids = flat_ids if flat_ids.is_cuda else flat_ids.to(self.device, non_blocking=True)
        if ids.dtype not in (torch.int64, torch.int32):
            ids = ids.to(torch.int64)
        ids = ids.contiguous()
        if self._nccl() and not self.replicated and n > 0:
            return self._lookup_nccl(members, ids, n, record)
        descs, outs = (ops.LookupTable * len(members))(), []
        for i, t in enumerate(members):
            # a table with a shadow has bf16 outputs: rows are copied at the shadow's width
            out = torch.empty((n, t.Dps if t.use_shadow else t.Dp), dtype=t.out_dtype,
                              device=self.device)
            descs[i] = _lookup_table(t, "shadow" if t.use_shadow else "table", out)
            outs.append(out if out.shape[1] == t.D else out[:, :t.D])
        pend = torch.empty(n, dtype=torch.int32, device=self.device) if record else None
        if record:
            self._fwd_calls += 1
        if n > 0:
            _count()
            ops.check(ops.lib().px_sparse_lookup(
                _vp(ids.data_ptr()), 1 if ids.dtype == torch.int64 else 0, n, descs,
                len(members), _vp(pend.data_ptr()) if pend is not None else _vp(0),
                ctypes.byref(self.geom), _vp(self.hdr_buf.local_ptr),
                _vp(self.ctl.data_ptr()), self._wait,
                _sp(torch.cuda.current_stream(self.device))), "sparse_lookup")
        return outs, pend

    # ------------------------------------------------------------- evaluation
    def _slot_maps(self):
        """(row counts, partition index), int32 [owners, slots] on the device, built once per
        layout: the real rows of the partition held in each (owner, slot) of the layout (the
        rest of a slot is padding), and that partition (-1: none), from which the top-k kernel
        recovers global row ids.  A replicated layout is one partition: owners = 1, [[0]]."""
        lay = self.layout
        if self._slots is None or self._slots[0] is not lay:
            shape = (1 if lay.replicated else lay.world, lay.parts_per_owner)
            cnt = torch.zeros(shape, dtype=torch.int32)
            part = torch.full(shape, -1, dtype=torch.int32)
            for p in range(lay.P):
                o = 0 if lay.replicated else lay.owners[p]
                cnt[o, lay.slots[p]] = lay.partition_rows(p)
                part[o, lay.slots[p]] = p
            self._slots = (lay, cnt.to(self.device), part.to(self.device))
        return self._slots[1:]

    def _eval_operands(self, x, what):
        """Checks the inputs of the eval entry point `what` and returns what
        px_full_softmax_nll, px_full_softmax_topk and px_full_softmax_sample share: (x, K,
        (bias source, bias pitch), head, tail, stream).  head is their ctypes arguments from the
        weight shadow pointers through the row counts, tail those from the slot count through
        `wait`; the top-k and sampling kernels take their partition index between the two.  The
        bias rows are the master rows: fp32, or bf16 rows of the shadow's layout with bf16
        masters (widened where they are added)."""
        tw, tb = self.tables
        if not tw.use_shadow or tb.D != 1 or x.dim() != 2 or x.shape[1] != tw.D or \
                x.dtype != torch.bfloat16:
            raise ValueError("%s needs bf16 inputs [N, %d], a weight table with a bf16 shadow "
                             "and a bias table of width 1" % (what, tw.D))
        x = x.contiguous()
        if x.data_ptr() % 16:                      # TMA needs a 16-byte aligned base
            x = x.clone()
        b_bf16 = tb.weight_dtype == torch.bfloat16
        b_src, b_pitch = ("shadow", tb.Dps) if b_bf16 else ("table", tb.Dp)
        cnt, _ = self._slot_maps()
        head = (_vp(tw.dev_ptrs("shadow").data_ptr()), tw.Dps, _vp(tb.dev_ptrs(b_src).data_ptr()),
                b_pitch, int(b_bf16), _vp(cnt.data_ptr()))
        tail = (int(cnt.shape[1]), ctypes.byref(self.geom), self.rank,
                _vp(self.hdr_buf.local_ptr), _vp(self.ctl.data_ptr()), self._wait)
        return (x, int(x.shape[1]), (b_src, b_pitch), head, tail,
                _sp(torch.cuda.current_stream(self.device)))

    def full_softmax_nll(self, x, targets):
        """Per-row full-softmax NLL, fp32 [N], of bf16 inputs `x` [N, K] against this
        group's (weight, bias) tables: ``cross_entropy(x @ W.T + b, targets)`` with fp32
        logits, computed from the rows where their owners store them — no gather of the
        table and no [N, V] logits (`ops/csrc/kernels/softmax_eval.cu`).  The targets' rows
        come from one launch of the group's lookup kernel.  A target outside [0, V) gives
        NaN in its row.  One-sided: no other rank takes part."""
        return self._nll(x, targets, False)[0]

    def full_softmax_nll_lse(self, x, targets):
        """``(nll, lse)``, fp32 [N] each: `full_softmax_nll` and each row's log-sum-exp, which
        the backward (`full_softmax_nll_grad`) takes."""
        return self._nll(x, targets, True)

    def _nll(self, x, targets, want_lse):
        L = ops.lib()
        tw, tb = self.tables
        x, K, (b_src, b_pitch), head, tail, stream = self._eval_operands(x, "full_softmax_nll")
        n = int(x.shape[0])
        out = torch.empty(n, dtype=torch.float32, device=self.device)
        lse = torch.empty(n, dtype=torch.float32, device=self.device) if want_lse else None
        if n == 0:
            return out, lse
        ids = targets.reshape(-1).to(self.device, torch.int64).contiguous()
        # target bias from the master rows like every bias row the eval kernel reads
        w_t = torch.empty((n, tw.Dps), dtype=torch.bfloat16, device=self.device)
        b_t = torch.empty((n, b_pitch), dtype=tb.weight_dtype, device=self.device)
        descs = (ops.LookupTable * 2)(_lookup_table(tw, "shadow", w_t),
                                      _lookup_table(tb, b_src, b_t))
        _count()
        ops.check(L.px_sparse_lookup(
            _vp(ids.data_ptr()), 1, n, descs, 2, _vp(0), ctypes.byref(self.geom),
            _vp(self.hdr_buf.local_ptr), _vp(self.ctl.data_ptr()), self._wait, stream),
            "sparse_lookup(full softmax targets)")
        ws = torch.empty(consts.NUM_SMS * n * 2, dtype=torch.float32, device=self.device)
        _count(2)
        ops.check(L.px_full_softmax_nll(
            _vp(x.data_ptr()), n, K, *head, *tail, _vp(ws.data_ptr()), consts.NUM_SMS,
            _vp(ids.data_ptr()), _vp(w_t.data_ptr()), _vp(b_t.data_ptr()),
            _vp(out.data_ptr()), _vp(lse.data_ptr() if want_lse else 0), stream),
            "full_softmax_nll")
        return out, lse

    def _all_rows(self):
        """int32 [V]: every global id of the group, allocated once."""
        if self._all_ids is None:
            self._all_ids = torch.arange(self.tables[0].V, dtype=torch.int32, device=self.device)
        return self._all_ids

    def record_all_rows(self):
        """Counts one forward call whose gradient rows are every row of the group, in global
        id order, without a lookup, and returns its token (the fused full-softmax training
        forward; its backward hands the rows to `add_pending` like a lookup's)."""
        self._fwd_calls += 1
        return self._all_rows()

    def full_softmax_train_chunk(self, n):
        """Rows of one vocabulary chunk of `full_softmax_nll_grad` for n input rows: the
        chunk's gathered rows and its bf16 [n, Vc] softmax gradient fit in
        `consts.FULL_SOFTMAX_TRAIN_WS_BYTES`; a multiple of BV · NUM_SMS where that fits
        (whole waves of the gradient kernel's blocks of BV = `full_softmax_block_rows(K)`
        rows), else of BV."""
        tw, tb = self.tables
        b_bytes = tb.Dps * 2 if tb.weight_dtype == torch.bfloat16 else tb.Dp * 4
        rows = consts.FULL_SOFTMAX_TRAIN_WS_BYTES // (2 * n + 2 * tw.Dps + b_bytes)
        bv = full_softmax_block_rows(tw.D)
        wave = bv * consts.NUM_SMS
        vc = rows // wave * wave if rows >= wave else max(bv, rows // bv * bv)
        return min(vc, (tw.V + bv - 1) // bv * bv)

    def full_softmax_nll_grad(self, x, targets, lse, g, want_x=True, want_tables=True,
                              chunk=None):
        """Backward of `full_softmax_nll_lse` for the gradient `g` [N] of the NLL: ``(dx,
        dW, db)`` with dx [N, K] in `x`'s dtype and the table gradient as every row in
        global id order, dW [V, K] and db [V, 1] in the tables' lookup dtypes (what
        `add_pending` takes); None for what is not wanted.  Over vocabulary chunks of
        `chunk` rows (default `full_softmax_train_chunk`): one lookup launch gathers the
        chunk's rows, the gradient kernel recomputes its logits and writes G = g · (softmax −
        onehot) in bf16 and db, then dx += G·W_c (fp32) and dW_c = Gᵀ·x.  One-sided: no other
        rank takes part."""
        L = ops.lib()
        tw, tb = self.tables
        x, K, (b_src, b_pitch), _, _, stream = self._eval_operands(x, "full_softmax_nll_grad")
        n, V, dev = int(x.shape[0]), tw.V, self.device
        dx = torch.zeros(n, K, dtype=torch.float32, device=dev) if want_x else None
        dW = torch.empty(V, K, dtype=torch.bfloat16, device=dev) if want_tables else None
        db = torch.zeros(V, dtype=torch.float32, device=dev)
        if n > 0:
            ids = targets.reshape(-1).to(dev, torch.int64).contiguous()
            lse = lse.to(dev, torch.float32).contiguous()
            g = g.reshape(-1).to(dev, torch.float32).contiguous()
            vc = int(chunk) if chunk else self.full_softmax_train_chunk(n)
            bv = full_softmax_block_rows(K)
            gp = (vc + bv - 1) // bv * bv                  # >= the chunk's blocks · BV, even
            wc = torch.empty((vc, tw.Dps), dtype=torch.bfloat16, device=dev)
            bc = torch.empty((vc, b_pitch), dtype=tb.weight_dtype, device=dev)
            G = torch.empty((n, gp), dtype=torch.bfloat16, device=dev)
            all_ids = self._all_rows()
            descs = (ops.LookupTable * 2)(_lookup_table(tw, "shadow", wc),
                                          _lookup_table(tb, b_src, bc))
            for v0 in range(0, V, vc):
                m = min(vc, V - v0)
                _count(2)
                ops.check(L.px_sparse_lookup(
                    _vp(all_ids[v0:].data_ptr()), 0, m, descs, 2, _vp(0),
                    ctypes.byref(self.geom), _vp(self.hdr_buf.local_ptr),
                    _vp(self.ctl.data_ptr()), self._wait, stream),
                    "sparse_lookup(full softmax chunk)")
                ops.check(L.px_full_softmax_grad(
                    _vp(x.data_ptr()), n, K, _vp(wc.data_ptr()), tw.Dps, _vp(bc.data_ptr()),
                    b_pitch, int(tb.weight_dtype == torch.bfloat16), m, v0,
                    _vp(lse.data_ptr()), _vp(g.data_ptr()), _vp(ids.data_ptr()),
                    _vp(G.data_ptr()), gp, _vp(db[v0:].data_ptr()), consts.NUM_SMS, stream),
                    "full_softmax_grad")
                Gc = G[:, :m]
                if want_x:
                    dx.add_(torch.mm(Gc, wc[:m, :K], out_dtype=torch.float32))
                if want_tables:
                    torch.mm(Gc.t(), x, out=dW[v0:v0 + m])
        if want_x:
            dx = dx.to(x.dtype)
        if not want_tables:
            return dx, None, None
        return dx, dW.to(tw.out_dtype), db.to(tb.out_dtype)[:, None]

    def full_softmax_topk(self, x, k):
        """The k largest full-softmax logits of each row of bf16 inputs `x` [N, K] against
        this group's (weight, bias) tables: ``(log_probs fp32 [N, k], ids int64 [N, k])``, logit
        descending and equal logits by ascending id, with fp32 logits computed from the rows
        where their owners store them (`ops/csrc/kernels/softmax_eval.cu`).  1 <= k <= 32.
        Scratch is per call and O(NUM_SMS · rows · k): rows are taken in chunks so that the
        per-CTA lists fit in `consts.TOPK_WS_BYTES`.  One-sided: no other rank takes part."""
        return self._ranked(x, k, "full_softmax_topk", "k")

    def full_softmax_sample(self, x, n, inv_tau, seed, top_k=None, top_p=None):
        """n draws without replacement from ``softmax((x @ W.T + b) · inv_tau)`` for each row
        of bf16 inputs `x` [N, K], in draw order: ``(log_probs fp32 [N, n], ids int64 [N, n])``,
        where log_probs are the tempered log-probabilities of the ids.  The kernel keeps the n
        largest Gumbel keys ``s − log E`` of each row (s the scaled fp32 logit, E the noise of
        (seed, row, id), `engine.sample_log_e`), so the draws depend on the seed, the row's
        index in `x` and the ids only.  1 <= n <= 32, inv_tau = fp32(1/τ) > 0, seed in
        [0, 2^32).  Chunked, one-sided and fresh as `full_softmax_topk`.

        `top_k` (an int in [n, V]) and `top_p` (a real in (0, 1]) truncate each row to T = {v :
        s_v >= θ*}, θ* the largest θ with count(θ) >= top_k or (mass(θ) >= top_p and count(θ)
        >= n) (`parallax.nn.full_softmax_sample`); the draws are the n best keys within T and
        log_probs stay those of the untruncated softmax.  Per row chunk: one log-sum-exp pass,
        32 / `consts.SAMPLE_RADIX_BITS` histogram passes that find θ*, and the sampling pass
        with keys below θ* dropped, each reading the table once."""
        trunc = None
        if top_k is not None or top_p is not None:
            V = self.tables[0].V
            if top_k is not None and (isinstance(top_k, bool) or not isinstance(top_k, int) or
                                      not n <= top_k <= V):
                raise ValueError("full_softmax_sample: top_k must be an int in [num_samples, "
                                 "%d], got %r" % (V, top_k))
            if top_p is not None and (isinstance(top_p, bool) or
                                      not isinstance(top_p, numbers.Real) or
                                      not 0.0 < top_p <= 1.0):
                raise ValueError("full_softmax_sample: top_p must be a real number in (0, 1], "
                                 "got %r" % (top_p,))
            trunc = (top_k or 0, 0.0 if top_p is None else float(top_p))
        return self._ranked(x, n, "full_softmax_sample", "num_samples", (inv_tau, seed), trunc)

    def _ranked(self, x, k, what, k_name, sample=None, trunc=None):
        """The list-keeping eval kernels: top-k (`sample` None) or sampling (`sample` =
        (inv_tau, seed)), truncated when `trunc` = (top_k or 0, top_p or 0), in row chunks
        whose per-CTA lists (and digit bins, which reuse their memory) fit in
        `consts.TOPK_WS_BYTES`."""
        L = ops.lib()
        V = self.tables[0].V
        if isinstance(k, bool) or not isinstance(k, int) or not 1 <= k <= min(32, V):
            raise ValueError("%s: %s must be an int in [1, %d], got %r"
                             % (what, k_name, min(32, V), k))
        x, K, _, head, tail, stream = self._eval_operands(x, what)
        n = int(x.shape[0])
        log_probs = torch.empty(n, k, dtype=torch.float32, device=self.device)
        ids = torch.empty(n, k, dtype=torch.int64, device=self.device)
        if n == 0:
            return log_probs, ids
        _, part = self._slot_maps()
        ctas = consts.NUM_SMS
        d = consts.SAMPLE_RADIX_BITS
        per_row = max(k, 1 << d) if trunc else k          # 8-byte entries per (CTA, row)
        chunk = max(128, consts.TOPK_WS_BYTES // (ctas * per_row * 8) // 128 * 128)
        chunk = min(chunk, n)
        ws = torch.empty(ctas * chunk * 2, dtype=torch.float32, device=self.device)
        tk = torch.empty(ctas * chunk * per_row * 2, dtype=torch.int32, device=self.device)
        rows = torch.empty(chunk * 4, dtype=torch.int32, device=self.device) if trunc else None
        for r0 in range(0, n, chunk):
            m = min(chunk, n - r0)
            args = (_vp(x[r0:].data_ptr()), m, K, *head, _vp(part.data_ptr()), *tail,
                    _vp(ws.data_ptr()), ctas, k, _vp(tk.data_ptr()),
                    _vp(log_probs[r0:].data_ptr()), _vp(ids[r0:].data_ptr()))
            _count(2)
            if sample is None:
                rc = L.px_full_softmax_topk(*args, stream)
            elif trunc is None:
                rc = L.px_full_softmax_sample(*args, sample[0], sample[1], r0, stream)
            else:
                # θ* of every row of the chunk (into `rows`), then the masked sampling pass
                common = (_vp(x[r0:].data_ptr()), m, K, *head, *tail)
                ops.check(L.px_full_softmax_sample_lse(
                    *common, _vp(ws.data_ptr()), ctas, sample[0], _vp(rows.data_ptr()), stream),
                    what)
                for lo in range(32 - d, -1, -d):
                    _count(2)
                    ops.check(L.px_full_softmax_radix(
                        *common, _vp(tk.data_ptr()), ctas, sample[0], _vp(rows.data_ptr()), lo,
                        trunc[0], trunc[1], k, stream), what)
                _count(2)
                rc = L.px_full_softmax_sample_masked(*args, sample[0], sample[1], r0,
                                                     _vp(rows.data_ptr()), stream)
            ops.check(rc, what)
        return log_probs, ids

    def add_pending(self, token, grads):
        gs = []
        for t, g in zip(self.tables, grads):
            g = g.reshape(-1, t.D)
            if t.Dp != t.D:
                g = torch.nn.functional.pad(g, (0, t.Dp - t.D))
            if g.dtype not in _DT:
                g = g.float()
            gs.append(g.contiguous())
        dts = {g.dtype for g in gs}
        if len(dts) > 1:
            gs = [g.float() for g in gs]
        self.calls.append((token, gs))
        self._bwd_calls += 1
        if self.early_push and self._bwd_calls == self._fwd_calls and self._cur_step > 0 \
                and self._last_mb and self.ring_ready():
            self._run_step(self._cur_step)

    def ring_ready(self):
        """Early push needs every lazy allocation done (first step runs at the end)."""
        if self._nccl():
            return True
        return self.scratch_n > 0 and (not self.route.sync or self.ids_buf is not None)

    # ----------------------------------------------------------------- capacity
    def _negotiated(self, n):
        """Largest per-rank row count of this step (Horovod negotiates allgather sizes on
        every cycle, `collective_operations.cc:80-90`).  With a `sparse_capacity` hint, in
        a simulated world or under stream capture nothing is exchanged."""
        if (not self.route.sync or self.world == 1 or not self.comm.distributed or
                self.capacity_hint or torch.cuda.is_current_stream_capturing()):
            return n
        return self.comm.all_reduce_max_int(n)

    def _ensure_capacity(self, n):
        dev = self.device
        if n > self.scratch_n:
            cap_n = max(int(n * 1.25) + 16, 64)
            for t in self.tables:
                # fp32 rows for ids carried by several positions (kept zero between steps
                # by the push kernel's flush pass)
                t.staging = torch.zeros(cap_n // 2 + 2, t.Dp, dtype=torch.float32, device=dev)
            self.scratch_n = cap_n
        if not self.route.sync:
            return
        m = self._negotiated(n)
        if self.ids_buf is not None and m <= self.cap:
            return
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError(
                "sparse group %s: %d gradient rows exceed the ring capacity %d inside a "
                "captured CUDA graph (shapes must be static under cuda_graph)" %
                (self.name, n, self.cap))
        want = int(self.capacity_hint or max(int(m * 1.5) + 16, 64))
        if self.capacity_hint and m > want:
            raise RuntimeError(
                "sparse group %s: %d gradient rows in one step exceed sess_config"
                "['sparse_capacity'] = %d" % (self.name, m, want))
        if self.ids_buf is not None:
            parallax_log.info("sparse group %s: growing receive rings %d -> %d rows/source",
                              self.name, self.cap, want)
            torch.cuda.synchronize(dev)
            if self.comm.distributed:
                self.comm.barrier()
            self.heap.free(self.ids_buf)
            for t in self.tables:
                self.heap.free(t.ring_buf)
                t._ptrs.pop("ring", None)
        self.cap = want
        W = self.world
        for t in self.tables:
            t.ring_buf = self.heap.alloc(W * self.cap * t.Dp * 4, "ring:" + t.name)
        self.ids_buf = self.heap.alloc(W * self.cap * 4, "ring_ids:" + self.name)
        self.next = torch.empty(W * self.cap, dtype=torch.int32, device=dev)
        self._ids_dev = None
        if self.comm.distributed:
            torch.cuda.synchronize(dev)
            self.comm.barrier()

    @property
    def hdrs_dev(self):
        if self._hdrs_dev is None:
            self._hdrs_dev = self.hdr_buf.dev_ptrs()
        return self._hdrs_dev

    @property
    def ids_dev(self):
        if self._ids_dev is None:
            self._ids_dev = self.ids_buf.dev_ptrs()
        return self._ids_dev

    def warm(self, n):
        """Allocate everything a step of `n` gradient rows needs (no lazy allocation /
        pointer upload will happen inside the step)."""
        self._ensure_capacity(n)
        for t in self.tables:
            t.dev_ptrs("table")
            for i in range(t.nslots):
                t.dev_ptrs("slot%d" % i)
            if t.use_shadow:
                t.dev_ptrs("shadow")
            if self.route.sync:
                t.dev_ptrs("ring")
        if self.route.sync:
            self.ids_dev, self.hdrs_dev

    # --------------------------------------------------------------------- step
    def begin_step(self, step):
        self.hp.upload(step)
        self._cur_step = step
        self._fwd_calls = self._bwd_calls = 0

    def micro_batch(self, k, K):
        """The engine runs micro-batch `k` of `K` of the step next: only the last one's
        backward may push."""
        self._last_mb = k == K - 1

    def finish_step(self, step, stream=None):
        if self._done_step == step and not self.calls:
            return                           # already pushed from the backward pass
        self._run_step(step, stream)

    def _run_step(self, step, stream=None):
        from ..utils import timeline
        self._done_step = step
        if self._nccl():
            cs = stream if stream is not None else self.fabric.comm_stream
            pend_ids, grads = self._take_calls()
            if pend_ids is None:
                raise RuntimeError("protocol='nccl': every rank must look the group %s up in "
                                   "every step (collective)" % self.name)
            cur = torch.cuda.current_stream(self.device)
            if cs is not cur:
                cs.wait_stream(cur)
            self._push_apply_nccl(pend_ids, grads, int(pend_ids.numel()), cs)
            return
        if timeline.enabled():
            cs = stream if stream is not None else self.fabric.comm_stream
            with timeline.activity(self.name, "SPARSE_PUSH_APPLY", gpu=True, stream=cs,
                                   args="rows=%d" % sum(c[0].numel() for c in self.calls)):
                self._push_then_apply(step, stream)
        else:
            self._push_then_apply(step, stream)

    def _push_then_apply(self, step, stream):
        self.stage_push(step, stream)
        if self.joint_clip is not None:
            # the apply waits for the rule's norm: the dense group issues it after the
            # rule's last contributor (`NVDenseGroup.contributed`)
            dense, st = self.joint_clip
            cs = stream if stream is not None else self.fabric.comm_stream
            self.stage_norm(st.local if self.norm_counts() else None, cs)
            dense.contributed(st, cs)
        elif self.route.sync:
            self.stage_apply(step, stream)

    def _take_calls(self):
        """Pending ids and per-table gradient rows of this step's lookups, concatenated,
        or (None, None) when there were none; the list starts empty again."""
        calls, self.calls = self.calls, []
        if len(calls) <= 1:
            return calls[0] if calls else (None, None)
        ids, grads = zip(*calls)
        return torch.cat(ids), [torch.cat(g) for g in zip(*grads)]

    def stage_push(self, step, stream=None):
        """Sender side, one kernel: local aggregation + push (or remote apply in async
        mode).  Separate from `stage_apply` so that a world simulated on one GPU can
        enqueue every rank's push before any rank's (spinning) owner kernel."""
        cs = stream if stream is not None else self.fabric.comm_stream
        pend_ids, grads = self._take_calls()
        if pend_ids is None:
            pend_ids = torch.empty(0, dtype=torch.int32, device=self.device)
            grads = [torch.empty((0, t.Dp), dtype=torch.float32, device=self.device)
                     for t in self.tables]
        n = int(pend_ids.numel())
        self._ensure_capacity(max(n, 1))
        self._last_n = n
        for t in self.tables:
            t.stats["pushed_rows"] += n
            t.stats["steps"] += 1
        gdt = grads[0].dtype
        sync = self.route.sync
        if sync:
            if self.wire_dtype is None:
                # fixed for the lifetime of the rings: bf16 gradients stay bf16 on the wire
                # when the boundary optimisation is on, everything else travels as fp32
                self.wire_dtype = torch.bfloat16 if (gdt == torch.bfloat16 and self.boundary) \
                    else torch.float32
            if self.wire_dtype == torch.bfloat16 and gdt != torch.bfloat16:
                grads = [g.to(torch.bfloat16) for g in grads]   # dtype changed mid-run
                gdt = torch.bfloat16
        cur = torch.cuda.current_stream(self.device)
        if cs is not cur:
            cs.wait_stream(cur)
            if not torch.cuda.is_current_stream_capturing():
                pend_ids.record_stream(cs)
                for g in grads:
                    g.record_stream(cs)
        descs = self._push_tables(grads, sync)
        self._keep = (pend_ids, grads, descs)
        _count()
        ops.check(ops.lib().px_sparse_push(
            _vp(pend_ids.data_ptr()), n, descs, len(self.tables), _DT[gdt],
            _DT[self.wire_dtype] if sync else 0, 0 if sync else 1,
            _vp(self.ids_dev.data_ptr()) if sync else _vp(0),
            _vp(self.hdrs_dev.data_ptr()) if sync else _vp(0), self.cap,
            ctypes.byref(self.geom), _vp(self.ctl.data_ptr()), self.rank,
            1 if self.local_aggregation else 0, self.max_blocks, _sp(cs)), "sparse_push")

    def _push_tables(self, grads, sync):
        """PushTable per member table, shipping gradient rows `grads[i]`: into every owner's
        receive ring (`sync`, ScaleGradients on the sender when the boundary optimisation is
        on), or through the optimizer onto every owner's table rows (async)."""
        descs = (ops.PushTable * len(self.tables))()
        for d, t, g in zip(descs, self.tables, grads):
            d.grads, d.staging = g.data_ptr(), t.staging.data_ptr()
            d.hp, d.D4, d.kind = self.hp.dev.data_ptr(), t.D4, _optim.KIND_ID[t.kind]
            if sync:
                d.rings = t.dev_ptrs("ring").data_ptr()
                d.scale = t.scale if self.boundary else 1.0
            else:
                d.tables = t.dev_ptrs("table").data_ptr()
                d.slot0s = t.dev_ptrs("slot0").data_ptr() if t.nslots > 0 else 0
                d.slot1s = t.dev_ptrs("slot1").data_ptr() if t.nslots > 1 else 0
                d.slot2s = t.dev_ptrs("slot2").data_ptr() if t.nslots > 2 else 0
                d.shadows = t.dev_ptrs("shadow").data_ptr() if t.use_shadow else 0
                d.scale = t.scale
        return descs

    def _owner_tables(self, rings, sender_scaled, hp=None):
        """OwnerTable per member table, merging the rows at device address rings[i]; the
        owner applies the ScaleGradients factor unless the sender did (`sender_scaled`).
        `hp`: the device hyper-parameter vector to use instead of the shared one."""
        hp_ptr = (hp if hp is not None else self.hp.dev).data_ptr()
        descs = (ops.OwnerTable * len(self.tables))()
        for d, t, ring in zip(descs, self.tables, rings):
            d.ring, d.table = ring, t.table.data_ptr()
            d.slot0 = t.slots[0].data_ptr() if t.nslots > 0 else 0
            d.slot1 = t.slots[1].data_ptr() if t.nslots > 1 else 0
            d.slot2 = t.slots[2].data_ptr() if t.nslots > 2 else 0
            bf16 = t.weight_dtype == torch.bfloat16
            d.shadow = t.shadow.data_ptr() if t.use_shadow and not bf16 else 0
            d.hp, d.D4, d.D, d.kind = hp_ptr, t.D4, t.D, _optim.KIND_ID[t.kind]
            d.w_bf16, d.seed, d.slot_part = int(bf16), t.sr_seed, self._slot_part_dev.data_ptr()
            avg = (1.0 / self.world) if t.average else 1.0
            if self.micro_batches > 1:
                avg /= self.micro_batches
            d.avg = avg if sender_scaled else avg * t.scale
        return descs

    def _owner_blocks(self):
        n = max(self._last_n, 1)
        # 16 half-warps per CTA, one entry per half-warp: as many CTAs as fit on the device at once
        # (4 per SM at 64 registers; the merge variant is a cooperative launch)
        return max(1, min(max(self.max_blocks, consts.NUM_SMS * 4)
                          if self.max_blocks >= consts.NUM_SMS
                          else self.max_blocks,
                          (n * (self.world if self.replicated else 1) + 15) // 16))

    def _use_merge(self):
        return self.world > 1 or not self.local_aggregation

    def stage_apply(self, step, stream=None, hp=None):
        """Owner side, one kernel: merge rows from all sources, apply the optimizer
        (with the hyper-parameter vector `hp` instead of the shared one when given)."""
        cs = stream if stream is not None else self.fabric.comm_stream
        blocks = self._owner_blocks()
        use_merge = self._use_merge()
        descs = self._owner_tables([t.ring_buf.local_ptr for t in self.tables],
                                   sender_scaled=self.boundary, hp=hp)
        self._keep_o = descs
        _count()
        ops.check(ops.lib().px_sparse_owner(
            descs, len(self.tables), _DT[self.wire_dtype], _vp(self.ids_buf.local_ptr),
            _vp(self.hdr_buf.local_ptr), _vp(self.hdrs_dev.data_ptr()),
            _vp(self.slotmap.data_ptr()), _vp(self.next.data_ptr()), self.cap,
            ctypes.byref(self.geom), _vp(self.ctl.data_ptr()), self.rank,
            1 if use_merge else 0, blocks, -1, _sp(cs)), "sparse_owner")

    def norm_counts(self):
        """Whether this rank's `stage_norm` adds to the global norm: every owner of a
        partitioned group, only rank 0 of a replicated one (every replica merges every row)."""
        return not self.replicated or self.rank == 0

    def stage_norm(self, sumsq, stream=None):
        """Owner side, after `stage_push` and before `stage_apply`: add to the fp32 device
        scalar `sumsq` the squared norm of the rows `stage_apply` will hand to the optimizer
        (merged over sources, × average × ScaleGradients × hp[HP_GSCALE]).  Nothing is
        launched when `sumsq` is None."""
        if sumsq is None:
            return
        cs = stream if stream is not None else self.fabric.comm_stream
        descs = self._owner_tables([t.ring_buf.local_ptr for t in self.tables],
                                   sender_scaled=self.boundary)
        self._keep_nrm = descs
        _count()
        ops.check(ops.lib().px_sparse_owner_norm(
            descs, len(self.tables), _DT[self.wire_dtype], _vp(self.ids_buf.local_ptr),
            _vp(self.hdr_buf.local_ptr), _vp(self.slotmap.data_ptr()),
            _vp(self.next.data_ptr()), self.cap, ctypes.byref(self.geom),
            _vp(self.ctl.data_ptr()), 1 if self._use_merge() else 0, self._owner_blocks(),
            _vp(sumsq.data_ptr()), _sp(cs)), "sparse_owner_norm")

    def clip_hp(self, scale, stream=None):
        """The group's private hyper-parameters for a clipped apply: the shared vector with
        hp[HP_GSCALE] × the device scalar `scale`."""
        from . import nvops
        nvops.clip_hp(self.hp.dev, scale, self.hp_clip,
                      stream if stream is not None else self.fabric.comm_stream)
        return self.hp_clip

    # ---------------------------------------------------------------- inspection
    def device_times(self):
        """%globaltimer stamps (ns) written by the last push / owner kernels:
        push start, pushed flag published, owner start, all sources arrived, applied
        published.  Valid under CUDA-graph replay (the kernels write them every run)."""
        off = ops.sparse_abi()["ctl_time_offset"]
        raw = self.ctl.view(torch.uint8)[off:off + 104].clone().view(torch.int64).tolist()
        d = dict(zip(("push_start", "pushed", "owner_start", "arrived", "applied"), raw))
        d["push_phases"] = raw[5:13]        # CTA 0 of the push kernel: end of each phase
        return d

    def overflow_count(self):
        off = ops.sparse_abi()["ctl_overflow_offset"]
        return int(self.ctl.view(torch.uint8)[off:off + 4].clone().view(torch.int32).item())

    def release_shared(self):
        for b in (self.hdr_buf, self.ids_buf):
            if b is not None:
                self.heap.free(b)
        self.hdr_buf = self.ids_buf = None
