"""NVLink fabric backend: the engine's production path on H100.

Dense variables → `NVDenseGroup` (buckets in symmetric memory, fused
reduce-scatter + optimizer + parameter all-gather kernel per bucket, launched
from autograd hooks on a dedicated comm stream so it overlaps backward).
Sparse variables → `nv_sparse.NVSparseTable` / `NVSparseGroup` (row-partitioned
shards in symmetric memory; remote-gather lookup; one push kernel and one owner
kernel per co-lookup group and step).

Static schedule: every kernel that synchronises with peers is issued on ONE
comm stream in an order fixed by the model (sparse groups when their last gradient
of the step arrives, dense buckets in index order, the last bucket after the sparse
groups) — identical on all ranks, so no cross-rank wait cycle
can form and no per-step negotiation is needed (what Horovod's coordinator
does every 5 ms tick, `horovod/common/operations.cc:1274-1590`).
"""
import ctypes
import math

import torch

from .. import consts, optim as _optim
from ..log import parallax_log
from ..ops import sinks as _sinks
from . import modes, nvops
from .layout import TableLayout, assign_owners
from .nv_sparse import NVSparseTable, NVSparseGroup, hp_stage     # noqa: F401 (re-export)
from .symmetric import (SymmetricHeap, IpcExchange, CH_COMM, CH_MAIN, CH_SMALL)

MODE_FUSED, MODE_REDUCE, MODE_UPDATE, MODE_ACCUMULATE = 0, 1, 2, 3
_ES = {torch.float32: 4, torch.bfloat16: 2}
# segments (tensors) of one layer-wise bucket: its [nseg, 2] fp32 sums must fit one half of the
# fabric's one-shot stage (2 × 64 KiB)
LW_MAX_SEGMENTS = 65536 // 8


class NVFabric(object):
    def __init__(self, comm, exchange=None, options=None):
        self.comm = comm
        self.device = comm.device
        self.rank, self.world = comm.rank, comm.world
        self.options = options or {}
        ex = exchange if exchange is not None else IpcExchange(comm)
        if exchange is None and comm.distributed:
            import socket
            hosts = set(comm.all_gather_object(socket.gethostname()))
            if len(hosts) > 1:
                raise RuntimeError(
                    "the NVLink fabric addresses peers through CUDA IPC / NVSwitch "
                    "multicast and therefore spans ONE NVLink domain (one HGX/DGX box); "
                    "this job spans hosts %s. Run one job per box, or use "
                    "sess_config={'fabric': 'library'} (same engine on torch.distributed/"
                    "NCCL collectives) across boxes."
                    % sorted(hosts))
        self.heap = SymmetricHeap(self.device, ex)
        self.comm_stream = torch.cuda.Stream(self.device, priority=-1)
        # double-buffered staging for the one-shot all-reduce (norms, scalars)
        self.small_stage = self.heap.alloc(2 * 65536, "oneshot_stage")
        self.max_blocks = int(self.options.get("comm_blocks", 32))
        # CTAs of the fused dense step: its barriers are rank-level, so the grid is not tied to
        # the barrier slots — one CTA of 512 threads per SM (at 110 registers more would run as
        # a second wave behind the first one's system-scope fence); an explicit comm_blocks
        # (tests simulating several ranks on one GPU need small grids) applies to it as well
        self.dense_blocks = int(self.options.get(
            "dense_blocks", self.options.get("comm_blocks", consts.NUM_SMS)))
        if isinstance(ex, IpcExchange):
            self.heap.pads_dev()        # eager: no lazy H2D inside a step
        if comm.distributed:
            comm.barrier()

    def close(self):
        torch.cuda.synchronize(self.device)
        if self.comm.distributed:
            self.comm.barrier()
        self.heap.close()


class _Bucket(object):
    pass


class NVDenseGroup(object):
    def __init__(self, named_params, optimizer, fabric, route, graph,
                 options=None, sparse_groups=()):
        self.fabric, self.route, self.graph = fabric, route, graph
        self.sparse_groups = list(sparse_groups)
        self.optimizer = optimizer
        self.heap = fabric.heap
        self.rank, self.world = fabric.rank, fabric.world
        self.device = fabric.device
        opts = options or {}
        self.options = opts
        # bucket size: sess_config["bucket_bytes"], else PARALLAX_FUSION_THRESHOLD (Horovod's
        # HOROVOD_FUSION_THRESHOLD, `operations.cc:1030`), else 32 MiB
        import os
        from .. import consts
        self.bucket_bytes = int(opts.get("bucket_bytes") or
                                os.environ.get(consts.PARALLAX_FUSION_THRESHOLD) or (32 << 20))
        self.update = opts.get("dense_update", "sharded")   # or "replicated"
        if not route.sync:
            self.update = "async"
        # PSConfig.protocol == "nccl": library fallback for the dense reduction
        # (the in-engine baseline); every other protocol value = NVLink kernels.
        self.protocol = opts.get("_protocol", "nvlink")
        if self.protocol == "nccl" and route.sync:
            self.update = "replicated"
        # PSConfig.replicate_variables (PS run option): True = owners push the
        # updated values into every mirror right after the update; False =
        # workers pull the owners' slices at the start of the next step.
        self.pull_mirrors = (route.run_option == "PS" and route.sync and
                             not opts.get("_replicate_variables", True) and
                             self.update == "sharded" and self.world > 1)
        self.names = [n for n, _ in named_params]
        self.params = [p for _, p in named_params]
        _optim.require_fused(optimizer.kind, "NVLink fabric")
        self.kind = optimizer.kind
        self.nslots = _optim.NUM_SLOTS[self.kind]
        # LARS / LAMB: every bucket reduces with MODE_REDUCE, then runs the norm pass, the
        # all-reduce of its per-tensor sums and the update pass (`_layerwise_update`)
        self.layerwise = self.kind in _optim.LAYERWISE_KINDS
        self.clip_rules = graph.clip_rules()
        self.ema_rule = graph.ema
        self.last_grad_norm = {}
        self._hp = hp_stage(fabric, optimizer)
        self.hp = self._hp.dev
        # the last bucket to launch is held back until the sparse groups of the step have
        # been pushed (`finish_step`): it becomes ready right when backward reaches the
        # embedding gradients, and must not sit in front of their push on the comm stream
        self.defer_last = bool(opts.get("dense_defer_last", True))
        # sess_config["micro_batches"] = K: micro-batch k < K-1 of a step reduces every bucket
        # into its fp32 accumulator `red` (MODE_ACCUMULATE); the last one runs the step's
        # usual kernels with the accumulator folded in.  Every gradient is weighted 1/(W·K).
        self.micro_batches = int(opts.get("micro_batches", 1))
        self._mb = 0
        self._build_buckets()
        self._install_hooks()
        self._next = 0
        self._clip_pending = {}

    # ---------------------------------------------------------------- build
    def _clip_index(self, name):
        for i, r in enumerate(self.clip_rules):
            if r.applies_to(name):
                return i
        return -1

    def _build_buckets(self):
        W = self.world
        open_b, buckets = {}, []
        for name, p in reversed(list(zip(self.names, self.params))):
            assert p.dtype in _ES, "unsupported parameter dtype %s" % p.dtype
            key = (p.dtype, self._clip_index(name))
            b = open_b.get(key)
            if b is None:
                b = _Bucket()
                b.dtype, b.clip = key
                b.items, b.n = [], 0
                open_b[key] = b
                buckets.append(b)
            vn = 16 // _ES[p.dtype]
            off = b.n
            b.items.append((name, p, off, p.numel()))
            b.n = off + (p.numel() + vn - 1) // vn * vn
            if b.n * _ES[p.dtype] >= self.bucket_bytes or \
                    (self.layerwise and len(b.items) >= LW_MAX_SEGMENTS):
                del open_b[key]
        self.buckets = buckets
        heap = self.heap
        # NVLS: bucket buffers bound to an NVSwitch multicast object, the fused
        # kernel then reduces with multimem.ld_reduce and broadcasts parameters
        # with multimem.st.  It pays off on large buckets across many GPUs and not at
        # 2 (tools/allreduce_sweep.py measures the crossover).  "auto" enables it on a
        # full 8-GPU box; `dense_nvls=True` forces it for 4..7.
        want = self.options.get("dense_nvls", "auto")
        self.nvls = False
        if W > 1 and self.update == "sharded" and not self.pull_mirrors and want:
            from . import multicast
            if want is True or (want == "auto" and W >= 8):
                try:
                    self.nvls = multicast.supported(self.fabric.comm)
                except Exception:
                    self.nvls = False
        for bi, b in enumerate(buckets):
            vn = 16 // _ES[b.dtype]
            quantum = W * vn * 32
            b.index = bi
            b.n = (b.n + quantum - 1) // quantum * quantum
            es = _ES[b.dtype]
            b.mc = False
            if self.nvls:
                from . import multicast
                try:
                    b.grad_buf = multicast.MulticastBuffer(self.fabric, b.n * es)
                    b.param_buf = multicast.MulticastBuffer(self.fabric, b.n * es)
                    b.mc = True
                except multicast.MulticastError as e:
                    # MulticastBuffer agrees on success/failure across ranks, so
                    # every rank takes this branch together
                    parallax_log.warning("NVLS unavailable (%s); using P2P kernels", e)
                    self.nvls = False
            if not b.mc:
                b.grad_buf = heap.alloc(b.n * es, "grad%d" % bi)
                b.param_buf = heap.alloc(b.n * es, "param%d" % bi)
            b.grad_flat = b.grad_buf.tensor(b.dtype, b.n)
            b.param_flat = b.param_buf.tensor(b.dtype, b.n)
            b.grad_views, b.scales = [], []
            with torch.no_grad():
                for name, p, off, numel in b.items:
                    b.param_flat[off:off + numel].copy_(p.detach().reshape(-1))
                    p.data = b.param_flat[off:off + numel].view(p.shape)
                    b.grad_views.append(b.grad_flat[off:off + numel].view(p.shape))
                    b.scales.append(self.graph.scale_for(name))
            b.need_scale = any(s != 1.0 for s in b.scales)
            b.pending = [None] * len(b.items)
            b.ready = 0
            b.launched = False
            b.event = torch.cuda.Event()
        # every replica starts from rank 0's values
        if W > 1:
            torch.cuda.synchronize(self.device)
            for b in buckets:
                if b.mc:      # bootstrap only: no peer unicast mappings on NVLS buffers
                    self.fabric.comm.broadcast_(b.param_flat, 0)
                else:
                    nvops.broadcast(heap, b.param_buf.c_ptrs(), b.n * _ES[b.dtype], 0,
                                    CH_MAIN, self.fabric.max_blocks)
            torch.cuda.synchronize(self.device)
        for b in buckets:
            self._alloc_state(b)
        # clip-rule scalars.  A rule's contributors are its dense buckets and, with
        # include_sparse, the sparse groups whose tables it matches; the norm is complete,
        # and the rule's updates are issued, once the last of them has been enqueued
        self.clip_state = {}
        joint = {self.graph.joint_clip_index(grp.tables[0].name) for grp in self.sparse_groups}
        for ci in sorted({b.clip for b in buckets if b.clip >= 0} | (joint - {-1})):
            st = _Bucket()
            st.index = ci
            st.local = torch.zeros(4, dtype=torch.float32, device=self.device)
            st.total = torch.zeros(4, dtype=torch.float32, device=self.device)
            st.scale = torch.ones(1, dtype=torch.float32, device=self.device)
            st.norm = torch.zeros(1, dtype=torch.float32, device=self.device)
            st.buckets = [b for b in buckets if b.clip == ci]
            self.clip_state[ci] = st
        self.link_groups(self.sparse_groups)

    def link_groups(self, groups):
        """Attach the sparse groups of `include_sparse` clip rules to their rule's state
        (at build, and again when re-partitioning replaced the groups)."""
        self.sparse_groups = list(groups)
        for ci, st in self.clip_state.items():
            st.groups = sorted((grp for grp in groups
                                if self.graph.joint_clip_index(grp.tables[0].name) == ci),
                               key=lambda grp: grp.name)
            st.left = len(st.buckets) + len(st.groups)
            for grp in st.groups:
                grp.joint_clip = (self, st)
                grp.hp_clip = torch.zeros_like(grp.hp.dev)

    def _alloc_state(self, b):
        W, dev = self.world, self.device
        sharded = self.update == "sharded"
        b.slice = b.n // W if (sharded or self.update == "async") else b.n
        lo = self.rank * b.slice if b.slice != b.n else 0
        init = self.optimizer.slot_init()

        def mk(fill=None, src=None):
            if self.update == "async":
                sb = self.heap.alloc(b.slice * 4, "state")
                t = sb.tensor(torch.float32, b.slice)
                t._symm = sb
            else:
                t = torch.empty(b.slice, dtype=torch.float32, device=dev)
                t._symm = None
            if src is not None:
                t.copy_(src)
            else:
                t.fill_(fill)
            return t
        b.master = mk(src=b.param_flat[lo:lo + b.slice].float())
        b.slots = [mk(fill=v) for v in init]
        b.ema = None
        if self.ema_rule is not None and any(
                self.ema_rule.applies_to(n) for n, _, _, _ in b.items):
            b.ema = mk(src=b.master)
        b.red = torch.empty(b.slice, dtype=torch.float32, device=dev) \
            if ((b.clip >= 0 or self.micro_batches > 1 or self.layerwise) and sharded) else None
        b.lw = None
        if self.layerwise and sharded:
            b.lw = nvops.LayerwiseMap([(off, numel) for _, _, off, numel in b.items], lo,
                                      b.slice, 16 // _ES[b.dtype],
                                      [self.optimizer.layer_flags(n) for n, _, _, _ in b.items],
                                      dev)

    def _install_hooks(self):
        for b in self.buckets:
            b.async_events = []
            for idx, (name, p, off, numel) in enumerate(b.items):
                p.register_post_accumulate_grad_hook(self._make_hook(b, idx))
                _sinks.register(p, b.grad_views[idx], self._make_deliver(b, idx))

    def _make_deliver(self, b, idx):
        def deliver(event=None):
            # a fused op wrote this gradient straight into the bucket (`ops.sinks`)
            b.pending[idx] = b.grad_views[idx]
            if event is not None:
                b.async_events.append(event)
            b.ready += 1
            if b.ready == len(b.items):
                self._bucket_ready(b)
        return deliver

    def _make_hook(self, b, idx):
        def hook(p):
            b.pending[idx] = p.grad
            p.grad = None
            b.ready += 1
            if b.ready == len(b.items):
                self._bucket_ready(b)
        return hook

    # ----------------------------------------------------------------- step
    def begin_step(self, step):
        self._hp.upload(step)
        if self.pull_mirrors and step > 1:
            # mirror refresh deferred to "first use": all-gather of the owners'
            # parameter slices before the forward pass
            cur = torch.cuda.current_stream(self.device)
            for b in self.buckets:
                nvops.allgather(self.heap, b.param_buf.c_ptrs(),
                                (b.n // self.world) * _ES[b.dtype], CH_MAIN,
                                self.fabric.max_blocks, stream=cur)

    def _bucket_ready(self, b):
        views, grads = [], []
        for v, g in zip(b.grad_views, b.pending):
            if g is None:
                v.zero_()
            elif g is v:
                pass        # delivered in place (`ops.sinks`): no pack copy
            else:
                views.append(v)
                grads.append(g if g.dtype == v.dtype else g.to(v.dtype))
        if grads:
            torch._foreach_copy_(views, grads)
            nvops._count(1)
        if b.need_scale:
            for ev in b.async_events:     # scaled in place: the producer must be done
                torch.cuda.current_stream(self.device).wait_event(ev)
            for v, s in zip(b.grad_views, b.scales):
                if s != 1.0:
                    v.mul_(s)
        b.pending = [None] * len(b.items)
        b.event.record(torch.cuda.current_stream(self.device))
        b.is_ready = True
        self._drain()

    def _drain(self, final=False):
        """Launch consecutive ready buckets in index order on the comm stream."""
        last = len(self.buckets) - 1
        while self._next < len(self.buckets) and \
                getattr(self.buckets[self._next], "is_ready", False):
            if self._next == last and self.defer_last and not final and \
                    self._mb == self.micro_batches - 1:
                break
            b = self.buckets[self._next]
            self._launch(b)
            self._next += 1

    def _launch(self, b):
        from ..utils import timeline
        if timeline.enabled():
            with timeline.activity("bucket%d" % b.index, "DENSE_STEP", gpu=True,
                                   stream=self.fabric.comm_stream,
                                   args="%s n=%d %s" % (self.update, b.n, self.kind)):
                self._launch_impl(b)
        else:
            self._launch_impl(b)

    def _launch_impl(self, b):
        fab, heap, cs = self.fabric, self.heap, self.fabric.comm_stream
        cs.wait_event(b.event)
        for ev in b.async_events:        # side-stream producers of in-place gradients
            cs.wait_event(ev)
        if getattr(self, "stamp_before", None) and b.index == len(self.buckets) - 1:
            nvops.stamp(self.stamp_before, cs)
        W = self.world
        mb = fab.dense_blocks
        ema_decay = self.ema_rule.decay if self.ema_rule is not None else 0.0
        s0 = b.slots[0] if self.nslots > 0 else None
        s1 = b.slots[1] if self.nslots > 1 else None
        s2 = b.slots[2] if self.nslots > 2 else None
        st = self.clip_state.get(b.clip)
        K = self.micro_batches
        avg = 1.0 / (W * K)
        acc_in = self._mb > 0
        if self.update == "sharded" and self._mb < K - 1:
            nvops.dense_step(heap, self._grad_sources(b), self._param_targets(b),
                             b.master, s0, s1, b.ema, b.red, self.hp, None, None, b.n, avg,
                             ema_decay, self.kind, MODE_ACCUMULATE, b.dtype, CH_COMM,
                             max_blocks=mb, stream=cs, use_mc=b.mc, slot2=s2, acc_in=acc_in)
        elif self.update == "sharded":
            if st is None and self.layerwise:
                nvops.dense_step(heap, self._grad_sources(b), self._param_targets(b),
                                 b.master, s0, s1, b.ema, b.red, self.hp, None, None, b.n,
                                 avg, ema_decay, self.kind, MODE_REDUCE, b.dtype, CH_COMM,
                                 max_blocks=mb, stream=cs, use_mc=b.mc, acc_in=acc_in)
                self._layerwise_update(b, None, cs)
            elif st is None:
                nvops.dense_step(heap, self._grad_sources(b), self._param_targets(b),
                                 b.master, s0, s1, b.ema, b.red if acc_in else None,
                                 self.hp, None, None, b.n, avg, ema_decay, self.kind,
                                 MODE_FUSED, b.dtype, CH_COMM, max_blocks=mb,
                                 stream=cs, use_mc=b.mc, slot2=s2, acc_in=acc_in)
            else:
                nvops.dense_step(heap, self._grad_sources(b), self._param_targets(b),
                                 b.master, s0, s1, b.ema, b.red, self.hp, None,
                                 st.local, b.n, avg, ema_decay, self.kind,
                                 MODE_REDUCE, b.dtype, CH_COMM, max_blocks=mb,
                                 stream=cs, use_mc=b.mc, slot2=s2, acc_in=acc_in)
                self.contributed(st, cs)
        elif self.update == "replicated":
            # classic AR: all-reduce (mean) then every replica updates itself
            if self.protocol == "nccl" and W > 1:
                import torch.distributed as dist
                with torch.cuda.stream(cs):
                    dist.all_reduce(b.grad_flat, group=self.fabric.comm.group)
                    b.grad_flat.mul_(1.0 / W)
                    if st is not None:
                        # slice-local Σg² so the cross-rank sum equals the global norm²
                        sl = b.n // W
                        st.local[0] += b.grad_flat[self.rank * sl:(self.rank + 1) * sl] \
                            .float().pow(2).sum()
            else:
                nvops.allreduce_twoshot(heap, b.grad_buf.c_ptrs(), b.n, b.dtype,
                                        1.0 / W, CH_COMM,
                                        sumsq=st.local if st is not None else None,
                                        max_blocks=mb, stream=cs)
            if st is None:
                self._local_update(b, None, cs)
            else:
                self.contributed(st, cs)
        else:  # async PS
            clip = None
            if st is not None:
                nvops.sumsq(b.grad_flat, b.n, b.dtype, 1.0, st.local, stream=cs)
                if b is st.buckets[-1]:
                    nvops.clip_scale(st.local, self.clip_rules[b.clip].max_norm,
                                     st.scale, st.norm, st.local, stream=cs)
                    for bb in st.buckets:
                        self._async_update(bb, st.scale, cs)
            else:
                self._async_update(b, clip, cs)
        b.launched = True

    def _grad_sources(self, b):
        return b.grad_buf.mc_c_ptrs() if b.mc else b.grad_buf.c_ptrs()

    def _param_targets(self, b):
        """Where the fused kernel stores updated parameters: every peer's mirror
        (push; one multimem.st on NVLS buffers) or only the local buffer (pull
        mode; peers fetch later)."""
        if b.mc:
            return b.param_buf.mc_c_ptrs()
        if not self.pull_mirrors:
            return b.param_buf.c_ptrs()
        arr = getattr(b, "_self_targets", None)
        if arr is None:
            arr = (ctypes.c_void_p * self.world)(*([b.param_buf.local_ptr] * self.world))
            b._self_targets = arr
        return arr

    def contributed(self, st, cs):
        """One contributor of clip rule `st` (a dense bucket's Σg² reduction or a sparse
        group's `stage_norm`) has been enqueued on `cs`.  After the last one: the global
        norm and scale, each group's clipped hyper-parameters, the rule's dense updates,
        then the groups' deferred owner kernels in name order — the same order on every
        rank, since the contributors arrive in autograd order."""
        st.left -= 1
        if st.left:
            return
        st.left = len(st.buckets) + len(st.groups)
        self._finish_clip(st, cs)
        hps = [grp.clip_hp(st.scale, cs) for grp in st.groups]
        W, mb = self.world, self.fabric.dense_blocks
        ema_decay = self.ema_rule.decay if self.ema_rule is not None else 0.0
        for bb in st.buckets:
            if self.update == "sharded" and self.layerwise:
                self._layerwise_update(bb, st.scale, cs)
            elif self.update == "sharded":
                t0 = bb.slots[0] if self.nslots > 0 else None
                t1 = bb.slots[1] if self.nslots > 1 else None
                t2 = bb.slots[2] if self.nslots > 2 else None
                nvops.dense_step(self.heap, self._grad_sources(bb),
                                 self._param_targets(bb), bb.master, t0, t1,
                                 bb.ema, bb.red, self.hp, st.scale, None,
                                 bb.n, 1.0 / (W * self.micro_batches), ema_decay, self.kind,
                                 MODE_UPDATE, bb.dtype, CH_COMM,
                                 max_blocks=mb, stream=cs, use_mc=bb.mc, slot2=t2)
            else:
                self._local_update(bb, st.scale, cs)
        for grp, hp in zip(st.groups, hps):
            grp.stage_apply(grp._cur_step, cs, hp=hp)

    def _layerwise_update(self, b, clip, cs):
        """Passes 2-4 of a layer-wise bucket whose gradient is in `b.red`: the norm pass over
        this rank's slice, the one-shot all-reduce of the [nseg, 2] sums (bitwise identical
        on every rank, so a tensor split across owners gets one trust ratio), the update
        pass with the push of the parameters and the end barrier."""
        s0 = b.slots[0]
        s1 = b.slots[1] if self.nslots > 1 else None
        lw, W = b.lw, self.world
        nvops.layerwise_norm(b.red, b.master, s0, s1, self.hp, clip, lw, self.kind, b.dtype,
                             stream=cs)
        if W > 1:
            nvops.allreduce_oneshot(self.heap, lw.sums, lw.total, self.fabric.small_stage,
                                    2 * lw.nseg, torch.float32, 1.0, CH_SMALL, stream=cs)
        ema_decay = self.ema_rule.decay if self.ema_rule is not None else 0.0
        nvops.layerwise_update(self.heap, self._param_targets(b), b.red, b.master, s0, s1,
                               b.ema, self.hp, clip, lw, lw.total if W > 1 else lw.sums, b.n,
                               ema_decay, self.kind, b.dtype, CH_COMM,
                               max_blocks=self.fabric.dense_blocks, stream=cs, use_mc=b.mc)

    def _finish_clip(self, st, cs):
        rule = self.clip_rules[st.index]
        if self.world > 1:
            nvops.allreduce_oneshot(self.heap, st.local, st.total,
                                    self.fabric.small_stage, 4, torch.float32,
                                    1.0, CH_SMALL, stream=cs)
            nvops.clip_scale(st.total, rule.max_norm, st.scale, st.norm, st.local,
                             stream=cs)
        else:
            nvops.clip_scale(st.local, rule.max_norm, st.scale, st.norm, st.local,
                             stream=cs)

    def _local_update(self, b, clip, cs):
        ema_decay = self.ema_rule.decay if self.ema_rule is not None else 0.0
        s0 = b.slots[0] if self.nslots > 0 else None
        s1 = b.slots[1] if self.nslots > 1 else None
        s2 = b.slots[2] if self.nslots > 2 else None
        g = (ctypes.c_void_p * 1)(b.grad_buf.local_ptr)
        p = (ctypes.c_void_p * 1)(b.param_buf.local_ptr)
        b._keep = (g, p)
        nvops.dense_step(self.heap, g, p, b.master, s0, s1, b.ema, None, self.hp,
                         clip, None, b.n, 1.0, ema_decay, self.kind, MODE_FUSED,
                         b.dtype, CH_COMM, rank=0, world=1, stream=cs, slot2=s2)

    def _async_update(self, b, clip, cs):
        W = self.world
        mc = b.master._symm.c_ptrs()
        s0 = b.slots[0]._symm.c_ptrs() if self.nslots > 0 else None
        s1 = b.slots[1]._symm.c_ptrs() if self.nslots > 1 else None
        s2 = b.slots[2]._symm.c_ptrs() if self.nslots > 2 else None
        nvops.dense_async(b.grad_flat, b.param_flat, mc, s0, s1, self.hp, clip,
                          b.n, self.kind, b.dtype, self.rank, W,
                          max_blocks=self.fabric.max_blocks * 2, stream=cs, slot2_c=s2)

    def close(self):
        _sinks.unregister_all(self.params)

    def micro_batch(self, k, K):
        """The engine runs micro-batch `k` of `K` of the step next."""
        self._mb = k

    def end_micro_batch(self):
        """After the backward pass of a micro-batch that is not the step's last: every
        bucket has been reduced into its accumulator (MODE_ACCUMULATE) or is now; the
        bucket state starts over for the next micro-batch."""
        self._flush_buckets()
        self._reset_buckets()

    def _flush_buckets(self):
        # buckets whose parameters received no gradient this (micro-)step
        for b in self.buckets:
            if not getattr(b, "is_ready", False):
                self._bucket_ready(b)
        self._drain(final=True)
        assert self._next == len(self.buckets)

    def _reset_buckets(self):
        for b in self.buckets:
            b.ready, b.is_ready, b.launched = 0, False, False
            b.async_events = []
        self._next = 0

    def finish_step(self, step):
        self._flush_buckets()
        torch.cuda.current_stream(self.device).wait_stream(self.fabric.comm_stream)
        self._reset_buckets()
        self._mb = 0

    def zero_grad(self):
        for p in self.params:
            p.grad = None

    # ----------------------------------------------------------- checkpoint
    def _gather_full(self, attr, idx=None):
        """name -> full fp32 tensor (CPU) reconstructed from slices."""
        out = {}
        comm = self.fabric.comm
        for b in self.buckets:
            t = getattr(b, attr)
            if idx is not None:
                t = t[idx] if t is not None and idx < len(t) else None
            if t is None:
                continue
            if b.slice != b.n and self.world > 1:
                full = torch.cat(comm.all_gather_tensors(t.contiguous()))
            else:
                full = t
            full = full.detach().float().cpu()
            for name, p, off, numel in b.items:
                out[name] = full[off:off + numel].view(p.shape).clone()
        return out

    def state_dict(self):
        torch.cuda.synchronize(self.device)
        sd = {"master": self._gather_full("master"), "slots": {}, "ema": {}}
        per_slot = [self._gather_full("slots", i) for i in range(self.nslots)]
        for n in self.names:
            sd["slots"][n] = [ps[n] for ps in per_slot]
        if self.ema_rule is not None:
            full = self._gather_full("ema")
            sd["ema"] = {n: v for n, v in full.items()
                         if self.ema_rule.applies_to(n)}
        return sd

    def load_state_dict(self, sd):
        torch.cuda.synchronize(self.device)
        for b in self.buckets:
            lo = self.rank * b.slice if b.slice != b.n else 0
            hi = lo + b.slice

            def fill(dst, src_by_name):
                full = torch.zeros(b.n, dtype=torch.float32)
                have = dst.detach().float().cpu()
                full[lo:hi] = have
                for name, p, off, numel in b.items:
                    if name in src_by_name:
                        full[off:off + numel] = src_by_name[name].reshape(-1).float()
                dst.copy_(full[lo:hi].to(self.device))
                return full
            full = fill(b.master, sd["master"])
            # parameters (all of them, not just my slice)
            pf = b.param_flat.detach().float().cpu()
            for name, p, off, numel in b.items:
                if name in sd["master"]:
                    pf[off:off + numel] = sd["master"][name].reshape(-1).float()
            b.param_flat.copy_(pf.to(self.device).to(b.dtype))
            for i in range(self.nslots):
                fill(b.slots[i], {n: v[i] for n, v in sd["slots"].items()
                                  if len(v) > i})
            if b.ema is not None:
                fill(b.ema, sd.get("ema", {}))
        torch.cuda.synchronize(self.device)

    def ema_value(self, name):
        return self._gather_full("ema")[name]


# ===========================================================================
def build_nvlink(engine):
    """Module surgery for the NVLink fabric (called by `TrainEngine._build`)."""
    from .engine import ShardedEmbedding, _set_submodule
    from .. import ops
    if not torch.cuda.is_available():
        raise RuntimeError("the NVLink fabric needs a CUDA device")
    ops.lib()      # loud failure if the native library is missing
    g, comm, cfg = engine.graph, engine.comm, engine.config
    # convolution algorithms are picked by measurement during the eager warm-up
    # steps (shapes are static per graph); TF's cuDNN autotune did the same for the
    # reference (tensorflow/core/kernels/conv_ops.cc:746-783)
    torch.backends.cudnn.benchmark = bool(
        (cfg.sess_config or {}).get("cudnn_benchmark", True)
        if isinstance(cfg.sess_config, dict) else True)
    opts = dict(cfg.sess_config) if isinstance(cfg.sess_config, dict) else {}
    ps_cfg = cfg.communication_config.ps_config
    opts["_protocol"] = "nccl" if ps_cfg.protocol == "nccl" else "nvlink"
    opts["_replicate_variables"] = bool(ps_cfg.replicate_variables)
    fabric = NVFabric(comm, exchange=opts.get("_exchange"), options=opts)
    engine.fabric = fabric
    dev = comm.device
    cdt = opts.get("compute_dtype")
    cdt = {None: None, "float32": torch.float32, "fp32": torch.float32,
           "bfloat16": torch.bfloat16, "bf16": torch.bfloat16}.get(cdt, cdt)
    # sparse tables first (their weights may be meta / huge)
    sparse_items = sorted(engine.analysis.sparse_modules.items(), key=lambda kv: kv[0])
    pname_of = lambda path: path + ".weight" if path else "weight"
    # co-lookup groups: tables that the model looks up with the same ids in one call
    # (`parallax.nn.lookup_many`); declared by the model (`co_lookup_groups`, module
    # paths) or sess_config["sparse_groups"]
    declared = list(opts.get("sparse_groups") or
                    getattr(engine.model, "co_lookup_groups", None) or [])
    known = {path for path, _ in sparse_items}
    group_of, groups = {}, []
    for paths in declared:
        paths = [p_ for p_ in paths if p_ in known]
        if len(paths) > 1:
            groups.append(paths)
            for p_ in paths:
                group_of[p_] = len(groups) - 1
    # byte-greedy placement of every partition of every sparse variable on its owner
    # (`ps/between_graph_parallel.py:49-70`); PSConfig.boundary_among_servers=False keeps
    # the naive round-robin placement
    kind = g.sparse_optimizer.kind
    def item_bytes(path, mod):
        info = engine.analysis.variables[pname_of(path)]
        rows = (int(mod.weight.shape[0]) + info.partitions - 1) // info.partitions
        return info.partitions, rows * _optim.table_row_bytes(kind, int(mod.weight.shape[1]),
                                                              engine.sparse_weight_dtype)
    mods = dict(sparse_items)
    place_items, seen = [], set()
    for path, mod in sparse_items:
        key = ("g", group_of[path]) if path in group_of else ("t", path)
        if key in seen:
            continue
        seen.add(key)
        members = groups[group_of[path]] if path in group_of else [path]
        parts = {item_bytes(m_, mods[m_])[0] for m_ in members}
        if len(parts) != 1:
            raise ValueError("co-lookup group %s: members differ in partition count" % members)
        place_items.append((key, parts.pop(),
                            sum(item_bytes(m_, mods[m_])[1] for m_ in members)))
    owners = assign_owners(place_items, comm.world) \
        if bool(ps_cfg.boundary_among_servers) else {}
    for path, mod in sparse_items:
        pname = pname_of(path)
        info = engine.analysis.variables[pname]
        part = getattr(mod, "partitioner", None)
        key = ("g", group_of[path]) if path in group_of else ("t", path)
        t = NVSparseTable(
            pname, mod.weight, info.partitions,
            part.strategy if part is not None else "mod", g.sparse_optimizer,
            fabric, engine.route, g, cfg,
            init={"seed": getattr(mod, "init_seed", 1234),
                  "scale": getattr(mod, "init_scale", 0.05)},
            out_dtype=cdt or torch.float32, options=opts, owners=owners.get(key),
            auto_group=False)
        engine.tables[pname] = t
        _set_submodule(engine.model, path, ShardedEmbedding(t))
    engine.sparse_groups = []
    for paths in groups:
        engine.sparse_groups.append(NVSparseGroup([engine.tables[pname_of(p_)] for p_ in paths]))
    for path, _ in sparse_items:
        if path not in group_of:
            engine.sparse_groups.append(NVSparseGroup([engine.tables[pname_of(path)]]))
    engine.model.to(dev)
    if cdt is not None:
        for p in engine.model.parameters():
            if p.is_floating_point() and not getattr(p, "_parallax_skip", False):
                p.data = p.data.to(cdt)
        for b in engine.model.buffers():
            if b.is_floating_point() and opts.get("cast_buffers", False):
                b.data = b.data.to(cdt)
    dense_named = [(n, p) for n, p in engine.model.named_parameters()
                   if p.requires_grad and not getattr(p, "_parallax_skip", False)]
    joint = any(r.include_sparse for r in g.clip_rules())
    if g.trainable() and (dense_named or joint):
        engine.dense = NVDenseGroup(dense_named, g.optimizer, fabric, engine.route,
                                    g, options=opts, sparse_groups=engine.sparse_groups)
    torch.cuda.synchronize(dev)
    parallax_log.info(
        "nvlink fabric: rank %d/%d, %d dense buckets, %d sparse tables, "
        "symmetric heap %.1f MiB", comm.rank, comm.world,
        len(engine.dense.buckets) if engine.dense else 0, len(engine.tables),
        ops.lib().px_symm_live_bytes() / 2 ** 20)
