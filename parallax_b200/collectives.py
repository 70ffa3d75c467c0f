"""Horovod-style collective API over the NVLink fabric.

Parity: `horovod/tensorflow/__init__.py:36-82` (`allreduce` — dense mean/sum;
``IndexedSlices`` ⇒ allgather of values + indices), `:85-138` (broadcast of
variables), `horovod/torch/mpi_ops.py:86-422` (handle API: `*_async`, `poll`,
`synchronize`), `horovod/common/operations.cc:1625-1803` (init/rank/size,
name-keyed enqueue, DUPLICATE_NAME_ERROR `:1713-1716`), fusion buffer
(`fusion_buffer_manager.{h,cc}`, 64 MiB default `operations.cc:1030`).

Design: there is no background negotiation thread.  Every rank calls the same
ops in the same order (torch programs are rank-symmetric); an op is one or
two kernels on the caller's stream:

* ≤ `oneshot_bytes`  : staged one-shot all-reduce (one barrier, latency-bound)
* larger              : copy into the symmetric workspace (the "fusion
  buffer") → two-shot in-place reduce-scatter/all-gather kernel → copy out,
  chunked by the workspace size.  Tensors allocated with `symmetric_empty`
  skip both copies.
The 1/size scaling and dtype handling are inside the kernel epilogue (Horovod
runs a separate `div` kernel, `horovod/torch/mpi_ops_v2.cc:66-71`).

Cross-rank validation (Horovod's coordinator errors, `operations.cc:213-415`)
is done the first time a *name* is seen: shape/dtype/op digests are exchanged
once and cached (`registry` — the analogue of the response cache,
`response_cache.{h,cc}`); later calls with the same name skip the exchange.
"""
import ctypes
import functools
import os
import threading

import torch
import torch.distributed as dist

from .log import parallax_log
from .parallel.fabric import Comm

_state = None


class HorovodInternalError(RuntimeError):
    pass


class _State(object):
    def __init__(self, comm, workspace_bytes, oneshot_bytes):
        self.comm = comm
        self.cuda = comm.is_cuda
        self.fabric = None
        self.handles = {}
        self.next_handle = 1
        self.inflight_names = set()
        self.registry = {}
        self.lock = threading.Lock()
        self.timeline = None
        if self.cuda:
            from .parallel.nvlink_backend import NVFabric
            self.fabric = NVFabric(comm)
            heap = self.fabric.heap
            self.ws_bytes = int(workspace_bytes)
            self.ws = heap.alloc(self.ws_bytes, "fusion_workspace")
            self.oneshot_bytes = int(oneshot_bytes)
            self.stage = heap.alloc(2 * self.oneshot_bytes, "oneshot_stage")
            self.user_bufs = {}
            # NVLS workspace from 256 KB up at >= 4 GPUs (tools/allreduce_sweep.py measures
            # the crossover)
            self.ws_mc = None
            self.nvls_min_bytes = 256 << 10
            if comm.world >= 4:
                try:
                    from .parallel import multicast
                    if multicast.supported(comm):
                        self.ws_mc = multicast.MulticastBuffer(self.fabric, self.ws_bytes)
                except Exception as e:  # pragma: no cover
                    parallax_log.warning("NVLS workspace unavailable: %s", e)
                    self.ws_mc = None


def init(comm=None, workspace_bytes=64 << 20, oneshot_bytes=256 << 10):
    """Initialise (idempotent).  `comm` defaults to the torchrun environment."""
    global _state
    if _state is not None:
        return
    comm = comm or Comm.from_env()
    _state = _State(comm, workspace_bytes, oneshot_bytes)
    import os
    _registry_lib().px_registry_reset(int(os.environ.get("PARALLAX_CACHE_CAPACITY", 1024)))
    if comm.rank == 0:
        from . import consts
        from .log import parallax_log
        for name, why in consts.inert_horovod_env().items():
            parallax_log.info("%s is set but has no effect: %s", name, why)


def shutdown():
    global _state
    if _state is None:
        return
    if _state.fabric is not None:
        _state.fabric.close()
    _state = None


def _st():
    if _state is None:
        raise ValueError("parallax collectives have not been initialised; "
                         "call init() first")
    return _state


def is_initialized():
    return _state is not None


def rank():
    return _st().comm.rank


def size():
    return _st().comm.world


def local_rank():
    return _st().comm.local_rank


def local_size():
    import os
    return int(os.environ.get("LOCAL_WORLD_SIZE", _st().comm.world))


# ---------------------------------------------------------------------------
def _sig_hash(sig):
    import hashlib
    return int.from_bytes(hashlib.blake2b(repr(sig).encode(), digest_size=8).digest(),
                          "little")


def _validate(name, kind, tensor, extra=()):
    """First use of `name`: exchange (kind, dtype, shape[1:] or shape) and
    raise on every rank if they differ — Horovod's mismatch errors.  Validated
    signatures live in the native LRU registry (`runtime/registry.cpp`, the
    response-cache analogue): a HIT skips the exchange entirely."""
    st = _st()
    if name is None:
        return
    shape = tuple(tensor.shape[1:]) if kind == "allgather" else tuple(tensor.shape)
    sig = (kind, str(tensor.dtype), shape, tensor.device.type) + tuple(extra)
    L = _registry_lib()
    _coordinate_cache(st, L)
    h = _sig_hash(sig)
    state = L.px_registry_lookup(name.encode(), h)
    if state == 1:
        return                                  # cache hit: no negotiation
    if st.comm.distributed:
        sigs = st.comm.all_gather_object(sig)
        if len(set(sigs)) != 1:
            L.px_registry_erase(name.encode())
            raise HorovodInternalError(
                "Mismatched %s for tensor %r across ranks: %s" % (kind, name, sigs))
    L.px_registry_put(name.encode(), h)


def _coordinate_cache(st, L, force=False):
    """Horovod's `CacheCoordinator::sync` (`response_cache.cc:303-432`): a local cache HIT
    skips a *collective* exchange, which is only safe while every rank holds the same cache.
    Every `PARALLAX_CACHE_SYNC_EVERY` named ops (same count on all ranks — collectives are
    issued in one program order) the ranks exchange a digest of their cache plus its bit
    vector; on any disagreement every rank drops its cache, so the next use of each name
    is validated by all ranks together instead of hanging."""
    if not st.comm.distributed:
        return
    st.validate_calls = getattr(st, "validate_calls", 0) + 1
    every = int(os.environ.get("PARALLAX_CACHE_SYNC_EVERY", "64"))
    if not force and (every <= 0 or st.validate_calls % every):
        return
    words = max(1, L.px_registry_bits(None, 0))
    bits = (ctypes.c_uint64 * words)()
    L.px_registry_bits(bits, words)
    mine = (int(L.px_registry_digest()), tuple(int(b) for b in bits))
    everyone = st.comm.all_gather_object(mine)
    st.cache_syncs = getattr(st, "cache_syncs", 0) + 1
    if len({d for d, _ in everyone}) != 1:
        n = min(len(b) for _, b in everyone)
        common = sum(bin(functools.reduce(lambda a, c: a & c, [b[i] for _, b in everyone]))
                     .count("1") for i in range(n))
        parallax_log.warning(
            "collective signature caches diverged across ranks (%d entries in common): "
            "resetting them; every name is re-validated on next use", common)
        L.px_registry_reset(0)
        st.cache_resets = getattr(st, "cache_resets", 0) + 1


def _registry_lib():
    from . import ops
    global _reg_ready
    if not globals().get("_reg_ready"):
        u64 = ctypes.c_uint64
        ops.register_signatures({
            "px_registry_reset": (None, [ctypes.c_int]),
            "px_registry_lookup": (ctypes.c_int, [ctypes.c_char_p, u64]),
            "px_registry_put": (ctypes.c_int, [ctypes.c_char_p, u64]),
            "px_registry_erase": (ctypes.c_int, [ctypes.c_char_p]),
            "px_registry_bits": (ctypes.c_int, [ctypes.POINTER(u64), ctypes.c_int]),
            "px_registry_digest": (u64, []),
            "px_registry_stats": (None, [ctypes.POINTER(ctypes.c_long)] * 5),
        })
        _reg_ready = True
    return ops.lib()


def registry_stats():
    L = _registry_lib()
    v = [ctypes.c_long() for _ in range(5)]
    L.px_registry_stats(*[ctypes.byref(x) for x in v])
    return dict(zip(("hits", "misses", "invalid", "evictions", "size"),
                    [x.value for x in v]))


def _vn(dtype):
    return 16 // torch.empty((), dtype=dtype).element_size()


def symmetric_empty(numel, dtype=torch.float32):
    """A tensor in symmetric memory (collective call: every rank must allocate
    the same sequence).  `allreduce_` on it is zero-copy."""
    st = _st()
    es = torch.empty((), dtype=dtype).element_size()
    q = st.comm.world * _vn(dtype)
    n = (int(numel) + q - 1) // q * q
    buf = st.fabric.heap.alloc(n * es, "user")
    t = buf.tensor(dtype, n)[:numel]
    st.user_bufs[t.data_ptr()] = (buf, n)
    return t


def _allreduce_cuda(x, out, scale):
    from .parallel import nvops
    from .parallel.symmetric import CH_USER
    st = _st()
    heap, W = st.fabric.heap, st.comm.world
    dt = x.dtype
    if dt == torch.float16:
        # widened on the way in: an fp16 sum of W addends is exact in fp32
        y = torch.empty_like(x, dtype=torch.float32)
        _allreduce_cuda(x.float(), y, scale)
        out.copy_(y.to(dt))
        return out
    if dt not in nvops.DT:
        # int32 / int64 / fp64 / uint8 …: exact reduction through the library (Horovod
        # reduces these dtypes natively, `nccl_operations.cc:22-38`); an fp32 detour would
        # corrupt counts above 2^24 and truncate float64
        y = x.clone()
        dist.all_reduce(y, group=st.comm.group)
        if scale != 1.0:
            y = y / W if dt.is_floating_point else torch.div(y, W, rounding_mode="floor")
        out.copy_(y.view(out.shape))
        return out
    es = x.element_size()
    n = x.numel()
    if n == 0:
        return out
    flat, oflat = x.reshape(-1), out.reshape(-1)
    ub = st.user_bufs.get(x.data_ptr())
    if ub is not None and out.data_ptr() == x.data_ptr():
        buf, npad = ub
        nvops.allreduce_twoshot(heap, buf.c_ptrs(), npad, dt, scale, CH_USER,
                                max_blocks=st.fabric.max_blocks)
        return out
    if n * es <= st.oneshot_bytes and flat.data_ptr() % 16 == 0:
        # storage may be shorter than the 16 B-padded length: stage a copy then
        if (n * es) % 16 != 0:
            pad = torch.zeros((n * es + 15) // 16 * 16 // es, dtype=dt, device=x.device)
            pad[:n] = flat
            dst = torch.empty_like(pad)
            nvops.allreduce_oneshot(heap, pad, dst, st.stage, n, dt, scale,
                                    CH_USER[0])
            oflat.copy_(dst[:n])
        else:
            nvops.allreduce_oneshot(heap, flat, oflat, st.stage, n, dt, scale,
                                    CH_USER[0])
        return out
    use_mc = st.ws_mc is not None and n * es >= st.nvls_min_bytes
    ws = (st.ws_mc if use_mc else st.ws).tensor(dt)
    q = W * _vn(dt)
    chunk = (min(ws.numel(), st.ws_bytes // es) // q) * q
    for s in range(0, n, chunk):
        m = min(chunk, n - s)
        mp = (m + q - 1) // q * q
        ws[:m].copy_(flat[s:s + m])
        if mp != m:
            ws[m:mp].zero_()
        if use_mc:
            st.ws_mc.allreduce_(mp, dt, scale, CH_USER, max_blocks=64)
        else:
            nvops.allreduce_twoshot(heap, st.ws.c_ptrs(), mp, dt, scale, CH_USER,
                                    max_blocks=st.fabric.max_blocks)
        oflat[s:s + m].copy_(ws[:m])
    return out


class Compression(object):
    """Gradient compression for all-reduce (`horovod/tensorflow/compression.py:46-64`:
    ``Compression.none`` / ``Compression.fp16``).  bf16 is the Hopper-native
    16-bit wire format; fp16 is kept for parity."""

    class none(object):
        @staticmethod
        def compress(t):
            return t, None

        @staticmethod
        def decompress(t, ctx):
            return t

    class fp16(object):
        @staticmethod
        def compress(t):
            return (t.to(torch.float16), t.dtype) if t.is_floating_point() else (t, None)

        @staticmethod
        def decompress(t, ctx):
            return t.to(ctx) if ctx is not None else t

    class bf16(object):
        @staticmethod
        def compress(t):
            return (t.to(torch.bfloat16), t.dtype) if t.is_floating_point() else (t, None)

        @staticmethod
        def decompress(t, ctx):
            return t.to(ctx) if ctx is not None else t


def allreduce(tensor, average=True, name=None, out=None, compression=None):
    if out is None and compression is None and _wants_grad(tensor):
        return _AllreduceFn.apply(tensor, average, name)
    if compression is not None and compression is not Compression.none:
        c, ctx = compression.compress(tensor)
        r = compression.decompress(allreduce(c, average, name), ctx)
        if out is not None:
            out.copy_(r)
            return out
        return r
    return _allreduce_impl(tensor, average, name, out)


def _allreduce_impl(tensor, average=True, name=None, out=None):
    """Sum (or mean) of `tensor` over all ranks.  A ``torch.sparse`` tensor is
    reduced Horovod-style: all-gather of indices and values (duplicates kept,
    values ÷ size when `average`)."""
    st = _st()
    if tensor.is_sparse:
        t = tensor.coalesce()
        idx = allgather(t.indices().t().contiguous(),
                        name=None if name is None else name + ".indices")
        val = allgather(t.values(), name=None if name is None else name + ".values")
        if average:
            val = val / st.comm.world
        return torch.sparse_coo_tensor(idx.t(), val, tensor.shape)
    _validate(name, "allreduce", tensor)
    W = st.comm.world
    scale = (1.0 / W) if average else 1.0
    if out is None:
        out = torch.empty_like(tensor, memory_format=torch.contiguous_format)
    if not tensor.is_cuda or not st.cuda:
        out.copy_(tensor)
        if W > 1:
            dist.all_reduce(out, group=st.comm._grp_for(out))
        if average:
            out.div_(W) if out.is_floating_point() else out.floor_divide_(W)
        return out
    x = tensor.contiguous()
    if W == 1:
        out.copy_(x)
        return out
    if not out.is_contiguous():
        # `out.reshape(-1)` of a transposed / channels_last tensor is a copy: reduce into a
        # contiguous temporary and lay the result out afterwards
        tmp = torch.empty_like(x)
        _allreduce_cuda(x, tmp, scale)
        out.copy_(tmp.view(out.shape))
        return out
    return _allreduce_cuda(x, out, scale)


def allreduce_(tensor, average=True, name=None):
    return allreduce(tensor, average, name, out=tensor)


def grouped_allreduce(tensors, average=True, name=None):
    """Fuse several tensors of one dtype into the workspace, reduce once,
    scatter the results back (Horovod tensor fusion,
    `horovod/common/operations.cc:465-588`)."""
    st = _st()
    if not tensors:
        return []
    if not st.cuda or st.comm.world == 1 or len({t.dtype for t in tensors}) != 1:
        return [allreduce(t, average, None) for t in tensors]
    flat = torch.cat([t.reshape(-1) for t in tensors])
    red = allreduce(flat, average, name)
    outs, off = [], 0
    for t in tensors:
        outs.append(red[off:off + t.numel()].view_as(t))
        off += t.numel()
    return outs


def allgather(tensor, name=None):
    """Concatenate `tensor` from all ranks along dim 0 (first dims may differ)."""
    if _wants_grad(tensor):
        return _AllgatherFn.apply(tensor, name)
    return _allgather_impl(tensor, name)


def _allgather_impl(tensor, name=None):
    st = _st()
    _validate(name, "allgather", tensor)
    W = st.comm.world
    if W == 1:
        return tensor.clone()
    sizes = st.comm.all_gather_object(int(tensor.shape[0]))
    if not tensor.is_cuda or not st.cuda:
        return torch.cat(st.comm.all_gather_varlen(tensor))
    from .parallel import nvops
    from .parallel.symmetric import CH_USER
    x = tensor.contiguous()
    row = x[0].numel() if x.dim() > 1 and x.shape[0] else \
        (int(torch.tensor(x.shape[1:]).prod()) if x.dim() > 1 else 1)
    es = x.element_size()
    slice_bytes = (max(sizes) * row * es + 15) // 16 * 16
    if slice_bytes * W > st.ws_bytes:
        # too large for the workspace: library fallback (rare, control-sized)
        return torch.cat(st.comm.all_gather_varlen(tensor))
    wsb = st.ws.bytes_tensor()
    mine = wsb[st.comm.rank * slice_bytes:st.comm.rank * slice_bytes + x.numel() * es]
    mine.copy_(x.reshape(-1).view(torch.uint8))
    nvops.allgather(st.fabric.heap, st.ws.c_ptrs(), slice_bytes, CH_USER,
                    max_blocks=st.fabric.max_blocks)
    parts = []
    for r, n in enumerate(sizes):
        b = wsb[r * slice_bytes:r * slice_bytes + n * row * es]
        parts.append(b.view(x.dtype).view((n,) + tuple(x.shape[1:])))
    return torch.cat(parts)


def broadcast(tensor, root_rank, name=None, out=None):
    if out is None and _wants_grad(tensor):
        return _BroadcastFn.apply(tensor, root_rank, name)
    return _broadcast_impl(tensor, root_rank, name, out)


def _broadcast_impl(tensor, root_rank, name=None, out=None):
    st = _st()
    _validate(name, "broadcast", tensor, extra=(root_rank,))
    W = st.comm.world
    if out is None:
        out = torch.empty_like(tensor)
    out.copy_(tensor)
    if W == 1:
        return out
    if not tensor.is_cuda or not st.cuda:
        dist.broadcast(out, src=root_rank, group=st.comm._grp_for(out))
        return out
    from .parallel import nvops
    from .parallel.symmetric import CH_USER
    flat = out.reshape(-1).view(torch.uint8) if out.is_contiguous() else None
    src = out.contiguous().reshape(-1).view(torch.uint8)
    wsb = st.ws.bytes_tensor()
    n = src.numel()
    for s in range(0, n, st.ws_bytes):
        m = min(st.ws_bytes, n - s)
        mp = (m + 15) // 16 * 16
        if st.comm.rank == root_rank:
            wsb[:m].copy_(src[s:s + m])
        nvops.broadcast(st.fabric.heap, st.ws.c_ptrs(), mp, root_rank, CH_USER,
                        st.fabric.max_blocks)
        src[s:s + m].copy_(wsb[:m])
    if flat is None:
        out.copy_(src.view(out.dtype).view(out.shape))
    return out


def broadcast_(tensor, root_rank, name=None):
    return broadcast(tensor, root_rank, name, out=tensor)


def broadcast_parameters(params, root_rank=0):
    """Broadcast a state_dict / named parameters from `root_rank`
    (`horovod/torch/__init__.py` `broadcast_parameters`,
    `horovod/tensorflow/__init__.py:85-104`)."""
    items = sorted(params.items()) if isinstance(params, dict) else sorted(params)
    for name, p in items:
        if torch.is_tensor(p):
            with torch.no_grad():
                broadcast_(p.data if hasattr(p, "data") else p, root_rank,
                           name="broadcast." + name)


# ---------------------------------------------------------------- autograd
# Horovod registers gradients for its collective ops
# (`horovod/tensorflow/mpi_ops.py:82-173`, `horovod/torch/mpi_ops.py` autograd Functions):
# d(allreduce) = allreduce of the upstream gradient; d(allgather) = this rank's rows of the
# summed gradient; d(broadcast) = the summed gradient on the root, zero elsewhere.
def _wants_grad(t):
    return torch.is_grad_enabled() and torch.is_tensor(t) and t.requires_grad and \
        not t.is_sparse


def _gname(name):
    return None if name is None else name + ".grad"


class _AllreduceFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, tensor, average, name):
        ctx.average, ctx.name = average, name
        return _allreduce_impl(tensor.detach(), average, name)

    @staticmethod
    def backward(ctx, grad):
        return _allreduce_impl(grad.contiguous(), ctx.average, _gname(ctx.name)), None, None


class _AllgatherFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, tensor, name):
        st = _st()
        ctx.name, ctx.n = name, int(tensor.shape[0])
        sizes = st.comm.all_gather_object(ctx.n) if st.comm.world > 1 else [ctx.n]
        ctx.offset = sum(sizes[:st.comm.rank])
        return _allgather_impl(tensor.detach(), name)

    @staticmethod
    def backward(ctx, grad):
        summed = _allreduce_impl(grad.contiguous(), False, _gname(ctx.name))
        return summed[ctx.offset:ctx.offset + ctx.n], None


class _BroadcastFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, tensor, root_rank, name):
        ctx.root, ctx.name = root_rank, name
        return _broadcast_impl(tensor.detach(), root_rank, name)

    @staticmethod
    def backward(ctx, grad):
        summed = _allreduce_impl(grad.contiguous(), False, _gname(ctx.name))
        if _st().comm.rank != ctx.root:
            summed = torch.zeros_like(summed)
        return summed, None, None


# ------------------------------------------------------------- handle API
def _enqueue(kind, fn, name):
    st = _st()
    with st.lock:
        if name is not None:
            if name in st.inflight_names:
                raise HorovodInternalError(
                    "Duplicate tensor name %r: a previous %s with this name has "
                    "not completed" % (name, kind))
            st.inflight_names.add(name)
        h = st.next_handle
        st.next_handle += 1
    result = fn()
    ev = None
    if torch.is_tensor(result) and result.is_cuda:
        ev = torch.cuda.Event()
        ev.record()
    st.handles[h] = (result, ev, name)
    return h


def allreduce_async(tensor, average=True, name=None):
    return _enqueue("allreduce", lambda: allreduce(tensor, average, name), name)


def allreduce_async_(tensor, average=True, name=None):
    return _enqueue("allreduce", lambda: allreduce_(tensor, average, name), name)


def allgather_async(tensor, name=None):
    return _enqueue("allgather", lambda: allgather(tensor, name), name)


def broadcast_async(tensor, root_rank, name=None):
    return _enqueue("broadcast", lambda: broadcast(tensor, root_rank, name), name)


def broadcast_async_(tensor, root_rank, name=None):
    return _enqueue("broadcast", lambda: broadcast_(tensor, root_rank, name), name)


def poll(handle):
    result, ev, _ = _st().handles[handle]
    return True if ev is None else ev.query()


def synchronize(handle):
    st = _st()
    if handle not in st.handles:
        raise ValueError("unknown handle %r" % handle)
    result, ev, name = st.handles.pop(handle)
    if ev is not None:
        ev.synchronize()
    if name is not None:
        st.inflight_names.discard(name)
    return result


class DistributedOptimizer(object):
    """Wrap a ``torch.optim.Optimizer``: gradients are averaged across ranks
    before `step()` (`horovod/torch/__init__.py:44-177`: per-parameter hooks
    fire `allreduce_async_` during backward, `synchronize()` waits).  Here the
    per-parameter hooks only count backward passes; `synchronize()` — called by
    `step()` — reduces all dense gradients of one dtype as ONE fused group
    (`grouped_allreduce`) on the fabric kernels, i.e. after the backward pass,
    not underneath it (the `parallel_run` engine is the path that launches
    bucket kernels from autograd hooks on a comm stream while backward still
    runs).  Sparse gradients are all-gathered unless `sparse_as_dense`
    (`horovod/tensorflow/__init__.py:189-192`)."""

    def __init__(self, optimizer, named_parameters=None, sparse_as_dense=False,
                 compression=None, backward_passes_per_step=1):
        self.optimizer = optimizer
        self.sparse_as_dense = sparse_as_dense
        # `compression`: gradients travel in the compressed dtype
        # (`horovod/torch/compression.py`); `backward_passes_per_step` = N: the gradients
        # of up to N backward passes accumulate locally in `.grad`; `step()` — called ONCE
        # after them — always reduces and applies (`horovod/torch/__init__.py:79-154`: the
        # per-parameter hooks count passes, `step()` synchronizes)
        self.compression = compression
        self.backward_passes_per_step = int(backward_passes_per_step)
        assert self.backward_passes_per_step >= 1
        params = [p for g in optimizer.param_groups for p in g["params"]]
        if named_parameters is not None:
            names = {id(p): n for n, p in named_parameters}
        else:
            names = {}
        self._names = {id(p): names.get(id(p), "param.%d" % i)
                       for i, p in enumerate(params)}
        dup = len(set(self._names.values())) != len(self._names)
        if dup:
            raise ValueError("parameter names must be unique")
        self._params = params
        self._synchronized = False
        self._delay = {id(p): self.backward_passes_per_step for p in params}
        self._hooks = [p.register_post_accumulate_grad_hook(self._count_pass)
                       for p in params if p.requires_grad]

    def _count_pass(self, p):
        if self._delay[id(p)] <= 0:
            raise AssertionError(
                "Gradients were computed more than backward_passes_per_step times before "
                "call to step(). Increase backward_passes_per_step to accumulate gradients "
                "locally.")
        self._delay[id(p)] -= 1

    def synchronize(self):
        dense = [p for p in self._params if p.grad is not None and not p.grad.is_sparse]
        by_dtype = {}
        for p in dense:
            by_dtype.setdefault(p.grad.dtype, []).append(p)
        comp = self.compression if self.compression is not None and \
            self.compression is not Compression.none else None
        for dt, ps in by_dtype.items():
            if comp is None:
                outs = grouped_allreduce([p.grad for p in ps], average=True)
            else:
                packed = [comp.compress(p.grad) for p in ps]
                red = grouped_allreduce([c for c, _ in packed], average=True)
                outs = [comp.decompress(r, ctx) for r, (_, ctx) in zip(red, packed)]
            for p, o in zip(ps, outs):
                p.grad.copy_(o)
        for p in self._params:
            if p.grad is not None and p.grad.is_sparse:
                if self.sparse_as_dense:
                    p.grad = allreduce(p.grad.to_dense(), True)
                else:
                    p.grad = allreduce(p.grad, True, name="grad." + self._names[id(p)])
        self._synchronized = True

    def step(self, closure=None):
        """Reduce whatever accumulated in `.grad` since the last step (1..N backward
        passes) and apply it."""
        if not self._synchronized:
            self.synchronize()
        self._synchronized = False
        for k in self._delay:
            self._delay[k] = self.backward_passes_per_step
        return self.optimizer.step(closure)

    def zero_grad(self, set_to_none=True):
        return self.optimizer.zero_grad(set_to_none=set_to_none)

    def __getattr__(self, k):
        return getattr(self.optimizer, k)


# --------------------------------------------------- more of the Horovod surface
def mpi_threads_supported():
    """Horovod reports whether MPI was initialised with MPI_THREAD_MULTIPLE
    (`horovod/common/operations.cc:1675-1680`).  There is no MPI here: ops are
    stream-ordered launches that any thread may issue, provided all ranks issue
    them in the same order."""
    _st()
    return True


def mpi_built():
    """Horovod scripts branch on this to pick a launcher; nothing here links MPI."""
    return False


def mpi_enabled():
    return False


def gloo_built():
    """the host fabric (CPU tensors, bootstrap) runs over torch.distributed's gloo backend"""
    import torch.distributed as dist
    return bool(dist.is_available() and dist.is_gloo_available())


def nccl_built():
    """NCCL is reachable (`protocol="nccl"`, int / fp64 reductions, the bench's same-engine
    arm); the default data path is the hand-written NVLink fabric, not NCCL."""
    import torch.distributed as dist
    return bool(dist.is_available() and dist.is_nccl_available())


def cuda_built():
    return bool(torch.cuda.is_available())


def broadcast_object(obj, root_rank=0):
    """pickle-able python object from `root_rank` to everyone"""
    return _st().comm.broadcast_object(obj, root_rank)


def broadcast_optimizer_state(optimizer, root_rank=0):
    """Broadcast a ``torch.optim.Optimizer``'s state (slot tensors, step counters,
    hyper-parameters in `param_groups`) from `root_rank`
    (`horovod/torch/__init__.py` `broadcast_optimizer_state`).  State that does not
    exist yet on a rank (fresh optimizer) is created from the root's layout."""
    if isinstance(optimizer, DistributedOptimizer):
        optimizer = optimizer.optimizer
    st = _st()
    sd = optimizer.state_dict()
    # scalars / structure travel as one object; tensors with the tensor broadcast
    meta = {"param_groups": sd["param_groups"],
            "state": {k: {n: (("T", tuple(v.shape), str(v.dtype)) if torch.is_tensor(v) else
                              ("V", v)) for n, v in d.items()}
                      for k, d in sd["state"].items()}}
    meta = st.comm.broadcast_object(meta, root_rank)
    new_state = {}
    for k, d in sorted(meta["state"].items(), key=lambda kv: str(kv[0])):
        new_state[k] = {}
        for n, desc in sorted(d.items()):
            if desc[0] == "V":
                new_state[k][n] = desc[1]
                continue
            have = sd["state"].get(k, {}).get(n)
            dtype = getattr(torch, desc[2].split(".")[-1])
            if have is None or tuple(have.shape) != desc[1]:
                ref = optimizer.param_groups[0]["params"][0]
                have = torch.zeros(desc[1], dtype=dtype, device=ref.device)
            t = have.detach().clone()
            broadcast_(t, root_rank, name="opt_state.%s.%s" % (k, n))
            new_state[k][n] = t
    optimizer.load_state_dict({"state": new_state, "param_groups": meta["param_groups"]})


def allreduce_gradients(params, average=True, compression=None, sparse_as_dense=False):
    """Reduce the `.grad` of `params` in place (fused per dtype).  The building
    block of `DistributedGradientTape`."""
    params = [p for p in params if p.grad is not None]
    dense = [p for p in params if not p.grad.is_sparse]
    by_dtype = {}
    for p in dense:
        by_dtype.setdefault(p.grad.dtype, []).append(p)
    comp = compression if compression is not None and compression is not Compression.none \
        else None
    for ps in by_dtype.values():
        if comp is None:
            outs = grouped_allreduce([p.grad for p in ps], average=average)
        else:
            packed = [comp.compress(p.grad) for p in ps]
            red = grouped_allreduce([c for c, _ in packed], average=average)
            outs = [comp.decompress(r, ctx) for r, (_, ctx) in zip(red, packed)]
        for p, o in zip(ps, outs):
            p.grad.copy_(o)
    for i, p in enumerate(params):
        if p.grad.is_sparse:
            p.grad = allreduce(p.grad.to_dense(), average) if sparse_as_dense else \
                allreduce(p.grad, average, name=None)


class DistributedGradientTape(object):
    """`horovod/tensorflow/__init__.py:242-316`: a gradient "tape" whose
    `gradient(target, sources)` returns gradients already averaged over the
    ranks.  The torch counterpart wraps `torch.autograd.grad`."""

    def __init__(self, compression=None, sparse_as_dense=False):
        self.compression, self.sparse_as_dense = compression, sparse_as_dense

    def gradient(self, target, sources, retain_graph=False):
        sources = list(sources)
        grads = torch.autograd.grad(target, sources, retain_graph=retain_graph,
                                    allow_unused=True)
        out = []
        for i, g in enumerate(grads):
            if g is None:
                out.append(None)
            elif g.is_sparse:
                out.append(allreduce(g.to_dense(), True) if self.sparse_as_dense
                           else allreduce(g, True))
            else:
                out.append(allreduce(g, True, compression=self.compression))
        return out
