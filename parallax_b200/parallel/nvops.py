"""Thin, allocation-free Python wrappers around the native kernels.

Each function launches exactly one kernel (or a fixed short sequence) on the
given/current stream; all are CUDA-graph capturable.
"""
import ctypes

import torch

from .. import ops
from ..optim import KIND_ID

_vp = ctypes.c_void_p
DT = {torch.float32: 0, torch.bfloat16: 1}

# launch counter — bench.py reports `gpu_launches` from it
launches = {"n": 0}


def _count(k=1):
    launches["n"] += k


def _s(stream):
    if stream is None:
        stream = torch.cuda.current_stream()
    return _vp(stream.cuda_stream)


def _p(t):
    return _vp(t.data_ptr()) if t is not None else _vp(0)


def allreduce_twoshot(heap, buf_cptrs, n, dtype, scale, channels, sumsq=None,
                      max_blocks=32, stream=None):
    L = ops.lib()
    _count()
    ops.check(L.px_allreduce_twoshot(
        buf_cptrs, _p(heap.pads_dev()), _p(heap.epoch), channels[0], channels[1],
        n, DT[dtype], scale, _p(sumsq), heap.rank, heap.world, max_blocks,
        _s(stream)), "allreduce_twoshot")


def allreduce_twoshot_bulk(heap, buf_cptrs, n, dtype, scale, channels, max_blocks=128,
                           stream=None):
    """TMA (cp.async.bulk) variant of the two-shot all-reduce — kept for comparison
    (tools/allreduce_sweep.py); the engine uses the ld.global / multimem kernels."""
    L = ops.lib()
    _count()
    ops.check(L.px_allreduce_twoshot_bulk(
        buf_cptrs, _p(heap.pads_dev()), _p(heap.epoch), channels[0], channels[1], n, DT[dtype],
        scale, heap.rank, heap.world, max_blocks, _s(stream)), "allreduce_twoshot_bulk")


def allreduce_oneshot(heap, src, dst, stage_buf, n, dtype, scale, channel,
                      sumsq=None, max_blocks=8, stream=None):
    L = ops.lib()
    _count()
    ops.check(L.px_allreduce_oneshot(
        _p(src), _p(dst), stage_buf.c_ptrs(), stage_buf.nbytes // 2,
        _p(heap.pads_dev()), _p(heap.epoch), channel, n, DT[dtype], scale,
        _p(sumsq), heap.rank, heap.world, max_blocks, _s(stream)),
        "allreduce_oneshot")


def broadcast(heap, buf_cptrs, nbytes, root, channels, max_blocks=32, stream=None):
    L = ops.lib()
    _count()
    ops.check(L.px_broadcast(buf_cptrs, _p(heap.pads_dev()), _p(heap.epoch),
                             channels[0], channels[1], nbytes, root, heap.rank,
                             heap.world, max_blocks, _s(stream)), "broadcast")


def allgather(heap, buf_cptrs, slice_bytes, channels, max_blocks=32, stream=None):
    L = ops.lib()
    _count()
    ops.check(L.px_allgather(buf_cptrs, _p(heap.pads_dev()), _p(heap.epoch),
                             channels[0], channels[1], slice_bytes, heap.rank,
                             heap.world, max_blocks, _s(stream)), "allgather")


def dense_step(heap, grads_cptrs, params_cptrs, master, slot0, slot1, ema, red,
               hp, clip, sumsq, n, avg, ema_decay, kind, mode, dtype, channels,
               rank=None, world=None, max_blocks=32, stream=None, use_mc=False,
               slot2=None, acc_in=False):
    """One fused dense step (`kernels/dense_step.cu`).  `acc_in`: `red` holds the scaled
    gradient sum of the step's earlier micro-batches; modes 0, 1 and 3 add it first."""
    L = ops.lib()
    _count()
    ops.check(L.px_dense_step(
        grads_cptrs, params_cptrs, _p(master), _p(slot0), _p(slot1), _p(slot2), _p(ema),
        _p(red), _p(hp), _p(clip), _p(sumsq), n, avg, ema_decay, KIND_ID[kind],
        mode, 1 if acc_in else 0, DT[dtype], _p(heap.pads_dev()) if heap is not None else _vp(0),
        _p(heap.epoch) if heap is not None else _vp(0), channels[0], channels[1],
        heap.rank if rank is None else rank,
        heap.world if world is None else world, max_blocks, 1 if use_mc else 0,
        _s(stream)), "dense_step")


def clip_scale(sumsq_total, max_norm, scale_out, norm_out, zero_after, stream=None):
    L = ops.lib()
    _count()
    ops.check(L.px_clip_scale(_p(sumsq_total), max_norm, _p(scale_out),
                              _p(norm_out), _p(zero_after), _s(stream)),
              "clip_scale")


def clip_hp(hp, scale, out, stream=None):
    """out = hp with out[HP_GSCALE] multiplied by the device scalar `scale`."""
    L = ops.lib()
    _count()
    ops.check(L.px_clip_hp(_p(hp), _p(scale), _p(out), _s(stream)), "clip_hp")


def dense_async(my_grads, my_params, master_c, slot0_c, slot1_c, hp, clip, n,
                kind, dtype, rank, world, max_blocks=64, stream=None, slot2_c=None):
    L = ops.lib()
    _count()
    ops.check(L.px_dense_async(_p(my_grads), _p(my_params), master_c, slot0_c,
                               slot1_c, slot2_c, _p(hp), _p(clip), n, KIND_ID[kind],
                               DT[dtype], rank, world, max_blocks, _s(stream)),
              "dense_async")


def sumsq(x, n, dtype, mul, out, stream=None):
    L = ops.lib()
    _count()
    ops.check(L.px_sumsq(_p(x), n, DT[dtype], mul, _p(out), _s(stream)), "sumsq")


class LayerwiseMap(object):
    """Segment map of one layer-wise bucket (kinds `optim.LAYERWISE_KINDS`) on one rank, for
    `layerwise_norm` / `layerwise_update`.  `items`: the bucket's (offset, numel) per tensor in
    elements, in offset order; `lo`, `slice_n`: this rank's slice; `vn`: elements per 16-byte
    vector; `flags`: `optim.LW_*` bits per tensor.  A tensor is one segment; its vectors in the
    slice are split into chunks of at most `chunk` vectors, none spanning two tensors, so that
    every chunk's partial sums come from one CTA, without atomics.  A chunk's fourth entry
    counts its elements inside the tensor, so the tail of a tensor's last vector is left out
    of the norms."""
    CHUNK = 2048

    def __init__(self, items, lo, slice_n, vn, flags, device, chunk=None):
        chunk = chunk or self.CHUNK
        assert lo % vn == 0 and slice_n % vn == 0
        v_lo, v_hi = lo // vn, (lo + slice_n) // vn
        rows, rng = [], []
        for seg, (off, numel) in enumerate(items):
            assert off % vn == 0
            a, b = max(off // vn, v_lo), min((off + numel + vn - 1) // vn, v_hi)
            first = len(rows)
            for v in range(a, b, chunk):
                nv = min(chunk, b - v)
                rows.append((v - v_lo, nv, seg, min(nv * vn, off + numel - v * vn)))
            rng.append((first, len(rows)))
        assert v_hi - v_lo < 2 ** 31
        self.nseg, self.nchunks = len(items), len(rows)
        self.chunks = torch.tensor(rows or [(0, 0, 0, 0)], dtype=torch.int32, device=device)
        self.seg_chunks = torch.tensor(rng or [(0, 0)], dtype=torch.int32, device=device)
        self.flags = torch.tensor(list(flags) or [0], dtype=torch.int32, device=device)
        self.partials = torch.zeros(2 * max(self.nchunks, 1), dtype=torch.float32, device=device)
        self.sums = torch.zeros(2 * max(self.nseg, 1), dtype=torch.float32, device=device)
        self.total = torch.zeros_like(self.sums)


def layerwise_norm(red, master, slot0, slot1, hp, clip, lw, kind, dtype, max_blocks=0,
                   stream=None):
    """Norm pass of a layer-wise bucket: Σw² and Σx² of every segment over this rank's slice
    into `lw.sums` ([nseg, 2]; zero for segments outside the slice)."""
    L = ops.lib()
    _count(2)
    ops.check(L.px_layerwise_norm(
        _p(red), _p(master), _p(slot0), _p(slot1), _p(hp), _p(clip), _p(lw.chunks),
        lw.nchunks, _p(lw.flags), _p(lw.seg_chunks), lw.nseg, _p(lw.partials), _p(lw.sums),
        KIND_ID[kind], DT[dtype], max_blocks, _s(stream)), "layerwise_norm")


def layerwise_update(heap, params_cptrs, red, master, slot0, slot1, ema, hp, clip, lw, total,
                     n, ema_decay, kind, dtype, channels, rank=None, world=None, max_blocks=32,
                     stream=None, use_mc=False):
    """Update pass of a layer-wise bucket: trust ratios from `total` (the all-reduced
    `lw.sums`, or `lw.sums` itself at world 1), the rule, the EMA, the push of the parameters
    and the end barrier of `channels`."""
    L = ops.lib()
    _count()
    ops.check(L.px_layerwise_update(
        params_cptrs, _p(red), _p(master), _p(slot0), _p(slot1), _p(ema), _p(hp), _p(clip),
        _p(lw.chunks), lw.nchunks, _p(lw.flags), lw.nseg, _p(total), n, ema_decay,
        KIND_ID[kind], DT[dtype], _p(heap.pads_dev()) if heap is not None else _vp(0),
        _p(heap.epoch) if heap is not None else _vp(0), channels[1],
        heap.rank if rank is None else rank, heap.world if world is None else world,
        max_blocks, 1 if use_mc else 0, _s(stream)), "layerwise_update")


def stamp(slot_ptr, stream=None):
    """Write %globaltimer (ns) into a device u64 — a graph-capturable timestamp."""
    L = ops.lib()
    ops.check(L.px_stamp(_vp(slot_ptr), _s(stream)), "stamp")
