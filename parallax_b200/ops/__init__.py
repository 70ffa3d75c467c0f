"""Native library loader (ctypes over a C ABI — no torch headers, so the
whole library compiles in seconds and loads into any torch build).

`lib()` returns the loaded `libparallax_b200.so`.  On a machine with a CUDA
device a missing/unloadable library is a hard error — the engine never
silently falls back to a library/eager path.
"""
import ctypes
import os

from .build import LIB, build as _build, nvcc as _nvcc

_lib = None
_abi = None

c_void_p, c_int, c_size_t, c_float = \
    ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t, ctypes.c_float
PP = ctypes.POINTER(ctypes.c_void_p)


# ctypes mirrors of the sparse-group descriptors, named like their C structs (sparse_group.cuh,
# sparse.cu); `lib()` checks their layout against the library's `px_sparse_abi()`.
class GroupGeom(ctypes.Structure):
    _fields_ = [(n, c_int) for n in ("V", "P", "W", "rows_per_part", "strategy",
                                     "replicated", "extras", "base")] + \
        [("part_owner", c_void_p), ("part_slot", c_void_p)]


class LookupTable(ctypes.Structure):
    _fields_ = [("srcs", c_void_p), ("out", c_void_p), ("D4", c_int),
                ("src_bf16", c_int), ("out_bf16", c_int)]


class PushTable(ctypes.Structure):
    _fields_ = [("grads", c_void_p), ("staging", c_void_p), ("rings", c_void_p),
                ("tables", c_void_p), ("slot0s", c_void_p), ("slot1s", c_void_p),
                ("slot2s", c_void_p), ("shadows", c_void_p), ("hp", c_void_p),
                ("D4", c_int), ("kind", c_int), ("scale", c_float)]


class OwnerTable(ctypes.Structure):
    _fields_ = [("ring", c_void_p), ("table", c_void_p), ("slot0", c_void_p),
                ("slot1", c_void_p), ("slot2", c_void_p), ("shadow", c_void_p),
                ("hp", c_void_p), ("D4", c_int), ("kind", c_int), ("avg", c_float),
                ("D", c_int), ("slot_part", c_void_p), ("seed", ctypes.c_uint32),
                ("w_bf16", c_int)]


_SIGS = {
    "px_last_error": (ctypes.c_char_p, []),
    "px_device_count": (c_int, []),
    "px_set_device": (c_int, [c_int]),
    "px_symm_alloc": (c_int, [c_size_t, PP]),
    "px_symm_free": (c_int, [c_void_p]),
    "px_ipc_export": (c_int, [c_void_p, ctypes.c_char_p]),
    "px_ipc_import": (c_int, [ctypes.c_char_p, PP]),
    "px_ipc_close": (c_int, [c_void_p]),
    "px_enable_peer": (c_int, [c_int]),
    "px_memcpy_h2d_async": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p]),
    "px_memset_async": (c_int, [c_void_p, c_int, c_size_t, c_void_p]),
    "px_symm_live_bytes": (c_size_t, []),
    "px_barrier": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "px_allreduce_twoshot": (c_int, [PP, c_void_p, c_void_p, c_int, c_int, c_size_t,
                                     c_int, c_float, c_void_p, c_int, c_int, c_int,
                                     c_void_p]),
    "px_allreduce_twoshot_bulk": (c_int, [PP, c_void_p, c_void_p, c_int, c_int, c_size_t,
                                          c_int, c_float, c_int, c_int, c_int, c_void_p]),
    "px_allreduce_oneshot": (c_int, [c_void_p, c_void_p, PP, c_size_t, c_void_p,
                                     c_void_p, c_int, c_size_t, c_int, c_float,
                                     c_void_p, c_int, c_int, c_int, c_void_p]),
    "px_broadcast": (c_int, [PP, c_void_p, c_void_p, c_int, c_int, c_size_t, c_int,
                             c_int, c_int, c_int, c_void_p]),
    "px_allgather": (c_int, [PP, c_void_p, c_void_p, c_int, c_int, c_size_t, c_int,
                             c_int, c_int, c_void_p]),
    "px_dense_step": (c_int, [PP, PP, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                              c_void_p, c_void_p, c_void_p, c_void_p, c_size_t,
                              c_float, c_float, c_int, c_int, c_int, c_int, c_void_p,
                              c_void_p, c_int, c_int, c_int, c_int, c_int, c_int,
                              c_void_p]),
    "px_clip_scale": (c_int, [c_void_p, c_float, c_void_p, c_void_p, c_void_p,
                              c_void_p]),
    "px_dense_async": (c_int, [c_void_p, c_void_p, PP, PP, PP, PP, c_void_p, c_void_p,
                               c_size_t, c_int, c_int, c_int, c_int, c_int,
                               c_void_p]),
    "px_sumsq": (c_int, [c_void_p, c_size_t, c_int, c_float, c_void_p, c_void_p]),
    "px_layerwise_norm": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                  c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p,
                                  c_void_p, c_int, c_int, c_int, c_void_p]),
    "px_layerwise_update": (c_int, [PP, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                    c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int,
                                    c_void_p, c_size_t, c_float, c_int, c_int, c_void_p,
                                    c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "px_sparse_lookup": (c_int, [c_void_p, c_int, c_int, ctypes.POINTER(LookupTable),
                                 c_int, c_void_p, ctypes.POINTER(GroupGeom), c_void_p,
                                 c_void_p, c_int, c_void_p]),
    "px_full_softmax_nll": (c_int, [c_void_p, c_int, c_int, c_void_p, c_int, c_void_p, c_int,
                                    c_int, c_void_p, c_int, ctypes.POINTER(GroupGeom), c_int,
                                    c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p,
                                    c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "px_full_softmax_grad": (c_int, [c_void_p, c_int, c_int, c_void_p, c_int, c_void_p, c_int,
                                     c_int, c_int, ctypes.c_longlong, c_void_p, c_void_p,
                                     c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p]),
    "px_full_softmax_topk": (c_int, [c_void_p, c_int, c_int, c_void_p, c_int, c_void_p, c_int,
                                     c_int, c_void_p, c_void_p, c_int, ctypes.POINTER(GroupGeom),
                                     c_int, c_void_p, c_void_p, c_int, c_void_p, c_int, c_int,
                                     c_void_p, c_void_p, c_void_p, c_void_p]),
    "px_full_softmax_sample": (c_int, [c_void_p, c_int, c_int, c_void_p, c_int, c_void_p,
                                       c_int, c_int, c_void_p, c_void_p, c_int,
                                       ctypes.POINTER(GroupGeom), c_int, c_void_p, c_void_p,
                                       c_int, c_void_p, c_int, c_int, c_void_p, c_void_p,
                                       c_void_p, c_float, ctypes.c_uint32, c_int, c_void_p]),
    "px_full_softmax_sample_lse": (c_int, [c_void_p, c_int, c_int, c_void_p, c_int, c_void_p,
                                           c_int, c_int, c_void_p, c_int,
                                           ctypes.POINTER(GroupGeom), c_int, c_void_p, c_void_p,
                                           c_int, c_void_p, c_int, c_float, c_void_p, c_void_p]),
    "px_full_softmax_radix": (c_int, [c_void_p, c_int, c_int, c_void_p, c_int, c_void_p, c_int,
                                      c_int, c_void_p, c_int, ctypes.POINTER(GroupGeom), c_int,
                                      c_void_p, c_void_p, c_int, c_void_p, c_int, c_float,
                                      c_void_p, c_int, c_int, c_float, c_int, c_void_p]),
    "px_full_softmax_sample_masked": (c_int, [c_void_p, c_int, c_int, c_void_p, c_int, c_void_p,
                                              c_int, c_int, c_void_p, c_void_p, c_int,
                                              ctypes.POINTER(GroupGeom), c_int, c_void_p,
                                              c_void_p, c_int, c_void_p, c_int, c_int, c_void_p,
                                              c_void_p, c_void_p, c_float, ctypes.c_uint32,
                                              c_int, c_void_p, c_void_p]),
    "px_sparse_push": (c_int, [c_void_p, c_int, ctypes.POINTER(PushTable), c_int, c_int,
                               c_int, c_int, c_void_p, c_void_p, c_int,
                               ctypes.POINTER(GroupGeom), c_void_p, c_int, c_int, c_int,
                               c_void_p]),
    "px_sparse_owner": (c_int, [ctypes.POINTER(OwnerTable), c_int, c_int, c_void_p,
                                c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                                ctypes.POINTER(GroupGeom), c_void_p, c_int, c_int, c_int,
                                c_int, c_void_p]),
    "px_sparse_owner_norm": (c_int, [ctypes.POINTER(OwnerTable), c_int, c_int, c_void_p,
                                     c_void_p, c_void_p, c_void_p, c_int,
                                     ctypes.POINTER(GroupGeom), c_void_p, c_int, c_int,
                                     c_void_p, c_void_p]),
    "px_linear_xent_tile_cols": (c_int, []),
    "px_linear_xent_logits": (c_int, [c_void_p, c_int, c_int, c_void_p, c_int, c_void_p, c_int,
                                      c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "px_linear_xent_rows": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                    c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "px_clip_hp": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p]),
    "px_stamp": (c_int, [c_void_p, c_void_p]),
}


def available():
    return os.path.exists(LIB)


def check_struct(cls, abi):
    """Raise RuntimeError unless ctypes class `cls` has the layout `abi` (`sparse_abi()`)
    gives the C struct of the same name: the same fields at the same offsets, same size."""
    name = cls.__name__
    ours = {"%s.%s" % (name, f): getattr(cls, f).offset for f, _ in cls._fields_}
    ours[name] = ctypes.sizeof(cls)
    for k in [k for k in abi if k.startswith(name + ".")] + list(ours):
        if abi.get(k) != ours.get(k):
            raise RuntimeError(
                "%s and parallax_b200.ops disagree on %s (%s vs %s; a bare struct name is its "
                "size): rebuild it with `python -m parallax_b200.ops.build`"
                % (LIB, k, abi.get(k), ours.get(k)))


def sparse_abi():
    """The library's `px_sparse_abi()` as a dict: ``group_max``, ``hdr_words``,
    ``ctl_bytes``, ``ctl_time_offset``, ``ctl_overflow_offset``, and per descriptor
    ``Struct`` (its size) and ``Struct.field`` (byte offsets)."""
    lib()
    return _abi


def lib(build_if_missing=True):
    global _lib, _abi
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB):
        if build_if_missing and _nvcc() is not None:
            _build()
        else:
            raise RuntimeError(
                "libparallax_b200.so is missing (%s) and cannot be built: run "
                "`python -m parallax_b200.ops.build`" % LIB)
    L = ctypes.CDLL(LIB, mode=ctypes.RTLD_GLOBAL)
    for name, (res, args) in _SIGS.items():
        try:
            fn = getattr(L, name)
        except AttributeError:
            continue        # optional symbol (added by later build stages)
        fn.restype = res
        fn.argtypes = args
    L.px_sparse_abi.restype = ctypes.c_char_p    # required: a library without it fails here
    abi = {k: int(v) for k, v in (kv.split("=") for kv in L.px_sparse_abi().decode().split())}
    for cls in (GroupGeom, LookupTable, PushTable, OwnerTable):
        check_struct(cls, abi)
    _lib, _abi = L, abi
    return L


def register_signatures(sigs):
    """Let other modules (gemm, runtime) declare their symbols."""
    _SIGS.update(sigs)
    if _lib is not None:
        for name, (res, args) in sigs.items():
            if hasattr(_lib, name):
                fn = getattr(_lib, name)
                fn.restype, fn.argtypes = res, args


def check(rc, what=""):
    if rc != 0:
        msg = ""
        try:
            msg = lib().px_last_error().decode()
        except Exception:
            pass
        raise RuntimeError("native call %s failed (rc=%d) %s" % (what, rc, msg))
