"""Python face of the wgmma/TMA GEMM (`csrc/kernels/gemm_tc.cu`).

`gemm_tn(A, Bt, addend=None, splits=None)` computes ``A @ Bt.T (+ addend)`` in
bf16 with fp32 accumulation, where both operands are K-contiguous
(A: [M, K], Bt: [N, K]) — the layout wgmma consumes directly through
128B-swizzled TMA tiles.  `splits` > 1 spreads the reduction over that many
CTAs per output tile (skinny products: M = batch, K or N huge).
"""
import ctypes

import torch

from .. import consts
from . import lib as _lib, check as _check, register_signatures

_vp, _i = ctypes.c_void_p, ctypes.c_int
register_signatures({
    "px_gemm_tc": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp]),
})

_ws_cache = {}


def _workspace(M, N, device):
    key = (M, N, str(device))
    w = _ws_cache.get(key)
    if w is None:
        w = (torch.zeros(M, N, dtype=torch.float32, device=device),
             torch.zeros(max(1, (M // 128) * (N // 64)), dtype=torch.int32, device=device))
        _ws_cache[key] = w
    return w


def pick_splits(M, N, K, bn=128, sms=consts.NUM_SMS):
    """Enough K-splits to put ~one CTA on every SM, each split ≥ 256 deep."""
    tiles = (M // 128) * (N // bn)
    s = max(1, min(K // 256, sms // max(tiles, 1)))
    while s > 1 and K % (s * 64) != 0:
        s -= 1
    return s


def supported(A, Bt):
    return (A.is_cuda and A.dtype == torch.bfloat16 and Bt.dtype == torch.bfloat16 and
            A.dim() == 2 and Bt.dim() == 2 and A.is_contiguous() and Bt.is_contiguous() and
            A.shape[0] % 128 == 0 and A.shape[1] % 64 == 0 and Bt.shape[0] % 64 == 0 and
            A.data_ptr() % 16 == 0 and Bt.data_ptr() % 16 == 0)


def gemm_tn(A, Bt, addend=None, splits=None, out=None, bn=None, cluster=True):
    M, K = A.shape
    N = Bt.shape[0]
    assert Bt.shape[1] == K
    if bn is None:
        bn = 128 if N % 128 == 0 else 64
    if splits is None:
        splits = pick_splits(M, N, K, bn)
    if out is None:
        out = torch.empty(M, N, dtype=torch.bfloat16, device=A.device)
    # cluster: split-K reduction through distributed shared memory (a thread-block cluster of
    # the K-splits) where the split count allows it, else L2 atomics + ticket + read-back
    cluster = bool(cluster) and 2 <= splits <= 16 and 128 % splits == 0
    ws = tk = None
    if splits > 1 and not cluster:
        ws, tk = _workspace(M, N, A.device)
    from ..parallel import nvops
    nvops.launches["n"] += 1
    rc = _lib().px_gemm_tc(
        _vp(A.data_ptr()), _vp(Bt.data_ptr()), _vp(out.data_ptr()),
        _vp(addend.data_ptr()) if addend is not None else _vp(0),
        _vp(ws.data_ptr()) if ws is not None else _vp(0),
        _vp(tk.data_ptr()) if tk is not None else _vp(0), M, N, K, splits, bn,
        1 if cluster else 0, _vp(torch.cuda.current_stream().cuda_stream))
    _check(rc, "gemm_tc")
    return out
