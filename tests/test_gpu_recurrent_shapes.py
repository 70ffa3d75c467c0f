"""The NMT and skip-thoughts recurrence kernels against fp64 at the edges of what their gates
accept: the LN-GRU cell (`kernels/ln_gru.cu`), the LN-LSTM cell of the `layer_norm_lstm` layer
(`kernels/ln_lstm.cu`, `ln_lstm_cell.cuh`) and the attention decoder's attention, LSTM cell and
LN-LSTM cell kernels (`kernels/nmt_decoder.cu`).  All of them run one 256-thread CTA per batch
row, and their shape-dependent code sits where the benchmark shapes never go:

| family          | shape               | what the shape is there for                                |
|-----------------|---------------------|------------------------------------------------------------|
| LN-GRU          | n 4096              | the largest accepted: every thread owns two full 8-unit groups (G = 2) |
| LN-GRU          | n 2056              | G = 2 with one thread owning a second group                 |
| LN-LSTM layer   | U 2048              | the largest accepted: every thread on, the last warp owns [1792, 2048) |
| LN-LSTM layer   | U 1032              | one thread past 1024 units                                  |
| attention       | S 1024, U 1024, M 2048 | the largest accepted: four passes of each softmax loop, the fp32 values loop's second pass over columns [1024, 2048) |
| attention       | S 1000, U 64, M 128 | a last partial block of 256 source positions                |
| decoder cells   | U 1024 / U 8        | the largest the decoder's gate accepts / one thread on       |

At each shape every kernel runs with NaN in every buffer it writes, a row gap of 8 elements
behind every output that takes a row stride and a NaN sentinel row past every output that does
not; every optional argument is set and every row stride is larger than its row.  The checks:
the written region is finite and within the calibrated bound of `test_gpu_lm1b_numerics`
(error against fp64 within twice that of the same computation in the kernel's dtype, plus a
floor) over each whole output and over each block of 256 units or source positions, so that one
wrong warp cannot hide inside a norm over the whole tensor; gaps and sentinels stay NaN; the
inputs keep their bits; accumulators (`acc` with first = 0, d_keys, d_values, the attention
parameter partials) start from random values and their increments are held to fp64; rows past
their length carry state and gradient through bit for bit; a second launch gives the same bits;
γ/β views at a 2-byte (bf16) or 4-byte (fp32) offset give the bits of aligned copies.

The gates: the largest accepted shape takes the fused node (the launch counts of the layer and
node tests in `test_gpu_ln_gru.py`, `test_gpu_ln_lstm.py` and `test_gpu_nmt_decoder.py`, and the
decoder below), the first refused shape and misaligned weights take the composition, every raw
entry point returns -2 past its limit without launching anything, and the `px_*_max_*` queries
give the documented limits.  Measured ratios are printed (`pytest -s`)."""
import copy
import ctypes
import types

import pytest
import torch
import torch.nn.functional as F

from tests.test_gpu_lm1b_numerics import FACTOR, _assert_calibrated, _errs, _floor
from tests.test_gpu_ln_gru import _cell_operands, _lengths
from tests.test_gpu_nmt_decoder import _DT, _attn_params, _gen, _lib, _p, _pad, _stream

pytestmark = pytest.mark.gpu

_vp = ctypes.c_void_p
NAN = float("nan")
EPS = 1e-5
DTS = [torch.bfloat16, torch.float32]
GAP = 8          # extra elements per row behind every strided output


# ===========================================================================
# helpers
# ===========================================================================
def _bits(t):
    return t.contiguous().reshape(-1).view(torch.uint8)


def _nan(*shape, dt=torch.float32):
    return torch.full(shape, NAN, dtype=dt, device="cuda")


def _strided(x):
    """x [B, w] in the first w columns of a NaN buffer [B, w + GAP]"""
    buf = _nan(x.shape[0], x.shape[1] + GAP, dt=x.dtype)
    buf[:, :x.shape[1]].copy_(x)
    return buf


def _rows(x):
    """x [B, ...] in the first B rows of a NaN buffer [B + 1, ...]"""
    buf = _nan(x.shape[0] + 1, *x.shape[1:], dt=x.dtype)
    buf[:-1].copy_(x)
    return buf


def _at_offset(x):
    """a copy of x as a view one element into a larger buffer (2 bytes in bf16, 4 in fp32)"""
    buf = torch.empty(x.numel() + 1, dtype=x.dtype, device=x.device)
    buf[1:].copy_(x.reshape(-1))
    return buf[1:].view(x.shape)


def _assert_nan(t, what):
    assert torch.isnan(t.float()).all(), "written into " + what


def _share(got, ref, low, dt):
    """the share of its calibrated bound that got's error uses (max of the max-abs and the
    Frobenius criteria of `_within`)"""
    e_k, f_k = _errs(got, ref)
    e_t, f_t = _errs(low, ref)
    floor = _floor(dt, ref.numel())
    bounds = (FACTOR * e_t + floor * float(ref.abs().max()), FACTOR * f_t + floor)
    return max(0.0 if e == 0 else (e / b if b > 0 else float("inf"))
               for e, b in zip((e_k, f_k), bounds))


def _edges(n, step=256):
    return list(range(0, n, step)) + [n]


def _assert_regions(name, got, ref, low, dt, blocks=1, edges=None, dim=-1):
    """the calibrated bound on each region: `dim` split into `blocks` equal blocks, each cut at
    `edges` (default: 256 at a time)"""
    got, ref, low = got.double(), ref.double(), low.double()
    w = ref.shape[dim] // blocks
    edges = edges or _edges(w)
    shares = {}
    for k in range(blocks):
        for a, b in zip(edges[:-1], edges[1:]):
            sl = lambda t: t.narrow(dim, k * w + a, b - a)
            shares[(k, a, b)] = _share(sl(got), sl(ref), sl(low), dt)
    worst = max(shares, key=shares.get)
    print("regions %-40s %3d, worst block %d [%d, %d) at %.3f of its bound"
          % (name, len(shares), *worst, shares[worst]))
    assert all(s <= 1 for s in shares.values()), \
        (name, {k: v for k, v in shares.items() if v > 1})


def _check(name, got, ref, low, dt, blocks=1, edges=None, dim=-1):
    _assert_calibrated(name, got.double(), ref, low.double(), dt)
    _assert_regions(name, got, ref, low, dt, blocks, edges, dim)


def _assert_same_bits(a, b, tag):
    for k in a:
        assert torch.equal(_bits(a[k]), _bits(b[k])), (tag, k)


def _row_leaves(params, B, cdt):
    """γ/β repeated per row as leaves: their gradients are the per-row sums the kernels add to
    their accumulators"""
    return [q.to(cdt).expand(B, -1).clone().requires_grad_(True) for q in params]


def _ln(x, g, b):
    return F.layer_norm(x, x.shape[1:], eps=EPS) * g + b


# ===========================================================================
# LN-GRU cells
# ===========================================================================
def _gru_ref(ops, live, acc0, cdt):
    """one step of the composition in `cdt` by autograd (fp64 is the oracle), acc = acc0 + the
    per-row γ/β gradients in hh's column order"""
    hh, gx, cx, h, prm, dout, carry, drec = ops
    B, n = h.shape
    x = [q.detach().to(cdt).requires_grad_(True) for q in (hh, gx, cx, h)]
    g_wh, b_wh, g_u, b_u = _row_leaves(prm, B, cdt)
    zr = torch.sigmoid(_ln(x[0][:, :2 * n], g_wh, b_wh) + x[1])
    z, r = zr[:, :n], zr[:, n:]
    cand = torch.tanh(r * _ln(x[0][:, 2 * n:], g_u, b_u) + x[2])
    h2 = (1.0 - z) * x[3] + z * cand
    state, out = torch.where(live, h2, x[3]), torch.where(live, h2, torch.zeros_like(h2))
    torch.autograd.backward([out, state], [dout.to(cdt), (carry + drec).to(cdt)])
    inc = torch.cat([g_wh.grad, g_u.grad, b_wh.grad, b_u.grad], 1)
    acc = acc0.double() + inc.double() if cdt == torch.float64 else acc0 + inc.float()
    return {"state": state.detach(), "out": out.detach(), "dhh": x[0].grad, "dgx": x[1].grad,
            "dcx": x[2].grad, "carry": x[3].grad, "acc": acc}


def _gru_run(ops, gx_buf, cx_buf, dout_buf, prm, acc0, lengths, t, dt):
    """both cell kernels with strided gx/cx/dout/out/dgx/dcx and NaN everywhere they write ->
    the whole output buffers (gaps and sentinel rows included)"""
    hh, _, _, h, _, _, carry, drec = ops
    B, n = h.shape
    L, st = _lib(), _stream()
    o = {"state": _nan(B + 1, n, dt=dt), "out": _nan(B, n + GAP, dt=dt), "stats": _nan(B + 1, 4),
         "carry": _rows(carry), "dhh": _nan(B + 1, 3 * n, dt=dt),
         "dgx": _nan(B, 2 * n + GAP, dt=dt), "dcx": _nan(B, n + GAP, dt=dt), "acc": _rows(acc0)}
    pp = [_p(q) for q in prm]
    assert L.px_ln_gru_fwd(_p(hh), _p(gx_buf), gx_buf.stride(0), _p(cx_buf), cx_buf.stride(0),
                           _p(h), _p(o["state"]), _p(o["out"]), n + GAP, _p(o["stats"]), *pp,
                           _p(lengths), t, B, n, EPS, EPS, _DT[dt], st) == 0
    assert L.px_ln_gru_bwd(_p(hh), _p(o["stats"]), _p(gx_buf), gx_buf.stride(0), _p(cx_buf),
                           cx_buf.stride(0), _p(h), _p(dout_buf), dout_buf.stride(0), _p(drec),
                           _p(o["carry"]), _p(o["dhh"]), _p(o["dgx"]), 2 * n + GAP, _p(o["dcx"]),
                           n + GAP, _p(o["acc"]), 0, *pp, _p(lengths), t, B, n, _DT[dt], st) == 0
    torch.cuda.synchronize()
    return o


@pytest.mark.parametrize("n", [4096, 2056])
@pytest.mark.parametrize("dt", DTS)
def test_ln_gru_cells(n, dt):
    B, t = 4, 4
    tag = "gru/%d/%s" % (n, str(dt)[6:])
    ops = _cell_operands(B, n, dt, seed=n + 11)
    hh, gx, cx, h, prm, dout, carry, drec = ops
    lengths = _lengths(B, 9, seed=n)          # row 0 live, row 1 finished at t 4
    live = (lengths > t)[:, None]
    gx_buf, cx_buf, dout_buf = _strided(gx), _strided(cx), _strided(dout)
    acc0 = torch.randn(B, 6 * n, device="cuda", generator=_gen(n)) * 0.1
    inputs = dict(hh=hh, gx=gx_buf, cx=cx_buf, h=h, dout=dout_buf, drec=drec, lengths=lengths,
                  **{"prm%d" % i: q for i, q in enumerate(prm)})
    before = {k: v.clone() for k, v in inputs.items()}
    o = _gru_run(ops, gx_buf, cx_buf, dout_buf, prm, acc0, lengths, t, dt)
    _assert_same_bits(inputs, before, tag + " input")
    for k in ("state", "stats", "carry", "dhh", "acc"):
        _assert_nan(o[k][-1], "%s: the sentinel row of %s" % (tag, k))
    for k, w in (("out", n), ("dgx", 2 * n), ("dcx", n)):
        _assert_nan(o[k][:, w:], "%s: the row gap of %s" % (tag, k))
    got = {"state": o["state"][:B], "out": o["out"][:, :n], "dhh": o["dhh"][:B],
           "dgx": o["dgx"][:, :2 * n], "dcx": o["dcx"][:, :n], "carry": o["carry"][:B],
           "acc": o["acc"][:B]}
    ref = _gru_ref(ops, live, acc0, torch.float64)
    low = _gru_ref(ops, live, acc0, dt)
    blocks = {"dhh": 3, "dgx": 2, "acc": 6}
    for k in got:
        # 256-unit blocks: [0, 2048) is every thread's first group, [2048, n) the second
        _check("%s/%s" % (tag, k), got[k], ref[k], low[k], dt, blocks.get(k, 1))
    dead = ~live[:, 0]
    assert torch.equal(_bits(got["state"][dead]), _bits(h[dead])), tag
    assert torch.equal(_bits(got["carry"][dead]), _bits((carry + drec)[dead])), tag
    assert torch.equal(_bits(got["acc"][dead]), _bits(acc0[dead])), tag
    for k in ("out", "dhh", "dgx", "dcx"):
        assert not got[k][dead].any(), (tag, k)
    _assert_same_bits(o, _gru_run(ops, gx_buf, cx_buf, dout_buf, prm, acc0, lengths, t, dt),
                      tag + " second launch")
    _assert_same_bits(o, _gru_run(ops, gx_buf, cx_buf, dout_buf, [_at_offset(q) for q in prm],
                                  acc0, lengths, t, dt), tag + " γ/β at an offset")


# ===========================================================================
# LN-LSTM cells: the layer's kernels and the decoder's
# ===========================================================================
def _ln_lstm_ref(pre, c, gam, bet, fb, cdt):
    """`LayerNormLSTM.cell` from the pre-LayerNorm gate terms in `cdt`, γ/β as per-row leaves
    -> (h', c', γ leaves, β leaves)"""
    B, U = c.shape
    g, b = _row_leaves(gam, B, cdt), _row_leaves(bet, B, cdt)
    a = [_ln(x, g[k], b[k]) for k, x in enumerate(pre.split(U, 1))]
    c2 = c * torch.sigmoid(a[2] + fb) + torch.sigmoid(a[0]) * torch.tanh(a[1])
    return torch.tanh(_ln(c2, g[4], b[4])) * torch.sigmoid(a[3]), c2, g, b


def _acc_total(acc0, g, b, cdt):
    inc = torch.cat([q.grad for q in g + b], 1)
    return acc0.double() + inc.double() if cdt == torch.float64 else acc0 + inc.float()


def _ln_operands(B, U, dt, seed):
    g = _gen(seed)
    f32 = dict(device="cuda", dtype=torch.float32)
    r = lambda *s: torch.randn(*s, generator=g, **f32)
    x = {"P": r(B, 4 * U) * 2.0 + 0.3, "gx": r(B, 4 * U), "c": r(B, U), "h": r(B, U).to(dt),
         "dout": r(B, U).to(dt), "carry_h": r(B, U), "carry_c": r(B, U), "drec": r(B, U),
         "acc": r(B, 10 * U) * 0.1}
    gam = [(1.0 + 0.3 * r(U)).to(dt) for _ in range(5)]
    bet = [(0.2 * r(U)).to(dt) for _ in range(5)]
    return x, gam, bet


def _ln_ptrs(gam, bet):
    return (_vp * 10)(*[q.data_ptr() for q in gam + bet]), (ctypes.c_float * 5)(*[EPS] * 5)


def _lstm_run(x, bufs, gam, bet, fb, lengths, t, dt):
    """both `px_ln_lstm_*` cell kernels, every row stride U + GAP (4U + GAP) -> output buffers"""
    B, U = x["c"].shape
    L, st = _lib(), _stream()
    ln, ep = _ln_ptrs(gam, bet)
    o = {"c_new": _nan(B + 1, U), "h_next": _nan(B, U + GAP, dt=dt),
         "out": _nan(B, U + GAP, dt=dt), "stats": _nan(B + 1, 10), "carry_h": _rows(x["carry_h"]),
         "carry_c": _rows(x["carry_c"]), "dpre": _nan(B, 4 * U + GAP, dt=dt),
         "acc": _rows(x["acc"])}
    gxb, hb, db = bufs["gx"], bufs["h"], bufs["dout"]
    assert L.px_ln_lstm_fwd(_p(x["P"]), _p(gxb), gxb.stride(0), _p(x["c"]), _p(o["c_new"]), _p(hb),
                            hb.stride(0), _p(o["h_next"]), U + GAP, _p(o["out"]), U + GAP,
                            _p(o["stats"]), ln, ep, fb, _p(lengths), t, B, U, _DT[dt], st) == 0
    assert L.px_ln_lstm_bwd(_p(x["P"]), _p(gxb), gxb.stride(0), _p(o["stats"]), _p(x["c"]),
                            _p(db), db.stride(0), _p(x["drec"]), _p(o["carry_h"]),
                            _p(o["carry_c"]), _p(o["dpre"]), 4 * U + GAP, _p(o["acc"]), 0, ln, ep,
                            fb, _p(lengths), t, B, U, _DT[dt], st) == 0
    torch.cuda.synchronize()
    return o


@pytest.mark.parametrize("U", [2048, 1032])
@pytest.mark.parametrize("dt", DTS)
def test_ln_lstm_cells(U, dt):
    B, t, fb = 4, 2, 1.0
    tag = "ln-lstm/%d/%s" % (U, str(dt)[6:])
    x, gam, bet = _ln_operands(B, U, dt, seed=U + 3)
    lengths = torch.tensor([3, 1, 3, 1], device="cuda")      # rows 0 and 2 live at t 2
    live = (lengths > t)[:, None]
    bufs = {k: _strided(x[k]) for k in ("gx", "h", "dout")}
    inputs = dict(P=x["P"], c=x["c"], drec=x["drec"], lengths=lengths, **bufs,
                  **{"ln%d" % i: q for i, q in enumerate(gam + bet)})
    before = {k: v.clone() for k, v in inputs.items()}
    o = _lstm_run(x, bufs, gam, bet, fb, lengths, t, dt)
    _assert_same_bits(inputs, before, tag + " input")
    for k in ("c_new", "stats", "carry_h", "carry_c", "acc"):
        _assert_nan(o[k][-1], "%s: the sentinel row of %s" % (tag, k))
    for k, w in (("h_next", U), ("out", U), ("dpre", 4 * U)):
        _assert_nan(o[k][:, w:], "%s: the row gap of %s" % (tag, k))
    got = {"c_new": o["c_new"][:B], "h_next": o["h_next"][:, :U], "out": o["out"][:, :U],
           "dpre": o["dpre"][:, :4 * U], "carry_h": o["carry_h"][:B],
           "carry_c": o["carry_c"][:B], "acc": o["acc"][:B]}

    def run(cdt):
        pre = (x["P"].to(cdt) + x["gx"].to(cdt)).requires_grad_(True)
        c = x["c"].to(cdt).requires_grad_(True)
        h2, c2, g, b = _ln_lstm_ref(pre, c, gam, bet, fb, cdt)
        h, dh_t = x["h"].to(cdt), (x["carry_h"] + x["drec"]).to(cdt)
        zero = torch.zeros_like(dh_t)
        dh = torch.where(live, x["dout"].to(cdt) + dh_t, zero)
        dc = torch.where(live, x["carry_c"].to(cdt), zero)
        torch.autograd.backward([h2, c2], [dh, dc])
        return {"c_new": torch.where(live, c2, c).detach(),
                "h_next": torch.where(live, h2, h).detach(),
                "out": torch.where(live, h2, zero).detach(), "dpre": pre.grad,
                "carry_h": torch.where(live, zero, dh_t),
                "carry_c": torch.where(live, c.grad, x["carry_c"].to(cdt)),
                "acc": _acc_total(x["acc"], g, b, cdt)}
    ref, low = run(torch.float64), run(dt)
    blocks = {"dpre": 4, "acc": 10}
    for k in got:
        # 256-unit blocks, one per warp: at U 2048 the last warp owns [1792, 2048)
        _check("%s/%s" % (tag, k), got[k], ref[k], low[k], dt, blocks.get(k, 1))
    dead = ~live[:, 0]
    assert torch.equal(_bits(got["h_next"][dead]), _bits(x["h"][dead])), tag
    assert torch.equal(_bits(got["c_new"][dead]), _bits(x["c"][dead])), tag
    assert torch.equal(_bits(got["carry_h"][dead]), _bits((x["carry_h"] + x["drec"])[dead])), tag
    assert torch.equal(_bits(got["carry_c"][dead]), _bits(x["carry_c"][dead])), tag
    assert torch.equal(_bits(got["acc"][dead]), _bits(x["acc"][dead])), tag
    assert not got["out"][dead].any() and not got["dpre"][dead].any(), tag
    _assert_same_bits(o, _lstm_run(x, bufs, gam, bet, fb, lengths, t, dt), tag + " second launch")
    _assert_same_bits(o, _lstm_run(x, bufs, [_at_offset(q) for q in gam],
                                   [_at_offset(q) for q in bet], fb, lengths, t, dt),
                      tag + " γ/β at an offset")


def _dec_grad_inputs(B, U, dt, seed):
    """the decoder cells' optional inputs, each in a buffer with a row gap"""
    g = _gen(seed)
    r = lambda *s: torch.randn(*s, device="cuda", generator=g)
    y = {"resid": r(B, U).to(dt), "mask": ((r(B, U) > -0.8).float() * 1.25).to(dt),
         "dA": r(B, U), "dA_mask": ((r(B, U) > -0.8).float() * 1.25).to(dt), "dR": r(B, U),
         "dO": r(B, U).to(dt), "drec": r(B, U), "dc": r(B, U)}
    return y, {k: _strided(y[k]) for k in ("resid", "mask", "dA", "dA_mask", "dO", "drec")}


def _dec_dy(y, cdt):
    return (y["dA"].to(cdt) * y["dA_mask"].to(cdt) + y["dR"].to(cdt) + y["dO"].to(cdt))


def _dec_outs(B, U, dt):
    return {"c": _nan(B + 1, U), "h": _nan(B, U + GAP, dt=dt), "y": _nan(B, U + GAP, dt=dt),
            "xn": _nan(B, U + GAP, dt=dt), "dG": _nan(B + 1, 4 * U, dt=dt),
            "dY": _nan(B + 1, U)}


def _dec_ld(b, name):
    return _p(b[name]), b[name].stride(0)


def _dec_check_layout(o, B, U, tag):
    for k in ("c", "dG", "dY", "dc") + (("stats", "acc") if "acc" in o else ()):
        _assert_nan(o[k][-1], "%s: the sentinel row of %s" % (tag, k))
    for k in ("h", "y", "xn"):
        _assert_nan(o[k][:, U:], "%s: the row gap of %s" % (tag, k))
    got = {k: o[k][:, :U] if k in ("h", "y", "xn") else o[k][:B] for k in o if k != "stats"}
    return got


def _ln_dec_run(x, y, bufs, gam, bet, fb, dt):
    """`px_nmt_ln_lstm_cell_fwd` / `bwd` with every optional argument and row stride"""
    B, U = x["c"].shape
    L, st = _lib(), _stream()
    ln, ep = _ln_ptrs(gam, bet)
    o = _dec_outs(B, U, dt)
    o.update(stats=_nan(B + 1, 10), dc=_rows(y["dc"]), acc=_rows(x["acc"]))
    assert L.px_nmt_ln_lstm_cell_fwd(_p(x["P"]), _p(x["gx"]), _p(x["c"]), _p(o["c"]), _p(o["h"]),
                                     U + GAP, *_dec_ld(bufs, "resid"), _p(o["y"]), U + GAP,
                                     *_dec_ld(bufs, "mask"), _p(o["xn"]), U + GAP,
                                     _p(o["stats"]), ln, ep, fb, B, U, _DT[dt], st) == 0
    assert L.px_nmt_ln_lstm_cell_bwd(_p(x["P"]), _p(x["gx"]), _p(o["stats"]), _p(x["c"]),
                                     *_dec_ld(bufs, "dA"), *_dec_ld(bufs, "dA_mask"),
                                     _p(y["dR"]), *_dec_ld(bufs, "dO"), *_dec_ld(bufs, "drec"),
                                     _p(o["dc"]), _p(o["dG"]), _p(o["dY"]), _p(o["acc"]), 0, ln,
                                     ep, fb, B, U, _DT[dt], st) == 0
    torch.cuda.synchronize()
    return o


@pytest.mark.parametrize("U", [1024, 8])
@pytest.mark.parametrize("dt", DTS)
def test_decoder_ln_lstm_cells(U, dt):
    B, fb = 4, 1.0
    tag = "dec-ln/%d/%s" % (U, str(dt)[6:])
    x, gam, bet = _ln_operands(B, U, dt, seed=U + 5)
    y, bufs = _dec_grad_inputs(B, U, dt, seed=U + 6)
    inputs = dict(P=x["P"], gx=x["gx"], c=x["c"], dR=y["dR"], **bufs,
                  **{"ln%d" % i: q for i, q in enumerate(gam + bet)})
    before = {k: v.clone() for k, v in inputs.items()}
    o = _ln_dec_run(x, y, bufs, gam, bet, fb, dt)
    _assert_same_bits(inputs, before, tag + " input")
    got = _dec_check_layout(o, B, U, tag)

    def run(cdt):
        pre = (x["P"].to(cdt) + x["gx"].to(cdt)).requires_grad_(True)
        c = x["c"].to(cdt).requires_grad_(True)
        h2, c2, g, b = _ln_lstm_ref(pre, c, gam, bet, fb, cdt)
        yy = h2 + y["resid"].to(cdt)
        dy = _dec_dy(y, cdt)
        torch.autograd.backward([h2, c2], [dy + y["drec"].to(cdt), y["dc"].to(cdt)])
        return {"c": c2.detach(), "h": h2.detach(), "y": yy.detach(),
                "xn": (yy * y["mask"].to(cdt)).detach(), "dG": pre.grad, "dY": dy,
                "dc": c.grad, "acc": _acc_total(x["acc"], g, b, cdt)}
    ref, low = run(torch.float64), run(dt)
    blocks = {"dG": 4, "acc": 10}
    for k in got:
        _check("%s/%s" % (tag, k), got[k], ref[k], low[k], dt, blocks.get(k, 1))
    _assert_same_bits(o, _ln_dec_run(x, y, bufs, gam, bet, fb, dt), tag + " second launch")
    _assert_same_bits(o, _ln_dec_run(x, y, bufs, [_at_offset(q) for q in gam],
                                     [_at_offset(q) for q in bet], fb, dt),
                      tag + " γ/β at an offset")


def _plain_dec_run(x, y, bufs, b_ih, b_hh, dt):
    """`px_nmt_lstm_cell_fwd` / `bwd` with every optional argument and row stride"""
    B, U = x["c"].shape
    L, st = _lib(), _stream()
    o = _dec_outs(B, U, dt)
    o["dc"] = _rows(y["dc"])
    assert L.px_nmt_lstm_cell_fwd(_p(x["P"]), _p(x["gx"]), _p(b_ih), _p(b_hh), _p(x["c"]),
                                  _p(o["c"]), _p(o["h"]), U + GAP, *_dec_ld(bufs, "resid"),
                                  _p(o["y"]), U + GAP, *_dec_ld(bufs, "mask"), _p(o["xn"]),
                                  U + GAP, B, U, _DT[dt], st) == 0
    assert L.px_nmt_lstm_cell_bwd(_p(x["P"]), _p(x["gx"]), _p(b_ih), _p(b_hh), _p(x["c"]),
                                  _p(o["c"]), *_dec_ld(bufs, "dA"), *_dec_ld(bufs, "dA_mask"),
                                  _p(y["dR"]), *_dec_ld(bufs, "dO"), *_dec_ld(bufs, "drec"),
                                  _p(o["dc"]), _p(o["dG"]), _p(o["dY"]), B, U, _DT[dt], st) == 0
    torch.cuda.synchronize()
    return o


@pytest.mark.parametrize("dt", DTS)
def test_decoder_lstm_cells_strided(dt):
    B, U = 4, 1024
    tag = "dec-lstm/%d/%s" % (U, str(dt)[6:])
    x, _, _ = _ln_operands(B, U, dt, seed=U + 7)
    y, bufs = _dec_grad_inputs(B, U, dt, seed=U + 8)
    g = _gen(U + 9)
    b_ih = (torch.randn(4 * U, device="cuda", generator=g) * 0.3).to(dt)
    b_hh = (torch.randn(4 * U, device="cuda", generator=g) * 0.3).to(dt)
    inputs = dict(P=x["P"], gx=x["gx"], c=x["c"], dR=y["dR"], b_ih=b_ih, b_hh=b_hh, **bufs)
    before = {k: v.clone() for k, v in inputs.items()}
    o = _plain_dec_run(x, y, bufs, b_ih, b_hh, dt)
    _assert_same_bits(inputs, before, tag + " input")
    got = _dec_check_layout(o, B, U, tag)

    def run(cdt):
        pre = (x["P"].to(cdt) + x["gx"].to(cdt) + b_ih.to(cdt) + b_hh.to(cdt)).requires_grad_(True)
        c_prev = x["c"].to(cdt).requires_grad_(True)
        i, f, gg, og = pre.chunk(4, -1)
        c = torch.sigmoid(f) * c_prev + torch.sigmoid(i) * torch.tanh(gg)
        h = torch.sigmoid(og) * torch.tanh(c)
        yy = h + y["resid"].to(cdt)
        dy = _dec_dy(y, cdt)
        torch.autograd.backward([h, c], [dy + y["drec"].to(cdt), y["dc"].to(cdt)])
        return {"c": c.detach(), "h": h.detach(), "y": yy.detach(),
                "xn": (yy * y["mask"].to(cdt)).detach(), "dG": pre.grad, "dY": dy,
                "dc": c_prev.grad}
    ref, low = run(torch.float64), run(dt)
    for k in got:
        _check("%s/%s" % (tag, k), got[k], ref[k], low[k], dt, 4 if k == "dG" else 1)
    _assert_same_bits(o, _plain_dec_run(x, y, bufs, b_ih, b_hh, dt), tag + " second launch")


# ===========================================================================
# attention kernels
# ===========================================================================
def _attn_ref(x, prm, pad, bah, cdt):
    """one attention step in `cdt` by autograd with every optional term, and the attention
    parameters per row (their gradients are the kernel's per-row partials)"""
    B = x["keys"].shape[0]
    lv = [(x["pq"] if bah else x["q"]).to(cdt), x["keys"].to(cdt), x["values"].to(cdt)]
    lv = [t.detach().requires_grad_(True) for t in lv]
    pr = {k: None if t is None else t.reshape(1, -1).to(x["keys"].dtype).to(cdt)
          for k, t in prm.items()}
    if bah:
        pr["v"] = prm["v"].to(cdt).reshape(1, -1)
    rows = {k: t.expand(B, -1).clone().requires_grad_(True) for k, t in pr.items()
            if t is not None}
    if bah:
        hid = lv[1] + lv[0][:, None, :]
        if "b" in rows:
            hid = hid + rows["b"][:, None, :]
        s = (torch.tanh(hid) * rows["v"][:, None, :]).sum(-1)
    else:
        s = torch.bmm(lv[0][:, None, :], lv[1].transpose(1, 2))[:, 0]
        if "g" in rows:
            s = s * rows["g"]
    a = torch.softmax(s.masked_fill(pad, float("-inf")), -1)
    ctx = torch.bmm(a[:, None, :], lv[2])[:, 0]
    d_ctx = x["dA"].to(cdt) * x["dA_mask"].to(cdt) + x["dO"].to(cdt)
    ctx.backward(d_ctx)
    acc = lambda k, inc: x[k].double() + inc.double() if cdt == torch.float64 \
        else x[k] + inc.float()
    out = {"ctx": ctx.detach(), "feed": ctx.detach() * x["fmask"].to(cdt), "align": a.detach(),
           "dk": acc("dk", lv[1].grad), "dv": acc("dv", lv[2].grad), "dq": lv[0].grad}
    if bah:
        out["part_v"] = acc("part_v", rows["v"].grad)
        if "b" in rows:
            out["part_b"] = acc("part_b", rows["b"].grad)
    elif "g" in rows:
        out["part_g"] = acc("part_g", rows["g"].grad[:, 0])
    return out


def _attn_run(x, bufs, prm, pad, kind, dt):
    """both attention kernels with every optional argument and row stride set -> buffers"""
    B, S, U = x["keys"].shape
    M = x["values"].shape[2]
    L, st = _lib(), _stream()
    gt = None if prm["g"] is None else prm["g"].to(dt)
    bt = None if prm["b"] is None else prm["b"].to(dt)
    o = {"ctx": _nan(B, M + GAP, dt=dt), "feed": _nan(B, M + GAP, dt=dt),
         "align": _nan(B + 1, S), "dq": _nan(B + 1, U), "dpq": _nan(B + 1, U, dt=dt),
         "dk": _rows(x["dk"]), "dv": _rows(x["dv"]), "part_g": _rows(x["part_g"]),
         "part_v": _rows(x["part_v"]), "part_b": _rows(x["part_b"])}
    qb = bufs["q"]
    assert L.px_nmt_attn_fwd(_p(qb), qb.stride(0), _p(x["pq"]), _p(x["keys"]), _p(x["values"]),
                             _p(pad), _p(gt), _p(prm["v"]), _p(bt), _p(o["ctx"]), M + GAP,
                             *_dec_ld(bufs, "fmask"), _p(o["feed"]), M + GAP, _p(o["align"]),
                             B, S, U, M, kind, _DT[dt], st) == 0
    bah = kind == 1
    assert L.px_nmt_attn_bwd(*_dec_ld(bufs, "dA"), *_dec_ld(bufs, "dA_mask"),
                             *_dec_ld(bufs, "dO"), _p(o["align"]), _p(qb), qb.stride(0),
                             _p(x["pq"]), _p(x["keys"]), _p(x["values"]), _p(gt), _p(prm["v"]),
                             _p(bt), None if bah else _p(o["dq"]), _p(o["dpq"]) if bah else None,
                             _p(o["dk"]), _p(o["dv"]), _p(o["part_g"]),
                             _p(o["part_v"]) if bah else None,
                             _p(o["part_b"]) if bt is not None else None,
                             B, S, U, M, kind, _DT[dt], st) == 0
    torch.cuda.synchronize()
    return o


ATTN_SHAPES = [(3, 1024, 1024, 2048), (3, 1000, 64, 128)]


@pytest.mark.parametrize("B,S,U,M", ATTN_SHAPES, ids=["S%d-U%d-M%d" % s[1:] for s in ATTN_SHAPES])
@pytest.mark.parametrize("option", ["luong", "scaled_luong", "bahdanau", "normed_bahdanau"])
@pytest.mark.parametrize("dt", DTS)
def test_attention_kernels(B, S, U, M, option, dt):
    bah = option in ("bahdanau", "normed_bahdanau")
    tag = "attn/%s/S%d/%s" % (option, S, str(dt)[6:])
    g = _gen(S + U + M)
    r = lambda *s: torch.randn(*s, device="cuda", generator=g)
    pad = _pad(B, S, S + 1)
    x = {"q": (r(B, U) / U ** 0.5).to(dt), "pq": r(B, U) * 0.5, "keys": r(B, S, U).to(dt),
         "values": r(B, S, M).masked_fill(pad[..., None], 0).to(dt),
         "fmask": ((r(B, M) > -0.8).float() * 1.25).to(dt), "dA": r(B, M),
         "dA_mask": ((r(B, M) > -0.8).float() * 1.25).to(dt), "dO": r(B, M).to(dt),
         "dk": r(B, S, U) * 0.01, "dv": r(B, S, M) * 0.01, "part_g": r(B) * 0.1,
         "part_v": r(B, U) * 0.1, "part_b": r(B, U) * 0.1}
    prm = _attn_params(option, U, seed=U + 1)
    bufs = {k: _strided(x[k]) for k in ("q", "fmask", "dA", "dA_mask", "dO")}
    inputs = dict(pq=x["pq"], keys=x["keys"], values=x["values"], pad=pad, **bufs,
                  **{k: v for k, v in prm.items() if v is not None})
    before = {k: v.clone() for k, v in inputs.items()}
    kind = 1 if bah else 0
    o = _attn_run(x, bufs, prm, pad, kind, dt)
    _assert_same_bits(inputs, before, tag + " input")
    for k in ("ctx", "feed"):
        _assert_nan(o[k][:, M:], "%s: the row gap of %s" % (tag, k))
    outs = ["ctx", "feed", "align", "dk", "dv"] + (["dpq", "part_v"] if bah else ["dq"])
    if bah and prm["b"] is not None:
        outs.append("part_b")
    if not bah and prm["g"] is not None:
        outs.append("part_g")
    for k in outs:
        if k not in ("ctx", "feed"):
            _assert_nan(o[k][-1], "%s: the sentinel row of %s" % (tag, k))
    # untouched optional outputs keep their NaN or their start values
    for k in {"dq", "dpq", "part_g", "part_v", "part_b"} - set(outs):
        if k in ("dq", "dpq"):
            _assert_nan(o[k], "%s: %s, which this kind does not write" % (tag, k))
        else:
            assert torch.equal(_bits(o[k][:B]), _bits(x[k])), (tag, k)
    got = {k: o[k][:, :M] if k in ("ctx", "feed") else o[k][:B] for k in outs}
    got["dq"] = got.pop("dpq") if bah else got["dq"]
    ref = _attn_ref(x, prm, pad, bah, torch.float64)
    low = _attn_ref(x, prm, pad, bah, dt)
    s_edges = _edges(S)                                  # 256 source positions per pass
    m_edges = [0, 1024, M] if M > 1024 else None         # fp32: the values loop's two passes
    for k in got:
        name = "%s/%s" % (tag, k)
        _assert_calibrated(name, got[k].double(), ref[k], low[k].double(), dt)
        if k in ("align", "dk", "dv"):
            _assert_regions(name + "/s", got[k], ref[k], low[k], dt, edges=s_edges, dim=1)
        if k in ("ctx", "feed", "dv") and m_edges:
            _assert_regions(name + "/m", got[k], ref[k], low[k], dt, edges=m_edges)
    _assert_same_bits(o, _attn_run(x, bufs, prm, pad, kind, dt), tag + " second launch")


# ===========================================================================
# gates
# ===========================================================================
def test_limits_are_the_documented_ones():
    L = _lib()
    assert L.px_ln_gru_max_units() == 4096
    assert L.px_ln_lstm_max_units() == 2048
    assert (L.px_nmt_max_units(), L.px_nmt_max_memory(), L.px_nmt_max_source()) == \
        (1024, 2048, 1024)


def test_raw_entry_points_refuse_past_their_limits():
    """-2 at the first shape past each limit (and, for the LN-LSTM layer kernels, at a row stride
    that is not a multiple of 8), before any launch: every pointer is one zeroed scratch buffer
    large enough for the B 1 shape, and it is still zero afterwards"""
    L, st = _lib(), _stream()
    scratch = torch.zeros(1 << 23, device="cuda")
    z = _p(scratch)
    ln, ep = (_vp * 10)(*[scratch.data_ptr()] * 10), (ctypes.c_float * 5)(*[EPS] * 5)
    calls = {}
    for dt in (0, 1):
        n = 4104
        calls["gru_fwd", dt] = L.px_ln_gru_fwd(z, z, 2 * n, z, n, z, z, z, n, z, z, z, z, z, None,
                                               0, 1, n, EPS, EPS, dt, st)
        calls["gru_bwd", dt] = L.px_ln_gru_bwd(z, z, z, 2 * n, z, n, z, z, n, z, z, z, z, 2 * n,
                                               z, n, z, 1, z, z, z, z, None, 0, 1, n, dt, st)
        calls["gru_param", dt] = L.px_ln_gru_param_grad(z, 1, n, z, z, z, z, dt, st)
        for U, ld in ((2056, 0), (2048, 4)):      # past the limit / a stride off by 4 elements
            g4, u = 4 * U + ld, U + ld
            calls["lstm_fwd", U, dt] = L.px_ln_lstm_fwd(z, z, g4, z, z, z, u, z, u, z, u, z, ln,
                                                        ep, 1.0, None, 0, 1, U, dt, st)
            calls["lstm_bwd", U, dt] = L.px_ln_lstm_bwd(z, z, g4, z, z, z, u, z, z, z, z, g4, z,
                                                        1, ln, ep, 1.0, None, 0, 1, U, dt, st)
        calls["lstm_param", dt] = L.px_ln_lstm_param_grad(z, 1, 2056, z, dt, st)
        for S, U, M in ((1025, 64, 64), (16, 1032, 64), (16, 64, 2056)):
            for kind in (0, 1):
                calls["attn_fwd", S, U, M, kind, dt] = L.px_nmt_attn_fwd(
                    z, U, z, z, z, z, None, z, None, z, M, None, 0, z, M, z, 1, S, U, M, kind,
                    dt, st)
                calls["attn_bwd", S, U, M, kind, dt] = L.px_nmt_attn_bwd(
                    z, M, None, 0, None, 0, z, z, U, z, z, z, None, z, None, z, z, z, z, z, z,
                    None, 1, S, U, M, kind, dt, st)
        U = 2056
        calls["dec_ln_fwd", dt] = L.px_nmt_ln_lstm_cell_fwd(z, z, z, z, z, U, None, 0, z, U, None,
                                                            0, z, U, z, ln, ep, 1.0, 1, U, dt, st)
        calls["dec_ln_bwd", dt] = L.px_nmt_ln_lstm_cell_bwd(z, z, z, z, z, U, None, 0, z, None, 0,
                                                            z, U, z, z, z, z, 1, ln, ep, 1.0, 1,
                                                            U, dt, st)
    torch.cuda.synchronize()
    assert {k: v for k, v in calls.items() if v != -2} == {}
    assert not scratch.any(), "a refused call launched a kernel"


def _ns(**kw):
    return types.SimpleNamespace(**kw)


def _forbid(monkeypatch, name):
    from parallax_b200.ops import fused
    monkeypatch.setattr(fused, name, lambda *a, **k: pytest.fail("the fused node ran"))


def test_ln_gru_gate_boundary(monkeypatch):
    """n 4096 is accepted (the layer cases run it on the node), 4104 and a w_hu at a 4-byte
    offset take the composition, which matches fp64"""
    from parallax_b200.ops import fused
    from tests.test_gpu_ln_gru import _layer_data, _module, _run_layer
    x = torch.zeros(1, 1, 8, device="cuda")
    for n, ok in ((4096, True), (4104, False)):
        ln = lambda k: _ns(weight=torch.ones(k, device="cuda"), bias=torch.zeros(k, device="cuda"))
        assert fused.ln_gru_applies(x, torch.zeros(n, 3 * n, device="cuda"), ln(2 * n), ln(n)) == ok
    _forbid(monkeypatch, "ln_gru_layer")
    m = _module(8, 4104, seed=1)
    data = _layer_data(2, 8, 2, 4104, True, True, seed=2)
    got = _run_layer(m, torch.float32, data, composition=False)
    comp = _run_layer(m, torch.float32, data, composition=True)
    ref = _run_layer(m, torch.float64, data, composition=True)
    for k in got:
        assert torch.equal(got[k], comp[k]), k
        torch.testing.assert_close(got[k].double(), ref[k], rtol=1e-3, atol=1e-4)
    m = _module(8, 64, seed=3)
    w = m.w_hu.detach()
    m.w_hu = torch.nn.Parameter(_at_offset(w))
    assert m.w_hu.data_ptr() % 16
    a, fa = m(data[0], data[1], None, reverse=True)
    b, fb = m._composition(data[0], data[1], None, reverse=True)
    assert torch.equal(a, b) and torch.equal(fa, fb)


def test_ln_lstm_gate_boundary(monkeypatch):
    """U 2048 is accepted (the layer cases run it on the node), 2056 and a kernel weight at a
    4-byte offset take the composition, which matches fp64"""
    from parallax_b200.ops import fused
    from tests.test_gpu_ln_lstm import _layer_data, _module, _run_layer
    x = torch.zeros(1, 1, 8, device="cuda")
    for U, ok in ((2048, True), (2056, False)):
        ln = [_ns(weight=torch.ones(U, device="cuda"), bias=torch.zeros(U, device="cuda"), eps=EPS)
              for _ in range(5)]
        w = torch.zeros(4 * U, 8 + U, device="cuda")
        assert fused.ln_lstm_applies(x, w, ln[:4], ln[4]) == ok
    _forbid(monkeypatch, "ln_lstm_layer")
    m = _module(8, 2056, seed=1)
    data = _layer_data(2, 2, 8, 2056, True, seed=2)
    got = _run_layer(m, torch.float32, data, composition=False)
    comp = _run_layer(m, torch.float32, data, composition=True)
    ref = _run_layer(m, torch.float64, data, composition=True)
    for k in got:
        assert torch.equal(got[k], comp[k]), k
        torch.testing.assert_close(got[k].double(), ref[k], rtol=1e-3, atol=1e-4)
    m = _module(8, 64, seed=3)
    m.kernel.weight = torch.nn.Parameter(_at_offset(m.kernel.weight.detach()))
    assert m.kernel.weight.data_ptr() % 16
    st = (torch.zeros(2, 64, device="cuda"), torch.zeros(2, 64, device="cuda"))
    a, (ha, ca) = m(data[0], st, data[1])
    b, (hb, cb) = m._composition(data[0], st, data[1])
    assert torch.equal(a, b) and torch.equal(ha, hb) and torch.equal(ca, cb)


def test_ln_lstm_layer_with_layernorm_parameters_at_an_offset():
    """the layer node through its gate, with every γ/β a view at a 2-byte offset, gives the bits
    of the same values in fresh aligned tensors, forward and backward"""
    from parallax_b200.parallel import nvops
    from tests.test_gpu_ln_lstm import _layer_data, _module
    m = _module(16, 1032, seed=4).to(torch.bfloat16)
    m2 = copy.deepcopy(m)
    for ln in list(m2.ln) + [m2.ln_c]:
        ln.weight = torch.nn.Parameter(_at_offset(ln.weight.detach()))
        ln.bias = torch.nn.Parameter(_at_offset(ln.bias.detach()))
        assert ln.weight.data_ptr() % 4 == 2
    x, lengths, h0, c0 = _layer_data(3, 3, 16, 1032, True, seed=5)[:4]

    def run(mod):
        xl = x.to(torch.bfloat16).requires_grad_(True)
        st = (h0.to(torch.bfloat16), c0.to(torch.bfloat16))
        l0 = nvops.launches["n"]
        out, (h, c) = mod(xl, st, lengths)
        (out.float().sum() + h.float().sum() + c.float().sum()).backward()
        assert nvops.launches["n"] - l0 == 2 * 3 + 1       # the fused node ran: T fwd, T + 1 bwd
        return [out, h, c, xl.grad] + [p.grad for p in mod.parameters()]
    for a, b in zip(run(m), run(m2)):
        assert torch.equal(_bits(a), _bits(b))


def _decoder(U, M, unit, seed):
    import parallax_b200.models.nmt as nmt
    from parallax_b200.models.nmt.model import Decoder
    torch.manual_seed(seed)
    hp = nmt.create_hparams(num_units=U, num_layers=1, encoder_type="uni", attention="luong",
                            attention_architecture="standard", residual=False, dropout=0.0,
                            unit_type=unit)
    nmt.extend_hparams(hp, 40, 40)
    return Decoder(hp, M).cuda()


def _decode(dec, enc, lengths, emb, dt):
    d = copy.deepcopy(dec).to(dt)
    keys, values, pad = d.attention.prepare(enc.to(dt), lengths)
    B = emb.shape[0]
    state = {"cells": [l.zero_state(B, emb.device, dt) for l in d.layers],
             "attention": torch.zeros(B, d.attention_size, device=emb.device, dtype=dt)}
    with torch.no_grad():
        return d(emb.to(dt), state, (keys, values, pad)), \
            d._composition(emb.to(dt), state, (keys, values, pad))


@pytest.mark.parametrize("unit", ["lstm", "layer_norm_lstm"])
@pytest.mark.parametrize("U,M,S,fused_ok", [(1024, 2048, 1024, True), (1032, 64, 16, False),
                                            (64, 2056, 16, False), (64, 64, 1025, False)])
def test_decoder_gate_boundary(U, M, S, fused_ok, unit, monkeypatch):
    """the largest accepted (U, M, S) runs the node, the first refused U, M or S the
    composition; both match fp64"""
    from parallax_b200.ops import fused
    from parallax_b200.parallel import nvops
    B, T = 3, 2
    dec = _decoder(U, M, unit, seed=U + M + S)
    g = _gen(S)
    enc = torch.randn(B, S, M, device="cuda", generator=g)
    emb = torch.randn(B, T, U, device="cuda", generator=g)
    lengths = torch.tensor([S, 1, S // 2 + 1], device="cuda")
    calls = {"n": 0, "launches": 0}
    if fused_ok:
        real = fused.nmt_attention_decoder

        def spy(*a, **k):
            l0 = nvops.launches["n"]
            out = real(*a, **k)
            calls["n"] += 1
            calls["launches"] += nvops.launches["n"] - l0
            return out
        monkeypatch.setattr(fused, "nmt_attention_decoder", spy)
    else:
        _forbid(monkeypatch, "nmt_attention_decoder")
    got, comp = _decode(dec, enc, lengths, emb, torch.float32)
    assert calls["n"] == int(fused_ok)
    assert calls["launches"] == (T * 2 if fused_ok else 0)    # T steps of one layer + attention
    ref, _ = _decode(dec, enc, lengths, emb, torch.float64)
    tag = "dec-gate/%s/U%d/M%d/S%d" % (unit, U, M, S)
    if fused_ok:
        _assert_calibrated(tag, got.double(), ref, comp.double(), torch.float32)
    else:
        assert torch.equal(got, comp), tag
        torch.testing.assert_close(got.double(), ref, rtol=1e-3, atol=1e-4)
