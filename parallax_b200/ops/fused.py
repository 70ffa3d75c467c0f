"""Fused model-side ops (autograd Functions) for the LM1B hot path.

`lstm_layer`  — a whole unrolled LSTMP layer as ONE autograd node: the
  sequential part is one persistent kernel for all T forward steps and one for
  all T backward steps (bf16, batch 128; elsewhere, forward, 2 small GEMMs + 1
  fused cell kernel per time step and, backward, 2 GEMMs per step, the first
  with the cell backward in its epilogue for bf16, else 2 GEMMs + 1 fused
  kernel); every weight gradient is a single GEMM batched over all time steps
  (the reference's TF graph issues one small GEMM + ~25 elementwise kernels per
  step and direction:
  `examples/lm1b/language_model.py:76-87`).
`sampled_softmax_loss` — logits GEMM + one fused kernel that produces the
  loss and the softmax probabilities in place (= gradient wrt logits), so the
  backward is two GEMMs and a few row scalings.

Both have a pure-PyTorch implementation (`*_reference`) which is the numerics
oracle in the tests and the path used on the host fabric.
`ln_gru_layer` — the skip-thoughts layer-normalised GRU recurrence as ONE autograd node: per
  time step a cuBLAS product in fp32 and one cell kernel forward, one cell kernel and a cuBLAS
  product backward (`kernels/ln_gru.cu`); `w_hu`'s gradient is one GEMM over all steps.  Its
  oracle is the composition in `LayerNormGRU._composition`.
`ln_lstm_layer` — the NMT layer-normalised LSTM layer as ONE autograd node: the input side as
  one cuBLAS product before the loop, then per time step a cuBLAS product in fp32 and one cell
  kernel forward, one cell kernel and a cuBLAS product backward (`kernels/ln_lstm.cu`); the
  kernel weight's gradient and the input gradient are one GEMM each over all steps.  Its oracle
  is `LayerNormLSTM._composition`.
`nmt_attention_decoder` — the NMT decoder's attention recurrence (standard: every layer; gnmt:
  the bottom layer) as ONE autograd node: per time step a cuBLAS product and one cell kernel per
  layer and one attention kernel (`kernels/nmt_decoder.cu`) each way; every weight gradient is one
  GEMM over all steps; with `ln` the cells are layer-normalised LSTMs (`LayerNormLSTM.cell`).
  Its oracle is `nmt_attention_decoder_reference`, which equals
  `Decoder._composition`.
`linear_cross_entropy` — a dense output layer and its softmax cross entropy without the [N, V]
  logits: per chunk of rows one wgmma logits kernel with a log-sum-exp epilogue and one row
  kernel (`kernels/linear_xent.cu`), the gradient formed in the forward.  Its oracle is
  `linear_cross_entropy_reference`.
"""
import ctypes

import torch
import torch.nn.functional as F

from . import lib as _lib, check as _check, register_signatures

_vp, _i, _f = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
register_signatures({
    "px_lstm_cell_fwd": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _f, _i, _vp]),
    "px_lstm_cell_bwd": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "px_lstm_dm_cell_bwd": (_i, [_vp] * 7 + [_i, _i, _i, _i, _vp]),
    "px_lstm_fwd_persistent_grid": (_i, [_i, _i, _i]),
    "px_lstm_fwd_persistent": (_i, [_vp] * 8 + [_i, _i, _i, _i, _f, _vp]),
    "px_lstm_bwd_persistent_grid": (_i, [_i, _i, _i]),
    "px_lstm_bwd_persistent": (_i, [_vp] * 10 + [_i, _i, _i, _i, _vp]),
    "px_sampled_softmax": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "px_sampled_softmax_dot": (_i, [_vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i,
                                    _vp]),
    "px_ssm_bwd": (_i, [_vp, _vp, _vp, _vp, _i, _vp, _vp, _f, _vp, _vp, _vp, _i, _vp, _i, _i, _i,
                        _vp]),
    "px_ln_gru_max_units": (_i, []),
    "px_ln_gru_fwd": (_i, [_vp, _vp, _i, _vp, _i, _vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp, _vp,
                           _i, _i, _i, _f, _f, _i, _vp]),
    "px_ln_gru_bwd": (_i, [_vp, _vp, _vp, _i, _vp, _i, _vp, _vp, _i, _vp, _vp, _vp, _vp, _i, _vp,
                           _i, _vp, _i, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "px_ln_gru_param_grad": (_i, [_vp, _i, _i, _vp, _vp, _vp, _vp, _i, _vp]),
    "px_ln_lstm_max_units": (_i, []),
    "px_ln_lstm_fwd": (_i, [_vp, _vp, _i, _vp, _vp, _vp, _i, _vp, _i, _vp, _i, _vp, _vp, _vp, _f,
                            _vp, _i, _i, _i, _i, _vp]),
    "px_ln_lstm_bwd": (_i, [_vp, _vp, _i, _vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _i, _vp, _i, _vp,
                            _vp, _f, _vp, _i, _i, _i, _i, _vp]),
    "px_ln_lstm_param_grad": (_i, [_vp, _i, _i, _vp, _i, _vp]),
    "px_nmt_max_units": (_i, []),
    "px_nmt_max_memory": (_i, []),
    "px_nmt_max_source": (_i, []),
    "px_nmt_attn_fwd": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _vp, _i, _vp,
                             _i, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "px_nmt_attn_bwd": (_i, [_vp, _i, _vp, _i, _vp, _i, _vp, _vp, _i] + [_vp] * 13 +
                        [_i, _i, _i, _i, _i, _i, _vp]),
    "px_nmt_attn_param_grad": (_i, [_vp, _i, _i, _vp, _vp]),
    "px_nmt_lstm_cell_fwd": (_i, [_vp] * 6 + [_vp, _i, _vp, _i, _vp, _i, _vp, _i, _vp, _i,
                                              _i, _i, _i, _vp]),
    "px_nmt_lstm_cell_bwd": (_i, [_vp] * 6 + [_vp, _i, _vp, _i, _vp, _vp, _i, _vp, _i, _vp, _vp,
                                              _vp, _i, _i, _i, _vp]),
    "px_nmt_ln_lstm_cell_fwd": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _vp, _i, _vp, _i, _vp, _i, _vp,
                                     _i, _vp, _vp, _vp, _f, _i, _i, _i, _vp]),
    "px_nmt_ln_lstm_cell_bwd": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _vp, _i, _vp, _vp, _i, _vp, _i,
                                     _vp, _vp, _vp, _vp, _i, _vp, _vp, _f, _i, _i, _i, _vp]),
})
_DT = {torch.float32: 0, torch.bfloat16: 1}


def _p(t):
    return _vp(t.data_ptr())


def _stream():
    return _vp(torch.cuda.current_stream().cuda_stream)


def _count(n=1):
    from ..parallel import nvops
    nvops.launches["n"] += n


# ===========================================================================
# LSTM layer
# ===========================================================================
def _acc(t):
    """The references' accumulation type: fp32 for bf16/fp32 inputs, fp64 kept as fp64 (the
    tests' oracle)."""
    return t if t.dtype == torch.float64 else t.float()


# Columns of dm per CTA of `px_lstm_dm_cell_bwd` (dm_t = dh_t·W_P^T with the cell backward in
# its epilogue), measured with tools/bench_lstm_step.py at B 128, S 2048, P 512.
BWD_BN = 16


def _fused_bwd_ok(dt, Bsz, S, P, W_P):
    """dm_t = dh_t·W_P^T with the cell backward fits one `px_lstm_dm_cell_bwd` launch: bf16,
    whole 128-row tiles, S in BN-column tiles, P in 64-deep K-blocks, W_P as the K-contiguous
    operand (the other operands are the layer's own 16-byte-aligned buffers)."""
    return (dt == torch.bfloat16 and Bsz % 128 == 0 and S % BWD_BN == 0 and P % 64 == 0 and
            W_P.is_contiguous() and W_P.data_ptr() % 16 == 0)


_persistent_grid = {}


def _persistent_ok(entry, dt, Bsz, S, P, Wh, W_P):
    """bf16, Wh and W_P contiguous and 16-byte aligned, and `entry` (a persistent kernel's grid
    query: its shapes, and whether the device keeps the whole grid resident) takes the layer."""
    if not (dt == torch.bfloat16 and Wh.is_contiguous() and W_P.is_contiguous() and
            Wh.data_ptr() % 16 == 0 and W_P.data_ptr() % 16 == 0):
        return False
    key = (entry, torch.cuda.current_device(), Bsz, S, P)
    if key not in _persistent_grid:
        _persistent_grid[key] = getattr(_lib(), entry)(Bsz, S, P)
    return _persistent_grid[key] > 0


def _fwd_persistent_ok(dt, Bsz, S, P, Wh, W_P):
    """All T forward steps fit one `px_lstm_fwd_persistent` launch: bf16, one 128-row tile,
    S in 128-unit and P in 64-column tiles with P <= 512, Wh and W_P contiguous and 16-byte
    aligned, and the device keeps the whole grid (S/16 CTAs) resident."""
    return _persistent_ok("px_lstm_fwd_persistent_grid", dt, Bsz, S, P, Wh, W_P)


def _bwd_persistent_ok(dt, Bsz, S, P, Wh, W_P):
    """All T backward steps fit one `px_lstm_bwd_persistent` launch: the same conditions as
    the forward kernel's."""
    return _persistent_ok("px_lstm_bwd_persistent_grid", dt, Bsz, S, P, Wh, W_P)


def lstm_layer_reference(x, Wx, Wh, bias, W_P, c0, h0, forget_bias=1.0):
    """x: [T, B, E] → (H [T, B, P], c_T, h_T); plain autograd-able torch."""
    T, Bsz, E = x.shape
    S = W_P.shape[0]
    xw = torch.addmm(bias, x.reshape(T * Bsz, E), Wx).view(T, Bsz, 4 * S)
    c, h, outs = _acc(c0), h0, []
    for t in range(T):
        gates = _acc(torch.addmm(xw[t], h, Wh))
        i, j, f, o = gates.split(S, dim=1)
        c = torch.sigmoid(f + forget_bias) * c + torch.sigmoid(i) * torch.tanh(j)
        m = (torch.sigmoid(o) * torch.tanh(c)).to(x.dtype)
        h = m @ W_P
        outs.append(h)
    return torch.stack(outs), c, h


class _LSTMLayerFn(torch.autograd.Function):
    """`W` is either the stacked `[E+P, 4S]` kernel of the reference's LSTM cell
    (`Wh is None`; rows `[:E]` multiply x, rows `[E:]` multiply h — one parameter, one
    gradient written straight into its bucket sink) or just `Wx` with `Wh` separate."""

    @staticmethod
    def forward(ctx, x, W, Wh, bias, W_P, c0, h0, forget_bias):
        L = _lib()
        T, Bsz, E = x.shape
        S, P = W_P.shape
        dt = x.dtype
        dev = x.device
        x = x.contiguous()
        stacked = Wh is None
        ctx.stacked = stacked
        ctx.param_refs = (W, bias, W_P)
        if stacked:
            Wx, Wh = W.detach()[:E], W.detach()[E:]
        else:
            Wx = W
        # W_P^T for the unfused backward chain (dm_t = dh_t W_P^T as a plain NN GEMM): a 2 MB
        # true transpose, 17 us of uncoalesced copy — done here on the side stream, underneath
        # the forward chain, instead of at the head of the backward pass
        if any(ctx.needs_input_grad) and not _fused_bwd_ok(dt, Bsz, S, P, W_P):
            from . import sinks
            cur = torch.cuda.current_stream(dev)
            ws = sinks.side_stream(dev)
            ws.wait_stream(cur)
            with torch.cuda.stream(ws):
                ctx.WPT = W_P.detach().t().contiguous()
                ctx.WPT_ev = torch.cuda.Event()
                ctx.WPT_ev.record(ws)
            ctx.WPT.record_stream(cur)
        xw = torch.addmm(bias, x.view(T * Bsz, E), Wx).view(T, Bsz, 4 * S)
        act = torch.empty(T, Bsz, 4 * S, dtype=dt, device=dev)
        c_all = torch.empty(T + 1, Bsz, S, dtype=torch.float32, device=dev)
        m_all = torch.empty(T, Bsz, S, dtype=dt, device=dev)
        h_all = torch.empty(T + 1, Bsz, P, dtype=dt, device=dev)
        c_all[0].copy_(c0)
        h_all[0].copy_(h0)
        st = _stream()
        if _fwd_persistent_ok(dt, Bsz, S, P, Wh, W_P):
            # every time step in one cooperative launch, Wh and W_P resident in shared memory
            ws = torch.empty(S // 128, Bsz, P, dtype=torch.float32, device=dev)
            _check(L.px_lstm_fwd_persistent(_p(xw), _p(Wh), _p(W_P), _p(act), _p(c_all),
                                            _p(m_all), _p(h_all), _p(ws), T, Bsz, S, P,
                                            float(forget_bias), st), "lstm_fwd_persistent")
            _count(1)
        else:
            for t in range(T):
                # accumulate straight into xw[t] (an `out=` different from the addend makes
                # torch copy the 2 MB addend first — one more launch per step on the
                # critical path)
                gpre = xw[t].addmm_(h_all[t], Wh)
                _check(L.px_lstm_cell_fwd(_p(gpre), _p(c_all[t]), _p(act[t]),
                                          _p(c_all[t + 1]), _p(m_all[t]), Bsz, S,
                                          float(forget_bias), _DT[dt], st), "lstm_cell_fwd")
                torch.mm(m_all[t], W_P, out=h_all[t + 1])
            _count(T)
        ctx.save_for_backward(x, Wx, Wh, W_P, act, c_all, m_all, h_all)
        ctx.dims = (T, Bsz, E, S, P)
        return h_all[1:], c_all[T].clone(), h_all[T].clone()

    @staticmethod
    def backward(ctx, dH, dcT, dhT):
        from . import sinks
        L = _lib()
        x, Wx, Wh, W_P, act, c_all, m_all, h_all = ctx.saved_tensors
        T, Bsz, E, S, P = ctx.dims
        stacked = ctx.stacked
        W_ref, bias_ref, WP_ref = ctx.param_refs
        dt, dev = x.dtype, x.device
        dH = dH.contiguous()
        dgates = torch.empty(T, Bsz, 4 * S, dtype=dt, device=dev)
        dh_tot = torch.empty(T, Bsz, P, dtype=dt, device=dev)
        dc = torch.zeros(Bsz, S, dtype=torch.float32, device=dev) if dcT is None \
            else dcT.float().clone()
        dh_rec = None if dhT is None else dhT.to(dt)
        # dm_t = dh_t @ W_P^T: on the fused path one kernel with the cell backward in its
        # epilogue (W_P [S, P] is already the K-contiguous operand), else a plain NN GEMM on the
        # W_P^T made in forward followed by the cell kernel
        fused = _fused_bwd_ok(dt, Bsz, S, P, W_P)
        dm = None if fused else torch.empty(Bsz, S, dtype=dt, device=dev)
        cur = torch.cuda.current_stream(dev)
        if not fused:
            cur.wait_event(ctx.WPT_ev)
            WPT = ctx.WPT
        # dh_{t-1} = dH_{t-1} + dgates_t @ Wh^T : Wh [P, 4S] is already the
        # K-contiguous "B^T" operand, so this skinny product (M=B, N=P, K=4S)
        # goes to our wgmma split-K kernel with the +dH addend fused in, its 8 K-splits
        # per tile reducing through DSMEM in a cluster.  The reduction reads the addend 4 bf16 at
        # a time, so dH must be 8-byte aligned (an incoming gradient may be a view at any offset).
        from . import gemm as _gemm
        use_tc = (dt == torch.bfloat16 and Bsz % 128 == 0 and P % 64 == 0 and
                  (4 * S) % 1024 == 0 and Wh.is_contiguous() and dH.data_ptr() % 8 == 0)
        WhT = None if use_tc else Wh.t().contiguous()
        st = _stream()

        # ---- weight-gradient outputs: the parameters' bucket sinks when a dense group
        # registered them (no pack copy afterwards), else fresh tensors
        def sink_of(ref, shape):
            s_ = sinks.get(ref)
            if s_ is not None and s_.dtype == dt and tuple(s_.shape) == tuple(shape):
                return s_, True
            return torch.empty(shape, dtype=dt, device=dev), False
        if stacked:
            dW, w_sunk = sink_of(W_ref, (E + P, 4 * S))
            dWx_o, dWh_o = dW[:E], dW[E:]
        else:
            dWx_o, w_sunk = sink_of(W_ref, (E, 4 * S))
            dWh_o = torch.empty(P, 4 * S, dtype=dt, device=dev)
        dbias_o, b_sunk = sink_of(bias_ref, (4 * S,))
        dWP_o, p_sunk = sink_of(WP_ref, (S, P))
        ws = sinks.side_stream(dev)
        ws2 = sinks.side_stream(dev, 1)
        if dh_rec is None:
            dh_tot[T - 1].copy_(dH[T - 1])
        else:
            torch.add(dH[T - 1], dh_rec, out=dh_tot[T - 1])
        if _bwd_persistent_ok(dt, Bsz, S, P, Wh, W_P) and dH.data_ptr() % 16 == 0:
            # every time step in one cooperative launch, W_P's and Wh's tiles resident in
            # shared memory; dh_rec = dgates[0]·Wh^T with no addend
            dh_rec = torch.empty(Bsz, P, dtype=dt, device=dev)
            ws_ = torch.empty(4 * S // 512, Bsz, P, dtype=torch.float32, device=dev)
            _check(L.px_lstm_bwd_persistent(_p(dH), _p(act), _p(c_all), _p(Wh), _p(W_P), _p(dc),
                                            _p(dgates), _p(dh_tot), _p(dh_rec), _p(ws_), T, Bsz,
                                            S, P, st), "lstm_bwd_persistent")
            _count(1)
        else:
            for t in range(T - 1, -1, -1):
                if fused:
                    _check(L.px_lstm_dm_cell_bwd(_p(dh_tot[t]), _p(W_P), _p(dc), _p(act[t]),
                                                 _p(c_all[t]), _p(c_all[t + 1]), _p(dgates[t]),
                                                 Bsz, S, P, BWD_BN, st), "lstm_dm_cell_bwd")
                else:
                    torch.mm(dh_tot[t], WPT, out=dm)
                    _check(L.px_lstm_cell_bwd(_p(dm), _p(dc), _p(act[t]), _p(c_all[t]),
                                              _p(c_all[t + 1]), _p(dgates[t]), Bsz, S, _DT[dt],
                                              st), "lstm_cell_bwd")
                if t > 0:
                    if use_tc:
                        _gemm.gemm_tn(dgates[t], Wh, addend=dH[t - 1], splits=8, bn=64,
                                      out=dh_tot[t - 1])
                    else:
                        torch.addmm(dH[t - 1], dgates[t], WhT, out=dh_tot[t - 1])
                else:
                    dh_rec = _gemm.gemm_tn(dgates[0], Wh, splits=8, bn=64) if use_tc \
                        else torch.mm(dgates[0], WhT)
            _count(T)
        dg2 = dgates.view(T * Bsz, 4 * S)
        # the bias gradient, a bandwidth-bound column sum, runs on a second side stream next
        # to the compute-bound weight-gradient GEMMs
        ws2.wait_stream(cur)
        with torch.cuda.stream(ws2):
            torch.sum(dg2, 0, out=dbias_o)
        ev_b = torch.cuda.Event()
        ev_b.record(ws2)
        dgates.record_stream(ws2)
        dbias_o.record_stream(ws2)
        # dx first: the embedding gradient is what the rest of backward (and the sparse
        # push) is waiting for; the weight-gradient GEMMs go to the side stream
        dx = (dg2 @ Wx.t()).view(T, Bsz, E)
        ws.wait_stream(cur)
        with torch.cuda.stream(ws):
            torch.mm(h_all[:T].reshape(-1, P).t(), dg2, out=dWh_o)
            torch.mm(x.reshape(-1, E).t(), dg2, out=dWx_o)
            torch.mm(m_all.reshape(-1, S).t(), dh_tot.view(-1, P), out=dWP_o)
        ev = torch.cuda.Event()
        ev.record(ws)
        for t_ in (dgates, dh_tot, x, h_all, m_all, dWh_o, dWx_o, dbias_o, dWP_o):
            t_.record_stream(ws)
        outs, plain = [], False
        for ref, o, sunk, e_ in ((W_ref, dW if stacked else dWx_o, w_sunk, ev),
                                 (bias_ref, dbias_o, b_sunk, ev_b), (WP_ref, dWP_o, p_sunk, ev)):
            if sunk:
                # in the bucket already: hand it to the dense group directly (its fused
                # reduce/update kernel waits for the event), nothing goes through
                # AccumulateGrad
                sinks.deliver(ref, e_)
                outs.append(None)
            else:
                outs.append(o)
                plain = True
        if plain or not stacked:
            cur.wait_event(ev)        # plain tensors are consumed on the current stream
            cur.wait_event(ev_b)
        dW_out, dbias, dW_P = outs
        return dx, dW_out, None if stacked else dWh_o, dbias, dW_P, dc, dh_rec, None


def lstm_layer(x, Wx, Wh, bias, W_P, c0, h0, forget_bias=1.0):
    if x.is_cuda and x.dtype in _DT:
        return _LSTMLayerFn.apply(x, Wx, Wh, bias, W_P, c0, h0, forget_bias)
    return lstm_layer_reference(x, Wx, Wh, bias, W_P, c0, h0, forget_bias)


def lstm_layer_stacked(x, W, bias, W_P, c0, h0, forget_bias=1.0):
    """Same layer with the reference's stacked kernel `W = [Wx; Wh]` ([E+P, 4S],
    `examples/lm1b/language_model.py:76-87`) passed whole: one parameter, one gradient
    tensor, written by the weight-gradient GEMMs directly into the parameter's bucket."""
    E = x.shape[-1]
    if x.is_cuda and x.dtype in _DT:
        return _LSTMLayerFn.apply(x, W, None, bias, W_P, c0, h0, forget_bias)
    return lstm_layer_reference(x, W[:E], W[E:], bias, W_P, c0, h0, forget_bias)


# ===========================================================================
# layer-normalised GRU layer (skip-thoughts)
# ===========================================================================
def _addr(t, offset):
    """Device address of element `offset` of tensor `t`."""
    return _vp(t.data_ptr() + offset * t.element_size())


def _mm_f32(a, b, out):
    """out (fp32) = a·b on cuBLAS, with an fp32 output for bf16 operands too."""
    if a.dtype == torch.float32:
        return torch.mm(a, b, out=out)
    return torch.mm(a, b, out_dtype=torch.float32, out=out)


def ln_gru_applies(x, w_hu, ln_wh, ln_u, h0=None):
    """The fused node takes the layer: a CUDA tensor in bf16 or fp32 with w_hu and both
    LayerNorms' γ/β in the same dtype, w_hu contiguous and 16-byte aligned, n % 8 == 0 and
    n <= `px_ln_gru_max_units()` (4096: 8 units per thread, 2 groups per thread, one 256-thread
    CTA per row), and an initial state, if any, of the same dtype."""
    dt = x.dtype
    if not (x.is_cuda and dt in _DT and w_hu.dtype == dt):
        return False
    n = w_hu.shape[0]
    params = (ln_wh.weight, ln_wh.bias, ln_u.weight, ln_u.bias)
    if any(p is None or p.dtype != dt or not p.is_contiguous() for p in params):
        return False
    if h0 is not None and h0.dtype != dt:
        return False
    return (n % 8 == 0 and n <= _lib().px_ln_gru_max_units() and w_hu.is_contiguous() and
            w_hu.data_ptr() % 16 == 0)


def _ln_gru_forward(gx, cx, w_hu, lnp, h0, lengths, reverse, eps, save):
    """All T steps -> (out [B, T, n], hs, hh, stats).  hs [T+1, B, n] holds the state before
    each step in processing order, hh [T, B, 3n] (fp32) each step's h·w_hu and stats [T, B, 4]
    its LayerNorm (mean, rstd) pairs; without `save`, hs and hh are ping-pong / scratch buffers
    and stats is None."""
    L = _lib()
    B, T, n2 = gx.shape
    n = n2 // 2
    dt, dev = gx.dtype, gx.device
    hs = torch.empty(T + 1 if save else 2, B, n, dtype=dt, device=dev)
    if h0 is None:
        hs[0].zero_()
    else:
        hs[0].copy_(h0)
    hh = torch.empty(T if save else 1, B, 3 * n, dtype=torch.float32, device=dev)
    stats = torch.empty(T, B, 4, dtype=torch.float32, device=dev) if save else None
    out = torch.empty(B, T, n, dtype=dt, device=dev)
    st = _stream()
    for s in range(T):
        t = T - 1 - s if reverse else s
        i, o = (s, s + 1) if save else (s % 2, (s + 1) % 2)
        hh_s = hh[s] if save else hh[0]
        _mm_f32(hs[i], w_hu, hh_s)
        _check(L.px_ln_gru_fwd(_p(hh_s), _addr(gx, t * 2 * n), T * 2 * n, _addr(cx, t * n), T * n,
                               _p(hs[i]), _p(hs[o]), _addr(out, t * n), T * n,
                               _p(stats[s]) if save else None, *[_p(p) for p in lnp],
                               None if lengths is None else _p(lengths), t, B, n, eps[0], eps[1],
                               _DT[dt], st), "ln_gru_fwd")
    _count(T)
    return out, hs[T] if save else hs[T % 2], hs, hh, stats


class _LNGRULayerFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, gx, cx, w_hu, g_wh, b_wh, g_u, b_u, h0, lengths, reverse, eps_wh, eps_u):
        out, hT, hs, hh, stats = _ln_gru_forward(gx, cx, w_hu, (g_wh, b_wh, g_u, b_u), h0, lengths,
                                                 reverse, (eps_wh, eps_u), True)
        ctx.save_for_backward(gx, cx, w_hu, g_wh, b_wh, g_u, b_u, hs, hh, stats, lengths)
        ctx.reverse = reverse
        ctx.set_materialize_grads(False)
        return out, hT.clone()

    @staticmethod
    def backward(ctx, d_out, d_final):
        L = _lib()
        gx, cx, w_hu, g_wh, b_wh, g_u, b_u, hs, hh, stats, lengths = ctx.saved_tensors
        B, T, n2 = gx.shape
        n = n2 // 2
        dt, dev = gx.dtype, gx.device
        if d_out is not None:
            d_out = d_out.contiguous()
            if d_out.data_ptr() % 16:
                d_out = d_out.clone()
        carry = torch.zeros(B, n, dtype=torch.float32, device=dev) if d_final is None \
            else d_final.float().clone()
        drec = torch.empty(B, n, dtype=torch.float32, device=dev)
        dhh = torch.empty(T, B, 3 * n, dtype=dt, device=dev)
        dgx = torch.empty(B, T, 2 * n, dtype=dt, device=dev)
        dcx = torch.empty(B, T, n, dtype=dt, device=dev)
        acc = torch.empty(B, 6 * n, dtype=torch.float32, device=dev)
        lnp = [_p(p) for p in (g_wh, b_wh, g_u, b_u)]
        lp = None if lengths is None else _p(lengths)
        need_h0 = ctx.needs_input_grad[7]
        w_t = w_hu.t()
        st = _stream()
        for k in range(T):
            s = T - 1 - k
            t = T - 1 - s if ctx.reverse else s
            _check(L.px_ln_gru_bwd(_p(hh[s]), _p(stats[s]), _addr(gx, t * 2 * n), T * 2 * n,
                                   _addr(cx, t * n), T * n, _p(hs[s]),
                                   None if d_out is None else _addr(d_out, t * n), T * n,
                                   None if k == 0 else _p(drec), _p(carry), _p(dhh[s]),
                                   _addr(dgx, t * 2 * n), T * 2 * n, _addr(dcx, t * n), T * n,
                                   _p(acc), int(k == 0), *lnp, lp, t, B, n, _DT[dt], st),
                   "ln_gru_bwd")
            if s > 0 or need_h0:
                _mm_f32(dhh[s], w_t, drec)
        dh0 = drec.add_(carry).to(dt) if need_h0 else None
        dw_hu = torch.mm(hs[:T].reshape(T * B, n).t(), dhh.view(T * B, 3 * n))
        dln = [torch.empty_like(p) for p in (g_wh, b_wh, g_u, b_u)]
        _check(L.px_ln_gru_param_grad(_p(acc), B, n, *[_p(d) for d in dln], _DT[dt], st),
               "ln_gru_param_grad")
        _count(T + 1)
        return (dgx, dcx, dw_hu, *dln, dh0, None, None, None, None)


def ln_gru_layer(gx, cx, w_hu, ln_wh, ln_u, h0=None, lengths=None, reverse=False):
    """The recurrence of `LayerNormGRU` from its input-side terms gx = LN_wx(x·w_x) [B, T, 2n]
    and cx = LN_w(x·w) [B, T, n] -> (outputs [B, T, n], zero past each length; final state
    [B, n]).  `lengths` [B] masks each row as the composition does; `reverse` walks t from T−1
    down to 0.  Callers check `ln_gru_applies` first.  Without autograd (no_grad, or nothing
    requiring a gradient) nothing is kept for a backward pass."""
    gx, cx = gx.contiguous(), cx.contiguous()
    if lengths is not None:
        lengths = lengths.to(device=gx.device, dtype=torch.int64).contiguous()
    args = (gx, cx, w_hu, ln_wh.weight, ln_wh.bias, ln_u.weight, ln_u.bias, h0)
    eps = (float(ln_wh.eps), float(ln_u.eps))
    if torch.is_grad_enabled() and any(a is not None and a.requires_grad for a in args):
        return _LNGRULayerFn.apply(*args, lengths, bool(reverse), *eps)
    out, hT, _, _, _ = _ln_gru_forward(gx, cx, w_hu, args[3:7], h0, lengths, reverse, eps, False)
    return out, hT


# ===========================================================================
# layer-normalised LSTM layer (NMT)
# ===========================================================================
def _ln_lstm_params(ln_gates, ln_c):
    """γ of LN_i, LN_j, LN_f, LN_o, LN_c, then their β"""
    lns = list(ln_gates) + [ln_c]
    return [ln.weight for ln in lns] + [ln.bias for ln in lns], [float(ln.eps) for ln in lns]


def ln_lstm_applies(x, kernel_weight, ln_gates, ln_c, h0=None, c0=None):
    """The fused node takes the layer: a CUDA tensor [B, T, I] in bf16 or fp32 with the kernel
    weight [4U, I + U], the five LayerNorms' γ/β and any initial state in the same dtype, the
    kernel weight contiguous and 16-byte aligned, U % 8 == 0 and U <= `px_ln_lstm_max_units()`
    (2048: 8 units per thread, one 256-thread CTA per row)."""
    dt = x.dtype
    if not (x.is_cuda and x.dim() == 3 and dt in _DT and kernel_weight.dtype == dt):
        return False
    params, _ = _ln_lstm_params(ln_gates, ln_c)
    if any(p is None or p.dtype != dt or not p.is_contiguous() for p in params):
        return False
    if any(s is not None and s.dtype != dt for s in (h0, c0)):
        return False
    U = kernel_weight.shape[0] // 4
    return (U % 8 == 0 and U <= _lib().px_ln_lstm_max_units() and
            kernel_weight.shape == (4 * U, x.shape[2] + U) and kernel_weight.is_contiguous() and
            kernel_weight.data_ptr() % 16 == 0)


def _ln_lstm_ptrs(params, eps):
    return (_vp * 10)(*[p.data_ptr() for p in params]), (_f * 5)(*eps)


def _ln_lstm_forward(x, w, params, eps, fb, h0, c0, lengths, save):
    """All T steps -> (out [B, T, U], h_T, c_T (fp32), hs, C, P, gx, stats).  gx [B, T, 4U] (fp32)
    is x·W_xᵀ, hs [B, T, U] the state h before each step, C [T+1, B, U] (fp32) the cell states,
    P [T, B, 4U] (fp32) each step's h·W_hᵀ and stats [T, B, 10] its LayerNorm statistics;
    without `save`, hs, C and P are ping-pong / scratch buffers and stats is None."""
    L = _lib()
    B, T, I = x.shape
    U = w.shape[0] // 4
    dt, dev = x.dtype, x.device
    f32 = dict(dtype=torch.float32, device=dev)
    gx = torch.empty(B, T, 4 * U, **f32)
    _mm_f32(x.reshape(B * T, I), w[:, :I].t(), gx.view(B * T, 4 * U))
    w_h = w[:, I:].t()
    if save:
        hs = torch.empty(B, T, U, dtype=dt, device=dev)
        hT = torch.empty(B, U, dtype=dt, device=dev)
        h_at = lambda s: (hs[:, s], T * U) if s < T else (hT, U)
    else:
        hs = torch.empty(2, B, U, dtype=dt, device=dev)
        h_at = lambda s: (hs[s % 2], U)
    C = torch.empty(T + 1 if save else 2, B, U, **f32)
    h_at(0)[0].copy_(h0)
    C[0].copy_(c0)
    P = torch.empty(T if save else 1, B, 4 * U, **f32)
    stats = torch.empty(T, B, 10, **f32) if save else None
    out = torch.empty(B, T, U, dtype=dt, device=dev)
    ln, ep = _ln_lstm_ptrs(params, eps)
    lp = None if lengths is None else _p(lengths)
    st = _stream()
    for t in range(T):
        (h, h_ld), (hn, hn_ld) = h_at(t), h_at(t + 1)
        c_i, c_o = (t, t + 1) if save else (t % 2, (t + 1) % 2)
        Pt = P[t] if save else P[0]
        _mm_f32(h, w_h, Pt)
        _check(L.px_ln_lstm_fwd(_p(Pt), _addr(gx, t * 4 * U), T * 4 * U, _p(C[c_i]), _p(C[c_o]),
                                _p(h), h_ld, _p(hn), hn_ld, _addr(out, t * U), T * U,
                                _p(stats[t]) if save else None, ln, ep, fb, lp, t, B, U, _DT[dt],
                                st), "ln_lstm_fwd")
    _count(T)
    return out, h_at(T)[0], C[T if save else T % 2], hs, C, P, gx, stats


class _LNLSTMLayerFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, h0, c0, lengths, eps, fb, *params):
        out, hT, cT, hs, C, P, gx, stats = _ln_lstm_forward(x, w, params, eps, fb, h0, c0, lengths,
                                                            True)
        ctx.save_for_backward(x, w, hs, C, P, gx, stats, lengths, *params)
        ctx.eps, ctx.fb = eps, fb
        ctx.set_materialize_grads(False)
        return out, hT, cT.to(x.dtype, copy=True)

    @staticmethod
    def backward(ctx, d_out, d_hT, d_cT):
        L = _lib()
        x, w, hs, C, P, gx, stats, lengths, *params = ctx.saved_tensors
        B, T, I = x.shape
        U = w.shape[0] // 4
        dt, dev = x.dtype, x.device
        f32 = dict(dtype=torch.float32, device=dev)
        if d_out is not None:
            d_out = d_out.contiguous()
            if d_out.data_ptr() % 16:
                d_out = d_out.clone()
        carry_h, carry_c = (torch.zeros(B, U, **f32) if d is None else
                            torch.empty(B, U, **f32).copy_(d) for d in (d_hT, d_cT))
        drec = torch.empty(B, U, **f32)
        dpre = torch.empty(B, T, 4 * U, dtype=dt, device=dev)
        acc = torch.empty(B, 10 * U, **f32)
        ln, ep = _ln_lstm_ptrs(params, ctx.eps)
        lp = None if lengths is None else _p(lengths)
        need_h0 = ctx.needs_input_grad[2]
        w_h = w[:, I:]
        st = _stream()
        for k in range(T):
            t = T - 1 - k
            _check(L.px_ln_lstm_bwd(_p(P[t]), _addr(gx, t * 4 * U), T * 4 * U, _p(stats[t]),
                                    _p(C[t]), None if d_out is None else _addr(d_out, t * U),
                                    T * U, None if k == 0 else _p(drec), _p(carry_h),
                                    _p(carry_c), _addr(dpre, t * 4 * U), T * 4 * U, _p(acc),
                                    int(k == 0), ln, ep, ctx.fb, lp, t, B, U, _DT[dt], st),
                   "ln_lstm_bwd")
            if t > 0 or need_h0:
                _mm_f32(dpre[:, t], w_h, drec)
        dh0 = drec.add_(carry_h).to(dt) if need_h0 else None
        dc0 = carry_c.to(dt) if ctx.needs_input_grad[3] else None
        d2 = dpre.view(B * T, 4 * U)
        dx = torch.mm(d2, w[:, :I]).view(B, T, I) if ctx.needs_input_grad[0] else None
        dw = torch.cat([torch.mm(d2.t(), x.reshape(B * T, I)),
                        torch.mm(d2.t(), hs.view(B * T, U))], 1)
        dln = torch.empty(10, U, dtype=dt, device=dev)
        _check(L.px_ln_lstm_param_grad(_p(acc), B, U, _p(dln), _DT[dt], st), "ln_lstm_param_grad")
        _count(T + 1)
        return (dx, dw, dh0, dc0, None, None, None, *dln.unbind(0))


def ln_lstm_layer(x, kernel_weight, ln_gates, ln_c, forget_bias, h0, c0, lengths=None):
    """`LayerNormLSTM` over x [B, T, I] -> (outputs [B, T, U], zero past each length; (h_T, c_T)
    in x's dtype).  kernel_weight [4U, I + U] is the bias-free `nn.Linear` over [x | h] (gate
    order i, j, f, o), ln_gates the gates' four `nn.LayerNorm(U)`, ln_c the cell state's; c' is
    carried un-normalised, in fp32 between steps.  `lengths` [B] freezes each row's state past
    its length.  Callers check `ln_lstm_applies` first.  Without autograd (no_grad, or nothing
    requiring a gradient) nothing is kept for a backward pass."""
    B, T, _ = x.shape
    U = kernel_weight.shape[0] // 4
    if h0 is None:
        h0 = x.new_zeros(B, U)
    if c0 is None:
        c0 = x.new_zeros(B, U)
    if lengths is not None:
        lengths = lengths.to(device=x.device, dtype=torch.int64).contiguous()
    params, eps = _ln_lstm_params(ln_gates, ln_c)
    fb = float(forget_bias)
    args = [x, kernel_weight, h0, c0] + params
    if torch.is_grad_enabled() and any(a.requires_grad for a in args):
        out, hT, cT = _LNLSTMLayerFn.apply(x, kernel_weight, h0, c0, lengths, tuple(eps), fb,
                                           *params)
        return out, (hT, cT)
    out, hT, cT, *_ = _ln_lstm_forward(x, kernel_weight, params, eps, fb, h0, c0, lengths, False)
    return out, (hT.clone(), cT.to(x.dtype, copy=True))


# ===========================================================================
# NMT attention decoder
# ===========================================================================
def nmt_decoder_applies(emb, keys, values, weights, states, unit_type="lstm"):
    """The fused node takes the decoder: LSTM or layer_norm_lstm cells, a CUDA tensor in bf16 or
    fp32 with every weight and state in the same dtype, the matrices contiguous and 16-byte
    aligned (for layer_norm_lstm, each layer's whole kernel weight), keys
    [B, S, U] and values [B, S, M] contiguous and 16-byte aligned, U % 8 == 0 and M % 8 == 0,
    and U, M and S within `px_nmt_max_units` / `px_nmt_max_memory` / `px_nmt_max_source`
    (1024 / 2048 / 1024)."""
    dt = emb.dtype
    if unit_type not in ("lstm", "layer_norm_lstm") or not (emb.is_cuda and dt in _DT):
        return False
    if any(t is not None and t.dtype != dt for t in list(weights) + list(states) + [keys, values]):
        return False
    for w in weights:
        if w is not None and w.dim() == 2 and not (w.is_contiguous() and w.data_ptr() % 16 == 0):
            return False
    for t in (keys, values):
        if not (t.is_contiguous() and t.data_ptr() % 16 == 0):
            return False
    B, S, U = keys.shape
    M = values.shape[2]
    L = _lib()
    return (U % 8 == 0 and M % 8 == 0 and emb.shape[-1] == U and U <= L.px_nmt_max_units() and
            M <= L.px_nmt_max_memory() and S <= L.px_nmt_max_source())


def _mask_mul(x, m):
    return x if m is None else x * m


def _ln_cell_reference(gates, c, ln, dt):
    """`LayerNormLSTM.cell` from its pre-LayerNorm gate terms, in the accumulation type"""
    params, eps, fb = ln
    U = c.shape[1]
    F_ = torch.nn.functional
    a = [F_.layer_norm(x, (U,), _acc(params[k]), _acc(params[5 + k]), eps[k])
         for k, x in enumerate(gates.chunk(4, -1))]
    c = c * torch.sigmoid(a[2] + fb) + torch.sigmoid(a[0]) * torch.tanh(a[1])
    h = (torch.tanh(F_.layer_norm(c, (U,), _acc(params[4]), _acc(params[9]), eps[4])) *
         torch.sigmoid(a[3])).to(dt)
    return h, c


def nmt_attention_decoder_reference(emb, h0, c0, att0, keys, values, pad, w_ih, w_hh, b_ih, b_hh,
                                    residual, w_q=None, g=None, v=None, b=None, w_a=None,
                                    masks=None, output_attention=True, ln=None):
    """Pure-PyTorch version of `nmt_attention_decoder` (same arguments, same masks): the fp64
    oracle of the node's tests.  State and gates are kept in the accumulation type (fp32 for
    bf16/fp32 inputs)."""
    B, T, U = emb.shape
    L = len(w_ih)
    dt = emb.dtype
    h, c = list(h0), [_acc(x) for x in c0]
    feed = att0
    outs, qs, ctxs = [], [], []
    for t in range(T):
        x = torch.cat([emb[:, t], feed], -1)
        for l in range(L):
            inp = _mask_mul(x, None if masks is None else masks[l][t])
            bi, bh = (None, None) if b_ih is None else (b_ih[l], b_hh[l])
            gates = _acc(torch.nn.functional.linear(inp, w_ih[l], bi) +
                         torch.nn.functional.linear(h[l], w_hh[l], bh))
            if ln is not None:
                h[l], c[l] = _ln_cell_reference(gates, c[l], ln[l], dt)
            else:
                i, f, gg, o = gates.chunk(4, -1)
                c[l] = torch.sigmoid(f) * c[l] + torch.sigmoid(i) * torch.tanh(gg)
                h[l] = (torch.sigmoid(o) * torch.tanh(c[l])).to(dt)
            x = h[l] + x[..., :U] if residual[l] else h[l]
        q = x
        if v is not None:
            hid = keys + (q @ w_q.t())[:, None, :]
            if b is not None:
                hid = hid + b
            s = (torch.tanh(hid) * v.to(hid.dtype)).sum(-1)
        else:
            s = torch.bmm(q[:, None, :], keys.transpose(1, 2))[:, 0]
            if g is not None:
                s = s * g.to(s.dtype)
        a = torch.softmax(_acc(s).masked_fill(pad, float("-inf")), -1)
        ctx = torch.bmm(a[:, None, :].to(values.dtype), values)[:, 0]
        if w_a is not None:
            feed = torch.cat([q, ctx], -1) @ w_a.t()
            outs.append(feed if output_attention else q)
        else:
            feed = ctx
            qs.append(q)
            ctxs.append(ctx)
    if w_a is not None:
        return torch.stack(outs, 1)
    return torch.stack(qs, 1), torch.stack(ctxs, 1)


def _nmt_forward(cfg, emb, h0, c0, att0, keys, values, pad, W, attn, masks, save):
    """All T steps of the decoder -> dict of buffers (module docstring of
    `kernels/nmt_decoder.cu`; DESIGN.md §5).  Time-major per-step buffers:
    xh[l] [T+1, B, K_l] = [input ⊙ mask | h_{t-1}] (layer 0: [emb ⊙ mask | feed ⊙ mask | h]),
    P[l] [T, B, 4U] fp32 products, C[l] [T+1, B, U] fp32 cell states, qc [T, B, U+M] = [q | ctx],
    align [T, B, S] fp32, pq [T, B, U] fp32.  Without `save` the recurrent buffers are ping-pong
    pairs and only what the outputs need is kept."""
    Lb = _lib()
    L, std, bah, res = cfg["L"], cfg["standard"], cfg["bahdanau"], cfg["residual"]
    w_ih, w_hh, b_ih, b_hh = W["w_ih"], W["w_hh"], W["b_ih"], W["b_hh"]
    B, T, U = emb.shape
    S, M = keys.shape[1], values.shape[2]
    A = att0.shape[1]
    dt, dev = emb.dtype, emb.device
    nT = T + 1 if save else 2
    sl = (lambda t: t) if save else (lambda t: t % 2)
    I = [U + A] + [U] * (L - 1)
    K = [I[0] + U] + [I[l] + U for l in range(1, L)]
    xh = [torch.empty(nT, B, K[l], dtype=dt, device=dev) for l in range(L)]
    C = [torch.empty(nT, B, U, dtype=torch.float32, device=dev) for _ in range(L)]
    P = [torch.empty(T if save else 1, B, 4 * U, dtype=torch.float32, device=dev)
         for _ in range(L)]
    qc = torch.empty(T, B, U + M, dtype=dt, device=dev)
    lnc = cfg["ln"]
    stats = [torch.empty(T, B, 10, dtype=torch.float32, device=dev) if save else None
             for _ in range(L)] if lnc is not None else None
    lnp = [_ln_lstm_ptrs(W["ln"][l], lnc[l][0]) for l in range(L)] if lnc is not None else None
    align = torch.empty(T if save else 1, B, S, dtype=torch.float32, device=dev)
    pq = torch.empty(T if save else 1, B, U, dtype=torch.float32, device=dev) if bah else None
    att = torch.empty(T, B, U, dtype=dt, device=dev) if std else None
    ybuf = [torch.empty(B, U, dtype=dt, device=dev) for _ in range(L - 1)]
    # W_step[l]: the columns a step multiplies (layer 0: feed and h; the embedding part is one
    # product over all T before the loop)
    w_step = [torch.cat([w_ih[0][:, U:], w_hh[0]], 1)] + \
        [torch.cat([w_ih[l], w_hh[l]], 1) for l in range(1, L)]
    m0 = None if masks is None else masks[0]
    embT = emb.transpose(0, 1)
    e_part = xh[0][:T, :, :U] if save else torch.empty(T, B, U, dtype=dt, device=dev)
    if m0 is None:
        e_part.copy_(embT)
    else:
        torch.mul(embT, m0[:, :, :U], out=e_part)
    gx0 = torch.empty(T, B, 4 * U, dtype=torch.float32, device=dev)
    _mm_f32(e_part.reshape(T * B, U), w_ih[0][:, :U].t(), gx0.view(T * B, 4 * U))
    if m0 is None:
        xh[0][0, :, U:U + A].copy_(att0)
    else:
        torch.mul(att0, m0[0, :, U:], out=xh[0][0, :, U:U + A])
    for l in range(L):
        xh[l][0, :, I[l]:].copy_(h0[l])
        C[l][0].copy_(c0[l])
    kind = 1 if bah else 0
    g_p = _p(attn["g"]) if attn["g"] is not None else None
    v_p = _p(attn["v"]) if bah else None
    b_p = _p(attn["b"]) if attn["b"] is not None else None
    emb_ld = T * U
    st = _stream()
    for t in range(T):
        i0, i1 = sl(t), sl(t + 1)
        for l in range(L):
            Pt = P[l][t] if save else P[l][0]
            _mm_f32(xh[l][i0, :, U if l == 0 else 0:], w_step[l].t(), Pt)
            top = l == L - 1
            if res[l]:
                resid, r_ld = ((_addr(emb, t * U), emb_ld) if l == 0 else (_p(ybuf[l - 1]), U))
            else:
                resid, r_ld = None, 0
            y, y_ld = (_p(qc[t]), U + M) if top else (_p(ybuf[l]), U)
            if top:
                xn, xn_ld, mk, mk_ld = None, 0, None, 0
            else:
                xn, xn_ld = _p(xh[l + 1][i0]), K[l + 1]
                mk, mk_ld = (None, 0) if masks is None else (_p(masks[l + 1][t]), I[l + 1])
            if lnc is not None:
                _check(Lb.px_nmt_ln_lstm_cell_fwd(
                    _p(Pt), _p(gx0[t]) if l == 0 else None, _p(C[l][i0]), _p(C[l][i1]),
                    _addr(xh[l][i1], I[l]), K[l], resid, r_ld, y, y_ld, mk, mk_ld, xn, xn_ld,
                    _p(stats[l][t]) if save else None, *lnp[l], lnc[l][1], B, U, _DT[dt], st),
                    "nmt_ln_lstm_cell_fwd")
            else:
                _check(Lb.px_nmt_lstm_cell_fwd(
                    _p(Pt), _p(gx0[t]) if l == 0 else None, _p(b_ih[l]), _p(b_hh[l]),
                    _p(C[l][i0]), _p(C[l][i1]), _addr(xh[l][i1], I[l]), K[l], resid, r_ld, y,
                    y_ld, mk, mk_ld, xn, xn_ld, B, U, _DT[dt], st), "nmt_lstm_cell_fwd")
        q = qc[t][:, :U]
        pq_t = None
        if bah:
            pq_t = pq[t] if save else pq[0]
            _mm_f32(q, attn["w_q"].t(), pq_t)
        feed, feed_ld, fm, fm_ld = None, 0, None, 0
        if not std and t + 1 < T:
            feed, feed_ld = _addr(xh[0][i1], U), K[0]
            if m0 is not None:
                fm, fm_ld = _addr(m0[t + 1], U), I[0]
        _check(Lb.px_nmt_attn_fwd(
            _p(qc[t]), U + M, _p(pq_t) if bah else None, _p(keys), _p(values), _p(pad), g_p,
            v_p, b_p, _addr(qc[t], U), U + M, fm, fm_ld, feed, feed_ld,
            _p(align[t] if save else align[0]), B, S, U, M, kind, _DT[dt], st), "nmt_attn_fwd")
        if std:
            torch.mm(qc[t], W["w_a"].t(), out=att[t])
            if t + 1 < T:
                dst = xh[0][i1, :, U:U + A]
                if m0 is None:
                    dst.copy_(att[t])
                else:
                    torch.mul(att[t], m0[t + 1, :, U:], out=dst)
    _count(T * (L + 1))
    return dict(xh=xh, C=C, P=P, qc=qc, align=align, pq=pq, att=att, gx0=gx0, w_step=w_step,
                e_part=e_part, last=sl(T), stats=stats)


def _nmt_outputs(cfg, F, U, output_attention):
    if cfg["standard"]:
        if output_attention:
            return F["att"].transpose(0, 1)
        return F["qc"][:, :, :U].transpose(0, 1).contiguous()
    return (F["qc"][:, :, :U].transpose(0, 1).contiguous(),
            F["qc"][:, :, U:].transpose(0, 1).contiguous())


class _NMTDecoderFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, cfg, n_in, emb, att0, keys, values, pad, *rest):
        L = cfg["L"]
        h0, c0 = rest[:L], rest[L:2 * L]
        W = dict(w_ih=rest[2 * L:3 * L], w_hh=rest[3 * L:4 * L], b_ih=rest[4 * L:5 * L],
                 b_hh=rest[5 * L:6 * L], w_q=rest[6 * L], w_a=rest[6 * L + 4])
        attn = dict(w_q=rest[6 * L], g=rest[6 * L + 1], v=rest[6 * L + 2], b=rest[6 * L + 3])
        masks = None if rest[6 * L + 5] is None else rest[6 * L + 5:6 * L + 5 + L]
        W["ln"] = _nmt_ln_params(cfg, rest)
        F = _nmt_forward(cfg, emb, h0, c0, att0, keys, values, pad, W, attn, masks, True)
        ctx.cfg, ctx.n_in = cfg, n_in
        ctx.F = F
        ctx.save_for_backward(emb, att0, keys, values, pad, *rest)
        ctx.set_materialize_grads(False)
        return _nmt_outputs(cfg, F, emb.shape[2], cfg["output_attention"])

    @staticmethod
    def backward(ctx, *douts):
        cfg, F = ctx.cfg, ctx.F
        Lb = _lib()
        emb, att0, keys, values, pad, *rest = ctx.saved_tensors
        L, std, bah, res = cfg["L"], cfg["standard"], cfg["bahdanau"], cfg["residual"]
        w_ih, w_hh, b_ih, b_hh = rest[2 * L:3 * L], rest[3 * L:4 * L], rest[4 * L:5 * L], \
            rest[5 * L:6 * L]
        w_q, g, vp, bb, w_a = rest[6 * L:6 * L + 5]
        masks = None if rest[6 * L + 5] is None else rest[6 * L + 5:6 * L + 5 + L]
        B, T, U = emb.shape
        S, M = keys.shape[1], values.shape[2]
        A = att0.shape[1]
        dt, dev = emb.dtype, emb.device
        xh, C, P, qc, align, pq, gx0, w_step = (F[k] for k in ("xh", "C", "P", "qc", "align",
                                                                "pq", "gx0", "w_step"))
        lnc, stats = cfg["ln"], F["stats"]
        if lnc is not None:
            lnw = _nmt_ln_params(cfg, rest)
            lnp = [_ln_lstm_ptrs(lnw[l], lnc[l][0]) for l in range(L)]
            acc = [torch.empty(B, 10 * U, dtype=torch.float32, device=dev) for _ in range(L)]
        I = [U + A] + [U] * (L - 1)
        K = [I[0] + U] + [I[l] + U for l in range(1, L)]
        m0 = None if masks is None else masks[0]

        def _prep(d):
            if d is None:
                return None
            d = d.contiguous()
            return d if d.data_ptr() % 16 == 0 else d.clone()
        if std:
            d_main, d_ctx_out = _prep(douts[0]), None
        else:
            d_main, d_ctx_out = _prep(douts[0]), _prep(douts[1])
        f32 = dict(dtype=torch.float32, device=dev)
        dG = [torch.empty(T, B, 4 * U, dtype=dt, device=dev) for _ in range(L)]
        dXH = [torch.empty(B, K[l] - (U if l == 0 else 0), **f32) for l in range(L)]
        dc = [torch.zeros(B, U, **f32) for _ in range(L)]
        dY = [torch.empty(B, U, **f32) for _ in range(L)]
        dY0 = torch.empty(T, B, U, **f32) if res[0] else None
        dkeys = torch.zeros(B, S, U, **f32)
        dvalues = torch.zeros(B, S, M, **f32)
        part_g = torch.zeros(B, 1, **f32) if (not bah and g is not None) else None
        part_v = torch.zeros(B, U, **f32) if bah else None
        part_b = torch.zeros(B, U, **f32) if (bah and bb is not None) else None
        dq = torch.empty(B, U, **f32)
        dpq = torch.empty(T, B, U, dtype=dt, device=dev) if bah else None
        datt = torch.empty(T, B, U, dtype=dt, device=dev) if std else None
        dqc = torch.empty(B, U + M, **f32) if std else None
        g_p = _p(g) if g is not None else None
        kind = 1 if bah else 0
        st = _stream()
        for t in range(T - 1, -1, -1):
            last = t == T - 1
            if std:
                # d att_t = d_out_t (output_attention) + the feed's gradient from step t+1
                dst = datt[t]
                d_o = d_main[:, t] if (cfg["output_attention"] and d_main is not None) else None
                if last:
                    if d_o is None:
                        dst.zero_()
                    else:
                        dst.copy_(d_o)
                else:
                    dF = dXH[0][:, :A]
                    mf = None if m0 is None else m0[t + 1, :, U:]
                    if d_o is None:
                        dst.copy_(dF if mf is None else dF * mf)
                    elif mf is None:
                        torch.add(d_o, dF, out=dst)
                    else:
                        torch.addcmul(d_o, dF, mf, out=dst)
                _mm_f32(datt[t], w_a, dqc)
                dA, dA_ld, dAm, dAm_ld = _addr(dqc, U), U + M, None, 0
                dO, dO_ld = None, 0
            else:
                dA, dA_ld, dAm, dAm_ld = (None, 0, None, 0) if last else \
                    (_p(dXH[0]), K[0] - U, None if m0 is None else _addr(m0[t + 1], U), I[0])
                dO, dO_ld = (None, 0) if d_ctx_out is None else (_addr(d_ctx_out, t * M), T * M)
            _check(Lb.px_nmt_attn_bwd(
                dA, dA_ld, dAm, dAm_ld, dO, dO_ld, _p(align[t]), _p(qc[t]), U + M,
                _p(pq[t]) if bah else None, _p(keys), _p(values), g_p,
                _p(vp) if bah else None, _p(bb) if bb is not None else None,
                None if bah else _p(dq), _p(dpq[t]) if bah else None, _p(dkeys), _p(dvalues),
                _p(part_g) if part_g is not None else None,
                _p(part_v) if bah else None, _p(part_b) if part_b is not None else None,
                B, S, U, M, kind, _DT[dt], st), "nmt_attn_bwd")
            if bah:
                _mm_f32(dpq[t], w_q, dq)
            for l in range(L - 1, -1, -1):
                top = l == L - 1
                if top:
                    a_, a_ld, am, am_ld = (_p(dqc), U + M, None, 0) if std else (None, 0, None, 0)
                    dR = _p(dq)
                    if std:
                        o_ = None if (cfg["output_attention"] or d_main is None) else \
                            _addr(d_main, t * U)
                    else:
                        o_ = None if d_main is None else _addr(d_main, t * U)
                    o_ld = T * U
                else:
                    a_, a_ld = _p(dXH[l + 1]), K[l + 1]
                    am, am_ld = (None, 0) if masks is None else (_p(masks[l + 1][t]), I[l + 1])
                    dR = _p(dY[l + 1]) if res[l + 1] else None
                    o_, o_ld = None, 0
                off = A if l == 0 else I[l]
                drec, drec_ld = (None, 0) if last else (_addr(dXH[l], off), dXH[l].shape[1])
                dYp = _p(dY0[t]) if (l == 0 and res[0]) else (_p(dY[l]) if l > 0 and res[l]
                                                              else None)
                if lnc is not None:
                    _check(Lb.px_nmt_ln_lstm_cell_bwd(
                        _p(P[l][t]), _p(gx0[t]) if l == 0 else None, _p(stats[l][t]),
                        _p(C[l][t]), a_, a_ld, am, am_ld, dR, o_, o_ld, drec, drec_ld,
                        _p(dc[l]), _p(dG[l][t]), dYp, _p(acc[l]), int(last), *lnp[l],
                        lnc[l][1], B, U, _DT[dt], st), "nmt_ln_lstm_cell_bwd")
                else:
                    _check(Lb.px_nmt_lstm_cell_bwd(
                        _p(P[l][t]), _p(gx0[t]) if l == 0 else None, _p(b_ih[l]), _p(b_hh[l]),
                        _p(C[l][t]), _p(C[l][t + 1]), a_, a_ld, am, am_ld, dR, o_, o_ld, drec,
                        drec_ld, _p(dc[l]), _p(dG[l][t]), dYp, B, U, _DT[dt], st),
                        "nmt_lstm_cell_bwd")
                _mm_f32(dG[l][t], w_step[l], dXH[l])
        _count(T * (L + 1))
        nd = ctx.needs_input_grad
        # gradients of the inputs: (cfg, n_in, emb, att0, keys, values, pad, *rest)
        dG2 = [d.view(T * B, 4 * U) for d in dG]
        gl = [None] * len(rest)
        demb = None
        if nd[2]:
            de = torch.empty(T * B, U, **f32)
            _mm_f32(dG2[0], w_ih[0][:, :U], de)
            de = de.view(T, B, U)
            if m0 is not None:
                de = de * m0[:, :, :U]
            if dY0 is not None:
                de = de + dY0
            demb = de.transpose(0, 1).to(dt)
        datt0 = None
        if nd[3]:
            d = dXH[0][:, :A]
            datt0 = (d if m0 is None else d * m0[0, :, U:]).to(dt)
        dk = dkeys.to(dt) if nd[4] else None
        dv = dvalues.to(dt) if nd[5] else None
        for l in range(L):
            off = A if l == 0 else I[l]
            gl[l] = dXH[l][:, off:].to(dt)                         # h0
            gl[L + l] = dc[l].to(rest[L + l].dtype)                # c0
            if l == 0:
                gl[2 * L] = torch.mm(dG2[0].t(), xh[0][:T, :, :U + A].reshape(T * B, U + A))
            else:
                gl[2 * L + l] = torch.mm(dG2[l].t(), xh[l][:T, :, :I[l]].reshape(T * B, I[l]))
            gl[3 * L + l] = torch.mm(dG2[l].t(), xh[l][:T, :, I[l]:].reshape(T * B, U))
            if lnc is not None:
                dln = torch.empty(10, U, dtype=dt, device=dev)
                _check(Lb.px_ln_lstm_param_grad(_p(acc[l]), B, U, _p(dln), _DT[dt], st),
                       "ln_lstm_param_grad")
                o = 7 * L + 5 + 10 * l
                gl[o:o + 10] = list(dln.unbind(0))
                continue
            db = torch.sum(dG2[l], 0, dtype=torch.float32)
            gl[4 * L + l] = db.to(rest[4 * L + l].dtype)
            gl[5 * L + l] = db.to(rest[5 * L + l].dtype)
        qrows = qc[:, :, :U].reshape(T * B, U)
        if bah:
            gl[6 * L] = torch.mm(dpq.view(T * B, U).t(), qrows)
            out = torch.empty(U, **f32)
            _check(Lb.px_nmt_attn_param_grad(_p(part_v), B, U, _p(out), st), "nmt_attn_param_grad")
            gl[6 * L + 2] = out.to(vp.dtype)
            if part_b is not None:
                out = torch.empty(U, **f32)
                _check(Lb.px_nmt_attn_param_grad(_p(part_b), B, U, _p(out), st),
                       "nmt_attn_param_grad")
                gl[6 * L + 3] = out.to(bb.dtype)
        elif part_g is not None:
            out = torch.empty(1, **f32)
            _check(Lb.px_nmt_attn_param_grad(_p(part_g), B, 1, _p(out), st), "nmt_attn_param_grad")
            gl[6 * L + 1] = out.view(()).to(g.dtype)
        if std:
            gl[6 * L + 4] = torch.mm(datt.view(T * B, U).t(), qc.view(T * B, U + M))
        ctx.F = None
        return (None, None, demb, datt0, dk, dv, None, *gl)


def _nmt_args(h0, c0, w_ih, w_hh, b_ih, b_hh, w_q, g, v, b, w_a, masks, ln=None):
    """the node's tensor arguments; with LN-LSTM cells the 10 γ/β of each layer come last"""
    L = len(w_ih)
    if b_ih is None:
        b_ih = b_hh = [None] * L
    return (list(h0) + list(c0) + list(w_ih) + list(w_hh) + list(b_ih) + list(b_hh) +
            [w_q, g, v, b, w_a] + (list(masks) if masks is not None else [None] * L) +
            ([p for x in ln for p in x[0]] if ln is not None else []))


def _nmt_ln_params(cfg, rest):
    """per layer the 10 γ/β tensors from the node's tensor arguments (None for LSTM cells)"""
    if cfg["ln"] is None:
        return None
    L = cfg["L"]
    return [rest[7 * L + 5 + 10 * l:7 * L + 15 + 10 * l] for l in range(L)]


def _nmt_cfg(L, residual, v, w_a, output_attention, ln=None):
    return {"L": L, "standard": w_a is not None, "bahdanau": v is not None,
            "residual": tuple(bool(r) for r in residual),
            "output_attention": bool(output_attention),
            "ln": None if ln is None else tuple((tuple(float(e) for e in x[1]), float(x[2]))
                                                for x in ln)}


def nmt_attention_decoder(emb, h0, c0, att0, keys, values, pad, w_ih, w_hh, b_ih, b_hh, residual,
                          w_q=None, g=None, v=None, b=None, w_a=None, masks=None,
                          output_attention=True, ln=None):
    """All T steps of the NMT attention decoder's recurrence as ONE autograd node
    (`kernels/nmt_decoder.cu`).

    emb [B, T, U] (the decoder inputs), h0/c0 (per layer [B, U]), att0 [B, A] (the fed-back
    attention state), keys [B, S, U], values [B, S, M], pad [B, S] bool (True past each source
    length); per layer w_ih [4U, I_l], w_hh [4U, U], b_ih, b_hh (torch.nn.LSTM, gates i, f, g,
    o) and `residual` flags.  The attention: luong (`g`: scaled_luong's scale or None) or, with
    `v` = v′ (g·v/‖v‖ for normed_bahdanau, else v) and `w_q`, bahdanau (`b`: normed's bias).
    With `w_a` the architecture is *standard*: the L layers feed att_t = W_a·[q_t, ctx_t] back
    and the output is att_t or q_t (`output_attention`) -> [B, T, U].  Without it, *gnmt*: the
    layers (the bottom layer only) feed ctx_t back -> (h [B, T, U], ctx [B, T, M]).

    `masks` (per layer [T, B, I_l] in emb's dtype, or None) multiply each layer's input: the
    caller draws dropout there, from the same distribution as `F.dropout` but not from its
    random stream.

    `ln` (or None) makes every layer a layer-normalised LSTM (`LayerNormLSTM.cell`, gates i, j,
    f, o): per layer (the 10 γ/β of LN_i, LN_j, LN_f, LN_o, LN_c then their β, the 5 eps, the
    forget bias), with w_ih / w_hh the input and h columns of the bias-free kernel weight and
    b_ih = b_hh = None.  Callers check `nmt_decoder_applies` first.  Without autograd nothing is
    kept for a backward pass; the node never synchronises with the host."""
    L = len(w_ih)
    cfg = _nmt_cfg(L, residual, v, w_a, output_attention, ln)
    emb, att0 = emb.contiguous(), att0.contiguous()
    pad = pad.to(torch.bool).contiguous()
    if masks is not None:
        masks = [m.contiguous() for m in masks]
    args = _nmt_args(h0, c0, w_ih, w_hh, b_ih, b_hh, w_q, g, v, b, w_a, masks, ln)
    ins = [emb, att0, keys, values] + args
    if torch.is_grad_enabled() and any(a is not None and a.requires_grad for a in ins):
        return _NMTDecoderFn.apply(cfg, len(args), emb, att0, keys, values, pad, *args)
    W = dict(w_ih=w_ih, w_hh=w_hh, b_ih=b_ih, b_hh=b_hh, w_q=w_q, w_a=w_a,
             ln=None if ln is None else [x[0] for x in ln])
    attn = dict(w_q=w_q, g=g, v=v, b=b)
    F = _nmt_forward(cfg, emb, h0, c0, att0, keys, values, pad, W, attn, masks, False)
    return _nmt_outputs(cfg, F, emb.shape[2], output_attention)


@torch.no_grad()
def nmt_attention_decoder_step(emb_t, h0, c0, att0, keys, values, pad, w_ih, w_hh, b_ih, b_hh,
                               residual, w_q=None, g=None, v=None, b=None, w_a=None, masks=None,
                               ln=None):
    """One decoding step (T = 1, nothing saved) of `nmt_attention_decoder` from emb_t [B, U] ->
    (q [B, U] the top layer's output, att [B, A] the new fed-back state: W_a·[q, ctx] for
    standard, ctx for gnmt, h per layer, c per layer in c0's dtype)."""
    L = len(w_ih)
    cfg = _nmt_cfg(L, residual, v, w_a, True, ln)
    U = emb_t.shape[1]
    W = dict(w_ih=w_ih, w_hh=w_hh, b_ih=b_ih, b_hh=b_hh, w_q=w_q, w_a=w_a,
             ln=None if ln is None else [x[0] for x in ln])
    attn = dict(w_q=w_q, g=g, v=v, b=b)
    F = _nmt_forward(cfg, emb_t[:, None, :].contiguous(), h0, c0, att0, keys, values,
                     pad.to(torch.bool).contiguous(), W, attn, masks, False)
    last = F["last"]
    I = [U + att0.shape[1]] + [U] * (L - 1)
    hs = [F["xh"][l][last, :, I[l]:].clone() for l in range(L)]
    cs = [F["C"][l][last].to(c0[l].dtype) for l in range(L)]
    q = F["qc"][0, :, :U]
    att = F["att"][0] if w_a is not None else F["qc"][0, :, U:]
    return q, att, hs, cs


# ===========================================================================
# sampled softmax
# ===========================================================================
def sampled_softmax_reference(inputs, true_w, samp_w, true_b, samp_b, logq_true,
                              logq_samp, targets, sampled):
    """Per-example loss [N] (tf.nn.sampled_softmax_loss semantics)."""
    true_logits = _acc((inputs * true_w).sum(-1)) + _acc(true_b) - logq_true
    samp_logits = _acc(inputs @ samp_w.t()) + (_acc(samp_b) - logq_samp)
    hits = targets.unsqueeze(1) == sampled.unsqueeze(0)
    samp_logits = samp_logits.masked_fill(hits, float("-inf"))
    lse = torch.logsumexp(torch.cat([true_logits.unsqueeze(1), samp_logits], 1), 1)
    return lse - true_logits


class _SampledSoftmaxFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, inputs, true_w, samp_w, true_b, samp_b, logq_true, logq_samp,
                targets, sampled):
        L = _lib()
        N, S = inputs.shape[0], samp_w.shape[0]
        dt = inputs.dtype
        logits = inputs @ samp_w.t()                               # [N, S]  (cuBLAS)
        true_dot = (inputs.float() * true_w.float()).sum(-1)
        adj_t = (true_b.float() - logq_true).contiguous()
        adj_s = (samp_b.float() - logq_samp).contiguous()
        loss = torch.empty(N, dtype=torch.float32, device=inputs.device)
        dtrue = torch.empty(N, dtype=torch.float32, device=inputs.device)
        tg = targets.to(torch.int64).contiguous()
        sm = sampled.to(torch.int64).contiguous()
        _check(L.px_sampled_softmax(_p(logits), _p(true_dot), _p(adj_t), _p(adj_s), _p(tg),
                                    _p(sm), _p(loss), _p(dtrue), N, S, _DT[dt], _stream()),
               "sampled_softmax")
        _count(1)
        ctx.save_for_backward(inputs, true_w, samp_w, logits, dtrue)
        return loss

    @staticmethod
    def backward(ctx, g):
        inputs, true_w, samp_w, probs, dtrue = ctx.saved_tensors
        dt = inputs.dtype
        g = g.float()
        gt = (g * dtrue).unsqueeze(1)                              # [N,1]
        d_inputs = ((probs @ samp_w).float() * g.unsqueeze(1) +
                    gt * true_w.float()).to(dt)
        gi = (inputs.float() * g.unsqueeze(1)).to(dt)              # diag(g)·H
        d_samp_w = probs.t() @ gi
        d_true_w = (gt * inputs.float()).to(dt)
        d_samp_b = (probs.float().t() @ g) if probs.dtype == torch.float32 else \
            torch.mm(probs.t(), g.to(dt).unsqueeze(1), out_dtype=torch.float32).squeeze(1)
        d_true_b = gt.squeeze(1)
        return d_inputs, d_true_w, d_samp_w, d_true_b, d_samp_b, None, None, None, None


def sampled_softmax_loss(inputs, true_w, samp_w, true_b, samp_b, logq_true, logq_samp,
                         targets, sampled):
    if inputs.is_cuda and inputs.dtype in _DT and samp_w.shape[0] <= 256 * 64:
        return _SampledSoftmaxFn.apply(inputs, true_w.to(inputs.dtype),
                                       samp_w.to(inputs.dtype), true_b, samp_b,
                                       logq_true, logq_samp, targets, sampled)
    return sampled_softmax_reference(inputs, true_w, samp_w, true_b, samp_b, logq_true,
                                     logq_samp, targets, sampled)


# ---------------------------------------------------------------------------
# the whole loss head as one node
# ---------------------------------------------------------------------------
def _head_forward(inputs, w_all, adj, targets, sampled):
    """-> (probs [N,S] in inputs.dtype, loss [N] fp32, dtrue [N] fp32).  `w_all` holds the
    N true-class rows followed by the S sampled rows; `adj` = bias - log Q for the same
    N + S positions."""
    N, S = inputs.shape[0], w_all.shape[0] - inputs.shape[0]
    P = inputs.shape[1]
    logits = inputs @ w_all[N:].t()                                # [N, S]
    if inputs.is_cuda:
        loss = torch.empty(N, dtype=torch.float32, device=inputs.device)
        dtrue = torch.empty(N, dtype=torch.float32, device=inputs.device)
        _check(_lib().px_sampled_softmax_dot(
            _p(logits), _p(inputs), _p(w_all), P, _p(adj), _vp(adj.data_ptr() + 4 * N),
            _p(targets), _p(sampled), _p(loss), _p(dtrue), N, S, _DT[inputs.dtype], _stream()),
            "sampled_softmax_dot")
        _count(1)
        return logits, loss, dtrue
    # same math in PyTorch (host fabric / CPU tests of the node's algebra)
    tl = (inputs.float() * w_all[:N].float()).sum(-1) + adj[:N]
    a = logits.float() + adj[N:]
    a = a.masked_fill(targets.unsqueeze(1) == sampled.unsqueeze(0), float("-inf"))
    mx = torch.maximum(a.max(1).values, tl)
    e, et = torch.exp(a - mx.unsqueeze(1)), torch.exp(tl - mx)
    denom = e.sum(1) + et
    return (e / denom.unsqueeze(1)).to(inputs.dtype), mx + torch.log(denom) - tl, et / denom - 1.0


def _head_backward(G, inputs, w_all, g, row_w, dtrue, gi, d_w_all, db, grow):
    """in place: G -> d_inputs; fills gi, d_w_all[:N], db[:N], grow (see `px_ssm_bwd`)."""
    N, P = inputs.shape
    if inputs.is_cuda:
        _check(_lib().px_ssm_bwd(
            _p(G), _p(inputs), _p(w_all), _p(g), 0 if g.numel() == 1 else 1,
            _p(row_w) if row_w is not None else None, _p(dtrue), 1.0 / N, _p(gi), _p(d_w_all),
            _p(db), 1 if db.dtype == torch.bfloat16 else 0, _p(grow), N, P, _DT[inputs.dtype],
            _stream()), "ssm_bwd")
        _count(1)
        return
    gr = g.reshape(-1).float() * (1.0 / N)
    gr = gr.expand(N) if gr.numel() == 1 else gr
    if row_w is not None:
        gr = gr * row_w
    gt = gr * dtrue
    x, wt = inputs.float(), w_all[:N].float()
    G.copy_(G.float() * gr.unsqueeze(1) + gt.unsqueeze(1) * wt)
    gi.copy_(x * gr.unsqueeze(1))
    d_w_all[:N].copy_(x * gt.unsqueeze(1))
    db[:N].copy_(gt)
    grow.copy_(gr)


class _SampledSoftmaxHeadFn(torch.autograd.Function):
    """mean (optionally row-weighted) sampled-softmax loss of `inputs` [N, P] against the
    rows `w_all` / `b_all` of (targets ++ sampled).  Forward: logits GEMM + one kernel
    (true-class dot product, bias - log Q, accidental hits, log-sum-exp, loss, softmax
    probabilities in place).  Backward: two GEMMs, one GEMV and ONE glue kernel; the
    gradients of the looked-up rows come out as single [N+S, ·] tensors in lookup order —
    exactly what the co-lookup group's push kernel consumes (no slice / cat / cast
    launches in between).  Reference: tf.nn.sampled_softmax_loss as used by
    `examples/lm1b/language_model.py:96-107`."""

    @staticmethod
    def forward(ctx, inputs, w_all, b_all, adj, targets, sampled, row_w):
        probs, loss, dtrue = _head_forward(inputs, w_all, adj, targets, sampled)
        ctx.save_for_backward(inputs, w_all, probs, dtrue, row_w)
        ctx.b_meta = (tuple(b_all.shape), b_all.dtype)
        if row_w is not None:
            loss = loss * row_w
        return loss.mean()

    @staticmethod
    def backward(ctx, g):
        inputs, w_all, probs, dtrue, row_w = ctx.saved_tensors
        N, P = inputs.shape
        S = w_all.shape[0] - N
        dt, dev = inputs.dtype, inputs.device
        b_shape, b_dt = ctx.b_meta
        g = g.float().contiguous()
        G = probs @ w_all[N:]                                      # [N, P] -> d_inputs
        d_w_all = torch.empty(N + S, P, dtype=dt, device=dev)
        db = torch.empty(N + S, dtype=b_dt if b_dt in _DT else torch.float32, device=dev)
        gi = torch.empty(N, P, dtype=dt, device=dev)
        grow = torch.empty(N, dtype=dt, device=dev)
        _head_backward(G, inputs, w_all, g, row_w, dtrue, gi, d_w_all, db, grow)
        torch.mm(probs.t(), gi, out=d_w_all[N:])                   # d w_sampled
        if db.dtype == dt:                                         # d b_sampled
            torch.mm(probs.t(), grow.view(N, 1), out=db[N:].view(S, 1))
        elif dt == torch.bfloat16 and db.dtype == torch.float32:
            # fp32 straight out of the product: a bf16 result would round the gradient of an
            # fp32 bias to 8 bits
            db[N:].copy_(torch.mm(probs.t(), grow.view(N, 1), out_dtype=torch.float32).view(S))
        else:
            db[N:].copy_((probs.t() @ grow.view(N, 1)).view(S))
        db = db.view(b_shape)
        if db.dtype != b_dt:
            db = db.to(b_dt)
        return G, d_w_all, db, None, None, None, None


def sampled_softmax_head(inputs, w_all, b_all, logq, targets, sampled, row_w=None, adj=None):
    """Scalar mean sampled-softmax loss.  `w_all` [N+S, P], `b_all` [N+S] or [N+S, 1] and
    `logq` [N+S] are ordered (targets ++ sampled); `adj` may carry a precomputed
    ``b - log Q`` (fp32, no gradient — the bias gradient is produced from `b_all`)."""
    N, P = inputs.shape
    S = w_all.shape[0] - N
    dt = inputs.dtype
    vec = 4 if dt == torch.float32 else 8
    fused = (inputs.is_cuda and dt in _DT and w_all.dtype == dt and
             0 < S <= 256 * 64 and P % vec == 0 and b_all.numel() == N + S)
    if fused:
        inputs = inputs.contiguous()
        w_all = w_all.contiguous()
        fused = inputs.data_ptr() % 16 == 0 and w_all.data_ptr() % 16 == 0
    if not fused:
        b = b_all.reshape(-1)
        loss = sampled_softmax_loss(inputs, w_all[:N], w_all[N:], b[:N], b[N:], logq[:N],
                                    logq[N:], targets, sampled)
        if row_w is not None:
            loss = loss * row_w.to(loss.dtype)
        return loss.mean()
    if adj is None:
        adj = b_all.detach().reshape(-1).float() - logq
    adj = adj.float().contiguous()
    tg = targets.to(torch.int64).contiguous()
    sm = sampled.to(torch.int64).contiguous()
    rw = None if row_w is None else row_w.detach().float().contiguous()
    return _SampledSoftmaxHeadFn.apply(inputs, w_all, b_all, adj, tg, sm, rw)


# ===========================================================================
# dense linear cross-entropy (output layer + softmax loss)
# ===========================================================================
_LX_K_MAX = 8192


def linear_xent_applies(inputs, weight, bias):
    """The fused kernels take the head: CUDA tensors, bf16 inputs and weight, a bias that is None
    or bf16/fp32 [V], 8 <= K <= 8192 with K % 8 == 0 (the TMA row pitch is a multiple of 16
    bytes), and a contiguous, 16-byte-aligned weight (it is read in place)."""
    if not (inputs.is_cuda and weight.is_cuda and inputs.dtype == torch.bfloat16 and
            weight.dtype == torch.bfloat16 and inputs.dim() == 2 and weight.dim() == 2):
        return False
    V, K = weight.shape
    if bias is not None and not (bias.is_cuda and bias.dtype in (torch.bfloat16, torch.float32)
                                 and tuple(bias.shape) == (V,)):
        return False
    return (K % 8 == 0 and 8 <= K <= _LX_K_MAX and V >= 1 and weight.is_contiguous() and
            weight.data_ptr() % 16 == 0)


def linear_xent_chunk_rows(N, V):
    """Rows per chunk: the most whole 128-row tiles whose fp32 logits and bf16 softmax gradient
    ([n, V] each, rows padded to 8 columns) fit `consts.LINEAR_XENT_WS_BYTES`, never fewer than
    128, never more than N."""
    from .. import consts
    vp = (V + 7) // 8 * 8
    return min(N, max(128, consts.LINEAR_XENT_WS_BYTES // (vp * 6) // 128 * 128))


def linear_cross_entropy_reference(inputs, targets, weight, bias=None, row_weights=None):
    """The composition: ``(cross_entropy(linear(x, W, b).float(), t, reduction="none") * w).sum()``
    -> (loss, nll), with NaN in the nll of a target outside [0, V).  The oracle of the fused path
    and the path taken wherever `linear_xent_applies` is false."""
    if bias is not None and bias.dtype != inputs.dtype:
        bias = bias.to(inputs.dtype)
    V = weight.shape[0]
    valid = (targets >= 0) & (targets < V)
    nll = F.cross_entropy(F.linear(inputs, weight, bias).float(), targets.clamp(0, V - 1),
                          reduction="none")
    nll = torch.where(valid, nll, torch.full_like(nll, float("nan")))
    if row_weights is None:
        return nll.sum(), nll
    return (nll * row_weights.detach().to(nll.dtype)).sum(), nll


def _linear_xent(x, targets, weight, bias, row_w, want, chunk=None):
    """Chunked fused forward -> (nll [N] fp32, dX, fp32 dW, fp32 db), each gradient of the
    unscaled loss Σ w_i · nll_i or None as `want` (x, weight, bias) asks.  Per chunk of n rows:
    the logits kernel, the rows kernel (writing the bf16 gradient G when anything is wanted),
    then dX_c = G·W, dW += Gᵀ·X_c and db += Σ_rows G on cuBLAS."""
    L = _lib()
    N, K = x.shape
    V = weight.shape[0]
    dev = x.device
    grad = any(want)
    vp = (V + 7) // 8 * 8
    n = min(N, int(chunk)) if chunk else linear_xent_chunk_rows(N, V)
    nvt = (V + L.px_linear_xent_tile_cols() - 1) // L.px_linear_xent_tile_cols()
    nll = torch.empty(N, dtype=torch.float32, device=dev)
    dx = torch.empty(N, K, dtype=x.dtype, device=dev) if want[0] else None
    dw = torch.zeros(V, K, dtype=torch.float32, device=dev) if want[1] and N == 0 else None
    db = torch.zeros(1, V, dtype=torch.float32, device=dev) if want[2] and N == 0 else None
    if N == 0:
        return nll, dx, dw, db
    S = torch.empty(n, vp, dtype=torch.float32, device=dev)
    part = torch.empty(n, nvt, 2, dtype=torch.float32, device=dev)
    tgt = torch.empty(n, dtype=torch.float32, device=dev)
    G = torch.empty(n, vp, dtype=torch.bfloat16, device=dev) if grad else None
    ones = torch.ones(1, n, dtype=torch.bfloat16, device=dev) if want[2] else None
    kind = 0 if bias is None else (1 if bias.dtype == torch.bfloat16 else 2)
    st = _stream()
    for c0 in range(0, N, n):
        m = min(n, N - c0)
        _check(L.px_linear_xent_logits(_addr(x, c0 * K), m, K, _p(weight), V,
                                       None if bias is None else _p(bias), kind,
                                       _addr(targets, c0), _p(S), vp, _p(part), _p(tgt), st),
               "linear_xent_logits")
        _check(L.px_linear_xent_rows(_p(S), vp, _p(part), _p(tgt), _addr(targets, c0),
                                     None if row_w is None else _addr(row_w, c0), _addr(nll, c0),
                                     None if G is None else _p(G), m, V, st),
               "linear_xent_rows")
        _count(2)
        if not grad:
            continue
        Gc = G[:m, :V]
        if want[0]:
            torch.mm(Gc, weight, out=dx[c0:c0 + m])
        if want[1]:
            if c0 == 0:
                dw = torch.mm(Gc.t(), x[:m], out_dtype=torch.float32)
            else:
                torch.addmm(dw, Gc.t(), x[c0:c0 + m], out_dtype=torch.float32, out=dw)
        if want[2]:
            if c0 == 0:
                db = torch.mm(ones[:, :m], Gc, out_dtype=torch.float32)
            else:
                torch.addmm(db, ones[:, :m], Gc, out_dtype=torch.float32, out=db)
    return nll, dx, dw, db


def _weighted_sum(nll, row_w):
    return nll.sum() if row_w is None else (nll * row_w).sum()


class _LinearXentFn(torch.autograd.Function):
    """Forms the gradient of the loss during the forward (the row weights are known then), so
    the backward only scales the saved dX, dW and db by the incoming scalar."""

    @staticmethod
    def forward(ctx, x, weight, bias, targets, row_w, chunk):
        want = tuple(bool(w) for w in ctx.needs_input_grad[:3])
        nll, dx, dw, db = _linear_xent(x, targets, weight, bias, row_w, want, chunk)
        ctx.grads = (dx, dw, db)
        ctx.out_dtypes = (weight.dtype, None if bias is None else bias.dtype)
        ctx.mark_non_differentiable(nll)
        return _weighted_sum(nll, row_w), nll

    @staticmethod
    def backward(ctx, g, _):
        dx, dw, db = ctx.grads
        w_dt, b_dt = ctx.out_dtypes
        g = g.float()
        gx = None if dx is None else dx * g
        gw = None if dw is None else torch.mul(dw, g, out=torch.empty(dw.shape, dtype=w_dt,
                                                                      device=dw.device))
        gb = None if db is None else (db.view(-1) * g).to(b_dt)
        return gx, gw, gb, None, None, None


def linear_cross_entropy(inputs, targets, weight, bias=None, row_weights=None, chunk=None):
    """The fused head: (loss = Σ_i w_i · nll_i, nll [N] fp32) for bf16 inputs [N, K] against a
    dense output layer `weight` [V, K] (+ `bias` [V]), without an [N, V] logits tensor beyond
    one chunk of `chunk` rows (default `linear_xent_chunk_rows`).  Callers check
    `linear_xent_applies` first.  With autograd the gradient is formed during the forward; without
    it (no_grad, or nothing requiring a gradient) only the logits and rows kernels run."""
    x = inputs.contiguous()
    if x.data_ptr() % 16:
        x = x.clone()
    t = targets.to(device=x.device, dtype=torch.int64).contiguous()
    rw = None if row_weights is None else \
        row_weights.detach().to(device=x.device, dtype=torch.float32).contiguous()
    if torch.is_grad_enabled() and any(a is not None and a.requires_grad
                                       for a in (inputs, weight, bias)):
        return _LinearXentFn.apply(x, weight, bias, t, rw, chunk)
    nll = _linear_xent(x, t, weight, bias, rw, (False, False, False), chunk)[0]
    return _weighted_sum(nll, rw), nll
