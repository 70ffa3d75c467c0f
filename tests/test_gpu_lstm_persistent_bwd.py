"""The persistent backward LSTM recurrence (`px_lstm_bwd_persistent`: all T steps in one
cooperative launch) against fp64 at the benchmark's layer, against the per-step kernels
(`px_lstm_dm_cell_bwd` + the split-K `gemm_tn`) through the whole layer, under CUDA-graph replay,
and the shapes and dtypes that must keep the per-step kernels.

The oracle is the fp64 recurrence over exact bf16 operands (act, c_all, dH and the weights).  The
low-precision arm rounds where the per-step path rounds: dm to bf16, dgates to bf16, and the dh
product plus its addend to bf16.  Bounds are the calibrated ones of `test_gpu_lm1b_numerics`."""
import ctypes

import pytest
import torch

from tests.test_gpu_lm1b_numerics import (_assert_calibrated, _errs, _floor, _run_layer, _NAMES,
                                          _FACTOR_OF, FACTOR)

pytestmark = pytest.mark.gpu

_vp = ctypes.c_void_p
B_, S_, P_ = 128, 2048, 512
BF = torch.bfloat16


def _p(t):
    return _vp(t.data_ptr())


def _lib():
    from parallax_b200 import ops
    from parallax_b200.ops import fused  # noqa: F401  (register the signatures)
    return ops.lib()


def _bwd_inputs(T, B=B_, S=S_, P=P_, seed=0, tails=True):
    """Exact bf16 operands of the backward recurrence: activations as the forward stores them
    (σ(i), tanh(j), σ(f), σ(o) in bf16), fp32 cell states, dH, Wh, W_P; dL/dc_T and dL/dh_T
    (zero and None when `tails` is False).  Wh and W_P scale with their forward fan-in, as in
    `_chain_inputs` (0.04 and 0.03 at the bench layer)."""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    rn = lambda sc, *s: torch.randn(*s, device="cuda", generator=gen) * sc
    mk = lambda sc, *s: rn(sc, *s).to(BF)
    i, j, f, o = rn(1.5, T, B, 4 * S).split(S, -1)
    act = torch.cat([torch.sigmoid(i), torch.tanh(j), torch.sigmoid(f + 1.0), torch.sigmoid(o)],
                    -1).to(BF)
    return dict(act=act, c_all=rn(0.8, T + 1, B, S), dH=mk(0.05, T, B, P),
                Wh=mk(0.04 * (512 / P) ** 0.5, P, 4 * S), WP=mk(0.03 * (2048 / S) ** 0.5, S, P),
                dcT=rn(0.1, B, S) if tails else torch.zeros(B, S, device="cuda"),
                dhT=mk(0.05, B, P) if tails else None)


def _head(inp, dt):
    """dh_tot[T-1] = dH[T-1] + dh_T, in `dt` (the host's bf16 add for the low arm)."""
    dH, dhT = inp["dH"].to(dt), inp["dhT"]
    T = dH.shape[0]
    return dH[T - 1].clone() if dhT is None else dH[T - 1] + dhT.to(dt)


def _bwd_torch(inp, dt):
    """(dgates [T,B,4S], dh_tot [T,B,P], dh_rec [B,P], dc_0 [B,S]) of the recurrence in PyTorch:
    dt = float64 is the oracle, bfloat16 rounds where the per-step kernels round."""
    f64 = dt == torch.float64
    acc = torch.float64 if f64 else torch.float32
    dH, act, c_all = inp["dH"], inp["act"], inp["c_all"]
    Wh, WP = inp["Wh"].to(acc), inp["WP"].to(acc)
    T, S = dH.shape[0], WP.shape[0]
    dc = inp["dcT"].to(acc)
    dh = _head(inp, dt)
    dgs, dhs, dh_rec = [None] * T, [None] * T, None
    dhs[T - 1] = dh
    for t in range(T - 1, -1, -1):
        dm = dh.to(acc) @ WP.t()
        if not f64:
            dm = dm.to(BF).to(acc)                     # the dm tile rounded to bf16
        si, tj, sf, so = act[t].to(acc).split(S, 1)
        tc = torch.tanh(c_all[t + 1].to(acc))
        dcv = dc + dm * so * (1 - tc * tc)
        dg = torch.cat([dcv * tj * si * (1 - si), dcv * si * (1 - tj * tj),
                        dcv * c_all[t].to(acc) * sf * (1 - sf), dm * tc * so * (1 - so)], 1)
        dc = dcv * sf
        dg = dg.to(dt)
        dgs[t] = dg
        prod = dg.to(acc) @ Wh.t()
        if t > 0:
            dh = (prod + dH[t - 1].to(acc)).to(dt)
            dhs[t - 1] = dh
        else:
            dh_rec = prod.to(dt)
    return torch.stack(dgs), torch.stack(dhs), dh_rec, dc


def _buffers(inp):
    T, B, P = inp["dH"].shape
    S = inp["WP"].shape[0]
    dev = "cuda"
    return dict(dgates=torch.empty(T, B, 4 * S, dtype=BF, device=dev),
                dh_tot=torch.empty(T, B, P, dtype=BF, device=dev),
                dh_rec=torch.empty(B, P, dtype=BF, device=dev),
                dc=torch.empty(B, S, device=dev),
                ws=torch.empty(4 * S // 512, B, P, device=dev))


def _reset(inp, bufs):
    """The launch's in/out state: dc <- dL/dc_T, dh_tot[T-1] <- dH[T-1] + dL/dh_T."""
    bufs["dc"].copy_(inp["dcT"])
    bufs["dh_tot"][-1].copy_(_head(inp, BF))


def _launch(L, inp, bufs):
    T, B, P = inp["dH"].shape
    S = inp["WP"].shape[0]
    rc = L.px_lstm_bwd_persistent(_p(inp["dH"]), _p(inp["act"]), _p(inp["c_all"]), _p(inp["Wh"]),
                                  _p(inp["WP"]), _p(bufs["dc"]), _p(bufs["dgates"]),
                                  _p(bufs["dh_tot"]), _p(bufs["dh_rec"]), _p(bufs["ws"]),
                                  T, B, S, P, _vp(torch.cuda.current_stream().cuda_stream))
    assert rc == 0, rc


def _run_kernel(inp):
    L = _lib()
    bufs = _buffers(inp)
    _reset(inp, bufs)
    _launch(L, inp, bufs)
    torch.cuda.synchronize()
    return bufs["dgates"], bufs["dh_tot"], bufs["dh_rec"], bufs["dc"]


def _bits(t):
    return t.reshape(-1).view(torch.uint8)


def _skip_unless_bench_grid():
    """The bench layer needs 128 co-resident CTAs; a device with fewer SMs runs it per step."""
    if _lib().px_lstm_bwd_persistent_grid(B_, S_, P_) == 0:
        pytest.skip("this device cannot keep the bench layer's %d CTAs resident" % (S_ // 16))


@pytest.mark.parametrize("tails", [True, False])
@pytest.mark.parametrize("T", [1, 20])
def test_persistent_bwd_vs_fp64_bench_shape(T, tails):
    """B 128, S 2048, P 512 (the bench layer), with and without nonzero dL/dc_T and dL/dh_T:
    dgates, dh_tot[0 .. T-2], dh_rec and dL/dc_0 against fp64 on exact bf16 operands; a second
    launch gives the same bits."""
    _skip_unless_bench_grid()
    inp = _bwd_inputs(T, seed=T + 2 * tails, tails=tails)
    got = _run_kernel(inp)
    ref = _bwd_torch(inp, torch.float64)
    low = _bwd_torch(inp, BF)
    dg, dh_tot, dh_rec, dc = got
    _assert_calibrated("dgates", dg, ref[0], low[0], BF)
    if T > 1:
        _assert_calibrated("dh_tot", dh_tot[:T - 1], ref[1][:T - 1], low[1][:T - 1], BF)
    _assert_calibrated("dh_rec", dh_rec, ref[2], low[2], BF)
    _assert_calibrated("dc_0", dc, ref[3], low[3], BF)
    # the row the kernel reads, dh_tot[T-1], is left as it was
    assert torch.equal(dh_tot[T - 1], _head(inp, BF))
    again = _run_kernel(inp)
    for name, a_, b_ in zip(("dgates", "dh_tot", "dh_rec", "dc"), got, again):
        assert torch.equal(_bits(a_), _bits(b_)), name


def _bench_layer_inputs(T, E=512, seed=7, S=S_, P=P_):
    """Operands and output gradients of a layer; the weights scale with their fan-in (0.04 for
    both row blocks of W and 0.03 for W_P at the bench layer)."""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    rn = lambda sc, *s: torch.randn(*s, device="cuda", generator=gen) * sc
    mk = lambda sc, *s: rn(sc, *s).to(BF)
    fan_in = torch.tensor([0.04 * (512 / E) ** 0.5] * E + [0.04 * (512 / P) ** 0.5] * P,
                          device="cuda")[:, None]
    return dict(x=mk(1.0, T, B_, E), W=(rn(1.0, E + P, 4 * S) * fan_in).to(BF), b=mk(0.1, 4 * S),
                WP=mk(0.03 * (2048 / S) ** 0.5, S, P), c0=rn(0.5, B_, S), h0=mk(0.3, B_, P),
                gH=mk(0.1, T, B_, P), gc=rn(0.1, B_, S), gh=mk(0.1, B_, P))


def _layer_backward_launches(inp, dt, persistent, monkeypatch):
    """[outputs and gradients of `_run_layer("stacked")`], native launches of its backward."""
    from parallax_b200.ops import fused
    from parallax_b200.parallel import nvops
    with monkeypatch.context() as m:
        if not persistent:
            m.setattr(fused, "_bwd_persistent_ok", lambda *a: False)
        n0 = []
        out = _run_layer("stacked", inp, dt, before_backward=lambda: n0.append(nvops.launches["n"]))
        return out, nvops.launches["n"] - n0[0]


def test_persistent_bwd_layer_matches_per_step_kernels(monkeypatch):
    """The bench layer (T 20) through `_LSTMLayerFn` with the persistent backward against the same
    layer with the per-step backward (`px_lstm_dm_cell_bwd` + `gemm_tn`): the outputs are equal
    (same forward), every gradient (dx, dW, dbias, dW_P, dc0, dh0) is within the calibrated bound
    of fp64 with the per-step path as the low-precision arm, and the two are apart by no more than
    twice the per-step path's own error.  The backward is one native launch instead of 2T; two
    runs agree bit for bit."""
    import tests.test_gpu_lm1b_numerics as N
    from parallax_b200.ops import fused
    _skip_unless_bench_grid()
    T, E = 20, 512
    monkeypatch.setattr(N, "E_", E)
    inp = _bench_layer_inputs(T, E)
    W = inp["W"]
    assert fused._bwd_persistent_ok(BF, B_, S_, P_, W[E:], inp["WP"])
    new, n_new = _layer_backward_launches(inp, BF, True, monkeypatch)
    again, _ = _layer_backward_launches(inp, BF, True, monkeypatch)
    old, n_old = _layer_backward_launches(inp, BF, False, monkeypatch)
    assert n_new == 1 and n_old == 2 * T, (n_new, n_old)
    ref = _run_layer("reference", inp, torch.float64)
    for name, a_, b_ in zip(_NAMES, new, again):
        assert torch.equal(_bits(a_), _bits(b_)), name
    for name, n, o in zip(_NAMES[:3], new[:3], old[:3]):
        assert torch.equal(_bits(n), _bits(o)), name
    for name, n, o, r in zip(_NAMES[3:], new[3:], old[3:], ref[3:]):
        _assert_calibrated(name, n, r, o, BF, _FACTOR_OF.get(name, FACTOR))
        d = float((n.double() - o.double()).abs().max())
        e_old = _errs(o, r)[0]
        assert d <= 2 * e_old + _floor(BF, r.numel()) * float(r.abs().max()), (name, d, e_old)


def _check_graph_replay(S=S_, P=P_):
    """The kernel captured in a CUDA graph at (S, P), replayed three times with different dH, act
    and c_all copied in between (and dc, dh_tot[T-1] reset): each replay matches an eager launch
    on the same inputs bit for bit (the grid barriers start every replay in the right state)."""
    L = _lib()
    T = 6
    static = _bwd_inputs(T, S=S, P=P, seed=100)
    bufs = _buffers(static)
    _reset(static, bufs)
    _launch(L, static, bufs)                           # warm-up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        _launch(L, static, bufs)
    for r in range(3):
        fresh = _bwd_inputs(T, S=S, P=P, seed=200 + r)
        for k in ("dH", "act", "c_all", "dcT", "dhT"):
            static[k].copy_(fresh[k])
        _reset(static, bufs)
        g.replay()
        torch.cuda.synchronize()
        fresh["Wh"], fresh["WP"] = static["Wh"], static["WP"]
        eager = _run_kernel(fresh)
        for name, a_, b_ in zip(("dgates", "dh_tot", "dh_rec", "dc"),
                                (bufs["dgates"], bufs["dh_tot"], bufs["dh_rec"], bufs["dc"]),
                                eager):
            assert torch.equal(_bits(a_), _bits(b_)), (S, P, r, name)


def test_persistent_bwd_graph_replay_bit_identical():
    """`_check_graph_replay` at the bench layer (128 CTAs)."""
    _skip_unless_bench_grid()
    _check_graph_replay()


@pytest.mark.parametrize("dt,B,S,P", [(torch.float32, 128, 256, 128), (BF, 64, 256, 128),
                                      (BF, 256, 256, 128), (BF, 128, 200, 128),
                                      (BF, 128, 256, 576)])
def test_refused_shapes_take_the_per_step_kernels(monkeypatch, dt, B, S, P):
    """fp32, batches that are not one 128-row tile, S not a multiple of 128 units and P above 512
    run the per-step backward (more than one native launch) and still match fp64."""
    import tests.test_gpu_lm1b_numerics as N
    from tests.test_gpu_lstm_fused_step import _small_inputs
    from parallax_b200.ops import fused
    T, E = 3, 64
    L = _lib()
    ok = B == 128 and S % 128 == 0 and P <= 512
    assert L.px_lstm_bwd_persistent_grid(B, S, P) == (S // 16 if ok else 0)
    monkeypatch.setattr(N, "E_", E)
    inp = _small_inputs(T, B, E, S, P)
    W = inp["W"].to(dt)
    assert not fused._bwd_persistent_ok(dt, B, S, P, W[E:], inp["WP"].to(dt))
    got, n = _layer_backward_launches(inp, dt, True, monkeypatch)
    assert n >= T, n
    ref = _run_layer("reference", inp, torch.float64)
    low = _run_layer("reference", inp, dt)
    for name, g_, r, lo in zip(_NAMES, got, ref, low):
        _assert_calibrated("%s B%d S%d P%d/%s" % (dt, B, S, P, name), g_, r, lo, dt,
                           _FACTOR_OF.get(name, FACTOR))
