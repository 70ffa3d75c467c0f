"""The persistent forward LSTM recurrence (`px_lstm_fwd_persistent`: all T steps in one cooperative
launch) against fp64 at the benchmark's layer, against the per-step kernels, under CUDA-graph
replay, and the shapes and dtypes that must keep the per-step kernels.

Bounds are the calibrated ones of `test_gpu_lm1b_numerics`: the kernel's error against fp64 is held
to twice that of the same chain in PyTorch bf16 (addmm rounded to bf16, the cell in fp32, m and h
in bf16) plus a floor."""
import ctypes

import pytest
import torch

from tests.test_gpu_lm1b_numerics import _assert_calibrated, _errs, _floor

pytestmark = pytest.mark.gpu

_vp = ctypes.c_void_p
B_, S_, P_ = 128, 2048, 512


def _p(t):
    return _vp(t.data_ptr())


def _lib():
    from parallax_b200 import ops
    from parallax_b200.ops import fused  # noqa: F401  (register the signatures)
    return ops.lib()


def _chain_inputs(T, B=B_, S=S_, P=P_, seed=0):
    """Exact bf16 operands of the recurrence: xw = x·Wx + b, Wh, W_P, and fp32 c0.  Wh and W_P
    scale with their fan-in (0.04 and 0.03 at the bench layer), so the gates stay O(1) at every
    S and P."""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    mk = lambda sc, *s: (torch.randn(*s, device="cuda", generator=gen) * sc).bfloat16()
    return dict(xw=mk(1.0, T, B, 4 * S), Wh=mk(0.04 * (512 / P) ** 0.5, P, 4 * S),
                WP=mk(0.03 * (2048 / S) ** 0.5, S, P),
                c0=torch.randn(B, S, device="cuda", generator=gen) * 0.5, h0=mk(0.3, B, P))


def _chain_torch(inp, dt, fb=1.0):
    """(act [T,B,4S], c_all [T+1,B,S], m_all [T,B,S], h_all [T+1,B,P]) of the recurrence in
    PyTorch: dt = float64 is the oracle, bfloat16 rounds where the per-step kernels round."""
    acc = torch.float64 if dt == torch.float64 else torch.float32
    xw, Wh, WP = (inp[k].to(dt) for k in ("xw", "Wh", "WP"))
    S = WP.shape[0]
    c, h = inp["c0"].to(acc), inp["h0"].to(dt)
    acts, cs, ms, hs = [], [c], [], [h]
    for t in range(xw.shape[0]):
        g = torch.addmm(xw[t], h, Wh).to(acc)
        i, j, f, o = g.split(S, dim=1)
        si, tj, sf, so = torch.sigmoid(i), torch.tanh(j), torch.sigmoid(f + fb), torch.sigmoid(o)
        c = sf * c + si * tj
        m = (so * torch.tanh(c)).to(dt)
        h = m @ WP
        acts.append(torch.cat([si, tj, sf, so], 1).to(dt))
        cs.append(c)
        ms.append(m)
        hs.append(h)
    return torch.stack(acts), torch.stack(cs), torch.stack(ms), torch.stack(hs)


def _buffers(inp):
    T, B, G = inp["xw"].shape
    S, P = inp["WP"].shape
    dev, bf = "cuda", torch.bfloat16
    act = torch.empty(T, B, G, dtype=bf, device=dev)
    c_all = torch.empty(T + 1, B, S, device=dev)
    m_all = torch.empty(T, B, S, dtype=bf, device=dev)
    h_all = torch.empty(T + 1, B, P, dtype=bf, device=dev)
    ws = torch.empty(S // 128, B, P, device=dev)
    return act, c_all, m_all, h_all, ws


def _launch(L, inp, bufs, fb=1.0):
    act, c_all, m_all, h_all, ws = bufs
    T, B, _ = inp["xw"].shape
    S, P = inp["WP"].shape
    rc = L.px_lstm_fwd_persistent(_p(inp["xw"]), _p(inp["Wh"]), _p(inp["WP"]), _p(act), _p(c_all),
                                  _p(m_all), _p(h_all), _p(ws), T, B, S, P, fb,
                                  _vp(torch.cuda.current_stream().cuda_stream))
    assert rc == 0, rc


def _run_kernel(inp, fb=1.0):
    L = _lib()
    bufs = _buffers(inp)
    bufs[1][0].copy_(inp["c0"])
    bufs[3][0].copy_(inp["h0"])
    _launch(L, inp, bufs, fb)
    torch.cuda.synchronize()
    return bufs[:4]


_NAMES = ("act", "c_all", "m_all", "h_all")


def _skip_unless_bench_grid():
    """The bench layer needs 128 co-resident CTAs; a device with fewer SMs runs it per step."""
    if _lib().px_lstm_fwd_persistent_grid(B_, S_, P_) == 0:
        pytest.skip("this device cannot keep the bench layer's %d CTAs resident" % (S_ // 16))


@pytest.mark.parametrize("T", [1, 20])
def test_persistent_fwd_vs_fp64_bench_shape(T):
    """B 128, S 2048, P 512 (the bench layer): H, c_T, h_T and the tensors the backward chain
    reads (act, c_all, m_all) against fp64 on exact bf16 operands."""
    _skip_unless_bench_grid()
    inp = _chain_inputs(T, seed=T)
    got = _run_kernel(inp)
    ref = _chain_torch(inp, torch.float64)
    low = _chain_torch(inp, torch.bfloat16)
    act, c_all, m_all, h_all = got
    _assert_calibrated("H", h_all[1:], ref[3][1:], low[3][1:], torch.bfloat16)
    _assert_calibrated("c_T", c_all[T], ref[1][T], low[1][T], torch.bfloat16)
    _assert_calibrated("h_T", h_all[T], ref[3][T], low[3][T], torch.bfloat16)
    for name, g, r, lo in zip(_NAMES[:3], got[:3], ref[:3], low[:3]):
        _assert_calibrated(name, g[-T:], r[-T:], lo[-T:], torch.bfloat16)
    # the rows the kernel reads, c0 and h0, are left as they were
    assert torch.equal(c_all[0], inp["c0"]) and torch.equal(h_all[0], inp["h0"])


def test_persistent_fwd_matches_per_step_kernels_and_is_deterministic():
    """The layer through the persistent kernel against the same layer through the per-step
    kernels (addmm, cell kernel, mm): their difference stays within the bf16 chain's own error
    against fp64; and two runs of the persistent kernel agree bit for bit."""
    from parallax_b200.ops import fused
    from parallax_b200.parallel import nvops
    _skip_unless_bench_grid()
    T, E = 20, 512
    gen = torch.Generator(device="cuda").manual_seed(7)
    mk = lambda sc, *s: (torch.randn(*s, device="cuda", generator=gen) * sc).bfloat16()
    x, W, b = mk(1.0, T, B_, E), mk(0.04, E + P_, 4 * S_), mk(0.1, 4 * S_)
    WP, h0 = mk(0.03, S_, P_), mk(0.3, B_, P_)
    c0 = torch.randn(B_, S_, device="cuda", generator=gen) * 0.5
    assert fused._fwd_persistent_ok(torch.bfloat16, B_, S_, P_, W[E:], WP)
    outs = []
    with torch.no_grad():
        for persistent in (True, True, False):
            ok = fused._fwd_persistent_ok
            try:
                if not persistent:
                    fused._fwd_persistent_ok = lambda *a: False
                n0 = nvops.launches["n"]
                outs.append(fused.lstm_layer_stacked(x, W, b, WP, c0, h0, 1.0))
                torch.cuda.synchronize()
                assert nvops.launches["n"] - n0 == (1 if persistent else T)
            finally:
                fused._fwd_persistent_ok = ok
        ref = fused.lstm_layer_reference(x.double(), W[:E].double(), W[E:].double(), b.double(),
                                         WP.double(), c0.double(), h0.double(), 1.0)
    new, again, old = outs
    for a_, b_ in zip(new, again):
        assert torch.equal(a_.reshape(-1).view(torch.uint8), b_.reshape(-1).view(torch.uint8))
    for name, n, o, r in zip(("H", "c_T", "h_T"), new, old, ref):
        # the persistent kernel within the calibrated bound, with the per-step kernels as the
        # low-precision run; and the two apart by no more than twice the per-step error
        _assert_calibrated(name, n, r, o, torch.bfloat16)
        d = float((n.double() - o.double()).abs().max())
        e_old = _errs(o, r)[0]
        assert d <= 2 * e_old + _floor(torch.bfloat16, r.numel()) * float(r.abs().max()), \
            (name, d, e_old)


def _check_graph_replay(S=S_, P=P_):
    """The kernel captured in a CUDA graph at (S, P), replayed three times with different xw, h0
    and c0 copied in between: each replay matches an eager launch on the same inputs bit for bit
    (the grid barriers start every replay in the right state)."""
    L = _lib()
    T = 6
    static = _chain_inputs(T, S=S, P=P, seed=100)
    bufs = _buffers(static)
    bufs[1][0].copy_(static["c0"])
    bufs[3][0].copy_(static["h0"])
    _launch(L, static, bufs)                           # warm-up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        _launch(L, static, bufs)
    for r in range(3):
        fresh = _chain_inputs(T, S=S, P=P, seed=200 + r)
        static["xw"].copy_(fresh["xw"])
        bufs[1][0].copy_(fresh["c0"])
        bufs[3][0].copy_(fresh["h0"])
        g.replay()
        torch.cuda.synchronize()
        fresh["Wh"], fresh["WP"] = static["Wh"], static["WP"]
        eager = _run_kernel(fresh)
        for name, a_, b_ in zip(_NAMES, bufs[:4], eager):
            assert torch.equal(a_.reshape(-1).view(torch.uint8), b_.reshape(-1).view(torch.uint8)), \
                (S, P, r, name)


def test_persistent_fwd_graph_replay_bit_identical():
    """`_check_graph_replay` at the bench layer (128 CTAs)."""
    _skip_unless_bench_grid()
    _check_graph_replay()


@pytest.mark.parametrize("dt,B,S", [(torch.float32, 128, 256), (torch.bfloat16, 64, 256),
                                    (torch.bfloat16, 128, 200)])
def test_refused_shapes_take_the_per_step_kernels(dt, B, S):
    """fp32, a batch that is not one 128-row tile, and S not a multiple of 128 units run the
    per-step kernels (T native launches, not one) and still match fp64."""
    from parallax_b200.ops import fused
    from parallax_b200.parallel import nvops
    T, E, P = 4, 64, 128
    L = _lib()
    assert L.px_lstm_fwd_persistent_grid(B, S, P) == (S // 16 if B == 128 and S % 128 == 0 else 0)
    gen = torch.Generator(device="cuda").manual_seed(B + S)
    mk = lambda sc, *s: (torch.randn(*s, device="cuda", generator=gen) * sc).to(dt)
    x, W, b = mk(1.0, T, B, E), mk(0.1, E + P, 4 * S), mk(0.1, 4 * S)
    WP, h0 = mk(0.06, S, P), mk(0.3, B, P)
    c0 = torch.randn(B, S, device="cuda", generator=gen) * 0.5
    assert not fused._fwd_persistent_ok(dt, B, S, P, W[E:], WP)
    with torch.no_grad():
        n0 = nvops.launches["n"]
        got = fused.lstm_layer_stacked(x, W, b, WP, c0, h0, 1.0)
        torch.cuda.synchronize()
        assert nvops.launches["n"] - n0 == T
        ref = fused.lstm_layer_reference(x.double(), W[:E].double(), W[E:].double(), b.double(),
                                         WP.double(), c0.double(), h0.double(), 1.0)
        low = fused.lstm_layer_reference(x, W[:E], W[E:], b, WP, c0, h0, 1.0)
    for name, g_, r, lo in zip(("H", "c_T", "h_T"), got, ref, low):
        _assert_calibrated(name, g_, r, lo, dt)
