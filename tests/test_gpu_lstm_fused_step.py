"""The backward LSTM time step with the cell fused into the dm product (`px_lstm_dm_cell_bwd`)
at the bench layer's shape (B 128, S 2048, P 512): against fp64 on the exact operands the
kernel receives, and against the unfused pair (cuBLAS product + cell kernel) it replaces.  The
layer-level cases run shapes on both sides of the fused path's conditions."""
import pytest
import torch

from tests.test_gpu_lm1b_numerics import (_assert_calibrated, _gen, _lib, _p, _run_layer,
                                          _stream, _NAMES, _FACTOR_OF, FACTOR)

pytestmark = pytest.mark.gpu

B, S, P = 128, 2048, 512
BF = torch.bfloat16


def _cell_bwd64(act, cp, cn, dm, dc):
    si, tj, sf, so = act.double().split(act.shape[1] // 4, dim=1)
    tc = torch.tanh(cn.double())
    dmv = dm.double()
    dcv = dc.double() + dmv * so * (1 - tc * tc)
    dg = torch.cat([dcv * tj * si * (1 - si), dcv * si * (1 - tj * tj),
                    dcv * cp.double() * sf * (1 - sf), dmv * tc * so * (1 - so)], 1)
    return dg, dcv * sf


def _agree_bf16(name, got, ref):
    """Same quantity through two bf16 computations that differ in accumulation order only."""
    d = (got.double() - ref.double())
    rel_fro = float(d.norm()) / max(float(ref.double().norm()), 1e-300)
    rel_max = float(d.abs().max()) / max(float(ref.double().abs().max()), 1e-300)
    print("fused vs unfused %-8s rel-diff max %.2e fro %.2e" % (name, rel_max, rel_fro))
    assert rel_fro <= 2.0 ** -8 and rel_max <= 2.0 ** -7, (name, rel_max, rel_fro)


def _bwd_operands(seed):
    gen = _gen(seed)
    rn = lambda *s: torch.randn(*s, device="cuda", generator=gen)
    act = torch.cat([torch.sigmoid(rn(B, S) * 3), torch.tanh(rn(B, S) * 2),
                     torch.sigmoid(rn(B, S) * 3 + 1), torch.sigmoid(rn(B, S) * 3)], 1).to(BF)
    cp = rn(B, S) * 2.0
    cn = rn(B, S) * 2.0
    cn.view(-1)[::9] = 30.0                                # tanh(c) = 1: 1 − tanh² cancels
    dh = (rn(B, P) * 0.5).to(BF)
    WP = (rn(S, P) * 0.03).to(BF)
    dc = rn(B, S) * 0.5
    return act, cp, cn, dh, WP, dc


@pytest.mark.parametrize("bn", [16, 32, 64])
def test_dm_cell_bwd(bn):
    L = _lib()
    act, cp, cn, dh, WP, dc_in = _bwd_operands(21)
    # unfused pair: cuBLAS dm = dh·W_P^T, then the cell kernel
    dm0 = torch.mm(dh, WP.t())
    dc0 = dc_in.clone()
    dg0 = torch.empty(B, 4 * S, dtype=BF, device="cuda")
    assert L.px_lstm_cell_bwd(_p(dm0), _p(dc0), _p(act), _p(cp), _p(cn), _p(dg0), B, S, 1,
                              _stream()) == 0
    dc1 = dc_in.clone()
    dg1 = torch.full_like(dg0, float("nan"))
    assert L.px_lstm_dm_cell_bwd(_p(dh), _p(WP), _p(dc1), _p(act), _p(cp), _p(cn), _p(dg1),
                                 B, S, P, bn, _stream()) == 0
    torch.cuda.synchronize()
    # fp64 through the whole step on the exact operands; the unfused pair calibrates the bound
    dg64, dc64 = _cell_bwd64(act, cp, cn, dh.double() @ WP.double().t(), dc_in)
    _assert_calibrated("dgates bn%d" % bn, dg1, dg64, dg0, BF)
    _assert_calibrated("dc bn%d" % bn, dc1, dc64, dc0, BF)
    _agree_bf16("dgates", dg1, dg0)
    _agree_bf16("dc", dc1, dc0)
    # the epilogue rounds dm to bf16 as the product's output is rounded: given cuBLAS's dm, the
    # cell math is the unfused kernel's, so only elements whose dm rounded differently differ
    dm1 = (dh.double() @ WP.double().t()).to(BF)
    dg_r, dc_r = torch.empty_like(dg0), dc_in.clone()
    assert L.px_lstm_cell_bwd(_p(dm1), _p(dc_r), _p(act), _p(cp), _p(cn), _p(dg_r), B, S, 1,
                              _stream()) == 0
    torch.cuda.synchronize()
    same = (dg1.view(torch.int16) == dg_r.view(torch.int16)).double().mean()
    print("dgates bit-equal to the cell kernel on the exactly rounded dm: %.4f" % float(same))
    assert float(same) > 0.99


def test_fused_path_taken_at_bench_shape():
    from parallax_b200.ops import fused
    WP = torch.empty(S, P, dtype=BF, device="cuda")
    assert fused._fused_bwd_ok(BF, B, S, P, WP)
    assert not fused._fused_bwd_ok(torch.float32, B, S, P, WP.float())
    assert not fused._fused_bwd_ok(BF, 64, S, P, WP)
    assert not fused._fused_bwd_ok(BF, B, S, P, WP.t())


def test_dm_cell_bwd_rejects_bad_shapes():
    L = _lib()
    act, cp, cn, dh, WP, dc = _bwd_operands(22)
    dg = torch.empty(B, 4 * S, dtype=BF, device="cuda")
    args = (_p(dh), _p(WP), _p(dc), _p(act), _p(cp), _p(cn), _p(dg))
    assert L.px_lstm_dm_cell_bwd(*args, 64, S, P, 32, _stream()) == -1     # M not 128·k
    assert L.px_lstm_dm_cell_bwd(*args, B, S, P, 128, _stream()) == -1    # BN not 16/32/64
    assert L.px_lstm_dm_cell_bwd(*args, B, S - 8, P, 32, _stream()) == -1  # S not BN·k
    assert L.px_lstm_dm_cell_bwd(_p(dh), _p(WP), _p(dc[:, 1:]), *args[3:], B, S, P, 32,
                                 _stream()) == -1                         # misaligned dc


# ---------------------------------------------------------------------------
# whole layer on the shapes that fall back to the unfused pair
# ---------------------------------------------------------------------------
def _small_inputs(T, Bsz, E, S_, P_):
    gen = _gen(T * 1000 + Bsz)
    mk = lambda sc, *s: (torch.randn(*s, device="cuda", generator=gen) * sc).bfloat16()
    return dict(x=mk(1.0, T, Bsz, E), W=mk(0.08, E + P_, 4 * S_), b=mk(0.1, 4 * S_),
                WP=mk(0.06, S_, P_), c0=torch.randn(Bsz, S_, device="cuda", generator=gen) * 0.5,
                h0=mk(0.3, Bsz, P_), gH=mk(0.1, T, Bsz, P_),
                gc=torch.randn(Bsz, S_, device="cuda", generator=gen) * 0.1, gh=mk(0.1, Bsz, P_))


@pytest.mark.parametrize("Bsz,E,S_,P_,fused_bwd", [
    (128, 64, 256, 64, True),       # the smallest fused shape: one K-block of P
    (64, 128, 512, 128, False),     # batch not a whole 128-row tile: unfused pair
    (128, 128, 520, 128, False),    # S not a whole number of BN-column tiles: unfused pair
])
def test_layer_fused_and_fallback_shapes(monkeypatch, Bsz, E, S_, P_, fused_bwd):
    """The stacked layer (T 3) against fp64 on both sides of the fused path's conditions, with
    the layer's own input width patched into the numerics module's helpers.  Both persistent
    kernels are switched off, so the per-step kernels run even where the persistent ones would
    take the layer ((128, 256, 64) is in `test_gpu_lstm_persistent_shapes`)."""
    import tests.test_gpu_lm1b_numerics as N
    from parallax_b200.ops import fused
    WP = torch.empty(S_, P_, dtype=BF, device="cuda")
    assert fused._fused_bwd_ok(BF, Bsz, S_, P_, WP) == fused_bwd
    monkeypatch.setattr(N, "E_", E)
    monkeypatch.setattr(fused, "_fwd_persistent_ok", lambda *a: False)
    monkeypatch.setattr(fused, "_bwd_persistent_ok", lambda *a: False)
    inp = _small_inputs(3, Bsz, E, S_, P_)
    ref = _run_layer("reference", inp, torch.float64)
    low = _run_layer("reference", inp, BF)
    got = _run_layer("stacked", inp, BF)
    for name, g, r, lo in zip(_NAMES, got, ref, low):
        _assert_calibrated("B%d S%d P%d/%s" % (Bsz, S_, P_, name), g, r, lo, BF,
                           _FACTOR_OF.get(name, FACTOR))
