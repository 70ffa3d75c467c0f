"""The persistent LSTM kernels (`px_lstm_fwd_persistent`, `px_lstm_bwd_persistent`) against fp64
at every kind of layer their grid queries accept, not only the bench layer (S 2048, P 512), and
the boundary of those queries.

The kernels take B 128 in bf16, S any multiple of 128 while the S/16 CTAs stay resident (S <= 2048
on a 132-SM H100) and P any multiple of 64 up to 512.  Their shape-dependent logic is idle at the
bench layer, where every CTA takes part in the split-K product (phase B forward, phase 2 backward:
(P/64)·(S/128) participants of S/16), the slot sum runs over 16 slots and h_t / dh_t has all 8
K-blocks.  The sweep covers the rest:

| S    | P   | grid | participants | slots | what the row is there for                            |
|------|-----|------|--------------|-------|------------------------------------------------------|
| 128  | 64  | 8    | 1            | 1     | smallest grid; one participant, slot and K-block     |
| 128  | 512 | 8    | 8            | 1     | one slot (the slot loop's body never runs), 8 K-blocks |
| 256  | 64  | 16   | 2            | 2     | one slot step; 1 CTA in 8 takes part                 |
| 384  | 128 | 24   | 6            | 3     | odd slot count, 2 K-blocks                           |
| 640  | 192 | 40   | 15           | 5     | odd K-block count (3) and odd participant count      |
| 1024 | 256 | 64   | 32           | 8     | half the grid; the parked gate tile sizes the forward's A region (P <= 256) |
| 1920 | 320 | 120  | 75           | 15    | 5 K-blocks; grid just under 128, odd slot count      |
| 2048 | 384 | 128  | 96           | 16    | full grid with 3/4 of it taking part, 6 K-blocks     |
| 1536 | 448 | 96   | 84           | 12    | 7 K-blocks                                           |
| 2048 | 64  | 128  | 16           | 16    | full grid, one K-block, 1/8 of the grid takes part   |

Each kernel runs with NaN in everything it must write and a sentinel row past every output, and is
held to the calibrated bound of `test_gpu_lm1b_numerics` (error against fp64 within twice the
PyTorch bf16 chain's, plus a floor) over each whole output and over each CTA's own tile.  The
weights scale with their fan-in (`_chain_inputs`, `_bwd_inputs`), so the gates stay O(1) at every
shape.  Measured ratios are printed (`pytest -s`)."""
import os
import subprocess
import sys

import pytest
import torch

from tests.test_gpu_lm1b_numerics import (_assert_calibrated, _errs, _floor, _run_layer, _NAMES,
                                          _FACTOR_OF, FACTOR)
from tests.test_gpu_lstm_persistent_fwd import (_chain_inputs, _chain_torch, _run_kernel, _lib,
                                                _launch as _fwd_launch,
                                                _check_graph_replay as _fwd_graph_replay)
from tests.test_gpu_lstm_persistent_bwd import (_bwd_inputs, _bwd_torch, _head, _bits,
                                                _bench_layer_inputs,
                                                _launch as _bwd_launch,
                                                _run_kernel as _bwd_run_kernel,
                                                _check_graph_replay as _bwd_graph_replay)

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
NAN = float("nan")
SHAPES = [(128, 64), (128, 512), (256, 64), (384, 128), (640, 192), (1024, 256), (1920, 320),
          (2048, 384), (1536, 448), (2048, 64)]
_IDS = ["S%d-P%d" % sp for sp in SHAPES]
_QUERIES = ("px_lstm_fwd_persistent_grid", "px_lstm_bwd_persistent_grid")


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _expected_grid(B, S, P):
    """The documented rule: S/16 CTAs for B 128, S a multiple of 128, P a multiple of 64 up to 512,
    while the device keeps one CTA per SM resident; else 0."""
    ok = B == 128 and S > 0 and S % 128 == 0 and 0 < P <= 512 and P % 64 == 0
    return S // 16 if ok and S // 16 <= _sms() else 0


def _first_refused_S():
    """The first multiple of 128 whose S/16 CTAs outnumber the SMs (2176 on a 132-SM H100)."""
    return 128 * (16 * _sms() // 128 + 1)


def _require_persistent(S, P):
    """Both grid queries give the documented answer for (128, S, P); skip where that answer is no
    because this device has too few SMs for S/16 CTAs."""
    want = _expected_grid(128, S, P)
    for q in _QUERIES:
        assert getattr(_lib(), q)(128, S, P) == want, (q, S, P, want)
    if want == 0:
        pytest.skip("S %d needs %d co-resident CTAs; this device has %d SMs"
                    % (S, S // 16, _sms()))


def _per_step_bwd_launches(T, S, P):
    """Native launches of the per-step backward of a bf16 batch-128 layer: T of the dm/cell
    kernel, plus T of the split-K `gemm_tn` where it takes the dh product (P in 64-column tiles,
    4S in 1024-column tiles)."""
    return T * (2 if P % 64 == 0 and (4 * S) % 1024 == 0 else 1)


# ---------------------------------------------------------------------------------------- tiles
def _gate_tiles(x):
    """[T, 128, 4S] -> [S/16, n]: row j holds CTA j's rows 64·(j % 2) … +63 and units
    32·(j // 2) … +31 of all four gate blocks."""
    T, _, G = x.shape
    S = G // 4
    return x.reshape(T, 2, 64, 4, S // 32, 32).permute(4, 1, 0, 2, 3, 5).reshape(S // 16, -1)


def _unit_tiles(x):
    """[T, 128, S] -> [S/16, n]: CTA j's rows and units, as `_gate_tiles`."""
    T, _, S = x.shape
    return x.reshape(T, 2, 64, S // 32, 32).permute(3, 1, 0, 2, 4).reshape(S // 16, -1)


def _col_tiles(x):
    """[T, 128, P] -> [P/64, n]: one 64-column N-tile of the split-K product per row."""
    T, B, P = x.shape
    return x.reshape(T, B, P // 64, 64).permute(2, 0, 1, 3).reshape(P // 64, -1)


def _assert_tiles(name, got, ref, low, factor=FACTOR):
    """`_assert_calibrated`'s bf16 criterion on every row of [tiles, n]: one misplaced or stale
    tile must not hide inside a norm taken over all of them."""
    d_k, d_t = got.double() - ref, low.double() - ref
    nr = ref.norm(dim=1)
    nr = torch.where(nr > 0, nr, torch.ones_like(nr))
    floor = _floor(BF, ref.shape[1])
    bound_max = factor * d_t.abs().amax(1) + floor * ref.abs().amax(1)
    bound_fro = factor * d_t.norm(dim=1) / nr + floor
    used = torch.maximum(d_k.abs().amax(1) / bound_max, d_k.norm(dim=1) / nr / bound_fro)
    worst = int(used.argmax())
    print("tiles %-32s %3d tiles, worst (%d) at %.3f of its bound"
          % (name, used.numel(), worst, float(used[worst])))
    assert bool((used <= 1).all()), (name, [int(i) for i in torch.nonzero(used > 1)[:, 0]])


def _sentinel_rows(full):
    """Fill the last row of every buffer with a fixed bit pattern -> copies to compare against."""
    rows = {}
    for k, v in full.items():
        bits = v[-1].view(torch.int16 if v.element_size() == 2 else torch.int32)
        bits.fill_(0x5A5A if v.element_size() == 2 else 0x5A5A5A5A)
        rows[k] = v[-1].clone()
    return rows


def _assert_sentinels(full, rows, tag):
    for k, v in full.items():
        assert torch.equal(_bits(v[-1]), _bits(rows[k])), "%s: written past the end of %s" % (tag, k)


# ------------------------------------------------------------------------------ forward kernel
@pytest.mark.parametrize("T", [1, 2, 7])
@pytest.mark.parametrize("S,P", SHAPES, ids=_IDS)
def test_fwd_kernel_vs_fp64(S, P, T):
    """act, c, m and H against fp64, whole and per CTA tile (per N-tile for H), from buffers
    poisoned with NaN; nothing written past T steps or into the inputs; a second launch gives the
    same bits.  T 1 has no trailing barrier, T 2 one handoff, T 7 ends on the other mbarrier
    phase."""
    _require_persistent(S, P)
    tag = "fwd S%d P%d T%d" % (S, P, T)
    inp = _chain_inputs(T, S=S, P=P, seed=S + P + T)
    B = 128
    full = dict(act=torch.full((T + 1, B, 4 * S), NAN, dtype=BF, device="cuda"),
                c_all=torch.full((T + 2, B, S), NAN, device="cuda"),
                m_all=torch.full((T + 1, B, S), NAN, dtype=BF, device="cuda"),
                h_all=torch.full((T + 2, B, P), NAN, dtype=BF, device="cuda"),
                ws=torch.full((S // 128 + 1, B, P), NAN, device="cuda"))
    full["c_all"][0].copy_(inp["c0"])
    full["h_all"][0].copy_(inp["h0"])
    tails = _sentinel_rows(full)
    before = {k: inp[k].clone() for k in ("xw", "Wh", "WP")}
    _fwd_launch(_lib(), inp, tuple(full[k][:-1] for k in ("act", "c_all", "m_all", "h_all", "ws")))
    torch.cuda.synchronize()
    _assert_sentinels(full, tails, tag)
    for k, v in before.items():
        assert torch.equal(_bits(inp[k]), _bits(v)), (tag, k)
    assert torch.equal(_bits(full["c_all"][0]), _bits(inp["c0"])), tag
    assert torch.equal(_bits(full["h_all"][0]), _bits(inp["h0"])), tag

    act, c_all, m_all, h_all = (full[k][:-1] for k in ("act", "c_all", "m_all", "h_all"))
    ref = _chain_torch(inp, torch.float64)
    low = _chain_torch(inp, BF)
    outs = (("act", act, ref[0], low[0], _gate_tiles),
            ("c", c_all[1:], ref[1][1:], low[1][1:], _unit_tiles),
            ("m", m_all, ref[2], low[2], _unit_tiles),
            ("H", h_all[1:], ref[3][1:], low[3][1:], _col_tiles))
    for name, g, r, lo, tiles in outs:
        _assert_calibrated("%s/%s" % (tag, name), g, r, lo, BF)
        _assert_tiles("%s/%s" % (tag, name), tiles(g), tiles(r), tiles(lo))

    again = _run_kernel(inp)
    for name, a_, b_ in zip(("act", "c_all", "m_all", "h_all"), (act, c_all, m_all, h_all), again):
        assert torch.equal(_bits(a_), _bits(b_)), (tag, name)


# ----------------------------------------------------------------------------- backward kernel
@pytest.mark.parametrize("T,tails", [(1, True), (2, True), (7, True), (7, False)])
@pytest.mark.parametrize("S,P", SHAPES, ids=_IDS)
def test_bwd_kernel_vs_fp64(S, P, T, tails):
    """dgates, dh_tot[0 .. T-2], dh_rec and dL/dc_0 against fp64, whole and per CTA tile (per
    N-tile for dh), from buffers poisoned with NaN; nothing written past the outputs or into the
    inputs; a second launch gives the same bits."""
    _require_persistent(S, P)
    tag = "bwd S%d P%d T%d%s" % (S, P, T, "" if tails else " no-tails")
    inp = _bwd_inputs(T, S=S, P=P, seed=S + P + T + 2 * tails, tails=tails)
    B = 128
    full = dict(dgates=torch.full((T + 1, B, 4 * S), NAN, dtype=BF, device="cuda"),
                dh_tot=torch.full((T + 1, B, P), NAN, dtype=BF, device="cuda"),
                dh_rec=torch.full((2, B, P), NAN, dtype=BF, device="cuda"),
                dc=torch.full((B + 1, S), NAN, device="cuda"),
                ws=torch.full((4 * S // 512 + 1, B, P), NAN, device="cuda"))
    full["dc"][:B].copy_(inp["dcT"])
    full["dh_tot"][T - 1].copy_(_head(inp, BF))
    sentinels = _sentinel_rows(full)
    bufs = {k: v[:-1] for k, v in full.items()}
    bufs["dh_rec"] = full["dh_rec"][0]
    before = {k: inp[k].clone() for k in ("dH", "act", "c_all", "Wh", "WP")}
    _bwd_launch(_lib(), inp, bufs)
    torch.cuda.synchronize()
    _assert_sentinels(full, sentinels, tag)
    for k, v in before.items():
        assert torch.equal(_bits(inp[k]), _bits(v)), (tag, k)
    assert torch.equal(_bits(bufs["dh_tot"][T - 1]), _bits(_head(inp, BF))), tag

    ref = _bwd_torch(inp, torch.float64)
    low = _bwd_torch(inp, BF)
    dg, dh_tot, dh_rec, dc = bufs["dgates"], bufs["dh_tot"], bufs["dh_rec"], bufs["dc"]
    outs = [("dgates", dg, ref[0], low[0], _gate_tiles),
            ("dh_rec", dh_rec[None], ref[2][None], low[2][None], _col_tiles),
            ("dc_0", dc[None], ref[3][None], low[3][None], _unit_tiles)]
    if T > 1:
        outs.append(("dh_tot", dh_tot[:T - 1], ref[1][:T - 1], low[1][:T - 1], _col_tiles))
    for name, g, r, lo, tiles in outs:
        _assert_calibrated("%s/%s" % (tag, name), g, r, lo, BF)
        _assert_tiles("%s/%s" % (tag, name), tiles(g), tiles(r), tiles(lo))

    again = _bwd_run_kernel(inp)
    for name, a_, b_ in zip(("dgates", "dh_tot", "dh_rec", "dc"), (dg, dh_tot, dh_rec, dc), again):
        assert torch.equal(_bits(a_), _bits(b_)), (tag, name)


# --------------------------------------------------------------------------------- whole layer
def _layer(inp, fwd, bwd, monkeypatch):
    """`_run_layer("stacked")` with the persistent forward / backward left on or switched off ->
    (outputs and gradients, native launches of the forward, native launches of the backward)."""
    from parallax_b200.ops import fused
    from parallax_b200.parallel import nvops
    with monkeypatch.context() as m:
        if not fwd:
            m.setattr(fused, "_fwd_persistent_ok", lambda *a: False)
        if not bwd:
            m.setattr(fused, "_bwd_persistent_ok", lambda *a: False)
        n = [nvops.launches["n"]]
        out = _run_layer("stacked", inp, BF, before_backward=lambda: n.append(nvops.launches["n"]))
        return out, n[1] - n[0], nvops.launches["n"] - n[1]


def _assert_layer(tag, got, low, ref):
    for name, g, lo, r in zip(_NAMES, got, low, ref):
        _assert_calibrated("%s/%s" % (tag, name), g, r, lo, BF, _FACTOR_OF.get(name, FACTOR))


@pytest.mark.parametrize("S,P,E", [(1024, 256, 256), (512, 128, 128), (2048, 256, 512)])
def test_layer_persistent_vs_fp64_and_per_step(monkeypatch, S, P, E):
    """The stacked layer (T 8) with autograd: one native launch each way; outputs and every
    gradient within the calibrated bound of fp64 with the per-step kernels as the low arm, and no
    further from the per-step result than twice the per-step path's own error."""
    import tests.test_gpu_lm1b_numerics as N
    _require_persistent(S, P)
    T = 8
    tag = "layer S%d P%d E%d" % (S, P, E)
    monkeypatch.setattr(N, "E_", E)
    inp = _bench_layer_inputs(T, E, seed=S + P + E, S=S, P=P)
    new, nf, nb = _layer(inp, True, True, monkeypatch)
    old, of, ob = _layer(inp, False, False, monkeypatch)
    assert (nf, nb, of, ob) == (1, 1, T, _per_step_bwd_launches(T, S, P)), (nf, nb, of, ob)
    ref = _run_layer("reference", inp, torch.float64)
    _assert_layer(tag, new, old, ref)
    for name, n, o, r in zip(_NAMES, new, old, ref):
        d = float((n.double() - o.double()).abs().max())
        e_old = _errs(o, r)[0]
        assert d <= 2 * e_old + _floor(BF, r.numel()) * float(r.abs().max()), (tag, name, d, e_old)


@pytest.mark.parametrize("offset", [4, 1])
def test_layer_persistent_fwd_then_per_step_bwd(monkeypatch, offset):
    """S 1024, P 256, T 8 with dL/dH `offset` bf16 elements past a 16-byte boundary: the
    persistent backward refuses it, so the per-step backward runs on the act, c_all, m_all and
    h_all the persistent forward wrote.  At 8 bytes the dh product is the split-K `gemm_tn`
    (2T launches); at 2 bytes, which `gemm_tn`'s 8-byte addend loads cannot take, it is cuBLAS
    (T launches).  Every gradient is within the bound of fp64, the per-step layer the low arm."""
    import tests.test_gpu_lm1b_numerics as N
    S, P, E, T = 1024, 256, 256, 8
    _require_persistent(S, P)
    monkeypatch.setattr(N, "E_", E)
    inp = _bench_layer_inputs(T, E, seed=offset, S=S, P=P)
    low, _, _ = _layer(inp, False, False, monkeypatch)
    gH = inp["gH"]
    buf = torch.empty(gH.numel() + 8, dtype=BF, device="cuda")
    inp["gH"] = buf[offset:offset + gH.numel()].view_as(gH).copy_(gH)
    assert inp["gH"].data_ptr() % 16 == 2 * offset
    got, nf, nb = _layer(inp, True, True, monkeypatch)
    assert (nf, nb) == (1, 2 * T if offset == 4 else T), (nf, nb)
    ref = _run_layer("reference", inp, torch.float64)
    _assert_layer("mixed S%d P%d dH+%dB" % (S, P, 2 * offset), got, low, ref)


# ------------------------------------------------------------------------- the gate's boundary
def test_grid_queries_follow_the_documented_rule():
    """Both grid queries over B {64, 128, 256} × S {64, 128, 200, 256, 2048, first S beyond
    residency} × P {32, 64, 96, 448, 512, 576} equal the documented rule (`_expected_grid`).  Its
    residency cap is one CTA per SM (DESIGN.md §5: 512 threads at 84 and 95 registers); if ptxas
    ever lets two CTAs share an SM, the cap and this expectation change together."""
    L = _lib()
    wrong = []
    for q in _QUERIES:
        for B in (64, 128, 256):
            for S in (64, 128, 200, 256, 2048, _first_refused_S()):
                for P in (32, 64, 96, 448, 512, 576):
                    got, want = getattr(L, q)(B, S, P), _expected_grid(B, S, P)
                    if got != want:
                        wrong.append((q, B, S, P, got, want))
    assert not wrong, wrong


_QUERY_SCRIPT = """
import sys
sys.path.insert(0, sys.argv[1])
from parallax_b200 import ops
from parallax_b200.ops import fused  # noqa: F401
L = ops.lib()
S = int(sys.argv[2])
for P in map(int, sys.argv[3:]):
    print(L.px_lstm_fwd_persistent_grid(128, S, P), L.px_lstm_bwd_persistent_grid(128, S, P))
"""


def test_narrow_query_does_not_lower_the_wide_answer():
    """In a fresh process, querying P 64 first leaves the answer for P 512 what it is when P 512
    is the only query (the residency check sizes the shared-memory limit for the widest P)."""
    S = 128 * min(16, 16 * _sms() // 128)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = {k: v for k, v in os.environ.items() if not k.startswith("PARALLAX_")}

    def answers(*ps):
        r = subprocess.run([sys.executable, "-c", _QUERY_SCRIPT, root, str(S)] +
                           [str(p) for p in ps], env=env, cwd=root, capture_output=True,
                           text=True, timeout=300)
        assert r.returncode == 0, r.stderr[-2000:]
        return [tuple(map(int, line.split())) for line in r.stdout.split("\n") if line.strip()]
    narrow_first = answers(64, 512)
    alone = answers(512)
    assert narrow_first == [(S // 16, S // 16)] * 2, narrow_first
    assert alone == narrow_first[1:], (alone, narrow_first)


def test_python_gate_refuses_transposed_wh_and_offset_wp():
    """`_fwd_persistent_ok` / `_bwd_persistent_ok` take contiguous, 16-byte-aligned weights and
    refuse a transposed Wh and a W_P view 2 bytes past an aligned base."""
    from parallax_b200.ops import fused
    S, P = 1024, 256
    _require_persistent(S, P)
    Wh = torch.empty(P, 4 * S, dtype=BF, device="cuda")
    WP = torch.empty(S, P, dtype=BF, device="cuda")
    Wh_t = torch.empty(4 * S, P, dtype=BF, device="cuda").t()
    WP_2 = torch.empty(S * P + 8, dtype=BF, device="cuda")[1:1 + S * P].view(S, P)
    for ok in (fused._fwd_persistent_ok, fused._bwd_persistent_ok):
        assert ok(BF, 128, S, P, Wh, WP), ok
        assert not ok(BF, 128, S, P, Wh_t, WP), ok
        assert not ok(BF, 128, S, P, Wh, WP_2), ok


@pytest.mark.parametrize("S,P", [(None, 256), (256, 96), (256, 576)],
                         ids=["S-first-beyond-residency-P256", "S256-P96", "S256-P576"])
def test_refused_layer_runs_per_step(monkeypatch, S, P):
    """Layers the queries refuse, the first S beyond residency (2176 on a 132-SM H100) and P 96
    and 576, run the per-step kernels both ways (launch counts) and match fp64, with the PyTorch
    bf16 layer as the low arm."""
    import tests.test_gpu_lm1b_numerics as N
    from parallax_b200.ops import fused
    S = S or _first_refused_S()
    T, E = 4, 128
    for q in _QUERIES:
        assert getattr(_lib(), q)(128, S, P) == 0, (q, S, P)
    monkeypatch.setattr(N, "E_", E)
    inp = _bench_layer_inputs(T, E, seed=S + P, S=S, P=P)
    W, WP = inp["W"], inp["WP"]
    assert not fused._fwd_persistent_ok(BF, 128, S, P, W[E:], WP)
    assert not fused._bwd_persistent_ok(BF, 128, S, P, W[E:], WP)
    got, nf, nb = _layer(inp, True, True, monkeypatch)
    assert (nf, nb) == (T, _per_step_bwd_launches(T, S, P)), (nf, nb)
    ref = _run_layer("reference", inp, torch.float64)
    low = _run_layer("reference", inp, BF)
    _assert_layer("refused S%d P%d" % (S, P), got, low, ref)


# ------------------------------------------------------------------------ graphs, second device
def test_fwd_graph_replay_at_a_small_grid():
    """The forward kernel's graph replays at S 256, P 128 (16 CTAs, 4 in phase B) equal eager
    launches bit for bit."""
    _require_persistent(256, 128)
    _fwd_graph_replay(256, 128)


def test_bwd_graph_replay_at_a_small_grid():
    """The backward kernel's graph replays at S 256, P 128 (16 CTAs, 4 in phase 2) equal eager
    launches bit for bit."""
    _require_persistent(256, 128)
    _bwd_graph_replay(256, 128)


@pytest.mark.multigpu
def test_second_device_gives_the_same_bits():
    """One forward and one backward launch at S 1024, P 256 on cuda:1 (its own residency query and
    shared-memory attribute) give the bits cuda:0 gives on the same inputs."""
    S, P, T = 1024, 256, 5
    with torch.cuda.device(0):
        _require_persistent(S, P)
        fwd_in = _chain_inputs(T, S=S, P=P, seed=11)
        bwd_in = _bwd_inputs(T, S=S, P=P, seed=12)
        first = list(_run_kernel(fwd_in)) + list(_bwd_run_kernel(bwd_in))
    on1 = lambda d: {k: None if v is None else v.to("cuda:1") for k, v in d.items()}
    with torch.cuda.device(1):
        _require_persistent(S, P)
        second = list(_run_kernel(on1(fwd_in))) + list(_bwd_run_kernel(on1(bwd_in)))
    names = ("act", "c_all", "m_all", "h_all", "dgates", "dh_tot", "dh_rec", "dc")
    for name, a_, b_ in zip(names, first, second):
        assert a_.device.index == 0 and b_.device.index == 1, name
        assert torch.equal(_bits(a_.cpu()), _bits(b_.cpu())), name
