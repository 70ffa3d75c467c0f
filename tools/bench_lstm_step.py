"""Device time per time step of the LM1B LSTM backward recurrence, unfused against fused, each
arm captured as a CUDA graph of T dependent time steps (the regime of the real step) and
replayed alternately with the other arms:
  unfused: dm = dh·W_P^T (cuBLAS), cell kernel, dh' = dH + dgates·Wh^T (wgmma split-K 8)
  fused:   px_lstm_dm_cell_bwd (BN swept), the same split-K product
  persistent: px_lstm_bwd_persistent, all T steps in one cooperative launch
The forward chain is timed the same way, per step (xw[t] += h·Wh, cell kernel, h' = m·W_P) against
the persistent kernel that runs all T steps in one cooperative launch (px_lstm_fwd_persistent).
Usage: python tools/bench_lstm_step.py [--rounds R]"""
import argparse
import ctypes
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from parallax_b200 import ops
from parallax_b200.ops import fused, gemm as G  # noqa: F401  (register the signatures)

ap = argparse.ArgumentParser()
ap.add_argument("--rounds", type=int, default=20)
ap.add_argument("--T", type=int, default=20)
a = ap.parse_args()

B, E, S, P, T = 128, 512, 2048, 512, a.T
dev, bf = "cuda", torch.bfloat16
L = ops.lib()
_vp = ctypes.c_void_p


def p_(t):
    return _vp(t.data_ptr())


def st():
    return _vp(torch.cuda.current_stream().cuda_stream)


def check(rc, what):
    assert rc == 0, (what, rc)


gen = torch.Generator(device=dev).manual_seed(0)
rn = lambda sc, *s: torch.randn(*s, device=dev, generator=gen) * sc
Wh = rn(0.04, P, 4 * S).to(bf)
WP = rn(0.03, S, P).to(bf)
WPT = WP.t().contiguous()
xw0 = rn(1.0, T, B, 4 * S).to(bf)
xw = xw0.clone()
act = torch.empty(T, B, 4 * S, dtype=bf, device=dev)
c_all = torch.empty(T + 1, B, S, device=dev)
c_all[0] = rn(0.5, B, S)
m_all = torch.empty(T, B, S, dtype=bf, device=dev)
h_all = torch.empty(T + 1, B, P, dtype=bf, device=dev)
h_all[0] = rn(0.3, B, P).to(bf)
dm = torch.empty(B, S, dtype=bf, device=dev)
dH = rn(0.1, T, B, P).to(bf)
dh_tot = torch.empty(T, B, P, dtype=bf, device=dev)
dh_tot[T - 1] = dH[T - 1]
dgates = torch.empty(T, B, 4 * S, dtype=bf, device=dev)
dc = torch.zeros(B, S, device=dev)


def fwd_unfused():
    for t in range(T):
        g = xw[t].addmm_(h_all[t], Wh)
        check(L.px_lstm_cell_fwd(p_(g), p_(c_all[t]), p_(act[t]), p_(c_all[t + 1]),
                                 p_(m_all[t]), B, S, 1.0, 1, st()), "cell_fwd")
        torch.mm(m_all[t], WP, out=h_all[t + 1])


ws_fwd = torch.empty(S // 128, B, P, device=dev)


def fwd_persistent():
    check(L.px_lstm_fwd_persistent(p_(xw), p_(Wh), p_(WP), p_(act), p_(c_all), p_(m_all),
                                   p_(h_all), p_(ws_fwd), T, B, S, P, 1.0, st()), "fwd_persistent")


def dh_step(t):
    if t > 0:
        G.gemm_tn(dgates[t], Wh, addend=dH[t - 1], splits=8, bn=64, out=dh_tot[t - 1])


def bwd_unfused():
    for t in range(T - 1, -1, -1):
        torch.mm(dh_tot[t], WPT, out=dm)
        check(L.px_lstm_cell_bwd(p_(dm), p_(dc), p_(act[t]), p_(c_all[t]), p_(c_all[t + 1]),
                                 p_(dgates[t]), B, S, 1, st()), "cell_bwd")
        dh_step(t)


def bwd_fused(bn):
    def run():
        for t in range(T - 1, -1, -1):
            check(L.px_lstm_dm_cell_bwd(p_(dh_tot[t]), p_(WP), p_(dc), p_(act[t]), p_(c_all[t]),
                                        p_(c_all[t + 1]), p_(dgates[t]), B, S, P, bn, st()),
                  "dm_cell_bwd")
            dh_step(t)
    return run


ws_bwd = torch.empty(4 * S // 512, B, P, device=dev)
dh_rec = torch.empty(B, P, dtype=bf, device=dev)


def bwd_persistent():
    check(L.px_lstm_bwd_persistent(p_(dH), p_(act), p_(c_all), p_(Wh), p_(WP), p_(dc),
                                   p_(dgates), p_(dh_tot), p_(dh_rec), p_(ws_bwd), T, B, S, P,
                                   st()), "bwd_persistent")


def graph_of(fn):
    for _ in range(2):
        xw.copy_(xw0)
        fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g


arms = [("fwd (addmm, cell, mm)", fwd_unfused), ("fwd persistent", fwd_persistent),
        ("bwd unfused (mm, cell, gemm_tn)", bwd_unfused)]
for bn in (16, 32, 64):
    arms.append(("bwd fused  BN %2d" % bn, bwd_fused(bn)))
arms.append(("bwd persistent", bwd_persistent))
graphs = [(name, graph_of(fn)) for name, fn in arms]
times = {name: [] for name, _ in graphs}
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
for _ in range(a.rounds):
    for name, g in graphs:
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        times[name].append(e0.elapsed_time(e1) * 1e3 / T)
print("%s, %d dependent time steps per graph, %d alternating rounds; us per time step"
      % (torch.cuda.get_device_name(), T, a.rounds))
for name, _ in graphs:
    v = sorted(times[name])
    print("%-36s median %6.2f  min %6.2f  max %6.2f" % (name, statistics.median(v), v[0], v[-1]))
