"""Device time of the per-time-step products of the LM1B LSTM backward chain, each captured
in a CUDA graph of 40 back-to-back dependent launches (the regime of the real step):
  A  today:   dm = dh @ W_P^T (cuBLAS)  then  dh' = dH + dgates @ Wh^T (wgmma split-K 16)
  B  fused W: dm' = DMH + dgates @ (W_P Wh)^T   cuBLAS addmm
  C  fused W: same product on the wgmma split-K kernel (several tilings)
Usage: python tools/bench_lstm_gemms.py"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from parallax_b200.ops import gemm as G

B, P, S = 128, 512, 2048
dev = "cuda"
bf = torch.bfloat16
dh = torch.randn(B, P, device=dev).to(bf)
dH = torch.randn(B, P, device=dev).to(bf)
WPT = (torch.randn(P, S, device=dev) * 0.02).to(bf)
Wh = (torch.randn(P, 4 * S, device=dev) * 0.02).to(bf)
Wc = (torch.randn(S, 4 * S, device=dev) * 0.02).to(bf)
dg = torch.randn(B, 4 * S, device=dev).to(bf)
DMH = torch.randn(B, S, device=dev).to(bf)
dm = torch.empty(B, S, device=dev, dtype=bf)
out_h = torch.empty(B, P, device=dev, dtype=bf)


def timed(name, fn, iters=40, reps=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(iters):
            fn()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / (iters * reps)
    print("%-64s %7.2f us" % (name, us), flush=True)
    return us


def a_today():
    torch.mm(dh, WPT, out=dm)
    G.gemm_tn(dg, Wh, addend=dH, splits=16, bn=64, out=out_h)


timed("A  mm(128x512x2048) + tc splitK16 (128x8192x512)+addend", a_today)
timed("A1 mm(128x512x2048) cuBLAS alone", lambda: torch.mm(dh, WPT, out=dm))
timed("A2 tc splitK16 128x8192->512 alone (L2 red.add + ticket + read-back)",
      lambda: G.gemm_tn(dg, Wh, addend=dH, splits=16, bn=64, out=out_h, cluster=False))
timed("A3 tc splitK16, 16-CTA cluster DSMEM reduction",
      lambda: G.gemm_tn(dg, Wh, addend=dH, splits=16, bn=64, out=out_h, cluster=True))
timed("A4 tc splitK8, 8-CTA cluster DSMEM reduction",
      lambda: G.gemm_tn(dg, Wh, addend=dH, splits=8, bn=64, out=out_h, cluster=True))
WcT = Wc.t()
timed("B  cuBLAS addmm(DMH, dg[128x8192], Wc^T[8192x2048])",
      lambda: torch.addmm(DMH, dg, WcT, out=dm))
for bn, sp in ((64, 4), (128, 8), (64, 2), (128, 4), (64, 8), (128, 16)):
    try:
        timed("C  tc gemm_tn N=2048 K=8192 bn=%d splits=%d" % (bn, sp),
              lambda: G.gemm_tn(dg, Wc, addend=DMH, splits=sp, bn=bn, out=dm))
    except Exception as e:
        print("C bn=%d splits=%d failed: %s" % (bn, sp, e))
# forward counterparts
h = torch.randn(B, P, device=dev).to(bf)
m = torch.randn(B, S, device=dev).to(bf)
xw = torch.randn(B, 4 * S, device=dev).to(bf)
W_P = (torch.randn(S, P, device=dev) * 0.02).to(bf)
gp = torch.empty(B, 4 * S, device=dev, dtype=bf)
h2 = torch.empty(B, P, device=dev, dtype=bf)
Wf = (torch.randn(S, 4 * S, device=dev) * 0.02).to(bf)
timed("F  today fwd: addmm(xw, h[128x512], Wh) + mm(m[128x2048], W_P)",
      lambda: (torch.addmm(xw, h, Wh, out=gp), torch.mm(m, W_P, out=h2)))
timed("F' fused W fwd: addmm(xw, m[128x2048], W'[2048x8192])",
      lambda: torch.addmm(xw, m, Wf, out=gp))
# forward projection h = m @ W_P on the cluster split-K kernel (needs W_P^T, K-contiguous)
WPt = W_P.t().contiguous()
timed("F1 cuBLAS mm(m[128x2048], W_P[2048x512])", lambda: torch.mm(m, W_P, out=h2))
for sp in (2, 4, 8):
    timed("F2 tc cluster splitK%d 128x2048->512" % sp,
          lambda: G.gemm_tn(m, WPt, splits=sp, bn=64, out=h2, cluster=True))
