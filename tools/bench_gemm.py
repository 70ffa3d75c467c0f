"""Time the wgmma GEMM against cuBLAS (torch.mm) on the LSTM's skinny shapes."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from parallax_b200.ops.gemm import gemm_tn, pick_splits

def timeit(fn, n=40):
    """Device time per call: n calls captured in one CUDA graph (no launch gaps),
    weights L2-resident exactly as inside the unrolled LSTM."""
    for _ in range(3): fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(n): fn()
    g.replay(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5): g.replay()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (5 * n)

shapes = [("dh_rec  dgates@Wh^T", 128, 512, 8192), ("proj    m@W_P", 128, 512, 2048),
          ("gates   h@Wh", 128, 8192, 512), ("dm      dh@W_P^T", 128, 2048, 512)]
print("%-22s %6s %6s %6s | %9s | %s" % ("shape", "M", "N", "K", "cuBLAS us", "wgmma us (splits,bn)"))
for name, M, N, K in shapes:
    A = torch.randn(M, K, device="cuda").bfloat16()
    Bt = torch.randn(N, K, device="cuda").bfloat16()
    B = Bt.t().contiguous()
    t_cublas = min(timeit(lambda: torch.mm(A, B)), timeit(lambda: torch.mm(A, Bt.t())))
    res = []
    for bn in (128, 64):
        for s in sorted({1, 2, 4, 8, 16, 32, pick_splits(M, N, K, bn)}):
            if K % (s * 64): continue
            try:
                t = timeit(lambda: gemm_tn(A, Bt, splits=s, bn=bn))
                res.append((t, s, bn))
            except Exception as e:
                res.append((float("inf"), s, bn))
    res.sort()
    print("%-22s %6d %6d %6d | %9.2f | %s" % (name, M, N, K, t_cublas,
          "  ".join("%.2f(%d,%d)" % r for r in res[:5])))
