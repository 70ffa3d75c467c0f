"""Launch each hand-written hot kernel a few times at its production shape so
`ncu --set full -k regex:px_` can capture them on ONE GPU:

  ncu --set full --clock-control none --import-source on -k regex:px_ -c 40 \
      -o gpurun_out/prof python tools/ncu_targets.py
"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import parallax_b200 as parallax
from parallax_b200 import optim
from parallax_b200.ops.gemm import gemm_tn
from parallax_b200.ops import fused
from parallax_b200.parallel import nvops, modes
from parallax_b200.parallel.symmetric import CH_COMM
from parallax_b200.parallel.nvlink_backend import NVSparseTable
from parallax_b200.graph import Graph
from tests.gpu_utils import make_world

torch.manual_seed(0)
dev = "cuda"
REP = 2
# ---- wgmma split-K GEMM at the LSTM backward shape ----------------------------
A = torch.randn(128, 8192, device=dev).bfloat16()
Bt = torch.randn(512, 8192, device=dev).bfloat16()
D = torch.randn(128, 512, device=dev).bfloat16()
for _ in range(REP):
    gemm_tn(A, Bt, addend=D, splits=16, bn=64)
A2 = torch.randn(128, 512, device=dev).bfloat16()
B2 = torch.randn(8192, 512, device=dev).bfloat16()
for _ in range(REP):
    gemm_tn(A2, B2, splits=1, bn=128)
# ---- fused dense step (world 1 = fused multi-tensor Adagrad + EMA), 32 MiB bucket
fabs = make_world(1)
f = fabs[0]
n = 16 << 20
gb, pb = f.heap.alloc(n * 2, "g"), f.heap.alloc(n * 2, "p")
gb.tensor(torch.bfloat16, n).normal_()
master = torch.randn(n, device=dev)
acc = torch.ones(n, device=dev)
ema = master.clone()
hp = torch.tensor(optim.Adagrad(0.2, 1.0).hyper(1), device=dev)
for _ in range(REP):
    nvops.dense_step(f.heap, gb.c_ptrs(), pb.c_ptrs(), master, acc, None, ema, None, hp,
                     None, None, n, 1.0, 0.999, "adagrad", 0, torch.bfloat16, CH_COMM)
# ---- two-shot all-reduce with a 2-rank world simulated on this GPU.  ncu serialises
# kernels, so spinning peer kernels cannot be profiled: only with --with-allreduce
# (plain run, no ncu) is this section executed.
if "--with-allreduce" not in sys.argv:
    fabs2 = []
else:
  fabs2 = make_world(2, options={"comm_blocks": 32})
n2 = 8 << 20
bufs = [ff.heap.alloc(n2 * 2, "x") for ff in fabs2]
for b in bufs:
    b.tensor(torch.bfloat16, n2).normal_()
torch.cuda.synchronize()
for _ in range(REP if fabs2 else 0):
    for r, ff in enumerate(fabs2):
        nvops.allreduce_twoshot(ff.heap, bufs[r].c_ptrs(), n2, torch.bfloat16, 0.5, CH_COMM,
                                max_blocks=32, stream=ff.comm_stream)
    torch.cuda.synchronize()
# ---- sparse path at the LM1B softmax-table shape --------------------------------
V, Dm, n_ids = 793470, 512, 10752
route = modes.route_for("HYBRID", True)
cfg = parallax.Config()
opt = optim.Adagrad(0.2, 1.0)
graph = Graph(torch.nn.Linear(1, 1), optimizer=opt)
W0 = torch.empty(V, Dm, device="meta")
t = NVSparseTable("softmax_w.weight", W0, 32, "mod", opt, f, route, graph, cfg,
                  init={"seed": 1, "scale": 0.05}, out_dtype=torch.bfloat16,
                  options={"sparse_capacity": {"softmax_w.weight": 16384},
                           "sparse_early_push": False})
t.warm(n_ids)
for step in range(1, REP + 1):
    ids = torch.randint(0, V, (n_ids,), device=dev)
    ids[:2560] = (ids[:2560] % 50)            # Zipf-like head: many duplicates
    rows, pend = t.lookup(ids)
    t.add_pending(pend, torch.randn(n_ids, Dm, device=dev).bfloat16())
    t.begin_step(step)
    t.finish_step(step)
    torch.cuda.synchronize()
# ---- LSTM cell + sampled softmax ---------------------------------------------------
T, B, E, S, P = 2, 128, 512, 2048, 512
x = torch.randn(T, B, E, device=dev).bfloat16().requires_grad_(True)
Wx = (torch.randn(E, 4 * S, device=dev) * 0.02).bfloat16().requires_grad_(True)
Wh = (torch.randn(P, 4 * S, device=dev) * 0.02).bfloat16().requires_grad_(True)
bias = torch.zeros(4 * S, device=dev).bfloat16().requires_grad_(True)
WP = (torch.randn(S, P, device=dev) * 0.02).bfloat16().requires_grad_(True)
c0 = torch.zeros(B, S, device=dev)
h0 = torch.zeros(B, P, device=dev).bfloat16()
H, cT, hT = fused.lstm_layer(x, Wx, Wh, bias, WP, c0, h0)
H.float().sum().backward()
N, Sn = 2560, 8192
inp = torch.randn(N, P, device=dev).bfloat16().requires_grad_(True)
tw = torch.randn(N, P, device=dev).bfloat16()
sw = torch.randn(Sn, P, device=dev).bfloat16()
loss = fused.sampled_softmax_loss(inp, tw, sw, torch.zeros(N, device=dev),
                                  torch.zeros(Sn, device=dev), torch.zeros(N, device=dev),
                                  torch.zeros(Sn, device=dev),
                                  torch.randint(0, V, (N,), device=dev),
                                  torch.randint(0, V, (Sn,), device=dev))
loss.sum().backward()
# ---- the loss head as one node (dot product inside the softmax kernel, one backward glue
# kernel) at the LM1B shape
w_all = torch.randn(N + Sn, P, device=dev).bfloat16().requires_grad_(True)
b_all = torch.zeros(N + Sn, 1, device=dev).bfloat16().requires_grad_(True)
head = fused.sampled_softmax_head(inp, w_all, b_all, torch.zeros(N + Sn, device=dev),
                                  torch.randint(0, V, (N,), device=dev),
                                  torch.randint(0, V, (Sn,), device=dev))
head.backward()
torch.cuda.synchronize()
print("ncu targets done")
