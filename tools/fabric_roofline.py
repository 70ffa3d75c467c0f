"""Achieved fraction of the NVLink roofline for every fused compute+collective path, at the
LM1B shapes, on N real GPUs (run under torchrun).  Device-timed (CUDA events on the launching
stream, max over ranks; the push / owner kernels also stamp %globaltimer themselves).

  python -m torch.distributed.run --nproc-per-node 8 --master-addr 127.0.0.1 \
      --master-port 29541 tools/fabric_roofline.py --out gpurun_out/fabric_roofline_8.json

Roofline: bytes that must cross NVLink per GPU and direction / NVLink bandwidth, or the HBM side
(bytes / HBM bandwidth) when that is slower.
Paths: fused dense step (reduce-scatter by load + optimizer + all-gather by store; P2P and
NVLS), remote-gather lookup, push (all-to-all of bf16 rows + ids), owner (HBM-bound)."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import torch.distributed as dist

import parallax_b200 as parallax
from parallax_b200 import optim
from parallax_b200.graph import Graph
from parallax_b200.parallel import modes, nvops, multicast
from parallax_b200.parallel.fabric import Comm
from parallax_b200.parallel.nvlink_backend import NVFabric, NVSparseTable, NVSparseGroup
from parallax_b200.parallel.symmetric import CH_COMM

ap = argparse.ArgumentParser()
ap.add_argument("--out", default=None)
ap.add_argument("--iters", type=int, default=30)
args = ap.parse_args()
NVLINK, HBM = 450.0, 3350.0      # H100 SXM data sheet, GB/s: NVLink 4 per direction, HBM3
try:
    HBM = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"]
except Exception:
    pass

comm = Comm.from_env()
W, rank, dev = comm.world, comm.rank, comm.device
fab = NVFabric(comm, options={})
heap = fab.heap
res = {"world": W, "nvlink_gbs_per_dir": NVLINK, "hbm_gbs": HBM, "paths": {}}


def tmax(ms):
    t = torch.tensor([ms], device=dev)
    if W > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t)


def timed(fn, iters, stream=None):
    """`iters` back-to-back launches captured in ONE CUDA graph (an eager launch loop of
    these short kernels is bound by the ~25 us host cost of a launch, not by the GPU)."""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    comm.barrier()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, capture_error_mode="thread_local"):
        for _ in range(iters):
            fn()
    g.replay()
    torch.cuda.synchronize()
    comm.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(3):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return tmax(e0.elapsed_time(e1) / (3 * iters)) * 1e3          # us


# ------------------------------------------------------------------ dense step
n = 9_453_568                      # LM1B dense parameters: W 1024x8192, B 8192, W_P 2048x512
q = W * 8 * 32
n = (n + q - 1) // q * q
opt = optim.Adagrad(0.2, 1.0)
hp = torch.tensor(opt.hyper(1), device=dev)
sl = n // W
master = torch.randn(sl, device=dev)
acc = torch.ones(sl, device=dev)
ema = master.clone()


def dense(use_mc):
    if use_mc:
        gb = multicast.MulticastBuffer(fab, n * 2)
        pb = multicast.MulticastBuffer(fab, n * 2)
        gsrc, pdst = gb.mc_c_ptrs(), pb.mc_c_ptrs()
        gb.tensor(torch.bfloat16, n).normal_()
    else:
        gb, pb = heap.alloc(n * 2, "g"), heap.alloc(n * 2, "p")
        gsrc, pdst = gb.c_ptrs(), pb.c_ptrs()
        gb.tensor(torch.bfloat16, n).normal_()
    torch.cuda.synchronize()
    comm.barrier()
    us = timed(lambda: nvops.dense_step(heap, gsrc, pdst, master, acc, None, ema, None, hp, None,
                                        None, n, 1.0 / W, 0.999, "adagrad", 0, torch.bfloat16,
                                        CH_COMM, max_blocks=fab.dense_blocks,
                                        use_mc=use_mc), args.iters)
    torch.cuda.synchronize()
    st_ = heap.epoch[7 * 128:7 * 128 + 10].clone().view(torch.int64).tolist()
    phases = {"start_wait_us": (st_[1] - st_[0]) / 1e3, "loop_cta0_us": (st_[2] - st_[1]) / 1e3,
              "to_last_cta_fenced_us": (st_[3] - st_[2]) / 1e3,
              "end_wait_us": (st_[4] - st_[3]) / 1e3}
    # NVLink bytes per GPU and direction.  P2P: I pull my slice from W-1 peers (in) and the
    # peers pull theirs from me (out), then I store my updated slice into W-1 peers (out) and
    # receive theirs (in).  NVLS: the switch still fetches every GPU's whole gradient (out)
    # but returns only my reduced slice (in); parameters leave once (multimem.st) and arrive
    # replicated by the switch (in).
    rs = (W - 1) * sl * 2                       # bytes of one phase in the busier direction
    if use_mc:
        link_in = sl * 2 + rs
        link_out = rs + sl * 2
    else:
        link_in = rs + rs
        link_out = rs + rs
    hbm = sl * (2 + 8 + 8 + 8 + 2) + (W - 1) * sl * 2 * 2      # own slice + serving the peers
    t_link = max(link_in, link_out) / (NVLINK * 1e3)              # us
    t_hbm = hbm / (HBM * 1e3)
    return {"us": us, "phases_last_launch": phases, "n_params": n, "nvlink_bytes_in": link_in, "nvlink_bytes_out": link_out,
            "hbm_bytes": hbm, "roofline_us": max(t_link, t_hbm),
            "bound": "nvlink" if t_link > t_hbm else "hbm",
            "fraction_of_roofline": max(t_link, t_hbm) / us,
            "nvlink_gbs_achieved": max(link_in, link_out) / us / 1e3}


res["paths"]["dense_step_p2p"] = dense(False)
if W > 1 and multicast.supported(comm):
    try:
        res["paths"]["dense_step_nvls"] = dense(True)
    except Exception as e:
        res["paths"]["dense_step_nvls"] = {"error": repr(e)}

# ---------------------------------------------------------------- sparse paths
V = 793470
route = modes.route_for("HYBRID", True)
cfg = parallax.Config(run_option="HYBRID")
graph = Graph(torch.nn.Linear(1, 1), optimizer=opt)
meta = lambda d: torch.empty(V, d, device="meta")
o = {"sparse_early_push": False, "sparse_capacity": {"softmax_w": 16384, "softmax_b": 16384,
                                                      "emb": 4096}}
mk = lambda name, d: NVSparseTable(name, meta(d), 32, "mod", opt, fab, route, graph, cfg,
                                   init={"seed": 1, "scale": 0.05}, out_dtype=torch.bfloat16,
                                   options=o, auto_group=False)
groups = {"softmax(w+b)": (NVSparseGroup([mk("softmax_w", 512), mk("softmax_b", 1)]), 10752),
          "emb": (NVSparseGroup([mk("emb", 512)]), 2560)}
for name, (grp, nrows) in groups.items():
    grp.warm(nrows)
    torch.cuda.synchronize()
    comm.barrier()
    cs = torch.cuda.current_stream()
    tl = tp = to = 0.0
    dl = dp = do = 0.0
    ITERS = args.iters
    for it in range(ITERS + 3):
        ids = torch.randint(0, V, (nrows,), device=dev)
        grads = [torch.randn(nrows, t.D, device=dev).bfloat16() for t in grp.tables]
        grp.begin_step(it + 1)
        torch.cuda.synchronize()
        comm.barrier()
        e = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        e[0].record()
        outs, tok = grp.lookup(ids)
        e[1].record()
        grp.add_pending(tok, grads)
        grp.stage_push(it + 1, stream=cs)
        e[2].record()
        grp.stage_apply(it + 1, stream=cs)
        e[3].record()
        torch.cuda.synchronize()
        if it >= 3:
            d = grp.device_times()
            tl += e[0].elapsed_time(e[1])
            dp += (d["pushed"] - d["push_start"]) / 1e3
            do += (d["applied"] - d["arrived"]) / 1e3
    rowb = sum(t.Dp for t in grp.tables) * 2                       # bf16 wire / shadow bytes
    remote = (W - 1) / W
    ids_fix = torch.randint(0, V, (nrows,), device=dev)
    lk_us = timed(lambda: grp.lookup(ids_fix, record=False), 10)
    push_us, own_us = tmax(dp / ITERS), tmax(do / ITERS)
    link = nrows * rowb * remote
    res["paths"]["lookup " + name] = {
        "us": lk_us, "rows": nrows, "nvlink_bytes_in": link,
        "roofline_us": max(link / (NVLINK * 1e3), nrows * rowb / (HBM * 1e3)),
        "fraction_of_roofline": max(link / (NVLINK * 1e3), nrows * rowb / (HBM * 1e3)) / lk_us,
        "note": "10 lookups per CUDA graph; random 1 KB rows: page-walk / latency bound"}
    res["paths"]["push " + name] = {
        "us_device_timer": push_us, "rows": nrows, "nvlink_bytes_out": link + nrows * 4 * remote,
        "roofline_us": max(link / (NVLINK * 1e3), 2 * nrows * rowb / (HBM * 1e3)),
        "fraction_of_roofline": max(link / (NVLINK * 1e3), 2 * nrows * rowb / (HBM * 1e3)) / push_us}
    hbm_o = nrows * (rowb + sum(t.Dp for t in grp.tables) * (4 * 4 + 2))
    res["paths"]["owner " + name] = {
        "us_device_timer": own_us, "rows": nrows, "hbm_bytes": hbm_o,
        "roofline_us": hbm_o / (HBM * 1e3), "fraction_of_roofline": hbm_o / (HBM * 1e3) / own_us,
        "note": "random 2 KB rows in three multi-GB arrays: page-walk bound (about 1 ns per "
                "distinct page touched), not bandwidth bound"}
if rank == 0:
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(args.out), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
fab.close()
comm.shutdown()
