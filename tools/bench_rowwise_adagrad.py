"""Row-wise Adagrad against Adagrad on one GPU.

    python tools/bench_rowwise_adagrad.py [--rounds 3] [--out result.json] [--small]

Three measurements; the two arms alternate for `--rounds` rounds and the median is reported:

1. ``owner`` — the sparse owner kernel alone on a simulated group (W = 1 and 8 ranks on this
   GPU): 65 536 touched rows, pushed once per iteration by every rank's push kernel, of
   (a) a 50 M-row D = 64 fp32 table and (b) a 793 470 x 512 table with a bf16 shadow.
   Kernel time is the device time of the `px_sparse_owner_kernel` launches taken from
   `torch.profiler` (summed over the W owners of one step).  The bytes are those the rule
   moves per touched row — Adagrad reads w and s and writes w, s (16·D) and the shadow
   (2·D); row-wise reads and writes w (8·D) and 4 B of s each way (8) and writes the shadow
   (2·D) — the ring rows are not counted.
2. ``ncf`` — NeuMF at 50 M users (bf16, CUDA graph), Adagrad against row-wise Adagrad on the
   embeddings (the dense layers use Adagrad in both arms): ms/step from CUDA events, and the
   symmetric-heap bytes the build allocated.
3. ``ncf_100m`` — one build and 20 steps of NeuMF at 100 M users with row-wise Adagrad on
   one GPU: ms/step, heap bytes and the peak device memory.

The card name, power limit and max SM clock are read in the same run and printed with the
numbers.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import parallax_b200 as parallax  # noqa: E402
from parallax_b200 import ops, optim  # noqa: E402

ARMS = ("adagrad", "rowwise_adagrad")
TOUCHED = 65536


def card():
    try:
        return subprocess.run(
            ["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
             "--format=csv,noheader"], capture_output=True, text=True,
            timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # pragma: no cover
        return "unknown (%s)" % e


def make_opt(arm):
    return optim.Adagrad(0.05, 0.1) if arm == "adagrad" else optim.RowWiseAdagrad(0.05, 0.1)


def rule_bytes(arm, D, shadow):
    """Bytes the rule moves per touched row (see the module docstring)."""
    sh = 2 * D if shadow else 0
    return (16 * D if arm == "adagrad" else 8 * D + 8) + sh


# ------------------------------------------------------------------- 1. owner kernel
def owner_arm(arm, world, V, D, bf16, iters):
    from tests.gpu_utils import make_world
    from parallax_b200.parallel import modes
    from parallax_b200.parallel.nvlink_backend import NVSparseTable, NVSparseGroup
    opt = make_opt(arm)
    fabs = make_world(world)
    route = modes.route_for("HYBRID", True)
    cfg = parallax.Config(run_option="HYBRID")
    graph = parallax.Graph(torch.nn.Linear(1, 1), optimizer=optim.Adagrad(0.1),
                           sparse_optimizer=opt)
    weight = torch.empty(V, D, device="meta")
    o = {"sparse_early_push": False}
    n = TOUCHED // world
    groups = []
    for f in fabs:
        t = NVSparseTable("t", weight, 8 * world, "mod", opt, f, route, graph, cfg,
                          init={"seed": 1, "scale": 0.05}, options=o,
                          out_dtype=torch.bfloat16 if bf16 else torch.float32,
                          auto_group=False)
        groups.append(NVSparseGroup([t]))
    gen = torch.Generator(device="cuda").manual_seed(3)
    ids = torch.unique(torch.randint(0, V, (TOUCHED * 2,), device="cuda", generator=gen))
    ids = ids[torch.randperm(ids.numel(), device="cuda", generator=gen)[:TOUCHED]]
    gdt = torch.bfloat16 if bf16 else torch.float32
    grads = torch.randn(n, D, device="cuda", generator=gen).to(gdt) * 1e-2
    for grp in groups:               # every rank's rings exist before any rank's pointers
        grp._ensure_capacity(n)
    for grp in groups:
        grp.warm(n)
    torch.cuda.synchronize()

    def step(s):
        for r, grp in enumerate(groups):
            _, pend = grp.lookup(ids[r * n:(r + 1) * n])
            grp.add_pending(pend, [grads])
            grp.begin_step(s)
        torch.cuda.synchronize()
        for grp in groups:
            grp.stage_push(s)
        torch.cuda.synchronize()
        for grp in groups:
            grp.stage_apply(s)
        torch.cuda.synchronize()

    for s in range(1, 4):
        step(s)
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for s in range(4, 4 + iters):
            step(s)
    total_us, launches = 0.0, 0
    for e in prof.key_averages():
        if "px_sparse_owner_kernel" in e.key:
            total_us += getattr(e, "device_time_total", None) or e.cuda_time_total
            launches += e.count
    for f in fabs:
        f.close()
    per_step_us = total_us / iters
    nbytes = TOUCHED * rule_bytes(arm, D, bf16)
    return {"owner_us_per_step": per_step_us, "launches": launches,
            "rule_bytes": nbytes, "rule_GBps": nbytes / (per_step_us * 1e-6) / 1e9}


# ------------------------------------------------------------------------ 2/3. NCF
def ncf_arm(arm, users, items, batch, warmup, steps):
    from parallax_b200.models.ncf import NeuMF
    torch.cuda.reset_peak_memory_stats()
    heap0 = ops.lib().px_symm_live_bytes()
    model = NeuMF(users, items, num_partitions=8, lazy=True)
    graph = parallax.Graph(model, optimizer=optim.Adagrad(0.05, 0.1),
                           sparse_optimizer=make_opt(arm), name="ncf")
    cfg = parallax.Config(run_option="HYBRID", search_partitions=False,
                          sess_config={"compute_dtype": "bf16", "cuda_graph": True})
    sess, *_ = parallax.parallel_run(graph, "localhost:0", sync=True, parallax_config=cfg)
    eng = sess.engine
    heap = ops.lib().px_symm_live_bytes() - heap0
    dev = eng.comm.device
    gen = torch.Generator().manual_seed(5)
    batches = [{"users": torch.randint(0, users, (batch,), generator=gen).to(dev),
                "items": torch.randint(0, items, (batch,), generator=gen).to(dev),
                "labels": torch.randint(0, 2, (batch,), generator=gen).to(dev)}
               for _ in range(4)]
    for i in range(warmup):
        eng.train_step(batches[i % 4])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        out = eng.train_step(batches[i % 4])
    e1.record()
    torch.cuda.synchronize()
    res = {"ms_per_step": e0.elapsed_time(e1) / steps, "heap_bytes": heap,
           "peak_allocated_bytes": torch.cuda.max_memory_allocated(),
           "loss": float(out["loss"]),
           "graph_captured": bool(getattr(eng, "graph_captured", False))}
    sess.close()
    torch.cuda.empty_cache()
    return res


def median_of(rs, key):
    return statistics.median(r[key] for r in rs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20, help="owner-kernel steps profiled")
    ap.add_argument("--steps", type=int, default=50, help="timed NCF steps per round")
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--small", action="store_true", help="small tables (plumbing check)")
    ap.add_argument("--skip", default="", help="comma list of owner,ncf,ncf_100m to skip")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_rowwise_adagrad needs a CUDA device")
    skip = set(filter(None, args.skip.split(",")))
    big = not args.small
    result = {"card": card(), "rounds": args.rounds, "shape": "full" if big else "small"}
    if "owner" not in skip:
        tables = {"emb_50M_d64_fp32": (50_000_000 if big else 1_000_000, 64, False),
                  "lm1b_793470_d512_bf16": (793_470 if big else 100_000, 512, True)}
        result["owner"] = {}
        for tname, (V, D, bf16) in tables.items():
            for world in (1, 8):
                runs = {a: [] for a in ARMS}
                for _ in range(args.rounds):
                    for a in ARMS:
                        runs[a].append(owner_arm(a, world, V, D, bf16, args.iters))
                key = "%s_W%d" % (tname, world)
                result["owner"][key] = {
                    a: {"owner_us_per_step_median": median_of(rs, "owner_us_per_step"),
                        "owner_us_per_step": [r["owner_us_per_step"] for r in rs],
                        "rule_GBps_median": median_of(rs, "rule_GBps"),
                        "rule_bytes": rs[0]["rule_bytes"]} for a, rs in runs.items()}
                print(json.dumps({key: result["owner"][key]}), flush=True)
    users, items = (50_000_000, 1_000_000) if big else (1_000_000, 100_000)
    batch = 65536 if big else 4096
    if "ncf" not in skip:
        runs = {a: [] for a in ARMS}
        for _ in range(args.rounds):
            for a in ARMS:
                runs[a].append(ncf_arm(a, users, items, batch, args.warmup, args.steps))
        result["ncf"] = {"users": users, "batch": batch}
        for a, rs in runs.items():
            result["ncf"][a] = {"ms_per_step_median": median_of(rs, "ms_per_step"),
                                "ms_per_step": [r["ms_per_step"] for r in rs],
                                "heap_bytes": rs[-1]["heap_bytes"],
                                "peak_allocated_bytes": rs[-1]["peak_allocated_bytes"],
                                "graph_captured": rs[-1]["graph_captured"]}
        print(json.dumps({"ncf": result["ncf"]}), flush=True)
    if "ncf_100m" not in skip:
        r = ncf_arm("rowwise_adagrad", 100_000_000 if big else 2_000_000, items, batch, 5, 20)
        result["ncf_100m"] = dict(r, users=100_000_000 if big else 2_000_000, batch=batch)
        print(json.dumps({"ncf_100m": result["ncf_100m"]}), flush=True)
    print(json.dumps(result))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
