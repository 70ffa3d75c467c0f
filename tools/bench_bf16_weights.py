"""fp32 against bf16 master rows for sparse variables (sess_config["sparse_weights"]) on one GPU.

    python tools/bench_bf16_weights.py [--rounds 3] [--out result.json] [--small]
                                       [--skip owner,ncf,lm1b]

The two arms alternate in one process for `--rounds` rounds and the median is reported:

1. ``owner`` — the sparse owner kernel alone on a simulated group (W = 1 and 8 ranks on this
   GPU), at the shapes of `tools/bench_rowwise_adagrad.py`: 65 536 touched rows of a 50 M x 64
   table and of a 793 470 x 512 table, Adagrad and row-wise Adagrad, bf16 lookups (both arms
   read bf16 rows: the shadow or the bf16 master).  Kernel time is the device time of the
   `px_sparse_owner_kernel` launches from `torch.profiler`, summed over the W owners of a step.
2. ``ncf`` — NeuMF (bf16, CUDA graph, Adam on the embeddings) at 50 M and 100 M users: ms/step
   from CUDA events and the symmetric-heap bytes of the build; an arm that does not fit is
   reported with its error.
3. ``lm1b`` — words/s of `bench.py`'s LM1B configuration, and the loss after the timed steps.

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

ARMS = ("fp32", "bf16")
TOUCHED = 65536


def card():
    try:
        return subprocess.run(
            ["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
             "--format=csv,noheader"], capture_output=True, text=True,
            timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # pragma: no cover
        return "unknown (%s)" % e


def make_opt(kind):
    return optim.Adagrad(0.05, 0.1) if kind == "adagrad" else optim.RowWiseAdagrad(0.05, 0.1)


# ------------------------------------------------------------------- 1. owner kernel
def owner_arm(arm, kind, world, V, D, iters):
    from tests.gpu_utils import make_world
    from parallax_b200.parallel import modes
    from parallax_b200.parallel.nvlink_backend import NVSparseTable, NVSparseGroup
    opt = make_opt(kind)
    fabs = make_world(world)
    route = modes.route_for("HYBRID", True)
    cfg = parallax.Config(run_option="HYBRID")
    graph = parallax.Graph(torch.nn.Linear(1, 1), optimizer=optim.Adagrad(0.1),
                           sparse_optimizer=opt)
    weight = torch.empty(V, D, device="meta")
    o = {"sparse_early_push": False, "sparse_weights": arm}
    n = TOUCHED // world
    groups = []
    for f in fabs:
        t = NVSparseTable("t", weight, 8 * world, "mod", opt, f, route, graph, cfg,
                          init={"seed": 1, "scale": 0.05}, options=o,
                          out_dtype=torch.bfloat16, auto_group=False)
        groups.append(NVSparseGroup([t]))
    gen = torch.Generator(device="cuda").manual_seed(3)
    ids = torch.unique(torch.randint(0, V, (TOUCHED * 2,), device="cuda", generator=gen))
    ids = ids[torch.randperm(ids.numel(), device="cuda", generator=gen)[:TOUCHED]]
    grads = torch.randn(n, D, device="cuda", generator=gen).to(torch.bfloat16) * 1e-2
    for grp in groups:
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
    total_us = 0.0
    for e in prof.key_averages():
        if "px_sparse_owner_kernel" in e.key:
            total_us += getattr(e, "device_time_total", None) or e.cuda_time_total
    for f in fabs:
        f.close()
    return total_us / iters


# ------------------------------------------------------------------------ 2. NCF
def ncf_arm(arm, users, items, batch, warmup, steps):
    from parallax_b200.models.ncf import NeuMF
    torch.cuda.reset_peak_memory_stats()
    heap0 = ops.lib().px_symm_live_bytes()
    sess = None
    try:
        model = NeuMF(users, items, num_partitions=8, lazy=True)
        graph = parallax.Graph(model, optimizer=optim.Adam(1e-3),
                               sparse_optimizer=optim.Adam(1e-3), name="ncf")
        cfg = parallax.Config(run_option="HYBRID", search_partitions=False,
                              sess_config={"compute_dtype": "bf16", "cuda_graph": True,
                                           "sparse_weights": arm})
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
               "loss": float(out["loss"])}
    except (RuntimeError, torch.cuda.OutOfMemoryError) as e:
        res = {"error": str(e).splitlines()[0][:200]}
    finally:
        if sess is not None:
            sess.close()
        torch.cuda.empty_cache()
    return res


# ------------------------------------------------------------------------ 3. LM1B
def lm1b_arm(arm, warmup, steps, small):
    """bench.py's LM1B configuration (HYBRID, bf16, CUDA graph) with one change: the
    sparse_weights arm."""
    import bench
    graph, make_batch, desc, _, _, _ = bench.build_lm1b(
        argparse.Namespace(small=small, batch=None), parallax, torch)
    cfg = parallax.Config(run_option="HYBRID", search_partitions=False,
                          sess_config={"compute_dtype": "bf16", "cuda_graph": True,
                                       "sparse_weights": arm})
    sess, *_ = parallax.parallel_run(graph, "localhost:0", sync=True, parallax_config=cfg)
    eng = sess.engine
    dev = eng.comm.device
    gen = torch.Generator().manual_seed(11)
    batches = [{k: v.to(dev) for k, v in make_batch(gen).items()} for _ in range(4)]
    for i in range(warmup):
        eng.train_step(batches[i % 4])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        out = eng.train_step(batches[i % 4])
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    res = {"words_per_s": desc["items_per_step"] / (ms * 1e-3), "ms_per_step": ms,
           "loss": float(out["loss"])}
    sess.close()
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20, help="owner-kernel steps profiled")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--small", action="store_true", help="small shapes (plumbing check)")
    ap.add_argument("--skip", default="", help="comma list of owner,ncf,lm1b to skip")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_bf16_weights needs a CUDA device")
    skip = set(filter(None, args.skip.split(",")))
    big = not args.small
    result = {"card": card(), "rounds": args.rounds, "shape": "full" if big else "small"}
    print(json.dumps({"card": result["card"]}), flush=True)
    med = statistics.median
    if "owner" not in skip:
        result["owner"] = {}
        tables = {"emb_50M_d64": (50_000_000 if big else 1_000_000, 64),
                  "lm1b_793470_d512": (793_470 if big else 100_000, 512)}
        for tname, (V, D) in tables.items():
            for kind in ("adagrad", "rowwise_adagrad"):
                for world in (1, 8):
                    runs = {a: [] for a in ARMS}
                    for _ in range(args.rounds):
                        for a in ARMS:
                            runs[a].append(owner_arm(a, kind, world, V, D, args.iters))
                    key = "%s_%s_W%d" % (tname, kind, world)
                    result["owner"][key] = {a: {"owner_us_per_step_median": med(rs),
                                                "owner_us_per_step": rs}
                                            for a, rs in runs.items()}
                    print(json.dumps({key: result["owner"][key]}), flush=True)
    if "ncf" not in skip:
        result["ncf"] = {}
        batch = 65536 if big else 4096
        for users in ((50_000_000, 100_000_000) if big else (1_000_000, 2_000_000)):
            runs = {a: [] for a in ARMS}
            for _ in range(args.rounds):
                for a in ARMS:
                    runs[a].append(ncf_arm(a, users, 1_000_000 if big else 100_000, batch,
                                           args.warmup, args.steps))
            ent = {"batch": batch}
            for a, rs in runs.items():
                ok = [r for r in rs if "error" not in r]
                ent[a] = {"ms_per_step_median":
                          med(r["ms_per_step"] for r in ok) if ok else None,
                          "ms_per_step": [r.get("ms_per_step") for r in rs],
                          "heap_bytes": ok[-1]["heap_bytes"] if ok else None,
                          "loss": ok[-1]["loss"] if ok else None,
                          "error": rs[-1].get("error")}
            result["ncf"]["users_%d" % users] = ent
            print(json.dumps({"ncf_users_%d" % users: ent}), flush=True)
    if "lm1b" not in skip:
        runs = {a: [] for a in ARMS}
        for _ in range(args.rounds):
            for a in ARMS:
                runs[a].append(lm1b_arm(a, args.warmup, args.steps, not big))
        result["lm1b"] = {a: {"words_per_s_median": med(r["words_per_s"] for r in rs),
                              "words_per_s": [r["words_per_s"] for r in rs],
                              "loss": [r["loss"] for r in rs]} for a, rs in runs.items()}
        print(json.dumps({"lm1b": result["lm1b"]}), flush=True)
    print(json.dumps(result))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
