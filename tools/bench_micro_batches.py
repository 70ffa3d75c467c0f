"""Gradient accumulation (sess_config["micro_batches"]) on one GPU.

    python tools/bench_micro_batches.py [--rounds 3] [--steps 30] [--out result.json]
                                        [--skip kernel,lm1b,bert] [--parent DIR]

Arms alternate within each round and the median over `--rounds` rounds is reported:

1. ``kernel`` — the fused dense step on a 32 MiB bf16 bucket at W = 1 (Adagrad): MODE 0
   (reduce + update + parameter store), MODE 3 (reduce into the fp32 accumulator), MODE 3
   with the accumulator in, and MODE 0 with the accumulator in (a step's last micro-batch).
   Time from CUDA events over 50 launches; GB/s from the bytes each mode must move
   (`kernel_bytes`).
2. ``lm1b`` / ``bert`` — `bench.py`'s configurations: K = 1 at batch b, K = 4 at batch 4b and
   K = 1 at batch 4b: ms/step, items/s and `torch.cuda.max_memory_allocated`.  Each arm runs
   in a process of its own; an arm that does not fit is reported with its error.
3. ``--parent DIR``: `bench.py` (LM1B, K = 1) of another built checkout against this one,
   alternating, to show that K = 1 is unchanged.

The card name and power limit are read in the same run and printed with the numbers.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        return subprocess.run(
            ["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
             "--format=csv,noheader"], capture_output=True, text=True,
            timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # pragma: no cover
        return "unknown (%s)" % e


def kernel_bytes(mode, acc_in, n):
    """Bytes a W = 1 Adagrad step on n bf16 elements moves: the gradient read, then
    MODE 0: master and accumulator slot read + written (fp32), parameters stored (bf16);
    MODE 3: the fp32 accumulator written (and read with the accumulator in)."""
    b = 2 * n
    if mode == 0:
        b += 16 * n + 2 * n
    else:
        b += 4 * n
    if acc_in:
        b += 4 * n
    return b


def bench_kernel(rounds, iters=50):
    import torch
    from tests.gpu_utils import make_world
    from parallax_b200 import optim
    from parallax_b200.parallel import nvops
    from parallax_b200.parallel.symmetric import CH_COMM
    n = 16 << 20                                       # 32 MiB of bf16
    fab = make_world(1)[0]
    gb, pb = fab.heap.alloc(n * 2, "g"), fab.heap.alloc(n * 2, "p")
    gb.tensor(torch.bfloat16, n).normal_()
    pb.tensor(torch.bfloat16, n).normal_()
    master = pb.tensor(torch.bfloat16, n).float()
    slot = torch.full((n,), 0.1, device="cuda")
    red = torch.zeros(n, device="cuda")
    opt = optim.Adagrad(1e-6, 0.1)
    hp = torch.tensor(opt.hyper(1), device="cuda")
    arms = {"mode0": (0, False), "mode3": (3, False), "mode3_acc": (3, True),
            "mode0_acc": (0, True)}

    def launch(mode, acc_in):
        nvops.dense_step(fab.heap, gb.c_ptrs(), pb.c_ptrs(), master, slot, None, None,
                         red, hp, None, None, n, 1.0, 0.0, "adagrad", mode, torch.bfloat16,
                         CH_COMM, max_blocks=fab.dense_blocks, stream=fab.comm_stream,
                         acc_in=acc_in)
    for mode, acc in arms.values():
        launch(mode, acc)
    times = {k: [] for k in arms}
    for _ in range(rounds):
        for name, (mode, acc) in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record(fab.comm_stream)
            for _ in range(iters):
                launch(mode, acc)
            e1.record(fab.comm_stream)
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / iters)
    out = {}
    for name, (mode, acc) in arms.items():
        ms = statistics.median(times[name])
        out[name] = {"us": ms * 1e3, "GB/s": kernel_bytes(mode, acc, n) / (ms / 1e3) / 1e9,
                     "rounds_us": [t * 1e3 for t in times[name]]}
    fab.close()
    return out


def _step_arm(model, K, batch, steps, warmup):
    """One arm in this process: ms/step, items/s and peak memory of `bench.py`'s model."""
    import torch
    import bench
    import parallax_b200 as parallax
    args = argparse.Namespace(small=False, batch=batch, model=model, dtype="bf16")
    builder = {"lm1b": bench.build_lm1b, "bert": bench.build_bert}[model]
    graph, make_batch, desc, _, unit, _ = builder(args, parallax, torch)
    sc = {"compute_dtype": "bf16", "cuda_graph": True}
    if K > 1:
        sc["micro_batches"] = K
    cfg = parallax.Config(run_option="HYBRID", search_partitions=False, sess_config=sc)
    sess, *_ = parallax.parallel_run(graph, "localhost:0", sync=True, parallax_config=cfg)
    eng = sess.engine
    gen = torch.Generator().manual_seed(99)
    batches = [{k: v.to(eng.comm.device) for k, v in make_batch(gen).items()}
               for _ in range(2)]
    for i in range(warmup):
        eng.train_step(batches[i % 2])
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        out = eng.train_step(batches[i % 2])
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    res = {"ms_per_step": ms, "items_per_s": desc["items_per_step"] / (ms / 1e3),
           "unit": unit, "max_memory_allocated_GiB": torch.cuda.max_memory_allocated() / 2 ** 30,
           "loss": float(out["loss"]), "graph": bool(getattr(eng, "graph_captured", False))}
    sess.close()
    return res


def _run_sub(argv, cwd=ROOT, timeout=900):
    r = subprocess.run([sys.executable] + argv, cwd=cwd, capture_output=True, text=True,
                       timeout=timeout)
    for line in reversed(r.stdout.strip().splitlines()):
        if line.startswith("{"):
            return json.loads(line)
    return {"error": (r.stderr or r.stdout).strip().splitlines()[-1:]}


def bench_model(model, b, rounds, steps):
    arms = [("K1_b", 1, b), ("K4_4b", 4, 4 * b), ("K1_4b", 1, 4 * b)]
    res = {name: [] for name, _, _ in arms}
    for _ in range(rounds):
        for name, K, batch in arms:
            res[name].append(_run_sub([__file__, "--_arm", model, str(K), str(batch),
                                       str(steps)]))
    out = {}
    for name, K, batch in arms:
        ok = [r for r in res[name] if "ms_per_step" in r]
        if not ok:
            out[name] = {"K": K, "batch": batch, "error": res[name][-1].get("error")}
            continue
        med = statistics.median(r["ms_per_step"] for r in ok)
        out[name] = {"K": K, "batch": batch, "ms_per_step": med,
                     "items_per_s": ok[0]["items_per_s"] * ok[0]["ms_per_step"] / med,
                     "max_memory_allocated_GiB": max(r["max_memory_allocated_GiB"] for r in ok),
                     "rounds_ms": [r["ms_per_step"] for r in ok], "loss": ok[-1]["loss"]}
    return out


def bench_parent(parent, rounds, steps):
    res = {"parent": [], "this": []}
    for _ in range(rounds):
        for name, cwd in (("parent", parent), ("this", ROOT)):
            r = _run_sub(["bench.py", "--gpus", "1", "--steps", str(steps), "--warmup", "10",
                          "--no-extras", "--no-e2e"], cwd=cwd)
            res[name].append(r.get("ms_per_step"))
    return {k: {"ms_per_step": statistics.median([x for x in v if x is not None] or [0.0]),
                "rounds_ms": v} for k, v in res.items()}


def main():
    if len(sys.argv) > 1 and sys.argv[1] == "--_arm":
        model, K, batch, steps = sys.argv[2], int(sys.argv[3]), int(sys.argv[4]), \
            int(sys.argv[5])
        try:
            print(json.dumps(_step_arm(model, K, batch, steps, warmup=6)))
        except Exception as e:
            print(json.dumps({"error": "%s: %s" % (type(e).__name__, e)}))
        return
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--skip", default="")
    ap.add_argument("--parent", default=None)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    skip = set(args.skip.split(",")) - {""}
    res = {"card": card()}
    print("card:", res["card"], flush=True)
    if "kernel" not in skip:
        res["kernel"] = bench_kernel(args.rounds)
        print(json.dumps({"kernel": res["kernel"]}), flush=True)
    for model, b in (("lm1b", 128), ("bert", 16)):
        if model not in skip:
            res[model] = bench_model(model, b, args.rounds, args.steps)
            print(json.dumps({model: res[model]}), flush=True)
    if args.parent:
        res["parent_vs_this"] = bench_parent(args.parent, args.rounds, 100)
        print(json.dumps({"parent_vs_this": res["parent_vs_this"]}), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
