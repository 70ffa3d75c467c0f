"""Full-softmax training of the LM1B output layer on one GPU: the gather + matmul + cross_entropy
composition against the fused forward and backward (``sess_config["full_softmax_train"] =
"fused"``), and an LM1B(num_sampled=0) training step under each setting.

    python tools/bench_full_softmax_train.py [--n 640 2560] [--steps 10] [--out result.json]

Head: LM1B's (softmax_w, softmax_b) co-lookup group built through the engine on the NVLink
fabric: V = 793 470, K = 512, bf16 shadow rows, 32 partitions.  For each N the composition's
forward plus backward, the fused forward plus backward and the fused NLL (no gradient) alternate
over --rounds rounds of --iters calls (median).  The backward's table gradient rows are dropped
after each call (no step is run).  Per arm: ms per call (CUDA events, after warm-up), the growth
of `torch.cuda.max_memory_allocated` during one call, and TFLOP/s counted as 8·N·V·K for forward
plus backward (2·N·V·K for the NLL alone).  The records carry the relative Frobenius difference
of the two arms' input gradients.

Step: LM1B(num_sampled=0) at the benchmark's shapes (batch 128, 20 steps, LSTM 2048 -> 512,
bf16, CUDA graph), each setting in a process of its own: ms per step over --steps steps after
--warmup, and the peak allocation from the first step on.  The card name, power limit and max SM clock are read in the
same run.
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
from parallax_b200.models.lm1b import LM1B, lm1b_graph  # noqa: E402
from parallax_b200.parallel.engine import full_softmax_composition  # noqa: E402
from tools.bench_full_softmax import alternate, card  # noqa: E402


def head(a, info):
    torch.manual_seed(0)
    model = LM1B(lazy=True, state_size=512, num_sampled=0)
    sess, *_ = parallax.parallel_run(
        lm1b_graph(model, batch_size=128), "localhost:0",
        parallax_config=parallax.Config(sess_config={"fabric": "nvlink", "compute_dtype": "bf16",
                                                     "full_softmax_train": "fused"}))
    m = sess.engine.model
    w, b = m.softmax_w, m.softmax_b
    grp = w.table.group
    assert b.table.group is grp and w.table.use_shadow
    V, K = w.num_embeddings, w.embedding_dim
    out = []
    for n in a.n:
        gen = torch.Generator(device="cuda").manual_seed(n)
        x = (torch.randn(n, K, device="cuda", generator=gen) * 0.5).bfloat16().requires_grad_()
        t = torch.randint(0, V, (n,), device="cuda", generator=gen)
        gvec = torch.full((n,), 1.0 / n, device="cuda")

        def fwd_bwd(fn):
            def run():
                nll = fn(x, t, w, b)
                nll.backward(gvec)
                grp.calls.clear()             # drop the table gradient rows: no step is run
                grp._fwd_calls = grp._bwd_calls = 0
                dx, x.grad = x.grad, None
                return dx
            return run
        comp = fwd_bwd(full_softmax_composition)
        fused = fwd_bwd(parallax.nn.full_softmax_nll)

        def nll():
            with torch.no_grad():
                return parallax.nn.full_softmax_nll(x, t, w, b)
        dc, df = comp(), fused()                                    # warm-up + values
        nll()
        diff = float((df.float() - dc.float()).norm() / dc.float().norm())
        del dc, df
        res = alternate([("composition", comp, a.iters), ("fused", fused, a.iters),
                         ("fused_nll", nll, a.iters)], a.rounds)
        med = {}
        for arm, (ms, grow) in res.items():
            med[arm] = statistics.median(ms)
            flop = (2.0 if arm == "fused_nll" else 8.0) * n * V * K
            r = {"part": "head", "arm": arm, "N": n, "V": V, "K": K,
                 "ms": round(med[arm], 3), "ms_all": [round(v, 3) for v in ms],
                 "mem_growth_MB": round(grow / 2 ** 20, 1),
                 "tflops": round(flop / (med[arm] * 1e-3) / 1e12, 1),
                 "chunk_rows": grp.full_softmax_train_chunk(n),
                 "rel_diff_dx": round(diff, 5), "card": info}
            out.append(r)
            print(json.dumps(r), flush=True)
        r = {"part": "head", "N": n,
             "fused_over_composition": round(med["fused"] / med["composition"], 3),
             "fused_over_fused_nll": round(med["fused"] / med["fused_nll"], 3)}
        out.append(r)
        print(json.dumps(r), flush=True)
    sess.close()
    return out


def step(a, setting, info):
    torch.manual_seed(0)
    model = LM1B(lazy=True, vocab_size=793470, emb_size=512, state_size=2048,
                 projected_size=512, num_sampled=0, num_steps=20, num_shards=32)
    sess, *_ = parallax.parallel_run(
        lm1b_graph(model, batch_size=128), "localhost:0",
        parallax_config=parallax.Config(sess_config={
            "fabric": "nvlink", "compute_dtype": "bf16", "cuda_graph": True,
            "full_softmax_train": setting}))
    gen = torch.Generator().manual_seed(1)
    feeds = [{"x": torch.randint(0, 793470, (128, 20), generator=gen),
              "y": torch.randint(0, 793470, (128, 20), generator=gen)} for _ in range(4)]
    # the peak over the eager warm-up steps and the capture, where the step's buffers are
    # allocated (replays reuse the graph's pool)
    torch.cuda.reset_peak_memory_stats()
    for i in range(a.warmup):
        sess.run(["loss", "train_op"], feeds[i % 4])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(a.steps):
        loss = sess.run(["loss", "train_op"], feeds[i % 4])[0][0]
    e1.record()
    torch.cuda.synchronize()
    r = {"part": "lm1b_step", "full_softmax_train": setting, "num_sampled": 0,
         "ms_per_step": round(e0.elapsed_time(e1) / a.steps, 2),
         "peak_allocated_GB": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2),
         "loss": float(loss), "cuda_graph": bool(getattr(sess.engine, "graph_captured", False)),
         "card": info}
    print(json.dumps(r), flush=True)
    sess.close()
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="*", default=[640, 2560])
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--step_settings", nargs="*", default=["composition", "fused"])
    ap.add_argument("--step_only", default=None, help=argparse.SUPPRESS)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_full_softmax_train needs a CUDA device")
    info = card()
    if a.step_only:
        step(a, a.step_only, info)
        return
    print("card: %s" % info, flush=True)
    results = []
    # the steps first, before this process holds any device memory
    for setting in a.step_settings:
        # each setting in its own process: peak allocation and allocator state of its own
        p = subprocess.run([sys.executable, os.path.abspath(__file__), "--step_only", setting,
                            "--steps", str(a.steps), "--warmup", str(a.warmup)],
                           capture_output=True, text=True)
        lines = [ln for ln in p.stdout.splitlines() if ln.startswith("{")]
        if p.returncode != 0 or not lines:
            r = {"part": "lm1b_step", "full_softmax_train": setting,
                 "error": (p.stderr or p.stdout)[-2000:]}
        else:
            r = json.loads(lines[-1])
        results.append(r)
        print(json.dumps(r), flush=True)
    if a.n:
        results += head(a, info)
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"card": info, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
