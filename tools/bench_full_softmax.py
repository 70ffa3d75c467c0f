"""Full-softmax evaluation of the LM1B output layer: the gather + matmul + cross_entropy
composition against the fused kernel (`parallax.nn.full_softmax_nll`), in one process.

    python tools/bench_full_softmax.py [--n 640 2560] [--iters 10] [--out result.json]

Builds LM1B's (softmax_w, softmax_b) co-lookup group through the engine on the NVLink
fabric, one GPU: V = 793 470, K = 512, bf16 shadow rows, 32 partitions.  For each N the two
arms alternate; per arm it reports ms per call (CUDA events, after warm-up), the growth of
`torch.cuda.max_memory_allocated` during one call, the achieved TFLOP/s from 2·N·V·K, and
the largest |Δ| between the arms' NLL (the composition rounds logits to bf16).  The card
name, power limit and max SM clock are read in the same run.
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


def card():
    try:
        return subprocess.run(
            ["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
             "--format=csv,noheader"], capture_output=True, text=True,
            timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # pragma: no cover
        return "unknown (%s)" % e


def timed(fn, iters):
    """ms per call over `iters` back-to-back calls, and the allocation peak of one call."""
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = fn()
    torch.cuda.synchronize()
    growth = torch.cuda.max_memory_allocated() - base
    del out
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters, growth


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[640, 2560])
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_full_softmax needs a CUDA device")
    info = card()
    print("card: %s" % info, flush=True)
    torch.manual_seed(0)
    model = LM1B(lazy=True, state_size=512)          # the output layer is LM1B's exactly
    sess, *_ = parallax.parallel_run(
        lm1b_graph(model, batch_size=128), "localhost:0",
        parallax_config=parallax.Config(sess_config={"fabric": "nvlink",
                                                     "compute_dtype": "bf16"}))
    m = sess.engine.model
    w, b = m.softmax_w, m.softmax_b
    assert w.table.group is b.table.group and w.table.use_shadow
    V, K = w.num_embeddings, w.embedding_dim
    arms = {
        "composition": lambda x, t: full_softmax_composition(x, t, w, b),
        "fused": lambda x, t: parallax.nn.full_softmax_nll(x, t, w, b),
    }
    results = []
    with torch.no_grad():
        for n in a.n:
            g = torch.Generator(device="cuda").manual_seed(n)
            x = (torch.randn(n, K, device="cuda", generator=g) * 0.5).bfloat16()
            t = torch.randint(0, V, (n,), device="cuda", generator=g)
            outs = {k: f(x, t) for k, f in arms.items()}             # warm-up + values
            for k, f in arms.items():
                f(x, t)
            diff = float((outs["fused"] - outs["composition"]).abs().max())
            del outs
            ms = {k: [] for k in arms}
            mem = {}
            for _ in range(a.rounds):                                # arms alternate
                for k, f in arms.items():
                    t_ms, grow = timed(lambda: f(x, t), a.iters)
                    ms[k].append(t_ms)
                    mem[k] = grow
            for k in arms:
                med = statistics.median(ms[k])
                r = {"arm": k, "N": n, "V": V, "K": K, "ms": round(med, 3),
                     "ms_all": [round(v, 3) for v in ms[k]],
                     "mem_growth_MB": round(mem[k] / 2 ** 20, 1),
                     "tflops": round(2.0 * n * V * K / (med * 1e-3) / 1e12, 1),
                     "max_abs_diff_nll": diff, "card": info}
                results.append(r)
                print(json.dumps(r), flush=True)
    sess.close()
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"card": info, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
