"""Top-k next-word prediction over LM1B's output layer: the gather + matmul + log_softmax + top-k
composition against the fused top-k kernel (`parallax.nn.full_softmax_topk`), next to the fused
NLL (`parallax.nn.full_softmax_nll`) at the same N, in one process.

    python tools/bench_full_softmax_topk.py [--n 640 2560] [--k 1 10 32] [--out result.json]

Builds LM1B's (softmax_w, softmax_b) co-lookup group through the engine on the NVLink fabric,
one GPU: V = 793 470, K = 512, bf16 shadow rows, 32 partitions.  For each (N, k) the fused
top-k and the fused NLL alternate over 3 rounds (median); the composition is timed once per
round after them.  Per arm: ms per call (CUDA events, after warm-up), the growth of
`torch.cuda.max_memory_allocated` during one call, and TFLOP/s from 2·N·V·K.  The fused ids are
compared with the composition's where its consecutive log-probabilities, the (k+1)-th
included, differ by > 2e-2 (the composition's logits are rounded to bf16).  The card name,
power limit and max SM clock are read in the same run.
"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import parallax_b200 as parallax  # noqa: E402
from parallax_b200.models.lm1b import LM1B, lm1b_graph  # noqa: E402
from parallax_b200.parallel.engine import full_softmax_topk_composition  # noqa: E402
from tools.bench_full_softmax import card, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[640, 2560])
    ap.add_argument("--k", type=int, nargs="+", default=[1, 10, 32])
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--comp_iters", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_full_softmax_topk needs a CUDA device")
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
    results = []

    def report(arm, n, k, ms, grow, extra=None):
        med = statistics.median(ms)
        r = {"arm": arm, "N": n, "k": k, "V": V, "K": K, "ms": round(med, 3),
             "ms_all": [round(v, 3) for v in ms], "mem_growth_MB": round(grow / 2 ** 20, 1),
             "tflops": round(2.0 * n * V * K / (med * 1e-3) / 1e12, 1), "card": info}
        r.update(extra or {})
        results.append(r)
        print(json.dumps(r), flush=True)
        return med

    with torch.no_grad():
        for n in a.n:
            g = torch.Generator(device="cuda").manual_seed(n)
            x = (torch.randn(n, K, device="cuda", generator=g) * 0.5).bfloat16()
            t = torch.randint(0, V, (n,), device="cuda", generator=g)
            nll = lambda: parallax.nn.full_softmax_nll(x, t, w, b)       # noqa: E731
            nll()
            for k in a.k:
                topk = lambda: parallax.nn.full_softmax_topk(x, w, b, k)    # noqa: E731
                comp = lambda: full_softmax_topk_composition(x, w, b, k)     # noqa: E731
                lp, ids = topk()
                clp, cids = full_softmax_topk_composition(x, w, b, k + 1)
                d = clp[:, :-1] - clp[:, 1:]                  # [N, k]: the (k+1)-th included
                ok = d > 2e-2
                ok[:, 1:] &= d[:, :-1] > 2e-2
                agree = {"ids_checked": int(ok.sum()),
                         "ids_equal": bool(torch.equal(ids[ok], cids[:, :k][ok])),
                         "max_abs_diff_log_probs": float((lp - clp[:, :k]).abs().max())}
                del lp, ids, clp, cids, d, ok
                ms = {"fused_topk": [], "fused_nll": [], "composition": []}
                mem = {}
                for _ in range(a.rounds):
                    for arm, f in (("fused_topk", topk), ("fused_nll", nll)):   # alternate
                        t_ms, grow = timed(f, a.iters)
                        ms[arm].append(t_ms)
                        mem[arm] = grow
                    t_ms, grow = timed(comp, a.comp_iters)
                    ms["composition"].append(t_ms)
                    mem["composition"] = grow
                report("composition", n, k, ms["composition"], mem["composition"])
                tk = report("fused_topk", n, k, ms["fused_topk"], mem["fused_topk"], agree)
                nl = report("fused_nll", n, k, ms["fused_nll"], mem["fused_nll"])
                print(json.dumps({"N": n, "k": k, "topk_over_nll": round(tk / nl, 3)}),
                      flush=True)
    sess.close()
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"card": info, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
