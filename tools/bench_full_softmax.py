"""Full-softmax evaluation of the LM1B output layer, in one process: the NLL's gather + matmul +
cross_entropy composition against the fused kernel (`parallax.nn.full_softmax_nll`), and top-k
next-word prediction's gather + matmul + log_softmax + top-k composition against the fused top-k
kernel (`parallax.nn.full_softmax_topk`), next to the fused NLL at the same N, and sampling's
gather + matmul + log_softmax + noise + top-n composition against the fused sampler
(`parallax.nn.full_softmax_sample`), next to the fused top-k at the same n and the fused NLL.

    python tools/bench_full_softmax.py [--n 640 2560] [--k 1 10 32] [--sample 1 10 32]
                                       [--trunc 1 10] [--top_k 40] [--top_p 0.9 0.95]
                                       [--temperature 1.0] [--K 512] [--out result.json]

Builds LM1B's (softmax_w, softmax_b) co-lookup group through the engine on the NVLink fabric,
one GPU: V = 793 470, K = --K (LM1B's projected_size, default 512), bf16 shadow rows, 32
partitions.  For each N:
- NLL: the composition and the fused kernel alternate over --rounds rounds of --iters calls
  (median).  The records carry the largest |Δ| between the arms' NLL (the composition rounds
  logits to bf16).  At K != 512 a second group 512 wide is built and its fused NLL
  (`fused_nll_k512`) is timed in the same rounds.
- top-k, for each k of --k (an empty list times the NLL only): the fused top-k and the fused NLL
  alternate over the rounds, and the composition is timed after them in each round over
  --comp_iters calls.  The fused ids are compared with the composition's where its consecutive
  log-probabilities, the (k+1)-th included, differ by > 2e-2.
- sampling, for each n of --sample (default none) at --temperature: the fused sampler, the fused
  top-k at k = n and the fused NLL alternate over the rounds, and the composition is timed after
  them.  The records carry the share of first draws equal to the composition's (same seed; its
  logits are rounded to bf16, so keys closer than that may swap).
- truncated sampling, for each n of --trunc (default none) and each truncation of --top_k
  (alone) and --top_p (each alone): the fused truncated sampler, the fused untruncated sampler
  at the same n and the fused NLL alternate over the rounds, and the truncated composition is
  timed after them.  The records carry the share of rows whose draws equal the composition's.
Per arm: ms per call (CUDA events, after warm-up), the growth of `torch.cuda.max_memory_allocated`
during one call, and the achieved TFLOP/s from 2·N·V·K.  The card name, power limit and max SM
clock are read in the same run.
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
from parallax_b200.parallel.engine import (full_softmax_composition,  # noqa: E402
                                           full_softmax_sample_composition,
                                           full_softmax_topk_composition)


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


def alternate(arms, rounds):
    """{name: (ms per call of each round, allocation growth)} of arms [(name, fn, iters)],
    timed in turn in every round."""
    ms, mem = {name: [] for name, _, _ in arms}, {}
    for _ in range(rounds):
        for name, fn, iters in arms:
            t_ms, mem[name] = timed(fn, iters)
            ms[name].append(t_ms)
    return {name: (ms[name], mem[name]) for name in ms}


def output_layer(K, sess_config, **model_kw):
    """(session, softmax_w, softmax_b) of an LM1B whose output layer is LM1B's with K columns,
    built through the engine on the NVLink fabric, one GPU"""
    model = LM1B(lazy=True, state_size=512, projected_size=K, **model_kw)
    sess, *_ = parallax.parallel_run(
        lm1b_graph(model, batch_size=128), "localhost:0",
        parallax_config=parallax.Config(sess_config=dict({"fabric": "nvlink",
                                                          "compute_dtype": "bf16"},
                                                         **sess_config)))
    m = sess.engine.model
    w, b = m.softmax_w, m.softmax_b
    assert w.table.group is b.table.group and w.table.use_shadow and w.embedding_dim == K
    return sess, w, b


def k512_nll(sess_config, n_list, **model_kw):
    """{N: a call of the fused NLL on a second output layer 512 wide}, timed next to a wider
    layer's arms, and its session"""
    sess, w, b = output_layer(512, sess_config, **model_kw)
    calls = {}
    for n in n_list:
        g = torch.Generator(device="cuda").manual_seed(n)
        x = (torch.randn(n, 512, device="cuda", generator=g) * 0.5).bfloat16()
        t = torch.randint(0, w.num_embeddings, (n,), device="cuda", generator=g)

        def call(x=x, t=t):
            with torch.no_grad():
                return parallax.nn.full_softmax_nll(x, t, w, b)
        call()
        calls[n] = call
    return sess, calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[640, 2560])
    ap.add_argument("--k", type=int, nargs="*", default=[1, 10, 32])
    ap.add_argument("--sample", type=int, nargs="*", default=[])
    ap.add_argument("--trunc", type=int, nargs="*", default=[])
    ap.add_argument("--top_k", type=int, default=40)
    ap.add_argument("--top_p", type=float, nargs="*", default=[0.9, 0.95])
    ap.add_argument("--temperature", type=float, default=1.0)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--comp_iters", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--K", type=int, default=512,
                    help="columns of the output layer (LM1B's projected_size)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_full_softmax needs a CUDA device")
    info = card()
    print("card: %s" % info, flush=True)
    torch.manual_seed(0)
    # the output layer is LM1B's exactly, --K wide
    sess, w, b = output_layer(a.K, {})
    V, K = w.num_embeddings, w.embedding_dim
    sess512, nll512 = k512_nll({}, a.n) if K != 512 else (None, {})
    results = []

    def report(arm, n, timing, k=None, extra=None, Kx=None):
        ms, grow = timing
        med = statistics.median(ms)
        Kx = Kx or K
        r = {"arm": arm, "N": n, **({} if k is None else {"k": k}), "V": V, "K": Kx,
             **({} if k is None or "sample" not in arm else {"temperature": a.temperature}),
             "ms": round(med, 3), "ms_all": [round(v, 3) for v in ms],
             "mem_growth_MB": round(grow / 2 ** 20, 1),
             "tflops": round(2.0 * n * V * Kx / (med * 1e-3) / 1e12, 1), **(extra or {}),
             "card": info}
        results.append(r)
        print(json.dumps(r), flush=True)
        return med

    with torch.no_grad():
        for n in a.n:
            g = torch.Generator(device="cuda").manual_seed(n)
            x = (torch.randn(n, K, device="cuda", generator=g) * 0.5).bfloat16()
            t = torch.randint(0, V, (n,), device="cuda", generator=g)
            comp = lambda: full_softmax_composition(x, t, w, b)          # noqa: E731
            nll = lambda: parallax.nn.full_softmax_nll(x, t, w, b)       # noqa: E731
            ref, fused = comp(), nll()                                   # warm-up + values
            comp(), nll()
            diff = {"max_abs_diff_nll": float((fused - ref).abs().max())}
            del ref, fused
            arms = [("composition", comp, a.iters), ("fused", nll, a.iters)]
            if nll512:
                arms.append(("fused_nll_k512", nll512[n], a.iters))
            res = alternate(arms, a.rounds)
            for arm in ("composition", "fused"):
                report(arm, n, res[arm], extra=diff)
            if nll512:
                report("fused_nll_k512", n, res["fused_nll_k512"], Kx=512)
            for k in a.k:
                topk = lambda: parallax.nn.full_softmax_topk(x, w, b, k)    # noqa: E731
                tcomp = lambda: full_softmax_topk_composition(x, w, b, k)   # noqa: E731
                lp, ids = topk()
                clp, cids = full_softmax_topk_composition(x, w, b, k + 1)
                d = clp[:, :-1] - clp[:, 1:]                  # [N, k]: the (k+1)-th included
                ok = d > 2e-2
                ok[:, 1:] &= d[:, :-1] > 2e-2
                agree = {"ids_checked": int(ok.sum()),
                         "ids_equal": bool(torch.equal(ids[ok], cids[:, :k][ok])),
                         "max_abs_diff_log_probs": float((lp - clp[:, :k]).abs().max())}
                del lp, ids, clp, cids, d, ok
                res = alternate([("fused_topk", topk, a.iters), ("fused_nll", nll, a.iters),
                                 ("composition", tcomp, a.comp_iters)], a.rounds)
                report("composition", n, res["composition"], k)
                tk = report("fused_topk", n, res["fused_topk"], k, agree)
                nl = report("fused_nll", n, res["fused_nll"], k)
                print(json.dumps({"N": n, "k": k, "topk_over_nll": round(tk / nl, 3)}),
                      flush=True)
            inv_tau = float(torch.tensor(1.0 / a.temperature, dtype=torch.float32))
            for k in a.sample:
                smp = lambda: parallax.nn.full_softmax_sample(    # noqa: E731
                    x, w, b, k, a.temperature, 12345)
                scomp = lambda: full_softmax_sample_composition(  # noqa: E731
                    x, w, b, k, inv_tau, 12345)
                topk = lambda: parallax.nn.full_softmax_topk(x, w, b, k)    # noqa: E731
                lp, ids = smp()
                clp, cids = scomp()
                agree = {"first_draw_equal": round(float((ids[:, 0] == cids[:, 0]).float()
                                                         .mean()), 4),
                         "max_abs_diff_log_probs_equal_ids": float(
                             (lp - clp).abs()[ids == cids].max())}
                del lp, ids, clp, cids
                res = alternate([("fused_sample", smp, a.iters), ("fused_topk", topk, a.iters),
                                 ("fused_nll", nll, a.iters),
                                 ("composition_sample", scomp, a.comp_iters)], a.rounds)
                report("composition_sample", n, res["composition_sample"], k)
                sm = report("fused_sample", n, res["fused_sample"], k, agree)
                tk = report("fused_topk", n, res["fused_topk"], k)
                nl = report("fused_nll", n, res["fused_nll"], k)
                print(json.dumps({"N": n, "n": k, "sample_over_topk": round(sm / tk, 3),
                                  "sample_over_nll": round(sm / nl, 3)}), flush=True)
            truncs = ([{"top_k": a.top_k}] if a.top_k else []) + [{"top_p": p} for p in a.top_p]
            for k in a.trunc:
                for tr in truncs:
                    trs = lambda: parallax.nn.full_softmax_sample(    # noqa: E731
                        x, w, b, k, a.temperature, 12345, **tr)
                    smp = lambda: parallax.nn.full_softmax_sample(    # noqa: E731
                        x, w, b, k, a.temperature, 12345)
                    tcomp = lambda: full_softmax_sample_composition(  # noqa: E731
                        x, w, b, k, inv_tau, 12345, tr.get("top_k"), tr.get("top_p"))
                    ids, cids = trs()[1], tcomp()[1]
                    agree = {**tr, "rows_equal": round(float((ids == cids).all(1).float()
                                                             .mean()), 4)}
                    del ids, cids
                    res = alternate([("fused_trunc_sample", trs, a.iters),
                                     ("fused_sample", smp, a.iters),
                                     ("fused_nll", nll, a.iters),
                                     ("composition_trunc_sample", tcomp, a.comp_iters)],
                                    a.rounds)
                    report("composition_trunc_sample", n, res["composition_trunc_sample"], k,
                           tr)
                    tt = report("fused_trunc_sample", n, res["fused_trunc_sample"], k, agree)
                    sm = report("fused_sample", n, res["fused_sample"], k)
                    nl = report("fused_nll", n, res["fused_nll"], k)
                    cm = statistics.median(res["composition_trunc_sample"][0])
                    print(json.dumps({"N": n, "n": k, **tr, "trunc_over_sample": round(tt / sm, 3),
                                      "trunc_over_nll": round(tt / nl, 3),
                                      "composition_over_trunc": round(cm / tt, 2)}), flush=True)
    sess.close()
    if sess512 is not None:
        sess512.close()
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"card": info, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
