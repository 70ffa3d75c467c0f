"""Cost of clipping LM1B's embeddings jointly with its LSTM variables, one GPU.

    python tools/bench_joint_clip.py [--steps 100] [--rounds 3] [--out result.json]

Two arms on the bench LM1B shape (`bench.py`'s model: V = 793 470, bf16, CUDA graph):

* ``shipped`` — `lm1b_graph` as it is: the clip rule covers ``W, B, W_P`` only;
* ``joint``   — the same graph with ONE ``ClipByGlobalNorm(include_sparse=True)`` over
  ``W, B, W_P, emb.weight, softmax_w.weight, softmax_b.weight``.  The owner kernels of
  the embedding groups then wait for the norm, i.e. for the whole backward pass, and the
  next step's lookups wait for them.

The arms alternate for `--rounds` rounds; each round builds the session, runs the warm-up
steps and times `--steps` steps with CUDA events.  Reported: the median ms/step per arm and
the last step's pre-clip norm of the clip rule (`TrainEngine.grad_norm(0)`), with the card
name, power limit and max SM clock read in the same run.
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
from parallax_b200.graph import ClipByGlobalNorm  # noqa: E402
from parallax_b200.models.lm1b import LM1B, lm1b_graph  # noqa: E402

JOINT = ["W", "B", "W_P", "emb.weight", "softmax_w.weight", "softmax_b.weight"]


def card():
    try:
        return subprocess.run(
            ["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
             "--format=csv,noheader"], capture_output=True, text=True,
            timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # pragma: no cover
        return "unknown (%s)" % e


def build(arm, small, batch):
    kw = dict(vocab_size=50000, emb_size=128, state_size=512, projected_size=128,
              num_sampled=1024, num_steps=8, num_shards=8) if small else \
        dict(vocab_size=793470, emb_size=512, state_size=2048, projected_size=512,
             num_sampled=8192, num_steps=20, num_shards=32)
    model = LM1B(lazy=True, **kw)
    graph = lm1b_graph(model, batch_size=batch)
    if arm == "joint":
        clip = graph.clip_rules()[0]
        graph.grad_rules = [r for r in graph.grad_rules if r is not clip] + \
            [ClipByGlobalNorm(clip.max_norm, params=JOINT, include_sparse=True)]
    cfg = parallax.Config(run_option="HYBRID", search_partitions=False,
                          sess_config={"compute_dtype": "bf16", "cuda_graph": True})
    sess, *_ = parallax.parallel_run(graph, "localhost:0", sync=True, parallax_config=cfg)
    return sess, kw["vocab_size"], kw["num_steps"]


def run_arm(arm, args):
    sess, V, T = build(arm, args.small, args.batch)
    eng = sess.engine
    dev = eng.comm.device
    gen = torch.Generator().manual_seed(99)
    batches = [{"x": torch.randint(0, V, (args.batch, T), generator=gen).to(dev),
                "y": torch.randint(0, V, (args.batch, T), generator=gen).to(dev)}
               for _ in range(4)]
    for i in range(args.warmup):
        eng.train_step(batches[i % 4])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(args.steps):
        out = eng.train_step(batches[i % 4])
    e1.record()
    torch.cuda.synchronize()
    res = {"ms_per_step": e0.elapsed_time(e1) / args.steps, "grad_norm": eng.grad_norm(0),
           "loss": float(out["loss"]), "graph_captured": bool(getattr(eng, "graph_captured",
                                                                        False))}
    sess.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--small", action="store_true", help="a small LM1B (plumbing check)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_joint_clip needs a CUDA device")
    runs = {"shipped": [], "joint": []}
    for _ in range(args.rounds):
        for arm in ("shipped", "joint"):
            runs[arm].append(run_arm(arm, args))
    result = {"card": card(), "steps": args.steps, "rounds": args.rounds,
              "shape": "small" if args.small else "bench", "batch": args.batch}
    for arm, rs in runs.items():
        result[arm] = {"ms_per_step_median": statistics.median(r["ms_per_step"] for r in rs),
                       "ms_per_step": [r["ms_per_step"] for r in rs],
                       "grad_norm_last": rs[-1]["grad_norm"], "loss_last": rs[-1]["loss"],
                       "graph_captured": rs[-1]["graph_captured"]}
    result["joint_over_shipped"] = result["joint"]["ms_per_step_median"] / \
        result["shipped"]["ms_per_step_median"]
    print(json.dumps(result))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
