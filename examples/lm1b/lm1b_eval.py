"""LM1B evaluation (reference `examples/lm1b/lm1b_eval.py`): restore the latest
checkpoint written by `lm1b_distributed_driver.py --ckpt_dir …` and report test
perplexity with the FULL softmax (num_sampled = 0 at evaluation,
`language_model.py:30`).  Checkpoints hold full logical tensors keyed by the
single-device variable names, so no partition-name remapping is needed (the
reference remaps `emb/part_i` — `lm1b_eval.py:96-104`); with `--use_ema` the LSTM
variables are replaced by their exponential moving averages.

    python examples/lm1b/lm1b_eval.py --ckpt_dir /tmp/lm1b_ckpt --datadir … [--tiny]
"""
import argparse
import math
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np
import torch

import parallax_b200 as parallax
from parallax_b200.checkpoint import latest_checkpoint
from parallax_b200.models.lm1b import LM1B, lm1b_graph
from parallax_b200.models.lm1b_data import Vocabulary, Dataset

ap = argparse.ArgumentParser()
ap.add_argument("--ckpt_dir", required=True)
ap.add_argument("--datadir", default=None)
ap.add_argument("--use_synthetic", action="store_true")
ap.add_argument("--use_ema", action="store_true")
ap.add_argument("--batch_size", type=int, default=32)
ap.add_argument("--num_steps", type=int, default=20)
ap.add_argument("--vocab_size", type=int, default=793470)
ap.add_argument("--max_batches", type=int, default=100)
ap.add_argument("--tiny", action="store_true")
ap.add_argument("--top_k", type=int, default=0,
                help="also report accuracy@1 and accuracy@K of the K most likely next words "
                     "(parallax.nn.full_softmax_topk); this reads the softmax table a second "
                     "time per batch, after the perplexity's pass")
FLAGS = ap.parse_args()


def topk_hits(top, y, w):
    """(Σ w where the target is the first prediction, Σ w where it is among all k) of one
    batch: `top` [B, T, k] predicted ids, `y` [B, T] targets, `w` [B, T] weights."""
    top = torch.as_tensor(top).cpu()
    y = torch.as_tensor(np.asarray(y)).to(torch.int64)
    w = torch.as_tensor(np.asarray(w, dtype=np.float32))
    eq = top == y[..., None]
    return float((eq[..., 0].float() * w).sum()), float((eq.any(-1).float() * w).sum())


def main():
    kw = dict(vocab_size=FLAGS.vocab_size, num_steps=FLAGS.num_steps, lazy=True,
              eval_top_k=FLAGS.top_k)
    if FLAGS.tiny:
        kw.update(vocab_size=min(FLAGS.vocab_size, 10000), emb_size=32, state_size=64,
                  projected_size=32, num_sampled=64, lazy=False)
    model = LM1B(**kw)
    graph = lm1b_graph(model, FLAGS.batch_size)
    cfg = parallax.Config(ckpt_config=parallax.CheckPointConfig(ckpt_dir=FLAGS.ckpt_dir))
    path = latest_checkpoint(FLAGS.ckpt_dir)
    assert path is not None, "no checkpoint under %s" % FLAGS.ckpt_dir
    sess, *_ = parallax.parallel_run(graph, "localhost", parallax_config=cfg)   # restores on start
    eng = sess.engine
    if FLAGS.use_ema and eng.dense is not None:
        # evaluate with the EMA shadows of the LSTM variables (`lm1b_eval.py:96-104`); only
        # the dense group is touched — the sparse tables stay where they are
        d = eng.dense.state_dict()
        d["master"].update(d["ema"])
        eng.dense.load_state_dict(d)
    eng.model.eval()                       # full softmax, no dropout
    V = model.vocab_size
    if FLAGS.use_synthetic or not FLAGS.datadir:
        rng = np.random.RandomState(0)
        batches = ((rng.randint(0, V, (FLAGS.batch_size, FLAGS.num_steps)),
                    rng.randint(0, V, (FLAGS.batch_size, FLAGS.num_steps)),
                    np.ones((FLAGS.batch_size, FLAGS.num_steps), np.float32))
                   for _ in range(FLAGS.max_batches))
    else:
        vocab = Vocabulary.from_file(os.path.join(FLAGS.datadir, "1b_word_vocab.txt"))
        ds = Dataset(vocab, os.path.join(FLAGS.datadir, "heldout-monolingual.tokenized.shuffled/*"),
                     deterministic=True)
        batches = ds.iterate_once(FLAGS.batch_size, FLAGS.num_steps)
    tot, cnt, hit1, hitk = 0.0, 0.0, 0.0, 0.0
    for i, (x, y, w) in enumerate(batches):
        if i >= FLAGS.max_batches:
            break
        feeds = {"x": [x], "y": [y], "w": [w]}
        if FLAGS.top_k > 0:
            loss, top = sess.run(["loss", "top_k_ids"], feeds)
            hit1_, hitk_ = topk_hits(top[0], y, w)
            hit1 += hit1_
            hitk += hitk_
        else:
            loss = sess.run("loss", feeds)
        n = float(np.sum(w))
        tot += float(loss[0]) * x.size     # `loss` is the mean over batch×steps of loss·w
        cnt += n
    ppl = math.exp(tot / max(cnt, 1.0))
    parallax.log.info("checkpoint %s (global_step %d): perplexity = %.3f over %d words",
                      path, eng.global_step, ppl, int(cnt))
    print("perplexity %.3f" % ppl)
    if FLAGS.top_k > 0:
        print("accuracy@1 %.4f accuracy@%d %.4f" % (hit1 / max(cnt, 1.0), FLAGS.top_k,
                                                    hitk / max(cnt, 1.0)))
    sess.close()


if __name__ == "__main__":
    main()
