"""LM1B text generation: restore the latest checkpoint written by
`lm1b_distributed_driver.py --ckpt_dir …` (as `lm1b_eval.py` does, `--use_ema` included), prime
the LSTM with a prefix and draw one word at a time from the full softmax at a temperature
(`parallax.nn.full_softmax_sample`, fused on the rows' owners for bf16 tables on the NVLink
fabric), optionally truncated to the `--top_k` most likely words and the `--top_p` nucleus.
Each step feeds the previous words [B, 1] and the previous LSTM state, with no target, so the
softmax table is read once per word (ten times when truncated).  The same `--seed` gives the same
text.

    python examples/lm1b/lm1b_generate.py --ckpt_dir /tmp/lm1b_ckpt --datadir … \\
        --prefix "The meeting" --num_words 30 --temperature 0.8 --top_p 0.9 --num_sequences 4 \\
        --compute_dtype bf16
    python examples/lm1b/lm1b_generate.py --ckpt_dir … --use_synthetic --tiny --prefix "5 17"
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
import numpy as np

import parallax_b200 as parallax
from parallax_b200 import optim
from parallax_b200.checkpoint import latest_checkpoint
from parallax_b200.models.lm1b import LM1B, lm1b_graph, parse_hpconfig
from parallax_b200.models.lm1b_data import Vocabulary

ap = argparse.ArgumentParser()
ap.add_argument("--ckpt_dir", required=True)
ap.add_argument("--datadir", default=None, help="holds 1b_word_vocab.txt")
ap.add_argument("--use_synthetic", action="store_true",
                help="no vocabulary: the prefix and the output are word ids")
ap.add_argument("--use_ema", action="store_true")
ap.add_argument("--vocab_size", type=int, default=793470)
ap.add_argument("--tiny", action="store_true")
ap.add_argument("--hpconfig", default="",
                help="model hyper-parameters as lm1b_distributed_driver.py takes them: "
                     "name=value,... (emb_size, state_size, projected_size, num_sampled, "
                     "keep_prob); give the values the checkpoint was trained with")
ap.add_argument("--prefix", default="",
                help="words the sequences start with (ids with --use_synthetic or --tiny); "
                     "the sentence start <S> (id 0 without a vocabulary) is put in front")
ap.add_argument("--num_words", type=int, default=20, help="words to generate at most")
ap.add_argument("--num_sequences", type=int, default=4, help="sequences generated together")
ap.add_argument("--temperature", type=float, default=1.0)
ap.add_argument("--top_k", type=int, default=None,
                help="sample only among the K most likely words (and words tied with the K-th)")
ap.add_argument("--top_p", type=float, default=None,
                help="sample only from the smallest set of most likely words of mass >= P")
ap.add_argument("--seed", type=int, default=0)
ap.add_argument("--compute_dtype", default=None,
                help="bf16: bf16 LSTM outputs, which the fused sampler takes on the NVLink fabric")
FLAGS = ap.parse_args()


def step_seed(seed, step):
    """the sampling seed of generation step `step`: a 32-bit hash of (--seed, step)"""
    return optim.sr_mix(optim.sr_mix(seed & 0xffffffff) ^ step)


def main():
    model_kw = parse_hpconfig(FLAGS.hpconfig, FLAGS)
    kw = dict(vocab_size=FLAGS.vocab_size, lazy=True, eval_sample=1,
              sample_temperature=FLAGS.temperature, sample_top_k=FLAGS.top_k,
              sample_top_p=FLAGS.top_p)
    if FLAGS.tiny:
        kw.update(vocab_size=min(FLAGS.vocab_size, 10000), emb_size=32, state_size=64,
                  projected_size=32, num_sampled=64, lazy=False)
    kw.update(model_kw)
    model = LM1B(**kw)
    B = FLAGS.num_sequences
    cfg = parallax.Config(ckpt_config=parallax.CheckPointConfig(ckpt_dir=FLAGS.ckpt_dir),
                          sess_config={"compute_dtype": FLAGS.compute_dtype}
                          if FLAGS.compute_dtype else None)
    path = latest_checkpoint(FLAGS.ckpt_dir)
    assert path is not None, "no checkpoint under %s" % FLAGS.ckpt_dir
    sess, *_ = parallax.parallel_run(lm1b_graph(model, B), "localhost", parallax_config=cfg)
    eng = sess.engine
    if FLAGS.use_ema and eng.dense is not None:
        d = eng.dense.state_dict()
        d["master"].update(d["ema"])
        eng.dense.load_state_dict(d)
    eng.model.eval()                       # full softmax, no dropout

    vocab = None
    if not (FLAGS.use_synthetic or FLAGS.tiny or not FLAGS.datadir):
        vocab = Vocabulary.from_file(os.path.join(FLAGS.datadir, "1b_word_vocab.txt"))
    if vocab is not None:
        start = vocab.s_id
        prefix = [vocab.get_id(w) for w in FLAGS.prefix.split()]
        eos = vocab.get_id("</S>")
        eos = vocab.s_id if eos == vocab.unk_id else eos   # this vocabulary ends sentences with <S>
        word = vocab.get_token
    else:
        start, eos, word = 0, None, str
        prefix = [int(w) for w in FLAGS.prefix.split()]
        assert all(0 <= i < model.vocab_size for i in prefix), "prefix ids out of range"
    x = np.array([[start] + prefix] * B, dtype=np.int64)
    c = np.zeros((B, model.state_size), np.float32)
    h = np.zeros((B, model.projected_size), np.float32)
    fetches = ["sample_ids", "final_state_c", "final_state_h"]
    out = [[] for _ in range(B)]
    done = np.zeros(B, dtype=bool)
    for step in range(FLAGS.num_words):
        ids, c, h = (v[0] for v in sess.run(fetches, {
            "x": [x], "initial_state_c": [c], "initial_state_h": [h],
            "sample_seed": [step_seed(FLAGS.seed, step)]}))
        nxt = np.asarray(ids)[:, -1, 0]
        for b in range(B):
            if not done[b]:
                if eos is not None and nxt[b] == eos:
                    done[b] = True
                else:
                    out[b].append(int(nxt[b]))
        if done.all():
            break
        x = nxt[:, None].astype(np.int64)
    parallax.log.info("checkpoint %s (global_step %d), temperature %g, top_k %s, top_p %s, "
                      "seed %d", path, eng.global_step, FLAGS.temperature, FLAGS.top_k,
                      FLAGS.top_p, FLAGS.seed)
    for b in range(B):
        print(" ".join(word(i) for i in prefix + out[b]))
    sess.close()


if __name__ == "__main__":
    main()
