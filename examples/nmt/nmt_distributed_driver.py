"""NMT driver (reference `examples/nmt/nmt_distributed_driver.py:76-189`,
flag set of `examples/nmt/nmt.py:40-290`): vanilla / attention / GNMT
sequence-to-sequence training with partitioned embeddings; the parallel corpus
is sharded across workers through `parallax.shard`; only worker 0 logs
statistics (`:147-163`).  Also runs file inference (`--inference_input_file`).

    # synthetic corpus, GNMT, 4 GPUs
    python examples/nmt/nmt_distributed_driver.py --synthetic \
        --hparams_path wmt16_gnmt_4_layer --hparams num_units=256,num_train_steps=200 \
        --resource_info_file localhost:0,1,2,3
    # real data
    python examples/nmt/nmt_distributed_driver.py --src vi --tgt en \
        --vocab_prefix /data/vocab --train_prefix /data/train --dev_prefix /data/tst2012 \
        --out_dir /tmp/nmt_model --hparams_path iwslt15
"""
import argparse
import os
import random
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

import parallax_b200 as parallax
import parallax_b200.models.nmt as nmt
from parallax_b200.models.nmt import inference, vocab_utils
import parallax_config

ap = parallax_config.add_flags(argparse.ArgumentParser())
# data
ap.add_argument("--src", default="src", help="source language suffix")
ap.add_argument("--tgt", default="tgt", help="target language suffix")
ap.add_argument("--train_prefix", default=None)
ap.add_argument("--dev_prefix", default=None)
ap.add_argument("--test_prefix", default=None)
ap.add_argument("--vocab_prefix", default=None)
ap.add_argument("--embed_prefix", default=None, help="pretrained embeddings <prefix>.<lang>")
ap.add_argument("--out_dir", default="/tmp/nmt_model")
ap.add_argument("--synthetic", action="store_true",
                help="generate a toy reversal corpus under out_dir/synthetic")
# hyper-parameters: a standard file and/or a comma separated override string
ap.add_argument("--hparams_path", default=None,
                help="standard hparams name (%s) or json path" %
                ", ".join(nmt.hparams.standard_hparams_names()))
ap.add_argument("--hparams", default="", help="name=value,... overrides")
ap.add_argument("--num_train_steps", type=int, default=None)
ap.add_argument("--steps_per_eval", type=int, default=None)
ap.add_argument("--random_seed", type=int, default=None)
ap.add_argument("--clip_embeddings_jointly", action="store_true",
                help="clip embeddings and dense variables by one global norm, as the "
                     "reference does (default: each embedding's gradient on its own)")
ap.add_argument("--eval_only", action="store_true",
                help="restore the latest checkpoint of out_dir / --ckpt_dir and run the internal "
                     "(perplexity) and external (BLEU, …) evaluations — the reference's nmt_eval.py")
# inference
ap.add_argument("--inference_input_file", default=None)
ap.add_argument("--inference_output_file", default=None)
ap.add_argument("--inference_ref_file", default=None)
ap.add_argument("--num_workers", type=int, default=1, help="inference workers")
ap.add_argument("--jobid", type=int, default=0, help="inference worker id")
FLAGS = ap.parse_args()


def synthetic_corpus(d, n_train=20000, n_dev=200, vocab=1000, min_len=5, max_len=30):
    """target = reversed source with renamed words; written once"""
    if os.path.exists(os.path.join(d, "vocab.tgt")):
        return d
    os.makedirs(d, exist_ok=True)
    rng = random.Random(0)
    for name, n in (("train", n_train), ("dev", n_dev), ("test", n_dev)):
        with open(os.path.join(d, name + ".src"), "w") as fs, \
                open(os.path.join(d, name + ".tgt"), "w") as ft:
            for _ in range(n):
                s = [rng.randrange(vocab) for _ in range(rng.randint(min_len, max_len))]
                fs.write(" ".join("w%d" % i for i in s) + "\n")
                ft.write(" ".join("t%d" % i for i in reversed(s)) + "\n")
    for lang, pre in (("src", "w"), ("tgt", "t")):
        with open(os.path.join(d, "vocab." + lang), "w") as f:
            f.write("\n".join(["<unk>", "<s>", "</s>"] + [pre + str(i) for i in range(vocab)]) + "\n")
    return d


def build_hparams():
    hp = nmt.create_hparams(FLAGS.hparams_path)
    hp.src, hp.tgt, hp.out_dir = FLAGS.src, FLAGS.tgt, FLAGS.out_dir
    if FLAGS.synthetic:
        d = synthetic_corpus(os.path.join(FLAGS.out_dir, "synthetic"))
        hp.train_prefix, hp.dev_prefix = d + "/train", d + "/dev"
        hp.test_prefix, hp.vocab_prefix = d + "/test", d + "/vocab"
        hp.subword_option = ""
    for k in ("train_prefix", "dev_prefix", "test_prefix", "vocab_prefix", "embed_prefix"):
        if getattr(FLAGS, k):
            setattr(hp, k, getattr(FLAGS, k))
    if FLAGS.num_train_steps:
        hp.num_train_steps = FLAGS.num_train_steps
    if FLAGS.steps_per_eval:
        hp.steps_per_eval = FLAGS.steps_per_eval
    if FLAGS.random_seed is not None:
        hp.random_seed = FLAGS.random_seed
    if FLAGS.clip_embeddings_jointly:
        hp.clip_embeddings_jointly = True
    hp.parse(FLAGS.hparams)
    if not hp.vocab_prefix:
        raise ValueError("--vocab_prefix (or --synthetic) is required")
    # a previous run's hparams win unless told otherwise (`nmt.py:476-510`)
    loaded = nmt.load_hparams(hp.out_dir)
    if loaded is not None and not hp.override_loaded_hparams:
        hp = loaded
    return hp


def run_inference(hp):
    """restore the latest checkpoint of out_dir and translate a file"""
    nmt.train.prepare_vocab(hp)
    model = nmt.create_model(hp)
    cfg = parallax_config.build_config(FLAGS)
    cfg.ckpt_config = parallax.CheckPointConfig(ckpt_dir=FLAGS.ckpt_dir or hp.out_dir)
    sess, *_ = parallax.parallel_run(nmt.nmt_graph(model, hp), "localhost", sync=True,
                                     parallax_config=cfg)
    sv, tv = vocab_utils.create_vocab_tables(hp.src_vocab_file, hp.tgt_vocab_file, hp.share_vocab)
    out = FLAGS.inference_output_file or os.path.join(hp.out_dir, "translations")
    if FLAGS.num_workers > 1:
        inference.multi_worker_inference(model, hp, FLAGS.inference_input_file, out, sv, tv,
                                         FLAGS.num_workers, FLAGS.jobid)
    else:
        inference.single_worker_inference(model, hp, FLAGS.inference_input_file, out, sv, tv)
    if FLAGS.inference_ref_file and FLAGS.jobid == 0:
        inference.decode_and_evaluate("infer", model, hp, None, sv, tv, out,
                                      ref_file=FLAGS.inference_ref_file, decode=False)
    sess.close()


def run_eval(hp):
    """`nmt_eval.py:571-630` eval_fn: latest checkpoint → dev/test perplexity + scores"""
    cfg = parallax_config.build_config(FLAGS)
    cfg.ckpt_config = parallax.CheckPointConfig(ckpt_dir=FLAGS.ckpt_dir or hp.out_dir)
    tr = nmt.train.train(hp, "localhost", cfg, num_train_steps=0, final_eval=True)
    parallax.log.info("global step %d: dev/test ppl %s, scores %s", tr.sess.engine.global_step,
                      tr.final_ppl, tr.final_scores)
    tr.sess.close()
    return tr


def main():
    hp = build_hparams()
    if FLAGS.inference_input_file:
        return run_inference(hp)
    if FLAGS.eval_only:
        return run_eval(hp)
    cfg = parallax_config.build_config(FLAGS)
    if cfg.ckpt_config.ckpt_dir is None:
        cfg.ckpt_config = parallax.CheckPointConfig(
            ckpt_dir=hp.out_dir, save_ckpt_steps=FLAGS.save_ckpt_steps or
            10 * int(hp.steps_per_stats))
    tr = nmt.train.train(hp, FLAGS.resource_info_file, cfg, sync=FLAGS.sync)
    if tr.worker_id == 0:
        parallax.log.info("final: dev/test ppl %s, scores %s", tr.final_ppl, tr.final_scores)
        if hp.avg_ckpts:
            nmt.train.avg_checkpoints(cfg.ckpt_config.ckpt_dir, hp.num_keep_ckpts)
    tr.sess.close()


if __name__ == "__main__":
    main()
