"""LM1B training driver (reference `examples/lm1b/lm1b_distributed_driver.py:49-113`).

    python examples/lm1b/lm1b_distributed_driver.py --use_synthetic \
        --resource_info_file localhost:0,1,2,3,4,5,6,7 --compute_dtype bf16 --cuda_graph

Logs words/sec = Δglobal_step × batch × num_steps × num_workers / Δt.
"""
import argparse
import os
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np
import torch

import parallax_b200 as parallax
from parallax_b200.models.lm1b import LM1B, lm1b_graph, parse_hpconfig
import parallax_config
from parallax_b200.models.lm1b_data import Vocabulary, Dataset

ap = parallax_config.add_flags(argparse.ArgumentParser())
ap.add_argument("--datadir", default=None)
ap.add_argument("--logdir", default="/tmp/lm1b", help="logging directory (analysis reports)")
ap.add_argument("--hpconfig", default="",
                help="override hyper-parameters: name=value,... (batch_size, num_steps, "
                     "learning_rate, max_grad_norm, keep_prob, num_sampled, emb_size, state_size, "
                     "projected_size, vocab_size, num_variable_shards)")
ap.add_argument("--save_n_ckpts_per_epoch", type=int, default=-1,
                help="checkpoints per epoch of the 1B-word corpus (overrides save_ckpt_steps)")
ap.add_argument("--use_synthetic", action="store_true")
ap.add_argument("--batch_size", type=int, default=128)
ap.add_argument("--num_steps", type=int, default=20)
ap.add_argument("--num_variable_shards", type=int, default=32)
ap.add_argument("--learning_rate", type=float, default=0.2)
ap.add_argument("--max_grad_norm", type=float, default=10.0)
ap.add_argument("--max_steps", type=int, default=1000000)
ap.add_argument("--log_frequency", type=int, default=100)
ap.add_argument("--vocab_size", type=int, default=793470)
ap.add_argument("--tiny", action="store_true", help="small model for smoke runs")
FLAGS = ap.parse_args()

NUM_TRAIN_WORDS = 798945280          # words in the 1B-word training shards


def main():
    model_kw = parse_hpconfig(FLAGS.hpconfig, FLAGS)
    kw = dict(vocab_size=FLAGS.vocab_size, num_steps=FLAGS.num_steps,
              num_shards=FLAGS.num_variable_shards, lazy=True)
    if FLAGS.tiny:
        kw.update(vocab_size=min(FLAGS.vocab_size, 10000), emb_size=32, state_size=64,
                  projected_size=32, num_sampled=64, lazy=False)
    kw.update(model_kw)
    model = LM1B(**kw)
    single_gpu_graph = lm1b_graph(model, FLAGS.batch_size, FLAGS.learning_rate,
                                  FLAGS.max_grad_norm)
    dataset = None
    if not FLAGS.use_synthetic:
        vocab = Vocabulary.from_file(os.path.join(FLAGS.datadir, "1b_word_vocab.txt"))
        dataset = Dataset(vocab, os.path.join(
            FLAGS.datadir, "training-monolingual.tokenized.shuffled/*"))

    def run(sess, num_workers, worker_id, num_replicas_per_worker):
        B, T, V = FLAGS.batch_size, FLAGS.num_steps, model.vocab_size
        state_c = [np.zeros([B, model.state_size], np.float32)] * num_replicas_per_worker
        state_h = [np.zeros([B, model.projected_size], np.float32)] * num_replicas_per_worker
        it = None if dataset is None else dataset.iterate_forever(
            B * num_replicas_per_worker, T, num_workers, worker_id)
        prev_step = sess.run("global_step")[0]
        prev_time = time.time()
        fetches = {"global_step": "global_step", "loss": "loss", "train_op": "train_op",
                   "final_state_c": "final_state_c", "final_state_h": "final_state_h"}
        for local_step in range(FLAGS.max_steps):
            if it is None:
                x = np.random.randint(0, V, size=(B * num_replicas_per_worker, T))
                y = np.random.randint(0, V, size=(B * num_replicas_per_worker, T))
                w = np.ones((B * num_replicas_per_worker, T), np.float32)
            else:
                x, y, w = next(it)
            feeds = {"x": np.split(x, num_replicas_per_worker),
                     "y": np.split(y, num_replicas_per_worker),
                     "w": np.split(w, num_replicas_per_worker),
                     "initial_state_c": state_c, "initial_state_h": state_h}
            fetched = sess.run(fetches, feeds)
            state_c, state_h = fetched["final_state_c"], fetched["final_state_h"]
            if local_step % FLAGS.log_frequency == 0:
                now = time.time()
                gs = fetched["global_step"][0]
                elapsed = max(now - prev_time, 1e-9)
                wps = (gs - prev_step) * B * T * num_workers / elapsed
                prev_step, prev_time = gs, now
                parallax.log.info("Iteration %d, time = %.2fs, wps = %.0f, train loss = %.4f",
                                  gs, elapsed, wps, fetched["loss"][0])
        sess.close()

    cfg = parallax_config.build_config(FLAGS)
    if cfg.export_graph_path is None:
        cfg.export_graph_path = FLAGS.logdir
    if FLAGS.save_n_ckpts_per_epoch > 0 and FLAGS.ckpt_dir:
        # steps per epoch depend on the number of workers, known from the resource spec
        from parallax_b200.resource import parse_resource_info, worker_layout
        nw = len(worker_layout(parse_resource_info(FLAGS.resource_info_file,
                                                   cfg.normalized_run_option())))
        per_epoch = NUM_TRAIN_WORDS // (FLAGS.batch_size * FLAGS.num_steps * nw)
        cfg.ckpt_config = parallax.CheckPointConfig(
            ckpt_dir=FLAGS.ckpt_dir,
            save_ckpt_steps=max(per_epoch // FLAGS.save_n_ckpts_per_epoch, 1))
    sess, num_workers, worker_id, num_replicas_per_worker = parallax.parallel_run(
        single_gpu_graph, FLAGS.resource_info_file, sync=FLAGS.sync, parallax_config=cfg)
    run(sess, num_workers, worker_id, num_replicas_per_worker)


if __name__ == "__main__":
    main()
