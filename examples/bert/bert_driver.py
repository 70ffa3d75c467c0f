"""BERT masked-LM driver (BASELINE.json config 5: BERT-large, hybrid mode — transformer
weights on the fused dense path, the word-embedding table on the sparse path).  Not a
reference example.

    python examples/bert/bert_driver.py --size large --compute_dtype bf16 --cuda_graph \
        --resource_info_file localhost:0,1,2,3,4,5,6,7
"""
import argparse
import os
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import torch

import parallax_b200 as parallax
from parallax_b200.models.bert import Bert, bert_graph
import parallax_config

SIZES = {"tiny": dict(hidden=64, layers=2, heads=4, ff=128),
         "base": dict(hidden=768, layers=12, heads=12, ff=3072),
         "large": dict(hidden=1024, layers=24, heads=16, ff=4096)}

ap = parallax_config.add_flags(argparse.ArgumentParser())
ap.add_argument("--size", default="large", choices=sorted(SIZES))
ap.add_argument("--vocab_size", type=int, default=30522)
ap.add_argument("--batch_size", type=int, default=16)
ap.add_argument("--seq_len", type=int, default=512)
ap.add_argument("--mlm_fraction", type=float, default=0.15)
ap.add_argument("--learning_rate", type=float, default=1e-4)
ap.add_argument("--optimizer", default="adam", choices=["adam", "lamb"],
                help="lamb: LAMB for the dense variables (the large-batch recipe), Adam for "
                     "the word embedding")
ap.add_argument("--num_partitions", type=int, default=8)
ap.add_argument("--max_steps", type=int, default=100)
ap.add_argument("--log_frequency", type=int, default=10)
FLAGS = ap.parse_args()


def main():
    model = Bert(vocab=FLAGS.vocab_size, max_len=FLAGS.seq_len,
                 num_partitions=FLAGS.num_partitions, **SIZES[FLAGS.size])
    graph = bert_graph(model, FLAGS.learning_rate, optimizer=FLAGS.optimizer)
    sess, num_workers, worker_id, _ = parallax.parallel_run(
        graph, FLAGS.resource_info_file, sync=FLAGS.sync,
        parallax_config=parallax_config.build_config(FLAGS))
    gen = torch.Generator().manual_seed(5 + worker_id)
    B, T, V = FLAGS.batch_size, FLAGS.seq_len, FLAGS.vocab_size
    nm = max(1, int(T * FLAGS.mlm_fraction))
    t0 = time.time()
    for step in range(1, FLAGS.max_steps + 1):
        ids = torch.randint(5, V, (B, T), generator=gen)
        pos = torch.stack([torch.randperm(T, generator=gen)[:nm] for _ in range(B)])
        labels = torch.gather(ids, 1, pos)                  # predict the token that was there
        masked = ids.scatter(1, pos, 4)                     # id 4 = [MASK]
        loss, _ = sess.run(["loss", "train_op"], {"input_ids": [masked], "mlm_positions": [pos],
                                                  "mlm_labels": [labels]})
        if worker_id == 0 and step % FLAGS.log_frequency == 0:
            dt = time.time() - t0
            t0 = time.time()
            parallax.log.info("step %d  mlm loss %.4f  %.1fk tokens/sec (total)", step, loss[0],
                              FLAGS.log_frequency * B * T * num_workers / dt / 1e3)
    sess.close()


if __name__ == "__main__":
    main()
