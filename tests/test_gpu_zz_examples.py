"""The example model families on the NVLink fabric (one H100): NMT (GNMT),
skip-thoughts and the CNN benchmark harness take training steps in bf16 and agree
with the host-fabric oracle in fp32.  (Named to run after the kernel suites.)"""
import numpy as np
import pytest
import torch

import parallax_b200 as parallax

pytestmark = pytest.mark.gpu


def _nmt_losses(fabric, dtype, steps):
    import parallax_b200.models.nmt as nmt
    torch.manual_seed(0)
    hp = nmt.create_hparams(num_units=32, num_layers=2, encoder_type="gnmt",
                            attention="normed_bahdanau", attention_architecture="gnmt_v2",
                            residual=True, dropout=0.0, num_embeddings_partitions=2,
                            learning_rate=0.5)
    nmt.extend_hparams(hp, 40, 40)
    m = nmt.create_model(hp)
    sc = {"fabric": fabric}
    if dtype:
        sc["compute_dtype"] = dtype
    sess, *_ = parallax.parallel_run(nmt.nmt_graph(m, hp), "localhost:0",
                                     parallax_config=parallax.Config(search_partitions=False,
                                                                     sess_config=sc))
    g = torch.Generator().manual_seed(1)
    B, S, T = 8, 7, 6
    feed = {"source": [torch.randint(3, 40, (B, S), generator=g)],
            "target_input": [torch.randint(3, 40, (B, T), generator=g)],
            "target_output": [torch.randint(3, 40, (B, T), generator=g)],
            "source_sequence_length": [torch.tensor([7, 5, 3, 6, 7, 2, 4, 7])],
            "target_sequence_length": [torch.tensor([6, 4, 6, 2, 5, 6, 3, 6])]}
    losses = [sess.run(["loss", "train_op"], feed)[0][0] for _ in range(steps)]
    from parallax_b200.models.nmt import inference
    dev = next(m.parameters()).device
    ids, _ = inference.greedy_decode(m, feed["source"][0].to(dev),
                                     feed["source_sequence_length"][0].to(dev), 1, 2, 5)
    sess.close()
    return losses, ids.cpu()


def test_nmt_gnmt_on_nvlink_fabric():
    ref, _ = _nmt_losses("host", None, 6)
    nv, ids = _nmt_losses("nvlink", None, 6)
    np.testing.assert_allclose(nv, ref, rtol=2e-3, atol=2e-3)
    bf, _ = _nmt_losses("nvlink", "bf16", 12)
    assert np.isfinite(bf).all() and bf[-1] < bf[0]
    assert ids.shape[0] == 8 and ids.shape[1] <= 5


def test_skip_thoughts_on_nvlink_fabric():
    from parallax_b200.models import skip_thoughts as st
    from parallax_b200.models.skip_thoughts.input_ops import parse_example_batch
    torch.manual_seed(0)
    mc = st.model_config(vocab_size=48, word_embedding_dim=16, encoder_dim=32, batch_size=4,
                         num_embedding_partitions=2, bidirectional_encoder=True)
    tc = st.training_config(learning_rate=0.01)
    model = st.SkipThoughtsModel(mc)
    sess, *_ = parallax.parallel_run(
        st.skip_thoughts_graph(model, tc), "localhost:0",
        parallax_config=parallax.Config(search_partitions=False,
                                        sess_config={"fabric": "nvlink", "compute_dtype": "bf16"}))
    batch = parse_example_batch([([3, 4, 5, 0], [6, 7, 0], [8, 0]), ([9, 0], [3, 0], [4, 5, 6, 0]),
                                 ([10, 11, 0], [12, 0], [13, 14, 0]), ([5, 0], [6, 0], [7, 0])])
    losses = [sess.run(["loss", "train_op"], st.feed_from_batch(batch))[0][0] for _ in range(15)]
    sess.close()
    assert np.isfinite(losses).all() and losses[-1] < losses[0]


def test_cnn_benchmark_harness_on_nvlink_fabric():
    from parallax_b200.models import cnn_benchmarks as cb
    bench = cb.BenchmarkCNN(cb.make_params(model="lenet", batch_size=16, num_batches=8,
                                           num_warmup_batches=4, display_every=4, use_fp16=True,
                                           optimizer="momentum", learning_rate=0.01))
    cfg = parallax.Config(run_option="MPI", search_partitions=False,
                          sess_config=dict(bench.sess_config(), fabric="nvlink"))
    sess, nw, wid, _ = parallax.parallel_run(bench.build_graph(), "localhost:0",
                                             parallax_config=cfg)
    res = bench.run(sess, nw, wid)
    captured = bool(getattr(sess.engine, "graph_captured", False))
    sess.close()
    assert res["num_steps"] == 8 and np.isfinite(res["average_loss"]) and captured
