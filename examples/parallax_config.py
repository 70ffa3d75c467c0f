"""Shared flag → `parallax.Config` mapping used by every example (the
reference copy-pastes this file per example:
`examples/lm1b/parallax_config.py:19-79`)."""
import argparse

import parallax_b200 as parallax


def add_flags(ap):
    ap.add_argument("--resource_info_file", default="localhost",
                    help="resource file (host[:gpu,gpu...] per line) or its text")
    ap.add_argument("--run_option", default="HYBRID", help="PS | MPI(AR) | HYBRID")
    ap.add_argument("--sync", type=lambda s: s.lower() != "false", default=True)
    ap.add_argument("--redirect_path", default=None)
    ap.add_argument("--ckpt_dir", default=None)
    ap.add_argument("--save_ckpt_steps", type=int, default=None)
    ap.add_argument("--save_ckpt_secs", type=int, default=None)
    ap.add_argument("--profile_dir", default=None)
    ap.add_argument("--profile_steps", default=None, help="comma separated steps")
    ap.add_argument("--profile_range", default=None, help="start,end")
    ap.add_argument("--profile_worker", type=int, default=None)
    ap.add_argument("--local_aggregation", type=lambda s: s.lower() != "false", default=True)
    ap.add_argument("--replicate_variables", type=lambda s: s.lower() != "false", default=True)
    ap.add_argument("--boundary_among_servers", type=lambda s: s.lower() != "false", default=True)
    ap.add_argument("--boundary_between_workers_and_servers",
                    type=lambda s: s.lower() != "false", default=True)
    ap.add_argument("--protocol", default="grpc")
    ap.add_argument("--mpirun_options", default="")
    ap.add_argument("--search_partitions", type=lambda s: s.lower() != "false", default=False)
    ap.add_argument("--average_sparse", action="store_true")
    ap.add_argument("--export_graph_path", default=None)
    ap.add_argument("--compute_dtype", default=None, help="bf16 | float32")
    ap.add_argument("--cuda_graph", action="store_true")
    # K forward/backward passes per optimizer step: every feed of a step is split into K
    # equal micro-batches along dim 0, so the per-worker batch a driver feeds is K·b.  Give
    # graph builders that take a batch size the per-worker K·b: `lm1b_graph(batch_size=...)`
    # scales the embedding gradients by it (ScaleGradients), and its 1/K weighting expects it.
    ap.add_argument("--micro_batches", type=int, default=1,
                    help="forward/backward passes per optimizer step (gradient accumulation)")
    # how parallax.nn.full_softmax_nll trains (LM1B with num_sampled=0): "fused" needs the
    # NVLink fabric and --compute_dtype bf16
    ap.add_argument("--full_softmax_train", default="composition",
                    choices=["composition", "fused"],
                    help="full-softmax training: gather + matmul composition, or fused kernels")
    return ap


def build_config(FLAGS):
    ckpt = parallax.CheckPointConfig(ckpt_dir=FLAGS.ckpt_dir,
                                     save_ckpt_steps=FLAGS.save_ckpt_steps,
                                     save_ckpt_secs=FLAGS.save_ckpt_secs)
    ps = parallax.PSConfig(
        protocol=FLAGS.protocol, replicate_variables=FLAGS.replicate_variables,
        local_aggregation=FLAGS.local_aggregation,
        boundary_among_servers=FLAGS.boundary_among_servers,
        boundary_between_workers_and_servers=FLAGS.boundary_between_workers_and_servers)
    mpi = parallax.MPIConfig(mpirun_options=FLAGS.mpirun_options)
    steps = [int(s) for s in FLAGS.profile_steps.split(",")] if FLAGS.profile_steps else None
    rng = tuple(int(s) for s in FLAGS.profile_range.split(",")) if FLAGS.profile_range else None
    prof = parallax.ProfileConfig(profile_dir=FLAGS.profile_dir, profile_steps=steps,
                                  profile_range=rng, profile_worker=FLAGS.profile_worker)
    sc = {}
    if FLAGS.compute_dtype:
        sc["compute_dtype"] = FLAGS.compute_dtype
    if FLAGS.cuda_graph:
        sc["cuda_graph"] = True
    if getattr(FLAGS, "micro_batches", 1) != 1:
        sc["micro_batches"] = FLAGS.micro_batches
    if getattr(FLAGS, "full_softmax_train", "composition") != "composition":
        sc["full_softmax_train"] = FLAGS.full_softmax_train
    cfg = parallax.Config()
    cfg.run_option = FLAGS.run_option
    cfg.average_sparse = FLAGS.average_sparse
    cfg.redirect_path = FLAGS.redirect_path
    cfg.search_partitions = FLAGS.search_partitions
    cfg.export_graph_path = FLAGS.export_graph_path
    cfg.sess_config = sc or None
    cfg.communication_config = parallax.CommunicationConfig(ps, mpi)
    cfg.ckpt_config = ckpt
    cfg.profile_config = prof
    return cfg
