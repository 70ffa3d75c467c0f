"""Multi-GPU correctness matrix; run under torchrun with >= 2 GPUs (tests/test_multigpu.py
does, at every world size the box offers):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 \
        --master-addr 127.0.0.1 --master-port 29533 tests/mp_nvlink_worker.py [--quick]

Every line is one configuration of the NVLink fabric (CUDA IPC symmetric heap, P2P / NVLS
kernels, flags) checked end to end against the single-device oracle of
`parallax_b200.utils.selfcheck`, plus the public collectives against torch.distributed (NCCL).
Model: Horovod's test suite runs every op under 2 real ranks
(`horovod/test/test_tensorflow.py:70-948`)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
import torch.distributed as dist

import parallax_b200 as parallax
from parallax_b200.utils import selfcheck as sc


def main():
    from parallax_b200.parallel.fabric import Comm
    quick = "--quick" in sys.argv
    comm = Comm.from_env()
    world, rank = comm.world, comm.rank
    ok = True

    def check(name, cond):
        nonlocal ok
        flags = comm.all_gather_object(bool(cond))
        if rank == 0:
            print("%-74s %s" % (name, "OK" if all(flags) else "FAIL %s" % flags), flush=True)
        ok = ok and all(flags)

    def engine(name, run_option, opt, steps=4, average=True, **kw):
        r = sc.check(world, rank, run_option, opt, steps=steps, average=average, **kw)
        check("%s (max err %.1e)" % (name, r["max_abs_err"]),
              r["ok"] and r["backend"] == "nvlink")

    from parallax_b200.parallel import multicast
    nvls = multicast.supported(comm)
    if rank == 0:
        print("world %d, NVLS multicast %s" % (world, "available" if nvls else "unavailable"),
              flush=True)
    fabrics = [("p2p", False)] + ([("nvls", True)] if nvls else [])
    for run_option in ("HYBRID", "MPI", "PS"):
        for opt in ("sgd", "adagrad"):
            for graph in (False, True):
                for fname, mc in fabrics:
                    if quick and (opt == "sgd" or (mc and not graph)):
                        continue
                    steps = 6 if graph else 4
                    engine("engine %s/%s graph=%s dense=%s" % (run_option, opt, graph, fname),
                           run_option, opt, steps,
                           sess_config={"cuda_graph": graph, "dense_nvls": mc})
    engine("early push off (sparse groups pushed after backward)", "HYBRID", "adagrad", 4,
           sess_config={"sparse_early_push": False})
    engine("early push off + graph", "HYBRID", "adagrad", 6,
           sess_config={"sparse_early_push": False, "cuda_graph": True})
    engine("dense last bucket not deferred", "HYBRID", "adagrad", 4,
           sess_config={"dense_defer_last": False})
    engine("sparse SUM semantics (average_sparse=False)", "HYBRID", "adagrad", 4, average=False)
    engine("AR replicated update (two-shot all-reduce + local optimizer)", "MPI", "momentum", 4,
           sess_config={"dense_update": "replicated"})
    engine("PS replicate_variables=False (pull mirrors at next step)", "PS", "adagrad", 4,
           ps=parallax.PSConfig(replicate_variables=False))
    engine("PS local_aggregation=False (owner merges raw entries)", "PS", "adagrad", 4,
           ps=parallax.PSConfig(local_aggregation=False))
    engine("boundary_between_workers_and_servers=False (fp32 wire, owner scales)", "HYBRID",
           "adagrad", 4, ps=parallax.PSConfig(boundary_between_workers_and_servers=False))
    engine("boundary_among_servers=False (round-robin placement)", "HYBRID", "adagrad", 4,
           ps=parallax.PSConfig(boundary_among_servers=False))
    for graph in (False, True):
        for ro in ("HYBRID", "MPI"):
            engine("protocol=nccl (in-engine NCCL arm) %s graph=%s" % (ro, graph), ro, "adagrad",
                   6 if graph else 4, ps=parallax.PSConfig(protocol="nccl"),
                   sess_config={"cuda_graph": graph})
    for opt in ("ftrl", "centered_rmsprop"):
        engine("extended optimizer %s (rule family 1) graph" % opt, "HYBRID", opt, 6,
               sess_config={"cuda_graph": True})
    def trains(losses):
        """finite everywhere, and the loss averaged over ALL ranks went down (one rank's
        8-sample batch is too noisy a signal, Hogwild with 8 writers even more so)"""
        every = comm.all_gather_object([float(x) for x in losses])
        mean = np.mean(np.asarray(every), axis=0)
        return bool(np.isfinite(every).all() and mean[-4:].mean() < mean[:2].mean())
    losses, _, _ = sc.train(world, rank, "PS", "adagrad", 24, False, sync=False)
    check("async PS trains (finite, mean loss over ranks decreases)", trains(losses))
    losses, _, _ = sc.train(world, rank, "HYBRID", "adagrad", 24, True,
                            sess_config={"compute_dtype": "bf16", "cuda_graph": True})
    check("bf16 + graph trains (bf16 wire, bf16 shadow lookups)", trains(losses))
    variable_rows(comm, check)
    sharded_checkpoint(comm, check)
    lm1b_flagship(comm, check)

    # public collectives vs NCCL
    from parallax_b200 import collectives as hvd
    hvd.init(comm)
    sizes = (1, 1000, 65536, 1 << 20, (1 << 22) + 8)
    for n in sizes if not quick else (1000, (1 << 20) + 8):
        for dt in (torch.float32, torch.bfloat16, torch.float16, torch.float64, torch.int32,
                   torch.int64):
            if dt.is_floating_point:
                x = torch.randn(n, device=comm.device).to(dt)
            else:
                x = torch.randint(-1000, 1000, (n,), device=comm.device).to(dt) + \
                    (2 ** 40 if dt == torch.int64 else 0)          # beyond fp32's 2^24
            ref_t = x.clone() if dt != torch.bfloat16 and dt != torch.float16 else x.float()
            dist.all_reduce(ref_t)
            got = hvd.allreduce(x, average=False)
            if dt in (torch.int32, torch.int64):
                good = torch.equal(got, ref_t)
            else:
                tol = {torch.float32: 1e-4, torch.float64: 1e-12}.get(dt, 5e-2)
                good = torch.allclose(got.to(ref_t.dtype), ref_t, rtol=tol, atol=tol)
            check("allreduce n=%d %s" % (n, str(dt).split(".")[-1]), good and got.dtype == dt)
    # non-contiguous inputs (transposed / channels_last) reduce correctly and in place
    x = torch.randn(64, 48, device=comm.device)
    ref_t = x.t().contiguous()
    dist.all_reduce(ref_t)
    check("allreduce of a transposed view", torch.allclose(hvd.allreduce(x.t(), average=False),
                                                           ref_t, rtol=1e-4, atol=1e-4))
    y = torch.randn(4, 8, 6, 6, device=comm.device).contiguous(memory_format=torch.channels_last)
    ref_t = y.clone()
    dist.all_reduce(ref_t)
    hvd.allreduce_(y, average=False)
    check("in-place allreduce_ of a channels_last tensor",
          torch.allclose(y, ref_t, rtol=1e-4, atol=1e-4))
    cnt = torch.tensor([7 + rank, 3], device=comm.device, dtype=torch.int64)
    check("integer average floor-divides",
          torch.equal(hvd.allreduce(cnt, average=True),
                      torch.tensor([(7 * world + world * (world - 1) // 2) // world, 3],
                                   device=comm.device)))
    x = torch.full((1000,), float(rank), device=comm.device)
    got = hvd.broadcast(x, root_rank=world - 1)
    check("broadcast", bool((got == world - 1).all()))
    x = torch.full((10 + rank, 3), float(rank), device=comm.device)
    got = hvd.allgather(x)
    exp = torch.cat([torch.full((10 + r, 3), float(r)) for r in range(world)])
    check("allgather (variable first dim)", torch.equal(got.cpu(), exp))
    hvd.shutdown()
    if rank == 0:
        print("ALL OK" if ok else "SOME FAILED", flush=True)
    comm.shutdown()
    sys.exit(0 if ok else 1)


def variable_rows(comm, check):
    """Row counts that differ between ranks and grow over the steps: the receive rings are
    re-negotiated and re-allocated (no sparse_capacity hint, eager steps)."""
    from parallax_b200 import optim
    from parallax_b200.models.simple import MLPWithEmbedding
    world, rank = comm.world, comm.rank
    V = sc.VOCAB
    model = MLPWithEmbedding(V, partitioner=parallax.get_partitioner(5))
    g = parallax.Graph(model, optimizer=optim.GradientDescent(0.5))
    cfg = parallax.Config(run_option="HYBRID", average_sparse=True, search_partitions=False)
    sess, *_ = parallax.parallel_run(g, "localhost", sync=True, parallax_config=cfg)
    ref = MLPWithEmbedding(V)
    ref.emb.sparse = False
    ropt = torch.optim.SGD(ref.parameters(), lr=0.5)
    for s in range(5):
        gen = torch.Generator().manual_seed(500 + s)
        per_rank = [4 * (1 + ((r + s) % world)) * (1 + s * 3) for r in range(world)]
        ids_all = [torch.randint(0, V, (b, 3), generator=gen) for b in per_rank]
        lab_all = [torch.randint(0, 4, (b,), generator=gen) for b in per_rank]
        sess.run(["loss", "train_op"], {"ids": [ids_all[rank]], "labels": [lab_all[rank]]})
        # oracle: mean over ranks of each rank's mean loss
        ropt.zero_grad()
        sum(ref(i, l)["loss"] for i, l in zip(ids_all, lab_all)).div(world).backward()
        ropt.step()
    grp = sess.engine.sparse_groups[0]
    grew = grp.cap >= max(4 * world * 13 * 3, 64)
    sd = sess.engine.state_dict()
    sess.close()
    good = torch.allclose(sd["sparse"]["emb.weight"]["weight"], ref.emb.weight.detach(),
                          rtol=2e-4, atol=2e-5)
    for n, p in ref.named_parameters():
        if n != "emb.weight":
            good = good and torch.allclose(sd["dense"]["master"][n], p.detach(),
                                           rtol=2e-4, atol=2e-5)
    check("variable rows per rank/step: rings re-negotiated (cap %d)" % grp.cap, good and grew)


def lm1b_flagship(comm, check):
    """The flagship step on N ranks (the smoke() shape: wgmma recurrent product, fused LSTM
    and loss-head nodes, co-lookup group, gradient sinks, CUDA graph, bf16): finite losses and
    bit-identical parameter replicas on every rank after 8 steps of different data per rank."""
    from parallax_b200.models.lm1b import LM1B, lm1b_graph
    world, rank = comm.world, comm.rank
    torch.manual_seed(0)
    B, T, V = 128, 4, 4096
    model = LM1B(vocab_size=V, emb_size=64, state_size=256, projected_size=64, num_sampled=128,
                 num_steps=T, num_shards=8)
    cfg = parallax.Config(run_option="HYBRID", search_partitions=False,
                          sess_config={"compute_dtype": "bf16", "cuda_graph": True})
    sess, *_ = parallax.parallel_run(lm1b_graph(model, batch_size=B), "localhost", sync=True,
                                     parallax_config=cfg)
    g = torch.Generator().manual_seed(7 + rank)
    losses = []
    for _ in range(8):
        x, y = torch.randint(0, V, (B, T), generator=g), torch.randint(0, V, (B, T), generator=g)
        losses.append(float(sess.run(["loss", "train_op"], {"x": [x], "y": [y]})[0][0]))
    m = sess.engine.model
    digest = [float(p.detach().double().abs().sum()) for p in (m.W, m.B, m.W_P)]
    sess.close()
    every = comm.all_gather_object(digest)
    same = all(d == every[0] for d in every)
    check("LM1B flagship step (bf16, graph): finite, replicas identical (|W| %.6g)" % digest[0],
          bool(np.isfinite(losses).all()) and same and losses[-1] < 2 * np.log(V))


def sharded_checkpoint(comm, check):
    """Per-owner checkpoint shards + manifest; restore into a different partitioning."""
    import tempfile
    from parallax_b200 import checkpoint as ckpt
    world, rank = comm.world, comm.rank
    d = comm.broadcast_object(tempfile.mkdtemp(prefix="px_ckpt_") if rank == 0 else None, 0)
    sc.train(world, rank, "HYBRID", "adagrad", 3, True, ckpt_dir=d, save=True)
    _, wa, _ = sc.train(world, rank, "HYBRID", "adagrad", 5, True)
    _, wb, _ = sc.train(world, rank, "HYBRID", "adagrad", 5, True, nparts=3, ckpt_dir=d)
    good = all(torch.allclose(wa[n], wb[n], rtol=2e-4, atol=2e-5) for n in wa)
    files = []
    if rank == 0:
        sub = [f for f in os.listdir(d) if f.startswith("model.ckpt-")][0]
        files = sorted(os.listdir(os.path.join(d, sub)))
    files = comm.broadcast_object(files, 0)
    check("sharded checkpoint (%d files) restored into another partitioning" % len(files),
          good and sum(f.startswith("sparse-") for f in files) >= world)


if __name__ == "__main__":
    main()
