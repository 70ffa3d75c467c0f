"""Gradient accumulation (`sess_config["micro_batches"]`) on real GPUs; run under torchrun
(tests/test_multigpu_micro_batches.py does, at every world size the box offers):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 \
        --master-addr 127.0.0.1 --master-port 29541 tests/mp_micro_batches_worker.py

Every line is one configuration of the NVLink fabric at K = 3 micro-batches: P2P and (where the
box has NVSwitch multicast) NVLS buckets, eager and CUDA graph, checked against the
single-device oracle on the concatenated global batch; the joint global-norm clip and bf16
master rows against K = 1 on the same rows.  Prints `ALL OK` when every line passes."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

import parallax_b200 as parallax
from parallax_b200 import optim
from parallax_b200.models.simple import MLPWithEmbedding
from parallax_b200.utils import selfcheck as sc

K, B, T, VOCAB, STEPS = 3, 12, 3, 64, 4          # B rows per rank, divisible by K


def make_batch(step, world, rank=None):
    g = torch.Generator().manual_seed(300 + step)
    ids = torch.randint(0, VOCAB, (B * world, T), generator=g)
    ids[:, 0] = ids[0, 0]            # one row in every micro-batch of every rank
    labels = torch.randint(0, 4, (B * world,), generator=g)
    if rank is None:
        return ids, labels
    return ids[rank * B:(rank + 1) * B], labels[rank * B:(rank + 1) * B]


def oracle(world, opt):
    """Single-device training on the concatenated global batch (sparse gradients averaged
    over workers, i.e. the plain gradient of the global mean loss)."""
    model = MLPWithEmbedding(VOCAB)
    model.emb.sparse = False
    params = dict(model.named_parameters())
    slots = {n: tuple(torch.full_like(p, v) for v in opt.slot_init())
             for n, p in params.items()}
    for s in range(STEPS):
        ids, labels = make_batch(s, world)
        model.zero_grad()
        model(ids, labels)["loss"].backward()
        hp = opt.hyper(s + 1)
        with torch.no_grad():
            for n, p in params.items():
                if n == "emb.weight":
                    rows = torch.unique(ids.reshape(-1))
                    optim.apply_sparse_rows_(opt.kind, p.data, rows, p.grad[rows], slots[n], hp)
                else:
                    optim.apply_dense_(opt.kind, p.data, p.grad, slots[n], hp)
    return {n: p.detach().clone() for n, p in params.items()}


def train(world, rank, run_option, micro_batches, sess_config=None, clip=None):
    model = MLPWithEmbedding(VOCAB, partitioner=parallax.get_partitioner(5))
    rules = [parallax.ClipByGlobalNorm(clip, include_sparse=True)] if clip else []
    g = parallax.Graph(model, optimizer=sc.make_opt("adagrad"), grad_rules=rules)
    scfg = dict(sess_config or {})
    scfg["micro_batches"] = micro_batches
    cfg = parallax.Config(run_option=run_option, average_sparse=True, sess_config=scfg,
                          search_partitions=False)
    sess, nw, wid, _ = parallax.parallel_run(g, "localhost", parallax_config=cfg)
    assert (nw, wid) == (world, rank)
    losses, norms = [], []
    for s in range(STEPS):
        ids, labels = make_batch(s, world, rank)
        loss, _ = sess.run(["loss", "train_op"], {"ids": [ids], "labels": [labels]})
        losses.append(loss[0])
        if clip:
            norms.append(sess.engine.grad_norm(0))
    sd = sess.engine.state_dict()
    backend = sess.engine.backend
    sess.close()
    w = dict(sd["dense"]["master"])
    w["emb.weight"] = sd["sparse"]["emb.weight"]["weight"]
    return losses, {n: v.float().cpu() for n, v in w.items()}, norms, backend


def max_err(a, b):
    return max(float((a[n] - b[n]).abs().max()) for n in b)


def main():
    from parallax_b200.parallel.fabric import Comm
    from parallax_b200.parallel import multicast
    comm = Comm.from_env()
    world, rank = comm.world, comm.rank
    ok = True

    def check(name, cond):
        nonlocal ok
        flags = comm.all_gather_object(bool(cond))
        if rank == 0:
            print("%-74s %s" % (name, "OK" if all(flags) else "FAIL %s" % flags), flush=True)
        ok = ok and all(flags)

    nvls = multicast.supported(comm) if world > 1 else False
    if rank == 0:
        print("world %d, K %d, NVLS multicast %s" % (world, K, "available" if nvls else
                                                      "unavailable"), flush=True)
    ref = oracle(world, sc.make_opt("adagrad"))
    fabrics = [("p2p", False)] + ([("nvls", True)] if nvls else [])
    for run_option in ("HYBRID", "MPI", "PS"):
        for graph in (False, True):
            for fname, mc in fabrics:
                _, w, _, backend = train(world, rank, run_option, K, {
                    "cuda_graph": graph, "graph_warmup": 2, "dense_nvls": mc})
                err = max_err(w, ref)
                ok_w = all(torch.allclose(w[n], ref[n], rtol=2e-4, atol=2e-5) for n in ref)
                check("K=%d %s graph=%s dense=%s vs oracle (max err %.1e)"
                      % (K, run_option, graph, fname, err), ok_w and backend == "nvlink")
    # the joint clip: its norm is that of the accumulated gradient, dense and sparse
    l1, w1, n1, _ = train(world, rank, "HYBRID", 1, clip=0.05)
    lk, wk, nk, _ = train(world, rank, "HYBRID", K, clip=0.05)
    check("K=%d joint clip vs K=1 (norm %.4f / %.4f, max err %.1e)"
          % (K, nk[-1], n1[-1], max_err(wk, w1)),
          all(abs(a - b) <= 1e-4 * b for a, b in zip(nk, n1)) and min(n1) > 0.05 and
          all(torch.allclose(wk[n], w1[n], rtol=2e-4, atol=2e-5) for n in w1))
    # bf16 compute and bf16 master rows: each micro-batch's bf16 gradient is rounded on its own
    bf = {"compute_dtype": "bf16", "sparse_weights": "bf16"}
    _, w1, _, _ = train(world, rank, "HYBRID", 1, bf)
    _, wk, _, _ = train(world, rank, "HYBRID", K, bf)
    check("K=%d bf16 compute + bf16 master rows vs K=1 (max err %.1e)" % (K, max_err(wk, w1)),
          all(torch.allclose(wk[n], w1[n], rtol=3e-2, atol=3e-3) for n in w1))
    if rank == 0:
        print("ALL OK" if ok else "SOME FAILED", flush=True)
    comm.shutdown()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
