"""Layer-wise optimizers (LARS, LAMB) on real GPUs; run under torchrun
(tests/test_multigpu_layerwise.py does, at every world size the box offers):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 \
        --master-addr 127.0.0.1 --master-port 29551 tests/mp_layerwise_worker.py

Every line is one configuration of the NVLink fabric: each rank trains on its share of the
global batch, and the dense masters and slots must match the single-device oracle on the whole
batch (`tests.test_layerwise_cpu.oracle`).  The schedule runs at W > 1: MODE 1, the norm pass,
the one-shot all-reduce of the per-tensor sums and the update pass with its end barrier, right
after each bucket's reduce (no clip) or from the clip rule's `contributed()` (clip), eager and
under a CUDA graph, with two micro-batches, on P2P buckets and, at W >= 4 where the box has
NVSwitch multicast, on NVLS buckets (`dense_nvls=True`, whose update pass stores with
`multimem.st`).  Every rank's parameters must be bitwise equal.  Prints `ALL OK` when every
line passes."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

import parallax_b200 as parallax
from tests.test_layerwise_cpu import DenseNet, _batch, _make_opt, oracle

B, STEPS = 4, 4                  # rows per rank, divisible by the micro-batch count


def train(world, rank, kind, K, clip, sess_config):
    rules = [parallax.ClipByGlobalNorm(clip)] if clip is not None else []
    model = DenseNet()
    g = parallax.Graph(model, optimizer=_make_opt(kind), grad_rules=rules)
    scfg = dict(sess_config)
    scfg["micro_batches"] = K
    cfg = parallax.Config(run_option="HYBRID", sess_config=scfg, search_partitions=False)
    sess, nw, wid, _ = parallax.parallel_run(g, "localhost", parallax_config=cfg)
    assert (nw, wid) == (world, rank)
    for s in range(STEPS):
        x, y = _batch(s, B * world)
        sess.run(["loss", "train_op"], {"x": [x[rank * B:(rank + 1) * B]],
                                        "labels": [y[rank * B:(rank + 1) * B]]})
    torch.cuda.synchronize()
    params = torch.cat([p.detach().float().reshape(-1).cpu() for p in model.parameters()])
    sd = sess.engine.state_dict()
    backend = sess.engine.backend
    nvls = bool(getattr(sess.engine.dense, "nvls", False))
    sess.close()
    return sd["dense"], params, backend, nvls


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

    nvls = multicast.supported(comm) if world >= 4 else False
    if rank == 0:
        print("world %d, NVLS multicast %s" % (world, "used" if nvls else "not used"), flush=True)
    fabrics = [("p2p", False)] + ([("nvls", True)] if nvls else [])
    for kind in ("lars", "lars_nesterov", "lamb"):
        for K, clip, graph in ((1, None, False), (2, 0.05, True)):
            _, ref_w, ref_s = oracle(kind, steps=STEPS, clip=clip, rows=B * world)
            for fname, mc in fabrics:
                dense, params, backend, used_mc = train(world, rank, kind, K, clip, {
                    "cuda_graph": graph, "graph_warmup": 2, "dense_nvls": mc})
                err = max(float((dense["master"][n] - w).abs().max()) for n, w in ref_w.items())
                good = backend == "nvlink" and used_mc == mc and all(
                    torch.allclose(dense["master"][n], w, rtol=2e-4, atol=2e-5) and
                    all(torch.allclose(a, b, rtol=2e-4, atol=2e-5)
                        for a, b in zip(dense["slots"][n], ref_s[n]))
                    for n, w in ref_w.items())
                same = all(torch.equal(p, params) for p in comm.all_gather_object(params))
                check("%s K=%d clip=%s graph=%s dense=%s vs oracle (max err %.1e)"
                      % (kind, K, clip, graph, fname, err), good and same)
    if rank == 0:
        print("ALL OK" if ok else "SOME FAILED", flush=True)
    comm.shutdown()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
