"""Gradient accumulation on the NVLink fabric (`sess_config["micro_batches"]`): the fused
dense step's accumulate mode (MODE 3 and the accumulator-in flag) against the fp32 oracle
on simulated worlds, and the engine against the host fabric and against one pass."""
import numpy as np
import pytest
import torch

import parallax_b200 as parallax
from parallax_b200 import optim
from parallax_b200.models.simple import MLPWithEmbedding

pytestmark = pytest.mark.gpu

MODE_FUSED, MODE_REDUCE, MODE_UPDATE, MODE_ACCUMULATE = 0, 1, 2, 3


def _opt(name):
    return {"sgd": optim.GradientDescent(0.3), "adagrad": optim.Adagrad(0.2, 1.0),
            "adam": optim.Adam(0.01),
            "ftrl": optim.Ftrl(0.2, l1_regularization_strength=0.001)}[name]


def _world(world, dtype, n, opt, seed):
    from tests.gpu_utils import make_world
    fabs = make_world(world)
    sl = n // world
    gb = [f.heap.alloc(n * 4, "g") for f in fabs]
    pb = [f.heap.alloc(n * 4, "p") for f in fabs]
    gen = torch.Generator(device="cuda").manual_seed(seed)
    w0 = torch.randn(n, device="cuda", generator=gen).to(dtype).float()
    for r in range(world):
        pb[r].tensor(dtype, n).copy_(w0)
    master = [w0[r * sl:(r + 1) * sl].clone() for r in range(world)]
    slots = [[torch.full((sl,), v, device="cuda") for v in opt.slot_init()]
             for _ in range(world)]
    red = [torch.full((sl,), float("nan"), device="cuda") for _ in range(world)]
    return fabs, gb, pb, w0, master, slots, red, gen


def _fill_grads(gb, dtype, n, gen):
    """New gradients in every rank's bucket; returns their fp32 sum over ranks."""
    total = torch.zeros(n, device="cuda")
    for b in gb:
        g = (torch.randn(n, device="cuda", generator=gen) * 0.5).to(dtype)
        b.tensor(dtype, n).copy_(g)
        total += g.float()
    return total


def _slot_args(s):
    return (s[0] if len(s) > 0 else None, s[1] if len(s) > 1 else None,
            s[2] if len(s) > 2 else None)


@pytest.mark.parametrize("world", [1, 2, 3, 4, 5, 6, 7, 8])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("opt_name", ["sgd", "adagrad", "adam", "ftrl"])
def test_accumulate_then_fused_step(world, dtype, opt_name):
    """Three micro-batches: MODE 3, MODE 3 with the accumulator, MODE 0 with the
    accumulator, the buckets overwritten in between, equal one update with the fp32 mean
    gradient; every rank ends with the same parameters, bit for bit."""
    from parallax_b200.parallel import nvops
    from parallax_b200.parallel.symmetric import CH_COMM
    K, opt = 3, _opt(opt_name)
    vn = 4 if dtype == torch.float32 else 8
    n = world * vn * 32 * 5
    fabs, gb, pb, w0, master, slots, red, gen = _world(world, dtype, n, opt, 11)
    hp_list = opt.hyper(1)
    hp = torch.tensor(hp_list, device="cuda")
    gsum = torch.zeros(n, device="cuda")
    for k, (mode, acc_in) in enumerate([(MODE_ACCUMULATE, False), (MODE_ACCUMULATE, True),
                                        (MODE_FUSED, True)]):
        gsum += _fill_grads(gb, dtype, n, gen)
        torch.cuda.synchronize()
        # phase by phase: no simulated rank may enqueue a later phase in front of a peer's
        # earlier one
        for r, f in enumerate(fabs):
            s0, s1, s2 = _slot_args(slots[r])
            nvops.dense_step(f.heap, gb[r].c_ptrs(), pb[r].c_ptrs(), master[r], s0, s1,
                             None, red[r], hp, None, None, n, 1.0 / (world * K), 0.0,
                             opt.kind, mode, dtype, CH_COMM, max_blocks=4,
                             stream=f.comm_stream, slot2=s2, acc_in=acc_in)
        torch.cuda.synchronize()
        if mode == MODE_ACCUMULATE:       # no update before the step's last micro-batch
            for r in range(world):
                assert torch.equal(pb[r].tensor(dtype, n).float(), w0)
    ref_w = w0.clone()
    ref_slots = [torch.full((n,), v, device="cuda") for v in opt.slot_init()]
    optim.apply_dense_(opt.kind, ref_w, gsum / (world * K), tuple(ref_slots), hp_list)
    torch.testing.assert_close(torch.cat(master), ref_w, rtol=1e-5, atol=1e-5)
    for i, s in enumerate(ref_slots):
        torch.testing.assert_close(torch.cat([sl[i] for sl in slots]), s, rtol=1e-5, atol=1e-5)
    p0 = pb[0].tensor(dtype, n).clone()
    torch.testing.assert_close(p0.float(), ref_w.to(dtype).float(), rtol=1e-2 if
                               dtype == torch.bfloat16 else 1e-5, atol=1e-5)
    for r in range(1, world):
        assert torch.equal(pb[r].tensor(dtype, n), p0)
    for f in fabs:
        f.close()


@pytest.mark.parametrize("world", [1, 4])
def test_accumulate_then_two_phase_clip(world):
    """MODE 3, MODE 1 with the accumulator, one-shot all-reduce of Σg², clip scale, MODE 2:
    the norm is that of the accumulated gradient, and the update is clip-then-apply."""
    from parallax_b200.parallel import nvops
    from parallax_b200.parallel.symmetric import CH_COMM, CH_SMALL
    K, dtype, opt = 2, torch.float32, _opt("adagrad")
    n = world * 4 * 32 * 5
    fabs, gb, pb, w0, master, slots, red, gen = _world(world, dtype, n, opt, 5)
    loc = [torch.zeros(4, device="cuda") for _ in range(world)]
    tot = [torch.zeros(4, device="cuda") for _ in range(world)]
    scale = [torch.ones(1, device="cuda") for _ in range(world)]
    norm = [torch.zeros(1, device="cuda") for _ in range(world)]
    hp_list = opt.hyper(1)
    hp = torch.tensor(hp_list, device="cuda")
    max_norm = 1.0
    gsum = torch.zeros(n, device="cuda")
    for mode, acc_in in [(MODE_ACCUMULATE, False), (MODE_REDUCE, True)]:
        gsum += _fill_grads(gb, dtype, n, gen) * 3
        for b in gb:
            b.tensor(dtype, n).mul_(3)
        torch.cuda.synchronize()
        for r, f in enumerate(fabs):
            nvops.dense_step(f.heap, gb[r].c_ptrs(), pb[r].c_ptrs(), master[r], slots[r][0],
                             None, None, red[r], hp, None,
                             loc[r] if mode == MODE_REDUCE else None, n, 1.0 / (world * K),
                             0.0, "adagrad", mode, dtype, CH_COMM, max_blocks=4,
                             stream=f.comm_stream, acc_in=acc_in)
        torch.cuda.synchronize()
    for r, f in enumerate(fabs):
        if world > 1:
            nvops.allreduce_oneshot(f.heap, loc[r], tot[r], f.small_stage, 4,
                                    torch.float32, 1.0, CH_SMALL, stream=f.comm_stream)
    for r, f in enumerate(fabs):
        nvops.clip_scale(tot[r] if world > 1 else loc[r], max_norm, scale[r], norm[r],
                         loc[r], stream=f.comm_stream)
        nvops.dense_step(f.heap, gb[r].c_ptrs(), pb[r].c_ptrs(), master[r], slots[r][0],
                         None, None, red[r], hp, scale[r], None, n, 1.0 / (world * K),
                         0.0, "adagrad", MODE_UPDATE, dtype, CH_COMM, max_blocks=4,
                         stream=f.comm_stream)
    torch.cuda.synchronize()
    gmean = gsum / (world * K)
    gn = float(gmean.norm())
    assert gn > max_norm
    for r in range(world):
        assert abs(float(norm[r]) - gn) < 1e-4 * gn
    ref_w, ref_acc = w0.clone(), torch.full((n,), 1.0, device="cuda")
    optim.apply_dense_("adagrad", ref_w, gmean * (max_norm / gn), (ref_acc,), hp_list)
    torch.testing.assert_close(torch.cat(master), ref_w, rtol=1e-5, atol=1e-5)
    for r in range(world):
        torch.testing.assert_close(pb[r].tensor(dtype, n), ref_w, rtol=1e-5, atol=1e-5)
    for f in fabs:
        f.close()


def _run(fabric, run_option, K, steps=4, compute_dtype=None, clip=0.5, graph=False,
         include_sparse=False, sparse_weights=None, norms=None):
    model = MLPWithEmbedding(64, partitioner=parallax.get_partitioner(3))
    rules = [parallax.ClipByGlobalNorm(
        clip, params=None if include_sparse else ["fc1.*", "fc2.*"],
        include_sparse=include_sparse)] if clip else []
    g = parallax.Graph(model, optimizer=optim.Adagrad(0.2, 1.0), grad_rules=rules,
                       ema=parallax.ExponentialMovingAverage(0.9, ["fc2.*"]))
    sc = {"fabric": fabric, "cuda_graph": graph, "micro_batches": K}
    if compute_dtype:
        sc["compute_dtype"] = compute_dtype
    if sparse_weights:
        sc["sparse_weights"] = sparse_weights
    cfg = parallax.Config(run_option=run_option, average_sparse=True, sess_config=sc)
    sess, *_ = parallax.parallel_run(g, "localhost:0", parallax_config=cfg)
    gen = torch.Generator().manual_seed(0)
    losses = []
    for s in range(steps):
        ids = torch.randint(0, 64, (16, 3), generator=gen)
        ids[:, 0] = 5                 # one row in every micro-batch
        labels = torch.randint(0, 4, (16,), generator=gen)
        loss, _ = sess.run(["loss", "train_op"], {"ids": [ids], "labels": [labels]})
        losses.append(loss[0])
        if norms is not None:
            norms.append(sess.engine.grad_norm(0))
    sd = sess.engine.state_dict()
    sess.close()
    return losses, sd


def _same(a, b, tol):
    (l_a, sd_a), (l_b, sd_b) = a, b
    np.testing.assert_allclose(l_a, l_b, rtol=tol[0], atol=tol[1])
    for part in ("master", "ema"):
        for n, w in sd_b["dense"][part].items():
            torch.testing.assert_close(sd_a["dense"][part][n], w, rtol=tol[0], atol=tol[1])
    torch.testing.assert_close(sd_a["sparse"]["emb.weight"]["weight"],
                               sd_b["sparse"]["emb.weight"]["weight"], rtol=tol[0], atol=tol[1])


@pytest.mark.parametrize("run_option", ["HYBRID", "MPI", "PS"])
def test_engine_fp32_matches_host_and_one_pass(run_option):
    nv4 = _run("nvlink", run_option, 4)
    _same(nv4, _run("host", run_option, 4), (1e-4, 1e-5))
    _same(nv4, _run("nvlink", run_option, 1), (1e-4, 1e-5))


@pytest.mark.parametrize("run_option", ["HYBRID", "MPI", "PS"])
def test_engine_bf16_matches_one_pass(run_option):
    """bf16 compute: each micro-batch's bf16 gradient is rounded on its own, so K=4 and one
    pass differ at bf16 precision."""
    nv4 = _run("nvlink", run_option, 4, compute_dtype="bf16")
    _same(nv4, _run("nvlink", run_option, 1, compute_dtype="bf16"), (3e-2, 3e-3))


@pytest.mark.parametrize("run_option", ["HYBRID", "PS"])
def test_engine_joint_clip_matches_host_and_one_pass(run_option):
    """ClipByGlobalNorm(include_sparse=True): the owners' `stage_norm` sees the merged rows
    weighted 1/K, so the norm and the update are those of the accumulated gradient."""
    kw = dict(clip=0.05, include_sparse=True)
    n_nv, n_host, n_one = [], [], []
    nv4 = _run("nvlink", run_option, 4, norms=n_nv, **kw)
    _same(nv4, _run("host", run_option, 4, norms=n_host, **kw), (1e-4, 1e-5))
    _same(nv4, _run("nvlink", run_option, 1, norms=n_one, **kw), (1e-4, 1e-5))
    assert min(n_one) > 0.05              # every step clips
    np.testing.assert_allclose(n_nv, n_host, rtol=1e-4)
    np.testing.assert_allclose(n_nv, n_one, rtol=1e-4)


def test_engine_bf16_master_rows_match_one_pass():
    """sparse_weights="bf16" (stochastic rounding keyed by step, row and column) with bf16
    compute, the joint clip included: K=4 against one pass over the same rows."""
    kw = dict(compute_dtype="bf16", sparse_weights="bf16", clip=0.05, include_sparse=True)
    _same(_run("nvlink", "HYBRID", 4, **kw), _run("nvlink", "HYBRID", 1, **kw), (3e-2, 3e-3))


def test_engine_cuda_graph_matches_eager():
    eager = _run("nvlink", "HYBRID", 4, steps=7)
    replay = _run("nvlink", "HYBRID", 4, steps=7, graph=True)
    _same(replay, eager, (1e-5, 1e-6))


def _lm1b_session(K, B=128):
    from parallax_b200.models.lm1b import LM1B, lm1b_graph
    torch.manual_seed(0)
    model = LM1B(vocab_size=4096, emb_size=64, state_size=256, projected_size=64,
                 num_sampled=128, num_steps=4, num_shards=2)
    graph = lm1b_graph(model, batch_size=(K or 1) * B)
    sc = {"compute_dtype": "bf16", "cuda_graph": True, "graph_warmup": 3}
    if K is not None:
        sc["micro_batches"] = K
    cfg = parallax.Config(run_option="HYBRID", sess_config=sc)
    sess, *_ = parallax.parallel_run(graph, "localhost:0", parallax_config=cfg)
    gen = torch.Generator().manual_seed(1)
    x = torch.randint(0, 4096, ((K or 1) * B, 4), generator=gen)
    y = torch.randint(0, 4096, ((K or 1) * B, 4), generator=gen)
    return sess, {"x": [x], "y": [y]}


def _native_counter(monkeypatch):
    """Counts the calls of the native entry points that launch the sparse push, the sparse
    owner and the fused dense step kernels (by mode)."""
    from parallax_b200 import ops
    L = ops.lib()
    calls = {"push": 0, "owner": 0, "dense": []}

    def wrap(name, key, mode_arg=None):
        real = getattr(L, name)

        def fn(*a):
            if mode_arg is None:
                calls[key] += 1
            else:
                calls[key].append(a[mode_arg])
            return real(*a)
        monkeypatch.setattr(L, name, fn)
    wrap("px_sparse_push", "push")
    wrap("px_sparse_owner", "owner")
    wrap("px_dense_step", "dense", mode_arg=15)
    return calls


def test_lm1b_counts_one_push_and_k_dense_launches(monkeypatch):
    """Small LM1B, two micro-batches under the CUDA graph: finite losses.  In an eager step
    every sparse group launches its push kernel once and its owner kernel once; every dense
    bucket launches the fused step K times, plus its MODE 2 update when it is clipped."""
    K = 2
    calls = _native_counter(monkeypatch)
    sess, feed = _lm1b_session(K)
    losses = []
    for s in range(6):
        calls["push"], calls["owner"], calls["dense"] = 0, 0, []
        loss, _ = sess.run(["loss", "train_op"], feed)
        losses.append(loss[0])
        if s == 1:                        # an eager step with every lazy allocation done
            eng = sess.engine
            nb = len(eng.dense.buckets)
            clipped = sum(1 for b in eng.dense.buckets if b.clip >= 0)
            assert calls["push"] == calls["owner"] == len(eng.sparse_groups)
            modes = calls["dense"]
            assert modes.count(MODE_ACCUMULATE) == (K - 1) * nb
            assert modes.count(MODE_FUSED) + modes.count(MODE_REDUCE) == nb
            assert modes.count(MODE_UPDATE) == clipped
            assert len(modes) == K * nb + clipped
    assert sess.engine.graph_captured
    assert all(np.isfinite(l) for l in losses)
    sess.close()


def test_lm1b_k1_launches_as_without_the_key():
    """micro_batches=1 runs the step of a session without the key: the same launch count
    (`nvops.launches`) in an eager step and in a replayed one, and the same losses."""
    from parallax_b200.parallel import nvops
    per = {}
    for key in (None, 1):
        sess, feed = _lm1b_session(key)
        counts, losses = [], []
        for s in range(6):
            l0 = nvops.launches["n"]
            loss, _ = sess.run(["loss", "train_op"], feed)
            counts.append(nvops.launches["n"] - l0)
            losses.append(loss[0])
        assert sess.engine.graph_captured
        sess.close()
        per[key] = (counts[1], counts[-1], losses)
    assert per[1][:2] == per[None][:2]
    np.testing.assert_allclose(per[1][2], per[None][2], rtol=1e-6)
