"""Gradient accumulation (`sess_config["micro_batches"]`) on the host and library fabrics:
one step of K micro-batches over a per-worker batch of K·b rows gives the update of one
pass over the same rows, for every run option, optimizer, clip rule and weight format."""
import numpy as np
import pytest
import torch

import parallax_b200 as parallax
from parallax_b200 import optim
from parallax_b200.models.simple import MLPWithEmbedding
from tests.dist_utils import run_distributed
from tests.test_hybrid_cpu import VOCAB, make_batch, make_opt, oracle

STEPS = 3


def _opts(opt_name):
    """(dense optimizer, sparse optimizer or None)"""
    if opt_name == "rowwise":
        return optim.Adagrad(0.2, initial_accumulator_value=1.0), \
            optim.RowWiseAdagrad(0.3, 0.5, epsilon=1e-3)
    return make_opt(opt_name), None


def _train(world, rank, run_option, opt_name, K, clip=None, include_sparse=False,
           sparse_weights=None, fabric=None, average=True, steps=STEPS):
    """`steps` steps of the global batches of `tests.test_hybrid_cpu` (8 rows per worker
    of a world of 2), this rank's share of them per step."""
    opt, sparse_opt = _opts(opt_name)
    model = MLPWithEmbedding(VOCAB, partitioner=parallax.get_partitioner(3))
    rules = []
    if clip is not None:
        rules = [parallax.ClipByGlobalNorm(
            clip, params=None if include_sparse else ["fc1.*", "fc2.*"],
            include_sparse=include_sparse)]
    graph = parallax.Graph(model, optimizer=opt, sparse_optimizer=sparse_opt,
                           grad_rules=rules)
    sc = {}
    if K is not None:
        sc["micro_batches"] = K
    if fabric:
        sc["fabric"] = fabric
    if sparse_weights:
        sc["sparse_weights"] = sparse_weights
    cfg = parallax.Config(run_option=run_option, average_sparse=average, sess_config=sc)
    sess, nw, wid, _ = parallax.parallel_run(graph, "localhost", parallax_config=cfg)
    assert (nw, wid) == (world, rank)
    losses, norms = [], []
    for s in range(steps):
        ids, labels = make_batch(s, 2)
        n = ids.shape[0] // world
        loss, gs, _ = sess.run(["loss", "global_step", "train_op"],
                               {"ids": [ids[rank * n:(rank + 1) * n]],
                                "labels": [labels[rank * n:(rank + 1) * n]]})
        assert gs == [s + 1]              # one optimizer step per step, whatever K is
        losses.append(loss[0])
        if clip is not None:
            norms.append(sess.engine.grad_norm(0))
    sd = sess.engine.state_dict()
    sess.close()
    weights = dict(sd["dense"]["master"])
    weights["emb.weight"] = sd["sparse"]["emb.weight"]["weight"]
    slots = {n: v for n, v in sd["dense"]["slots"].items()}
    slots["emb.weight"] = sd["sparse"]["emb.weight"]["slots"]
    return losses, weights, slots, norms


def _worker(rank, world, specs):
    """Several runs in one process group: each is a kwargs dict of `_train`."""
    return [_train(world, rank, **spec) for spec in specs]


def _close(got, want, tol):
    rtol, atol = tol
    for n, w in want.items():
        if isinstance(w, (list, tuple)):
            for a, b in zip(got[n], w):
                torch.testing.assert_close(a, b, rtol=rtol, atol=atol)
        else:
            torch.testing.assert_close(got[n], w, rtol=rtol, atol=atol)


TOL = (1e-5, 1e-6)


def _check_two_ranks(results, ref, tol=TOL):
    """`results`: per rank, the `_train` results of one spec; `ref`: a world-1 result on
    the concatenated rows."""
    ref_losses, ref_w, ref_slots, ref_norms = ref
    np.testing.assert_allclose(np.mean([r[0] for r in results], axis=0), ref_losses,
                               rtol=tol[0], atol=tol[1])
    for losses, weights, slots, norms in results:
        _close(weights, ref_w, tol)
        _close(slots, ref_slots, tol)
        if ref_norms:
            np.testing.assert_allclose(norms, ref_norms, rtol=1e-5)


@pytest.mark.parametrize("run_option", ["HYBRID", "PS", "MPI"])
@pytest.mark.parametrize("opt_name", ["sgd", "adagrad", "adam", "rowwise"])
def test_two_workers_match_single_pass(run_option, opt_name):
    """K ∈ {2, 4} on two workers equals one pass over the concatenated global batch: the
    plain-torch oracle of `test_hybrid_cpu` for the element-wise rules, and the engine
    itself on one worker for row-wise Adagrad (which that oracle does not model)."""
    specs = [dict(run_option=run_option, opt_name=opt_name, K=K) for K in (2, 4)]
    res = run_distributed(_worker, 2, specs)
    if opt_name == "rowwise":
        ref = _train(1, 0, run_option, opt_name, None)
        for i in range(len(specs)):
            _check_two_ranks([r[i] for r in res], ref)
        return
    ref_losses, ref_w = oracle(2, STEPS, make_opt(opt_name), sparse_scale=1.0)
    for i in range(len(specs)):
        mean_losses = np.mean([r[i][0] for r in res], axis=0)
        np.testing.assert_allclose(mean_losses, ref_losses, rtol=1e-5, atol=1e-6)
        for _, weights, _, _ in (r[i] for r in res):
            _close(weights, ref_w, TOL)


@pytest.mark.parametrize("include_sparse", [False, True])
@pytest.mark.parametrize("run_option", ["HYBRID", "PS", "MPI"])
def test_global_norm_clip_of_accumulated_gradient(run_option, include_sparse):
    """ClipByGlobalNorm takes the norm of the accumulated gradient: the norm and the update
    equal those of one pass over the same rows (a small max_norm, so every step clips)."""
    spec = dict(run_option=run_option, opt_name="adagrad", clip=0.05,
                include_sparse=include_sparse)
    res = run_distributed(_worker, 2, [dict(spec, K=2), dict(spec, K=4)])
    ref = _train(1, 0, K=None, **spec)
    assert all(n > 0.05 for n in ref[3])
    for i in range(2):
        _check_two_ranks([r[i] for r in res], ref)


def test_bf16_master_rows():
    """sparse_weights="bf16": the stochastic rounding is keyed by step, row and column, so
    accumulated and single-pass updates round alike up to fp32 summation order."""
    spec = dict(run_option="HYBRID", opt_name="adagrad", sparse_weights="bf16")
    res = run_distributed(_worker, 2, [dict(spec, K=2), dict(spec, K=4)])
    ref = _train(1, 0, K=None, **spec)
    for i in range(2):
        _check_two_ranks([r[i] for r in res], ref, tol=(1e-2, 1e-3))


def test_sparse_sum_semantics_and_library_fabric():
    """average_sparse=False (sparse SUM over workers) against K=1 on the same two workers,
    and the library fabric against the single-pass oracle."""
    specs = [dict(run_option="HYBRID", opt_name="adam", K=K, average=False) for K in (1, 4)] + \
        [dict(run_option="HYBRID", opt_name="adagrad", K=2, fabric="library")]
    res = run_distributed(_worker, 2, specs)
    for r in res:
        _close(r[1][1], r[0][1], TOL)
        _close(r[1][2], r[0][2], TOL)
    ref_losses, ref_w = oracle(2, STEPS, make_opt("adagrad"), sparse_scale=1.0)
    for r in res:
        _close(r[2][1], ref_w, TOL)


def test_k1_is_bitwise_the_default():
    a = _train(1, 0, "HYBRID", "adam", None, clip=0.05, include_sparse=True)
    b = _train(1, 0, "HYBRID", "adam", 1, clip=0.05, include_sparse=True)
    assert a[0] == b[0] and a[3] == b[3]
    for n in a[1]:
        assert torch.equal(a[1][n], b[1][n]), n


def test_fetched_loss_is_mean_and_logits_concatenate():
    model = MLPWithEmbedding(VOCAB)
    graph = parallax.Graph(model, optimizer=optim.GradientDescent(0.5))
    cfg = parallax.Config(run_option="HYBRID", sess_config={"micro_batches": 2})
    sess, *_ = parallax.parallel_run(graph, "localhost", parallax_config=cfg)
    ids, labels = make_batch(0, 1)
    halves = [sess.run(["loss", "logits"], {"ids": [ids[k * 4:(k + 1) * 4]],
                                           "labels": [labels[k * 4:(k + 1) * 4]]})
              for k in range(2)]
    loss, logits, _ = sess.run(["loss", "logits", "train_op"],
                               {"ids": [ids], "labels": [labels]})
    assert sess.engine.global_step == 1
    np.testing.assert_allclose(loss[0], np.mean([h[0][0] for h in halves]), rtol=1e-6)
    np.testing.assert_allclose(logits[0], np.concatenate([h[1][0] for h in halves]),
                               rtol=1e-6)
    # fetches without train_op are not split
    full = sess.run(["logits"], {"ids": [ids], "labels": [labels]})
    assert full[0][0].shape == (8, 4)
    sess.close()


class _Counting(MLPWithEmbedding):
    """Returns integer 0-dim counts next to the loss, as the NMT model does."""

    def forward(self, ids, labels):
        out = super().forward(ids, labels)
        out["batch_size"] = torch.tensor(ids.shape[0])
        out["word_count"] = (ids >= 0).sum()
        out["first_is_zero"] = ids[0, 0] == 0
        return out


def test_integer_scalar_outputs_are_summed():
    """Counts add up over the micro-batches (their mean would be neither a count nor
    computable for an integer tensor); the float loss is still the mean, a 0-dim boolean
    is the last micro-batch's value."""
    graph = parallax.Graph(_Counting(VOCAB), optimizer=optim.GradientDescent(0.5))
    cfg = parallax.Config(run_option="HYBRID", sess_config={"micro_batches": 2})
    sess, *_ = parallax.parallel_run(graph, "localhost", parallax_config=cfg)
    ids, labels = make_batch(0, 1)
    ids[4, 0] = 0                       # the last micro-batch's first id
    ids[0, 0] = 1
    bs, wc, first, loss, _ = sess.run(["batch_size", "word_count", "first_is_zero", "loss",
                                       "train_op"], {"ids": [ids], "labels": [labels]})
    assert bs[0] == 8 and wc[0] == ids.numel()
    assert first[0]                     # a 0-dim boolean is the last micro-batch's value
    assert isinstance(loss[0], float)
    sess.close()


def test_indivisible_feed_names_the_placeholder():
    model = MLPWithEmbedding(VOCAB)
    graph = parallax.Graph(model, optimizer=optim.GradientDescent(0.5))
    cfg = parallax.Config(run_option="HYBRID", sess_config={"micro_batches": 3})
    sess, *_ = parallax.parallel_run(graph, "localhost", parallax_config=cfg)
    ids, labels = make_batch(0, 1)
    with pytest.raises(ValueError, match="'ids'.*micro_batches=3"):
        sess.run(["loss", "train_op"], {"ids": [ids], "labels": [labels]})
    assert sess.engine.global_step == 0
    sess.close()


def _build(sess_config, sync=True, protocol=None):
    model = MLPWithEmbedding(VOCAB)
    graph = parallax.Graph(model, optimizer=optim.GradientDescent(0.5))
    cfg = parallax.Config(run_option="HYBRID", sess_config=sess_config)
    if protocol:
        cfg.communication_config = parallax.CommunicationConfig(
            parallax.PSConfig(protocol=protocol))
    return parallax.parallel_run(graph, "localhost", sync=sync, parallax_config=cfg)


@pytest.mark.parametrize("value", [0, -2, 2.0, True, "2", None])
def test_refuses_non_positive_int(value):
    with pytest.raises(ValueError, match="positive int"):
        _build({"micro_batches": value})


def test_refusals_name_the_alternative(monkeypatch):
    """Refused at build, before the fabric allocates anything (the NVLink cases are
    refused on a machine without a GPU, before the fabric would need one)."""
    from parallax_b200.parallel import nvlink_backend

    def no_build(engine):
        raise AssertionError("the fabric was built")
    monkeypatch.setattr(nvlink_backend, "build_nvlink", no_build)
    with pytest.raises(ValueError, match="sync=True"):
        _build({"micro_batches": 2}, sync=False)
    with pytest.raises(ValueError, match="fabric': 'library'"):
        _build({"micro_batches": 2, "fabric": "nvlink", "dense_update": "replicated"})
    with pytest.raises(ValueError, match="fabric': 'library'"):
        _build({"micro_batches": 2, "fabric": "nvlink"}, protocol="nccl")
