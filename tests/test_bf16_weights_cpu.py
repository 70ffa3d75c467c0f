"""bf16 master rows for sparse variables (sess_config["sparse_weights"] = "bf16") without a
GPU: the stochastic rounding and its hash, the host-fabric engine against a plain-torch
oracle that rounds the same way, the placement byte counts, the build-time refusals, fp32 <->
bf16 checkpoint restores, and why round-to-nearest is not enough."""
import math

import pytest
import torch

import parallax_b200 as parallax
from parallax_b200 import optim
from parallax_b200.models.simple import MLPWithEmbedding
from tests.dist_utils import run_distributed

B, T, VOCAB, STEPS = 8, 3, 64, 4


# ------------------------------------------------------------------ the rounding
def _mix_int(x):
    """sr_mix in exact Python integers (the reference for the int64-tensor version)."""
    x ^= x >> 16
    x = (x * 0x7feb352d) % 2 ** 32
    x ^= x >> 15
    x = (x * 0x846ca68b) % 2 ** 32
    return x ^ (x >> 16)


def _sr(x, seed=0x1234567, step=3, gids=None):
    x = x.reshape(-1, 1) if x.dim() == 1 else x
    gids = torch.arange(x.shape[0]) if gids is None else gids
    return optim.round_bf16_stochastic(x, seed, step, gids)


def test_hash_matches_exact_integers():
    g = torch.Generator().manual_seed(0)
    xs = torch.randint(0, 2 ** 32, (4096,), generator=g, dtype=torch.int64)
    xs[:4] = torch.tensor([0, 1, 2 ** 32 - 1, 2 ** 31])
    got = optim.sr_mix(xs)
    assert got.tolist() == [_mix_int(int(v)) for v in xs]
    assert optim.sr_mix(12345) == _mix_int(12345)


def test_representable_values_unchanged():
    g = torch.Generator().manual_seed(1)
    x = torch.randn(1000, 7, generator=g).to(torch.bfloat16).float()
    x[0, :3] = torch.tensor([0.0, -0.0, 2.0 ** -133])
    out = _sr(x)
    assert torch.equal(out.float(), x)
    assert torch.equal(out.view(torch.int16), x.to(torch.bfloat16).view(torch.int16))


def test_output_is_a_bf16_neighbour():
    g = torch.Generator().manual_seed(2)
    x = torch.randn(2000, 16, generator=g) * torch.logspace(-20, 20, 16)
    out = _sr(x)
    bits = x.view(torch.int32).to(torch.int64) & 0xffffffff
    down = ((bits >> 16) & 0xffff)
    got = out.view(torch.int16).to(torch.int64) & 0xffff
    assert bool(((got == down) | (got == down + 1)).all())
    # exactly representable -> no move; otherwise both neighbours occur
    assert bool((got == down).any()) and bool((got == down + 1).any())


def test_mean_is_unbiased():
    """2^16 keys (global ids) rounding the same value: the mean is within 4 sigma of it."""
    for v in (1.0 + 2 ** -9, -3.3, 1e-30, 123456.7):
        x32 = torch.tensor(v, dtype=torch.float32)
        down = float(x32.view(torch.int32).bitwise_and(-65536).view(torch.float32))
        ulp = 2.0 ** (math.floor(math.log2(abs(float(x32)))) - 7)
        frac = abs(float(x32) - down) / ulp
        x = torch.full((1 << 16, 1), float(x32))
        mean = float(_sr(x).double().mean())
        sigma = ulp * math.sqrt(frac * (1 - frac) / x.shape[0])
        assert abs(mean - float(x32)) <= 4 * sigma + 1e-9 * ulp, (v, mean)


def test_same_key_same_result_and_keys_matter():
    g = torch.Generator().manual_seed(3)
    x = torch.randn(512, 64, generator=g)
    gids = torch.randint(0, 10 ** 6, (512,), generator=g)
    a = optim.round_bf16_stochastic(x, 7, 11, gids)
    assert torch.equal(a.view(torch.int16), optim.round_bf16_stochastic(x, 7, 11, gids)
                       .view(torch.int16))
    for other in (optim.round_bf16_stochastic(x, 8, 11, gids),
                  optim.round_bf16_stochastic(x, 7, 12, gids),
                  optim.round_bf16_stochastic(x, 7, 11, gids + 1)):
        assert not torch.equal(a.view(torch.int16), other.view(torch.int16))


def test_inf_and_nan_pass_through():
    nan_low = torch.tensor([0x7f800001], dtype=torch.int32).view(torch.float32)   # low bits only
    x = torch.cat([torch.tensor([float("inf"), -float("inf"), float("nan"), -float("nan")]),
                   nan_low, -nan_low])
    out = _sr(x).float().view(-1)
    assert out[0] == float("inf") and out[1] == -float("inf")
    assert bool(out[2:].isnan().all())


def test_sr_seed_is_a_stable_function_of_the_name():
    assert optim.sr_seed("emb.weight") == optim.sr_seed("emb.weight")
    assert optim.sr_seed("emb.weight") != optim.sr_seed("softmax_w.weight")
    assert 0 <= optim.sr_seed("x") < 2 ** 32


def test_drift_sgd_stochastic_vs_nearest():
    """1000 SGD updates of 2^-12 on weights of 1.0 (bf16 ulp below 1.0 is 2^-8, above 2^-7):
    stochastic rounding reaches 1 - 1000 * 2^-12 in expectation, round-to-nearest never
    moves."""
    n, steps, upd = 1 << 14, 1000, 2.0 ** -12
    w_sr = torch.ones(n, 1).to(torch.bfloat16)
    w_rn = torch.ones(n, 1).to(torch.bfloat16)
    gids = torch.arange(n)
    for s in range(1, steps + 1):
        w_sr = optim.round_bf16_stochastic(w_sr.float() - upd, 99, s, gids)
        w_rn = (w_rn.float() - upd).to(torch.bfloat16)           # round to nearest even
    want = 1.0 - steps * upd
    # each step adds at most one rounding of variance ulp^2 / 4 (ulp = 2^-8 below 1.0)
    sigma = math.sqrt(steps * (2.0 ** -8) ** 2 / 4 / n)
    assert abs(float(w_sr.double().mean()) - want) <= 4 * sigma
    assert bool((w_rn.float() == 1.0).all())


# ------------------------------------------------------------------ placement bytes
def test_table_row_bytes():
    bf = torch.bfloat16
    assert optim.table_row_bytes("adagrad", 512) == 4096
    assert optim.table_row_bytes("adagrad", 512, bf) == 3072
    assert optim.table_row_bytes("adam", 64, bf) == 640
    assert optim.table_row_bytes("adam", 64) == 768
    assert optim.table_row_bytes("rowwise_adagrad", 64, bf) == 132
    assert optim.table_row_bytes("rowwise_adagrad", 64) == 260
    assert optim.table_row_bytes("sgd", 1, bf) == 16            # one 8-column bf16 row
    assert optim.table_row_bytes("sgd", 1) == 16
    assert optim.table_row_bytes("adagrad", 500, bf) == 2 * 504 + 4 * 500


# ------------------------------------------------------------- engine vs oracle
def make_batch(step, world, rank=None):
    g = torch.Generator().manual_seed(700 + step)
    ids = torch.randint(0, VOCAB, (B * world, T), generator=g)
    ids[:, 0] = ids[0, 0]
    labels = torch.randint(0, 4, (B * world,), generator=g)
    if rank is None:
        return ids, labels
    return ids[rank * B:(rank + 1) * B], labels[rank * B:(rank + 1) * B]


def dense_opt():
    return optim.Adagrad(0.3, 0.5)


def sparse_opt(kind):
    return optim.RowWiseAdagrad(0.3, 0.5, epsilon=1e-3) if kind == "rowwise" else \
        optim.Adagrad(0.3, 0.5)


def oracle(world, max_norm, kind):
    """Single-device training on the concatenated batch: the embedding's master is a bf16
    tensor, every update is applied in fp32 on the widened rows and rounded with
    `round_bf16_stochastic` (seed of "emb.weight", the step, the rows' ids)."""
    torch.manual_seed(0)
    model = MLPWithEmbedding(VOCAB)
    model.emb.sparse = False
    named = dict(model.named_parameters())
    dopt, sopt = dense_opt(), sparse_opt(kind)
    master = named["emb.weight"].detach().to(torch.bfloat16)
    with torch.no_grad():
        named["emb.weight"].copy_(master.float())
    slots = {n: tuple(torch.full_like(p, v) for v in dopt.slot_init()) for n, p in named.items()}
    slots["emb.weight"] = tuple(torch.full((VOCAB, optim.slot_width(sopt.kind, master.shape[1])), v)
                                for v in sopt.slot_init())
    seed = optim.sr_seed("emb.weight")
    for s in range(STEPS):
        ids, labels = make_batch(s, world)
        out = model(ids, labels)
        model.zero_grad()
        out["loss"].backward()
        grads = {n: p.grad.clone() for n, p in named.items()}
        grads["emb.weight"] *= world
        if max_norm is not None:
            norm = math.sqrt(sum(float((g.double() ** 2).sum()) for g in grads.values()))
            scale = max_norm / max(norm, max_norm)
            grads = {n: g * scale for n, g in grads.items()}
        with torch.no_grad():
            for n, p in named.items():
                if n == "emb.weight":
                    rows = torch.unique(ids.reshape(-1))
                    optim.apply_sparse_rows_(sopt.kind, master, rows, grads[n][rows],
                                             slots[n], sopt.hyper(s + 1), seed, rows)
                    p.copy_(master.float())
                else:
                    optim.apply_dense_(dopt.kind, p.data, grads[n], slots[n], dopt.hyper(s + 1))
    return {n: p.detach().clone() for n, p in named.items()}


def train(world, rank, run_option, max_norm, kind, nparts=3):
    torch.manual_seed(0)
    model = MLPWithEmbedding(VOCAB, partitioner=parallax.get_partitioner(nparts))
    rules = [parallax.ClipByGlobalNorm(max_norm, include_sparse=True)] \
        if max_norm is not None else []
    graph = parallax.Graph(model, optimizer=dense_opt(), sparse_optimizer=sparse_opt(kind),
                           grad_rules=rules)
    cfg = parallax.Config(run_option=run_option, search_partitions=False,
                          sess_config={"fabric": "host", "sparse_weights": "bf16"})
    sess, *_ = parallax.parallel_run(graph, "localhost", parallax_config=cfg)
    try:
        tab = sess.engine.tables["emb.weight"]
        assert tab.shard.dtype == torch.bfloat16
        assert all(s.dtype == torch.float32 for s in tab.slots)
        for s in range(STEPS):
            ids, labels = make_batch(s, world, rank if world > 1 else None)
            sess.run(["loss", "train_op"], {"ids": [ids], "labels": [labels]})
        sd = sess.engine.state_dict()
    finally:
        sess.close()
    weights = dict(sd["dense"]["master"])
    weights["emb.weight"] = sd["sparse"]["emb.weight"]["weight"]
    return weights


def _compare(got, want):
    for n, w in want.items():
        g = got[n].view_as(w)
        if n == "emb.weight":
            # bf16 values; an fp32 sum taken in another order may round the other way
            assert torch.equal(g, g.to(torch.bfloat16).float())
            ulp = 2.0 ** (torch.floor(torch.log2(w.abs().clamp_min(1e-30))) - 7)
            assert bool(((g - w).abs() <= ulp).all())
            assert float((g != w).float().mean()) < 0.01
        else:
            torch.testing.assert_close(g, w, rtol=2e-3, atol=2e-4)


@pytest.mark.parametrize("run_option", ["HYBRID", "PS", "MPI"])
@pytest.mark.parametrize("max_norm", [None, 0.05])
@pytest.mark.parametrize("kind", ["adagrad", "rowwise"])
def test_host_engine_matches_oracle(run_option, max_norm, kind):
    _compare(train(1, 0, run_option, max_norm, kind), oracle(1, max_norm, kind))


def _worker(rank, world, run_option, max_norm, kind):
    return train(world, rank, run_option, max_norm, kind)


@pytest.mark.parametrize("run_option,max_norm", [
    ("HYBRID", None), ("PS", 0.05), ("MPI", 0.05), ("MPI", None)])
def test_host_engine_two_ranks(run_option, max_norm):
    res = run_distributed(_worker, 2, run_option, max_norm, "adagrad")
    want = oracle(2, max_norm, "adagrad")
    for got in res:
        _compare(got, want)
    # every replica and every owner rounds alike: both ranks hold the same logical table
    assert torch.equal(res[0]["emb.weight"], res[1]["emb.weight"])


def test_lookups_return_the_bf16_values_widened():
    torch.manual_seed(0)
    model = MLPWithEmbedding(VOCAB, partitioner=parallax.get_partitioner(3))
    w0 = model.emb.weight.detach().clone()
    graph = parallax.Graph(model, optimizer=dense_opt(), sparse_optimizer=sparse_opt("adagrad"))
    sess, *_ = parallax.parallel_run(graph, "localhost", parallax_config=parallax.Config(
        search_partitions=False, sess_config={"fabric": "host", "sparse_weights": "bf16"}))
    try:
        tab = sess.engine.tables["emb.weight"]
        rows, _ = tab.lookup(torch.arange(VOCAB))
        assert rows.dtype == torch.float32
        assert torch.equal(rows, w0.to(torch.bfloat16).float())
        assert torch.equal(tab.full_weight(), w0.to(torch.bfloat16).float())
    finally:
        sess.close()


# -------------------------------------------------------------------- refusals
def _run(sess_config, sync=True):
    graph = parallax.Graph(MLPWithEmbedding(VOCAB), optimizer=dense_opt(),
                           sparse_optimizer=sparse_opt("adagrad"))
    sess, *_ = parallax.parallel_run(graph, "localhost", sync=sync,
                                     parallax_config=parallax.Config(
                                         search_partitions=False, sess_config=sess_config))
    sess.close()


@pytest.mark.parametrize("value", ["fp16", "float32", True, None])
def test_unknown_value_refused(value):
    with pytest.raises(ValueError, match="sparse_weights"):
        _run({"fabric": "host", "sparse_weights": value})


def test_async_refused():
    with pytest.raises(ValueError, match="sync=True"):
        _run({"fabric": "host", "sparse_weights": "bf16"}, sync=False)


@pytest.mark.parametrize("cdt", [None, "float32"])
def test_nvlink_needs_bf16_lookups(cdt):
    """Refused before the fabric is built: this machine needs no GPU to see the error."""
    sc = {"fabric": "nvlink", "sparse_weights": "bf16"}
    if cdt is not None:
        sc["compute_dtype"] = cdt
    with pytest.raises(ValueError, match="compute_dtype"):
        _run(sc)


def test_fp32_default_unchanged():
    _run({"fabric": "host", "sparse_weights": "fp32"})
    _run({"fabric": "host"})


# ------------------------------------------------------------------ checkpoints
def _session(weights, seed=0):
    torch.manual_seed(seed)
    model = MLPWithEmbedding(VOCAB, partitioner=parallax.get_partitioner(3))
    graph = parallax.Graph(model, optimizer=dense_opt(), sparse_optimizer=sparse_opt("adagrad"))
    sess, *_ = parallax.parallel_run(graph, "localhost", parallax_config=parallax.Config(
        search_partitions=False, sess_config={"fabric": "host", "sparse_weights": weights}))
    return sess


def test_checkpoint_fp32_bf16_round_trip():
    """fp32 state into a bf16 table rounds to nearest even; bf16 state into an fp32 table
    is exact; slots stay fp32 both ways."""
    src = _session("fp32")
    try:
        for s in range(2):
            ids, labels = make_batch(s, 1)
            src.run(["loss", "train_op"], {"ids": [ids], "labels": [labels]})
        sd32 = src.engine.state_dict()
    finally:
        src.close()
    dst = _session("bf16", seed=1)
    try:
        dst.engine.load_state_dict(sd32)
        sd16 = dst.engine.state_dict()
    finally:
        dst.close()
    w32 = sd32["sparse"]["emb.weight"]["weight"]
    assert torch.equal(sd16["sparse"]["emb.weight"]["weight"], w32.to(torch.bfloat16).float())
    torch.testing.assert_close(sd16["sparse"]["emb.weight"]["slots"][0],
                               sd32["sparse"]["emb.weight"]["slots"][0], rtol=0, atol=0)
    back = _session("fp32", seed=2)
    try:
        back.engine.load_state_dict(sd16)
        sd = back.engine.state_dict()
    finally:
        back.close()
    assert torch.equal(sd["sparse"]["emb.weight"]["weight"], sd16["sparse"]["emb.weight"]["weight"])
