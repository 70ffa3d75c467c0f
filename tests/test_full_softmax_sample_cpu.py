"""`parallax.nn.full_softmax_sample` without a GPU: the torch noise against a pure-Python
reimplementation, the composition against an fp64 Gumbel-top-k, the distribution of the draws,
their independence of the partitioning and the world size, the argument checks, LM1B's
`eval_sample` outputs and `lm1b_generate.py` end to end."""
import itertools
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from scipy import stats

import parallax_b200 as parallax
import parallax_b200.nn as pnn
from parallax_b200.models.lm1b import LM1B, lm1b_graph
from parallax_b200.parallel.engine import sample_log_e, sample_uniform
from parallax_b200.partitions import FixedSizePartitioner

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
V = 301
M32 = 0xffffffff


# ------------------------------------------------------------------ noise
def _mix(x):
    x ^= x >> 16
    x = (x * 0x7feb352d) & M32
    x ^= x >> 15
    x = (x * 0x846ca68b) & M32
    return x ^ (x >> 16)


def _v_python(seed, row, gid):
    """(h, v) in exact Python integers and numpy fp32 scalars"""
    h = _mix(_mix(_mix(seed) ^ row) ^ gid)
    v = np.float32(h) * np.float32(2.0 ** -32) + np.float32(2.0 ** -33)
    return h, min(v, np.float32(1.0 - 2.0 ** -24))


def test_noise_matches_python_bit_for_bit():
    rows = torch.tensor([0, 1, 2, 1000, 123456, M32 - 1, M32], dtype=torch.int64)
    gids = torch.cat([torch.arange(200), torch.tensor([793469, 2 ** 31 - 1, M32])])
    for seed in (0, 1, 0xdeadbeef, M32):
        v = sample_uniform(seed, rows, gids)
        assert v.dtype == torch.float32 and v.shape == (rows.numel(), gids.numel())
        want = np.array([[_v_python(seed, int(r), int(g))[1] for g in gids] for r in rows],
                        dtype=np.float32)
        assert np.array_equal(v.numpy().view(np.uint32), want.view(np.uint32)), seed
        assert (v > 0).all() and (v < 1).all()
        le = sample_log_e(seed, rows, gids)
        assert torch.isfinite(le).all()
    # the clamp: h rounds up to 2^32 in fp32 for the largest hashes
    assert _v_python(0, 0, 0)[1] < 1


# ------------------------------------------------------------------ composition vs fp64
def _session(eval_sample=0, train=(), temperature=1.0, num_shards=3):
    torch.manual_seed(0)
    m = LM1B(vocab_size=V, emb_size=16, state_size=32, projected_size=16, num_sampled=0,
             num_steps=4, num_shards=num_shards, keep_prob=1.0, eval_sample=eval_sample,
             sample_temperature=temperature)
    sess, *_ = parallax.parallel_run(lm1b_graph(m, batch_size=8), "localhost",
                                     parallax_config=parallax.Config(
                                         sess_config={"fabric": "host"}))
    for feeds in train:
        sess.run(["loss", "train_op"], feeds)
    return sess, m


def _batch(seed):
    x = torch.randint(0, V, (8, 4), generator=torch.Generator().manual_seed(seed))
    return {"x": [x], "y": [torch.roll(x, -1, dims=1)]}


@pytest.fixture(scope="module")
def lm1b():
    sess, m = _session(train=[_batch(0), _batch(1)])
    yield sess, m
    sess.close()


def _fp64_gumbel(inputs, weight, bias, tau, seed):
    """fp64 tempered log-probabilities [N, V] and keys [N, V] from the same uniforms"""
    ids = torch.arange(weight.num_embeddings)
    w, b = pnn.lookup_many([weight, bias], ids)
    s = (inputs.double() @ w.double().t() + b.double().t()) / tau
    v = sample_uniform(seed, torch.arange(inputs.shape[0]), ids).double()
    keys = s - torch.log(-torch.log1p(-v))
    return torch.log_softmax(s, dim=-1), keys


@pytest.mark.parametrize("n,tau", [(1, 1.0), (5, 0.7), (32, 1.5), (40, 1.0)])
def test_composition_matches_fp64_gumbel_top_k(lm1b, n, tau):
    sess, m = lm1b
    seed = 1000 + n
    inputs = torch.randn(37, 16, generator=torch.Generator().manual_seed(n))
    with torch.no_grad():
        lp, ids = pnn.full_softmax_sample(inputs, m.softmax_w, m.softmax_b, n, tau, seed)
    assert lp.shape == (37, n) and lp.dtype == torch.float32
    assert ids.shape == (37, n) and ids.dtype == torch.int64
    ref_lp, keys = _fp64_gumbel(inputs, m.softmax_w, m.softmax_b, tau, seed)
    assert ((ids >= 0) & (ids < V)).all()
    assert all(len(set(r)) == n for r in ids.tolist())
    torch.testing.assert_close(lp.double(), ref_lp.gather(1, ids), rtol=0, atol=1e-5)
    k = keys.gather(1, ids)
    assert (k[:, 1:] <= k[:, :-1] + 1e-5).all()           # draw order: keys descending
    order = torch.sort(keys, dim=1, descending=True, stable=True).indices
    srt = keys.gather(1, order[:, :n + 1])
    d = srt[:, :-1] - srt[:, 1:]
    ok = d[:, :n] > 1e-4
    ok[:, 1:] &= d[:, :n - 1] > 1e-4
    assert ok.float().mean() > 0.5
    assert torch.equal(ids[ok], order[:, :n][ok])


def test_gradients_flow_into_log_probs(lm1b):
    sess, m = lm1b
    inputs = torch.randn(5, 16, requires_grad=True)
    lp, _ = pnn.full_softmax_sample(inputs, m.softmax_w, m.softmax_b, 3, 0.8, 5)
    lp.sum().backward()
    assert inputs.grad is not None and torch.isfinite(inputs.grad).all()
    assert inputs.grad.abs().sum() > 0


# ------------------------------------------------------------------ distribution
def _tabled(logits):
    """(weight, bias) embeddings and one input row whose logits are `logits` [V]"""
    Vn = logits.numel()
    w, b = torch.nn.Embedding(Vn, 1), torch.nn.Embedding(Vn, 1)
    with torch.no_grad():
        w.weight.copy_(logits[:, None])
        b.weight.zero_()
    return w, b


@pytest.mark.parametrize("tau", [0.5, 1.0, 2.0])
def test_first_draws_follow_the_tempered_softmax(tau):
    Vn, N = 50, 200000
    logits = torch.randn(Vn, generator=torch.Generator().manual_seed(4)) * 1.5
    w, b = _tabled(logits)
    x = torch.ones(N, 1)
    _, ids = pnn.full_softmax_sample(x, w, b, 1, tau, 77)
    p = torch.softmax(logits.double() / tau, 0).numpy()
    cnt = np.bincount(ids[:, 0].numpy(), minlength=Vn)
    big = p * N >= 5                             # pool the rare ids into one cell
    obs = np.append(cnt[big], cnt[~big].sum())
    exp = np.append(p[big] * N, p[~big].sum() * N)
    keep = exp > 0
    assert stats.chisquare(obs[keep], exp[keep]).pvalue > 1e-4


@pytest.mark.parametrize("tau", [0.5, 1.0, 2.0])
def test_pairwise_inclusion_matches_sampling_without_replacement(tau):
    Vn, N, n = 50, 200000, 3
    logits = torch.randn(Vn, generator=torch.Generator().manual_seed(5)) * 1.5
    w, b = _tabled(logits)
    _, ids = pnn.full_softmax_sample(torch.ones(N, 1), w, b, n, tau, 78)
    assert all(len(set(r)) == n for r in ids[:1000].tolist())
    p = torch.softmax(logits.double() / tau, 0).numpy()
    # exact P(i and j among the 3 draws): sum over the ordered triples that contain both
    incl = np.zeros((Vn, Vn))
    for a, bb, c in itertools.permutations(range(Vn), 3):
        pr = p[a] * p[bb] / (1 - p[a]) * p[c] / (1 - p[a] - p[bb])
        incl[a, bb] += pr
        incl[a, c] += pr
        incl[bb, c] += pr
    incl = incl + incl.T
    got = np.zeros((Vn, Vn))
    s = ids.numpy()
    for u, v in ((0, 1), (0, 2), (1, 2)):
        np.add.at(got, (s[:, u], s[:, v]), 1)
    got = (got + got.T) / N
    iu = np.triu_indices(Vn, 1)
    sd = np.sqrt(incl[iu] * (1 - incl[iu]) / N)
    assert abs(incl[iu].sum() - 3.0) < 1e-9             # 3 pairs per draw
    assert (np.abs(got[iu] - incl[iu]) <= 5 * sd + 2.0 / N).all()


# ------------------------------------------------------------------ path independence
class _Head(torch.nn.Module):
    co_lookup_groups = [("w", "b")]

    def __init__(self, P, strategy):
        super().__init__()
        part = FixedSizePartitioner(P, strategy)
        self.w = pnn.Embedding(V, 16, partitioner=part, seed=11)
        self.b = pnn.Embedding(V, 1, partitioner=part, seed=12)
        self.lin = torch.nn.Linear(16, 16)

    def forward(self, x):
        with torch.no_grad():
            lp, ids = pnn.full_softmax_sample(x, self.w, self.b, 6, 0.9, 2024)
        return {"loss": self.lin(x).sum(), "ids": ids, "lp": lp}


def _draw(world=1, rank=0, P=3, strategy="mod"):
    torch.manual_seed(0)
    graph = parallax.Graph(_Head(P, strategy), optimizer=parallax.optim.Adagrad(0.1, 1.0))
    sess, nw, wid, _ = parallax.parallel_run(graph, "localhost", parallax_config=parallax.Config(
        sess_config={"fabric": "host"}))
    assert (nw, wid) == (world, rank)
    x = torch.randn(23, 16, generator=torch.Generator().manual_seed(1))
    sess.engine.model.eval()
    ids, lp = sess.run(["ids", "lp"], {"x": [x]})
    sess.close()
    return torch.as_tensor(ids[0]), torch.as_tensor(lp[0])


def _worker(rank, world):
    return _draw(world, rank)


def test_same_seed_same_draws_across_partitionings_and_world_sizes():
    from tests.dist_utils import run_distributed
    ref_ids, ref_lp = _draw()
    for P, strategy in itertools.product((1, 3, 7), ("mod", "div")):
        ids, lp = _draw(P=P, strategy=strategy)
        assert torch.equal(ids, ref_ids), (P, strategy)
        torch.testing.assert_close(lp, ref_lp, rtol=0, atol=1e-6)
    for ids, lp in run_distributed(_worker, 2):
        assert torch.equal(ids, ref_ids)


def test_seed_none_differs_between_calls(lm1b):
    sess, m = lm1b
    x = torch.randn(64, 16)
    with torch.no_grad():
        a = pnn.full_softmax_sample(x, m.softmax_w, m.softmax_b, 4)[1]
        b = pnn.full_softmax_sample(x, m.softmax_w, m.softmax_b, 4)[1]
        c = pnn.full_softmax_sample(x, m.softmax_w, m.softmax_b, 4, seed=9)[1]
        d = pnn.full_softmax_sample(x, m.softmax_w, m.softmax_b, 4, seed=9)[1]
    assert not torch.equal(a, b)
    assert torch.equal(c, d)


def test_argument_validation(lm1b):
    sess, m = lm1b
    x = torch.randn(5, 16)
    fs = pnn.full_softmax_sample
    for n in (0, -1, V + 1, True, False, 2.0, "3", None):
        with pytest.raises(ValueError, match="num_samples must be"):
            fs(x, m.softmax_w, m.softmax_b, n)
    for t in (0, 0.0, -1.0, float("inf"), float("nan"), True, "1", None, 1e-50):
        with pytest.raises(ValueError, match="temperature"):
            fs(x, m.softmax_w, m.softmax_b, 2, t)
    for s in (-1, 1 << 32, 1.0, True, "7"):
        with pytest.raises(ValueError, match="seed must be"):
            fs(x, m.softmax_w, m.softmax_b, 2, 1.0, s)
    with pytest.raises(ValueError, match="inputs must be"):
        fs(x.reshape(5, 4, 4), m.softmax_w, m.softmax_b)
    with pytest.raises(ValueError, match="columns"):
        fs(torch.randn(5, 8), m.softmax_w, m.softmax_b)
    with pytest.raises(ValueError, match="bias must be"):
        fs(x, m.softmax_w, m.softmax_w)
    fs(x, m.softmax_w, m.softmax_b, V, 2, np.uint32(M32))   # the bounds themselves are accepted


# ------------------------------------------------------------------ LM1B
def _eval(sess, m, fetches, feeds):
    m.eval()
    try:
        return sess.run(fetches, feeds)
    finally:
        m.train()


def test_lm1b_eval_sample_outputs(monkeypatch):
    seen = {}
    orig = pnn.full_softmax_sample

    def sample(inputs, w, b, n, tau, seed):
        seen["args"] = (n, tau, seed)
        seen["out"] = orig(inputs, w, b, n, tau, seed)
        return seen["out"]
    monkeypatch.setattr(pnn, "full_softmax_sample", sample)
    sess, m = _session(eval_sample=3, temperature=0.8)
    sess.run(["loss", "train_op"], _batch(0))
    assert "args" not in seen                      # training: no samples
    ids, lp = _eval(sess, m, ["sample_ids", "sample_log_probs"], dict(_batch(2), sample_seed=[5]))
    ids, lp = torch.as_tensor(ids[0]), torch.as_tensor(lp[0])
    assert seen["args"] == (3, 0.8, 5)
    assert ids.shape == (8, 4, 3) and ids.dtype == torch.int64 and lp.shape == (8, 4, 3)
    # rows of the op are time-major (t, b); the outputs are batch-major like x
    assert torch.equal(ids, seen["out"][1].reshape(4, 8, 3).transpose(0, 1))
    assert torch.equal(lp, seen["out"][0].reshape(4, 8, 3).transpose(0, 1))
    # y = None: no loss and no NLL pass; the same samples
    calls = []
    monkeypatch.setattr(pnn, "full_softmax_nll", lambda *a: calls.append(1))
    m.eval()
    try:
        out = sess.engine.eval_step({"x": _batch(2)["x"][0], "sample_seed": 5})
        ids2 = sess.run("sample_ids", {"x": _batch(2)["x"], "sample_seed": [5]})[0]
    finally:
        m.train()
    assert calls == [] and "loss" not in out
    assert set(out) == {"final_state_c", "final_state_h", "sample_ids", "sample_log_probs"}
    assert torch.equal(out["sample_ids"], ids) and torch.equal(torch.as_tensor(ids2), ids)
    with pytest.raises(ValueError, match="needs targets"):
        sess.engine.forward({"x": _batch(2)["x"][0]})
    sess.close()


def test_eval_sample_zero_leaves_the_outputs_unchanged():
    outs = []
    for n in (0, 2):
        sess, m = _session(eval_sample=n)
        train = sess.run(["loss", "train_op"], _batch(0))[0][0]
        m.eval()
        try:
            out = sess.engine.forward({"x": _batch(5)["x"][0], "y": _batch(5)["y"][0]})
        finally:
            m.train()
        outs.append((train, out))
        sess.close()
    (t0, o0), (t2, o2) = outs
    assert float(t0) == float(t2)
    assert list(o0) == ["loss", "final_state_c", "final_state_h"]
    assert set(o2) == set(o0) | {"sample_ids", "sample_log_probs"}
    for key in o0:
        assert torch.equal(o0[key], o2[key]), key


# ------------------------------------------------------------------ generation script
def test_generate_from_a_trained_tiny_checkpoint(tmp_path):
    env = {k: v for k, v in os.environ.items()
           if not k.startswith("PARALLAX_") and k not in ("RANK", "WORLD_SIZE", "LOCAL_RANK")}
    env.update(PARALLAX_FABRIC="host", CUDA_VISIBLE_DEVICES="", OMP_NUM_THREADS="2")
    ck = str(tmp_path / "ck")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "examples/lm1b/lm1b_distributed_driver.py"),
                        "--use_synthetic", "--tiny", "--max_steps", "4", "--ckpt_dir", ck,
                        "--save_ckpt_steps", "4", "--logdir", str(tmp_path / "log")],
                       env=env, cwd=str(tmp_path), capture_output=True, text=True, timeout=400)
    assert r.returncode == 0, r.stderr[-1500:]

    def generate(seed, extra=()):
        r = subprocess.run([sys.executable, os.path.join(ROOT, "examples/lm1b/lm1b_generate.py"),
                            "--use_synthetic", "--tiny", "--ckpt_dir", ck, "--prefix", "5 17",
                            "--num_words", "7", "--num_sequences", "3", "--seed", str(seed)]
                           + list(extra), env=env, cwd=str(tmp_path), capture_output=True,
                           text=True, timeout=400)
        assert r.returncode == 0, r.stderr[-1500:]
        assert "global_step 4" in r.stderr + r.stdout
        return r.stdout.strip().splitlines()[-3:]
    a, b, c = generate(1), generate(1), generate(2, ["--temperature", "0.7", "--use_ema"])
    for lines in (a, c):
        for line in lines:
            words = line.split()
            assert words[:2] == ["5", "17"] and len(words) == 2 + 7
            assert all(0 <= int(w) < 10000 for w in words)
    assert a == b and a != c
