"""Truncated sampling (`parallax.nn.full_softmax_sample(..., top_k=, top_p=)`) without a GPU: the
composition against an fp64 oracle of the truncation predicate, the distribution of the
draws against the softmax renormalised on the kept set, their independence of the partitioning,
the argument checks, LM1B's `sample_top_k` / `sample_top_p` and `lm1b_generate.py --top_p`."""
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
from parallax_b200.parallel.engine import _gathered_logits, _ordered_top, sample_log_e
from parallax_b200.partitions import FixedSizePartitioner

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
V = 301


def _kept(s, n, top_k=None, top_p=None):
    """bool [N, V]: each row's T by the definition, in fp64, one candidate θ at a time: the
    row's distinct values, largest first, until count(θ) >= top_k or (mass(θ) >= top_p and
    count(θ) >= n)."""
    s = np.asarray(s, dtype=np.float64)
    out = np.ones(s.shape, dtype=bool)
    for i, row in enumerate(s):
        q = np.exp(row - row.max())
        q /= q.sum()
        for th in np.unique(row)[::-1]:
            sel = row >= th
            c, m = int(sel.sum()), float(q[sel].sum())
            if (top_k is not None and c >= top_k) or (top_p is not None and m >= top_p and
                                                      c >= n):
                out[i] = sel
                break
    return torch.from_numpy(out)


def _embeddings(Vn, K, seed, dup=0):
    """(weight, bias) torch embeddings; with dup > 0 the first dup rows repeat rows dup..2·dup,
    so every input row has tied logits"""
    g = torch.Generator().manual_seed(seed)
    w, b = torch.nn.Embedding(Vn, K), torch.nn.Embedding(Vn, 1)
    with torch.no_grad():
        w.weight.copy_(torch.randn(Vn, K, generator=g))
        b.weight.copy_(torch.randn(Vn, 1, generator=g))
        if dup:
            w.weight[:dup] = w.weight[dup:2 * dup]
            b.weight[:dup] = b.weight[dup:2 * dup]
    return w, b


def _inv(tau):
    return float(torch.tensor(1.0 / tau, dtype=torch.float32))


@pytest.mark.parametrize("n,top_k,top_p,tau", [
    (1, 5, None, 1.0),
    (5, 5, None, 0.7),           # n = top_k
    (3, V, None, 1.0),           # top_k = V: every word
    (1, None, 0.9, 1.0),
    (8, None, 0.05, 1.0),        # the n floor: the nucleus alone is smaller than n
    (2, 10, 0.7, 1.5),           # both: the smaller set
    (4, 40, 0.95, 0.7),
])
def test_composition_matches_the_fp64_predicate(n, top_k, top_p, tau):
    N, K, seed = 29, 8, 77
    w, b = _embeddings(V, K, 3, dup=40)
    x = torch.randn(N, K, generator=torch.Generator().manual_seed(n))
    lp, ids = pnn.full_softmax_sample(x, w, b, n, tau, seed, top_k=top_k, top_p=top_p)
    assert lp.shape == (N, n) and ids.shape == (N, n) and ids.dtype == torch.int64
    with torch.no_grad():
        s = _gathered_logits(x, w, b) * _inv(tau)
    keep = _kept(s, n, top_k, top_p)
    assert (keep.sum(1) >= n).all()
    if top_k is not None and top_p is None:
        assert (keep.sum(1) >= top_k).all()
    # ties: tied words are kept or dropped together
    assert torch.equal(keep[:, :40], keep[:, 40:80])
    # the draws: the untruncated keys' order filtered to T, and untruncated log-probabilities
    keys = s - sample_log_e(seed, torch.arange(N), torch.arange(V))
    assert torch.equal(ids, _ordered_top(keys.masked_fill(~keep, -float("inf")), n))
    assert keep.gather(1, ids).all()
    torch.testing.assert_close(lp, torch.log_softmax(s, -1).gather(1, ids), rtol=0, atol=1e-6)
    if top_k == V:
        lp0, ids0 = pnn.full_softmax_sample(x, w, b, n, tau, seed)
        assert torch.equal(ids, ids0) and torch.equal(lp, lp0)


def test_top_p_one_is_the_untruncated_call():
    w, b = _embeddings(V, 8, 4)
    x = torch.randn(11, 8)
    a = pnn.full_softmax_sample(x, w, b, 3, 0.8, 5, top_p=1.0)
    c = pnn.full_softmax_sample(x, w, b, 3, 0.8, 5)
    assert torch.equal(a[0], c[0]) and torch.equal(a[1], c[1])


def test_truncation_changes_only_the_kept_set():
    """a truncated draw is the untruncated draw order filtered to T: with n = |T| words kept
    (top_k alone, no ties), the ids are T in the untruncated draw order"""
    w, b = _embeddings(V, 8, 5)
    x = torch.randn(7, 8)
    _, full = pnn.full_softmax_sample(x, w, b, V, 1.0, 9)
    _, top = pnn.full_softmax_sample(x, w, b, 6, 1.0, 9, top_k=6)
    with torch.no_grad():
        keep = _kept(_gathered_logits(x, w, b), 6, top_k=6)
    for r in range(7):
        order = [i for i in full[r].tolist() if keep[r, i]]
        assert top[r].tolist() == order


# ------------------------------------------------------------------ distribution
@pytest.mark.parametrize("tau,top_k,top_p", [(0.7, 10, None), (1.0, None, 0.8), (1.5, 12, 0.9)])
def test_first_draws_follow_the_truncated_softmax(tau, top_k, top_p):
    Vn, N = 50, 200000
    logits = torch.randn(Vn, generator=torch.Generator().manual_seed(4)) * 1.5
    w, b = torch.nn.Embedding(Vn, 1), torch.nn.Embedding(Vn, 1)
    with torch.no_grad():
        w.weight.copy_(logits[:, None])
        b.weight.zero_()
    _, ids = pnn.full_softmax_sample(torch.ones(N, 1), w, b, 1, tau, 91, top_k=top_k, top_p=top_p)
    s = logits[None] * _inv(tau)
    keep = _kept(s, 1, top_k, top_p)[0].numpy()
    p = torch.softmax(s[0].double(), 0).numpy() * keep
    p /= p.sum()
    cnt = np.bincount(ids[:, 0].numpy(), minlength=Vn)
    assert cnt[~keep].sum() == 0
    big = keep & (p * N >= 5)
    obs = np.append(cnt[big], cnt[keep & ~big].sum())
    exp = np.append(p[big] * N, p[keep & ~big].sum() * N)
    ok = exp > 0
    assert stats.chisquare(obs[ok], exp[ok]).pvalue > 1e-4


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
            lp, ids = pnn.full_softmax_sample(x, self.w, self.b, 4, 0.9, 2024, top_k=30,
                                              top_p=0.6)
        return {"loss": self.lin(x).sum(), "ids": ids, "lp": lp}


def _draw(P, strategy):
    torch.manual_seed(0)
    graph = parallax.Graph(_Head(P, strategy), optimizer=parallax.optim.Adagrad(0.1, 1.0))
    sess, *_ = parallax.parallel_run(graph, "localhost", parallax_config=parallax.Config(
        sess_config={"fabric": "host"}))
    x = torch.randn(23, 16, generator=torch.Generator().manual_seed(1))
    sess.engine.model.eval()
    ids, lp = sess.run(["ids", "lp"], {"x": [x]})
    sess.close()
    return torch.as_tensor(ids[0]), torch.as_tensor(lp[0])


def test_same_seed_same_truncated_draws_across_partitionings():
    ref_ids, ref_lp = _draw(1, "mod")
    for P, strategy in [(3, "mod"), (3, "div"), (7, "mod"), (7, "div"), (1, "div")]:
        ids, lp = _draw(P, strategy)
        assert torch.equal(ids, ref_ids), (P, strategy)
        torch.testing.assert_close(lp, ref_lp, rtol=0, atol=1e-6)


# ------------------------------------------------------------------ arguments
def test_argument_validation():
    w, b = _embeddings(V, 8, 6)
    x = torch.randn(5, 8)
    fs = pnn.full_softmax_sample
    for k in (0, -1, V + 1, True, False, 2.0, "3"):
        with pytest.raises(ValueError, match="top_k must be"):
            fs(x, w, b, 1, top_k=k)
    with pytest.raises(ValueError, match="must not exceed top_k"):
        fs(x, w, b, 4, top_k=3)
    for p in (0, 0.0, -0.1, 1.0000001, 2, float("nan"), float("inf"), True, "0.9"):
        with pytest.raises(ValueError, match="top_p must be"):
            fs(x, w, b, 1, top_p=p)
    # the existing refusals come first, with their messages
    with pytest.raises(ValueError, match="num_samples must be"):
        fs(x, w, b, 0, top_k=3)
    with pytest.raises(ValueError, match="temperature"):
        fs(x, w, b, 1, 0.0, top_p=0.5)
    # the bounds are accepted
    fs(x, w, b, V, top_k=np.int64(V))
    fs(x, w, b, 3, top_k=3, top_p=np.float32(1e-3))
    fs(x, w, b, 1, top_p=1)


# ------------------------------------------------------------------ LM1B
def _session(**kw):
    torch.manual_seed(0)
    m = LM1B(vocab_size=V, emb_size=16, state_size=32, projected_size=16, num_sampled=0,
             num_steps=4, num_shards=3, keep_prob=1.0, **kw)
    sess, *_ = parallax.parallel_run(lm1b_graph(m, batch_size=8), "localhost",
                                     parallax_config=parallax.Config(
                                         sess_config={"fabric": "host"}))
    return sess, m


def _batch(seed):
    x = torch.randint(0, V, (8, 4), generator=torch.Generator().manual_seed(seed))
    return {"x": [x], "y": [torch.roll(x, -1, dims=1)]}


def test_lm1b_truncated_sample_outputs(monkeypatch):
    seen = {}
    orig = pnn.full_softmax_sample

    def sample(inputs, w, b, n, tau, seed, **kw):
        seen["args"] = (n, tau, seed, kw)
        seen["out"] = orig(inputs, w, b, n, tau, seed, **kw)
        return seen["out"]
    monkeypatch.setattr(pnn, "full_softmax_sample", sample)
    sess, m = _session(eval_sample=2, sample_temperature=0.8, sample_top_k=7, sample_top_p=0.9)
    sess.run(["loss", "train_op"], _batch(0))
    m.eval()
    try:
        ids, lp = sess.run(["sample_ids", "sample_log_probs"], dict(_batch(2), sample_seed=[5]))
    finally:
        m.train()
    ids, lp = torch.as_tensor(ids[0]), torch.as_tensor(lp[0])
    assert seen["args"] == (2, 0.8, 5, {"top_k": 7, "top_p": 0.9})
    assert ids.shape == (8, 4, 2) and lp.shape == (8, 4, 2)
    assert torch.equal(ids, seen["out"][1].reshape(4, 8, 2).transpose(0, 1))
    assert torch.equal(lp, seen["out"][0].reshape(4, 8, 2).transpose(0, 1))
    sess.close()


def test_lm1b_top_k_only_passes_top_k(monkeypatch):
    seen = {}
    orig = pnn.full_softmax_sample

    def sample(inputs, w, b, n, tau, seed, **kw):
        seen["kw"] = kw
        return orig(inputs, w, b, n, tau, seed, **kw)
    monkeypatch.setattr(pnn, "full_softmax_sample", sample)
    sess, m = _session(eval_sample=1, sample_top_k=3)
    m.eval()
    try:
        sess.run("sample_ids", dict(_batch(3), sample_seed=[1]))
    finally:
        m.train()
    assert seen["kw"] == {"top_k": 3}
    sess.close()


# ------------------------------------------------------------------ generation script
def test_generate_top_p_from_a_trained_tiny_checkpoint(tmp_path):
    env = {k: v for k, v in os.environ.items()
           if not k.startswith("PARALLAX_") and k not in ("RANK", "WORLD_SIZE", "LOCAL_RANK")}
    env.update(PARALLAX_FABRIC="host", CUDA_VISIBLE_DEVICES="", OMP_NUM_THREADS="2")
    ck = str(tmp_path / "ck")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "examples/lm1b/lm1b_distributed_driver.py"),
                        "--use_synthetic", "--tiny", "--max_steps", "4", "--ckpt_dir", ck,
                        "--save_ckpt_steps", "4", "--logdir", str(tmp_path / "log")],
                       env=env, cwd=str(tmp_path), capture_output=True, text=True, timeout=400)
    assert r.returncode == 0, r.stderr[-1500:]

    def generate(seed, extra):
        r = subprocess.run([sys.executable, os.path.join(ROOT, "examples/lm1b/lm1b_generate.py"),
                            "--use_synthetic", "--tiny", "--ckpt_dir", ck, "--prefix", "5 17",
                            "--num_words", "7", "--num_sequences", "3", "--seed", str(seed)]
                           + list(extra), env=env, cwd=str(tmp_path), capture_output=True,
                           text=True, timeout=400)
        assert r.returncode == 0, r.stderr[-1500:]
        assert "top_p 0.9" in r.stderr + r.stdout
        return r.stdout.strip().splitlines()[-3:]
    a = generate(1, ["--top_p", "0.9"])
    b = generate(1, ["--top_p", "0.9"])
    c = generate(1, ["--top_p", "0.9", "--top_k", "5"])
    for lines in (a, c):
        for line in lines:
            words = line.split()
            assert words[:2] == ["5", "17"] and len(words) == 2 + 7
            assert all(0 <= int(w) < 10000 for w in words)
    assert a == b
