"""`ClipByGlobalNorm(include_sparse=True)` on the host fabric: one global norm over
the dense gradients and the aggregated, duplicate-merged embedding rows, checked
against `clip_grad_norm_` semantics on a plain single-device torch model whose
embedding has a dense gradient."""
import fnmatch
import math

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import parallax_b200 as parallax
from parallax_b200 import optim
from parallax_b200.models.simple import MLPWithEmbedding
from tests.dist_utils import run_distributed

B, T, VOCAB, STEPS = 8, 3, 64, 3
ALL = None
SPARSE_ONLY = ["emb.weight"]


def make_batch(step, world, rank=None):
    g = torch.Generator().manual_seed(300 + step)
    ids = torch.randint(0, VOCAB, (B * world, T), generator=g)
    ids[:, 0] = ids[0, 0]                     # duplicates inside and across workers
    labels = torch.randint(0, 4, (B * world,), generator=g)
    if rank is None:
        return ids, labels
    return ids[rank * B:(rank + 1) * B], labels[rank * B:(rank + 1) * B]


def make_opt(name):
    return {"sgd": lambda: optim.GradientDescent(0.5),
            "adagrad": lambda: optim.Adagrad(0.3, 0.5),
            "adam": lambda: optim.Adam(0.02)}[name]()


def oracle(world, opt, max_norm, params, emb_scale, average):
    """Single-device training on the concatenated batch: the loss is the mean over all
    workers' rows, so dense gradients are the worker mean and the embedding gradient
    is the worker mean too (× world for the sum semantics of sparse aggregation)."""
    model = MLPWithEmbedding(VOCAB)
    model.emb.sparse = False
    named = dict(model.named_parameters())
    slots = {n: tuple(torch.full_like(p, v) for v in opt.slot_init()) for n, p in named.items()}
    matched = [n for n in named
               if params is None or any(fnmatch.fnmatchcase(n, p) for p in params)]
    losses, norms = [], []
    for s in range(STEPS):
        ids, labels = make_batch(s, world)
        out = model(ids, labels)
        model.zero_grad()
        out["loss"].backward()
        losses.append(out["loss"].item())
        grads = {n: p.grad.clone() for n, p in named.items()}
        grads["emb.weight"] *= emb_scale * (1.0 if average else world)
        norm = math.sqrt(sum(float((grads[n].double() ** 2).sum()) for n in matched))
        norms.append(norm)
        scale = max_norm / max(norm, max_norm)
        for n in matched:
            grads[n] = grads[n] * scale
        hp = opt.hyper(s + 1)
        with torch.no_grad():
            for n, p in named.items():
                if n == "emb.weight":
                    rows = torch.unique(ids.reshape(-1))
                    optim.apply_sparse_rows_(opt.kind, p.data, rows, grads[n][rows], slots[n],
                                             hp)
                else:
                    optim.apply_dense_(opt.kind, p.data, grads[n], slots[n], hp)
    return losses, {n: p.detach().clone() for n, p in named.items()}, norms


def train(world, rank, run_option, opt_name, max_norm, params, emb_scale, average, local_agg,
          nparts=3):
    model = MLPWithEmbedding(VOCAB, partitioner=parallax.get_partitioner(nparts))
    rules = [parallax.ScaleGradients(emb_scale, params=["emb.weight"]),
             parallax.ClipByGlobalNorm(max_norm, params=params, include_sparse=True)]
    graph = parallax.Graph(model, optimizer=make_opt(opt_name), grad_rules=rules)
    cfg = parallax.Config(run_option=run_option, average_sparse=average,
                          search_partitions=False, sess_config={"fabric": "host"})
    cfg.communication_config = parallax.CommunicationConfig(
        parallax.PSConfig(local_aggregation=local_agg))
    sess, *_ = parallax.parallel_run(graph, "localhost", parallax_config=cfg)
    losses, norms = [], []
    try:
        for s in range(STEPS):
            ids, labels = make_batch(s, world, rank if world > 1 else None)
            loss, _ = sess.run(["loss", "train_op"], {"ids": [ids], "labels": [labels]})
            losses.append(loss[0])
            norms.append(sess.engine.grad_norm(0))
        sd = sess.engine.state_dict()
    finally:
        sess.close()
    weights = dict(sd["dense"]["master"])
    weights["emb.weight"] = sd["sparse"]["emb.weight"]["weight"]
    return losses, weights, norms


def _compare(got, want):
    l_got, w_got, n_got = got
    l_want, w_want, n_want = want
    for a, b in zip(l_got, l_want):
        assert abs(a - b) < 1e-4 * max(1.0, abs(b))
    for a, b in zip(n_got, n_want):
        assert abs(a - b) <= 1e-5 * b
    for n, w in w_want.items():
        torch.testing.assert_close(w_got[n].view_as(w), w, rtol=2e-4, atol=2e-5)


@pytest.mark.parametrize("run_option", ["HYBRID", "PS", "MPI"])
@pytest.mark.parametrize("average", [False, True])
@pytest.mark.parametrize("local_agg", [True, False])
@pytest.mark.parametrize("max_norm,params", [(0.05, ALL), (100.0, ALL), (0.02, SPARSE_ONLY)])
def test_host_joint_clip_matches_oracle(run_option, average, local_agg, max_norm, params):
    got = train(1, 0, run_option, "adagrad", max_norm, params, 4.0, average, local_agg)
    want = oracle(1, make_opt("adagrad"), max_norm, params, 4.0, average)
    _compare(got, want)
    if max_norm < 1:
        assert all(n > max_norm for n in want[2])        # the clip is active


@pytest.mark.parametrize("opt_name", ["sgd", "adam"])
def test_host_joint_clip_optimizers(opt_name):
    got = train(1, 0, "HYBRID", opt_name, 0.05, ALL, 2.0, False, True)
    _compare(got, oracle(1, make_opt(opt_name), 0.05, ALL, 2.0, False))


def _worker(rank, world, run_option, average, max_norm, params):
    return train(world, rank, run_option, "adagrad", max_norm, params, 4.0, average, True)


@pytest.mark.parametrize("run_option,average,max_norm,params", [
    ("HYBRID", False, 0.05, ALL), ("PS", True, 0.05, ALL), ("MPI", False, 0.05, ALL),
    ("HYBRID", True, 0.02, SPARSE_ONLY)])
def test_host_joint_clip_two_ranks(run_option, average, max_norm, params):
    """Partitioned tables: the owners' shares of Σg² are summed across ranks;
    replicated (MPI) tables were merged in full on every rank and count once."""
    res = run_distributed(_worker, 2, run_option, average, max_norm, params)
    want = oracle(2, make_opt("adagrad"), max_norm, params, 4.0, average)
    for rank, got in enumerate(res):
        for a, b in zip(got[2], want[2]):
            assert abs(a - b) <= 1e-5 * b, (rank, got[2], want[2])
        for n, w in want[1].items():
            torch.testing.assert_close(got[1][n].view_as(w), w, rtol=2e-4, atol=2e-5)


def test_default_rule_is_dense_only():
    """Without include_sparse the embedding is neither measured nor clipped."""
    model = MLPWithEmbedding(VOCAB)
    graph = parallax.Graph(model, optimizer=optim.GradientDescent(0.5),
                           grad_rules=[parallax.ClipByGlobalNorm(0.05)])
    assert graph.joint_clip_index("emb.weight") == -1
    sess, *_ = parallax.parallel_run(graph, "localhost", parallax_config=parallax.Config(
        search_partitions=False, sess_config={"fabric": "host"}))
    try:
        ids, labels = make_batch(0, 1)
        sess.run(["loss", "train_op"], {"ids": [ids], "labels": [labels]})
        assert sess.engine.dense.joint_tables == []
        ref = MLPWithEmbedding(VOCAB)
        out = ref(ids, labels)
        out["loss"].backward()
        dense = [p.grad for n, p in ref.named_parameters() if n != "emb.weight"]
        norm = math.sqrt(sum(float((g.double() ** 2).sum()) for g in dense))
        assert abs(sess.engine.grad_norm(0) - norm) <= 1e-5 * norm
    finally:
        sess.close()


def test_async_refused():
    model = MLPWithEmbedding(VOCAB)
    graph = parallax.Graph(model, optimizer=optim.GradientDescent(0.5), grad_rules=[
        parallax.ClipByGlobalNorm(1.0, include_sparse=True)])
    cfg = parallax.Config(run_option="PS", search_partitions=False,
                          sess_config={"fabric": "host"})
    with pytest.raises(ValueError, match="sync=True"):
        parallax.parallel_run(graph, "localhost", sync=False, parallax_config=cfg)


class _TwoTables(nn.Module):
    co_lookup_groups = [["a", "b"]]

    def __init__(self):
        super().__init__()
        self.a = parallax.nn.Embedding(16, 4)
        self.b = parallax.nn.Embedding(16, 1)
        self.fc = nn.Linear(4, 2)

    def forward(self, ids, labels):
        a, b = parallax.nn.lookup_many([self.a, self.b], ids)
        return {"loss": F.cross_entropy(self.fc(a) + b, labels)}


def test_split_co_lookup_group_refused():
    graph = parallax.Graph(_TwoTables(), optimizer=optim.GradientDescent(0.5), grad_rules=[
        parallax.ClipByGlobalNorm(1.0, params=["a.weight", "fc.*"], include_sparse=True)])
    cfg = parallax.Config(search_partitions=False, sess_config={"fabric": "host"})
    with pytest.raises(ValueError, match="co-lookup group"):
        parallax.parallel_run(graph, "localhost", parallax_config=cfg)


# ----------------------------------------------------------------------- NMT
def _nmt_hp(**kw):
    from parallax_b200.models import nmt
    kw = dict(dict(num_units=16, dropout=0.0, attention="luong", encoder_type="uni",
                   num_layers=1, num_embeddings_partitions=2, learning_rate=0.5,
                   max_gradient_norm=0.01), **kw)
    return nmt.extend_hparams(nmt.create_hparams(**kw), 30, 30)


def _nmt_feed():
    g = torch.Generator().manual_seed(0)
    src = torch.randint(3, 30, (4, 7), generator=g)
    tin = torch.randint(3, 30, (4, 6), generator=g)
    tout = torch.randint(3, 30, (4, 6), generator=g)
    return {"source": [src], "target_input": [tin], "target_output": [tout],
            "source_sequence_length": [torch.tensor([7, 5, 3, 6])],
            "target_sequence_length": [torch.tensor([6, 4, 6, 2])]}


def _nmt_train(hp, steps=2):
    from parallax_b200.models import nmt
    torch.manual_seed(0)
    m = nmt.create_model(hp)
    sess, *_ = parallax.parallel_run(nmt.nmt_graph(m, hp), "localhost",
                                     parallax_config=parallax.Config(
                                         search_partitions=False,
                                         sess_config={"fabric": "host"}))
    try:
        losses = [sess.run(["loss", "train_op"], _nmt_feed())[0][0] for _ in range(steps)]
        sd = sess.engine.state_dict()
        return losses, sd, sess.engine.grad_norm(0)
    finally:
        sess.close()


def test_nmt_joint_clip_matches_oracle():
    """clip_embeddings_jointly: one norm over every variable, embeddings included,
    as `clip_grad_norm_` over a single-device model with dense embedding gradients."""
    from parallax_b200.models import nmt
    hp = _nmt_hp(clip_embeddings_jointly=True)
    graph_rules = nmt.nmt_graph(nmt.create_model(hp), hp).clip_rules()
    assert len(graph_rules) == 1 and graph_rules[0].include_sparse
    losses, sd, norm = _nmt_train(hp)
    torch.manual_seed(0)
    ref = nmt.create_model(hp)
    ref.embedding_encoder.sparse = ref.embedding_decoder.sparse = False
    opt = nmt.nmt_graph(ref, hp).optimizer
    feed = {k: v[0] for k, v in _nmt_feed().items()}
    want, norms = [], []
    for step in (1, 2):
        ref.zero_grad()
        out = ref(**feed)
        out["loss"].backward()
        want.append(out["loss"].item())
        norms.append(float(torch.nn.utils.clip_grad_norm_(ref.parameters(), 0.01)))
        with torch.no_grad():
            for p in ref.parameters():
                p.sub_(opt.hyper(step)[0] * p.grad)
    assert min(norms) > 0.01                                   # the clip is active
    assert abs(norm - norms[-1]) <= 1e-5 * norms[-1]
    for a, b in zip(losses, want):
        assert abs(a - b) < 1e-5 * max(1.0, abs(b))
    for n, p in ref.named_parameters():
        got = sd["sparse"][n]["weight"] if n in sd["sparse"] else sd["dense"]["master"][n]
        torch.testing.assert_close(got.view_as(p), p.detach(), rtol=1e-4, atol=1e-6)


def test_nmt_default_clip_is_unchanged():
    """Without the hparam (as in hparams saved before it existed) and with it False,
    training is the same computation, bit for bit: dense-only rule + per-lookup clip."""
    from parallax_b200.models import nmt
    hp = _nmt_hp()
    assert hp.clip_embeddings_jointly is False
    rules = nmt.nmt_graph(nmt.create_model(hp), hp).clip_rules()
    assert len(rules) == 1 and not rules[0].include_sparse
    old = _nmt_hp()
    old._keys.remove("clip_embeddings_jointly")
    del old.__dict__["clip_embeddings_jointly"]
    l_new, sd_new, _ = _nmt_train(hp)
    l_old, sd_old, _ = _nmt_train(old)
    assert l_new == l_old
    for n, w in sd_old["dense"]["master"].items():
        assert torch.equal(sd_new["dense"]["master"][n], w)
    for n, t in sd_old["sparse"].items():
        assert torch.equal(sd_new["sparse"][n]["weight"], t["weight"])
