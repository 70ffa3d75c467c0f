"""Row-wise Adagrad on the host fabric: the host rule against a hand-written numpy step,
the engine against a single-device torch oracle on the concatenated batch, the build-time
refusals, checkpoints with the logical [V, 1] slot, and the placement byte counts."""
import math
import os

import numpy as np
import pytest
import torch

import parallax_b200 as parallax
from parallax_b200 import optim
from parallax_b200.models.simple import MLPWithEmbedding
from tests.dist_utils import run_distributed

B, T, VOCAB, STEPS = 8, 3, 64, 3


# ---------------------------------------------------------------------- the rule
@pytest.mark.parametrize("D", [1, 3, 64])
def test_host_rule_matches_numpy(D):
    rng = np.random.default_rng(D)
    V, lr, eps, s0 = 10, 0.3, 1e-3, 0.2
    w = rng.standard_normal((V, D)).astype(np.float32)
    s = np.full((V, 1), s0, dtype=np.float32)
    rows = np.array([1, 4, 7])
    g = rng.standard_normal((3, D)).astype(np.float32)
    opt = optim.RowWiseAdagrad(lr, initial_accumulator_value=s0, epsilon=eps)
    wt, st = torch.from_numpy(w.copy()), torch.from_numpy(s.copy())
    optim.apply_sparse_rows_(opt.kind, wt, torch.from_numpy(rows), torch.from_numpy(g), (st,),
                             opt.hyper(1))
    w_ref, s_ref = w.astype(np.float64), s.astype(np.float64)
    for i, r in enumerate(rows):
        s_ref[r, 0] += sum(float(x) ** 2 for x in g[i]) / D
        for j in range(D):
            w_ref[r, j] -= lr * g[i, j] / (math.sqrt(s_ref[r, 0]) + eps)
    np.testing.assert_allclose(st.numpy(), s_ref, rtol=1e-6)
    np.testing.assert_allclose(wt.numpy(), w_ref, rtol=1e-5, atol=1e-6)
    untouched = [r for r in range(V) if r not in rows]
    assert np.array_equal(wt.numpy()[untouched], w[untouched])
    assert np.array_equal(st.numpy()[untouched], s[untouched])


def test_width_one_is_adagrad():
    g = torch.Generator().manual_seed(0)
    w = torch.randn(12, 1, generator=g)
    rows = torch.tensor([0, 3, 5, 11])
    grads = [torch.randn(4, 1, generator=g) for _ in range(3)]
    rw, ad = optim.RowWiseAdagrad(0.2, 0.1), optim.Adagrad(0.2, 0.1)
    w1, w2 = w.clone(), w.clone()
    s1, s2 = (torch.full((12, 1), 0.1),), (torch.full((12, 1), 0.1),)
    for step, gr in enumerate(grads, 1):
        optim.apply_sparse_rows_(rw.kind, w1, rows, gr, s1, rw.hyper(step))
        optim.apply_sparse_rows_(ad.kind, w2, rows, gr, s2, ad.hyper(step))
    torch.testing.assert_close(w1, w2, rtol=1e-6, atol=0)
    torch.testing.assert_close(s1[0], s2[0], rtol=1e-6, atol=0)


def test_spec():
    opt = optim.RowWiseAdagrad(0.5, initial_accumulator_value=0.3, epsilon=1e-4)
    assert opt.kind == "rowwise_adagrad" and optim.KIND_ID[opt.kind] == 11
    assert optim.NUM_SLOTS[opt.kind] == 1 and optim.SLOT_NAMES[opt.kind] == ("accumulator",)
    assert opt.slot_init() == (0.3,)
    hp = opt.hyper(4)
    assert hp[optim.HP_LR] == 0.5 and abs(hp[optim.HP_EPS] - 1e-4) < 1e-12
    assert optim.kind_family(opt.kind) == 2
    assert optim.kind_family("adagrad") == 0 and optim.kind_family("ftrl") == 1


# ----------------------------------------------------------- engine vs oracle
def make_batch(step, world, rank=None):
    g = torch.Generator().manual_seed(500 + step)
    ids = torch.randint(0, VOCAB, (B * world, T), generator=g)
    ids[:, 0] = ids[0, 0]                     # duplicates inside and across workers
    labels = torch.randint(0, 4, (B * world,), generator=g)
    if rank is None:
        return ids, labels
    return ids[rank * B:(rank + 1) * B], labels[rank * B:(rank + 1) * B]


def dense_opt():
    return optim.Adagrad(0.3, 0.5)


def sparse_opt():
    return optim.RowWiseAdagrad(0.3, 0.5, epsilon=1e-3)


def oracle(world, max_norm, emb_scale, average):
    """Single-device training on the concatenated batch with a dense embedding gradient
    (× world for the sum semantics of sparse aggregation); the clip, when given, is
    `clip_grad_norm_` over every variable."""
    model = MLPWithEmbedding(VOCAB)
    model.emb.sparse = False
    named = dict(model.named_parameters())
    dopt, sopt = dense_opt(), sparse_opt()
    slots = {n: tuple(torch.full_like(p, v) for v in dopt.slot_init()) for n, p in named.items()}
    slots["emb.weight"] = (torch.full((VOCAB, 1), sopt.slot_init()[0]),)
    losses = []
    for s in range(STEPS):
        ids, labels = make_batch(s, world)
        out = model(ids, labels)
        model.zero_grad()
        out["loss"].backward()
        losses.append(out["loss"].item())
        grads = {n: p.grad.clone() for n, p in named.items()}
        grads["emb.weight"] *= emb_scale * (1.0 if average else world)
        if max_norm is not None:
            norm = math.sqrt(sum(float((g.double() ** 2).sum()) for g in grads.values()))
            scale = max_norm / max(norm, max_norm)
            grads = {n: g * scale for n, g in grads.items()}
        with torch.no_grad():
            for n, p in named.items():
                if n == "emb.weight":
                    rows = torch.unique(ids.reshape(-1))
                    optim.apply_sparse_rows_(sopt.kind, p.data, rows, grads[n][rows], slots[n],
                                             sopt.hyper(s + 1))
                else:
                    optim.apply_dense_(dopt.kind, p.data, grads[n], slots[n], dopt.hyper(s + 1))
    weights = {n: p.detach().clone() for n, p in named.items()}
    return losses, weights, slots["emb.weight"][0]


def train(world, rank, run_option, max_norm, emb_scale, average, local_agg, nparts=3):
    torch.manual_seed(0)
    model = MLPWithEmbedding(VOCAB, partitioner=parallax.get_partitioner(nparts))
    rules = [parallax.ScaleGradients(emb_scale, params=["emb.weight"])]
    if max_norm is not None:
        rules.append(parallax.ClipByGlobalNorm(max_norm, include_sparse=True))
    graph = parallax.Graph(model, optimizer=dense_opt(), sparse_optimizer=sparse_opt(),
                           grad_rules=rules)
    cfg = parallax.Config(run_option=run_option, average_sparse=average,
                          search_partitions=False, sess_config={"fabric": "host"})
    cfg.communication_config = parallax.CommunicationConfig(
        parallax.PSConfig(local_aggregation=local_agg))
    sess, *_ = parallax.parallel_run(graph, "localhost", parallax_config=cfg)
    losses = []
    try:
        for s in range(STEPS):
            ids, labels = make_batch(s, world, rank if world > 1 else None)
            loss, _ = sess.run(["loss", "train_op"], {"ids": [ids], "labels": [labels]})
            losses.append(loss[0])
        sd = sess.engine.state_dict()
    finally:
        sess.close()
    weights = dict(sd["dense"]["master"])
    weights["emb.weight"] = sd["sparse"]["emb.weight"]["weight"]
    return losses, weights, sd["sparse"]["emb.weight"]["slots"][0]


def _compare(got, want, losses=True):
    for a, b in zip(got[0], want[0] if losses else []):
        assert abs(a - b) < 1e-4 * max(1.0, abs(b))
    for n, w in want[1].items():
        torch.testing.assert_close(got[1][n].view_as(w), w, rtol=2e-4, atol=2e-5)
    assert tuple(got[2].shape) == (VOCAB, 1)
    torch.testing.assert_close(got[2], want[2], rtol=2e-4, atol=2e-6)


@pytest.mark.parametrize("run_option", ["HYBRID", "PS", "MPI"])
@pytest.mark.parametrize("average", [False, True])
@pytest.mark.parametrize("local_agg", [True, False])
@pytest.mark.parametrize("max_norm", [None, 0.05, 100.0])
def test_host_engine_matches_oracle(run_option, average, local_agg, max_norm):
    got = train(1, 0, run_option, max_norm, 4.0, average, local_agg)
    _compare(got, oracle(1, max_norm, 4.0, average))


def _worker(rank, world, run_option, average, max_norm):
    return train(world, rank, run_option, max_norm, 4.0, average, True)


@pytest.mark.parametrize("run_option,average,max_norm", [
    ("HYBRID", False, None), ("PS", True, 0.05), ("MPI", False, 0.05)])
def test_host_engine_two_ranks(run_option, average, max_norm):
    res = run_distributed(_worker, 2, run_option, average, max_norm)
    want = oracle(2, max_norm, 4.0, average)
    for got in res:                  # (each rank's loss is the mean over its own rows)
        _compare(got, want, losses=False)


def test_untouched_rows_and_accumulators_keep_their_bits():
    model = MLPWithEmbedding(VOCAB, partitioner=parallax.get_partitioner(3))
    graph = parallax.Graph(model, optimizer=dense_opt(), sparse_optimizer=sparse_opt())
    sess, *_ = parallax.parallel_run(graph, "localhost", parallax_config=parallax.Config(
        search_partitions=False, sess_config={"fabric": "host"}))
    try:
        ids, labels = make_batch(0, 1)
        sess.run(["loss", "train_op"], {"ids": [ids], "labels": [labels]})
        before = sess.engine.state_dict()["sparse"]["emb.weight"]
        ids, labels = make_batch(1, 1)
        sess.run(["loss", "train_op"], {"ids": [ids], "labels": [labels]})
        after = sess.engine.state_dict()["sparse"]["emb.weight"]
    finally:
        sess.close()
    touched = torch.zeros(VOCAB, dtype=torch.bool)
    touched[ids.reshape(-1)] = True
    assert torch.equal(after["weight"][~touched], before["weight"][~touched])
    assert torch.equal(after["slots"][0][~touched], before["slots"][0][~touched])
    assert bool((after["slots"][0][touched] > before["slots"][0][touched]).all())


# -------------------------------------------------------------------- refusals
def test_dense_use_refused():
    graph = parallax.Graph(MLPWithEmbedding(VOCAB), optimizer=sparse_opt())
    with pytest.raises(ValueError, match="sparse_optimizer"):
        parallax.parallel_run(graph, "localhost", parallax_config=parallax.Config(
            search_partitions=False, sess_config={"fabric": "host"}))


def test_async_refused():
    graph = parallax.Graph(MLPWithEmbedding(VOCAB), optimizer=dense_opt(),
                           sparse_optimizer=sparse_opt())
    cfg = parallax.Config(run_option="PS", search_partitions=False,
                          sess_config={"fabric": "host"})
    with pytest.raises(ValueError, match="sync=True"):
        parallax.parallel_run(graph, "localhost", sync=False, parallax_config=cfg)


def _session(opt, nparts=3):
    torch.manual_seed(0)
    model = MLPWithEmbedding(VOCAB, partitioner=parallax.get_partitioner(nparts))
    graph = parallax.Graph(model, optimizer=dense_opt(), sparse_optimizer=opt)
    sess, *_ = parallax.parallel_run(graph, "localhost", parallax_config=parallax.Config(
        search_partitions=False, sess_config={"fabric": "host"}))
    return sess


def test_slot_shape_mismatch_on_load_refused():
    sess = _session(optim.Adagrad(0.3, 0.5))
    try:
        ids, labels = make_batch(0, 1)
        sess.run(["loss", "train_op"], {"ids": [ids], "labels": [labels]})
        sd_adagrad = sess.engine.state_dict()
    finally:
        sess.close()
    sess = _session(sparse_opt())
    try:
        with pytest.raises(ValueError, match="emb.weight"):
            sess.engine.load_state_dict(sd_adagrad)             # [V, D] slot into [V, 1]
        sd = sess.engine.state_dict()
        assert tuple(sd["sparse"]["emb.weight"]["slots"][0].shape) == (VOCAB, 1)
    finally:
        sess.close()
    sess = _session(optim.Adagrad(0.3, 0.5))
    try:
        with pytest.raises(ValueError, match="emb.weight"):
            sess.engine.load_state_dict(sd)                     # [V, 1] slot into [V, D]
    finally:
        sess.close()


# ----------------------------------------------------------------- checkpoints
def test_state_dict_round_trip_and_repartition():
    sess = _session(sparse_opt())
    try:
        for s in range(2):
            ids, labels = make_batch(s, 1)
            sess.run(["loss", "train_op"], {"ids": [ids], "labels": [labels]})
        sd = sess.engine.state_dict()
        sess.engine.repartition(5)
        rp = sess.engine.state_dict()
    finally:
        sess.close()
    for k in ("weight", "slots"):
        torch.testing.assert_close(rp["sparse"]["emb.weight"][k], sd["sparse"]["emb.weight"][k])
    sess = _session(sparse_opt(), nparts=2)
    try:
        sess.engine.load_state_dict(sd)
        got = sess.engine.state_dict()
    finally:
        sess.close()
    for k in ("weight", "slots"):
        torch.testing.assert_close(got["sparse"]["emb.weight"][k], sd["sparse"]["emb.weight"][k])


class _Comm(object):
    distributed, is_cuda, device = False, False, torch.device("cpu")

    def __init__(self, rank, world):
        self.rank, self.world = rank, world

    def barrier(self):
        pass


class _Engine(object):
    dense, global_step, run_option = None, 5, "HYBRID"

    def __init__(self, comm, table):
        self.comm, self.tables = comm, {"emb.weight": table}
        self.model = torch.nn.Linear(1, 1)


def test_sharded_checkpoint_with_rowwise_slot(tmp_path):
    """Owners write [n, 1] slot rows; a reload at another world size and partition count
    re-scatters them, and the offline reader assembles a [V, 1] slot."""
    from parallax_b200 import checkpoint as ckpt
    from parallax_b200.parallel.layout import TableLayout
    from parallax_b200.tools import inspect_checkpoint as ic

    class _Table(object):
        """Row storage like NVSparseTable's, with a row-wise slot."""
        nslots, replicated, slot_dim = 1, False, 1

        def __init__(self, V, D, P, W, rank, full=None, slot=None):
            self.V, self.D, self.rank = V, D, rank
            self.layout = TableLayout(V, P, W, "mod")
            self.w = torch.zeros(self.layout.rows_local, D)
            self.s = torch.zeros(self.layout.rows_local, 1)
            if full is not None:
                for g, l in self.layout.owner_chunks(rank):
                    self.w[l], self.s[l] = full[g], slot[g]

        def local_rows(self, what="weight"):
            src = self.w if what == "weight" else self.s
            gs, rows = zip(*[(g, src[l]) for g, l in self.layout.owner_chunks(self.rank)])
            return torch.cat(gs), torch.cat(rows)

        def load_rows(self, ids, rows, what="weight"):
            own = self.layout.owner_of(ids) == self.rank
            dst = self.w if what == "weight" else self.s
            dst[self.layout.local_row_of(ids[own])] = rows[own]

    V, D = 53, 6
    full, slot = torch.randn(V, D), torch.rand(V, 1)
    d = str(tmp_path / "model.ckpt-5")
    os.makedirs(d)
    for r in range(2):
        ckpt.save_sharded(_Engine(_Comm(r, 2), _Table(V, D, 4, 2, r, full, slot)), d, r == 0)
    assert ckpt.read_manifest(d)["sparse"]["emb.weight"]["slot_dim"] == 1
    got = torch.zeros(V, 1)
    for r in range(3):
        t = _Table(V, D, 5, 3, r)
        ckpt.load_sharded(_Engine(_Comm(r, 3), t), d)
        g, l = t.layout.global_ids_of_owner(r)
        got[g] = t.s[l]
    torch.testing.assert_close(got, slot)
    tab = ckpt.assemble_table(d, "emb.weight")
    assert tuple(tab["slots"][0].shape) == (V, 1)
    torch.testing.assert_close(tab["slots"][0], slot)
    _, sd = ic.load(d)
    torch.testing.assert_close(sd["sparse"]["emb.weight"]["slots"][0], slot)
    # the byte estimate that decides what the reader assembles counts 4 B of slot per row
    _, small = ic.load(d, max_table_bytes=V * 4 * (D + 1))
    assert small["skipped"] == []
    _, small = ic.load(d, max_table_bytes=V * 4 * (D + 1) - 1)
    assert small["skipped"] == ["emb.weight"]

    class _DenseSlotTable(_Table):
        slot_dim = D                                      # e.g. Adagrad: [V, D] slots
    with pytest.raises(ValueError, match="emb.weight"):
        ckpt.load_sharded(_Engine(_Comm(0, 2), _DenseSlotTable(V, D, 4, 2, 0)), d)


# ------------------------------------------------------------------- placement
def test_placement_counts_four_bytes_of_slot_per_row():
    assert optim.table_row_bytes("rowwise_adagrad", 64) == 64 * 4 + 4
    assert optim.table_row_bytes("adagrad", 64) == 64 * 4 * 2
    assert optim.table_row_bytes("adam", 3) == 4 * 4 * 3         # padded to 4 columns
    assert optim.table_row_bytes("rowwise_adagrad", 3) == 4 * 4 + 4
    from parallax_b200.tools import launch_ps
    v = launch_ps._parse_var("emb:1000:64:4:rowwise_adagrad")
    assert launch_ps.row_bytes(v) == 64 * 4 + 4
    assert launch_ps.row_bytes(launch_ps._parse_var("emb:1000:64:4:1")) == 64 * 4 * 2
    _, load = launch_ps.plan([[v]], 4)
    assert load == [250 * (64 * 4 + 4)] * 4
    with pytest.raises(ValueError):
        launch_ps._parse_var("emb:1000:64:4:lion")


def test_host_engine_places_by_real_slot_bytes(monkeypatch):
    """The byte-greedy placement of the host / library fabric sees 4 B of slot per row."""
    from parallax_b200.parallel import layout
    seen = {}
    real = layout.assign_owners

    def spy(items, world):
        seen["items"] = list(items)
        return real(items, world)
    monkeypatch.setattr(layout, "assign_owners", spy)
    sess = _session(sparse_opt(), nparts=4)
    sess.close()
    (path, parts, nbytes), = seen["items"]
    D = MLPWithEmbedding(VOCAB).emb.weight.shape[1]
    assert parts == 4 and nbytes == (VOCAB // 4) * ((D + 3) // 4 * 16 + 4)
