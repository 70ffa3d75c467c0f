"""Layer-wise optimizers (LARS, LAMB) on the host and library fabrics: the update rules of
`optim.apply_dense_` against the reference LARS test and an fp64 LAMB, the per-name exclude
lists, the host engine against a single-device oracle, checkpoint resume and the refusals."""
import math

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import parallax_b200 as parallax
from parallax_b200 import optim
from tests.dist_utils import run_distributed

STEPS = 3


# --------------------------------------------------------------------------- rules
def _lars_expected(steps, lr=0.1, m=0.9, wd=0.1, eps=1e-5, eeta=0.1):
    """The reference `lars_optimizer_test.py` case in float64: var0 = var1 = [3, 3] ones,
    grads ones, the update computed from the formula."""
    w = np.ones((3, 3))
    g = np.ones((3, 3))
    vel = np.zeros((3, 3))
    for _ in range(steps):
        wn, gn = np.linalg.norm(w), np.linalg.norm(g)
        trust = eeta * wn / (gn + wd * wn + eps) if wn > 0 and gn > 0 else 1.0
        vel = m * vel + g
        w = w - lr * trust * vel
    return w, vel


@pytest.mark.parametrize("steps", [1, 10])
def test_lars_matches_reference_test_case(steps):
    opt = optim.LARSOptimizer(0.1, momentum=0.9, weight_decay=0.1, epsilon=1e-5, eeta=0.1)
    assert opt.kind == "lars" and optim.SLOT_NAMES["lars"] == ("momentum",)
    w = torch.ones(3, 3)
    (vel,) = (torch.zeros(3, 3),)
    for s in range(steps):
        optim.apply_dense_("lars", w, torch.ones(3, 3), (vel,), opt.hyper_for("var0", s + 1))
    want_w, want_vel = _lars_expected(steps)
    np.testing.assert_allclose(w.numpy(), want_w, rtol=1e-6)
    np.testing.assert_allclose(vel.numpy(), want_vel, rtol=1e-6)


def test_lars_nesterov_and_no_coupled_decay():
    """weight_decay enters only the trust ratio: with trust forced to 1 (skip_list), the step
    is plain momentum, whatever weight_decay is."""
    opt = optim.Lars(0.5, momentum=0.8, weight_decay=0.3, skip_list=["bias"],
                     use_nesterov=True)
    g = torch.randn(7, generator=torch.Generator().manual_seed(0))
    w = torch.randn(7, generator=torch.Generator().manual_seed(1))
    want, mom = w.clone(), torch.full((7,), 0.25)
    mom_new = 0.8 * mom + g
    want -= 0.5 * (g + 0.8 * mom_new)
    s0 = mom.clone()
    optim.apply_dense_("lars", w, g, (s0,), opt.hyper_for("fc.bias", 1))
    torch.testing.assert_close(w, want)
    torch.testing.assert_close(s0, mom_new)


def _lamb_fp64(w, g, m, v, t, lr, b1, b2, eps, wd, decay, adapt):
    w, g, m, v = (x.double() for x in (w, g, m, v))
    m = b1 * m + (1 - b1) * g
    v = b2 * v + (1 - b2) * g * g
    r = (m / (1 - b1 ** t)) / (torch.sqrt(v / (1 - b2 ** t)) + eps)
    if decay:
        r = r + wd * w
    wn, rn = float(w.norm()), float(r.norm())
    trust = wn / rn if adapt and wn > 0 and rn > 0 else 1.0
    return w - lr * trust * r, m, v


@pytest.mark.parametrize("name", ["enc.weight", "enc.LayerNorm.weight", "enc.bias"])
def test_lamb_matches_fp64(name):
    opt = optim.Lamb(0.01, beta1=0.8, beta2=0.95, epsilon=1e-6, weight_decay=0.05,
                     exclude_from_weight_decay=["LayerNorm", r"bias$"],
                     exclude_from_layer_adaptation=["LayerNorm"])
    decay = name == "enc.weight"
    adapt = name != "enc.LayerNorm.weight"
    gen = torch.Generator().manual_seed(3)
    w = torch.randn(5, 9, generator=gen)
    m, v = torch.zeros(5, 9), torch.zeros(5, 9)
    rw, rm, rv = w.double(), m.double(), v.double()
    for t in range(1, 6):
        g = torch.randn(5, 9, generator=gen)
        optim.apply_dense_("lamb", w, g, (m, v), opt.hyper_for(name, t))
        rw, rm, rv = _lamb_fp64(rw, g, rm, rv, t, 0.01, 0.8, 0.95, 1e-6, 0.05, decay, adapt)
    torch.testing.assert_close(w.double(), rw, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(m.double(), rm, rtol=1e-5, atol=1e-7)
    torch.testing.assert_close(v.double(), rv, rtol=1e-5, atol=1e-9)


def test_lamb_bias_corrections_are_host_doubles():
    opt = optim.Lamb(0.1, beta1=0.9, beta2=0.999)
    hp = opt.hyper(3)
    assert len(hp) == optim.HP_SIZE == 10
    assert hp[optim.HP_BC1] == 1.0 / (1.0 - 0.9 ** 3)
    assert hp[optim.HP_BC2] == 1.0 / (1.0 - 0.999 ** 3)
    assert hp[optim.HP_LR] == 0.1        # not folded, unlike Adam's


@pytest.mark.parametrize("kind", ["lars", "lamb"])
def test_trust_ratio_is_one_for_zero_norms(kind):
    """‖w‖ = 0 (a zero-initialised bias) or ‖x‖ = 0 (no gradient; for LAMB zero moments too):
    the step is that of trust = 1."""
    opt = optim.Lars(0.1, eeta=0.01) if kind == "lars" else optim.Lamb(0.1)
    hp = opt.hyper_for("b", 1)
    assert optim.trust_ratio(kind, 0.0, 2.0, hp) == 1.0
    assert optim.trust_ratio(kind, 2.0, 0.0, hp) == 1.0
    w, g = torch.zeros(4), torch.tensor([1.0, -2.0, 0.5, 0.0])
    slots = tuple(torch.zeros(4) for _ in optim.SLOT_NAMES[kind])
    optim.apply_dense_(kind, w, g, slots, hp)
    if kind == "lars":
        torch.testing.assert_close(w, -0.1 * g)
    else:
        torch.testing.assert_close(w, -0.1 * g / (g.abs() + 1e-6))
    w = torch.ones(4)
    slots = tuple(torch.zeros(4) for _ in optim.SLOT_NAMES[kind])
    optim.apply_dense_(kind, w, torch.zeros(4), slots, hp)
    torch.testing.assert_close(w, torch.ones(4))


def test_skip_and_exclude_patterns():
    lars = optim.Lars(0.1, skip_list=["bias", "bn"])
    assert lars.layer_flags("fc.weight") == optim.LW_ADAPT
    assert lars.layer_flags("fc.bias") == 0 and lars.layer_flags("layer1.bn1.weight") == 0
    assert optim.Lars(0.1).layer_flags("fc.bias") == optim.LW_ADAPT
    lamb = optim.Lamb(0.1, weight_decay=0.01, exclude_from_weight_decay=[r"\.bias$", "ln"])
    both = optim.LW_DECAY | optim.LW_ADAPT
    assert lamb.layer_flags("fc.weight") == both
    assert lamb.layer_flags("fc.bias") == 0          # adaptation follows the decay list
    assert lamb.layer_flags("ln1.weight") == 0
    assert lamb.layer_flags("fc.bias_gain") == both  # regex, not substring
    sep = optim.Lamb(0.1, weight_decay=0.01, exclude_from_weight_decay=["bias"],
                     exclude_from_layer_adaptation=[])
    assert sep.layer_flags("fc.bias") == optim.LW_ADAPT
    assert optim.Lamb(0.1).layer_flags("fc.weight") == optim.LW_ADAPT   # no decay at wd 0
    # the per-name hyper-parameters carry the flags; the other kinds have none
    assert int(lamb.hyper_for("fc.bias", 1)[optim.HP_FLAGS]) == 0
    nest = optim.Lars(0.1, skip_list=["bias"], use_nesterov=True)
    assert int(nest.hyper_for("fc.bias", 1)[optim.HP_FLAGS]) == optim.LW_NESTEROV
    # Nesterov is a per-tensor flag too: the dense step's segment map carries it
    assert nest.layer_flags("fc.weight") == optim.LW_NESTEROV | optim.LW_ADAPT
    assert nest.layer_flags("fc.bias") == optim.LW_NESTEROV
    assert optim.Adam(0.1).hyper_for("x", 2) == optim.Adam(0.1).hyper(2)


def test_kind_ids_and_families():
    old = ["sgd", "momentum", "adagrad", "adam", "rmsprop", "adadelta", "ftrl", "proximal_sgd",
           "proximal_adagrad", "adagrad_da", "centered_rmsprop", "rowwise_adagrad"]
    for i, k in enumerate(old):
        assert optim.KIND_ID[k] == i
    assert optim.KIND_ID["lars"] == 12 and optim.KIND_ID["lamb"] == 13
    assert optim.kind_family("lars") == optim.kind_family("lamb") == 3
    assert optim.kind_family("rowwise_adagrad") == 2
    assert optim.NUM_SLOTS["lars"] == 1 and optim.NUM_SLOTS["lamb"] == 2
    assert optim.SLOT_NAMES["lamb"] == ("m", "v")


# --------------------------------------------------------------------------- engine
class DenseNet(nn.Module):
    """Dense only: a weight, a zero-initialised bias, a scalar gain and a second layer."""

    def __init__(self, seed=0):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        self.fc1 = nn.Linear(6, 16)
        self.gain = nn.Parameter(torch.tensor(1.5))
        self.fc2 = nn.Linear(16, 4)
        with torch.no_grad():
            for p in (self.fc1.weight, self.fc1.bias, self.fc2.weight):
                p.copy_(torch.randn(p.shape, generator=g) * 0.3)
            self.fc2.bias.zero_()

    def forward(self, x, labels):
        logits = self.fc2(torch.tanh(self.fc1(x)) * self.gain)
        return {"loss": F.cross_entropy(logits, labels), "logits": logits}


def _batch(step, rows=8):
    g = torch.Generator().manual_seed(200 + step)
    return torch.randn(rows, 6, generator=g), torch.randint(0, 4, (rows,), generator=g)


def _make_opt(kind):
    """`kind`: "lars", "lars_nesterov" or "lamb"."""
    if kind.startswith("lars"):
        return optim.Lars(0.5, momentum=0.9, weight_decay=1e-3, eeta=0.02, skip_list=["bias"],
                          use_nesterov=kind == "lars_nesterov")
    return optim.Lamb(0.05, weight_decay=0.01, exclude_from_weight_decay=[r"bias$"],
                      exclude_from_layer_adaptation=["gain"])


def oracle(kind, steps=STEPS, clip=None, rows=8):
    """Single-device training on the whole batch of `rows` rows, one `apply_dense_` per
    tensor."""
    model = DenseNet()
    opt = _make_opt(kind)
    params = dict(model.named_parameters())
    slots = {n: tuple(torch.full_like(p, v) for v in opt.slot_init()) for n, p in params.items()}
    losses = []
    for s in range(steps):
        x, y = _batch(s, rows)
        model.zero_grad()
        out = model(x, y)
        out["loss"].backward()
        losses.append(float(out["loss"].detach()))
        grads = {n: p.grad.detach().clone() for n, p in params.items()}
        if clip is not None:
            norm = math.sqrt(sum(float((g ** 2).sum()) for g in grads.values()))
            scale = clip / max(norm, clip)
            grads = {n: g * scale for n, g in grads.items()}
        with torch.no_grad():
            for n, p in params.items():
                optim.apply_dense_(opt.kind, p.data, grads[n], slots[n],
                                   opt.hyper_for(n, s + 1))
    return losses, {n: p.detach().clone() for n, p in params.items()}, slots


def _train(world, rank, run_option, kind, K=None, clip=None, fabric=None, steps=STEPS,
           resume=None):
    """`resume=(start, state)`: load the engine state `state` into the new engine, then run
    steps start .. steps-1."""
    rules = [parallax.ClipByGlobalNorm(clip)] if clip is not None else []
    graph = parallax.Graph(DenseNet(), optimizer=_make_opt(kind), grad_rules=rules)
    sc = {}
    if K is not None:
        sc["micro_batches"] = K
    if fabric:
        sc["fabric"] = fabric
    cfg = parallax.Config(run_option=run_option, sess_config=sc)
    sess, nw, wid, _ = parallax.parallel_run(graph, "localhost", parallax_config=cfg)
    assert (nw, wid) == (world, rank)
    losses = []
    start = 0
    if resume is not None:
        start = resume[0]
        sess.engine.load_state_dict(resume[1])
    for s in range(start, steps):
        x, y = _batch(s)
        n = x.shape[0] // world
        loss, _ = sess.run(["loss", "train_op"], {"x": [x[rank * n:(rank + 1) * n]],
                                                  "labels": [y[rank * n:(rank + 1) * n]]})
        losses.append(loss[0])
    sd = sess.engine.state_dict()
    sess.close()
    return losses, sd


def _worker(rank, world, specs):
    return [_train(world, rank, **spec) for spec in specs]


def _check(result, ref, tol=(1e-5, 1e-6)):
    losses, sd = result
    ref_losses, ref_w, ref_slots = ref
    for n, w in ref_w.items():
        torch.testing.assert_close(sd["dense"]["master"][n], w, rtol=tol[0], atol=tol[1])
        for a, b in zip(sd["dense"]["slots"][n], ref_slots[n]):
            torch.testing.assert_close(a, b, rtol=tol[0], atol=tol[1])
    return losses, ref_losses


@pytest.mark.parametrize("kind", ["lars", "lars_nesterov", "lamb"])
def test_host_engine_world1_matches_oracle(kind):
    for clip in (None, 0.05):
        ref = oracle(kind, clip=clip)
        for K in (None, 2):
            losses, ref_losses = _check(_train(1, 0, "HYBRID", kind, K=K, clip=clip), ref)
            np.testing.assert_allclose(losses, ref_losses, rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("run_option", ["HYBRID", "MPI", "PS"])
@pytest.mark.parametrize("kind", ["lars", "lamb"])
def test_host_engine_two_workers_match_oracle(run_option, kind):
    specs = [dict(run_option=run_option, kind=kind),
             dict(run_option=run_option, kind=kind, clip=0.05),
             dict(run_option=run_option, kind=kind, K=2, clip=0.05)]
    res = run_distributed(_worker, 2, specs)
    refs = [oracle(kind), oracle(kind, clip=0.05), oracle(kind, clip=0.05)]
    for i, ref in enumerate(refs):
        for r in res:
            _check(r[i], ref)
        np.testing.assert_allclose(np.mean([r[i][0] for r in res], axis=0), ref[0],
                                   rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("kind", ["lars", "lamb"])
def test_checkpoint_resume_continues_identically(kind):
    """Dense slots are saved by name: a new engine, at its initial state, that loads the state
    saved after step 2 and runs steps 3..5 ends exactly where an uninterrupted run ends."""
    full = _train(1, 0, "HYBRID", kind, steps=5, clip=0.05)
    half = _train(1, 0, "HYBRID", kind, steps=2, clip=0.05)
    init = _train(1, 0, "HYBRID", kind, steps=0, clip=0.05)
    assert len(half[1]["dense"]["slots"]["fc1.weight"]) == optim.NUM_SLOTS[kind]
    for n, w in half[1]["dense"]["master"].items():      # the load has something to restore
        assert not torch.equal(init[1]["dense"]["master"][n], w), n
        for a, b in zip(init[1]["dense"]["slots"][n], half[1]["dense"]["slots"][n]):
            assert not torch.equal(a, b), n
    resumed = _train(1, 0, "HYBRID", kind, steps=5, clip=0.05, resume=(2, half[1]))
    assert resumed[0] == full[0][2:]
    for n, w in full[1]["dense"]["master"].items():
        assert torch.equal(resumed[1]["dense"]["master"][n], w), n
        for a, b in zip(resumed[1]["dense"]["slots"][n], full[1]["dense"]["slots"][n]):
            assert torch.equal(a, b), n


def test_library_fabric_matches_oracle():
    """fabric='library': the host code with library collectives (here gloo on the CPU)."""
    res = run_distributed(_worker, 2, [dict(run_option="HYBRID", kind="lamb", clip=0.05,
                                            fabric="library")])
    ref = oracle("lamb", clip=0.05)
    for r in res:
        _check(r[0], ref)


# --------------------------------------------------------------------------- refusals
def _build(opt, sess_config=None, sync=True, protocol=None, sparse_optimizer=None,
           sparse=True):
    from parallax_b200.models.simple import MLPWithEmbedding
    model = MLPWithEmbedding(64) if sparse else DenseNet()
    graph = parallax.Graph(model, optimizer=opt, sparse_optimizer=sparse_optimizer)
    cfg = parallax.Config(run_option="HYBRID", sess_config=sess_config or {})
    if protocol:
        cfg.communication_config = parallax.CommunicationConfig(
            parallax.PSConfig(protocol=protocol))
    return parallax.parallel_run(graph, "localhost", sync=sync, parallax_config=cfg)


@pytest.mark.parametrize("make", [lambda: optim.Lars(0.1), lambda: optim.Lamb(0.1)])
def test_refusals_name_the_alternative(make, monkeypatch):
    """Refused at build, before the fabric allocates anything (the NVLink cases are refused
    on a machine without a GPU, before the fabric would need one)."""
    from parallax_b200.parallel import nvlink_backend

    def no_build(engine):
        raise AssertionError("the fabric was built")
    monkeypatch.setattr(nvlink_backend, "build_nvlink", no_build)
    # the default sparse optimizer is the dense one
    with pytest.raises(ValueError, match=r"sparse_optimizer=Momentum\(\.\.\.\).*Adam"):
        _build(make())
    with pytest.raises(ValueError, match=r"sparse_optimizer=Momentum"):
        _build(optim.Adam(0.1), sparse_optimizer=make())
    with pytest.raises(ValueError, match="sync=True"):
        _build(make(), sync=False, sparse=False)
    with pytest.raises(ValueError, match="fabric': 'library'"):
        _build(make(), {"fabric": "nvlink", "dense_update": "replicated"}, sparse=False)
    with pytest.raises(ValueError, match="fabric': 'library'"):
        _build(make(), {"fabric": "nvlink"}, protocol="nccl", sparse=False)
    # a sparse model with its own sparse rule builds
    sess, *_ = _build(make(), sparse_optimizer=optim.Momentum(0.1))
    sess.close()


def test_bert_graph_lamb_recipe():
    from parallax_b200.models.bert import Bert, bert_graph
    model = Bert(vocab=50, hidden=16, layers=1, heads=2, ff=32, max_len=8, num_partitions=1)
    g = bert_graph(model, 1e-3, optimizer="lamb")
    assert g.optimizer.kind == "lamb" and g.optimizer.weight_decay == 0.01
    assert g.sparse_optimizer.kind == "adam"
    both = optim.LW_DECAY | optim.LW_ADAPT
    assert g.optimizer.layer_flags("layers.0.qkv.weight") == both
    for n in ("layers.0.qkv.bias", "layers.0.ln1.weight", "mlm_ln.bias", "ln.weight"):
        assert g.optimizer.layer_flags(n) == 0, n
    assert bert_graph(model, 1e-3).optimizer.kind == "adam"
    with pytest.raises(ValueError, match="lamb"):
        bert_graph(model, optimizer="lars")
