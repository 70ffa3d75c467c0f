"""Fused full-softmax training (`sess_config["full_softmax_train"]`) without a GPU: the option's
validation, and the fused backward's chunked schedule written in torch fp64 against autograd
through the composition.  `chunked_backward` is the oracle of `tests/test_gpu_full_softmax_train.py`."""
import pytest
import torch
import torch.nn.functional as F

import parallax_b200 as parallax
from parallax_b200 import optim
from parallax_b200.models.simple import MLPWithEmbedding
from parallax_b200.parallel.layout import TableLayout


def chunked_backward(x, targets, lse, g, gather, V, chunk):
    """fp64 ``(dx [N, K], dW [V, K], db [V])`` of the NLL's gradient `g` [N], in the fused
    backward's schedule: for each chunk of global ids [v0, v0 + chunk), gather its rows
    (`gather(ids)` -> (W_c [m, K], b_c [m])), recompute S = x·W_cᵀ + b_c, form
    G = g · (exp(S − lse) − onehot(targets)), then dx += G·W_c, dW_c = Gᵀ·x and db_c = Σ_rows G."""
    x, lse, g = x.double(), lse.double(), g.double()
    dx = torch.zeros_like(x)
    dW = torch.empty(V, x.shape[1], dtype=torch.float64)
    db = torch.empty(V, dtype=torch.float64)
    for v0 in range(0, V, chunk):
        ids = torch.arange(v0, min(V, v0 + chunk))
        w, b = gather(ids)
        w, b = w.double(), b.double()
        G = torch.exp(x @ w.t() + b[None, :] - lse[:, None])
        G -= (targets[:, None] == ids[None, :]).double()
        G *= g[:, None]
        dx += G @ w
        dW[ids] = G.t() @ x
        db[ids] = G.sum(0)
    return dx, dW, db


def layout_gather(W, B, layout):
    """`gather` from the tables stored by `layout`: each owner's local rows, read back by
    (owner, local row) of the global ids, as the group's lookup kernel reads them."""
    owners = 1 if layout.replicated else layout.world
    ids = torch.arange(layout.V)
    own = torch.zeros(layout.V, dtype=torch.int64) if layout.replicated else layout.owner_of(ids)
    loc = layout.local_row_of(ids)
    local_w = torch.full((owners, layout.rows_local, W.shape[1]), float("nan"), dtype=W.dtype)
    local_b = torch.full((owners, layout.rows_local), float("nan"), dtype=B.dtype)
    local_w[own, loc] = W
    local_b[own, loc] = B

    def gather(gids):
        o = torch.zeros_like(gids) if layout.replicated else layout.owner_of(gids)
        r = layout.local_row_of(gids)
        return local_w[o, r], local_b[o, r]
    return gather


def _composition_grads(x, targets, W, B, g):
    x, W, B = (t.double().clone().requires_grad_() for t in (x, W, B))
    nll = F.cross_entropy(x @ W.t() + B[None, :], targets, reduction="none")
    lse = torch.logsumexp((x @ W.t() + B[None, :]).detach(), dim=1)
    nll.backward(g.double())
    return nll.detach(), lse, x.grad, W.grad, B.grad


LAYOUTS = [
    # V, P, world, strategy, replicated
    (1000, 1, 1, "mod", False),
    (1001, 5, 2, "mod", False),
    (997, 7, 4, "div", False),
    (777, 1, 4, "mod", True),
]


@pytest.mark.parametrize("chunk", [128, 300, 4096])
@pytest.mark.parametrize("V,P,world,strategy,replicated", LAYOUTS)
@pytest.mark.parametrize("grads", ["ones", "zero", "random"])
def test_chunked_backward_matches_composition_autograd(V, P, world, strategy, replicated,
                                                       chunk, grads):
    gen = torch.Generator().manual_seed(V + chunk)
    N, K = 37, 24
    W = torch.randn(V, K, generator=gen, dtype=torch.float64) / K ** 0.5
    B = torch.randn(V, generator=gen, dtype=torch.float64)
    x = torch.randn(N, K, generator=gen, dtype=torch.float64)
    targets = torch.randint(0, V, (N,), generator=gen)
    targets[0], targets[-1] = 0, V - 1
    g = {"ones": torch.ones(N, dtype=torch.float64),
         "zero": torch.zeros(N, dtype=torch.float64),
         "random": torch.rand(N, generator=gen, dtype=torch.float64) * 3 - 1}[grads]
    g[3] = 0.0
    layout = TableLayout(V, P, world, strategy, replicated)
    _, lse, dx_ref, dW_ref, db_ref = _composition_grads(x, targets, W, B, g)
    dx, dW, db = chunked_backward(x, targets, lse, g, layout_gather(W, B, layout), V, chunk)
    torch.testing.assert_close(dx, dx_ref, rtol=1e-10, atol=1e-12)
    torch.testing.assert_close(dW, dW_ref, rtol=1e-10, atol=1e-12)
    torch.testing.assert_close(db, db_ref, rtol=1e-10, atol=1e-12)
    if grads == "zero":
        assert not dx.any() and not dW.any() and not db.any()


# ------------------------------------------------------------------ the option
def _build(sess_config, protocol=None):
    model = MLPWithEmbedding(50)
    graph = parallax.Graph(model, optimizer=optim.GradientDescent(0.5))
    cfg = parallax.Config(run_option="HYBRID", sess_config=sess_config)
    if protocol:
        cfg.communication_config = parallax.CommunicationConfig(
            parallax.PSConfig(protocol=protocol))
    return parallax.parallel_run(graph, "localhost", parallax_config=cfg)


class _FabricReached(Exception):
    pass


@pytest.fixture
def no_nvlink_build(monkeypatch):
    """The NVLink fabric's build raises `_FabricReached`: the option was accepted, and no GPU
    is needed to see it."""
    from parallax_b200.parallel import nvlink_backend

    def reached(engine):
        raise _FabricReached()
    monkeypatch.setattr(nvlink_backend, "build_nvlink", reached)


@pytest.mark.parametrize("sc", [{}, {"full_softmax_train": "composition"}])
def test_composition_is_the_default_and_builds_anywhere(sc):
    sess, *_ = _build(dict(sc, fabric="host"))
    sess.close()


def test_fused_is_accepted_on_nvlink_with_bf16(no_nvlink_build):
    with pytest.raises(_FabricReached):
        _build({"full_softmax_train": "fused", "fabric": "nvlink", "compute_dtype": "bf16"})
    with pytest.raises(_FabricReached):
        _build({"full_softmax_train": "composition", "fabric": "nvlink"})


@pytest.mark.parametrize("value", ["Fused", "gather", "", None, 1, True])
def test_refuses_unknown_values(value):
    with pytest.raises(ValueError, match="'composition' or 'fused'"):
        _build({"full_softmax_train": value, "fabric": "host"})


@pytest.mark.parametrize("fabric", ["host", "library"])
def test_fused_refused_on_host_and_library_fabrics(fabric):
    with pytest.raises(ValueError, match="needs the NVLink fabric"):
        _build({"full_softmax_train": "fused", "fabric": fabric, "compute_dtype": "bf16"})


def test_fused_refused_with_nccl_protocol_and_without_bf16(no_nvlink_build):
    with pytest.raises(ValueError, match="protocol='nccl'"):
        _build({"full_softmax_train": "fused", "fabric": "nvlink", "compute_dtype": "bf16"},
               protocol="nccl")
    for cdt in (None, "fp32"):
        with pytest.raises(ValueError, match="needs compute_dtype='bf16'"):
            _build({"full_softmax_train": "fused", "fabric": "nvlink", "compute_dtype": cdt})
