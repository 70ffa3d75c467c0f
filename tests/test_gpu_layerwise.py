"""Layer-wise optimizers (LARS, LAMB) on the NVLink fabric: the reduce, norm, all-reduce and
update passes against `optim.apply_dense_` per tensor on simulated worlds, the engine against
the host fabric, CUDA-graph replay, run-to-run reproducibility, and the refusal of kinds 12
and 13 by the elementwise entry points."""
import ctypes

import numpy as np
import pytest
import torch

import parallax_b200 as parallax
from parallax_b200 import optim
from tests.test_layerwise_cpu import DenseNet, _batch

pytestmark = pytest.mark.gpu

MODE_FUSED, MODE_REDUCE, MODE_UPDATE = 0, 1, 2


def _opt(kind):
    """`kind`: "lars", "lars_nesterov" or "lamb"."""
    if kind.startswith("lars"):
        return optim.Lars(0.5, momentum=0.9, weight_decay=1e-3, eeta=0.02, epsilon=1e-6,
                          skip_list=["skip"], use_nesterov=kind == "lars_nesterov")
    return optim.Lamb(0.05, weight_decay=0.01, exclude_from_weight_decay=["nodecay", "skip"],
                      exclude_from_layer_adaptation=["skip"])


def _shapes(world, vn):
    """(name, numel): a tensor straddling several slices, a numel that is not a multiple of
    the vector width, a scalar, a zero bias, a tensor without gradient, a tensor excluded from
    the trust ratio and, with the 110 small ones, more than 100 segments."""
    big = world * vn * 32 * 3 + 5
    items = [("big", big), ("odd", 3 * vn + 1), ("scalar", 1), ("zero_bias.nodecay", 40),
             ("nograd", 2 * vn), ("skip_me", 17)]
    items += [("small%d" % i, 1 + (i * 7) % 29) for i in range(110)]
    return items


def _layout(items, world, vn):
    off, out = 0, []
    for name, numel in items:
        out.append((name, off, numel))
        off += (numel + vn - 1) // vn * vn
    q = world * vn * 32
    return out, (off + q - 1) // q * q


@pytest.mark.parametrize("world", [1, 2, 4, 8])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("variant", ["lars", "lars_nesterov", "lamb"])
def test_passes_match_oracle(world, dtype, variant):
    from tests.gpu_utils import make_world
    from parallax_b200.parallel import nvops
    from parallax_b200.parallel.symmetric import CH_COMM, CH_SMALL
    opt = _opt(variant)
    kind = opt.kind
    vn = 4 if dtype == torch.float32 else 8
    items, n = _layout(_shapes(world, vn), world, vn)
    sl = n // world
    fabs = make_world(world)
    gb = [f.heap.alloc(n * 4, "g") for f in fabs]
    pb = [f.heap.alloc(n * 4, "p") for f in fabs]
    gen = torch.Generator(device="cuda").manual_seed(7)
    w0 = torch.zeros(n, device="cuda")
    for name, off, numel in items:
        if name != "zero_bias.nodecay":
            w0[off:off + numel] = torch.randn(numel, device="cuda", generator=gen)
    w0 = w0.to(dtype).float()
    gsum = torch.zeros(n, device="cuda")
    for r in range(world):
        pb[r].tensor(dtype, n).copy_(w0)
        g = (torch.randn(n, device="cuda", generator=gen) * 0.3)
        for name, off, numel in items:
            if name == "nograd":
                g[off:off + numel] = 0
        g = g.to(dtype)
        gb[r].tensor(dtype, n).copy_(g)
        gsum += g.float()
    steps = 2
    init = opt.slot_init()
    master = [w0[r * sl:(r + 1) * sl].clone() for r in range(world)]
    slots = [[torch.full((sl,), v, device="cuda") for v in init] for _ in range(world)]
    red = [torch.full((sl,), float("nan"), device="cuda") for _ in range(world)]
    flags = [opt.layer_flags(name) for name, _, _ in items]
    maps = [nvops.LayerwiseMap([(o, k) for _, o, k in items], r * sl, sl, vn, flags, "cuda",
                               chunk=64) for r in range(world)]
    assert maps[0].nseg > 100
    ref_w = {name: w0[off:off + numel].clone() for name, off, numel in items}
    ref_s = {name: tuple(torch.full((numel,), v, device="cuda") for v in init)
             for name, _, numel in items}
    for step in range(1, steps + 1):
        hp_list = opt.hyper(step)
        hp = torch.tensor(hp_list, device="cuda")
        for r, f in enumerate(fabs):
            nvops.dense_step(f.heap, gb[r].c_ptrs(), pb[r].c_ptrs(), master[r], slots[r][0],
                             None, None, red[r], hp, None, None, n, 1.0 / world, 0.0, kind,
                             MODE_REDUCE, dtype, CH_COMM, max_blocks=4, stream=f.comm_stream)
        torch.cuda.synchronize()
        for r, f in enumerate(fabs):
            s1 = slots[r][1] if len(slots[r]) > 1 else None
            nvops.layerwise_norm(red[r], master[r], slots[r][0], s1, hp, None, maps[r], kind,
                                 dtype, max_blocks=4, stream=f.comm_stream)
        torch.cuda.synchronize()
        if world > 1:
            for r, f in enumerate(fabs):
                nvops.allreduce_oneshot(f.heap, maps[r].sums, maps[r].total, f.small_stage,
                                        2 * maps[r].nseg, torch.float32, 1.0, CH_SMALL,
                                        stream=f.comm_stream)
            torch.cuda.synchronize()
        totals = [m.total if world > 1 else m.sums for m in maps]
        for r in range(1, world):
            assert torch.equal(totals[r], totals[0])
        # every trust ratio within 1e-5 of fp64 (from the fp64 norms of the oracle's inputs)
        gmean = gsum / world
        tot = totals[0].double().view(-1, 2).cpu()
        for i, (name, off, numel) in enumerate(items):
            w = ref_w[name].double()
            g = gmean[off:off + numel].double()
            if kind == "lars":
                x = g
            else:
                m = ref_s[name][0].double() * opt.beta1 + (1 - opt.beta1) * g
                v = ref_s[name][1].double() * opt.beta2 + (1 - opt.beta2) * g * g
                x = (m * hp_list[optim.HP_BC1]) / ((v * hp_list[optim.HP_BC2]).sqrt() +
                                                   opt.epsilon)
                if flags[i] & optim.LW_DECAY:
                    x = x + opt.weight_decay * w
            hpn = opt.hyper_for(name, step)
            want = optim.trust_ratio(kind, float(w.norm()), float(x.norm()), hpn)
            got = optim.trust_ratio(kind, float(tot[i, 0]) ** 0.5, float(tot[i, 1]) ** 0.5, hpn)
            assert abs(got - want) <= 1e-5 * abs(want), (name, got, want)
        for r, f in enumerate(fabs):
            s1 = slots[r][1] if len(slots[r]) > 1 else None
            nvops.layerwise_update(f.heap, pb[r].c_ptrs(), red[r], master[r], slots[r][0], s1,
                                   None, hp, None, maps[r], totals[r], n, 0.0, kind, dtype,
                                   CH_COMM, max_blocks=4, stream=f.comm_stream)
        torch.cuda.synchronize()
        for name, off, numel in items:
            optim.apply_dense_(kind, ref_w[name], gmean[off:off + numel], ref_s[name],
                               opt.hyper_for(name, step))
    got_w = torch.cat(master)
    got_s = [torch.cat([s[i] for s in slots]) for i in range(len(init))]
    for name, off, numel in items:
        torch.testing.assert_close(got_w[off:off + numel], ref_w[name], rtol=1e-5, atol=1e-6)
        for i in range(len(init)):
            torch.testing.assert_close(got_s[i][off:off + numel], ref_s[name][i], rtol=1e-5,
                                       atol=1e-6)
    p0 = pb[0].tensor(dtype, n).clone()
    for name, off, numel in items:
        assert torch.equal(p0[off:off + numel], got_w[off:off + numel].to(dtype)), name
    for r in range(1, world):
        assert torch.equal(pb[r].tensor(dtype, n), p0)
    for f in fabs:
        f.close()


def test_elementwise_entry_points_refuse_layerwise_kinds():
    """Kinds 12 and 13 through the fused dense step (modes 0 and 2), the async apply and the
    sparse push / owner kernels: an error, never a silent no-op or another family's rule."""
    from parallax_b200 import ops
    from parallax_b200.parallel import nvops
    from parallax_b200.parallel.symmetric import CH_COMM
    n = 4 * 32
    p = torch.zeros(n, device="cuda")
    g = torch.zeros(n, device="cuda")
    s0, s1 = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    hp = torch.zeros(optim.HP_SIZE, device="cuda")
    ptrs = (ctypes.c_void_p * 1)(g.data_ptr())
    pp = (ctypes.c_void_p * 1)(p.data_ptr())
    for kind in ("lars", "lamb"):
        for mode in (MODE_FUSED, MODE_UPDATE):
            with pytest.raises(RuntimeError, match="rc=-4"):
                nvops.dense_step(None, ptrs, pp, p, s0, s1, None, g if mode == 2 else None, hp,
                                 None, None, n, 1.0, 0.0, kind, mode, torch.float32, CH_COMM,
                                 rank=0, world=1)
        with pytest.raises(RuntimeError, match="rc=-4"):
            nvops.dense_async(g, p, pp, (ctypes.c_void_p * 1)(s0.data_ptr()),
                              (ctypes.c_void_p * 1)(s1.data_ptr()), hp, None, n, kind,
                              torch.float32, 0, 1)
    L = ops.lib()
    geom = ops.GroupGeom()
    for kid in (optim.KIND_ID["lars"], optim.KIND_ID["lamb"], 99):
        ot = (ops.OwnerTable * 1)()
        ot[0].kind = kid
        assert L.px_sparse_owner(ot, 1, 0, None, None, None, None, None, 0, ctypes.byref(geom),
                                 None, 0, 0, 1, -1, None) == -9
        pt = (ops.PushTable * 1)()
        pt[0].kind = kid
        assert L.px_sparse_push(None, 0, pt, 1, 0, 0, 0, None, None, 0, ctypes.byref(geom),
                                None, 0, 0, 1, None) == -9
    torch.cuda.synchronize()


# --------------------------------------------------------------------------- engine
def _run_dense(fabric, kind, K=None, clip=0.05, graph=False, steps=4):
    rules = [parallax.ClipByGlobalNorm(clip)] if clip is not None else []
    from tests.test_layerwise_cpu import _make_opt
    g = parallax.Graph(DenseNet(), optimizer=_make_opt(kind), grad_rules=rules,
                       ema=parallax.ExponentialMovingAverage(0.9, ["fc2.*"]))
    sc = {"fabric": fabric, "cuda_graph": graph}
    if K:
        sc["micro_batches"] = K
    cfg = parallax.Config(run_option="HYBRID", sess_config=sc)
    sess, *_ = parallax.parallel_run(g, "localhost:0", parallax_config=cfg)
    losses = []
    for s in range(steps):
        x, y = _batch(s)
        loss, _ = sess.run(["loss", "train_op"], {"x": [x], "labels": [y]})
        losses.append(loss[0])
    sd = sess.engine.state_dict()
    sess.close()
    return losses, sd


def _run_bert(fabric, K=None, graph=False, steps=4):
    from parallax_b200.models.bert import Bert, bert_graph
    torch.manual_seed(0)
    model = Bert(vocab=256, hidden=64, layers=2, heads=4, ff=128, max_len=16, num_partitions=2)
    g = bert_graph(model, 1e-3, optimizer="lamb")
    sc = {"fabric": fabric, "cuda_graph": graph}
    if K:
        sc["micro_batches"] = K
    cfg = parallax.Config(run_option="HYBRID", sess_config=sc)
    sess, *_ = parallax.parallel_run(g, "localhost:0", parallax_config=cfg)
    gen = torch.Generator().manual_seed(1)
    losses = []
    for s in range(steps):
        ids = torch.randint(5, 256, (4, 16), generator=gen)
        pos = torch.stack([torch.randperm(16, generator=gen)[:3] for _ in range(4)])
        labels = torch.gather(ids, 1, pos)
        loss, _ = sess.run(["loss", "train_op"], {"input_ids": [ids.scatter(1, pos, 4)],
                                                  "mlm_positions": [pos],
                                                  "mlm_labels": [labels]})
        losses.append(loss[0])
    sd = sess.engine.state_dict()
    sess.close()
    return losses, sd


def _same(a, b, tol, parts=("master", "ema")):
    np.testing.assert_allclose(a[0], b[0], rtol=tol[0], atol=tol[1])
    for part in parts:
        for n, w in b[1]["dense"][part].items():
            torch.testing.assert_close(a[1]["dense"][part][n], w, rtol=tol[0], atol=tol[1])
    for n, s in b[1]["dense"]["slots"].items():
        for x, y in zip(a[1]["dense"]["slots"][n], s):
            torch.testing.assert_close(x, y, rtol=tol[0], atol=tol[1])


def _bitwise(a, b):
    assert a[0] == b[0]
    for part in ("master", "ema"):
        for n, w in b[1]["dense"][part].items():
            assert torch.equal(a[1]["dense"][part][n], w), n


@pytest.mark.parametrize("kind", ["lars", "lars_nesterov", "lamb"])
@pytest.mark.parametrize("K", [None, 2])
@pytest.mark.parametrize("clip", [None, 0.05])
def test_engine_dense_model_matches_host(kind, K, clip):
    nv = _run_dense("nvlink", kind, K=K, clip=clip)
    _same(nv, _run_dense("host", kind, K=K, clip=clip), (1e-4, 1e-5))


@pytest.mark.parametrize("K", [None, 2])
def test_engine_small_bert_lamb_matches_host(K):
    """Small BERT with its LAMB recipe (clip on the dense variables, Adam on the table)."""
    nv = _run_bert("nvlink", K=K)
    host = _run_bert("host", K=K)
    _same(nv, host, (2e-4, 2e-5), parts=("master",))
    torch.testing.assert_close(nv[1]["sparse"]["word_emb.weight"]["weight"],
                               host[1]["sparse"]["word_emb.weight"]["weight"],
                               rtol=2e-4, atol=2e-5)


def test_cuda_graph_replay_is_bitwise_eager():
    for kind in ("lars", "lamb"):
        eager = _run_dense("nvlink", kind, K=2, steps=7)
        _bitwise(_run_dense("nvlink", kind, K=2, steps=7, graph=True), eager)


def test_two_runs_are_bitwise_equal():
    """The per-tensor sums are combined in a fixed order: no run-to-run difference."""
    for kind in ("lars", "lamb"):
        _bitwise(_run_dense("nvlink", kind), _run_dense("nvlink", kind))
