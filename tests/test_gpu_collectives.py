"""sm_90a collective kernels vs plain PyTorch fp32 references.  A world of W
ranks is simulated on one GPU (see tests/gpu_utils.py)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _setup(world):
    from tests.gpu_utils import make_world
    return make_world(world)


@pytest.mark.parametrize("world", [1, 2, 4, 8])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_allreduce_twoshot(world, dtype):
    from parallax_b200.parallel import nvops
    from parallax_b200.parallel.symmetric import CH_COMM
    fabs = _setup(world)
    n = world * 8 * 1000
    bufs = [f.heap.alloc(n * 4, "x") for f in fabs]
    g = torch.Generator(device="cuda").manual_seed(1)
    xs = []
    for b in bufs:
        t = b.tensor(dtype, n)
        t.copy_(torch.randn(n, device="cuda", generator=g))
        xs.append(t.float().clone())
    ref = torch.stack(xs).sum(0) / world
    sumsq = [torch.zeros(1, device="cuda") for _ in fabs]
    torch.cuda.synchronize()
    for r, f in enumerate(fabs):
        nvops.allreduce_twoshot(f.heap, bufs[r].c_ptrs(), n, dtype, 1.0 / world,
                                CH_COMM, sumsq=sumsq[r], max_blocks=4,
                                stream=f.comm_stream)
    torch.cuda.synchronize()
    tol = 1e-5 if dtype == torch.float32 else 2e-2
    for r, b in enumerate(bufs):
        torch.testing.assert_close(b.tensor(dtype, n).float(), ref, rtol=tol, atol=tol)
    total = sum(float(s) for s in sumsq)
    assert abs(total - float((bufs[0].tensor(dtype, n).float() ** 2).sum())) \
        <= 1e-2 * max(total, 1.0)
    # replicas are bitwise identical
    for b in bufs[1:]:
        assert torch.equal(b.tensor(dtype, n), bufs[0].tensor(dtype, n))
    for f in fabs:
        f.close()


@pytest.mark.parametrize("world,dtype", [(2, torch.bfloat16), (4, torch.float32),
                                         (8, torch.bfloat16)])
def test_allreduce_twoshot_bulk_tma_variant(world, dtype):
    """cp.async.bulk (TMA engine -> shared memory) variant of the reduce-scatter phase: same
    result as the register variant, several chunks per CTA so both stages are re-used."""
    from parallax_b200.parallel import nvops
    from parallax_b200.parallel.symmetric import CH_COMM
    fabs = _setup(world)
    es = 4 if dtype == torch.float32 else 2
    n = world * (8192 // es) * 5 + world * 8 * 3            # 5 full chunks + a partial one
    bufs = [f.heap.alloc(n * 4, "x") for f in fabs]
    g = torch.Generator(device="cuda").manual_seed(1)
    xs = []
    for b in bufs:
        t = b.tensor(dtype, n)
        t.copy_(torch.randn(n, device="cuda", generator=g))
        xs.append(t.float().clone())
    ref = torch.stack(xs).sum(0) / world
    torch.cuda.synchronize()
    for r, f in enumerate(fabs):
        nvops.allreduce_twoshot_bulk(f.heap, bufs[r].c_ptrs(), n, dtype, 1.0 / world, CH_COMM,
                                     max_blocks=2, stream=f.comm_stream)
    torch.cuda.synchronize()
    tol = 1e-5 if dtype == torch.float32 else 2e-2
    for b in bufs:
        torch.testing.assert_close(b.tensor(dtype, n).float(), ref, rtol=tol, atol=tol)
    for b in bufs[1:]:
        assert torch.equal(b.tensor(dtype, n), bufs[0].tensor(dtype, n))
    for f in fabs:
        f.close()


@pytest.mark.parametrize("world", [2, 8])
def test_allreduce_oneshot_repeated(world):
    from parallax_b200.parallel import nvops
    from parallax_b200.parallel.symmetric import CH_SMALL
    fabs = _setup(world)
    n = 1000
    for it in range(3):      # exercises the staging parity
        srcs = [torch.randn(n, device="cuda") + r + it for r in range(world)]
        dsts = [torch.empty(n, device="cuda") for _ in range(world)]
        torch.cuda.synchronize()
        for r, f in enumerate(fabs):
            nvops.allreduce_oneshot(f.heap, srcs[r], dsts[r], f.small_stage, n,
                                    torch.float32, 1.0, CH_SMALL, max_blocks=2,
                                    stream=f.comm_stream)
        torch.cuda.synchronize()
        ref = torch.stack(srcs).sum(0)
        for d in dsts:
            torch.testing.assert_close(d, ref, rtol=1e-5, atol=1e-5)
            assert torch.equal(d, dsts[0])
    for f in fabs:
        f.close()


@pytest.mark.parametrize("world", [2, 4])
def test_broadcast_and_allgather(world):
    from parallax_b200.parallel import nvops
    from parallax_b200.parallel.symmetric import CH_MAIN
    fabs = _setup(world)
    n = world * 4096
    bufs = [f.heap.alloc(n * 4, "x") for f in fabs]
    for r, b in enumerate(bufs):
        b.tensor(torch.float32, n).fill_(float(r + 1))
    torch.cuda.synchronize()
    for r, f in enumerate(fabs):
        nvops.broadcast(f.heap, bufs[r].c_ptrs(), n * 4, 1, CH_MAIN, 4,
                        stream=f.comm_stream)
    torch.cuda.synchronize()
    for b in bufs:
        assert float(b.tensor(torch.float32, n).min()) == 2.0
        assert float(b.tensor(torch.float32, n).max()) == 2.0
    sl = n // world
    for r, b in enumerate(bufs):
        b.tensor(torch.float32, n)[r * sl:(r + 1) * sl] = float(10 + r)
    torch.cuda.synchronize()
    for r, f in enumerate(fabs):
        nvops.allgather(f.heap, bufs[r].c_ptrs(), sl * 4, CH_MAIN, 4,
                        stream=f.comm_stream)
    torch.cuda.synchronize()
    ref = torch.arange(world, device="cuda").repeat_interleave(sl).float() + 10
    for b in bufs:
        assert torch.equal(b.tensor(torch.float32, n), ref)
    for f in fabs:
        f.close()


@pytest.mark.parametrize("world", [1, 2, 4])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("kind", ["sgd", "momentum", "adagrad", "adam", "rmsprop",
                                  "adadelta", "ftrl", "ftrl_p", "proximal_sgd",
                                  "proximal_adagrad", "adagrad_da", "centered_rmsprop"])
def test_dense_step_fused(world, dtype, kind):
    """reduce-scatter + optimizer + param all-gather in one kernel."""
    from parallax_b200 import optim
    from parallax_b200.parallel import nvops
    from parallax_b200.parallel.symmetric import CH_COMM
    fabs = _setup(world)
    opt = {"sgd": optim.GradientDescent(0.1), "momentum": optim.Momentum(0.1, 0.9, True),
           "adagrad": optim.Adagrad(0.1, 0.5), "adam": optim.Adam(0.01),
           "rmsprop": optim.RMSProp(0.01, momentum=0.9),
           "adadelta": optim.Adadelta(0.5, rho=0.9, epsilon=1e-4),
           "ftrl": optim.Ftrl(0.1, l1_regularization_strength=0.01,
                              l2_regularization_strength=0.02),
           "ftrl_p": optim.Ftrl(0.1, learning_rate_power=-0.3,
                                l1_regularization_strength=0.01),
           "proximal_sgd": optim.ProximalGradientDescent(0.1, 0.05, 0.1),
           "proximal_adagrad": optim.ProximalAdagrad(0.1, 0.5, l1_regularization_strength=0.05,
                                                     l2_regularization_strength=0.1),
           "adagrad_da": optim.AdagradDA(0.1, l1_regularization_strength=0.01,
                                         l2_regularization_strength=0.1),
           "centered_rmsprop": optim.CenteredRMSProp(0.01, momentum=0.9, epsilon=1e-3)}[kind]
    kind = opt.kind
    vn = 4 if dtype == torch.float32 else 8
    n = world * vn * 32 * 7
    sl = n // world
    es = 4 if dtype == torch.float32 else 2
    gb = [f.heap.alloc(n * es, "g") for f in fabs]
    pb = [f.heap.alloc(n * es, "p") for f in fabs]
    gen = torch.Generator(device="cuda").manual_seed(3)
    w0 = torch.randn(n, device="cuda", generator=gen)
    if dtype == torch.bfloat16:
        w0 = w0.bfloat16().float()
    master = [w0[r * sl:(r + 1) * sl].clone() for r in range(world)]
    slots = [[torch.full((sl,), v, device="cuda") for v in opt.slot_init()]
             for _ in range(world)]
    ema = [m.clone() for m in master]
    ref_w, ref_slots = w0.clone(), tuple(torch.full((n,), v, device="cuda")
                                         for v in opt.slot_init())
    ref_ema = w0.clone()
    for step in (1, 2, 3):
        grads = []
        for r in range(world):
            g = torch.randn(n, device="cuda", generator=gen)
            gb[r].tensor(dtype, n).copy_(g)
            grads.append(gb[r].tensor(dtype, n).float().clone())
            pb[r].tensor(dtype, n).zero_()
        hp_list = opt.hyper(step)
        hp = torch.tensor(hp_list, device="cuda")
        torch.cuda.synchronize()
        for r, f in enumerate(fabs):
            nvops.dense_step(f.heap, gb[r].c_ptrs(), pb[r].c_ptrs(), master[r],
                             slots[r][0] if len(slots[r]) > 0 else None,
                             slots[r][1] if len(slots[r]) > 1 else None, ema[r],
                             None, hp, None, None, n, 1.0 / world, 0.9, kind, 0,
                             dtype, CH_COMM, max_blocks=4, stream=f.comm_stream,
                             slot2=slots[r][2] if len(slots[r]) > 2 else None)
        torch.cuda.synchronize()
        gmean = torch.stack(grads).sum(0) / world
        optim.apply_dense_(kind, ref_w, gmean, ref_slots, hp_list)
        ref_ema.sub_((ref_ema - ref_w) * (1 - 0.9))
        got_master = torch.cat(master)
        torch.testing.assert_close(got_master, ref_w, rtol=2e-5, atol=2e-5)
        torch.testing.assert_close(torch.cat(ema), ref_ema, rtol=2e-5, atol=2e-5)
        for r in range(world):
            torch.testing.assert_close(pb[r].tensor(dtype, n).float(),
                                       ref_w.to(dtype).float(), rtol=1e-2, atol=1e-2)
            assert torch.equal(pb[r].tensor(dtype, n), pb[0].tensor(dtype, n))
    for f in fabs:
        f.close()


def test_dense_step_two_phase_clip():
    """REDUCE_ONLY + global-norm clip + UPDATE_PUSH equals clip-then-apply."""
    from parallax_b200 import optim
    from parallax_b200.parallel import nvops
    from parallax_b200.parallel.symmetric import CH_COMM, CH_SMALL
    world, dtype, n = 4, torch.float32, 4 * 4 * 32 * 5
    fabs = _setup(world)
    sl = n // world
    opt = optim.Adagrad(0.2, 1.0)
    gb = [f.heap.alloc(n * 4, "g") for f in fabs]
    pb = [f.heap.alloc(n * 4, "p") for f in fabs]
    gen = torch.Generator(device="cuda").manual_seed(5)
    w0 = torch.randn(n, device="cuda", generator=gen)
    master = [w0[r * sl:(r + 1) * sl].clone() for r in range(world)]
    acc = [torch.full((sl,), 1.0, device="cuda") for _ in range(world)]
    red = [torch.empty(sl, device="cuda") for _ in range(world)]
    loc = [torch.zeros(4, device="cuda") for _ in range(world)]
    tot = [torch.zeros(4, device="cuda") for _ in range(world)]
    scale = [torch.ones(1, device="cuda") for _ in range(world)]
    norm = [torch.zeros(1, device="cuda") for _ in range(world)]
    grads = []
    for r in range(world):
        g = torch.randn(n, device="cuda", generator=gen) * 3
        gb[r].tensor(dtype, n).copy_(g)
        grads.append(g)
    hp_list = opt.hyper(1)
    hp = torch.tensor(hp_list, device="cuda")
    max_norm = 10.0
    torch.cuda.synchronize()
    # phase-interleaved launches: the simulated ranks' streams share one process
    # (and possibly one hardware queue), so no rank may enqueue a later phase in
    # front of a peer's earlier one
    for r, f in enumerate(fabs):
        nvops.dense_step(f.heap, gb[r].c_ptrs(), pb[r].c_ptrs(), master[r], acc[r],
                         None, None, red[r], hp, None, loc[r], n, 1.0 / world, 0.0,
                         "adagrad", 1, dtype, CH_COMM, max_blocks=4, stream=f.comm_stream)
    for r, f in enumerate(fabs):
        nvops.allreduce_oneshot(f.heap, loc[r], tot[r], f.small_stage, 4,
                                torch.float32, 1.0, CH_SMALL, stream=f.comm_stream)
    for r, f in enumerate(fabs):
        nvops.clip_scale(tot[r], max_norm, scale[r], norm[r], loc[r], stream=f.comm_stream)
        nvops.dense_step(f.heap, gb[r].c_ptrs(), pb[r].c_ptrs(), master[r], acc[r],
                         None, None, red[r], hp, scale[r], None, n, 1.0 / world,
                         0.0, "adagrad", 2, dtype, CH_COMM, max_blocks=4,
                         stream=f.comm_stream)
    torch.cuda.synchronize()
    gmean = torch.stack(grads).sum(0) / world
    gn = float(gmean.norm())
    assert abs(float(norm[0]) - gn) < 1e-3 * gn
    gmean = gmean * (max_norm / max(gn, max_norm))
    ref_w, ref_acc = w0.clone(), torch.full((n,), 1.0, device="cuda")
    optim.apply_dense_("adagrad", ref_w, gmean, (ref_acc,), hp_list)
    torch.testing.assert_close(torch.cat(master), ref_w, rtol=1e-5, atol=1e-5)
    for r in range(world):
        torch.testing.assert_close(pb[r].tensor(dtype, n), ref_w, rtol=1e-5, atol=1e-5)
        assert float(loc[r].abs().sum()) == 0.0      # accumulator re-armed
    for f in fabs:
        f.close()
