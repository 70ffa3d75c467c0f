"""Fused LSTM layer / sampled-softmax kernels vs plain PyTorch fp32."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("dtype,tol", [(torch.float32, 2e-4), (torch.bfloat16, 6e-2)])
def test_lstm_layer_matches_reference(dtype, tol):
    from parallax_b200.ops.fused import lstm_layer, lstm_layer_reference
    torch.manual_seed(0)
    T, B, E, S, P = 5, 16, 24, 64, 24
    dev = "cuda"
    mk = lambda *s: (torch.randn(*s, device=dev) * 0.3)
    x, Wx, Wh, b, WP = mk(T, B, E), mk(E, 4 * S), mk(P, 4 * S), mk(4 * S), mk(S, P)
    c0, h0 = mk(B, S), mk(B, P)
    gH, gc, gh = mk(T, B, P), mk(B, S), mk(B, P)

    def run(fn, dt):
        args = [t.clone().to(dt).requires_grad_(True) for t in (x, Wx, Wh, b, WP)]
        c = c0.clone().requires_grad_(True)
        h = h0.clone().to(dt).requires_grad_(True)
        H, cT, hT = fn(args[0], args[1], args[2], args[3], args[4], c, h, 1.0)
        loss = (H.float() * gH).sum() + (cT.float() * gc).sum() + (hT.float() * gh).sum()
        loss.backward()
        return [H.float(), cT.float(), hT.float()] + \
            [a.grad.float() for a in args] + [c.grad.float(), h.grad.float()]
    ref = run(lstm_layer_reference, torch.float32)
    got = run(lstm_layer, dtype)
    for r, g in zip(ref, got):
        scale = float(r.abs().max()) + 1e-6
        assert float((r - g).abs().max()) <= tol * scale + tol, \
            (float((r - g).abs().max()), scale)


def test_lstm_layer_bf16_wgmma_backward_path():
    """B=128, 4S multiple of 1024: the recurrent backward product runs on the
    wgmma split-K kernel with the fused addend."""
    from parallax_b200.ops.fused import lstm_layer, lstm_layer_reference
    torch.manual_seed(0)
    T, B, E, S, P = 3, 128, 64, 256, 64
    mk = lambda *s: (torch.randn(*s, device="cuda") * 0.2)
    x, Wx, Wh, b, WP = mk(T, B, E), mk(E, 4 * S), mk(P, 4 * S), mk(4 * S), mk(S, P)
    c0, h0, gH = mk(B, S), mk(B, P), mk(T, B, P)

    def run(fn, dt):
        args = [t.clone().to(dt).requires_grad_(True) for t in (x, Wx, Wh, b, WP)]
        c = c0.clone().requires_grad_(True)
        h = h0.clone().to(dt).requires_grad_(True)
        H, cT, hT = fn(args[0], args[1], args[2], args[3], args[4], c, h, 1.0)
        (H.float() * gH).sum().backward()
        return [H.float()] + [a.grad.float() for a in args] + [h.grad.float()]
    ref = run(lstm_layer_reference, torch.float32)
    got = run(lstm_layer, torch.bfloat16)
    for r, g in zip(ref, got):
        scale = float(r.detach().abs().max()) + 1e-6
        assert float((r - g).detach().abs().max()) <= 6e-2 * scale + 6e-2


@pytest.mark.parametrize("dtype,tol", [(torch.float32, 1e-4), (torch.bfloat16, 4e-2)])
@pytest.mark.parametrize("S", [100, 1024, 8192])
def test_sampled_softmax_matches_reference(dtype, tol, S):
    from parallax_b200.ops.fused import sampled_softmax_loss, sampled_softmax_reference
    torch.manual_seed(1)
    N, P, V = 64, 32, 5000
    dev = "cuda"
    inputs = torch.randn(N, P, device=dev) * 0.5
    tw, sw = torch.randn(N, P, device=dev) * 0.5, torch.randn(S, P, device=dev) * 0.5
    tb, sb = torch.randn(N, device=dev), torch.randn(S, device=dev)
    lqt, lqs = torch.randn(N, device=dev), torch.randn(S, device=dev)
    targets = torch.randint(0, V, (N,), device=dev)
    sampled = torch.randint(0, V, (S,), device=dev)
    sampled[:5] = targets[:5]                      # accidental hits
    w = torch.rand(N, device=dev)

    def run(fn, dt):
        a = [t.clone().to(dt).requires_grad_(True) for t in (inputs, tw, sw)]
        b = [t.clone().requires_grad_(True) for t in (tb, sb)]
        loss = fn(a[0], a[1], a[2], b[0], b[1], lqt, lqs, targets, sampled)
        (loss.float() * w).sum().backward()
        return [loss.float()] + [t.grad.float() for t in a + b]
    ref = run(sampled_softmax_reference, torch.float32)
    got = run(sampled_softmax_loss, dtype)
    for r, g in zip(ref, got):
        scale = float(r.abs().max()) + 1e-6
        assert float((r - g).abs().max()) <= tol * scale + tol


@pytest.mark.parametrize("dtype,tol", [(torch.float32, 1e-4), (torch.bfloat16, 4e-2)])
@pytest.mark.parametrize("S,weighted,b_dtype", [(100, False, torch.float32),
                                               (1024, True, torch.bfloat16),
                                               (8192, False, torch.bfloat16)])
def test_sampled_softmax_head_matches_reference(dtype, tol, S, weighted, b_dtype):
    """The loss head as ONE node (true-class dot product inside the softmax kernel, one
    glue kernel in the backward pass, gradients of the looked-up rows as single [N+S, ·]
    tensors) against the fp32 PyTorch composition."""
    from parallax_b200.ops import fused
    torch.manual_seed(2)
    N, P, V = 96, 64, 5000
    dev = "cuda"
    inputs = torch.randn(N, P, device=dev) * 0.5
    w_all = torch.randn(N + S, P, device=dev) * 0.5
    b_all = torch.randn(N + S, 1, device=dev)
    logq = torch.randn(N + S, device=dev)
    targets = torch.randint(0, V, (N,), device=dev)
    sampled = torch.randint(0, V, (S,), device=dev)
    sampled[:5] = targets[:5]                      # accidental hits
    rw = torch.rand(N, device=dev) if weighted else None
    if dtype == torch.float32:
        b_dtype = torch.float32

    def run(head, dt, bdt):
        a = [t.clone().to(dt).requires_grad_(True) for t in (inputs, w_all)]
        b = b_all.clone().to(bdt).requires_grad_(True)
        if head:
            loss = fused.sampled_softmax_head(a[0], a[1], b, logq, targets, sampled, row_w=rw)
            assert loss.grad_fn.name().startswith("_SampledSoftmaxHeadFn"), loss.grad_fn
        else:
            bb = b.reshape(-1)
            loss = fused.sampled_softmax_reference(a[0], a[1][:N], a[1][N:], bb[:N], bb[N:],
                                                   logq[:N], logq[N:], targets, sampled)
            loss = (loss * rw if rw is not None else loss).mean()
        (loss.float() * 7.0).backward()
        return [loss.detach().float().reshape(1)] + [t.grad.float() for t in a] + \
            [b.grad.float()]
    ref = run(False, torch.float32, torch.float32)
    got = run(True, dtype, b_dtype)
    for r, g in zip(ref, got):
        assert r.shape == g.shape
        scale = float(r.abs().max()) + 1e-6
        assert float((r - g).abs().max()) <= tol * scale + tol, \
            (float((r - g).abs().max()), scale)


@pytest.mark.parametrize("weighted", [False, True])
def test_lm1b_model_fused_paths_match_plain_pytorch(weighted, monkeypatch):
    """LM1B forward + backward on the device (time-major rows, fused LSTM node, W_P^T on
    the side stream, fused loss head) against the same model evaluated by the PyTorch
    reference compositions on the CPU in fp32 — same weights, same negative samples."""
    from parallax_b200.models import lm1b as L
    torch.manual_seed(3)
    B, T, V = 16, 5, 400
    kw = dict(vocab_size=V, emb_size=32, state_size=64, projected_size=32, num_sampled=64,
              num_steps=T, num_shards=1, keep_prob=1.0)
    ref = L.LM1B(**kw)
    dev_m = L.LM1B(**kw)
    dev_m.load_state_dict(ref.state_dict())
    dev_m.cuda()
    x, y = torch.randint(0, V, (B, T)), torch.randint(0, V, (B, T))
    w = torch.rand(B, T) if weighted else None
    fixed = {}

    def sampler(S, Vv, device, oversample=3):
        if "s" not in fixed:
            fixed["s"] = (torch.randperm(Vv)[:S], torch.tensor(float(S + 5)))
        s, tries = fixed["s"]
        return s.to(device), tries.to(device)
    monkeypatch.setattr(L, "log_uniform_sample_unique", sampler)
    out_r = ref(x, y, w)
    out_r["loss"].backward()
    out_d = dev_m(x.cuda(), y.cuda(), None if w is None else w.cuda())
    assert out_d["loss"].grad_fn.name().startswith("_SampledSoftmaxHeadFn")
    out_d["loss"].backward()
    torch.cuda.synchronize()
    assert abs(float(out_r["loss"]) - float(out_d["loss"])) < 1e-3
    for k in ("final_state_c", "final_state_h"):
        assert torch.allclose(out_r[k], out_d[k].cpu().float(), atol=1e-4)
    for (n, p), (_, q) in zip(ref.named_parameters(), dev_m.named_parameters()):
        g_r = p.grad.to_dense() if p.grad.is_sparse else p.grad
        g_d = q.grad.to_dense() if q.grad.is_sparse else q.grad
        scale = float(g_r.abs().max()) + 1e-6
        assert float((g_r - g_d.cpu().float()).abs().max()) <= 2e-4 * scale + 1e-5, n
