"""Dense linear cross-entropy: the fused head (`parallax.nn.linear_cross_entropy` on its fused path,
`kernels/linear_xent.cu`) against the composition
``(cross_entropy(linear(x, W, b).float(), t, reduction="none") * w).sum()``, on one GPU, bf16.

Op arms, at (N, K, V, bias): (6400, 512, 7709, none) and (6400, 1024, 36548, none) (NMT, batch
128 × 50), (3968, 2400, 20000, bf16) (skip-thoughts default config, one decoder), (1216, 1024,
30522, bf16) (BERT's MLM head at the benchmark batch).  Forward (no_grad) and forward + backward
are timed with CUDA events, arms alternating, median (min–max) of --rounds rounds of --iters
calls.  TFLOP/s count 2·N·V·K for the forward and 6·N·V·K for forward + backward.  The logits
kernel alone (whole N as one chunk where the scratch allows, else the default chunk) is timed
against `torch.mm` of the same product into bf16.  Peak-allocation growth over one forward +
backward comes from the caching allocator.
Model arms (--model-rounds > 0): an NMT training step at the wmt16 shape with --vocab words and
the skip-thoughts default-config training step, through `parallel_run` (NVLink fabric, bf16);
each arm runs in a process of its own, the composition forced there by patching
`linear_xent_applies`.  Reported: ms per step, peak allocation, the first losses.
Usage: python tools/bench_linear_xent.py [--rounds 5] [--model-rounds 2]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = [(6400, 512, 7709, None), (6400, 1024, 36548, None), (3968, 2400, 20000, "bf16"),
          (1216, 1024, 30522, "bf16")]


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:           # report, do not guess
        return "unavailable (%s)" % e


def _events_ms(fn, iters):
    import torch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def _stat(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs)}


def op_arms(rounds, iters):
    import torch
    from parallax_b200.ops import fused
    out = []
    for N, K, V, bias in SHAPES:
        torch.manual_seed(0)
        x = (torch.randn(N, K, device="cuda") * 0.5).bfloat16().requires_grad_(True)
        w = (torch.randn(V, K, device="cuda") / K ** 0.5).bfloat16().requires_grad_(True)
        b = torch.randn(V, device="cuda").bfloat16().requires_grad_(True) if bias else None
        t = torch.randint(0, V, (N,), device="cuda")
        rw = torch.rand(N, device="cuda")
        assert fused.linear_xent_applies(x, w, b)
        params = [p for p in (x, w, b) if p is not None]

        def fused_fb():
            fused.linear_cross_entropy(x, t, w, b, rw)[0].backward()

        def comp_fb():
            fused.linear_cross_entropy_reference(x, t, w, b, rw)[0].backward()

        def fused_f():
            with torch.no_grad():
                fused.linear_cross_entropy(x, t, w, b, rw)

        def comp_f():
            with torch.no_grad():
                fused.linear_cross_entropy_reference(x, t, w, b, rw)
        arms = {"fused_fwd": fused_f, "comp_fwd": comp_f, "fused_fwd_bwd": fused_fb,
                "comp_fwd_bwd": comp_fb}
        for fn in arms.values():
            fn()
        times = {k: [] for k in arms}
        for _ in range(rounds):
            for k, fn in arms.items():
                for p in params:
                    p.grad = None
                times[k].append(_events_ms(fn, iters))
        peak = {}
        for k in ("fused_fwd_bwd", "comp_fwd_bwd"):
            for p in params:
                p.grad = None
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            arms[k]()
            torch.cuda.synchronize()
            peak[k] = (torch.cuda.max_memory_allocated() - base) / 2**20
        # the logits kernel alone against torch.mm into bf16
        L = fused._lib()
        n = fused.linear_xent_chunk_rows(N, V)
        vp = (V + 7) // 8 * 8
        nvt = (V + 255) // 256
        S = torch.empty(n, vp, device="cuda")
        part = torch.empty(n, nvt, 2, device="cuda")
        tgt = torch.empty(n, device="cuda")
        xd, wd = x.detach(), w.detach()
        kind = 0 if b is None else 1

        def logits():
            fused._check(L.px_linear_xent_logits(
                fused._p(xd), n, K, fused._p(wd), V, None if b is None else fused._p(b), kind,
                fused._p(t), fused._p(S), vp, fused._p(part), fused._p(tgt), fused._stream()))

        def mm():
            torch.mm(xd[:n], wd.t())
        logits()
        mm()
        lk, mk = [], []
        for _ in range(rounds):
            lk.append(_events_ms(logits, iters))
            mk.append(_events_ms(mm, iters))
        fl = 2.0 * N * V * K
        rec = {"N": N, "K": K, "V": V, "bias": bias or "none", "chunk_rows": n}
        for k, v in times.items():
            s = _stat(v)
            s["tflops"] = (fl if k.endswith("fwd") else 3 * fl) / (s["median"] * 1e-3) / 1e12
            rec[k + "_ms"] = s
        rec["logits_kernel_ms"] = _stat(lk)
        rec["logits_kernel_tflops"] = 2.0 * n * V * K / (rec["logits_kernel_ms"]["median"] * 1e-3) / 1e12
        rec["torch_mm_bf16_ms"] = _stat(mk)
        rec["peak_growth_mb"] = peak
        rec["fp32_logits_mb"] = N * V * 4 / 2**20
        print(json.dumps(rec), flush=True)
        out.append(rec)
        del x, w, b, S, part, tgt
        torch.cuda.empty_cache()
    return out


def model_step(which, composition, steps, vocab):
    """one arm in this process: ms per step after 2 warm-up steps, peak allocation, losses"""
    import torch
    import parallax_b200 as parallax
    from parallax_b200.ops import fused
    if composition:
        fused.linear_xent_applies = lambda *a, **k: False
    torch.manual_seed(0)
    cfg = parallax.Config(search_partitions=False, sess_config={"fabric": "nvlink",
                                                                "compute_dtype": "bf16"})
    if which == "nmt":
        import parallax_b200.models.nmt as nmt
        hp = nmt.create_hparams(standard="wmt16", dropout=0.0)
        nmt.extend_hparams(hp, vocab, vocab)
        m = nmt.create_model(hp)
        sess, *_ = parallax.parallel_run(nmt.nmt_graph(m, hp), "localhost:0", parallax_config=cfg)
        g = torch.Generator().manual_seed(1)
        B, S, T = 128, 50, 50
        feed = {"source": [torch.randint(3, vocab, (B, S), generator=g)],
                "target_input": [torch.randint(3, vocab, (B, T), generator=g)],
                "target_output": [torch.randint(3, vocab, (B, T), generator=g)],
                "source_sequence_length": [torch.randint(S // 2, S + 1, (B,), generator=g)],
                "target_sequence_length": [torch.randint(T // 2, T + 1, (B,), generator=g)]}
    else:
        from parallax_b200.models import skip_thoughts as st
        mc = st.model_config()
        model = st.SkipThoughtsModel(mc)
        sess, *_ = parallax.parallel_run(st.skip_thoughts_graph(model), "localhost:0",
                                         parallax_config=cfg)
        g = torch.Generator().manual_seed(1)
        B, T = mc.batch_size, 31

        def ids_mask():
            lens = torch.randint(T // 2, T + 1, (B,), generator=g)
            mask = (torch.arange(T)[None, :] < lens[:, None]).to(torch.int64)
            return torch.randint(1, mc.vocab_size, (B, T), generator=g) * mask, mask
        (ei, em), (pi, pm), (qi, qm) = ids_mask(), ids_mask(), ids_mask()
        feed = {"encode_ids": [ei], "encode_mask": [em], "decode_pre_ids": [pi],
                "decode_pre_mask": [pm], "decode_post_ids": [qi], "decode_post_mask": [qm]}
    losses = []
    for _ in range(2):
        losses.append(float(sess.run(["loss", "train_op"], feed)[0][0]))
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        losses.append(float(sess.run(["loss", "train_op"], feed)[0][0]))
    b.record()
    b.synchronize()
    rec = {"ms_per_step": a.elapsed_time(b) / steps,
           "peak_mb": torch.cuda.max_memory_allocated() / 2**20, "losses": losses[:3]}
    sess.close()
    return rec


def model_arms(rounds, steps, vocab):
    out = {}
    for which in ("nmt", "skip_thoughts"):
        for _ in range(rounds):
            for arm in ("fused", "composition"):
                r = subprocess.run([sys.executable, __file__, "--arm", which, arm, "--steps",
                                    str(steps), "--vocab", str(vocab)], capture_output=True,
                                   text=True)
                if r.returncode != 0:
                    raise RuntimeError(r.stderr[-3000:])
                rec = json.loads(r.stdout.strip().splitlines()[-1])
                out.setdefault(which, {}).setdefault(arm, []).append(rec)
        summary = {arm: {"ms_per_step": _stat([r["ms_per_step"] for r in recs]),
                         "peak_mb": max(r["peak_mb"] for r in recs),
                         "first_losses": recs[0]["losses"]}
                   for arm, recs in out[which].items()}
        print(json.dumps({"model": which, **summary}), flush=True)
        out[which] = summary
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--model-rounds", type=int, default=2)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--vocab", type=int, default=36548)
    ap.add_argument("--skip-ops", action="store_true")
    ap.add_argument("--arm", nargs=2, default=None)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if a.arm:
        print(json.dumps(model_step(a.arm[0], a.arm[1] == "composition", a.steps, a.vocab)))
        return
    res = {"gpu": gpu_info()}
    print(json.dumps(res), flush=True)
    if not a.skip_ops:
        res["ops"] = op_arms(a.rounds, a.iters)
    if a.model_rounds:
        res["models"] = model_arms(a.model_rounds, a.steps, a.vocab)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
