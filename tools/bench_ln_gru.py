"""Skip-thoughts' layer-normalised GRU: the fused node (`ops.fused.ln_gru_layer`) against the
composition (`LayerNormGRU._composition`, eager PyTorch one step at a time), on one GPU.

Layer arms: B 128, I 620, T 31, bf16, ragged lengths from a seed, an initial state, at n 2400 and
at n 1200 with reverse=True.  Forward (autograd recording, as in training) and forward + backward
are timed with CUDA events over --iters calls, arms alternating, median of --rounds rounds.
Launches per time step are counted with torch.profiler in a separate pass.
Model arm (--model-rounds > 0): a skip-thoughts training step through `parallel_run` at the
default configuration (vocab 20 000, word dim 620, encoder 2400, bf16, batch 128 of length 31),
with the fused layer and with every LayerNormGRU patched to the composition; each arm runs in a
process of its own, arms alternating, median over rounds.
Outputs are compared at the timed sizes: layer outputs and gradients, and the model's losses on
the same seeded batch.
Usage: python tools/bench_ln_gru.py [--rounds 5] [--model-rounds 3] [--dry-run]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def layer_counts(B, I, T, n):
    """FLOP of the recurrent products and bytes of the cell kernels of one layer call (bf16)."""
    mm = 2 * B * n * 3 * n                       # h·w_hu (and d(hh)·w_hu^T) per step
    fwd_flop = T * mm
    bwd_flop = T * mm + mm * T                   # per-step dh products + one dw_hu GEMM
    es = 2
    cell_fwd = B * (3 * n * 4 + 3 * n * es + n * es + 2 * n * es + 16)
    cell_bwd = B * (3 * n * 4 + 16 + 3 * n * es + n * es + n * es + 2 * n * 4 + n * 4 +
                    3 * n * es + 3 * n * es + 2 * 6 * n * 4)
    return {"product_gflop_per_step": mm / 1e9, "fwd_gflop": fwd_flop / 1e9,
            "bwd_gflop": bwd_flop / 1e9, "cell_fwd_mb_per_step": cell_fwd / 1e6,
            "cell_bwd_mb_per_step": cell_bwd / 1e6}


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:           # report, do not guess
        return "unavailable (%s)" % e


# ---------------------------------------------------------------------------
# layer arms
# ---------------------------------------------------------------------------
def layer_setup(B, I, T, n, reverse, seed=0):
    import torch
    from parallax_b200.models.skip_thoughts.gru_cell import LayerNormGRU
    torch.manual_seed(seed)
    m = LayerNormGRU(I, n).cuda().to(torch.bfloat16)
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    x = torch.randn(B, T, I, device="cuda", generator=g).to(torch.bfloat16)
    h0 = (torch.rand(B, n, device="cuda", generator=g) * 2 - 1).to(torch.bfloat16)
    lengths = torch.randint(1, T + 1, (B,), generator=torch.Generator().manual_seed(seed + 2))
    lengths[0] = T
    r = torch.randn(B, T, n, device="cuda", generator=g).to(torch.bfloat16)
    return m, x.requires_grad_(True), h0.requires_grad_(True), lengths.cuda(), r, reverse


def layer_call(arm, setup, backward):
    m, x, h0, lengths, r, reverse = setup
    fn = m.forward if arm == "fused" else m._composition
    out, fin = fn(x, lengths, h0, reverse=reverse)
    if backward:
        ((out * r).float().sum() + fin.float().sum()).backward()
    return out, fin


def time_layer(setup, backward, rounds, iters, warmup):
    import torch
    arms = ("fused", "composition")
    for a in arms:
        for _ in range(warmup):
            layer_call(a, setup, backward)
    torch.cuda.synchronize()
    res = {a: [] for a in arms}
    for k in range(rounds):
        for a in (arms if k % 2 == 0 else arms[::-1]):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                layer_call(a, setup, backward)
            e1.record()
            torch.cuda.synchronize()
            res[a].append(e0.elapsed_time(e1) / iters)
    return {a: {"median_ms": statistics.median(v), "min_ms": min(v), "max_ms": max(v)}
            for a, v in res.items()}


def count_launches(setup, arm, backward):
    """GPU activities (kernels, memcpy, memset) of one call, from torch.profiler"""
    import torch
    from torch.profiler import profile, ProfilerActivity
    layer_call(arm, setup, backward)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        layer_call(arm, setup, backward)
        torch.cuda.synchronize()
    return sum(e.count for e in prof.key_averages()
               if e.device_type == torch.autograd.DeviceType.CUDA)


def compare_layer(setup):
    import torch
    m = setup[0]
    outs = {}
    for arm in ("fused", "composition"):
        m.zero_grad(set_to_none=True)
        setup[1].grad = setup[2].grad = None
        out, fin = layer_call(arm, setup, True)
        outs[arm] = [out.detach().float(), fin.detach().float(), setup[1].grad.float(),
                     m.w_hu.grad.float(), setup[2].grad.float()]
    names = ("out", "final", "dx", "dw_hu", "dh0")
    rel = {}
    for k, a, b in zip(names, outs["fused"], outs["composition"]):
        rel[k] = float((a - b).norm() / b.norm().clamp_min(1e-30))
    return rel


# ---------------------------------------------------------------------------
# model arm (one process per arm)
# ---------------------------------------------------------------------------
def model_arm(arm, steps, warmup):
    import torch
    import parallax_b200 as parallax
    from parallax_b200.models import skip_thoughts as st
    from parallax_b200.models.skip_thoughts import gru_cell
    from parallax_b200.models.skip_thoughts.input_ops import parse_example_batch
    if arm == "composition":
        gru_cell.LayerNormGRU.forward = gru_cell.LayerNormGRU._composition
    torch.manual_seed(0)
    mc = st.model_config()
    model = st.SkipThoughtsModel(mc)
    sess, *_ = parallax.parallel_run(
        st.skip_thoughts_graph(model, st.training_config()), "localhost:0",
        parallax_config=parallax.Config(search_partitions=False, sess_config={
            "fabric": "nvlink", "compute_dtype": "bf16"}))
    g = torch.Generator().manual_seed(1)
    ex = [tuple(torch.randint(1, mc.vocab_size, (31,), generator=g).tolist() for _ in range(3))
          for _ in range(mc.batch_size)]
    feed = st.feed_from_batch(parse_example_batch(ex))
    losses = []
    for _ in range(warmup):
        losses.append(float(sess.run(["loss", "train_op"], feed)[0][0]))
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        sess.run(["loss", "train_op"], feed)
    e1.record()
    torch.cuda.synchronize()
    sess.close()
    print(json.dumps({"arm": arm, "step_ms": e0.elapsed_time(e1) / steps, "losses": losses}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--B", type=int, default=128)
    ap.add_argument("--I", type=int, default=620)
    ap.add_argument("--T", type=int, default=31)
    ap.add_argument("--units", default="2400,1200r",
                    help="comma-separated n, an 'r' suffix for reverse=True")
    ap.add_argument("--model-rounds", type=int, default=3)
    ap.add_argument("--model-steps", type=int, default=10)
    ap.add_argument("--model-warmup", type=int, default=3)
    ap.add_argument("--model-arm", choices=("fused", "composition"), help=argparse.SUPPRESS)
    ap.add_argument("--dry-run", action="store_true",
                    help="print the shapes and FLOP / byte counts without a GPU")
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    a = ap.parse_args()
    if a.model_arm:
        return model_arm(a.model_arm, a.model_steps, a.model_warmup)
    cases = [(int(u.rstrip("r")), u.endswith("r")) for u in a.units.split(",")]
    result = {"B": a.B, "I": a.I, "T": a.T, "dtype": "bf16",
              "counts": {"n%d" % n: layer_counts(a.B, a.I, a.T, n) for n, _ in cases}}
    if a.dry_run:
        print(json.dumps(result, indent=1))
        return
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_ln_gru.py needs a CUDA device")
    result["gpu"] = gpu_info()
    result["layer"] = {}
    for n, rev in cases:
        key = "n%d%s" % (n, "_reverse" if rev else "")
        setup = layer_setup(a.B, a.I, a.T, n, rev)
        r = {"fwd": time_layer(setup, False, a.rounds, a.iters, a.warmup),
             "fwd_bwd": time_layer(setup, True, a.rounds, a.iters, a.warmup)}
        for arm in ("fused", "composition"):
            r["launches_per_step_" + arm] = {
                "fwd": count_launches(setup, arm, False) / a.T,
                "fwd_bwd": count_launches(setup, arm, True) / a.T}
        r["rel_diff_fused_vs_composition"] = compare_layer(setup)
        result["layer"][key] = r
        print(key, json.dumps(r), flush=True)
        del setup
        torch.cuda.empty_cache()
    if a.model_rounds > 0:
        runs = {"fused": [], "composition": []}
        losses = {}
        arms = ("fused", "composition")
        for k in range(a.model_rounds):
            for arm in (arms if k % 2 == 0 else arms[::-1]):
                p = subprocess.run([sys.executable, os.path.abspath(__file__), "--model-arm", arm,
                                    "--model-steps", str(a.model_steps), "--model-warmup",
                                    str(a.model_warmup)], capture_output=True, text=True)
                line = [ln for ln in p.stdout.splitlines() if ln.startswith("{")]
                if p.returncode != 0 or not line:
                    raise SystemExit("model arm %s failed:\n%s" % (arm, p.stderr[-3000:]))
                d = json.loads(line[-1])
                runs[arm].append(d["step_ms"])
                losses[arm] = d["losses"]
                print("model", arm, d, flush=True)
        result["model"] = {arm: {"median_ms": statistics.median(v), "runs_ms": v}
                           for arm, v in runs.items()}
        result["model"]["losses"] = losses
        result["gpu_after"] = gpu_info()
    print(json.dumps(result))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
