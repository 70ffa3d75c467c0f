"""NMT's layer-normalised LSTM: the fused node (`ops.fused.ln_lstm_layer`) against the
composition (`LayerNormLSTM._composition`, eager PyTorch one time step at a time), on one GPU.

Layer arms: B 128, T 50, bf16, ragged lengths from a seed, an initial state, at U 512 (iwslt15,
I 512) and U 1024 (wmt16, I 1024).  Forward (autograd recording, as in training) and forward +
backward are timed with CUDA events over --iters calls, arms alternating, median (min–max) of
--rounds rounds.  GPU launches per time step come from torch.profiler in a separate pass.
Decoder arms: the attention decoder of iwslt15 (U 512, 2 layers, scaled_luong) and wmt16 (U 1024,
4 layers, normed_bahdanau) with unit_type=layer_norm_lstm, B 128, S = T = 50, bf16, the fused
node (`Decoder.forward`) against `Decoder._composition`, timed the same way.
Model arm (--model-rounds > 0): a whole NMT training step through `parallel_run` (NVLink fabric,
bf16) for iwslt15 and wmt16 with unit_type=layer_norm_lstm on a fixed synthetic batch
(B 128, S = T = 50, vocabularies of --vocab words), with the fused nodes and with every
LayerNormLSTM and the decoder patched to their compositions; each arm runs in a process of its own, arms
alternating, and reports its step time and peak allocation.
Outputs are compared at the timed sizes: layer outputs and gradients, and the model's losses.
Usage: python tools/bench_ln_lstm.py [--rounds 5] [--model-rounds 2] [--out FILE]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

LAYERS = {"iwslt15": 512, "wmt16": 1024}


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
def layer_setup(U, B=128, T=50, seed=0):
    import torch
    from parallax_b200.models.nmt.model import LayerNormLSTM
    torch.manual_seed(seed)
    m = LayerNormLSTM(U, U).cuda()
    with torch.no_grad():
        m.kernel.weight.uniform_(-0.1, 0.1)
    m = m.to(torch.bfloat16)
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    x = torch.randn(B, T, U, device="cuda", generator=g).to(torch.bfloat16).requires_grad_(True)
    h0 = (torch.rand(B, U, device="cuda", generator=g) * 2 - 1).to(torch.bfloat16)
    c0 = torch.randn(B, U, device="cuda", generator=g).to(torch.bfloat16)
    lengths = torch.randint(T // 2, T + 1, (B,), generator=torch.Generator().manual_seed(seed + 2))
    lengths[0] = T
    r = torch.randn(B, T, U, device="cuda", generator=g).to(torch.bfloat16)
    return m, x, (h0.requires_grad_(True), c0.requires_grad_(True)), lengths.cuda(), r


def decoder_setup(name, B=128, S=50, T=50, seed=0):
    import torch
    import parallax_b200.models.nmt as nmt
    torch.manual_seed(seed)
    hp = nmt.create_hparams(standard=name, dropout=0.0, unit_type="layer_norm_lstm")
    nmt.extend_hparams(hp, 64, 64)
    m = nmt.create_model(hp).cuda().to(torch.bfloat16)
    g = torch.Generator().manual_seed(seed + 1)
    src = torch.randint(3, 64, (B, S), generator=g).cuda()
    sl = torch.randint(S // 2, S + 1, (B,), generator=g)
    sl[0] = S
    with torch.no_grad():
        memory, state = m.encode(src, sl.cuda())
    keys, values, pad = memory
    memory = (keys.detach().requires_grad_(True), values.detach().requires_grad_(True), pad)
    cells = [tuple(x.detach().requires_grad_(True) for x in c) for c in state["cells"]]
    state = {"cells": cells, "attention": state["attention"]}
    emb = (torch.randn(B, T, hp.num_units, device="cuda", generator=torch.Generator(
        device="cuda").manual_seed(seed + 2)) * 0.1).to(torch.bfloat16).requires_grad_(True)
    r = torch.randn(B, T, hp.num_units, device="cuda").to(torch.bfloat16)
    return m.decoder, emb, state, memory, r


def decoder_call(arm, setup, backward):
    dec, emb, state, memory, r = setup
    out = (dec.forward if arm == "fused" else dec._composition)(emb, state, memory)
    if backward:
        (out * r).float().sum().backward()
    return out


def layer_call(arm, setup, backward):
    m, x, state, lengths, r = setup
    fn = m.forward if arm == "fused" else m._composition
    out, (h, c) = fn(x, state, lengths)
    if backward:
        ((out * r).float().sum() + h.float().sum() + c.float().sum()).backward()
    return out, h, c


def time_arms(call, backward, rounds, iters, warmup):
    import torch
    arms = ("fused", "composition")
    for a in arms:
        for _ in range(warmup):
            call(a, backward)
    torch.cuda.synchronize()
    res = {a: [] for a in arms}
    for k in range(rounds):
        for a in (arms if k % 2 == 0 else arms[::-1]):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                call(a, backward)
            e1.record()
            torch.cuda.synchronize()
            res[a].append(e0.elapsed_time(e1) / iters)
    return {a: {"median_ms": statistics.median(v), "min_ms": min(v), "max_ms": max(v)}
            for a, v in res.items()}


def count_launches(call, arm, backward):
    """GPU activities (kernels, memcpy, memset) of one call, from torch.profiler"""
    import torch
    from torch.profiler import profile, ProfilerActivity
    call(arm, backward)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call(arm, backward)
        torch.cuda.synchronize()
    return sum(e.count for e in prof.key_averages()
               if e.device_type == torch.autograd.DeviceType.CUDA)


def compare_layer(setup):
    """relative Frobenius differences of the outputs and gradients of the two arms"""
    import torch
    m, x, state, lengths, r = setup
    leaves = [x, *state] + list(m.parameters())
    outs = {}
    for arm in ("fused", "composition"):
        out, h, c = layer_call(arm, setup, False)
        loss = (out * r).float().sum() + h.float().sum() + c.float().sum()
        outs[arm] = [t.detach().float() for t in (out, h, c)] + \
            [g.float() for g in torch.autograd.grad(loss, leaves)]
    rel = [float((a - b).norm() / b.norm().clamp_min(1e-30))
           for a, b in zip(outs["fused"], outs["composition"])]
    return {"out": rel[0], "h_T": rel[1], "c_T": rel[2], "max_grad": max(rel[3:])}


# ---------------------------------------------------------------------------
# model arm (one process per arm)
# ---------------------------------------------------------------------------
def model_arm(name, arm, steps, warmup, vocab):
    import torch
    import parallax_b200 as parallax
    import parallax_b200.models.nmt as nmt
    from parallax_b200.models.nmt import model as nmt_model
    if arm == "composition":
        nmt_model.LayerNormLSTM.forward = nmt_model.LayerNormLSTM._composition
        nmt_model.Decoder.forward = nmt_model.Decoder._composition
    torch.manual_seed(0)
    hp = nmt.create_hparams(standard=name, dropout=0.0, unit_type="layer_norm_lstm")
    nmt.extend_hparams(hp, vocab, vocab)
    m = nmt.create_model(hp)
    sess, *_ = parallax.parallel_run(
        nmt.nmt_graph(m, hp), "localhost:0",
        parallax_config=parallax.Config(search_partitions=False, sess_config={
            "fabric": "nvlink", "compute_dtype": "bf16"}))
    g = torch.Generator().manual_seed(1)
    B, S, T = 128, 50, 50
    sl = torch.randint(S // 2, S + 1, (B,), generator=g)
    tl = torch.randint(T // 2, T + 1, (B,), generator=g)
    feed = {"source": [torch.randint(3, vocab, (B, S), generator=g)],
            "target_input": [torch.randint(3, vocab, (B, T), generator=g)],
            "target_output": [torch.randint(3, vocab, (B, T), generator=g)],
            "source_sequence_length": [sl], "target_sequence_length": [tl]}
    losses = []
    for _ in range(warmup):
        losses.append(float(sess.run(["loss", "train_op"], feed)[0][0]))
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        sess.run(["loss", "train_op"], feed)
    e1.record()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() / 2 ** 20
    sess.close()
    print(json.dumps({"config": name, "arm": arm, "step_ms": e0.elapsed_time(e1) / steps,
                      "peak_alloc_mb": peak, "losses": losses}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--layers", default=",".join(LAYERS))
    ap.add_argument("--decoders", default="iwslt15,wmt16")
    ap.add_argument("--model-rounds", type=int, default=2)
    ap.add_argument("--model-configs", default="iwslt15,wmt16")
    ap.add_argument("--model-steps", type=int, default=3)
    ap.add_argument("--model-warmup", type=int, default=2)
    ap.add_argument("--vocab", type=int, default=8192)
    ap.add_argument("--model-arm", help=argparse.SUPPRESS)
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    a = ap.parse_args()
    if a.model_arm:
        name, arm = a.model_arm.split(":")
        return model_arm(name, arm, a.model_steps, a.model_warmup, a.vocab)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_ln_lstm.py needs a CUDA device")
    result = {"B": 128, "T": 50, "dtype": "bf16", "gpu": gpu_info(), "layer": {}, "decoder": {}}
    for name in [s for s in a.layers.split(",") if s]:
        U = LAYERS[name]
        setup = layer_setup(U)
        T = setup[1].shape[1]
        call = lambda arm, bwd: layer_call(arm, setup, bwd)
        r = {"U": U, "I": U, "fwd": time_arms(call, False, a.rounds, a.iters, a.warmup),
             "fwd_bwd": time_arms(call, True, a.rounds, a.iters, a.warmup)}
        for arm in ("fused", "composition"):
            r["launches_per_step_" + arm] = {
                "fwd": count_launches(call, arm, False) / T,
                "fwd_bwd": count_launches(call, arm, True) / T}
        r["rel_diff_fused_vs_composition"] = compare_layer(setup)
        result["layer"][name] = r
        print(name, json.dumps(r), flush=True)
        del setup, call
        torch.cuda.empty_cache()
    for name in [s for s in a.decoders.split(",") if s]:
        setup = decoder_setup(name)
        T = setup[1].shape[1]
        call = lambda arm, bwd: decoder_call(arm, setup, bwd)
        r = {"fwd": time_arms(call, False, a.rounds, a.iters, a.warmup),
             "fwd_bwd": time_arms(call, True, a.rounds, a.iters, a.warmup)}
        for arm in ("fused", "composition"):
            r["launches_per_step_" + arm] = {
                "fwd": count_launches(call, arm, False) / T,
                "fwd_bwd": count_launches(call, arm, True) / T}
        result["decoder"][name] = r
        print("decoder", name, json.dumps(r), flush=True)
        del setup, call
        torch.cuda.empty_cache()
    if a.model_rounds > 0:
        result["model"] = {"vocab": a.vocab}
        arms = ("fused", "composition")
        for name in [s for s in a.model_configs.split(",") if s]:
            runs, peaks, losses = {x: [] for x in arms}, {}, {}
            for k in range(a.model_rounds):
                for arm in (arms if k % 2 == 0 else arms[::-1]):
                    p = subprocess.run([sys.executable, os.path.abspath(__file__), "--model-arm",
                                        "%s:%s" % (name, arm), "--model-steps",
                                        str(a.model_steps), "--model-warmup",
                                        str(a.model_warmup), "--vocab", str(a.vocab)],
                                       capture_output=True, text=True)
                    line = [ln for ln in p.stdout.splitlines() if ln.startswith("{")]
                    if p.returncode != 0 or not line:
                        raise SystemExit("model arm %s %s failed:\n%s" % (name, arm,
                                                                          p.stderr[-3000:]))
                    d = json.loads(line[-1])
                    runs[arm].append(d["step_ms"])
                    peaks[arm] = d["peak_alloc_mb"]
                    losses[arm] = d["losses"]
                    print("model", d, flush=True)
            result["model"][name] = {arm: {"median_ms": statistics.median(v), "runs_ms": v,
                                           "peak_alloc_mb": peaks[arm]}
                                     for arm, v in runs.items()}
            result["model"][name]["losses"] = losses
        result["gpu_after"] = gpu_info()
    print(json.dumps(result))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
