"""NMT attention decoder: the fused node (`ops.fused.nmt_attention_decoder`) against the
composition (`Decoder._composition`, eager PyTorch one time step at a time), on one GPU.

Decoder arms: the decoder shapes of three standard configurations at batch 128, S = T = 50, bf16,
ragged source lengths from a seed, dropout off:
  iwslt15            U 512,  2 layers, memory 1024, scaled_luong,    standard
  wmt16              U 1024, 4 layers, memory 2048, normed_bahdanau, standard
  wmt16_gnmt_4_layer U 1024, bottom layer (+3 cuDNN layers), memory 1024, normed_bahdanau, gnmt_v2
Forward (autograd recording, as in training) and forward + backward of `Decoder.forward` are
timed with CUDA events over --iters calls, arms alternating, median (min–max) of --rounds
rounds.  GPU launches per time step come from torch.profiler in a separate pass, and the growth
of peak allocation over one forward + backward from the caching allocator's statistics.
Model arm (--model-rounds > 0): a whole NMT training step through `parallel_run` (NVLink fabric,
bf16) for iwslt15 and wmt16 on a fixed synthetic batch, vocabularies of --vocab words each;
each arm runs in a process of its own, arms alternating.
Usage: python tools/bench_nmt_decoder.py [--rounds 5] [--model-rounds 3]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = ("iwslt15", "wmt16", "wmt16_gnmt_4_layer")


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:           # report, do not guess
        return "unavailable (%s)" % e


def _hparams(name, vocab):
    import parallax_b200.models.nmt as nmt
    hp = nmt.create_hparams(standard=name, dropout=0.0)
    nmt.extend_hparams(hp, vocab, vocab)
    return hp


def decoder_setup(name, B=128, S=50, T=50, seed=0):
    import torch
    import parallax_b200.models.nmt as nmt
    torch.manual_seed(seed)
    hp = _hparams(name, 64)
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
    fn = dec.forward if arm == "fused" else dec._composition
    out = fn(emb, state, memory)
    if backward:
        (out * r).float().sum().backward()
    return out


def time_decoder(setup, backward, rounds, iters, warmup):
    import torch
    arms = ("fused", "composition")
    for a in arms:
        for _ in range(warmup):
            decoder_call(a, setup, backward)
    torch.cuda.synchronize()
    res = {a: [] for a in arms}
    for k in range(rounds):
        for a in (arms if k % 2 == 0 else arms[::-1]):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                decoder_call(a, setup, backward)
            e1.record()
            torch.cuda.synchronize()
            res[a].append(e0.elapsed_time(e1) / iters)
    return {a: {"median_ms": statistics.median(v), "min_ms": min(v), "max_ms": max(v)}
            for a, v in res.items()}


def count_launches(setup, arm, backward):
    """GPU activities (kernels, memcpy, memset) of one call, from torch.profiler"""
    import torch
    from torch.profiler import profile, ProfilerActivity
    decoder_call(arm, setup, backward)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        decoder_call(arm, setup, backward)
        torch.cuda.synchronize()
    return sum(e.count for e in prof.key_averages()
               if e.device_type == torch.autograd.DeviceType.CUDA)


def peak_growth(setup, arm):
    """growth of the allocator's peak over one forward + backward (MB)"""
    import torch
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    decoder_call(arm, setup, True)
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def compare(setup):
    """relative Frobenius differences of the outputs and gradients of the two arms"""
    import torch
    dec, emb, state, memory, r = setup
    leaves = [emb, memory[0], memory[1]] + [x for c in state["cells"] for x in c]
    prm = [p for p in dec.parameters()]
    outs = {}
    for arm in ("fused", "composition"):
        out = decoder_call(arm, setup, False)
        gr = torch.autograd.grad((out * r).float().sum(), leaves + prm, allow_unused=True)
        outs[arm] = [out.detach().float()] + [None if x is None else x.float() for x in gr]
    rel = {}
    for i, (a, b) in enumerate(zip(outs["fused"], outs["composition"])):
        if a is None or b is None:
            continue
        rel[i] = float((a - b).norm() / b.norm().clamp_min(1e-30))
    return {"out": rel[0], "max_grad": max(v for k, v in rel.items() if k > 0)}


# ---------------------------------------------------------------------------
# model arm (one process per arm)
# ---------------------------------------------------------------------------
def model_arm(name, arm, steps, warmup, vocab):
    import torch
    import parallax_b200 as parallax
    import parallax_b200.models.nmt as nmt
    from parallax_b200.models.nmt import model as nmt_model
    if arm == "composition":
        nmt_model.Decoder.forward = nmt_model.Decoder._composition
    torch.manual_seed(0)
    hp = _hparams(name, vocab)
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
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        sess.run(["loss", "train_op"], feed)
    e1.record()
    torch.cuda.synchronize()
    sess.close()
    print(json.dumps({"config": name, "arm": arm, "step_ms": e0.elapsed_time(e1) / steps,
                      "losses": losses}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--model-rounds", type=int, default=3)
    ap.add_argument("--model-configs", default="iwslt15,wmt16")
    ap.add_argument("--model-steps", type=int, default=5)
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
        raise SystemExit("bench_nmt_decoder.py needs a CUDA device")
    result = {"B": 128, "S": 50, "T": 50, "dtype": "bf16", "gpu": gpu_info(), "decoder": {}}
    for name in [s for s in a.shapes.split(",") if s]:
        setup = decoder_setup(name)
        r = {"fwd": time_decoder(setup, False, a.rounds, a.iters, a.warmup),
             "fwd_bwd": time_decoder(setup, True, a.rounds, a.iters, a.warmup)}
        for arm in ("fused", "composition"):
            r["launches_per_step_" + arm] = {
                "fwd": count_launches(setup, arm, False) / 50,
                "fwd_bwd": count_launches(setup, arm, True) / 50}
            r["peak_growth_mb_" + arm] = peak_growth(setup, arm)
        r["rel_diff_fused_vs_composition"] = compare(setup)
        result["decoder"][name] = r
        print(name, json.dumps(r), flush=True)
        del setup
        torch.cuda.empty_cache()
    if a.model_rounds > 0:
        result["model"] = {"vocab": a.vocab}
        arms = ("fused", "composition")
        for name in [s for s in a.model_configs.split(",") if s]:
            runs, losses = {"fused": [], "composition": []}, {}
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
                    losses[arm] = d["losses"]
                    print("model", d, flush=True)
            result["model"][name] = {arm: {"median_ms": statistics.median(v), "runs_ms": v}
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
