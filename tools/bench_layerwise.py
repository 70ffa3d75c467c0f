"""Layer-wise optimizers (LARS, LAMB) on one GPU.

    python tools/bench_layerwise.py [--rounds 3] [--iters 50] [--bert] [--out result.json]

Arms alternate within each round and the median over `--rounds` rounds is reported:

1. Kernels at W = 1 on a 32 MiB bf16 bucket of 64 tensors: Adam MODE 0 against LAMB
   (MODE 1 reduce + norm pass + update pass), Momentum MODE 0 against LARS.  µs per pass and
   in total from CUDA events over `--iters` launches, and GB/s from this byte model (fp32
   master and slots, bf16 gradients and parameters, per element; a model, not a
   measurement): Adam 28, LAMB 52 = 6 + 16 + 30, Momentum 20, LARS 36 = 6 + 8 + 22.
2. ``--bert``: BERT-large step time (bf16, CUDA graph, batch 16 × 512) with Adam and with
   LAMB, each in a process of its own.

The card name and power limit are read in the same run and printed with the numbers.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BYTES = {"adam": 28, "lamb": 52, "momentum": 20, "lars": 36}
PASS_BYTES = {"lamb": (6, 16, 30), "lars": (6, 8, 22)}


def card():
    try:
        return subprocess.run(
            ["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
            capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # pragma: no cover
        return "unknown (%s)" % e


def _bucket(kind, n, ntensors):
    import torch
    from tests.gpu_utils import make_world
    from parallax_b200 import optim
    from parallax_b200.parallel import nvops
    f = make_world(1, options={"comm_blocks": 0})[0]
    gb, pb = f.heap.alloc(n * 2, "g"), f.heap.alloc(n * 2, "p")
    gb.tensor(torch.bfloat16, n).normal_()
    pb.tensor(torch.bfloat16, n).normal_()
    opt = {"adam": optim.Adam(1e-3), "lamb": optim.Lamb(1e-3, weight_decay=0.01),
           "momentum": optim.Momentum(0.1), "lars": optim.Lars(0.1)}[kind]
    master = pb.tensor(torch.bfloat16, n).float()
    slots = [torch.full((n,), v, device="cuda") for v in opt.slot_init()]
    hp = torch.tensor(opt.hyper(1), device="cuda")
    step = n // ntensors
    lw = nvops.LayerwiseMap([(i * step, step) for i in range(ntensors)], 0, n, 8,
                            [opt.layer_flags("w%d" % i) for i in range(ntensors)], "cuda") \
        if kind in optim.LAYERWISE_KINDS else None
    red = torch.empty(n, device="cuda") if lw is not None else None
    return f, gb, pb, master, slots, hp, lw, red


def bench_kernels(rounds, iters, mib=32, ntensors=64):
    import torch
    from parallax_b200.parallel import nvops
    from parallax_b200.parallel.symmetric import CH_COMM
    n = (mib << 20) // 2
    st = {k: _bucket(k, n, ntensors) for k in BYTES}
    s1 = lambda sl: sl[1] if len(sl) > 1 else None

    def fused(k):
        f, gb, pb, master, slots, hp, _, _ = st[k]
        nvops.dense_step(f.heap, gb.c_ptrs(), pb.c_ptrs(), master, slots[0], s1(slots), None,
                         None, hp, None, None, n, 1.0, 0.0, k, 0, torch.bfloat16, CH_COMM,
                         max_blocks=0, stream=torch.cuda.current_stream())

    def reduce(k):
        f, gb, pb, master, slots, hp, _, red = st[k]
        nvops.dense_step(f.heap, gb.c_ptrs(), pb.c_ptrs(), master, slots[0], s1(slots), None,
                         red, hp, None, None, n, 1.0, 0.0, k, 1, torch.bfloat16, CH_COMM,
                         max_blocks=0, stream=torch.cuda.current_stream())

    def norm(k):
        f, gb, pb, master, slots, hp, lw, red = st[k]
        nvops.layerwise_norm(red, master, slots[0], s1(slots), hp, None, lw, k, torch.bfloat16,
                             stream=torch.cuda.current_stream())

    def update(k):
        f, gb, pb, master, slots, hp, lw, red = st[k]
        nvops.layerwise_update(f.heap, pb.c_ptrs(), red, master, slots[0], s1(slots), None, hp,
                               None, lw, lw.sums, n, 0.0, k, torch.bfloat16, CH_COMM,
                               max_blocks=0, stream=torch.cuda.current_stream())

    arms = {"adam": [("fused", fused)], "momentum": [("fused", fused)],
            "lamb": [("reduce", reduce), ("norm", norm), ("update", update)],
            "lars": [("reduce", reduce), ("norm", norm), ("update", update)]}
    res = {k: {p: [] for p, _ in ps} for k, ps in arms.items()}
    for _ in range(rounds):
        for k, ps in arms.items():
            for p, fn in ps:
                for _ in range(3):
                    fn(k)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(iters):
                    fn(k)
                b.record()
                b.synchronize()
                res[k][p].append(a.elapsed_time(b) * 1e3 / iters)
    out = {}
    for k, ps in res.items():
        us = {p: statistics.median(v) for p, v in ps.items()}
        total = sum(us.values())
        row = {"us": us, "us_total": total, "model_bytes_per_elem": BYTES[k],
               "GBps_total": BYTES[k] * n / total / 1e3}
        if k in PASS_BYTES:
            row["GBps"] = {p: b * n / us[p] / 1e3 for p, b in zip(us, PASS_BYTES[k])}
        out[k] = row
    for f, *_ in st.values():
        f.close()
    return out


BERT_ARM = r"""
import json, sys, time, torch
sys.path.insert(0, %(root)r)
import parallax_b200 as parallax
from parallax_b200.models.bert import bert_large, bert_graph
torch.manual_seed(0)
g = bert_graph(bert_large(), 1e-4, optimizer=%(opt)r)
cfg = parallax.Config(run_option="HYBRID", sess_config={"compute_dtype": "bf16",
                                                        "cuda_graph": True})
sess, *_ = parallax.parallel_run(g, "localhost:0", parallax_config=cfg)
gen = torch.Generator().manual_seed(1)
B, T, V = 16, 512, 30522
ids = torch.randint(5, V, (B, T), generator=gen)
pos = torch.stack([torch.randperm(T, generator=gen)[:76] for _ in range(B)])
feed = {"input_ids": [ids.scatter(1, pos, 4)], "mlm_positions": [pos],
        "mlm_labels": [torch.gather(ids, 1, pos)]}
for _ in range(8):
    sess.run(["loss", "train_op"], feed)
torch.cuda.synchronize()
t = time.time()
for _ in range(%(steps)d):
    loss, _ = sess.run(["loss", "train_op"], feed)
torch.cuda.synchronize()
print(json.dumps({"ms_per_step": (time.time() - t) * 1e3 / %(steps)d, "loss": loss[0]}))
sess.close()
"""


def bench_bert(rounds, steps=20):
    res = {"adam": [], "lamb": []}
    for _ in range(rounds):
        for opt in res:
            r = subprocess.run([sys.executable, "-c", BERT_ARM % dict(root=ROOT, opt=opt,
                                                                       steps=steps)],
                               capture_output=True, text=True, timeout=1800)
            if r.returncode != 0:
                res[opt].append({"error": r.stderr.strip().splitlines()[-1:]})
            else:
                res[opt].append(json.loads(r.stdout.strip().splitlines()[-1]))
    out = {}
    for opt, v in res.items():
        ms = [x["ms_per_step"] for x in v if "ms_per_step" in x]
        out[opt] = {"ms_per_step_median": statistics.median(ms) if ms else None,
                    "runs": v}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--bert", action="store_true")
    ap.add_argument("--out")
    a = ap.parse_args()
    result = {"card": card(), "kernels_w1_32MiB_bf16": bench_kernels(a.rounds, a.iters)}
    result["bert_large_step"] = bench_bert(a.rounds) if a.bert else "not measured"
    result["card_after"] = card()
    s = json.dumps(result, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()
