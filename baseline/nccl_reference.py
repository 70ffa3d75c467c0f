"""Same-box baseline: the reference's *algorithm* on stock libraries.

The reference stack (TF 1.11 fork + Horovod 0.16.3 + OpenMPI) cannot be built
for sm_90 offline, so BASELINE.md defines the same-box comparison as a
reference-equivalent path written against `torch.distributed` with Horovod
semantics, using none of parallax_b200's kernels or engine:

* model math: the LM1B graph of `examples/lm1b/language_model.py:60-110`
  unrolled op by op in eager PyTorch (cuBLAS/ATen), bf16 autocast-free bf16
  weights for parity with the product arm;
* dense gradients: Horovod tensor fusion — gradients packed in ready order into
  a 64 MiB fusion buffer (`horovod/common/operations.cc:1030`), one NCCL
  all-reduce per buffer, then a separate ÷size kernel
  (`horovod/tensorflow/__init__.py:76-81`), unpack, per-variable Adagrad;
* sparse gradients (AR mode): all-gather of values and indices
  (`horovod/tensorflow/__init__.py:62-73`), every rank applies the full sparse
  Adagrad update to its replica of the table.

Run: ``python bench.py --impl nccl --gpus N ...`` (torchrun for N > 1).
"""
import json
import math
import os

import torch
import torch.distributed as dist
import torch.nn as nn
import torch.nn.functional as F

FUSION_BYTES = 64 << 20


class LM1BPlain(nn.Module):
    def __init__(self, V=793470, E=512, S=2048, P=512, num_sampled=8192, T=20, keep=0.9):
        super().__init__()
        self.V, self.E, self.S, self.P, self.ns, self.T, self.keep = V, E, S, P, num_sampled, T, keep
        sc = math.sqrt(3.0 / E)
        self.emb = nn.Embedding(V, E, sparse=True)
        self.softmax_w = nn.Embedding(V, P, sparse=True)
        self.softmax_b = nn.Embedding(V, 1, sparse=True)
        with torch.no_grad():
            self.emb.weight.uniform_(-sc, sc)
            self.softmax_w.weight.uniform_(-sc, sc)
            self.softmax_b.weight.zero_()
        k = E + P
        self.W = nn.Parameter(torch.empty(k, 4 * S).uniform_(-math.sqrt(3.0 / k), math.sqrt(3.0 / k)))
        self.B = nn.Parameter(torch.zeros(4 * S))
        self.W_P = nn.Parameter(torch.empty(S, P).uniform_(-math.sqrt(3.0 / S), math.sqrt(3.0 / S)))

    def forward(self, x, y):
        Bsz, T = x.shape
        dt = self.W.dtype
        e = F.dropout(self.emb(x).to(dt), 1 - self.keep)
        c = torch.zeros(Bsz, self.S, device=x.device, dtype=dt)
        h = torch.zeros(Bsz, self.P, device=x.device, dtype=dt)
        outs = []
        for t in range(T):
            gates = torch.addmm(self.B, torch.cat([e[:, t], h], 1), self.W)
            i, j, f, o = gates.split(self.S, 1)
            c = torch.sigmoid(f + 1.0) * c + torch.sigmoid(i) * torch.tanh(j)
            h = (torch.sigmoid(o) * torch.tanh(c)) @ self.W_P
            outs.append(F.dropout(h, 1 - self.keep))
        inputs = torch.stack(outs, 1).reshape(Bsz * T, -1)
        targets = y.reshape(-1)
        u = torch.rand(self.ns, device=x.device)
        sampled = (torch.exp(u * math.log(self.V + 1.0)) - 1).long().clamp_(0, self.V - 1)
        ids = torch.cat([targets, sampled])
        w_all = self.softmax_w(ids).to(dt)
        b_all = self.softmax_b(ids).squeeze(-1).float()
        idf = ids.float()
        logq = torch.log((torch.log(idf + 2) - torch.log(idf + 1)) / math.log(self.V + 1.0) * self.ns)
        N = targets.numel()
        true_logits = (inputs * w_all[:N]).sum(-1).float() + b_all[:N] - logq[:N]
        samp = (inputs @ w_all[N:].t()).float() + (b_all[N:] - logq[N:])
        samp = samp.masked_fill(targets.unsqueeze(1) == sampled.unsqueeze(0), -1e30)
        lse = torch.logsumexp(torch.cat([true_logits.unsqueeze(1), samp], 1), 1)
        return (lse - true_logits).mean()


class HorovodLikeTrainer(object):
    def __init__(self, model, world, lr=0.2, clip=10.0):
        self.m, self.world, self.lr, self.clip = model, world, lr, clip
        self.dense = [model.W, model.B, model.W_P]
        self.sparse = [model.emb.weight, model.softmax_w.weight, model.softmax_b.weight]
        self.acc = {id(p): torch.full_like(p, 1.0, dtype=torch.float32) for p in self.dense}
        self.master = {id(p): p.detach().float().clone() for p in self.dense}
        self.sacc = {id(p): torch.full_like(p, 1.0, dtype=torch.float32) for p in self.sparse}
        n = sum(p.numel() for p in self.dense)
        self.fusion = torch.empty(min(n, FUSION_BYTES // 2), dtype=self.dense[0].dtype,
                                  device=self.dense[0].device)

    def step(self, x, y):
        m, W = self.m, self.world
        for p in self.dense + self.sparse:
            p.grad = None
        loss = m(x, y)
        (loss * m.T).backward()
        # ---- dense: fusion buffer -> ncclAllReduce -> div -> unpack ------------
        off = 0
        grads = [p.grad for p in reversed(self.dense)]
        for g in grads:
            self.fusion[off:off + g.numel()].copy_(g.reshape(-1))       # memcpy-in
            off += g.numel()
        if W > 1:
            dist.all_reduce(self.fusion[:off])
            self.fusion[:off].div_(W)                                    # separate ÷size
        off = 0
        for g in grads:
            g.copy_(self.fusion[off:off + g.numel()].view_as(g))        # memcpy-out
            off += g.numel()
        torch.nn.utils.clip_grad_norm_(self.dense, self.clip)
        for p in self.dense:
            g = p.grad.float()
            a, w = self.acc[id(p)], self.master[id(p)]
            a.addcmul_(g, g)
            w.addcdiv_(g, a.sqrt(), value=-self.lr)
            p.data.copy_(w)
        # ---- sparse: allgather(values), allgather(indices), local apply --------
        for p in self.sparse:
            g = p.grad.coalesce()
            idx, val = g.indices()[0], g.values().float()
            if p is m.emb.weight:
                val = val * x.shape[0]
            if W > 1:
                n = torch.tensor([idx.numel()], device=idx.device)
                ns = [torch.zeros_like(n) for _ in range(W)]
                dist.all_gather(ns, n)
                mx = int(max(int(t) for t in ns))
                pi = torch.zeros(mx, dtype=idx.dtype, device=idx.device); pi[:idx.numel()] = idx
                pv = torch.zeros(mx, val.shape[1], device=val.device); pv[:idx.numel()] = val
                gi = [torch.empty_like(pi) for _ in range(W)]
                gv = [torch.empty_like(pv) for _ in range(W)]
                dist.all_gather(gi, pi)
                dist.all_gather(gv, pv)
                idx = torch.cat([a[:int(k)] for a, k in zip(gi, ns)])
                val = torch.cat([a[:int(k)] for a, k in zip(gv, ns)])
            u, inv = torch.unique(idx, return_inverse=True)
            gs = torch.zeros(u.numel(), val.shape[1], device=val.device).index_add_(0, inv, val)
            a = self.sacc[id(p)]
            ar = a[u] + gs * gs
            a[u] = ar
            p.data[u] = (p.data[u].float() - self.lr * gs / ar.sqrt()).to(p.dtype)
        return loss


def main(args):
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    lrank = int(os.environ.get("LOCAL_RANK", "0"))
    dev = torch.device("cuda", lrank)
    torch.cuda.set_device(dev)
    if world > 1 and not dist.is_initialized():
        dist.init_process_group("nccl", device_id=dev)
    torch.manual_seed(1 + rank)
    if args.small:
        kw, batch = dict(V=50000, E=128, S=512, P=128, num_sampled=1024, T=8), args.batch or 32
    else:
        kw, batch = dict(), args.batch or 128
    model = LM1BPlain(**kw).to(dev)
    for p in (model.W, model.B, model.W_P):
        p.data = p.data.bfloat16()
    tr = HorovodLikeTrainer(model, world)
    V, T = model.V, model.T
    gen = torch.Generator().manual_seed(5 + rank)
    batches = [(torch.randint(0, V, (batch, T), generator=gen).to(dev),
                torch.randint(0, V, (batch, T), generator=gen).to(dev)) for _ in range(4)]
    K, Wm = args.steps, max(args.warmup, 3)
    for i in range(Wm):
        tr.step(*batches[i % 4])
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(K):
        loss = tr.step(*batches[i % 4])
    e1.record()
    torch.cuda.synchronize()
    t = torch.tensor([e0.elapsed_time(e1)], device=dev)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms = float(t)
    if rank == 0:
        value = batch * T * world * K / (ms / 1e3)
        print(json.dumps({
            "metric": "lm1b_words_per_sec", "value": value, "unit": "words/s",
            "n_gpus": world, "steps": K, "warmup": Wm, "ms_per_step": ms / K,
            "higher_is_better": True, "scaling": "weak", "dtype": "bf16",
            "impl": "nccl_horovod_equivalent",
            "data": "synthetic", "loss": float(loss),
            "config": {"model": "lm1b", "global_batch": batch * world, "seq_len": T,
                       "parallelism": "dp%d/allreduce+sparse-allgather (Horovod semantics)" % world,
                       "note": "stock PyTorch eager + NCCL; no parallax_b200 code on this path"}}))
    if world > 1:
        dist.destroy_process_group()
    return 0
