"""BERT encoder with a sparse word-embedding table (BASELINE.json config 5:
BERT-large, hybrid mode — dense transformer weights on the all-reduce path,
the word embedding on the sparse path).  Not in the reference; a modern
dense-heavy + sparse-embedding workload for the same engine."""
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import nn as pnn
from .. import optim
from ..graph import Graph, ClipByGlobalNorm
from ..partitions import get_partitioner


class _Layer(nn.Module):
    def __init__(self, d, heads, ff):
        super().__init__()
        self.heads = heads
        self.qkv = nn.Linear(d, 3 * d)
        self.o = nn.Linear(d, d)
        self.ln1, self.ln2 = nn.LayerNorm(d), nn.LayerNorm(d)
        self.ff1, self.ff2 = nn.Linear(d, ff), nn.Linear(ff, d)

    def forward(self, x):
        B, T, D = x.shape
        q, k, v = self.qkv(x).view(B, T, 3, self.heads, D // self.heads).unbind(2)
        a = F.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2),
                                           v.transpose(1, 2))
        x = self.ln1(x + self.o(a.transpose(1, 2).reshape(B, T, D)))
        return self.ln2(x + self.ff2(F.gelu(self.ff1(x))))


class Bert(nn.Module):
    def __init__(self, vocab=30522, hidden=1024, layers=24, heads=16, ff=4096, max_len=512,
                 num_partitions=8):
        super().__init__()
        self.word_emb = pnn.Embedding(vocab, hidden, partitioner=get_partitioner(num_partitions),
                                      init_scale=0.02)
        self.pos_emb = nn.Parameter(torch.randn(max_len, hidden) * 0.02)
        self.ln = nn.LayerNorm(hidden)
        self.layers = nn.ModuleList(_Layer(hidden, heads, ff) for _ in range(layers))
        self.mlm = nn.Linear(hidden, hidden)
        self.mlm_ln = nn.LayerNorm(hidden)
        self.decoder = nn.Linear(hidden, vocab)

    def forward(self, input_ids, mlm_positions, mlm_labels):
        dt = self.decoder.weight.dtype
        B, T = input_ids.shape
        x = self.ln(self.word_emb(input_ids).to(dt) + self.pos_emb[:T])
        for l in self.layers:
            x = l(x)
        idx = mlm_positions.unsqueeze(-1).expand(-1, -1, x.shape[-1])
        h = self.mlm_ln(F.gelu(self.mlm(torch.gather(x, 1, idx))))
        logits = self.decoder(h).float()
        return {"loss": F.cross_entropy(logits.view(-1, logits.shape[-1]),
                                        mlm_labels.reshape(-1)), "logits": logits}


def bert_large(**kw):
    return Bert(hidden=1024, layers=24, heads=16, ff=4096, **kw)


# the parameters BERT's LAMB recipe neither decays nor adapts: LayerNorm gains and biases
LAMB_EXCLUDE = [r"(^|\.)(ln\d*|mlm_ln)\.", r"(^|\.)bias$"]


def bert_graph(model, learning_rate=1e-4, optimizer="adam"):
    """`optimizer="adam"` trains every variable with Adam.  `optimizer="lamb"` is the
    large-batch recipe: LAMB with weight decay 0.01, LayerNorm and bias parameters excluded
    from the decay and the trust ratio, for the dense variables, and Adam for the
    `word_emb` table."""
    dense = lambda n: n != "word_emb.weight"
    clip = [ClipByGlobalNorm(1.0, params=dense)]
    if optimizer == "adam":
        return Graph(model, optimizer=optim.Adam(learning_rate, weight_decay=0.0),
                     grad_rules=clip, name="bert")
    if optimizer == "lamb":
        return Graph(model, optimizer=optim.Lamb(learning_rate, weight_decay=0.01,
                                                 exclude_from_weight_decay=LAMB_EXCLUDE),
                     sparse_optimizer=optim.Adam(learning_rate, weight_decay=0.0),
                     grad_rules=clip, name="bert")
    raise ValueError("bert_graph: optimizer must be 'adam' or 'lamb', not %r" % (optimizer,))
