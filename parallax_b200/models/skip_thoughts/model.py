"""The skip-thoughts model: one sentence encoder, two sentence decoders.

Parity: `examples/skip_thoughts/skip_thoughts_model.py:60-387` — word embeddings
(uniform ±`uniform_init_scale`), layer-normalised GRU encoder (optionally
bidirectional with `encoder_dim`/2 units per direction, final states
concatenated) producing the *thought vector*; two decoders (previous and next
sentence) whose GRU starts from the thought vector and reads the target
embeddings shifted right by one zero step; ONE logits layer shared by both
decoders; loss = Σ masked cross-entropy (sum over the batch, not a mean),
perplexity statistics from the per-token losses and weights.  Training:
Adam, lr halved every `learning_rate_decay_steps`, global-norm clip
(`examples/skip_thoughts/train.py:44-99`).

Modes: ``forward(encode_ids, encode_mask, decode_pre_ids, …)`` (train / eval)
and ``encode(ids | embeddings, mask)`` (the "encode" mode used by
`SkipThoughtsEncoder`).
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from ... import nn as pnn
from ... import optim
from ...graph import Graph, ClipByGlobalNorm
from ...partitions import get_partitioner
from .gru_cell import LayerNormGRU


class SkipThoughtsModel(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.config = c = config
        part = get_partitioner(c.num_embedding_partitions) \
            if getattr(c, "num_embedding_partitions", 0) and c.num_embedding_partitions > 1 \
            else None
        self.word_embedding = pnn.Embedding(c.vocab_size, c.word_embedding_dim, partitioner=part,
                                            init_scale=c.uniform_init_scale, seed=21)
        if c.bidirectional_encoder:
            if c.encoder_dim % 2:
                raise ValueError("encoder_dim must be even when using a bidirectional encoder.")
            n = c.encoder_dim // 2
            self.encoder_fw = LayerNormGRU(c.word_embedding_dim, n, c.uniform_init_scale)
            self.encoder_bw = LayerNormGRU(c.word_embedding_dim, n, c.uniform_init_scale)
        else:
            self.encoder = LayerNormGRU(c.word_embedding_dim, c.encoder_dim, c.uniform_init_scale)
        self.decoder_pre = LayerNormGRU(c.word_embedding_dim, c.encoder_dim, c.uniform_init_scale)
        self.decoder_post = LayerNormGRU(c.word_embedding_dim, c.encoder_dim, c.uniform_init_scale)
        self.logits = nn.Linear(c.encoder_dim, c.vocab_size)
        with torch.no_grad():
            self.logits.weight.uniform_(-c.uniform_init_scale, c.uniform_init_scale)
            self.logits.bias.zero_()

    @property
    def compute_dtype(self):
        return self.logits.weight.dtype

    # -- encoder -----------------------------------------------------------------
    def encode_embeddings(self, emb, mask):
        """emb [B,T,D], mask [B,T] → thought vectors [B, encoder_dim]"""
        lengths = mask.to(emb.device).sum(1)
        if self.config.bidirectional_encoder:
            _, fw = self.encoder_fw(emb, lengths)
            _, bw = self.encoder_bw(emb, lengths, reverse=True)
            return torch.cat([fw, bw], 1)
        return self.encoder(emb, lengths)[1]

    def encode(self, encode_ids, encode_mask):
        return self.encode_embeddings(self.word_embedding(encode_ids).to(self.compute_dtype),
                                      encode_mask)

    # -- decoders ------------------------------------------------------------------
    def _decode(self, gru, thought, ids, mask):
        """The decoder GRU's outputs [B, T, encoder_dim] for target `ids`."""
        emb = self.word_embedding(ids).to(self.compute_dtype)
        inp = F.pad(emb[:, :-1, :], (0, 0, 1, 0))           # shift right, zero first step
        out, _ = gru(inp, mask.to(emb.device).sum(1), initial_state=thought)
        return out

    def _decoder_loss(self, gru, thought, ids, mask):
        """(Σ masked cross entropy, Σ weights) of one decoder, through
        `parallax.nn.linear_cross_entropy` with the shared logits layer (fused where it
        applies, so no [B·T, vocab] logits are kept)."""
        out = self._decode(gru, thought, ids, mask)
        weights = mask.to(out.device).reshape(-1).to(torch.float32)
        loss, _ = pnn.linear_cross_entropy(out.reshape(-1, out.shape[-1]), ids.reshape(-1),
                                           self.logits.weight, self.logits.bias,
                                           row_weights=weights)
        return loss, weights

    def forward(self, encode_ids, encode_mask, decode_pre_ids, decode_pre_mask,
                decode_post_ids, decode_post_mask):
        thought = self.encode(encode_ids, encode_mask)
        pre, w_pre = self._decoder_loss(self.decoder_pre, thought, decode_pre_ids,
                                        decode_pre_mask)
        post, w_post = self._decoder_loss(self.decoder_post, thought, decode_post_ids,
                                          decode_post_mask)
        return {"loss": pre + post, "loss_pre": pre.detach(), "loss_post": post.detach(),
                "sum_weights": (w_pre.sum() + w_post.sum()).detach(),
                "thought_vectors": thought.detach()}


def learning_rate_fn(training_config):
    """staircase exponential decay (`train.py:44-70`)"""
    base = float(training_config.learning_rate)
    f, every = training_config.learning_rate_decay_factor, training_config.learning_rate_decay_steps
    if not f:
        return lambda step: base
    return lambda step: base * float(f) ** (max(int(step) - 1, 0) // int(every))


def skip_thoughts_graph(model, training_config=None):
    """Adam + global-norm clipping of the dense variables; the (sparse) word
    embedding is updated with lazy Adam by its row owners."""
    from .configuration import training_config as _tc
    tc = training_config or _tc()
    dense = lambda n: not n.startswith("word_embedding")
    rules = [ClipByGlobalNorm(tc.clip_gradient_norm, params=dense)] if tc.clip_gradient_norm else []
    return Graph(model, optimizer=optim.Adam(learning_rate_fn(tc)), grad_rules=rules,
                 name="skip_thoughts")


def feed_from_batch(batch):
    """(encode, decode_pre, decode_post) `SentenceBatch`es → feed_dict"""
    enc, pre, post = batch
    return {"encode_ids": [enc.ids], "encode_mask": [enc.mask],
            "decode_pre_ids": [pre.ids], "decode_pre_mask": [pre.mask],
            "decode_post_ids": [post.ids], "decode_post_mask": [post.mask]}
