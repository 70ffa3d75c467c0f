"""Sequence-to-sequence NMT models: vanilla, attention and GNMT.

Parity (behaviour, not structure):

* `examples/nmt/model.py:41-677` `BaseModel`/`Model` — embeddings (shared or
  separate, *partitioned sparse variables* under `parallax.get_partitioner`,
  `model_helper.py:284-340`), uni/bi-directional encoders, decoder, bias-free
  output projection, loss = Σ masked cross-entropy / batch_size, learning-rate
  warm-up (`:207-232`) and decay schemes (`:234-263`), global-norm clipping.
* `examples/nmt/attention_model.py:31-183` `AttentionModel` — attention wrapper
  over the whole decoder stack with input feeding (previous attention vector
  concatenated to the next input), `output_attention`, `pass_hidden_state`.
* `examples/nmt/gnmt_model.py:32-285` `GNMTModel` — one bidirectional + N-1
  unidirectional encoder layers, attention computed from the *bottom* decoder
  layer and fed to every upper layer (`gnmt`: previous step's context,
  `gnmt_v2`: the current one), residual connections that add only the
  non-attention part of the input (`gnmt_residual_fn`, `:269-285`).
* cells (`model_helper.py:372-470`): lstm (forget bias), gru,
  layer_norm_lstm; dropout on every cell's input; residual wrappers on the
  top `num_*_residual_layers` layers.

GPU-first structure: there is no per-step cell graph.  Every layer is one
cuDNN sequence call wherever the data dependence allows it — whole encoder
stacks (packed by length), and in the GNMT decoder every layer above the
attention layer (those depend on the *contexts*, which the bottom layer
produces for all steps first); only the layers that feed attention back into
their own input run step by step.  The same modules serve the step API used by
greedy/sampling/beam decoding (`inference.py`).  On the GPU, with lstm or layer_norm_lstm cells,
those step-by-step layers and the attention are one fused autograd node (`ops/fused.py:
nmt_attention_decoder`), and every other layer_norm_lstm layer call is one fused autograd node
(`ops/fused.py: ln_lstm_layer`).
"""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.nn.utils.rnn import pack_padded_sequence, pad_packed_sequence

from ... import nn as pnn
from ... import optim
from ...graph import Graph, ClipByGlobalNorm
from ...ops import fused
from ...partitions import get_partitioner
from .attention import AttentionMechanism

UNIT_TYPES = ("lstm", "gru", "layer_norm_lstm")


# --------------------------------------------------------------------- cells
class LayerNormLSTM(nn.Module):
    """`tf.contrib.rnn.LayerNormBasicLSTMCell`: layer-normalised gate
    pre-activations and cell state.  On the GPU the whole layer is one fused autograd node
    (`fused.ln_lstm_layer`); elsewhere a Python time loop (no cuDNN equivalent)."""

    def __init__(self, input_size, num_units, forget_bias=1.0):
        super().__init__()
        self.num_units, self.forget_bias = num_units, forget_bias
        self.kernel = nn.Linear(input_size + num_units, 4 * num_units, bias=False)
        self.ln = nn.ModuleList([nn.LayerNorm(num_units) for _ in range(4)])
        self.ln_c = nn.LayerNorm(num_units)

    def cell(self, x, h, c):
        i, j, f, o = self.kernel(torch.cat([x, h], -1)).chunk(4, -1)
        i, j, f, o = (ln(g) for ln, g in zip(self.ln, (i, j, f, o)))
        c2 = c * torch.sigmoid(f + self.forget_bias) + torch.sigmoid(i) * torch.tanh(j)
        h2 = torch.tanh(self.ln_c(c2)) * torch.sigmoid(o)
        return h2, c2

    def forward(self, x, state, lengths=None):
        """x [B, T, I], state (h, c) -> (outputs [B, T, U], (h_T, c_T)).  The fused node when
        `fused.ln_lstm_applies` (CUDA, bf16/fp32, U % 8 == 0 and within the kernels' limit),
        else `_composition`."""
        h, c = state
        if fused.ln_lstm_applies(x, self.kernel.weight, self.ln, self.ln_c, h, c):
            return fused.ln_lstm_layer(x, self.kernel.weight, self.ln, self.ln_c, self.forget_bias,
                                       h, c, lengths)
        return self._composition(x, state, lengths)

    def _composition(self, x, state, lengths=None):
        """The layer as plain PyTorch ops, one time step at a time: the fallback of `forward`
        and the oracle of the fused node."""
        h, c = state
        outs = []
        for t in range(x.shape[1]):
            h2, c2 = self.cell(x[:, t], h, c)
            if lengths is not None:
                live = (lengths > t)[:, None]
                h2, c2 = torch.where(live, h2, h), torch.where(live, c2, c)
                outs.append(torch.where(live, h2, torch.zeros_like(h2)))
            else:
                outs.append(h2)
            h, c = h2, c2
        return torch.stack(outs, 1), (h, c)


class RNNLayer(nn.Module):
    """dropout(input) → one recurrent layer → optional residual.

    State: ``(h, c)`` for LSTM kinds, ``h`` for GRU, each ``[B, units]``."""

    def __init__(self, unit_type, input_size, num_units, forget_bias=1.0, dropout=0.0,
                 residual=False, init_weight=0.1):
        super().__init__()
        if unit_type not in UNIT_TYPES:
            raise ValueError("Unknown unit type %s!" % unit_type)
        self.unit_type, self.num_units = unit_type, num_units
        self.input_size, self.dropout, self.residual = input_size, float(dropout), residual
        if unit_type == "lstm":
            self.rnn = nn.LSTM(input_size, num_units, batch_first=True)
        elif unit_type == "gru":
            self.rnn = nn.GRU(input_size, num_units, batch_first=True)
        else:
            self.rnn = LayerNormLSTM(input_size, num_units, forget_bias)
        self.reset_parameters(init_weight, forget_bias)

    def reset_parameters(self, init_weight, forget_bias):
        with torch.no_grad():
            for n, p in self.rnn.named_parameters():
                if "weight" in n and p.dim() > 1:
                    p.uniform_(-init_weight, init_weight)
                elif "bias" in n:
                    p.zero_()
            if self.unit_type == "lstm":
                # TF adds forget_bias to the forget pre-activation at run time; a
                # bias initialised to it trains identically (gate order i,f,g,o)
                H = self.num_units
                self.rnn.bias_ih_l0[H:2 * H].fill_(forget_bias)

    @property
    def is_lstm(self):
        return self.unit_type != "gru"

    def zero_state(self, batch, device, dtype):
        z = torch.zeros(batch, self.num_units, device=device, dtype=dtype)
        return (z, z.clone()) if self.is_lstm else z

    def _to_rnn(self, state):
        if self.unit_type == "layer_norm_lstm":
            return state
        if self.is_lstm:
            return (state[0][None].contiguous(), state[1][None].contiguous())
        return state[None].contiguous()

    def _from_rnn(self, st):
        if self.unit_type == "layer_norm_lstm":
            return st
        return (st[0][0], st[1][0]) if self.is_lstm else st[0]

    def forward(self, x, state=None, lengths=None):
        """x [B,T,I]; `lengths` (CPU int64) → outputs past a sequence's end are
        zero and its state stops there (`dynamic_rnn(sequence_length=…)`)."""
        B, T = x.shape[0], x.shape[1]
        inp = F.dropout(x, self.dropout, True) if (self.training and self.dropout > 0) else x
        if state is None:
            state = self.zero_state(B, x.device, x.dtype)
        if self.unit_type == "layer_norm_lstm":
            ln = lengths.to(x.device) if lengths is not None else None
            out, st = self.rnn(inp, state, ln)
        elif lengths is not None:
            packed = pack_padded_sequence(inp, lengths, batch_first=True, enforce_sorted=False)
            out, st = self.rnn(packed, self._to_rnn(state))
            out, _ = pad_packed_sequence(out, batch_first=True, total_length=T)
        else:
            out, st = self.rnn(inp, self._to_rnn(state))
        if self.residual:
            out = out + x[..., :self.num_units]
        return out, self._from_rnn(st)

    def step(self, x, state):
        """One time step as explicit GEMMs + gate math (fp32) on the layer's own
        weights.  A length-1 cuDNN call would re-pack the weights on every step:
        on the NVLink fabric parameters are views into the symmetric buckets, never
        one flat cuDNN buffer."""
        if self.unit_type == "layer_norm_lstm":
            out, st = self.forward(x[:, None, :], state)
            return out[:, 0], st
        inp = F.dropout(x, self.dropout, True) if (self.training and self.dropout > 0) else x
        r = self.rnn
        n = self.num_units
        if self.unit_type == "lstm":
            h, c = state
            gates = (F.linear(inp, r.weight_ih_l0, r.bias_ih_l0) +
                     F.linear(h, r.weight_hh_l0, r.bias_hh_l0)).float()
            i, f, g, o = gates[:, :n], gates[:, n:2 * n], gates[:, 2 * n:3 * n], gates[:, 3 * n:]
            c2 = torch.sigmoid(f) * c.float() + torch.sigmoid(i) * torch.tanh(g)
            h2 = (torch.sigmoid(o) * torch.tanh(c2)).to(x.dtype)
            st = (h2, c2.to(c.dtype))
        else:                                   # torch / cuDNN GRU equations
            h = state
            gi = F.linear(inp, r.weight_ih_l0, r.bias_ih_l0).float()
            gh = F.linear(h, r.weight_hh_l0, r.bias_hh_l0).float()
            rg = torch.sigmoid(gi[:, :n] + gh[:, :n])
            z = torch.sigmoid(gi[:, n:2 * n] + gh[:, n:2 * n])
            cand = torch.tanh(gi[:, 2 * n:] + rg * gh[:, 2 * n:])
            h2 = ((1.0 - z) * cand + z * h.float()).to(x.dtype)
            st = h2
        out = h2
        if self.residual:
            out = out + x[..., :self.num_units]
        return out, st


def build_stack(unit_type, num_layers, num_residual_layers, input_size, num_units, hp,
                upper_input_size=None):
    """`model_helper._cell_list`: layer i is residual iff i ≥ n − n_residual."""
    layers = []
    for i in range(num_layers):
        isz = input_size if i == 0 else (upper_input_size or num_units)
        layers.append(RNNLayer(unit_type, isz, num_units, hp.forget_bias, hp.dropout,
                               residual=i >= num_layers - num_residual_layers,
                               init_weight=hp.init_weight))
    return nn.ModuleList(layers)


def reverse_by_length(x, lengths):
    """`tf.reverse_sequence` along time: element t ↔ len-1-t inside each
    sequence, padding left in place."""
    T = x.shape[1]
    t = torch.arange(T, device=x.device)[None, :]
    L = lengths.to(x.device)[:, None]
    idx = torch.where(t < L, L - 1 - t, t)
    return x.gather(1, idx[..., None].expand_as(x))


def run_stack(layers, x, lengths=None, states=None):
    out_states = []
    for i, layer in enumerate(layers):
        x, st = layer(x, None if states is None else states[i], lengths)
        out_states.append(st)
    return x, out_states


# ------------------------------------------------------------------- encoder
class Encoder(nn.Module):
    def __init__(self, hp):
        super().__init__()
        U, n, nres = hp.num_units, hp.num_encoder_layers, hp.num_encoder_residual_layers
        self.encoder_type = hp.encoder_type
        if hp.encoder_type == "uni":
            self.layers = build_stack(hp.unit_type, n, nres, U, U, hp)
            self.output_size = U
        elif hp.encoder_type == "bi":
            nb, nbres = n // 2, nres // 2
            self.fw = build_stack(hp.unit_type, nb, nbres, U, U, hp)
            self.bw = build_stack(hp.unit_type, nb, nbres, U, U, hp)
            self.output_size = 2 * U
        elif hp.encoder_type == "gnmt":
            self.fw = build_stack(hp.unit_type, 1, 0, U, U, hp)
            self.bw = build_stack(hp.unit_type, 1, 0, U, U, hp)
            self.layers = build_stack(hp.unit_type, n - 1, nres, 2 * U, U, hp)
            self.output_size = U
        else:
            raise ValueError("Unknown encoder_type %s" % hp.encoder_type)

    def _bidirectional(self, x, lengths):
        out_f, st_f = run_stack(self.fw, x, lengths)
        out_b, st_b = run_stack(self.bw, reverse_by_length(x, lengths), lengths)
        out_b = reverse_by_length(out_b, lengths)
        return torch.cat([out_f, out_b], -1), st_f, st_b

    def forward(self, emb, lengths):
        """emb [B,S,U], lengths CPU int64 [B] → (outputs [B,S,output_size], list of
        per-layer final states handed to the decoder)."""
        if self.encoder_type == "uni":
            return run_stack(self.layers, emb, lengths)
        out, st_f, st_b = self._bidirectional(emb, lengths)
        if self.encoder_type == "bi":
            if len(st_f) == 1:
                return out, [st_f[0], st_b[0]]
            states = []
            for f, b in zip(st_f, st_b):          # fw_0, bw_0, fw_1, bw_1, …
                states += [f, b]
            return out, states
        out, st_u = run_stack(self.layers, out, lengths)
        return out, [st_b[0]] + st_u


# ------------------------------------------------------------------- decoder
class Decoder(nn.Module):
    """Decoder stack; `architecture` ∈ none | standard | gnmt | gnmt_v2."""

    def __init__(self, hp, memory_size):
        super().__init__()
        U, n, nres = hp.num_units, hp.num_decoder_layers, hp.num_decoder_residual_layers
        self.num_units, self.memory_size = U, memory_size
        self.output_attention = bool(hp.output_attention)
        self.pass_hidden_state = bool(hp.pass_hidden_state)
        if not hp.attention:
            self.architecture = "none"
            self.layers = build_stack(hp.unit_type, n, nres, U, U, hp)
            return
        arch = hp.attention_architecture
        if arch not in ("standard", "gnmt", "gnmt_v2"):
            raise ValueError("Unknown attention architecture %s" % arch)
        self.architecture = arch
        self.attention = AttentionMechanism(hp.attention, U, memory_size, U, hp.init_weight)
        if arch == "standard":
            self.layers = build_stack(hp.unit_type, n, nres, 2 * U, U, hp)
            self.attention_layer = nn.Linear(U + memory_size, U, bias=False)
            self.attention_size = U
        else:
            self.layers = build_stack(hp.unit_type, n, nres, U + memory_size, U, hp,
                                      upper_input_size=U + memory_size)
            self.attention_size = memory_size

    # -- state ------------------------------------------------------------------
    def initial_state(self, encoder_state, batch, device, dtype):
        zero = [l.zero_state(batch, device, dtype) for l in self.layers]
        if self.architecture == "none":
            cells = list(encoder_state)         # vanilla model always passes the state
        elif self.pass_hidden_state:
            assert len(encoder_state) == len(self.layers), \
                "pass_hidden_state needs as many encoder states as decoder layers"
            cells = list(encoder_state)
        else:
            cells = zero
        st = {"cells": cells}
        if self.architecture != "none":
            st["attention"] = torch.zeros(batch, self.attention_size, device=device, dtype=dtype)
        return st

    @staticmethod
    def reorder_state(state, index):
        """gather batch entries (beam search parent selection / tiling)"""
        sel = lambda t: t.index_select(0, index)
        cells = [tuple(sel(x) for x in c) if isinstance(c, tuple) else sel(c)
                 for c in state["cells"]]
        out = {"cells": cells}
        if "attention" in state:
            out["attention"] = sel(state["attention"])
        return out

    # -- the fused node ---------------------------------------------------------------
    def node_arguments(self):
        """(layers, keyword arguments) of `fused.nmt_attention_decoder` (and of its reference)
        for this decoder's parameters: the layers that feed attention back into their input,
        every layer for standard and the bottom one for gnmt / gnmt_v2."""
        layers = self.layers if self.architecture == "standard" else self.layers[:1]
        rnn = [l.rnn for l in layers]
        a = self.attention
        if layers[0].unit_type == "layer_norm_lstm":
            # the bias-free kernel over [input | h]: its two column blocks, and the LayerNorms
            kw = dict(w_ih=[r.kernel.weight[:, :l.input_size] for l, r in zip(layers, rnn)],
                      w_hh=[r.kernel.weight[:, l.input_size:] for l, r in zip(layers, rnn)],
                      b_ih=None, b_hh=None, residual=[l.residual for l in layers],
                      ln=[([n.weight for n in list(r.ln) + [r.ln_c]] +
                           [n.bias for n in list(r.ln) + [r.ln_c]],
                           [n.eps for n in list(r.ln) + [r.ln_c]], r.forget_bias) for r in rnn])
        else:
            kw = dict(w_ih=[r.weight_ih_l0 for r in rnn], w_hh=[r.weight_hh_l0 for r in rnn],
                      b_ih=[r.bias_ih_l0 for r in rnn], b_hh=[r.bias_hh_l0 for r in rnn],
                      residual=[l.residual for l in layers])
        extra = []
        if a.option in ("bahdanau", "normed_bahdanau"):
            kw["w_q"] = a.query_layer.weight
            extra = [a.v]
            if a.option == "normed_bahdanau":
                kw["b"] = a.b
                extra.append(a.g)
        elif a.option == "scaled_luong":
            kw["g"] = a.g
        if self.architecture == "standard":
            kw["w_a"] = self.attention_layer.weight
        if a.option in ("bahdanau", "normed_bahdanau"):
            v = a.g * a.v / a.v.norm() if a.option == "normed_bahdanau" else a.v
            kw["v"] = v if v.dtype == torch.float64 else v.float().contiguous()
        return layers, kw, extra

    def _node(self, emb, state, memory):
        """`node_arguments` when the fused node takes this decoder, else None (no attention,
        GRU cells, CPU, fp64, shapes outside the kernels' limits)."""
        if self.architecture == "none":
            return None
        layers = self.layers if self.architecture == "standard" else self.layers[:1]
        unit = layers[0].unit_type
        if unit not in ("lstm", "layer_norm_lstm") or any(l.unit_type != unit for l in layers) \
                or not emb.is_cuda:
            return None
        layers, kw, extra = self.node_arguments()
        keys, values, _ = memory
        cells = state["cells"][:len(layers)]
        if unit == "lstm":
            weights = kw["w_ih"] + kw["w_hh"] + kw["b_ih"] + kw["b_hh"]
        else:
            weights = [l.rnn.kernel.weight for l in layers] + [p for x in kw["ln"] for p in x[0]]
        weights = weights + extra + [kw.get(k) for k in ("w_q", "g", "b", "w_a")]
        states = [x for c in cells for x in c] + [state["attention"]]
        if not fused.nmt_decoder_applies(emb, keys, values, weights, states, unit):
            return None
        return layers, kw

    def _dropout_masks(self, layers, T, emb):
        """Per layer [T, B, I_l] input masks (0 or 1/(1−p), in emb's dtype) when training with
        dropout, else None: the same distribution as the composition's `F.dropout`, drawn
        here because the fused node takes its masks as tensors."""
        if not (self.training and any(l.dropout > 0 for l in layers)):
            return None
        B = emb.shape[0]
        masks = []
        for l in layers:
            keep = 1.0 - l.dropout
            m = torch.empty(T, B, l.input_size, dtype=emb.dtype, device=emb.device)
            masks.append(m.bernoulli_(keep).div_(keep) if l.dropout > 0 else m.fill_(1.0))
        return masks

    def _gnmt_upper(self, x, ctx, state):
        """GNMT layers above the bottom one, as whole-sequence calls over (h⁰_t, context)"""
        if self.architecture == "gnmt":          # upper layers use the previous context
            ctx = torch.cat([state["attention"][:, None, :], ctx[:, :-1]], 1)
        for layer, st in zip(self.layers[1:], state["cells"][1:]):
            x, _ = layer(torch.cat([x, ctx], -1), st)
        return x

    # -- one step (inference; also the inner loop of the attention layers) --------
    def step(self, emb_t, state, memory):
        """emb_t [B,U] → (output [B,U], new state).  `memory` = attention.prepare(…)

        Without gradients and when the fused node applies, the attention layers run as one
        step of it (nothing saved); otherwise as `_step`."""
        grad = torch.is_grad_enabled() and (emb_t.requires_grad or
                                            any(p.requires_grad for p in self.parameters()))
        node = None if grad else self._node(emb_t, state, memory)
        if node is None:
            return self._step(emb_t, state, memory)
        layers, kw = node
        keys, values, pad = memory
        cells = state["cells"]
        n = len(layers)
        q, att, hs, cs = fused.nmt_attention_decoder_step(
            emb_t, [c[0] for c in cells[:n]], [c[1] for c in cells[:n]], state["attention"],
            keys, values, pad, masks=self._dropout_masks(layers, 1, emb_t), **kw)
        new_cells = list(zip(hs, cs))
        if self.architecture == "standard":
            return (att if self.output_attention else q), {"cells": new_cells, "attention": att}
        x, fed = q, (att if self.architecture == "gnmt_v2" else state["attention"])
        for layer, st in zip(self.layers[1:], cells[1:]):
            x, s2 = layer.step(torch.cat([x, fed], -1), st)
            new_cells.append(s2)
        return x, {"cells": new_cells, "attention": att}

    def _step(self, emb_t, state, memory):
        """One step of the composition: each layer's `RNNLayer.step`, the attention and the
        attention layer as separate PyTorch ops."""
        cells, new_cells = state["cells"], []
        if self.architecture == "none":
            x = emb_t
            for layer, st in zip(self.layers, cells):
                x, s2 = layer.step(x, st)
                new_cells.append(s2)
            return x, {"cells": new_cells}
        keys, values, pad = memory
        if self.architecture == "standard":
            x = torch.cat([emb_t, state["attention"]], -1)
            for layer, st in zip(self.layers, cells):
                x, s2 = layer.step(x, st)
                new_cells.append(s2)
            ctx, _ = self.attention(x, keys, values, pad)
            att = self.attention_layer(torch.cat([x, ctx], -1))
            out = att if self.output_attention else x
            return out, {"cells": new_cells, "attention": att}
        prev = state["attention"]
        x, s2 = self.layers[0].step(torch.cat([emb_t, prev], -1), cells[0])
        new_cells.append(s2)
        ctx, _ = self.attention(x, keys, values, pad)
        fed = ctx if self.architecture == "gnmt_v2" else prev
        for layer, st in zip(self.layers[1:], cells[1:]):
            x, s2 = layer.step(torch.cat([x, fed], -1), st)
            new_cells.append(s2)
        return x, {"cells": new_cells, "attention": ctx}

    # -- teacher-forced training pass ------------------------------------------------
    def forward(self, emb, state, memory):
        """emb [B,T,U] → outputs [B,T,U].

        With lstm or layer_norm_lstm cells on CUDA in bf16 or fp32 and shapes within the
        kernels' limits, the attention recurrence is one fused autograd node
        (`fused.nmt_attention_decoder`); every other case runs `_composition`.  With dropout the
        node's masks come from the same distribution as the composition's but not from the same
        random stream."""
        node = self._node(emb, state, memory)
        if node is None:
            return self._composition(emb, state, memory)
        layers, kw = node
        keys, values, pad = memory
        n = len(layers)
        cells = state["cells"][:n]
        out = fused.nmt_attention_decoder(
            emb, [c[0] for c in cells], [c[1] for c in cells], state["attention"], keys, values,
            pad, masks=self._dropout_masks(layers, emb.shape[1], emb),
            output_attention=self.output_attention, **kw)
        if self.architecture == "standard":
            return out
        return self._gnmt_upper(*out, state)

    def _composition(self, emb, state, memory):
        """The decoder as plain PyTorch ops, one time step at a time: the fallback of `forward`
        and the oracle of the fused node."""
        if self.architecture == "none":
            out, _ = run_stack(self.layers, emb, None, state["cells"])
            return out
        keys, values, pad = memory
        T = emb.shape[1]
        if self.architecture == "standard":
            outs = []
            for t in range(T):
                o, state = self._step(emb[:, t], state, memory)
                outs.append(o)
            return torch.stack(outs, 1)
        # GNMT: only the bottom layer is recurrent through attention; the layers
        # above see (h⁰_t, context) for every t and run as whole-sequence calls
        bottom, cell, prev = self.layers[0], state["cells"][0], state["attention"]
        hs, ctxs = [], []
        for t in range(T):
            h, cell = bottom.step(torch.cat([emb[:, t], prev], -1), cell)
            prev, _ = self.attention(h, keys, values, pad)
            hs.append(h)
            ctxs.append(prev)
        return self._gnmt_upper(torch.stack(hs, 1), torch.stack(ctxs, 1), state)


# --------------------------------------------------------------------- model
class _ClipGradNorm(torch.autograd.Function):
    """identity whose backward rescales the incoming gradient to norm ≤ max_norm"""

    @staticmethod
    def forward(ctx, x, max_norm):
        ctx.max_norm = max_norm
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        norm = g.float().norm()
        scale = torch.clamp(ctx.max_norm / (norm + 1e-6), max=1.0)
        return g * scale.to(g.dtype), None


class Seq2Seq(nn.Module):
    """placeholders: source, target_input, target_output [B,·] int64 and
    source_sequence_length, target_sequence_length [B]."""

    def __init__(self, hp):
        super().__init__()
        self.hp = hp
        U = hp.num_units
        part = get_partitioner(hp.num_embeddings_partitions) \
            if hp.num_embeddings_partitions and hp.num_embeddings_partitions > 1 else None
        self.embedding_encoder = pnn.Embedding(hp.src_vocab_size, U, partitioner=part,
                                               init_scale=hp.init_weight, seed=11)
        if hp.share_vocab:
            if hp.src_vocab_size != hp.tgt_vocab_size:
                raise ValueError("Share embedding but different src/tgt vocab sizes "
                                 "%d vs. %d" % (hp.src_vocab_size, hp.tgt_vocab_size))
            self.embedding_decoder = self.embedding_encoder
        else:
            self.embedding_decoder = pnn.Embedding(hp.tgt_vocab_size, U, partitioner=part,
                                                   init_scale=hp.init_weight, seed=13)
        self.encoder = Encoder(hp)
        self.decoder = Decoder(hp, self.encoder.output_size)
        self.output_layer = nn.Linear(U, hp.tgt_vocab_size, bias=False)
        self._init_dense(hp)

    def _init_dense(self, hp):
        """`model_helper.get_initializer`: uniform(±init_weight) | glorot_normal |
        glorot_uniform for every dense matrix outside the recurrent layers (those
        are initialised in `RNNLayer`)."""
        for name, p in self.named_parameters():
            if p.dim() < 2 or ".rnn." in name or name.startswith("embedding_"):
                continue
            with torch.no_grad():
                if hp.init_op == "uniform":
                    p.uniform_(-hp.init_weight, hp.init_weight)
                elif hp.init_op == "glorot_normal":
                    nn.init.xavier_normal_(p)
                elif hp.init_op == "glorot_uniform":
                    nn.init.xavier_uniform_(p)
                else:
                    raise ValueError("Unknown init_op %s" % hp.init_op)

    def load_pretrained_embeddings(self, which, matrix, num_trainable_tokens=3):
        """`embed_prefix`: initialise an embedding from a text file
        (`model_helper.py:248-281`).  The reference keeps only the first
        `num_trainable_tokens` rows trainable; here the table stays one ordinary
        sparse variable (all rows trainable) so it can be partitioned like any
        other — only rows ≥ `num_trainable_tokens` are overwritten."""
        emb = self.embedding_encoder if which == "encoder" else self.embedding_decoder
        with torch.no_grad():
            emb.weight[num_trainable_tokens:].copy_(matrix[num_trainable_tokens:])

    @property
    def compute_dtype(self):
        return self.output_layer.weight.dtype

    # -- pieces shared by training and inference --------------------------------
    def _embed(self, table, ids):
        """lookup + (training) clip of the gradient flowing back into the looked-up
        rows.  The reference clips embeddings and dense variables by ONE joint
        global norm (`model.py:196-205`); that is what ``clip_embeddings_jointly``
        selects (`nmt_graph`), and nothing is clipped here.  By default the
        engine's clip covers the dense variables only, and the sparse gradient of
        each lookup is clipped here by its own norm, per worker, before it is
        pushed to the row owners."""
        emb = table(ids).to(self.compute_dtype)
        if self.training and torch.is_grad_enabled() and self.hp.max_gradient_norm and \
                not self.hp.get("clip_embeddings_jointly", False):
            emb = _ClipGradNorm.apply(emb, float(self.hp.max_gradient_norm))
        return emb

    def encode(self, source, source_sequence_length):
        dt = self.compute_dtype
        emb = self._embed(self.embedding_encoder, source)
        lengths = source_sequence_length.detach().to("cpu", torch.int64).clamp(min=1)
        enc_out, enc_state = self.encoder(emb, lengths)
        memory = None
        if self.decoder.architecture != "none":
            memory = self.decoder.attention.prepare(enc_out, source_sequence_length)
        state = self.decoder.initial_state(enc_state, source.shape[0], enc_out.device, dt)
        return memory, state

    def decode_step(self, token_ids, state, memory):
        """token_ids [B] → (logits [B,V] fp32, new state)"""
        emb = self.embedding_decoder(token_ids).to(self.compute_dtype)
        out, state = self.decoder.step(emb, state, memory)
        return self.output_layer(out).float(), state

    def logits(self, source, target_input, source_sequence_length):
        memory, state = self.encode(source, source_sequence_length)
        emb = self._embed(self.embedding_decoder, target_input)
        return self.output_layer(self.decoder(emb, state, memory)).float()

    def forward(self, source, target_input, target_output, source_sequence_length,
                target_sequence_length):
        """Training loss: the masked cross entropy of the output layer summed over the batch
        and divided by B, through `parallax.nn.linear_cross_entropy` (fused where it applies,
        so no [B·T, V] logits are kept)."""
        memory, state = self.encode(source, source_sequence_length)
        emb = self._embed(self.embedding_decoder, target_input)
        out = self.decoder(emb, state, memory)
        B, T, U = out.shape
        tl = target_sequence_length.to(out.device)
        mask = (torch.arange(T, device=out.device)[None, :] < tl[:, None]).to(torch.float32)
        loss, _ = pnn.linear_cross_entropy(out.reshape(B * T, U), target_output.reshape(-1),
                                           self.output_layer.weight, None,
                                           row_weights=mask.reshape(-1))
        return {"loss": loss / B, "predict_count": tl.sum(),
                "word_count": tl.sum() + source_sequence_length.to(tl.device).sum(),
                "batch_size": torch.tensor(B, device=out.device)}


# --------------------------------------------------------- training "graph"
def learning_rate_fn(hp):
    """lr(step) with warm-up and decay (`model.py:207-263`).  `step` is the
    1-based index of the update being applied; TF evaluates the schedule with
    the number of *completed* steps, hence the ``step - 1``."""
    base, warm, total = float(hp.learning_rate), int(hp.warmup_steps), int(hp.num_train_steps)
    if hp.warmup_scheme != "t2t":
        raise ValueError("Unknown warmup scheme %s" % hp.warmup_scheme)
    scheme = hp.decay_scheme
    if scheme in ("luong5", "luong10", "luong234"):
        factor = 0.5
        if scheme == "luong5":
            start, times = total // 2, 5
        elif scheme == "luong10":
            start, times = total // 2, 10
        else:
            start, times = total * 2 // 3, 4
        every = max((total - start) // times, 1)
    elif not scheme:
        start, every, factor = total, 0, 1.0
    else:
        raise ValueError("Unknown decay scheme %s" % scheme)

    def lr(step):
        gs = max(int(step) - 1, 0)
        v = base
        if warm > 0 and gs < warm:          # t2t: start at 0.01·lr, ×100 over warm-up
            v *= math.exp(math.log(0.01) / warm) ** (warm - gs)
        if every and gs >= start:
            v *= factor ** ((gs - start) // every)
        return v
    return lr


def nmt_graph(model, hp=None):
    """SGD (with the decay schedule) or Adam + global-norm clipping
    (`model.py:160-205`).  The reference clips embeddings and dense variables
    jointly; ``hp.clip_embeddings_jointly`` does the same with one
    ``ClipByGlobalNorm(include_sparse=True)`` over every variable.  By default the
    engine's clip covers the dense variables and each embedding's sparse
    gradient is clipped by its own norm inside the model (`Seq2Seq._embed`)."""
    hp = hp or model.hp
    lr = learning_rate_fn(hp)
    if hp.optimizer == "sgd":
        opt = optim.GradientDescent(lr)
    elif hp.optimizer == "adam":
        assert float(hp.learning_rate) <= 0.001, \
            "! High Adam learning rate %g" % hp.learning_rate
        opt = optim.Adam(lr)
    else:
        raise ValueError("Unknown optimizer type %s" % hp.optimizer)
    dense = lambda n: not n.startswith("embedding_")
    if not hp.max_gradient_norm:
        rules = []
    elif hp.get("clip_embeddings_jointly", False):
        rules = [ClipByGlobalNorm(hp.max_gradient_norm, include_sparse=True)]
    else:
        rules = [ClipByGlobalNorm(hp.max_gradient_norm, params=dense)]
    return Graph(model, optimizer=opt, grad_rules=rules, name="nmt")


def create_model(hp):
    """model class by (attention, attention_architecture) like
    `nmt/train.py:275-291` `get_model_creator`; one class here covers all."""
    if hp.encoder_type == "gnmt" and hp.attention and \
            hp.attention_architecture not in ("gnmt", "gnmt_v2", "standard"):
        raise ValueError("Unknown attention architecture %s" % hp.attention_architecture)
    return Seq2Seq(hp)
