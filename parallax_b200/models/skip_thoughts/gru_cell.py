"""GRU with layer normalisation — the cell of the skip-thoughts encoder/decoders.

Parity: `examples/skip_thoughts/ops/gru_cell.py:27-134` `LayerNormGRUCell`:

    [z, r] = σ( LN(h·W_h) + LN(x·W_x) )
    ĥ      = tanh( r ⊙ LN(h·U) + LN(x·W) )
    h'     = (1 − z) ⊙ h + z ⊙ ĥ

recurrent matrices start as random orthonormal blocks, input matrices uniform
(`skip_thoughts_model.py:50-57,208-227`).

There is no cuDNN kernel for a layer-normalised GRU, so the layer is arranged
for the GPU rather than as a cell: both input projections and their layer norms
are computed for ALL time steps with two GEMMs before the recurrence, and each
step does a single fused ``h @ [W_h | U]`` GEMM.  On the GPU the recurrence is one autograd
node with one cell kernel per step each way (`ops/fused.py: ln_gru_layer`).
"""
import torch
import torch.nn as nn

from ...ops import fused


def random_orthonormal_(w):
    """fill the square matrix `w` with a random orthonormal basis (SVD of a
    uniform matrix, `skip_thoughts_model.py:50-57`)"""
    assert w.shape[0] == w.shape[1], "orthonormal init needs a square matrix"
    u, _, _ = torch.linalg.svd(torch.empty_like(w, dtype=torch.float32).uniform_(-1, 1))
    with torch.no_grad():
        w.copy_(u.to(w.dtype))
    return w


class LayerNormGRU(nn.Module):
    def __init__(self, input_size, num_units, init_scale=0.1):
        super().__init__()
        self.input_size, self.num_units = input_size, num_units
        self.w_x = nn.Parameter(torch.empty(input_size, 2 * num_units))     # gates, from x
        self.w = nn.Parameter(torch.empty(input_size, num_units))           # candidate, from x
        self.w_hu = nn.Parameter(torch.empty(num_units, 3 * num_units))     # [W_h | U], from h
        self.ln_wx = nn.LayerNorm(2 * num_units)
        self.ln_w = nn.LayerNorm(num_units)
        self.ln_wh = nn.LayerNorm(2 * num_units)
        self.ln_u = nn.LayerNorm(num_units)
        with torch.no_grad():
            self.w_x.uniform_(-init_scale, init_scale)
            self.w.uniform_(-init_scale, init_scale)
            n = num_units
            for k in range(3):           # three orthonormal blocks: z, r, candidate
                random_orthonormal_(self.w_hu[:, k * n:(k + 1) * n])

    def _cell(self, gx_t, cx_t, h):
        n = self.num_units
        hh = h @ self.w_hu
        zr = torch.sigmoid(self.ln_wh(hh[:, :2 * n]) + gx_t)
        z, r = zr[:, :n], zr[:, n:]
        cand = torch.tanh(r * self.ln_u(hh[:, 2 * n:]) + cx_t)
        return (1.0 - z) * h + z * cand

    def _input_side(self, x):
        """both input projections and their layer norms, for all steps at once"""
        return self.ln_wx(x @ self.w_x), self.ln_w(x @ self.w)

    def forward(self, x, lengths=None, initial_state=None, reverse=False):
        """x [B,T,I] → (outputs [B,T,U] zero past each length, final state [B,U]).
        `reverse=True` runs each sequence back to front (inside its own length).

        On CUDA in bf16 or fp32, with n % 8 == 0 and n <= 4096, the recurrence is one fused
        autograd node (`ops.fused.ln_gru_layer`: a product and one cell kernel per step each
        way); otherwise (CPU, fp64, other shapes) it is `_composition`."""
        if fused.ln_gru_applies(x, self.w_hu, self.ln_wh, self.ln_u, initial_state):
            gx, cx = self._input_side(x)
            return fused.ln_gru_layer(gx, cx, self.w_hu, self.ln_wh, self.ln_u, initial_state,
                                      lengths, reverse)
        return self._composition(x, lengths, initial_state, reverse)

    def _composition(self, x, lengths=None, initial_state=None, reverse=False):
        """The layer as plain PyTorch ops, one time step at a time: the fallback of `forward`
        and the oracle of the fused node."""
        B, T, _ = x.shape
        gx, cx = self._input_side(x)
        h = initial_state if initial_state is not None else \
            torch.zeros(B, self.num_units, device=x.device, dtype=x.dtype)
        outs = [None] * T
        order = range(T - 1, -1, -1) if reverse else range(T)
        for t in order:
            h2 = self._cell(gx[:, t], cx[:, t], h)
            if lengths is not None:
                live = (lengths > t)[:, None]
                h = torch.where(live, h2, h)
                outs[t] = torch.where(live, h2, torch.zeros_like(h2))
            else:
                h = h2
                outs[t] = h2
        return torch.stack(outs, 1), h
