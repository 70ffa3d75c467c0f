"""The bounds of `tests/full_softmax_ref.py` on the CPU: an fp32 emulation of the full-softmax
kernels in their operation order passes them at LM1B's geometry (V = 793 470, K = 512, 32
partitions, 47 work items per CTA on 132 CTAs), and the kernels' likely slips fail them."""
import math

import numpy as np
import pytest
import torch

from tests import full_softmax_ref as R

L2E = np.float32(math.log2(math.e))
GRID = 132


def _f32(a):
    return np.asarray(a, dtype=np.float64).astype(np.float32)


def _exp2f(a):
    return _f32(np.exp2(a.astype(np.float64)))


def _fma_arg(v, ms):
    """fmaf(v, L2E, −ms) in fp32 (the fp64 product of two fp32 values is exact)"""
    return _f32(v.astype(np.float64) * np.float64(L2E) - ms.astype(np.float64))


def _merge(cx, cy, mx, sy):
    """lse_merge over arrays; sy == 0 marks an empty incoming pair, cy == 0 an empty running one"""
    nx = np.maximum(cx, mx)
    with np.errstate(invalid="ignore", over="ignore"):
        e1 = _exp2f(_f32(_f32(cx - nx) * L2E))
        e2 = _exp2f(_f32(_f32(mx - nx) * L2E))
        y = _f32(cy.astype(np.float64) * e1 + _f32(sy * e2).astype(np.float64))
    take = cy == 0
    y = np.where(take, sy, y)
    nx = np.where(take, mx, nx)
    keep = sy == 0
    return np.where(keep, cx, nx), np.where(keep, cy, y)


def _local_order(V, P):
    """global id of each owner-local row of a one-owner "div" layout (−1: padding)"""
    rpp = -(-V // P)
    base, extras = divmod(V, P)
    lr = np.arange(P * rpp)
    p, idx = lr // rpp, lr % rpp
    rows = np.where(p < extras, base + 1, base)
    gid = np.where(p < extras, p * (base + 1) + idx, p * base + extras + idx)
    return np.where(idx < rows, gid, -1)


def emulate_lse(s, P, drop_item=None):
    """fp32 lse [R] of rows s [R, V] (exact fp32 values) in the kernel's order on one owner: per
    128-row block a quad of lanes (32 columns each) takes the block max, sums exp2f terms,
    adds over the quad, and merges into its CTA's pair; then the grid merge of one warp."""
    R_, V = s.shape
    gid = _local_order(V, P)
    nblk = -(-gid.size // 128)
    gid = np.concatenate([gid, -np.ones(nblk * 128 - gid.size, dtype=gid.dtype)])
    v = np.where(gid >= 0, s[:, np.clip(gid, 0, None)], -np.inf).astype(np.float32)
    v = v.reshape(R_, nblk, 16, 4, 2).transpose(0, 1, 3, 2, 4).reshape(R_, nblk, 4, 32)
    mx = v.max(axis=(2, 3))
    ms = _f32(mx * L2E)
    lane = np.zeros((R_, nblk, 4), dtype=np.float32)
    for i in range(32):
        lane = _f32(lane + _exp2f(_fma_arg(v[..., i], ms[..., None])))
    sm = _f32(_f32(lane[..., 0] + lane[..., 1]) + _f32(lane[..., 2] + lane[..., 3]))
    if drop_item is not None:
        sm[:, drop_item] = 0
    grid = min(GRID, nblk)
    cx = np.full((R_, grid), -np.inf, dtype=np.float32)
    cy = np.zeros((R_, grid), dtype=np.float32)
    for i0 in range(0, nblk, grid):
        it = np.arange(i0, min(nblk, i0 + grid))
        nx, ny = _merge(cx[:, :it.size], cy[:, :it.size], mx[:, it], sm[:, it])
        cx[:, :it.size], cy[:, :it.size] = nx, ny
    lx = np.full((R_, 32), -np.inf, dtype=np.float32)
    ly = np.zeros((R_, 32), dtype=np.float32)
    for g0 in range(0, grid, 32):
        n = min(32, grid - g0)
        nx, ny = _merge(lx[:, :n], ly[:, :n], cx[:, g0:g0 + n], cy[:, g0:g0 + n])
        lx[:, :n], ly[:, :n] = nx, ny
    for o in (16, 8, 4, 2, 1):
        p = np.arange(32) ^ o
        lx, ly = _merge(lx, ly, lx[:, p], ly[:, p])
    lse = _f32(lx[:, 0] + _f32(np.log(ly[:, 0].astype(np.float64))))
    return lse, -(-nblk // grid), grid


@pytest.fixture(scope="module")
def lm1b_rows():
    """fp64 logits of 4 fine and 2 coarse rows against LM1B's exact table"""
    W, b = R.exact_table(R.V_LM1B, R.K_LM1B, 11)
    x = R.exact_inputs(8, R.K_LM1B, 12)[[0, 1, 2, 3, 4, 7]]
    return R.logits64(x, W, b)


def test_emulated_lse_within_bound_and_a_dropped_item_outside(lm1b_rows):
    s = lm1b_rows
    lse64 = torch.logsumexp(s, 1)
    smax = s.abs().amax(1)
    s32 = s.float().numpy()
    assert np.array_equal(s32.astype(np.float64), s.numpy())      # exact operands
    lse, per_cta, grid = emulate_lse(s32, R.P_LM1B)
    assert per_cta == 47 and grid == GRID
    bound = R.lse_bound(lse64, smax, per_cta, grid)
    err = (torch.from_numpy(lse).double() - lse64).abs()
    assert (err <= 2 * bound).all(), (err / bound).max()
    # one item's (max, Σexp) pair dropped: the item at the middle of CTA 5's walk
    lse_d, _, _ = emulate_lse(s32, R.P_LM1B, drop_item=5 + 23 * GRID)
    err_d = (torch.from_numpy(lse_d).double() - lse64).abs()
    assert (err_d > 2 * bound).any(), (err_d / bound).max()


def test_tie_toward_the_higher_id_fails(lm1b_rows):
    s = lm1b_rows[4:]                                        # the coarse rows
    for k in (8, 9, 16, 17, 32):
        vals = torch.sort(s, dim=1, descending=True).values
        assert (vals[:, k - 1] == vals[:, k]).any()          # a tie across the k-th position
    ref = torch.sort(s, dim=1, descending=True, stable=True).indices[:, :32]
    V = s.shape[1]
    # (logit desc, id desc): the stable sort of the reversed row
    slip = (V - 1 - torch.sort(s.flip(1), dim=1, descending=True, stable=True).indices)[:, :32]
    assert not torch.equal(slip, ref)


def test_masking_words_equal_to_theta_fails():
    """masked draws with the words equal to θ* dropped differ from the reference's"""
    from parallax_b200.parallel.engine import sample_log_e
    W, b = R.exact_table(20011, 64, 3)
    x = R.exact_inputs(64, 64, 4, coarse_every=1)              # coarse rows: ties at θ*
    s = R.logits64(x, W, b)
    ref = R.reference(x, W, b, taus=(1.0,), seed=9, trunc_k=(40,))
    th = ref["th_40"]
    loge = sample_log_e(9, torch.arange(64), torch.arange(20011)).double()
    keys = (s - loge).masked_fill(s <= th[:, None], -math.inf)
    kv, ki = torch.sort(keys, dim=1, descending=True, stable=True)
    agree, ok = R.checked_draws(ki[:, :32], ref["mkey_40"], ref["mkid_40"], ref["mloge_40"], 32)
    assert ok.float().mean() >= 0.99 and not agree
    # and the correct mask agrees with itself through the same check
    keys = (s - loge).masked_fill(s < th[:, None], -math.inf)
    ki = torch.sort(keys, dim=1, descending=True, stable=True).indices
    assert R.checked_draws(ki[:, :32], ref["mkey_40"], ref["mkid_40"], ref["mloge_40"], 32)[0]


def _emulate_grad(s, lse32, g, t, v0):
    """fp32 G (before bf16) and the column sums db as the gradient kernel forms them: a lane
    holds rows m·128 + 64·cw + 16·w + 8·h + r (consumer warpgroup cw, warp w, quad row r) and sums
    its rows' G over m and then h; the 8 lanes of a column add by xor shuffles over r (bits 0, 1
    and 2), and the 8 consumer warps add into shared memory one after another"""
    nl2 = _f32(-lse32 * L2E)
    p = _exp2f(_f32(s.astype(np.float64) * np.float64(L2E) + nl2[:, None].astype(np.float64)))
    hot = (t[:, None] - v0) == np.arange(s.shape[1])[None, :]
    p = np.where(hot, _f32(p - np.float32(1)), p)
    gv = _f32(g[:, None] * p)
    N, C = gv.shape
    rows = gv.reshape(N // 128, 2, 4, 2, 8, C)              # (m, cw, w, h, r, column)
    lane = np.zeros((2, 4, 8, C), dtype=np.float32)
    for m in range(N // 128):
        for h in range(2):
            lane = _f32(lane + rows[m, :, :, h])
    r = np.arange(8)
    for bit in (0, 1, 2):
        lane = _f32(lane + lane[:, :, r ^ (1 << bit)])
    db = np.zeros(C, dtype=np.float32)
    for cw in range(2):
        for w in range(4):
            db = _f32(db + lane[cw, w, 0])
    return gv, db


def test_emulated_gradient_within_bound_and_db_across_blocks_outside():
    W, b = R.exact_table(256, 512, 5)
    x = R.exact_inputs(256, 512, 6)
    s = R.logits64(x, W, b)
    gen = torch.Generator().manual_seed(7)
    t = torch.randint(0, 256, (256,), generator=gen)
    g = (torch.rand(256, generator=gen) * 2 - 0.5).float()
    # the lse of a larger vocabulary: this chunk holds part of the softmax
    lse32 = (torch.logsumexp(s, 1) + 3.0).float()
    gv, db = _emulate_grad(s.float().numpy(), lse32.numpy(), g.numpy(), t.numpy(), 0)
    p = torch.exp(s - lse32.double()[:, None])
    G64 = g.double()[:, None] * (p - torch.nn.functional.one_hot(t, 256).double())
    gb = R.grad_bound(p, g.double(), s.abs().amax(1), lse32.double())
    Gb = torch.from_numpy(gv).bfloat16().double()
    assert ((Gb - G64).abs() <= 2 * (gb + R.bf16_half_ulp(G64.abs() + gb))).all()
    db_b = gb.sum(0) + (2 * 2 + 11) * R.U * G64.abs().sum(0)
    err = (torch.from_numpy(db).double() - G64.sum(0)).abs()
    assert (err <= 2 * db_b).all()
    # the second block's sums still holding the first block's (its s_db not re-zeroed)
    slip = db.copy()
    slip[128:] = _f32(slip[128:] + db[:128])
    err = (torch.from_numpy(slip).double() - G64.sum(0)).abs()
    assert (err[128:] > 2 * db_b[128:]).any()
