"""The optimizer-rule bounds of `tests/dense_plane_ref.py` (used by `test_gpu_dense_plane.py`)
hold for an fp32 emulation of the dense step and of the async apply, on states the calibration
never saw, and reject the slips a kernel is likely to make: a dropped 1/W, the neighbouring
owner's slice, the clip multiplier applied twice."""
import pytest
import torch

from tests import dense_plane_ref as R

N = 1 << 14


def _step(kind, world, seed, scale_mul=1.0, ref_mul=1.0, drop_avg=False):
    gen = torch.Generator().manual_seed(seed)
    opt = R.make_opt(kind)
    hp = opt.hyper(2)
    w0, s0 = R.random_state(gen, kind, N)
    xs = R.random_operands(gen, world, N, torch.float32)
    k_scale = (1.0 if drop_avg else 1.0 / world) * scale_mul
    w32, s32 = R.emulate_fp32(kind, w0, s0, xs, k_scale, hp, rank=world - 1)
    g64, G = R.reduce_ref(xs, 1.0 / world * ref_mul)
    w64, s64 = R.apply64(kind, w0, s0, g64, hp)
    return w32, s32, w0, s0, w64, s64, G, hp


@pytest.mark.parametrize("kind", R.DENSE_KINDS)
@pytest.mark.parametrize("world", [1, 3, 6, 8])
def test_fp32_step_emulation_within_bound(kind, world):
    """A fused step emulated in fp32 (rotated sum, one scale rounding, the rule in fp32) stays
    inside the calibrated bound on a fresh seed."""
    w32, s32, w0, s0, w64, s64, G, hp = _step(kind, world, seed=100 + world)
    assert R.check_rule("emulation", kind, w32, s32, w0, s0, w64, s64, G, world, hp) <= 1.0


@pytest.mark.parametrize("kind", R.ELEMENTWISE_KINDS)
def test_fp32_async_emulation_within_bound(kind):
    """W = 5 un-averaged applies in sequence, emulated in fp32, stay inside `ASYNC_C`."""
    gen = torch.Generator().manual_seed(7)
    hp = R.make_opt(kind).hyper(2)
    w0, s0 = R.random_state(gen, kind, N)
    xs = R.random_operands(gen, 5, N, torch.float32)
    w32, s32, w64, s64 = w0, s0, w0.double(), tuple(s.double() for s in s0)
    for x in xs:
        w32, s32 = R.emulate_fp32(kind, w32, s32, [x], 1.0, hp)
        w64, s64 = R.apply64(kind, w64, s64, x.double(), hp)
    G = sum(x.double().abs() for x in xs)
    R.check_rule("async", kind, w32, s32, w0, s0, w64, s64, G, 5, hp, R.ASYNC_C)


@pytest.mark.parametrize("kind", R.DENSE_KINDS)
def test_dropped_average_fails(kind):
    """The reduction without its 1/W (W = 4)."""
    w32, s32, w0, s0, w64, s64, G, hp = _step(kind, 4, seed=3, drop_avg=True)
    with pytest.raises(AssertionError):
        R.check_rule("slip", kind, w32, s32, w0, s0, w64, s64, G, 4, hp)


@pytest.mark.parametrize("kind", R.DENSE_KINDS)
def test_neighbouring_slice_fails(kind):
    """An owner that updates (or reports) the next rank's slice: the result shifted by one
    slice of a W = 4 bucket."""
    w32, s32, w0, s0, w64, s64, G, hp = _step(kind, 4, seed=4)
    sl = N // 4
    with pytest.raises(AssertionError):
        R.check_rule("slip", kind, w32.roll(sl), tuple(s.roll(sl) for s in s32), w0, s0,
                     w64, s64, G, 4, hp)


@pytest.mark.parametrize("kind", R.DENSE_KINDS)
def test_clip_applied_twice_fails(kind):
    """A clip multiplier of 0.5 applied twice against a reference that applies it once."""
    w32, s32, w0, s0, w64, s64, G, hp = _step(kind, 4, seed=5, scale_mul=0.25, ref_mul=0.5)
    with pytest.raises(AssertionError):
        R.check_rule("slip", kind, w32, s32, w0, s0, w64, s64, G, 4, hp)
