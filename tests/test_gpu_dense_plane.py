"""The dense NVLink data plane against fp64 at every world size 1..8 (`collectives.cu`,
`dense_step.cu`): two-shot, TMA two-shot and one-shot all-reduces, broadcast, all-gather, the
fused dense step, the async (Hogwild) apply, `sumsq` and `clip_scale`.

Every kernel of the plane is a template on the world size W; these tests run each
instantiation, 1..8, in a world simulated on one GPU (`tests/gpu_utils.py`).  Kernels with a
cross-rank barrier need all ranks' CTAs resident at once, so W·max_blocks <= 128, and the ranks
are launched phase by phase in rank order with nothing host-blocking in between.

Two kinds of operands (`tests/dense_plane_ref.py`):
  * exact -- k·2^-6, |k| <= 64: every W-way fp32 sum is exact, so the result is predicted bit
    for bit (the exact sum times fp32(scale) rounded once, then RNE to bf16).  A misplaced
    slice, vector, rank rotation or grid-stride round changes bits;
  * random -- randn, within |got - ref| <= (W-1)·u·|scale|·Σ|x_p| + u·|ref| (+ half a bf16 ulp).
Every case also checks that the replicas are bitwise identical and that the bytes past n in
every buffer (a guard of 0xFF bytes, a NaN pattern in both dtypes) keep their bits.

Sizes: the minimum n = W·VN, a slice of 777 vectors (not a multiple of 512), and a slice that
takes several grid-stride rounds of the grid with the last round partly filled; grids
max_blocks in {1, 3, 128 // W}."""
import ctypes
import math

import pytest
import torch

from tests import dense_plane_ref as R
from tests.lm1b_opt_ref import dense_grid, norm_bound, U

pytestmark = pytest.mark.gpu

WORLDS = [1, 2, 3, 4, 5, 6, 7, 8]
DTYPES = [torch.float32, torch.bfloat16]
GUARD = 512          # bytes past the last element of every buffer, checked after each call


def _vn(dtype):
    return 4 if dtype == torch.float32 else 8


def _es(dtype):
    return 4 if dtype == torch.float32 else 2


def _grids(world):
    return sorted({1, 3, 128 // world})


def _bits(t):
    return t.view(torch.int32) if t.element_size() == 4 else t.view(torch.int16)


def _world(world):
    from tests.gpu_utils import make_world
    return make_world(world)


def _close(fabs):
    for f in fabs:
        f.close()


def _arm(buf, nbytes):
    """0xFF over the whole buffer: the bytes from `nbytes` on are the guard."""
    buf.bytes_tensor().fill_(255)


def _guard_ok(buf, nbytes, what):
    g = buf.bytes_tensor()[nbytes:]
    assert g.numel() >= 16 and bool((g == 255).all()), "%s wrote past its end" % what


def _guarded(t):
    """An fp32 copy of `t` followed by GUARD bytes of 0xFF (a NaN pattern); the returned view
    holds the copy, `_tail_ok` checks the bytes after it."""
    full = torch.empty(t.numel() + GUARD // 4, dtype=torch.float32, device=t.device)
    _bits(full).fill_(-1)
    full[:t.numel()].copy_(t)
    return full[:t.numel()]


def _tail_ok(v, what):
    tail = v.as_strided((GUARD // 4,), (1,), v.storage_offset() + v.numel())
    assert bool((_bits(tail) == -1).all()), "%s: store past the end of the slice" % what


def _check_reduced(got, xs, scale, dtype, exact, world, what):
    """Bitwise against the exact-operand prediction, or within `reduce_bound`."""
    if exact:
        want = R.reduce_exact(xs, scale).to(dtype)
        assert torch.equal(_bits(got), _bits(want)), \
            "%s: %d of %d elements differ" % (what, int((_bits(got) != _bits(want)).sum()),
                                              got.numel())
    else:
        ref, G = R.reduce_ref(xs, scale)
        err = (got.double() - ref).abs()
        bound = R.reduce_bound(ref, G, world, dtype)
        assert bool((err <= bound).all()), \
            "%s: %d of %d out of bound, worst err/bound %g" % (
                what, int((err > bound).sum()), err.numel(), float((err / bound).max()))


def _operands(gen, world, n, dtype, exact):
    return R.exact_operands(gen, world, n, "cuda") if exact else \
        R.random_operands(gen, world, n, dtype, "cuda")


def _check_sumsq(got, vals, vn, iters, ctas, what, ranks=1):
    """fp32 Σx² (all terms >= 0) against the fp64 Σ of the fp32 values it squares."""
    ref = float((vals.double() ** 2).sum())
    rel = norm_bound(vn, iters, ctas, ranks=ranks)
    assert abs(float(got) - ref) <= rel * ref, "%s: Σx² %r vs %r (rel bound %g)" % (
        what, float(got), ref, rel)


# -------------------------------------------------------------------------- two-shot all-reduce
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("world", WORLDS)
def test_allreduce_twoshot_exact_and_bounded(world, dtype):
    """`px_allreduce_twoshot` at scale 1 and 1/W (inexact at W = 3, 5, 6, 7): exact operands
    bitwise, random ones within `reduce_bound`, every rank's Σx² of its own slice against the
    fp64 Σ of the pre-rounding fp32 values within `norm_bound(vn, iters, ctas)` (each thread
    squares vn·iters values in sequence, a two-level warp tree, one atomic per CTA).  Sizes
    include a slice of (2·UNROLL + 1)·ctas·512 + 37 vectors: two full UNROLL rounds of the
    grid and a third with one of its UNROLL slots partly filled.  Catches a wrong slice base,
    peer rotation, a skipped or doubled grid-stride / UNROLL step, a scale applied twice or
    not at all, and a Σx² taken before the scale or over the wrong slice."""
    from parallax_b200.parallel import nvops
    from parallax_b200.parallel.symmetric import CH_COMM
    vn, es = _vn(dtype), _es(dtype)
    unroll = 4 if world <= 4 else 2
    cases = [(mb, nv) for mb in _grids(world)
             for nv in (1, 777, (2 * unroll + 1) * mb * 512 + 37)]
    nmax = max(world * nv * vn for _, nv in cases)
    fabs = _world(world)
    bufs = [f.heap.alloc(nmax * es + GUARD, "x") for f in fabs]
    ss = [torch.zeros(1, device="cuda") for _ in fabs]
    gen = torch.Generator(device="cuda").manual_seed(11 + world)
    for mb, nv in cases:
        n = world * nv * vn
        ctas = max(1, min(-(-nv // 1024), mb))
        iters = -(-nv // (ctas * 512))
        for exact in (True, False):
            for scale in sorted({1.0, 1.0 / world}):
                xs = _operands(gen, world, n, dtype, exact)
                for r, b in enumerate(bufs):
                    _arm(b, n * es)
                    b.tensor(dtype, n).copy_(xs[r])
                    ss[r].zero_()
                torch.cuda.synchronize()
                for r, f in enumerate(fabs):
                    nvops.allreduce_twoshot(f.heap, bufs[r].c_ptrs(), n, dtype, scale, CH_COMM,
                                            sumsq=ss[r], max_blocks=mb, stream=f.comm_stream)
                torch.cuda.synchronize()
                what = "twoshot W=%d n=%d mb=%d exact=%s scale=%g" % (world, n, mb, exact, scale)
                out0 = bufs[0].tensor(dtype, n)
                _check_reduced(out0, xs, scale, dtype, exact, world, what)
                for r, b in enumerate(bufs):
                    assert torch.equal(_bits(b.tensor(dtype, n)), _bits(out0)), what
                    _guard_ok(b, n * es, what)
                if exact or dtype == torch.float32:
                    # the fp32 values the kernel squared: exact prediction, or its fp32 output
                    pre = R.reduce_exact(xs, scale) if exact else out0.float()
                    sl = n // world
                    for r in range(world):
                        _check_sumsq(ss[r], pre[r * sl:(r + 1) * sl], vn, iters, ctas,
                                     what + " rank %d" % r)
    _close(fabs)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("world", WORLDS)
def test_allreduce_twoshot_bulk_exact_and_bounded(world, dtype):
    """`px_allreduce_twoshot_bulk` (cp.async.bulk into 2·W·8 KB of shared memory): slices of
    less than one 8 KB chunk, exactly 5 chunks and 5 chunks plus a partial one, on 1 and 3
    CTAs, so the two-stage ring and its mbarrier parity wrap.  Exact operands bitwise, random
    ones within `reduce_bound`.  Catches a wrong stage or parity, a chunk read before its
    bytes land, a partial chunk's byte count and a wrong peer tile."""
    from parallax_b200.parallel import nvops
    from parallax_b200.parallel.symmetric import CH_COMM
    es = _es(dtype)
    slices = (16 * 100, 5 * 8192, 5 * 8192 + 16 * 37)
    nmax = world * max(slices) // es
    fabs = _world(world)
    bufs = [f.heap.alloc(nmax * es + GUARD, "x") for f in fabs]
    gen = torch.Generator(device="cuda").manual_seed(21 + world)
    for mb in (1, 3):
        for sb in slices:
            n = world * sb // es
            for exact in (True, False):
                for scale in sorted({1.0, 1.0 / world}):
                    xs = _operands(gen, world, n, dtype, exact)
                    for r, b in enumerate(bufs):
                        _arm(b, n * es)
                        b.tensor(dtype, n).copy_(xs[r])
                    torch.cuda.synchronize()
                    for r, f in enumerate(fabs):
                        nvops.allreduce_twoshot_bulk(f.heap, bufs[r].c_ptrs(), n, dtype, scale,
                                                     CH_COMM, max_blocks=mb,
                                                     stream=f.comm_stream)
                    torch.cuda.synchronize()
                    what = "bulk W=%d slice=%dB mb=%d exact=%s scale=%g" % (
                        world, sb, mb, exact, scale)
                    out0 = bufs[0].tensor(dtype, n)
                    _check_reduced(out0, xs, scale, dtype, exact, world, what)
                    for b in bufs:
                        assert torch.equal(_bits(b.tensor(dtype, n)), _bits(out0)), what
                        _guard_ok(b, n * es, what)
    _close(fabs)


# -------------------------------------------------------------------------- one-shot all-reduce
def _oneshot_round(fabs, srcs, dsts, ss, n, dtype, scale, channel, mb):
    from parallax_b200.parallel import nvops
    for r, f in enumerate(fabs):
        nvops.allreduce_oneshot(f.heap, srcs[r], dsts[r], f.small_stage, n, dtype, scale,
                                channel, sumsq=None if ss is None else ss[r], max_blocks=mb,
                                stream=f.comm_stream)


def _oneshot_io(xs, n, dtype, vn):
    """Zero-padded sources (whole 16-byte vectors) and 0xFF-armed destinations with a guard."""
    npad = -(-n // vn) * vn
    gel = GUARD // _es(dtype)
    srcs, dsts = [], []
    for x in xs:
        s = torch.zeros(npad, dtype=dtype, device="cuda")
        s[:n] = x
        srcs.append(s)
        d = torch.empty(npad + gel, dtype=dtype, device="cuda")
        _bits(d).fill_(-1)
        dsts.append(d)
    return srcs, dsts, npad


def _check_oneshot(dsts, xs, n, npad, scale, dtype, exact, world, what):
    out0 = dsts[0][:n]
    _check_reduced(out0, xs, scale, dtype, exact, world, what)
    for d in dsts:
        assert torch.equal(_bits(d[:n]), _bits(out0)), what + ": replicas differ"
        assert bool((_bits(d[n:npad]) == 0).all()), what + ": padding is not +0"
        assert bool((_bits(d[npad:]) == -1).all()), what + ": wrote past the padded end"


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("world", WORLDS)
def test_allreduce_oneshot_exact_and_bounded(world, dtype):
    """`px_allreduce_oneshot` at n in {1, VN - 1, VN, 3·512·VN + 5 (a ragged multi-CTA size),
    the largest the 64 KB stage half holds}, scale 1 and 1/W, grids 1, 3, 128 // W.  Zero
    padding up to the 16-byte vector reduces to +0 and nothing past it is written.  Every
    rank's Σx² (of the whole vector, the padding adding nothing) within `norm_bound`.  A size
    whose padded bytes exceed the stage half is refused with -2.  Catches a Σx² taken before
    the scale, a wrong stage half or peer, and a ragged tail read or written wrong."""
    from parallax_b200.parallel import nvops
    from parallax_b200.parallel.symmetric import CH_SMALL
    vn, es = _vn(dtype), _es(dtype)
    fabs = _world(world)
    half = fabs[0].small_stage.nbytes // 2
    ss = [torch.zeros(1, device="cuda") for _ in fabs]
    gen = torch.Generator(device="cuda").manual_seed(31 + world)
    for mb in _grids(world):
        for n in (1, vn - 1, vn, 3 * 512 * vn + 5, half // es):
            nvec = -(-n // vn)
            ctas = max(1, min(-(-nvec // 512), mb))
            iters = -(-nvec // (ctas * 512))
            for exact in (True, False):
                for scale in sorted({1.0, 1.0 / world}):
                    xs = _operands(gen, world, n, dtype, exact)
                    srcs, dsts, npad = _oneshot_io(xs, n, dtype, vn)
                    for s in ss:
                        s.zero_()
                    torch.cuda.synchronize()
                    _oneshot_round(fabs, srcs, dsts, ss, n, dtype, scale, CH_SMALL, mb)
                    torch.cuda.synchronize()
                    what = "oneshot W=%d n=%d mb=%d exact=%s scale=%g" % (
                        world, n, mb, exact, scale)
                    _check_oneshot(dsts, xs, n, npad, scale, dtype, exact, world, what)
                    if exact or dtype == torch.float32:
                        pre = R.reduce_exact(xs, scale) if exact else dsts[0][:n].float()
                        for r in range(world):
                            _check_sumsq(ss[r], pre, vn, iters, ctas, what + " rank %d" % r)
    n_big = half // es + 1
    with pytest.raises(RuntimeError, match=r"rc=-2"):
        nvops.allreduce_oneshot(fabs[0].heap, srcs[0], dsts[0], fabs[0].small_stage, n_big,
                                dtype, 1.0, CH_SMALL, stream=fabs[0].comm_stream)
    _close(fabs)


@pytest.mark.parametrize("world", WORLDS)
def test_allreduce_oneshot_stage_parity_sequences(world):
    """The one-shot kernel picks its stage half from the parity of each CTA's own barrier-slot
    epoch, which is safe because a CTA index covers the same vectors whatever the size (at a
    fixed max_blocks).  A sequence on one channel of one CTA, several, capped at max_blocks,
    and back, must be bitwise right at every call; so must one-shot calls on CH_USER[0]
    interleaved with two-shot calls on the CH_USER pair (whose start barrier advances the same
    slots), as the public all-reduce issues them.  Catches a parity taken from the wrong slot
    or epoch: a call would then read a peer's previous (or half-written) stage."""
    from parallax_b200.parallel import nvops
    from parallax_b200.parallel.symmetric import CH_SMALL, CH_USER
    dtype, vn = torch.float32, 4
    fabs = _world(world)
    gen = torch.Generator(device="cuda").manual_seed(41 + world)
    mb = 4
    one, several, capped = 100, 600 * vn, 3000 * vn      # 1, 2 and 4 (of 6) CTAs
    for n in (one, several, capped, one, capped, several, one, several, capped):
        xs = R.exact_operands(gen, world, n, "cuda")
        srcs, dsts, npad = _oneshot_io(xs, n, dtype, vn)
        torch.cuda.synchronize()
        _oneshot_round(fabs, srcs, dsts, None, n, dtype, 1.0 / world, CH_SMALL, mb)
        torch.cuda.synchronize()
        _check_oneshot(dsts, xs, n, npad, 1.0 / world, dtype, True, world,
                       "oneshot sequence W=%d n=%d" % (world, n))
    # interleaved with the two-shot on the public API's channel pair
    two_mb = min(32, 128 // world)
    nt = world * 3000 * vn
    bufs = [f.heap.alloc(nt * 4 + GUARD, "x") for f in fabs]
    for it, n in enumerate((one, capped, several, one, capped)):
        xs = R.exact_operands(gen, world, n, "cuda")
        srcs, dsts, npad = _oneshot_io(xs, n, dtype, vn)
        ys = R.exact_operands(gen, world, nt, "cuda")
        for r, b in enumerate(bufs):
            _arm(b, nt * 4)
            b.tensor(dtype, nt).copy_(ys[r])
        torch.cuda.synchronize()
        _oneshot_round(fabs, srcs, dsts, None, n, dtype, 1.0, CH_USER[0], 8)
        for r, f in enumerate(fabs):
            nvops.allreduce_twoshot(f.heap, bufs[r].c_ptrs(), nt, dtype, 1.0 / world, CH_USER,
                                    max_blocks=two_mb, stream=f.comm_stream)
        torch.cuda.synchronize()
        what = "interleaved W=%d it=%d" % (world, it)
        _check_oneshot(dsts, xs, n, npad, 1.0, dtype, True, world, what)
        want = R.reduce_exact(ys, 1.0 / world)
        for b in bufs:
            assert torch.equal(_bits(b.tensor(dtype, nt)), _bits(want)), what
            _guard_ok(b, nt * 4, what)
    _close(fabs)


# ------------------------------------------------------------------- broadcast and all-gather
def _pattern(rank, nbytes):
    """int32 `rank << 24 | index`: every element of every rank distinct."""
    return torch.arange(nbytes // 4, dtype=torch.int32, device="cuda") | (rank << 24)


@pytest.mark.parametrize("world", WORLDS)
def test_broadcast_and_allgather_distinct_elements(world):
    """`px_broadcast` from every root and `px_allgather` (templated on W) with every element
    distinct (rank << 24 | index), at 16 bytes, 777 vectors (not a multiple of the grid
    stride) and 4·ctas·512 + 99 vectors (several grid-stride rounds), grids 1, 3, 128 // W.
    Bitwise; guards intact.  Byte counts that are not a multiple of 16 are refused with -1.
    Catches a swapped, duplicated or misplaced 16-byte vector, a wrong root, a slice stored at
    the wrong offset or into the wrong peer -- none of which a constant fill can see."""
    from parallax_b200.parallel import nvops
    from parallax_b200.parallel.symmetric import CH_MAIN
    fabs = _world(world)
    sizes = lambda mb: (16, 777 * 16, (4 * mb * 512 + 99) * 16)   # noqa: E731
    top = max(sizes(mb)[-1] for mb in _grids(world))
    bufs = [f.heap.alloc(world * top + GUARD, "x") for f in fabs]
    for mb in _grids(world):
        for nb in sizes(mb):
            for root in range(world):
                for r, b in enumerate(bufs):
                    _arm(b, nb)
                    b.tensor(torch.int32, nb // 4).copy_(_pattern(r, nb))
                torch.cuda.synchronize()
                for r, f in enumerate(fabs):
                    nvops.broadcast(f.heap, bufs[r].c_ptrs(), nb, root, CH_MAIN, mb,
                                    stream=f.comm_stream)
                torch.cuda.synchronize()
                what = "broadcast W=%d bytes=%d mb=%d root=%d" % (world, nb, mb, root)
                want = _pattern(root, nb)
                for b in bufs:
                    assert torch.equal(b.tensor(torch.int32, nb // 4), want), what
                    _guard_ok(b, nb, what)
            # all-gather: slice r of every buffer comes from rank r
            tot = world * nb
            for r, b in enumerate(bufs):
                _arm(b, tot)
                b.tensor(torch.int32, tot // 4).copy_(_pattern(r, tot))
            torch.cuda.synchronize()
            for r, f in enumerate(fabs):
                nvops.allgather(f.heap, bufs[r].c_ptrs(), nb, CH_MAIN, mb, stream=f.comm_stream)
            torch.cuda.synchronize()
            what = "allgather W=%d slice=%d mb=%d" % (world, nb, mb)
            q = nb // 4
            want = torch.cat([_pattern(r, tot)[r * q:(r + 1) * q] for r in range(world)])
            for b in bufs:
                assert torch.equal(b.tensor(torch.int32, tot // 4), want), what
                _guard_ok(b, tot, what)
    with pytest.raises(RuntimeError, match=r"rc=-1"):
        nvops.broadcast(fabs[0].heap, bufs[0].c_ptrs(), 24, 0, CH_MAIN, 1,
                        stream=fabs[0].comm_stream)
    with pytest.raises(RuntimeError, match=r"rc=-1"):
        nvops.allgather(fabs[0].heap, bufs[0].c_ptrs(), 24, CH_MAIN, 1,
                        stream=fabs[0].comm_stream)
    _close(fabs)


# --------------------------------------------------------------------------- fused dense step
class _Step(object):
    """Per-rank buffers of one fused dense step over a bucket of up to `nmax` elements."""

    def __init__(self, fabs, nmax, dtype, nslots):
        W, es = len(fabs), _es(dtype)
        self.fabs, self.dtype, self.es = fabs, dtype, es
        self.gb = [f.heap.alloc(nmax * es + GUARD, "g") for f in fabs]
        self.pb = [f.heap.alloc(nmax * es + GUARD, "p") for f in fabs]
        self.loc = [torch.zeros(4, device="cuda") for _ in fabs]
        self.tot = [torch.zeros(4, device="cuda") for _ in fabs]
        self.scale = [torch.ones(1, device="cuda") for _ in fabs]
        self.norm = [torch.zeros(1, device="cuda") for _ in fabs]
        self.W, self.nslots = W, nslots

    def load(self, n, xs, w0, slots0, ema):
        """Gradients in, 0xFF-armed parameter buffers, fp32 slices of the shared state."""
        W, sl = self.W, n // self.W
        for r in range(W):
            _arm(self.gb[r], n * self.es)
            self.gb[r].tensor(self.dtype, n).copy_(xs[r])
            _arm(self.pb[r], n * self.es)
            self.loc[r].zero_()
        cut = lambda t, r: _guarded(t[r * sl:(r + 1) * sl])   # noqa: E731
        self.master = [cut(w0, r) for r in range(W)]
        self.slots = [[cut(s, r) for s in slots0] for r in range(W)]
        self.ema = [cut(w0, r) for r in range(W)] if ema else [None] * W
        self.red = [_guarded(torch.full((sl,), float("nan"), device="cuda"))
                    for _ in range(W)]
        self.n = n

    def run(self, hp, kind, mb, decay, two_phase, max_norm=None):
        from parallax_b200.parallel import nvops
        from parallax_b200.parallel.symmetric import CH_COMM, CH_SMALL
        fabs, n, W, dt = self.fabs, self.n, self.W, self.dtype

        def s(r, i):
            return self.slots[r][i] if len(self.slots[r]) > i else None

        def launch(r, f, mode, red, clip, sumsq):
            nvops.dense_step(f.heap, self.gb[r].c_ptrs(), self.pb[r].c_ptrs(), self.master[r],
                             s(r, 0), s(r, 1), self.ema[r], red, hp, clip, sumsq, n, 1.0 / W,
                             decay, kind, mode, dt, CH_COMM, max_blocks=mb,
                             stream=f.comm_stream, slot2=s(r, 2))
        torch.cuda.synchronize()
        if not two_phase:
            for r, f in enumerate(fabs):
                launch(r, f, 0, None, None, None)
        else:
            for r, f in enumerate(fabs):
                launch(r, f, 1, self.red[r], None, self.loc[r])
            for r, f in enumerate(fabs):
                nvops.allreduce_oneshot(f.heap, self.loc[r], self.tot[r], f.small_stage, 4,
                                        torch.float32, 1.0, CH_SMALL, stream=f.comm_stream)
            for r, f in enumerate(fabs):
                nvops.clip_scale(self.tot[r], max_norm, self.scale[r], self.norm[r], self.loc[r],
                                 stream=f.comm_stream)
                launch(r, f, 2, self.red[r], self.scale[r], None)
        torch.cuda.synchronize()

    def check_push(self, what):
        """Every rank's parameters are bitwise the RNE cast of the concatenated masters; no
        buffer was written past its end."""
        n = self.n
        want = torch.cat(self.master).to(self.dtype)
        for r, b in enumerate(self.pb):
            got = b.tensor(self.dtype, n)
            assert torch.equal(_bits(got), _bits(want)), "%s: rank %d params: %d of %d" % (
                what, r, int((_bits(got) != _bits(want)).sum()), n)
            _guard_ok(b, n * self.es, what + " params")
            _guard_ok(self.gb[r], n * self.es, what + " grads")
        for r in range(self.W):
            assert float(self.loc[r].abs().sum()) == 0.0, what + ": accumulator not re-armed"
            for name, t in [("master", self.master[r]), ("ema", self.ema[r]),
                            ("scratch", self.red[r])] + \
                    [("slot%d" % i, s) for i, s in enumerate(self.slots[r])]:
                if t is not None:
                    _tail_ok(t, "%s rank %d %s" % (what, r, name))


def _step_sizes(world, mb, vn):
    cap = 132 * 4 if world == 1 else mb
    return [world * vn * nv for nv in (1, 777, 3 * cap * 512 + 99)]


def _step_grids(world):
    return [0] if world == 1 else _grids(world)      # W = 1 ignores max_blocks (4·132 CTAs)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("world", WORLDS)
def test_dense_step_sgd_exact(world, dtype):
    """Mode 0 and the two-phase clip (mode 1 -> one-shot Σ of the ranks' Σg² -> `clip_scale`
    -> mode 2) with SGD at lr = 2^-3, weights on a 2^-10 grid and exact gradients: the kernel's
    g = fp32(Σx·fp32(1/W)) (times fp32(clip) in mode 2, one more rounding) and
    w = fmaf(-lr, g, w) are each one rounding of a value fp64 holds exactly, and so is the
    EMA at decay 0.75 ((1 - decay)·(m - w) is exact once m - w is rounded).  So the master,
    the mode-1 scratch, the EMA and the pushed parameters are predicted bitwise at every W,
    size and grid; the mode-1 norm is within `norm_bound(vn, iters, ctas, ranks=W)` of the
    fp64 norm of the exact scratch.  Catches a wrong slice, rank rotation, grid-stride round,
    a dropped or doubled 1/W or clip, and any rounding of the parameter push but RNE."""
    from parallax_b200 import optim
    vn = _vn(dtype)
    fabs = _world(world)
    nmax = max(max(_step_sizes(world, mb, vn)) for mb in _step_grids(world))
    st = _Step(fabs, nmax, dtype, 0)
    hp_list = optim.GradientDescent(2.0 ** -3).hyper(1)
    hp = torch.tensor(hp_list, device="cuda")
    lr, decay = 2.0 ** -3, 0.75
    gen = torch.Generator(device="cuda").manual_seed(51 + world)
    for mb in _step_grids(world):
        for n in _step_sizes(world, mb, vn):
            for two_phase in (False, True):
                xs = R.exact_operands(gen, world, n, "cuda")
                w0 = torch.randint(-4096, 4097, (n,), generator=gen, device="cuda").float() \
                    * 2.0 ** -10
                st.load(n, xs, w0, (), ema=True)
                g32 = R.reduce_exact(xs, 1.0 / world)
                what = "dense_step sgd W=%d n=%d mb=%d two_phase=%s" % (world, n, mb, two_phase)
                max_norm = None
                if two_phase:
                    n64 = float(g32.double().norm())
                    max_norm = R.f32(0.5 * n64) if n64 > 0 else 1.0
                st.run(hp, "sgd", mb, decay, two_phase, max_norm)
                g = g32
                if two_phase:
                    assert torch.equal(_bits(torch.cat(st.red)), _bits(g32)), what + ": scratch"
                    ctas, iters = dense_grid(n, world, mb, vn=vn)
                    ss = float((g32.double() ** 2).sum())
                    rel = norm_bound(vn, iters, ctas, ranks=world)
                    for r in range(world):
                        got = float(st.norm[r])
                        assert abs(got - math.sqrt(ss)) <= (rel / 2 + U) * math.sqrt(ss), \
                            "%s: norm %r vs %r" % (what, got, math.sqrt(ss))
                        assert torch.equal(st.scale[r], st.scale[0]), what + ": scales differ"
                    c = float(st.scale[0])
                    g = (g32.double() * c).float()
                w_want = (w0.double() - lr * g.double()).float()
                d = (w0.double() - w_want.double()).float()
                m_want = (w0.double() - (1 - decay) * d.double()).float()
                assert torch.equal(_bits(torch.cat(st.master)), _bits(w_want)), what + ": master"
                assert torch.equal(_bits(torch.cat(st.ema)), _bits(m_want)), what + ": ema"
                st.check_push(what)
    _close(fabs)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("world", WORLDS)
def test_dense_step_rules_random(world, dtype):
    """Momentum (Nesterov), Adagrad, Adam, FTRL and centered RMSProp, one step (mode 0, and the
    two-phase clip at the largest size) from a shared random fp32 state on randn gradients,
    against `optim.apply_dense_` on fp64 copies within the calibrated bound of
    `tests/dense_plane_ref.py` (C_kind·u·M; see its docstring for M and how C_kind was set).
    The parameters every rank holds are bitwise the RNE cast of the concatenated masters.
    Catches a slot stored to the wrong slice or owner, a rule read with the wrong slot, a
    gradient scaled by the wrong 1/W or clip."""
    vn = _vn(dtype)
    fabs = _world(world)
    nmax = max(max(_step_sizes(world, mb, vn)) for mb in _step_grids(world))
    st = _Step(fabs, nmax, dtype, 3)
    gen = torch.Generator(device="cuda").manual_seed(61 + world)
    for kind in R.DENSE_KINDS:
        opt = R.make_opt(kind)
        hp_list = opt.hyper(2)
        hp = torch.tensor(hp_list, device="cuda")
        for mb in _step_grids(world):
            sizes = _step_sizes(world, mb, vn)
            for n in sizes:
                for two_phase in ((False, True) if n == sizes[-1] else (False,)):
                    xs = R.random_operands(gen, world, n, dtype, "cuda")
                    w0, s0 = R.random_state(gen, kind, n, "cuda")
                    st.load(n, xs, w0, s0, ema=False)
                    g64, G = R.reduce_ref(xs, 1.0 / world)
                    max_norm = None
                    if two_phase:
                        max_norm = R.f32(0.5 * float(g64.norm()))
                    st.run(hp, kind, mb, 0.0, two_phase, max_norm)
                    if two_phase:
                        c = float(st.scale[0])
                        g64, G = g64 * c, G * c
                    w64, s64 = R.apply64(kind, w0, s0, g64, hp_list)
                    what = "dense_step %s W=%d n=%d mb=%d two_phase=%s" % (
                        kind, world, n, mb, two_phase)
                    R.check_rule(what, kind, torch.cat(st.master),
                                 [torch.cat([st.slots[r][i] for r in range(world)])
                                  for i in range(len(s0))], w0, s0, w64, s64, G, world, hp_list)
                    st.check_push(what)
    _close(fabs)


# ------------------------------------------------------------------------------ async apply
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("world", WORLDS)
def test_dense_async_every_kind(world, dtype):
    """`px_dense_async` (Hogwild apply of an async PS dense bucket) for all twelve elementwise
    rules (the eleven kinds and FTRL at learning-rate power -0.3), with and without the clip
    pointer, weight decay on SGD and Adam: ranks apply one at a time, each its un-averaged gradient × hp[GSCALE] × clip, onto the owners' fp32
    masters and slots, against the same applies in sequence in fp64 within the calibrated
    `ASYNC_C` bound (`tests/dense_plane_ref.py`).  After each apply the writer's parameters
    are bitwise the cast of the concatenated masters and every other rank's are untouched.
    Catches an ignored clip pointer, a wrong owner or offset inside the owner's slice, a slot
    of the wrong owner, a parameter store outside the writer."""
    from parallax_b200 import optim
    from parallax_b200.parallel import nvops
    vn, es = _vn(dtype), _es(dtype)
    big = -(-(3 * 128 * 512 + 99) // world)
    cases = ((1, 1), (3, 777), (128, big))           # (max_blocks, vectors per owner)
    nmax = world * vn * big
    gen = torch.Generator(device="cuda").manual_seed(71 + world)
    gel = GUARD // es
    grads = [torch.empty(nmax, dtype=dtype, device="cuda") for _ in range(world)]
    params = [torch.empty(nmax + gel, dtype=dtype, device="cuda") for _ in range(world)]
    clip_t = torch.tensor([0.625], device="cuda")
    for variant in R.ELEMENTWISE_VARIANTS:
        wd = 0.01 if variant in ("sgd", "adam") else 0.0
        opt = R.make_opt(variant, wd)
        kind = opt.kind
        hp_list = opt.hyper(2)
        hp = torch.tensor(hp_list, device="cuda")
        ns = optim.NUM_SLOTS[kind]
        for mb, nv in cases:
            n = world * vn * nv
            sl = n // world
            for clip in (None, clip_t):
                xs = R.random_operands(gen, world, n, dtype, "cuda")
                w0, s0 = R.random_state(gen, variant, n, "cuda")
                masters = [_guarded(w0[r * sl:(r + 1) * sl]) for r in range(world)]
                slots = [[_guarded(s[r * sl:(r + 1) * sl]) for r in range(world)] for s in s0]
                arr = lambda ts: (ctypes.c_void_p * world)(*[t.data_ptr() for t in ts])  # noqa
                m_c = arr(masters)
                s_c = [arr(s) for s in slots] + [None] * (3 - ns)
                for r in range(world):
                    grads[r][:n].copy_(xs[r])
                    _bits(params[r]).fill_(-1)
                c = R.f32(float(clip_t)) if clip is not None else 1.0
                w64, s64 = w0.double(), tuple(s.double() for s in s0)
                G = torch.zeros_like(w64)
                what = "async %s W=%d n=%d mb=%d clip=%s" % (variant, world, n, mb,
                                                             clip is not None)
                for r in range(world):
                    before = [p.clone() for p in params]
                    torch.cuda.synchronize()
                    nvops.dense_async(grads[r], params[r], m_c, s_c[0], s_c[1], hp, clip, n,
                                      kind, dtype, r, world, max_blocks=mb, slot2_c=s_c[2])
                    torch.cuda.synchronize()
                    w64, s64 = R.apply64(variant, w64, s64, xs[r].double() * c, hp_list)
                    G = G + xs[r].double().abs() * c
                    want = torch.cat(masters).to(dtype)
                    assert torch.equal(_bits(params[r][:n]), _bits(want)), \
                        "%s: writer %d's parameters" % (what, r)
                    assert bool((_bits(params[r][n:]) == -1).all()), what + ": past n"
                    for q in range(world):
                        if q != r:
                            assert torch.equal(_bits(params[q]), _bits(before[q])), \
                                "%s: rank %d's parameters changed by %d's apply" % (what, q, r)
                for r in range(world):
                    for t in [masters[r]] + [s[r] for s in slots]:
                        _tail_ok(t, "%s owner %d" % (what, r))
                R.check_rule(what, variant, torch.cat(masters),
                             [torch.cat(s) for s in slots], w0, s0, w64, s64, G, world,
                             hp_list, R.ASYNC_C)


# ------------------------------------------------------------------------- sumsq, clip_scale
@pytest.mark.parametrize("dtype", DTYPES)
def test_sumsq_against_fp64(dtype):
    """`px_sumsq` (Σ(x·mul)² of the async clip) with mul = 0.75 at one vector, 777 vectors and
    3·128·512 + 77 vectors (four grid-stride rounds of its 97 CTAs, one per 2048 vectors),
    against the fp64 sum within `norm_bound(vn, iters, ctas + 2)`: each term is rounded three times
    ((x·x)·mul)·mul instead of once.  A length that is not a whole number of 16-byte vectors is
    refused with -1 instead of having its tail dropped."""
    from parallax_b200.parallel import nvops
    vn = _vn(dtype)
    gen = torch.Generator(device="cuda").manual_seed(81)
    out = torch.zeros(1, device="cuda")
    mul = 0.75
    for nv in (1, 777, 3 * 128 * 512 + 77):
        n = nv * vn
        x = torch.randn(n, generator=gen, device="cuda").to(dtype)
        out.zero_()
        nvops.sumsq(x, n, dtype, mul, out)
        torch.cuda.synchronize()
        ctas = max(1, min(-(-nv // 2048), 128))
        iters = -(-nv // (ctas * 512))
        _check_sumsq(out, x.double() * mul, vn, iters, ctas + 2, "sumsq n=%d" % n)
    with pytest.raises(RuntimeError, match=r"rc=-1"):
        nvops.sumsq(x, 5 * vn + 1, dtype, 1.0, out)


def test_clip_scale_semantics():
    """`px_clip_scale` against the host fabric's clip (`host_backend.py`, `_clip`): norm 0 and
    a norm below max_norm give 1, above gives max_norm / norm, +inf gives 0, and NaN gives a
    multiplier of 1 (the host computes a NaN scale and skips scaling, since NaN < 1 is false;
    fmaxf drops the NaN).  The fp32 result is bitwise max_norm / max(sqrtf(Σ), max_norm);
    `norm_out` holds sqrtf(Σ) and `zero_after` is zeroed."""
    from parallax_b200.parallel import nvops
    max_norm = 10.0
    for tot in (0.0, 4.0, 99.0, 100.0, 400.0, 12345.678, float("inf"), float("nan")):
        t = torch.tensor([tot], device="cuda")
        scale = torch.full((1,), -1.0, device="cuda")
        norm = torch.full((1,), -1.0, device="cuda")
        zero = torch.full((4,), 7.0, device="cuda")
        nvops.clip_scale(t, max_norm, scale, norm, zero)
        torch.cuda.synchronize()
        n32 = torch.tensor([tot], dtype=torch.float32).sqrt()
        h_norm = float(n32)
        h_scale = max_norm / max(h_norm, max_norm)       # the host's expression
        h_mult = h_scale if h_scale < 1.0 else 1.0
        what = "clip_scale Σ=%r" % tot
        assert float(scale) == pytest.approx(h_mult, rel=2 * U, abs=0), what
        if tot == tot:
            want = torch.tensor([max_norm], dtype=torch.float32) / torch.maximum(
                n32, torch.tensor([max_norm], dtype=torch.float32))
            assert torch.equal(scale.cpu(), want), what
            assert torch.equal(norm.cpu(), n32), what
        else:
            assert float(scale) == 1.0 and math.isnan(float(norm)), what
        assert float(zero[0]) == 0.0 and bool((zero[1:] == 7.0).all()), what
