"""wgmma/TMA GEMM vs plain PyTorch fp64 references."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu


def _exact_operands(M, N, K, with_addend, seed):
    """Small integers × 2^-3 for A and B, × 2^-6 for the addend: every fp32 partial sum of
    the product is exact in any order and any split, so the bf16 output is fully determined."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    A = (torch.randint(-4, 5, (M, K), device="cuda", generator=g) * 0.125).bfloat16()
    Bt = (torch.randint(-4, 5, (N, K), device="cuda", generator=g) * 0.125).bfloat16()
    D = (torch.randint(-64, 65, (M, N), device="cuda", generator=g) / 64.0).bfloat16() \
        if with_addend else None
    ref = A.double() @ Bt.double().t()
    if D is not None:
        ref = ref + D.double()
    return A, Bt, D, ref.bfloat16()


def _assert_ws_clean(M, N):
    from parallax_b200.ops import gemm
    ws, tk = gemm._ws_cache[(M, N, str(torch.device("cuda", torch.cuda.current_device())))]
    assert int(torch.count_nonzero(ws)) == 0, "split-K workspace not re-zeroed"
    assert int(torch.count_nonzero(tk)) == 0, "split-K tickets not reset"


def _l2_path(splits, cluster):
    return splits > 1 and not (cluster and 2 <= splits <= 16 and 128 % splits == 0)


_EXACT = [
    # the products of ops/fused.py at the LM1B bench shape (B 128, P 512, S 2048):
    # dh_{t-1} = dH_{t-1} + dgates_t·Wh^T over 8 cluster splits or 16 L2 splits
    (128, 512, 8192, 8, 64, True), (128, 512, 8192, 16, 64, True),
    # a wide output (N 2048) over 4 splits: the shape of dm = dH·W_P^T + dgates·(W_P·Wh)^T,
    # one product per step with the combined weight (tools/bench_lstm_gemms.py times it)
    (128, 2048, 8192, 4, 64, True),
    # dh_rec of the first step: no addend
    (128, 512, 8192, 8, 64, False), (128, 512, 8192, 16, 64, False),
    # cluster sizes × tile widths, 9 K-blocks per split: the 4-stage ring wraps twice and
    # the last K-block lands on phase 0 of the second lap (odd number of full laps)
    *[(128, 256, s * 9 * 64, s, bn, True) for s in (2, 4, 8, 16) for bn in (64, 128)],
    # more than one row of tiles
    (256, 512, 4096, 8, 64, True), (384, 256, 2048, 4, 128, True),
    # splits that do not divide 128: no cluster, L2 workspace + ticket
    (128, 256, 3 * 9 * 64, 3, 64, True), (128, 512, 5 * 4 * 64, 5, 128, False),
    # no split
    (128, 512, 9 * 64, 1, 64, True), (256, 256, 17 * 64, 1, 128, False),
]


@pytest.mark.parametrize("M,N,K,splits,bn,with_addend", _EXACT)
@pytest.mark.parametrize("cluster", [False, True])
def test_gemm_tn_exact_on_small_integers(M, N, K, splits, bn, with_addend, cluster):
    """Bit-for-bit against fp64: any misplaced tile, row, column, K-block or split shows."""
    from parallax_b200.ops.gemm import gemm_tn
    A, Bt, D, ref = _exact_operands(M, N, K, with_addend, seed=M + N + K + splits + bn)
    for _ in range(2):                       # second call: the L2 workspace was re-zeroed
        out = gemm_tn(A, Bt, addend=D, splits=splits, bn=bn, cluster=cluster)
        torch.cuda.synchronize()
        bad = int((out.view(torch.int16) != ref.view(torch.int16)).sum())
        assert bad == 0, "%d of %d elements differ" % (bad, out.numel())
        if _l2_path(splits, cluster):
            _assert_ws_clean(M, N)


@pytest.mark.parametrize("M,N,K,splits,bn", [
    (128, 128, 64, 1, 128), (128, 128, 512, 1, 128), (128, 512, 8192, 1, 128),
    (128, 512, 8192, 16, 128), (128, 512, 8192, 32, 64), (128, 2048, 512, 2, 128),
    (128, 8192, 512, 1, 128), (256, 512, 2048, 4, 128), (128, 64, 256, 4, 64),
])
@pytest.mark.parametrize("with_addend", [False, True])
@pytest.mark.parametrize("cluster", [False, True])
def test_gemm_tn_matches_fp32(M, N, K, splits, bn, with_addend, cluster):
    """Random operands, per-element bound against fp64 of the same bf16 inputs: half a bf16
    ulp of output rounding (2^-8 relative) plus the fp32 accumulation term
    2^-16·(|A|·|B|^T)_ij.  cluster=True: the K-splits of a tile are one thread-block cluster
    and reduce through distributed shared memory (splits 2..16 dividing 128; others fall back
    to the L2 workspace)."""
    from parallax_b200.ops.gemm import gemm_tn
    torch.manual_seed(0)
    A = (torch.randn(M, K, device="cuda") * 0.5).bfloat16()
    Bt = (torch.randn(N, K, device="cuda") * 0.5).bfloat16()
    D = (torch.randn(M, N, device="cuda")).bfloat16() if with_addend else None
    ref = A.double() @ Bt.double().t()
    if D is not None:
        ref = ref + D.double()
    mag = A.double().abs() @ Bt.double().abs().t()
    bound = 2.0 ** -8 * ref.abs() + 2.0 ** -16 * mag
    for _ in range(2):                       # second call: workspace was re-zeroed
        out = gemm_tn(A, Bt, addend=D, splits=splits, bn=bn, cluster=cluster)
        torch.cuda.synchronize()
        err = (out.double() - ref).abs()
        worst = int(torch.argmax(err - bound))
        assert bool((err <= bound).all()), \
            (worst // N, worst % N, float(err.view(-1)[worst]), float(bound.view(-1)[worst]))
        if _l2_path(splits, cluster):
            _assert_ws_clean(M, N)


def test_gemm_tn_l2_workspace_reused_across_k_and_splits():
    """Back-to-back L2-path calls share one (M, N) workspace: each must leave it zeroed for the
    next one, whatever its K and split count."""
    from parallax_b200.ops.gemm import gemm_tn
    M, N = 128, 512
    for i, (K, splits, bn, add) in enumerate([(8192, 16, 64, True), (1024, 2, 128, False),
                                              (4096, 32, 64, True), (3 * 9 * 64, 3, 64, True),
                                              (8192, 16, 64, False)]):
        A, Bt, D, ref = _exact_operands(M, N, K, add, seed=100 + i)
        out = gemm_tn(A, Bt, addend=D, splits=splits, bn=bn, cluster=False)
        torch.cuda.synchronize()
        assert torch.equal(out.view(torch.int16), ref.view(torch.int16)), (K, splits, bn)
        _assert_ws_clean(M, N)


@pytest.mark.parametrize("cluster", [False, True])
def test_gemm_tn_out_and_addend_as_row_views(cluster):
    """`fused.py` passes `out=dh_tot[t-1]` and `addend=dH[t-1]`, rows of [T, B, P] buffers:
    the product lands in its row only and the neighbouring rows keep their bits."""
    from parallax_b200.ops.gemm import gemm_tn
    T, M, N, K = 4, 128, 512, 8192
    A, Bt, _, _ = _exact_operands(M, N, K, False, seed=7)
    g = torch.Generator(device="cuda").manual_seed(8)
    dH = (torch.randint(-64, 65, (T, M, N), device="cuda", generator=g) / 64.0).bfloat16()
    dh_tot = torch.full((T, M, N), float("nan"), dtype=torch.bfloat16, device="cuda")
    before = dh_tot.clone()
    t = 2
    out = gemm_tn(A, Bt, addend=dH[t - 1], splits=8 if cluster else 16, bn=64,
                  out=dh_tot[t - 1], cluster=cluster)
    torch.cuda.synchronize()
    assert out.data_ptr() == dh_tot[t - 1].data_ptr()
    ref = (A.double() @ Bt.double().t() + dH[t - 1].double()).bfloat16()
    assert torch.equal(dh_tot[t - 1].view(torch.int16), ref.view(torch.int16))
    for r in (0, 2, 3):
        assert torch.equal(dh_tot[r].view(torch.int16), before[r].view(torch.int16)), r


@pytest.mark.parametrize("M,N,K,splits,bn,cluster,with_ws,rc", [
    (192, 512, 1024, 1, 64, 0, False, -1),      # M % 128
    (128, 512, 1000, 1, 64, 0, False, -1),      # K % 64
    (128, 96, 1024, 1, 64, 0, False, -1),       # N % bn
    (128, 192, 1024, 1, 128, 0, False, -1),     # N % bn
    (128, 512, 1024, 1, 96, 0, False, -1),      # bn not 64 / 128
    (128, 512, 1024, 3, 64, 0, True, -2),       # K % (splits·64)
    (128, 512, 1024, 0, 64, 0, True, -2),       # splits < 1
    (128, 512, 8192, 32, 64, 1, False, -4),     # cluster of 32 splits
    (128, 512, 1536, 3, 64, 1, False, -4),      # cluster size not dividing 128
    (128, 512, 1024, 4, 64, 0, False, -3),      # L2 split-K without workspace
])
def test_px_gemm_tc_refuses_bad_shapes(M, N, K, splits, bn, cluster, with_ws, rc):
    """Argument checks return their negative codes before anything is launched.  The buffers
    cover whole tiles of every case (256 rows, 512 columns, K 8192), so a check that stopped
    refusing would fail the return-code assertion, not write out of bounds."""
    from parallax_b200 import ops
    from parallax_b200.ops import gemm  # noqa: F401  (registers the signature)
    vp = ctypes.c_void_p
    assert M <= 256 and N <= 512 and K <= 8192
    A = torch.zeros(256, 8192, dtype=torch.bfloat16, device="cuda")
    Bt = torch.zeros(512, 8192, dtype=torch.bfloat16, device="cuda")
    C = torch.zeros(256, 512, dtype=torch.bfloat16, device="cuda")
    ws = torch.zeros(256, 512, dtype=torch.float32, device="cuda")
    tk = torch.zeros(64, dtype=torch.int32, device="cuda")
    got = ops.lib().px_gemm_tc(
        vp(A.data_ptr()), vp(Bt.data_ptr()), vp(C.data_ptr()), vp(0),
        vp(ws.data_ptr()) if with_ws else vp(0), vp(tk.data_ptr()) if with_ws else vp(0),
        M, N, K, splits, bn, cluster, vp(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    assert got == rc
    assert int(torch.count_nonzero(C)) == 0
