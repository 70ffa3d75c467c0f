"""wgmma/TMA GEMM vs a plain PyTorch fp32 reference."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("M,N,K,splits,bn", [
    (128, 128, 64, 1, 128), (128, 128, 512, 1, 128), (128, 512, 8192, 1, 128),
    (128, 512, 8192, 16, 128), (128, 512, 8192, 32, 64), (128, 2048, 512, 2, 128),
    (128, 8192, 512, 1, 128), (256, 512, 2048, 4, 128), (128, 64, 256, 4, 64),
])
@pytest.mark.parametrize("with_addend", [False, True])
@pytest.mark.parametrize("cluster", [False, True])
def test_gemm_tn_matches_fp32(M, N, K, splits, bn, with_addend, cluster):
    """cluster=True: the K-splits of a tile are one thread-block cluster and reduce through
    distributed shared memory (splits 2..16 dividing 128; others fall back to the L2 workspace)."""
    from parallax_b200.ops.gemm import gemm_tn
    torch.manual_seed(0)
    A = (torch.randn(M, K, device="cuda") * 0.5).bfloat16()
    Bt = (torch.randn(N, K, device="cuda") * 0.5).bfloat16()
    D = (torch.randn(M, N, device="cuda")).bfloat16() if with_addend else None
    ref = A.float() @ Bt.float().t()
    if D is not None:
        ref = ref + D.float()
    for _ in range(2):                       # second call: workspace was re-zeroed
        out = gemm_tn(A, Bt, addend=D, splits=splits, bn=bn, cluster=cluster)
        torch.cuda.synchronize()
        err = (out.float() - ref).abs().max().item()
        scale = ref.abs().max().item()
        assert err <= 1e-2 * scale + 1e-2, (err, scale)
