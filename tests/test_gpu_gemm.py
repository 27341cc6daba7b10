"""wgmma GEMM core (descriptor / swizzle / major-ness validation) vs fp64 matmul.  GPU only."""
import pytest
import torch

pytestmark = pytest.mark.gpu

TOL = 2e-3   # TF32 operands (10-bit mantissa), fp32 accumulate


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


@pytest.mark.parametrize('a_mn,b_mn', [(0, 0), (1, 0), (0, 1), (1, 1)])
@pytest.mark.parametrize('M,N,K,batch', [(128, 128, 64, 1), (200, 300, 100, 2), (32, 200, 1024, 3), (256, 64, 40, 2)])
def test_gemm_majors(a_mn, b_mn, M, N, K, batch):
    from hawkeye_b200 import ops
    torch.manual_seed(M + N + K)
    A = torch.randn(batch, M, K, device='cuda')
    B = torch.randn(batch, K, N, device='cuda')
    ref = torch.bmm(A.double(), B.double())
    Ain = A.transpose(1, 2).contiguous() if a_mn else A            # [b,K,M] if MN-major
    Bin = B if b_mn else B.transpose(1, 2).contiguous()            # [b,K,N] if MN-major else [b,N,K]
    out = ops.gemm_tf32(Ain, Bin, a_mn=bool(a_mn), b_mn=bool(b_mn))
    torch.cuda.synchronize()
    err = _rel(out, ref)
    print(f'gemm a_mn={a_mn} b_mn={b_mn} {M}x{N}x{K} b{batch}: rel={err:.3e}')
    assert err < TOL


def test_gemm_epilogue():
    from hawkeye_b200 import ops
    torch.manual_seed(1)
    b, n = 3, 256
    A = torch.randn(b, n, n, device='cuda') / 16
    B = torch.randn(b, n, n, device='cuda') / 16
    D = torch.randn(b, n, n, device='cuda')
    av = torch.rand(b, device='cuda') + 0.5
    I = torch.eye(n, device='cuda', dtype=torch.float64)
    ref = -0.5 * av.double().view(b, 1, 1) * torch.bmm(A.double(), B.double()) + 1.5 * I + 0.25 * D.double()
    out = ops.gemm_tf32(A, B, b_mn=True, alpha=-0.5, alpha_vec=av, diag=1.5, D=D, beta=0.25)
    assert _rel(out, ref) < TOL
    out_t = ops.gemm_tf32(A, B, b_mn=True, alpha=-0.5, alpha_vec=av, diag=1.5, D=D, beta=0.25, trans_c=True)
    assert _rel(out_t, ref.transpose(1, 2)) < TOL
    # shared (2-D) B operand and row-broadcast D (ldd = 0)
    drow = torch.randn(b, 1, n, device='cuda')
    out = ops.gemm_tf32(A, B[0], b_mn=True, D=drow, beta=2.0)
    ref = torch.matmul(A.double(), B[0].double()) + 2.0 * drow.double()
    assert _rel(out, ref) < TOL
