"""Fused bilinear pooling kernels vs the oracle (oracle/hop_oracle.py) and the reference-generated fixtures."""
import pytest
import torch

import detgen
from conftest import rel_l2

pytestmark = pytest.mark.gpu


def test_fwd_bwd_golden(golden):
    from hawkeye_b200 import ops
    x = detgen.det_uniform((2, 128, 14, 14), 11).cuda().requires_grad_(True)
    y = ops.bilinear_pool(x)
    e = rel_l2(y.detach().cpu(), golden['bp_c128_y'])
    print('bp_c128 fwd rel', e)
    assert e < 1e-3
    dy = detgen.det(y.shape, 12).cuda()
    (dx,) = torch.autograd.grad(y, x, dy)
    e = rel_l2(dx.cpu(), golden['bp_c128_dx'])
    print('bp_c128 bwd rel', e)
    assert e < 2e-3


def test_full_size_golden(golden):
    from hawkeye_b200 import ops
    x = detgen.det_uniform((1, 512, 14, 14), 13).cuda().requires_grad_(True)
    y = ops.bilinear_pool(x)
    assert rel_l2(y.detach().cpu()[0, ::997], golden['bp_full_y_slice']) < 1e-3
    assert abs(y.detach().double().sum().item() - float(golden['bp_full_y_sum'])) / float(golden['bp_full_y_sum']) < 1e-3
    (dx,) = torch.autograd.grad(y, x, detgen.det(y.shape, 14).cuda())
    e = rel_l2(dx.cpu(), golden['bp_full_dx'])
    print('bp_full bwd rel', e)
    assert e < 2e-3


@pytest.mark.parametrize('B,C,H,W', [(3, 512, 14, 14), (2, 256, 8, 8), (5, 128, 6, 6), (2, 384, 14, 14), (2, 768, 4, 4)])
def test_vs_oracle(B, C, H, W):
    from hawkeye_b200 import ops
    from oracle import hop_oracle as O
    x = detgen.det_uniform((B, C, H, W), 5)
    dy = detgen.det((B, C * C), 6)
    xg = x.cuda().requires_grad_(True)
    y = ops.bilinear_pool(xg)
    (dx,) = torch.autograd.grad(y, xg, dy.cuda())
    y_ref = O.bilinear_pool_fwd(x.double())
    dx_ref = O.bilinear_pool_bwd(x.double(), dy.double())
    ef, eb = rel_l2(y.detach().cpu(), y_ref), rel_l2(dx.cpu(), dx_ref)
    print(f'bilinear {B}x{C}x{H}x{W}: fwd {ef:.2e} bwd {eb:.2e}')
    assert ef < 1e-3 and eb < 2e-3


def test_full_batch_properties():
    """benchmark size (B=32, C=512, 14x14): size-independent properties — unit row norm, symmetry, positivity."""
    from hawkeye_b200 import ops
    x = torch.rand(32, 512, 14, 14, device='cuda', generator=torch.Generator('cuda').manual_seed(0))
    y = ops.bilinear_pool(x)
    n = y.norm(dim=1)
    assert torch.allclose(n, torch.ones_like(n), atol=2e-4)
    Y = y.view(32, 512, 512)
    assert (Y - Y.transpose(1, 2)).abs().max().item() < 1e-6
    assert (y > 0).all()
    # unsupported shapes are loud errors, not fallbacks
    from hawkeye_b200._lib import HawkeyeLibError
    with pytest.raises(HawkeyeLibError):
        ops.bilinear_pool(torch.rand(1, 100, 4, 4, device='cuda'))


def test_baseline_batch_elementwise_vs_oracle():
    """benchmark size (B=32, C=512, 14x14) and B=40, forward AND backward, element-wise against the fp64 oracle, per
    image."""
    from hawkeye_b200 import ops
    from oracle import hop_oracle as O
    for B in (32, 40):
        x = torch.relu(detgen.det_uniform((B, 512, 14, 14), 31) - 0.2)       # sparse, non-negative: what a ReLU + pool stack emits
        dy = detgen.det((B, 512 * 512), 32)
        xg = x.cuda().requires_grad_(True)
        y = ops.bilinear_pool(xg)
        (dx,) = torch.autograd.grad(y, xg, dy.cuda())
        y_ref = O.bilinear_pool_fwd(x.double())
        dx_ref = O.bilinear_pool_bwd(x.double(), dy.double())
        wf = max(rel_l2(y[b].detach().cpu(), y_ref[b]) for b in range(B))
        wb = max(rel_l2(dx[b].cpu(), dx_ref[b]) for b in range(B))
        print(f'bilinear B={B}: worst image fwd {wf:.2e} bwd {wb:.2e}')
        assert wf < 1e-3 and wb < 2e-3


@pytest.mark.parametrize('shape', [(3, 14, 14), (37, 14, 14), (2, 2, 2), (150, 4, 4), (2, 7, 7), (3, 3, 3)])
def test_bilinear_pool_shapes(shape):
    """hk_bilinear_pool_fwd (closed-form norm + Gram with the sqrt / L2-normalise epilogue) across batch sizes below and past
    one wave of GEMM tiles and tiny maps whose H*W is padded to a multiple of 4, per image against the fp64 oracle."""
    from hawkeye_b200 import ops
    from oracle import hop_oracle as O
    B, H, W = shape
    x = torch.relu(detgen.det_uniform((B, 512, H, W), 5) - 0.3)
    y = ops.bilinear_pool(x.cuda())
    ref = O.bilinear_pool_fwd(x.double())
    worst = max(rel_l2(y[b].cpu(), ref[b]) for b in range(B))
    assert worst < 1e-3, worst
