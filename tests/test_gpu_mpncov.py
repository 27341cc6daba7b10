"""Fast MPN-COV pooling head (Covpool / Sqrtm / Triuvec, fwd + bwd) vs the oracle and reference fixtures, in both
precision modes."""
import math

import pytest
import torch

import detgen
from conftest import rel_l2
from kernel_check import precise  # noqa: F401  (a fixture)

pytestmark = pytest.mark.gpu

PATTERN = 0x7FA5A5A5   # guard words around the outputs (a NaN payload)
GUARD = 64


def _guarded(n):
    """device buffer of n floats between GUARD guard words on each side; returns (buffer, the n-float view)"""
    buf = torch.full((n + 2 * GUARD,), PATTERN, dtype=torch.int32).view(torch.float32).cuda()
    return buf, buf[GUARD:GUARD + n]


def _guards_intact(buf):
    bits = buf.cpu().view(torch.int32)
    return bool((bits[:GUARD] == PATTERN).all() and (bits[-GUARD:] == PATTERN).all())


def _per_image(label, out, ref, tol):
    """relative L2 and max-norm error of every batch entry on its own (a wrong per-image index cannot average out)"""
    for b in range(ref.shape[0]):
        e = rel_l2(out[b], ref[b])
        m = ((out[b].double() - ref[b]).abs().max() / ref[b].abs().max()).item()
        print(f'{label} [{b}]: rel {e:.2e} max {m:.2e} (tol {tol:.0e})')
        assert e < tol and m < 4 * tol, (label, b)


# cov, sqrt, dx tolerances (relative L2 to the fp32 reference's fixtures).  Measured on an H100 80GB HBM3 (700 W), worst
# over the three fixtures: 2.3e-4, 2.2e-4, 6.4e-4 single pass; 3.6e-6, 5.3e-6, 2.7e-6 in precise mode.
GOLDEN_TOL = {0: (1e-3, 1e-3, 3e-3), 1: (2e-5, 2e-5, 2e-5)}


@pytest.mark.parametrize('tag,shape,it', [('mpn_small', (2, 16, 3, 3), 5), ('mpn_it3', (2, 24, 4, 4), 3),
                                          ('mpn_c256', (1, 256, 14, 14), 5)])
def test_mpncov_golden(golden, tag, shape, it, precise):
    from hawkeye_b200 import ops
    x = detgen.det_uniform(shape, 31).cuda().requires_grad_(True)
    c = ops.CovpoolLayer(x)
    s = ops.SqrtmLayer(c, it)
    v = ops.TriuvecLayer(s)
    dv = detgen.det(v.shape, 32).cuda()
    (dx,) = torch.autograd.grad(v, x, dv)
    ec, es = rel_l2(c.detach().cpu(), golden[f'{tag}_cov']), rel_l2(s.detach().cpu(), golden[f'{tag}_sqrt'])
    ed = rel_l2(dx.cpu(), golden[f'{tag}_dx'])
    print(f'{tag} precise={precise}: cov {ec:.2e} sqrt {es:.2e} dx {ed:.2e}')
    assert v.shape == (shape[0], shape[1] * (shape[1] + 1) // 2, 1)
    tc, ts, td = GOLDEN_TOL[precise]
    assert ec < tc and es < ts and ed < td


# measured (H100 80GB HBM3, 700 W), worst relative L2 over every image: 5.5e-4 single pass (xc and g reach the MMA as
# tf32), 9.1e-7 in precise mode
COVPOOL_TOL = {0: 1.5e-3, 1: 5e-6}


@pytest.mark.parametrize('C', [16, 256])
@pytest.mark.parametrize('M', [9, 49, 196])
def test_covpool_vs_oracle_fp64(M, C, precise):
    """Covpool forward and backward at H*W = 3x3, 7x7 (the map of a 224x224 input) and 14x14.  For H*W % 4 != 0 the
    centred rows are kept at a 16-byte pitch (zero padding) and the backward writes dx at pitch H*W: nothing past
    [B, C, H*W] may change."""
    from hawkeye_b200 import _lib
    from oracle import hop_oracle as O
    B, H = 3, int(math.isqrt(M))
    Mp = (M + 3) // 4 * 4
    x = detgen.det_uniform((B, C, H, H), 40 + M + C)
    g = detgen.det((B, C, C), 41 + M + C)
    cov_buf, cov = _guarded(B * C * C)
    xc_buf, xc = _guarded(B * C * Mp)
    dx_buf, dx = _guarded(B * C * M)
    _lib.call('hk_covpool_fwd', x.cuda(), cov, xc, B, C, M, _lib.stream_ptr())
    _lib.call('hk_covpool_bwd', xc, g.cuda(), dx, B, C, M, _lib.stream_ptr())
    torch.cuda.synchronize()
    assert _guards_intact(cov_buf) and _guards_intact(xc_buf) and _guards_intact(dx_buf)
    assert (xc.cpu().view(B, C, Mp)[..., M:] == 0).all()          # the pitch padding adds nothing to the products
    tol = COVPOOL_TOL[precise]
    _per_image(f'covpool fwd M={M} C={C} precise={precise}', cov.cpu().view(B, C, C), O.covpool_fwd(x.double()), tol)
    _per_image(f'covpool bwd M={M} C={C} precise={precise}', dx.cpu().view(B, C, H, H),
               O.covpool_bwd(x.double(), g.double()), tol)


# fwd, bwd: the chain always runs in 3xTF32, whatever the precision mode.  Measured (H100 80GB HBM3, 700 W), worst
# relative L2 over every image: 4.4e-6 forward, 3.3e-6 backward
SQRTM_TOL = (3e-5, 3e-5)


@pytest.mark.parametrize('iterN', [2, 3, 5])
@pytest.mark.parametrize('n', [24, 100, 256])
def test_sqrtm_vs_oracle_fp64_per_image(n, iterN, precise):
    """Sqrtm forward and backward on one batch of three SPD matrices whose traces are 1e-3, 1 and 1e3: each image is
    normalised by its own trace.  n = 100 gives partial 64-wide tiles (scalar (hi, lo) stores); iterN = 2 leaves both
    Newton-Schulz loops empty."""
    from hawkeye_b200 import ops
    from oracle import hop_oracle as O
    B = 3
    f = detgen.det_uniform((B, n, 2 * n), 50 + n).double()
    f = f - f.mean(2, keepdim=True)
    cov = f @ f.transpose(1, 2) / (2 * n)
    traces = torch.tensor([1e-3, 1.0, 1e3], dtype=torch.float64)
    x = (cov * (traces / cov.diagonal(dim1=1, dim2=2).sum(1)).view(B, 1, 1)).float()
    g = detgen.det((B, n, n), 51 + n)
    xg = x.cuda().requires_grad_(True)
    y = ops.SqrtmLayer(xg, iterN)
    (gx,) = torch.autograd.grad(y, xg, g.cuda())
    y_ref, saved = O.sqrtm_fwd(x.double(), iterN)
    gx_ref = O.sqrtm_bwd(x.double(), saved, g.double(), iterN)
    _per_image(f'sqrtm fwd n={n} iterN={iterN} precise={precise}', y.detach().cpu(), y_ref, SQRTM_TOL[0])
    _per_image(f'sqrtm bwd n={n} iterN={iterN} precise={precise}', gx.cpu(), gx_ref, SQRTM_TOL[1])


@pytest.mark.parametrize('n', [1, 24, 129, 256])
def test_triuvec_vs_oracle(n, precise):
    """Triuvec forward is a gather and backward a scatter: both exact, and the strict lower triangle of dx is zero."""
    from hawkeye_b200 import _lib, ops
    from oracle import hop_oracle as O
    B, L = 2, n * (n + 1) // 2
    x = detgen.det((B, n, n), 60 + n)
    g = detgen.det((B, L, 1), 61 + n)
    v = ops.TriuvecLayer(x.cuda())
    dx = torch.full((B, n, n), float('nan'), device='cuda')
    _lib.call('hk_triuvec_bwd', g.cuda(), dx, B, n, _lib.stream_ptr())
    torch.cuda.synchronize()
    assert torch.equal(v.cpu(), O.triuvec_fwd(x))
    dx = dx.cpu()
    assert torch.equal(dx, O.triuvec_bwd(g, n))
    assert (torch.tril(dx, -1).view(torch.int32) == 0).all()


def test_sqrtm_chain_vs_oracle_fp64():
    """Sqrtm alone on an SPD batch at benchmark size (B=4, 256x256, iterN=5): 3xTF32 keeps the 12-GEMM chain at
    fp32-class accuracy; backward follows the reference formulae (incl. the transpose and diagonal term)."""
    from hawkeye_b200 import ops
    from oracle import hop_oracle as O
    B, n = 4, 256
    f = detgen.det_uniform((B, n, 196), 7).double()
    f = f - f.mean(2, keepdim=True)
    cov = (f @ f.transpose(1, 2) / 196).float()
    g = detgen.det((B, n, n), 8)
    cg = cov.cuda().requires_grad_(True)
    y = ops.SqrtmLayer(cg, 5)
    (gx,) = torch.autograd.grad(y, cg, g.cuda())
    y_ref, saved = O.sqrtm_fwd(cov.double(), 5)
    gx_ref = O.sqrtm_bwd(cov.double(), saved, g.double(), 5)
    ef, eb = rel_l2(y.detach().cpu(), y_ref), rel_l2(gx.cpu(), gx_ref)
    print(f'sqrtm fwd {ef:.2e} bwd {eb:.2e}')
    assert ef < 1e-4 and eb < 1e-3
    # triuvec round trip
    v = ops.TriuvecLayer(y.detach())
    back = ops.TriuvecFn.apply(y.detach().requires_grad_(True))
    assert torch.equal(v.cpu().squeeze(-1), O.triuvec_fwd(y.detach().cpu()).squeeze(-1))
