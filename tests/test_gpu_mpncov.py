"""Fast MPN-COV pooling head (Covpool / Sqrtm / Triuvec, fwd + bwd) vs the oracle and reference fixtures."""
import pytest
import torch

import detgen
from conftest import rel_l2

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('tag,shape,it', [('mpn_it3', (2, 24, 4, 4), 3), ('mpn_c256', (1, 256, 14, 14), 5)])
def test_mpncov_golden(golden, tag, shape, it):
    from hawkeye_b200 import ops
    x = detgen.det_uniform(shape, 31).cuda().requires_grad_(True)
    c = ops.CovpoolLayer(x)
    s = ops.SqrtmLayer(c, it)
    v = ops.TriuvecLayer(s)
    dv = detgen.det(v.shape, 32).cuda()
    (dx,) = torch.autograd.grad(v, x, dv)
    ec, es = rel_l2(c.detach().cpu(), golden[f'{tag}_cov']), rel_l2(s.detach().cpu(), golden[f'{tag}_sqrt'])
    ed = rel_l2(dx.cpu(), golden[f'{tag}_dx'])
    print(f'{tag}: cov {ec:.2e} sqrt {es:.2e} dx {ed:.2e}')
    assert v.shape == (shape[0], shape[1] * (shape[1] + 1) // 2, 1)
    assert ec < 1e-3 and es < 1e-3 and ed < 3e-3


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
