"""ChannelInteractionModule / CINClassifier against fixtures from the UNMODIFIED reference
(tests/golden/make_golden_cin.py): outputs in train and eval mode, input and parameter gradients, the 7x7 (WH = 49, padded
to 52 columns) case, and the full-size C = 2048, 14x14 forward."""
import os

import numpy as np
import pytest
import torch

import detgen
from conftest import load_golden, rel_l2

pytestmark = pytest.mark.gpu
G = load_golden('reference_cin')


@pytest.mark.parametrize('precise', [0, 1])
@pytest.mark.parametrize('tag,C,size,B', [('c256_8x8', 256, (8, 8), 4), ('c128_7x7', 128, (7, 7), 2)])
def test_channel_interaction_module(tag, C, size, B, precise):
    from hawkeye_b200 import _lib
    from hawkeye_b200.methods.cin import ChannelInteractionModule
    m = ChannelInteractionModule(in_channel=C, spatial_size=size)
    m.load_state_dict(detgen.state_like(m))
    m = m.cuda().train()
    x = detgen.det((B, C, size[0], size[1]), 91, positive=True).cuda().requires_grad_(True)
    _lib.set_precise(precise)
    try:
        z, zc = m(x)
        r1, r2 = detgen.det(z.shape, 92).cuda(), detgen.det(zc.shape, 93).cuda()
        ((z * r1).sum() + (zc * r2).sum()).backward()
        m.eval()
        with torch.no_grad():
            ze = m(x.detach())
    finally:
        _lib.set_precise(0)
    errs = {'z': rel_l2(z.detach().cpu(), G[f'{tag}_z']), 'zcci': rel_l2(zc.detach().cpu(), G[f'{tag}_zcci']),
            'z_eval': rel_l2(ze.cpu(), G[f'{tag}_z_eval']), 'dx': rel_l2(x.grad.cpu(), G[f'{tag}_dx']),
            'conv.weight': rel_l2(m.conv.weight.grad.cpu()[::4, ::4], G[f'{tag}_g_conv.weight_slice']),
            'conv.bias': rel_l2(m.conv.bias.grad.cpu(), G[f'{tag}_g_conv.bias']),
            'fc.weight': rel_l2(m.fc.weight.grad.cpu()[:, ::37], G[f'{tag}_g_fc.weight_slice']),
            'fc.bias': rel_l2(m.fc.bias.grad.cpu(), G[f'{tag}_g_fc.bias'])}
    print(tag, f'precise={precise}', {k: f'{v:.1e}' for k, v in errs.items()})
    # TF32: three chained single-pass products (W.X, conv, fc-weighted W_CCI.X) + the conv's tf32 store; precise: 3xTF32
    tol_f, tol_b = (3e-3, 5e-3) if not precise else (1e-4, 2e-4)
    assert max(errs['z'], errs['zcci'], errs['z_eval']) < tol_f
    assert max(errs[k] for k in ('dx', 'conv.weight', 'conv.bias', 'fc.weight', 'fc.bias')) < tol_b


@pytest.mark.parametrize('precise', [0, 1])
def test_cin_full_size_forward(precise):
    from hawkeye_b200 import _lib
    from hawkeye_b200.methods.cin import ChannelInteractionModule, CINClassifier
    m = ChannelInteractionModule(in_channel=2048, spatial_size=(14, 14))
    m.load_state_dict(detgen.state_like(m))
    cls = CINClassifier(2048, 200)
    cls.load_state_dict(detgen.state_like(cls))
    m, cls = m.cuda().eval(), cls.cuda().eval()
    x = detgen.det((2, 2048, 14, 14), 94, positive=True).cuda()
    _lib.set_precise(precise)
    try:
        with torch.no_grad():
            z = m(x)
            logits = cls(z)
    finally:
        _lib.set_precise(0)
    z4 = z.view(2, 2048, 196)
    ez, el = rel_l2(z4.cpu()[:, ::64, ::7], G['full_z_slice']), rel_l2(logits.cpu(), G['full_logits'])
    print(f'cin full size precise={precise}: z {ez:.2e} logits {el:.2e}')
    tol = 3e-3 if not precise else 1e-4
    assert ez < tol and el < tol
    assert abs(z.double().sum().item() - float(G['full_z_sum'])) / abs(float(G['full_z_sum'])) < 1e-3


@pytest.mark.parametrize('precise', [0, 1])
@pytest.mark.parametrize('tag,C,shape,B', [('osme_c256_7', 256, 7, 4), ('osme_c128_14', 128, (14, 14), 2)])
def test_osme_module(tag, C, shape, B, precise):
    """OSME against the reference: summed / per-attention features, input and all parameter grads."""
    from hawkeye_b200 import _lib
    from hawkeye_b200.methods.osme import OSME
    m = OSME(C, 64, feature_shape=shape, num_attention=2)
    m.load_state_dict(detgen.state_like(m))
    m = m.cuda().train()
    hw = shape if isinstance(shape, tuple) else (shape, shape)
    x = detgen.det((B, C, hw[0], hw[1]), 95, positive=True).cuda().requires_grad_(True)
    _lib.set_precise(precise)
    try:
        f, parts = m(x)
        ((f * detgen.det(f.shape, 96).cuda()).sum() + (parts * detgen.det(parts.shape, 97).cuda()).sum()).backward()
    finally:
        _lib.set_precise(0)
    errs = {'f': rel_l2(f.detach().cpu(), G[f'{tag}_f']), 'parts': rel_l2(parts.detach().cpu(), G[f'{tag}_parts']),
            'dx': rel_l2(x.grad.cpu(), G[f'{tag}_dx'])}
    for k, p in m.named_parameters():
        g = p.grad.cpu()
        g = g if g.numel() <= 65536 else g.reshape(g.shape[0], -1)[:, ::29]
        errs[k] = rel_l2(g, G[f'{tag}_g_{k}'])
    worst = max(errs, key=errs.get)
    print(tag, f'precise={precise}', {k: f'{v:.1e}' for k, v in errs.items() if k in ('f', 'parts', 'dx', worst)})
    assert errs[worst] < (3e-3 if not precise else 1e-4)
