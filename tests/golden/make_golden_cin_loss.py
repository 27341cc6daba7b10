"""Golden fixtures for CIN's training head from the UNMODIFIED reference (model/loss/CIN_loss.py, model/methods/CIN.py).
Run here only:  python tests/golden/make_golden_cin_loss.py  -> tests/golden/reference_cin_loss.<i>.npz
At the shape the shipped config trains (tests/cin_inputs.py): CINLoss on three label orders, and ChannelInteractionModule
in train mode at batch 20, C = 2048, 7x7.  Weights and inputs come from detgen, so the fixture carries slices and sums of
the outputs and gradients only."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tests'))
from conftest import save_golden  # noqa: E402
from oracle import ref_harness as rh  # noqa: E402
import cin_inputs as I  # noqa: E402
import detgen  # noqa: E402

rh.load_reference()
from model.loss.CIN_loss import CINLoss  # noqa: E402
from model.methods.CIN import ChannelInteractionModule  # noqa: E402

torch.set_num_threads(8)
out = {}
crit = CINLoss(rh.cfg(alpha=I.ALPHA, beta=0.5, channel=I.C, feature_size=I.WH, r_channel=I.R))
crit.load_state_dict(I.h_state())
for name in I.LABELS:
    z = I.logits().requires_grad_(True)
    zc = I.z_cci().requires_grad_(True)
    target = I.labels(name)
    crit.zero_grad()
    loss = crit((z, zc), target)
    loss.backward()
    out[f'{name}_loss'] = np.float64(loss.item())
    out[f'{name}_ce'] = np.float64(torch.nn.functional.cross_entropy(z.detach(), target, label_smoothing=0.1).item())
    out[f'{name}_dz'] = z.grad.numpy()
    out[f'{name}_dzc_slice'] = zc.grad.numpy()[:, ::64, ::7]
    out[f'{name}_dzc_sums'] = zc.grad.double().sum((1, 2)).numpy()
    gw = crit.h.weight.grad
    out[f'{name}_dw_slice'] = gw.numpy()[::16, ::389]
    out[f'{name}_dw_rowsums'] = gw.double().sum(1).numpy()
    out[f'{name}_db'] = crit.h.bias.grad.numpy()
    print(name, float(loss), 'pairs', int((target[:10] == target[10]).sum()))

# the module in train mode at the shape the shipped config trains
m = ChannelInteractionModule(in_channel=I.C, spatial_size=(7, 7))
m.load_state_dict(detgen.state_like(m))
m.train()
x = detgen.det((I.B, I.C, 7, 7), 6010, positive=True).requires_grad_(True)
z, zc = m(x)
r1, r2 = detgen.det(z.shape, 6011), detgen.det(zc.shape, 6012)
((z * r1).sum() + (zc * r2).sum()).backward()
out['module_z_slice'] = z.detach().numpy()[:, ::16, ::5]
out['module_zcci_slice'] = zc.detach().numpy()[:, ::16, ::5]
out['module_z_sums'] = z.detach().double().sum((1, 2)).numpy()
out['module_zcci_sums'] = zc.detach().double().sum((1, 2)).numpy()
out['module_dx_slice'] = x.grad.numpy()[:, ::16]
out['module_dx_sums'] = x.grad.double().sum((1, 2, 3)).numpy()
out['module_g_conv.weight_slice'] = m.conv.weight.grad.numpy()[::16, ::16]
out['module_g_conv.bias'] = m.conv.bias.grad.numpy()
out['module_g_fc.weight_slice'] = m.fc.weight.grad.numpy()[:, ::97]
out['module_g_fc.bias'] = m.fc.bias.grad.numpy()
save_golden('reference_cin_loss', out)                 # parts of under 1 MB: tests/golden/reference_cin_loss.<i>.npz
print('wrote', len(out), 'arrays')
