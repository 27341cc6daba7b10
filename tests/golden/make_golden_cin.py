"""Golden fixtures for the channel-interaction row from the UNMODIFIED reference (model/methods/CIN.py).
Run here only:  python tests/golden/make_golden_cin.py  -> tests/golden/reference_cin.<i>.npz
Weights come from detgen.state_like(module) and inputs from detgen seeds, so the fixture carries outputs only."""
import json
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
import detgen  # noqa: E402

rh.load_reference()
from model.methods.CIN import ChannelInteractionModule, CINClassifier  # noqa: E402
from model.registry import MODEL  # noqa: E402

torch.set_num_threads(8)
out = {}
for tag, C, size, B in (('c256_8x8', 256, (8, 8), 4), ('c128_7x7', 128, (7, 7), 2)):
    m = ChannelInteractionModule(in_channel=C, spatial_size=size)
    m.load_state_dict(detgen.state_like(m))
    m.train()
    x = detgen.det((B, C, size[0], size[1]), 91, positive=True).requires_grad_(True)
    z, zc = m(x)
    r1, r2 = detgen.det(z.shape, 92), detgen.det(zc.shape, 93)
    loss = (z * r1).sum() + (zc * r2).sum()
    m.zero_grad()
    loss.backward()
    out[f'{tag}_z'], out[f'{tag}_zcci'] = z.detach().numpy(), zc.detach().numpy()
    out[f'{tag}_dx'] = x.grad.numpy()
    out[f'{tag}_g_conv.weight_slice'] = m.conv.weight.grad.numpy()[::4, ::4]
    out[f'{tag}_g_conv.bias'] = m.conv.bias.grad.numpy()
    out[f'{tag}_g_fc.weight_slice'] = m.fc.weight.grad.numpy()[:, ::37]
    out[f'{tag}_g_fc.bias'] = m.fc.bias.grad.numpy()
    m.eval()
    out[f'{tag}_z_eval'] = m(x.detach()).detach().numpy()
    print(tag, float(loss))

# full-size forward (C = 2048, 14x14: a 448x448 input), eval mode, and the classifier on top
m = ChannelInteractionModule(in_channel=2048, spatial_size=(14, 14))
m.load_state_dict(detgen.state_like(m))
m.eval()
cls = CINClassifier(2048, 200)
cls.load_state_dict(detgen.state_like(cls))
x = detgen.det((2, 2048, 14, 14), 94, positive=True)
with torch.no_grad():
    z = m(x)
    logits = cls(z)
out['full_z_slice'] = z.numpy()[:, ::64, ::7]
out['full_z_sum'] = np.float64(z.double().sum().item())
out['full_logits'] = logits.numpy()
net = MODEL.get('CIN')(rh.cfg(name='CIN', num_classes=200))
out['cin_state_keys_json'] = np.frombuffer(json.dumps({k: list(v.shape) for k, v in net.state_dict().items()}, sort_keys=True).encode(), dtype=np.uint8)
save_golden('reference_cin', out)                 # parts of under 1 MB: tests/golden/reference_cin.<i>.npz
print('wrote', len(out), 'arrays')

# ---- OSME: the excitation module on its own + the OSMENet key list -----------
from model.methods.OSME import OSME  # noqa: E402

for tag, C, shape, B in (('osme_c256_7', 256, 7, 4), ('osme_c128_14', 128, (14, 14), 2)):
    m = OSME(C, 64, feature_shape=shape, num_attention=2)
    m.load_state_dict(detgen.state_like(m))
    hw = shape if isinstance(shape, tuple) else (shape, shape)
    x = detgen.det((B, C, hw[0], hw[1]), 95, positive=True).requires_grad_(True)
    f, parts = m(x)
    r1, r2 = detgen.det(f.shape, 96), detgen.det(parts.shape, 97)
    ((f * r1).sum() + (parts * r2).sum()).backward()
    out[f'{tag}_f'], out[f'{tag}_parts'], out[f'{tag}_dx'] = f.detach().numpy(), parts.detach().numpy(), x.grad.numpy()
    for k, p in m.named_parameters():
        g = p.grad.numpy()
        out[f'{tag}_g_{k}'] = g if g.size <= 65536 else g.reshape(g.shape[0], -1)[:, ::29]
net = MODEL.get('OSMENet')(rh.cfg(name='OSMENet', num_attention=2, num_classes=200))
out['osme_state_keys_json'] = np.frombuffer(json.dumps({k: list(v.shape) for k, v in net.state_dict().items()}, sort_keys=True).encode(), dtype=np.uint8)
save_golden('reference_cin', out)                 # parts of under 1 MB: tests/golden/reference_cin.<i>.npz
print('wrote', len(out), 'arrays (with OSME)')

# ---- MAMC / N-pairs loss: the criterion of OSMENet ---------------------------
from model.loss.MAMC_loss import MAMCLoss, NPairsLoss  # noqa: E402

for tag, b, p, D, ncls in (('npair_b8_p2', 8, 2, 64, 3), ('npair_b12_p3', 12, 3, 32, 4), ('npair_b6_p2_allsame', 6, 2, 16, 1),
                           ('npair_b4_p2_alldiff', 4, 2, 16, 4)):
    f = detgen.det((b, p, D), 201).requires_grad_(True)
    lab = torch.arange(b) % ncls                       # balanced classes, several samples per class (BalancedBatchSampler)
    loss = NPairsLoss()(f, lab)
    loss.backward()
    out[f'{tag}_feats'], out[f'{tag}_labels'] = f.detach().numpy(), lab.numpy()
    out[f'{tag}_loss'], out[f'{tag}_dfeats'] = np.float64(loss.item()), f.grad.numpy()
crit = MAMCLoss(rh.cfg(lambda_a=0.5, use_mamc=True))
pred = detgen.det((8, 200), 202).requires_grad_(True)
parts = detgen.det((8, 2, 64), 203).requires_grad_(True)
lab = torch.arange(8) % 3
loss = crit((pred, parts), lab)
loss.backward()
out['mamc_pred'], out['mamc_parts'], out['mamc_labels'] = pred.detach().numpy(), parts.detach().numpy(), lab.numpy()
out['mamc_loss'], out['mamc_dpred'], out['mamc_dparts'] = np.float64(loss.item()), pred.grad.numpy(), parts.grad.numpy()
save_golden('reference_cin', out)                 # parts of under 1 MB: tests/golden/reference_cin.<i>.npz
print('wrote', len(out), 'arrays (with OSME + MAMC)')
