"""Golden fixtures for Interp-Parts from the UNMODIFIED reference (model/methods/Interp_Parts.py, model/loss/InterpParts_loss.py).
Run here only:  HAWKEYE_REF=<Hawkeye checkout> python tests/golden/make_golden_interp_parts.py
    -> tests/golden/reference_interp_parts.<i>.npz
The model is built as ``ResNet(Bottleneck, ...)`` directly (IP_ResNet* would download torchvision's weights), and
``Tensor.cuda`` is the identity while this runs: the loss moves its prior and its Gaussian to ``.cuda(device)`` even when
the device is the CPU.  Inputs come from detgen seeds, so the tests rebuild them instead of reading them from here."""
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
torch.Tensor.cuda = lambda self, *a, **k: self
import model.loss.InterpParts_loss as L  # noqa: E402
from model.methods.Interp_Parts import Bottleneck, GroupingUnit, ResNet  # noqa: E402

torch.set_num_threads(8)
out = {}

# ---- the 101-layer state layout (IP_ResNet101 without the download) -------------------------------------------------
net = ResNet(Bottleneck, [3, 4, 23, 3], 200, 5)
out['state_keys_json'] = np.frombuffer(json.dumps([[k, list(v.shape)] for k, v in net.state_dict().items()]).encode(),
                                       dtype=np.uint8)
out['params_101'] = np.int64(sum(p.numel() for p in net.parameters()))

# ---- the Beta prior at several (N, alpha, beta) ------------------------------------------------------------------------
for i, (n, a, b) in enumerate([(16, 1, 0.001), (4, 1, 0.001), (7, 2.0, 3.0), (64, 1, 0.001), (1, 0.5, 0.5)]):
    L.update_prior_dist(n, a, b)
    out[f'prior_{i}'] = L.prior_dist.numpy().reshape(-1)
    out[f'prior_{i}_args'] = np.array([n, a, b], dtype=np.float64)


# ---- the grouping unit and the shaping loss alone at [4, 1024, 28, 28], 5 parts: x = 0.03 det(seed), centres
# 0.03 det(seed + 1), smooth 0.3 det(seed + 2), G = det(seed + 3) on the [N, C, K] outputs ---------------------------------
def unit_inputs(seed, N=4, C=1024, H=28, W=28, K=5):
    return (0.03 * detgen.det((N, C, H, W), seed), 0.03 * detgen.det((K, C, 1, 1), seed + 1), 0.3 * detgen.det((K,), seed + 2),
            detgen.det((N, C, K), seed + 3))


x, w, sf, G = unit_inputs(1500)
g = GroupingUnit(1024, 5)
with torch.no_grad():
    g.weight.copy_(w)
    g.smooth_factor.copy_(sf)
x.requires_grad_(True)
feats, assign = g(x)
shaping = L.ShapingLoss(assign, 2, 0.4, 5, 1, 0.001)
loss = (feats * G).sum() + 0.5 * shaping
loss.backward()
out['unit_seed'] = np.int64(1500)
out['unit_feats'] = feats.detach().numpy()
out['unit_assign'] = assign.detach().numpy()
out['unit_shaping'] = np.float64(shaping.item())
out['unit_dx_slice'] = x.grad[:, ::16].numpy()
out['unit_dweight'] = g.weight.grad.numpy()
out['unit_dsmooth'] = g.smooth_factor.grad.numpy()
print('unit', shaping.item())

# ---- the whole model end to end on a shallow trunk: [1, 1, 1] blocks, 5 parts, 4 images of 128x128, detgen.state_like
# weights, train mode, InterpPartsLoss and its backward ----------------------------------------------------------------
net = ResNet(Bottleneck, [1, 1, 1], 200, 5)
net.load_state_dict(detgen.state_like(net))
net.train()
x = detgen.det((4, 3, 128, 128), 1510)
labels = detgen.det_labels(4, 200, 1511)
logits, att, assign = net(x)
crit = L.InterpPartsLoss(rh.cfg(radius=2, std=0.4, num_parts=5, alpha=1, beta=0.001, coeff=0.5))
loss = crit((logits, att, assign), labels)
loss.backward()
out['e2e_logits'], out['e2e_att'], out['e2e_assign'] = logits.detach().numpy(), att.detach().numpy(), assign.detach().numpy()
out['e2e_loss'] = np.float64(loss.item())
names = ['grouping.weight', 'grouping.smooth_factor', 'attconv.2.weight', 'attconv.2.bias', 'attconv.3.weight',
         'groupingbn.weight', 'mylinear.bias', 'post_block.0.conv1.weight', 'layer3.0.conv2.weight', 'conv1.weight']
params = dict(net.named_parameters())
out['e2e_grad_names'] = np.frombuffer(json.dumps(names).encode(), dtype=np.uint8)
for i, k in enumerate(names):
    gr = params[k].grad.flatten()
    idx = torch.from_numpy(np.random.RandomState(1520 + i).choice(gr.numel(), min(gr.numel(), 256), replace=False))
    out[f'e2e_grad_{i}_idx'], out[f'e2e_grad_{i}'] = idx.numpy(), gr[idx].numpy()
out['e2e_running_var_att'] = net.attconv[3].running_var.numpy()
print('e2e', loss.item())

save_golden('reference_interp_parts', out)
print('wrote', len(out), 'arrays')
