"""Golden fixtures for Pairwise Confusion and the plain ResNet-50 classifier from the UNMODIFIED reference
(model/loss/pair_confusion.py, model/backbone/resnet.py ``ResNet50``, Examples/Baseline.py).
Run here only:  HAWKEYE_REF=<Hawkeye checkout> python tests/golden/make_golden_pc.py -> tests/golden/reference_pc.<i>.npz
* PairwiseConfusionLoss at batch 24, 200 classes, on the four label patterns of tests/pc_inputs.py and lambda_a 0.1 and 10:
  the loss and the logit gradient.
* ResNet50(num_classes=200) with detgen weights at batch 4, 224x224: one train-mode step, then one eval-mode step, each
  the logits, the PairwiseConfusionLoss (lambda_a 10) and slices or sums of the fc and conv1 gradients, in float32 and,
  through the same reference code, in float64.
* Examples/Baseline.py's training and validation transforms on a seeded image under a fixed torch seed."""
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
import pc_inputs as I  # noqa: E402

rh.load_reference()
from model.loss.pair_confusion import PairwiseConfusionLoss  # noqa: E402
from model.backbone.resnet import ResNet50  # noqa: E402

torch.set_num_threads(8)
out = {}
for lam in I.LAMBDAS:
    crit = PairwiseConfusionLoss(rh.cfg(lambda_a=lam))
    for name in I.NAMES:
        z = I.logits(name).requires_grad_(True)
        loss = crit(z, I.labels(name))
        loss.backward()
        out[f'loss_{name}_{lam}'] = np.float64(loss.item())
        out[f'dz_{name}_{lam}'] = z.grad.numpy()
        print('loss', name, lam, loss.item(), 'nan in dz:', bool(torch.isnan(z.grad).any()))

# ---- ResNet50, one train-mode then one eval-mode step --------------------------------------------------------------------
# The same steps in float64 (the reference's own code, net.double()) under the prefix net64_: a random-weight train-mode
# ResNet-50 loses most of its conv1 gradient to cancellation, so the fp32 run is itself far from exact there.
crit = PairwiseConfusionLoss(rh.cfg(lambda_a=I.NET_LAMBDA))
x, y = I.net_image(), I.net_labels()
for prefix, dtype in (('net', torch.float32), ('net64', torch.float64)):
    net = ResNet50(rh.cfg(num_classes=I.NET_K))
    net.load_state_dict(detgen.state_like(net, seed=71))
    net = net.to(dtype)
    for mode in ('train', 'eval'):
        net.train(mode == 'train')
        net.zero_grad()
        logits = net(x.to(dtype))
        loss = crit(logits, y)
        loss.backward()
        out[f'{prefix}_{mode}_logits'] = logits.detach().numpy()
        out[f'{prefix}_{mode}_loss'] = np.float64(loss.item())
        gw = net.fc.weight.grad
        out[f'{prefix}_{mode}_fc_w_slice'] = gw.numpy()[:, ::16]
        out[f'{prefix}_{mode}_fc_w_rowsums'] = gw.double().sum(1).numpy()
        out[f'{prefix}_{mode}_fc_b'] = net.fc.bias.grad.numpy()
        out[f'{prefix}_{mode}_conv1_w'] = net.conv1.weight.grad.numpy()
        print(prefix, mode, 'loss', loss.item())
    out[f'{prefix}_bn1_running_mean'] = net.bn1.running_mean.numpy()
    out[f'{prefix}_bn1_running_var'] = net.bn1.running_var.numpy()

# ---- Examples/Baseline.py's transforms -------------------------------------------------------------------------------------
sys.path.insert(0, rh.find_reference_root())
from Examples.Baseline import BaselineTrainer  # noqa: E402
from PIL import Image  # noqa: E402

tf = BaselineTrainer.get_transformers(None, None)
img = Image.fromarray((detgen.det_uniform((300, 260, 3), 7200).numpy() * 255).astype(np.uint8))
for split in ('train', 'val'):
    torch.manual_seed(7201)
    t = tf[split](img)
    out[f'tf_{split}_shape'] = np.array(t.shape)
    out[f'tf_{split}_slice'] = t.numpy()[:, ::8, ::8]
    out[f'tf_{split}_sums'] = t.double().sum((1, 2)).numpy()
save_golden('reference_pc', out)
print('wrote', len(out), 'arrays')
