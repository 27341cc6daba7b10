"""Golden fixtures for CrossX from the UNMODIFIED reference (model/methods/CrossX.py, model/loss/CrossX_loss.py,
Examples/CrossX.py).
Run here only:  HAWKEYE_REF=<Hawkeye checkout> python tests/golden/make_golden_crossx.py -> tests/golden/reference_crossx.<i>.npz
* CrossXLoss (gamma 0.5, 0.25, 0.5) at P in {2, 3}, N in {2, 8}, K = 200 on tests/crossx_inputs.py: the loss and the
  gradients of its six inputs (the feature lists as [N, C, 1, 1] tensors, copies: the reference overwrites them).
* CrossX(num_parts=2) with detgen weights at batch 4, 448x448: one train-mode step, then one eval-mode step, each the three
  logits, the loss and slices of the fc, me, conv3_1 and conv1 gradients, and the bn3_1 running statistics, in float32 and,
  through the same reference code, in float64.  Every BatchNorm has momentum 1, so the eval step normalises with the
  train step's batch statistics: on the initial ones (mean 0, variance 1) the random-weight activations grow block after
  block, softmax(xf) underflows to 0 and the reference's KL gradient through its target is NaN.  Every value is finite.
* The P = 1 and P = 3 models' logits (eval mode, float64) on the same image.
* The state_dict layout (keys and shapes) at P = 1, 2 and 3.
* Examples/CrossX.py's training and validation transforms on a seeded image under a fixed torch seed."""
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
import crossx_inputs as I  # noqa: E402
import detgen  # noqa: E402

rh.load_reference()
from model.loss.CrossX_loss import CrossXLoss  # noqa: E402
from model.methods.CrossX import ResNet, Bottleneck  # noqa: E402

torch.set_num_threads(16)
out = {}


for P, N in I.LOSS_CASES:
    xf, xp, xc, fu, fp, fc, y = I.loss_inputs(P, N)
    leaves = [t.clone().double().requires_grad_(True) for t in (xf, xp, xc, fu, fp, fc)]
    crit = CrossXLoss(rh.cfg(num_parts=P, gamma=list(I.GAMMA)))
    outs = tuple(leaves[:3]) + tuple([f[:, i, :, None, None] for i in range(P)] for f in leaves[3:])
    loss = crit(outs, y)
    loss.backward()
    out[f'loss_{P}_{N}'] = np.float64(loss.item())
    for name, t in zip(('xf', 'xp', 'xc', 'fu', 'fp', 'fc'), leaves):
        out[f'd{name}_{P}_{N}'] = t.grad.float().numpy()
    print('loss', P, N, loss.item())


def model(P):
    return ResNet(Bottleneck, [3, 4, 6, 3], nparts=P, meflag=P > 1, num_classes=I.K)


x, y = I.net_image(), I.net_labels()
crit = CrossXLoss(rh.cfg(num_parts=I.NET_P, gamma=list(I.GAMMA)))
for prefix, dtype in (('net', torch.float32), ('net64', torch.float64)):
    net = model(I.NET_P)
    net.load_state_dict(detgen.state_like(net, seed=81))
    net = net.to(dtype)
    for m in net.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.momentum = I.NET_BN_MOMENTUM
    for mode in ('train', 'eval'):
        net.train(mode == 'train')
        net.zero_grad()
        xf, xp, xc, ul, pl, cm = net(x.to(dtype))
        logits = [t.detach().clone() for t in (xf, xp, xc)]
        loss = crit((xf, xp, xc, ul, pl, cm), y)
        loss.backward()
        for n_, t in zip(('xf', 'xp', 'xc'), logits):
            out[f'{prefix}_{mode}_{n_}'] = t.numpy()
        out[f'{prefix}_{mode}_loss'] = np.float64(loss.item())
        for n_ in ('fc_ulti', 'fc_plty', 'fc_cmbn'):
            out[f'{prefix}_{mode}_{n_}_w_slice'] = getattr(net, n_).weight.grad.numpy()[:, ::32]
            out[f'{prefix}_{mode}_{n_}_b'] = getattr(net, n_).bias.grad.numpy()
        for blk in ('layer3', 'layer4'):
            me = getattr(net, blk)[-1].me.parts
            for i in range(I.NET_P):
                out[f'{prefix}_{mode}_{blk}_me{i}_0_w'] = me[i][0].weight.grad.numpy()[:, ::8]
                out[f'{prefix}_{mode}_{blk}_me{i}_2_b'] = me[i][2].bias.grad.numpy()
        out[f'{prefix}_{mode}_conv3_1_w_slice'] = net.conv3_1.weight.grad.numpy()[::16, ::16]
        out[f'{prefix}_{mode}_conv2_1_w_slice'] = net.conv2_1.weight.grad.numpy()[::16, ::16]
        out[f'{prefix}_{mode}_conv1_w'] = net.conv1.weight.grad.numpy()
        print(prefix, mode, 'loss', loss.item())
    bad = [k for k, v in out.items() if k.startswith(prefix + '_') and not np.isfinite(v).all()]
    assert not bad, bad
    out[f'{prefix}_bn3_1_running_mean'] = net.bn3_1.running_mean.numpy()
    out[f'{prefix}_bn3_1_running_var'] = net.bn3_1.running_var.numpy()

for P in (1, 3):
    net = model(P)
    net.load_state_dict(detgen.state_like(net, seed=81))
    net = net.double().eval()
    with torch.no_grad():
        o = net(x.double())
    if P == 1:
        out['p1_logits'] = o.float().numpy()
    else:
        for n_, t in zip(('xf', 'xp', 'xc'), o[:3]):
            out[f'p3_{n_}'] = t.float().numpy()
    print('P', P, 'done')

layout = {str(P): [[k, list(v.shape)] for k, v in model(P).state_dict().items()] for P in (1, 2, 3)}
out['layout'] = np.frombuffer(json.dumps(layout).encode(), dtype=np.uint8)

sys.path.insert(0, rh.find_reference_root())
from Examples.CrossX import CrossXTrainer  # noqa: E402
from PIL import Image  # noqa: E402

tf = CrossXTrainer.get_transformers(None, None)
img = Image.fromarray((detgen.det_uniform((500, 700, 3), 8200).numpy() * 255).astype(np.uint8))
for split in ('train', 'val'):
    torch.manual_seed(8201)
    t = tf[split](img)
    out[f'tf_{split}_shape'] = np.array(t.shape)
    out[f'tf_{split}_slice'] = t.numpy()[:, ::16, ::16]
    out[f'tf_{split}_sums'] = t.double().sum((1, 2)).numpy()
save_golden('reference_crossx', out)
print('wrote', len(out), 'arrays')
