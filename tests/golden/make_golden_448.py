"""Golden fixtures at the benchmark configuration (448x448, batch 2, 200 classes; the benchmark configurations) from the
UNMODIFIED reference: BCNN stage 1/2, CBCNN d=8192 and d=6000, MPN.  Needs the reference tree ($HAWKEYE_REF or baseline/_ref):
    python tests/golden/make_golden_448.py   -> tests/golden/reference_448.npz
    HK_GOLDEN_SIZE=224 python tests/golden/make_golden_448.py   -> tests/golden/reference_224.npz
Inputs and weights are regenerated from tests/detgen.py seeds by the tests; the fixture carries outputs only:
logits, loss, classifier gradients (bias, strided weight slice) and a few backbone gradients (whole small tensors, strided
slices of large ones).

For every gradient g the fixture also stores u_<name> = rel-L2 distance between the reference's fp32 gradient and an EXACT
(fp64, oracle/hop_oracle.py) evaluation of the same network on the same inputs.  It is not zero: the reference's own fp32
rounding flips ReLU / max-pool decisions (conv1_1's weight gradient is only reproducible to ~4e-3), so u is the floor any
faithful implementation can be held to; the GPU tests require  err <= 1e-3 + 3 u."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tests'))
from oracle import ref_harness as rh  # noqa: E402
from oracle.hop_oracle import VGG16_D  # noqa: E402
from oracle import hop_oracle as O  # noqa: E402
import detgen  # noqa: E402

rh.load_reference()
from model.registry import MODEL  # noqa: E402

torch.set_num_threads(8)
out = {}
SIZE, B = int(os.environ.get('HK_GOLDEN_SIZE', '448')), 2      # 224: the 7x7 (H*W = 49, not a multiple of 4) maps of the
#                                                                  reference's stock MPN / CBCNN / PeerLearning configs


def rel_l2(a, b):
    a, b = torch.as_tensor(a).double().flatten(), torch.as_tensor(b).double().flatten()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def uncertainties(tag, forward, x, labels, state, train_keys=None):
    """u_<key> for every stored gradient of `tag` (see the module docstring)."""
    st = {k: (v.double() if v.is_floating_point() else v) for k, v in state.items()}
    _, _, g = O.loss_and_grads(forward, x.double(), labels, st, train_keys)
    for key in [k for k in out if k.startswith(tag + '_g_')]:
        name = key[len(tag) + 3:]
        pname = name[:-len('_slice')] if name.endswith('_slice') else name
        full = g[pname]
        ref = torch.as_tensor(out[key])
        if name.endswith('_slice'):          # re-apply the slicing rule by matching shapes
            for sl in ((slice(None), slice(None, None, 4099)), (slice(None), slice(None, None, 61)),
                       (slice(None, None, 8), slice(None, None, 8)), (slice(None, None, 4), slice(None, None, 4)),
                       (slice(None), slice(None, None, 8), 0, 0), (slice(None, None, 4), slice(None, None, 4), 0, 0)):
                try:
                    cand = full[sl]
                except IndexError:
                    continue
                if tuple(cand.shape) == tuple(ref.shape):
                    full = cand
                    break
        out[f'{tag}_u_{name}'] = np.float32(rel_l2(full, ref))


def step(net, x, labels):
    net.train()
    logits = net(x)
    loss = torch.nn.CrossEntropyLoss(label_smoothing=0.1)(logits, labels)      # train.py:211-212
    net.zero_grad()
    loss.backward()
    return logits.detach().numpy(), np.float32(loss.item())


x = detgen.det((B, 3, SIZE, SIZE), 41)
labels = detgen.det_labels(B, 200, 42)
for stage in (1, 2):
    net = MODEL.get('BCNN')(rh.cfg(name='BCNN', stage=stage, num_classes=200))
    net.load_state_dict(detgen.vgg_bcnn_state(VGG16_D, 200, seed=100))
    t = f'bcnn_s{stage}'
    out[t + '_logits'], out[t + '_loss'] = step(net, x, labels)
    out[t + '_g_classifier.bias'] = net.classifier.bias.grad.numpy()
    out[t + '_g_classifier.weight_slice'] = net.classifier.weight.grad.numpy()[:, ::4099]
    if stage == 2:
        for k, p in net.named_parameters():
            if k.startswith('backbone') and k.endswith('bias'):
                out[f'{t}_g_{k}'] = p.grad.numpy()
        out[t + '_g_backbone.0.weight'] = net.backbone[0].weight.grad.numpy()
        out[t + '_g_backbone.10.weight_slice'] = net.backbone[10].weight.grad.numpy()[::8, ::8]
        out[t + '_g_backbone.28.weight_slice'] = net.backbone[28].weight.grad.numpy()[::8, ::8]
    st = detgen.vgg_bcnn_state(VGG16_D, 200, seed=100)
    uncertainties(t, lambda xx, s_, stage=stage: O.bcnn_forward(xx, s_, stage), x, labels, st,
                  None if stage == 2 else {'classifier.weight', 'classifier.bias'})
    print(t, float(out[t + '_loss']), {k: float(v) for k, v in out.items() if k.startswith(t + '_u_')}, flush=True)

for d in (8192, 6000):
    net = MODEL.get('CBCNN')(rh.cfg(name='CBCNN', stage=2, num_classes=200, input_channel=512, output_channel=d))
    net.load_state_dict(detgen.vgg_bcnn_state(VGG16_D, 200, seed=100, head_in=d))
    t = f'cbcnn_{d}'
    out[t + '_logits'], out[t + '_loss'] = step(net, x, labels)
    out[t + '_g_classifier.bias'] = net.classifier.bias.grad.numpy()
    out[t + '_g_classifier.weight_slice'] = net.classifier.weight.grad.numpy()[:, ::61]
    for k in ('backbone.0.bias', 'backbone.14.bias', 'backbone.28.bias'):
        out[f'{t}_g_{k}'] = dict(net.named_parameters())[k].grad.numpy()
    uncertainties(t, lambda xx, s_, d=d: O.cbcnn_forward(xx, s_, d, 2), x, labels,
                  detgen.vgg_bcnn_state(VGG16_D, 200, seed=100, head_in=d))
    print(t, float(out[t + '_loss']), {k: float(v) for k, v in out.items() if k.startswith(t + '_u_')}, flush=True)

net = MODEL.get('MPN')(rh.cfg(name='MPN', iter_num=5, is_sqrt=True, is_vec=True, input_dim=2048,
                              dimension_reduction=256, num_classes=200))
net.load_state_dict(detgen.state_like(net))
xm, lm = detgen.det((B, 3, SIZE, SIZE), 51), detgen.det_labels(B, 200, 52)
out['mpn_logits'], out['mpn_loss'] = step(net, xm, lm)
named = dict(net.named_parameters())
for k in ('classifier.bias', 'pool.conv_dr_block.1.weight', 'backbone.7.2.bn3.weight', 'backbone.4.0.bn1.bias', 'backbone.1.weight'):
    out[f'mpn_g_{k}'] = named[k].grad.numpy()
out['mpn_g_backbone.0.weight'] = named['backbone.0.weight'].grad.numpy()
out['mpn_g_pool.conv_dr_block.0.weight_slice'] = named['pool.conv_dr_block.0.weight'].grad.numpy()[:, ::8, 0, 0]
out['mpn_g_backbone.5.0.conv2.weight_slice'] = named['backbone.5.0.conv2.weight'].grad.numpy()[::4, ::4]
out['mpn_g_backbone.5.0.downsample.0.weight_slice'] = named['backbone.5.0.downsample.0.weight'].grad.numpy()[::4, ::4, 0, 0]
uncertainties('mpn', lambda xx, s_: O.mpn_forward(xx, s_, 5), xm, lm, detgen.state_like(net), set(named.keys()))
print('mpn', float(out['mpn_loss']), {k: float(v) for k, v in out.items() if k.startswith('mpn_u_')}, flush=True)

np.savez_compressed(os.path.join(HERE, f'reference_{SIZE}.npz'), **out)
print('wrote', len(out), 'arrays;', os.path.getsize(os.path.join(HERE, f'reference_{SIZE}.npz')) / 1e6, 'MB')
