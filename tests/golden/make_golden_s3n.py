"""Golden fixtures for S3N from the UNMODIFIED reference (model/methods/S3N.py, model/loss/S3N_loss.py).
Run here only:  HAWKEYE_REF=<Hawkeye checkout> python tests/golden/make_golden_s3n.py  -> tests/golden/reference_s3n.<p>.npz
Shims, none of which changes what the reference computes on the CPU:
- ``resnet50(pretrained=True)`` builds the reference's randomly initialised ResNet-50 (oracle/ref_harness, no download);
- ``random.uniform`` in the S3N module is wrapped to record each draw (p = 1), with the peak it was drawn for;
- ``peak_stimulation``, ``create_grid`` and ``F.grid_sample`` are wrapped to record their inputs and outputs.
Two 128x128 images, 200 classes, detgen.state_like weights except radius, radius_inv and filter, which keep their
initial values (radius 0.12, radius_inv 0.3, base_ratio 0.09 as in
configs/S3N.yaml), train mode; one fixture per p in {0, 1, 2}, all from the same weights and images.  The p = 2 fixture
also holds the eval-mode outputs of the checkpoint as loaded."""
import json
import os
import random
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
import model.methods  # noqa: E402,F401
from model.loss.S3N_loss import MultiSmoothLoss  # noqa: E402

S = sys.modules['model.methods.S3N']     # the package re-exports the class under the module's name
torch.set_num_threads(8)
N, SIZE, K = 2, 128, 200
CFG = dict(num_classes=K, image_size=SIZE, radius=0.12, radius_inv=0.3, base_ratio=0.09)
GRAD_NAMES = ['radius.scale', 'radius_inv.scale', 'filter.weight', 'raw_classifier.weight', 'sampler_classifier.bias',
              'sampler_classifier1.weight', 'con_classifier.weight', 'sampler_buffer.0.weight', 'sampler_buffer1.1.weight',
              'backbone.layer4.2.conv3.weight', 'backbone.conv1.weight', 'backbone.bn1.weight']

seen = {}
_peak, _grid, _gs, _uniform = S.peak_stimulation, S.S3N.create_grid, S.F.grid_sample, random.uniform


def rec_peak(dm, **kw):
    out = _peak(dm, **kw)
    seen.setdefault('peaks', []).append(out[0][:, 2:].numpy() if len(out[0]) else np.zeros((0, 2), np.int64))
    seen.setdefault('dm', []).append(dm.detach().reshape(-1).numpy().copy())
    return out


def rec_grid(self, x):
    g = _grid(self, x)
    seen.setdefault('maps', []).append(x[:, 0, 30:-30, 30:-30].detach().numpy().copy())
    seen.setdefault('grids', []).append(g.detach().numpy().copy())
    return g


def rec_gs(x, grid, **kw):
    out = _gs(x, grid, **kw)
    seen.setdefault('sampled', []).append(out.detach().numpy().copy())
    return out


def rec_uniform(a, b):
    u = _uniform(a, b)
    seen.setdefault('draws', []).append(u)
    return u


S.peak_stimulation, S.S3N.create_grid, S.F.grid_sample = rec_peak, rec_grid, rec_gs
S.random.uniform = rec_uniform

net = S.S3N(rh.cfg(**CFG))
state = detgen.state_like(net)
for k in ('radius.scale', 'radius_inv.scale', 'filter.weight'):       # the sampler's own initial values, not noise
    state[k] = net.state_dict()[k].clone()
keys = list(net.state_dict().keys())
x = detgen.det((N, 3, SIZE, SIZE), 5100)
labels = detgen.det_labels(N, K, 5101)
for p in (0, 1, 2):
    net.load_state_dict(state)
    evals = {}
    if p == 2:                                  # eval mode on the checkpoint itself (running statistics as loaded)
        net.eval()
        with torch.no_grad():
            for name, o in zip(('aggregation', 'agg_origin', 'agg_sampler', 'agg_sampler1'), net(x, 2)):
                evals['eval_' + name] = o.numpy()
    net.train()
    net.zero_grad()
    seen.clear()
    random.seed(5102 + p)
    crm_seen = {}
    h = net.map_origin.register_forward_hook(lambda m, i, o: crm_seen.__setitem__('crm', o.detach().clone()))
    outputs = net(x, p)
    h.remove()
    loss = MultiSmoothLoss(rh.cfg(smooth_ratio=0.85))(outputs, labels)
    loss.backward()
    out = {'state_keys_json': np.frombuffer(json.dumps(keys).encode(), dtype=np.uint8),
           'crm': crm_seen['crm'].numpy(), 'labels': labels.numpy(), 'loss': np.float64(loss.item())}
    for name, o in zip(('aggregation', 'agg_origin', 'agg_sampler', 'agg_sampler1'), outputs):
        out[name] = o.detach().numpy()
    out.update(evals)
    out['xs'], out['xs_inv'] = seen['maps'][0].reshape(N, -1), seen['maps'][1].reshape(N, -1)
    out['grid_zoom'] = seen['grids'][0][:, ::4, ::4].copy()      # every 4th row and column of the 128x128 grids
    out['grid_inv'] = seen['grids'][1][:, ::4, ::4].copy()
    sampled = np.concatenate(seen['sampled'])                      # [2N, 3, 128, 128]: zoom, then complementary
    pix = np.random.RandomState(5103).choice(sampled.size, 8192, replace=False)
    out['sampled_idx'], out['sampled'] = pix, sampled.reshape(-1)[pix]
    out['dm'] = np.stack(seen['dm'])
    for n in range(N):
        out[f'peaks_{n}'] = seen['peaks'][n].astype(np.int64)
    if p == 1:                                  # draws in order: image by image, peak by peak
        img, pos = [], []
        for n in range(N):
            for (r, c) in seen['peaks'][n]:
                img.append(n)
                pos.append(r * 31 + c)
        assert len(img) == len(seen['draws'])
        out['draw_image'], out['draw_pos'] = np.array(img, np.int64), np.array(pos, np.int64)
        out['draw_value'] = np.array(seen['draws'], np.float64)
    params = dict(net.named_parameters())
    for i, k in enumerate(GRAD_NAMES):
        g = params[k].grad                      # None: no peak went to that map (p = 1, 2)
        gr = (torch.zeros_like(params[k]) if g is None else g).flatten()
        sel = torch.from_numpy(np.random.RandomState(5110 + i).choice(gr.numel(), min(gr.numel(), 256), replace=False))
        out[f'grad_{i}_idx'], out[f'grad_{i}'] = sel.numpy(), gr[sel].numpy()
    out['grad_names'] = np.frombuffer(json.dumps(GRAD_NAMES).encode(), dtype=np.uint8)
    print('p', p, 'loss', loss.item(), 'peaks', [len(seen['peaks'][n]) for n in range(N)],
          'dradius', out['grad_0'], out['grad_1'])
    save_golden(f'reference_s3n.{p}', out)
