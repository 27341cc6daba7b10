"""Golden fixtures for AP-CNN from the UNMODIFIED reference (model/methods/APCNN.py, model/methods/nms.py).
Run here only:  HAWKEYE_REF=<Hawkeye checkout> python tests/golden/make_golden_apcnn.py -> tests/golden/reference_apcnn.<i>.npz
The models are built with the reference module's ``resnet50`` / ``ResNet`` — never its ``APCNN(config)`` factory, which
downloads weights.  ``random.random`` / ``random.randint`` are wrapped to record the drop-block draws of get_roi_crop_feat;
nothing else is patched.  Inputs and weights come from detgen seeds and tests/apcnn_inputs.py, so the tests rebuild them."""
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
import apcnn_inputs as I  # noqa: E402
import detgen  # noqa: E402

rh.load_reference()
R = sys.modules['model.methods.APCNN']       # `model.methods.APCNN` as an attribute is the factory function

torch.set_num_threads(8)
out = {}
DRAWS = []
_random, _randint = random.random, random.randint


def _rec_random():
    v = _random()
    DRAWS.append([v, -1.0])
    return v


def _rec_randint(a, b):
    v = _randint(a, b)
    DRAWS[-1][1] = float(v)
    return v


random.random, random.randint = _rec_random, _rec_randint

# ---- the state layout -------------------------------------------------------------------------------------------------
net = R.resnet50(200)
out['state_keys_json'] = np.frombuffer(json.dumps([[k, list(v.shape)] for k, v in net.state_dict().items()]).encode(),
                                       dtype=np.uint8)
out['params'] = np.int64(sum(p.numel() for p in net.parameters()))

# ---- get_att_roi on the seeded gates, both class switches; get_roi_crop_feat on the 200-class ROIs ----------------------
for nc in (200, 12):
    net.num_classes = nc
    g = I.gates(nc)
    rois = [net.get_att_roi(torch.from_numpy(g[l]).unsqueeze(1), 8 << l, 64 << l, I.ROI_IMAGE, I.ROI_IMAGE, iou_thred=0.05,
                            topk=(5, 3, 1)[l]) for l in range(3)]
    for l in range(3):
        b, c = I.pad_rois(rois[l].numpy(), I.ROI_BATCH, (5, 3, 1)[l])
        out[f'roi_{nc}_boxes_{l}'], out[f'roi_{nc}_counts_{l}'] = b, c
    print('roi', nc, [out[f'roi_{nc}_counts_{l}'].tolist() for l in range(3)])
    if nc == 200:
        x = detgen.det((I.ROI_BATCH, 8, 28, 28), 4100).requires_grad_(True)
        G = detgen.det((I.ROI_BATCH, 8, 28, 28), 4101)
        for mode in ('train', 'eval'):
            net.train(mode == 'train')
            random.seed(5)
            del DRAWS[:]
            y, _ = net.get_roi_crop_feat(x, rois, 8)
            x.grad = None
            (y * G).sum().backward()
            out[f'refine_{mode}_y'], out[f'refine_{mode}_dx'] = y.detach().numpy(), x.grad.numpy().copy()
            if mode == 'train':
                out['refine_draws'] = np.array(DRAWS, dtype=np.float64)
        print('refine draws', DRAWS)

# ---- PyramidAttentions forward and backward on seeded maps ---------------------------------------------------------------
apn = R.PyramidAttentions(256)
apn.load_state_dict(detgen.state_like(apn, seed=11))
Fs = [detgen.det((3, 256, s, s), 4200 + s).requires_grad_(True) for s in (12, 6, 3)]
A3, A4, A5, a3, a4, a5 = apn(Fs)
Gv = [detgen.det((3, 256), 4300 + i) for i in range(3)]
sum((A.mean((2, 3)) * g).sum() for A, g in zip((A3, A4, A5), Gv)).backward()
for i, (A, a, F) in enumerate(zip((A3, A4, A5), (a3, a4, a5), Fs)):
    out[f'att_pool_{i}'], out[f'att_gate_{i}'], out[f'att_dF_{i}'] = A.mean((2, 3)).detach().numpy(), a.detach().numpy(), F.grad.numpy()
out['att_dw_0'], out['att_db_0'] = apn.A3_1.conv.weight.grad.numpy(), apn.A3_1.conv.bias.grad.numpy()

# ---- end to end: a shallow trunk, 12 classes, 4 images of 160x160 (large enough that no single ROI covers the crop window), one train step ------------------------------------------
net = R.ResNet(I.E2E_CLASSES, R.Bottleneck, [1, 1, 1, 1])
net.load_state_dict(I.e2e_state(net))
net.train()
x = detgen.det((I.E2E_BATCH, 3, I.E2E_IMAGE, I.E2E_IMAGE), 4400)
labels = detgen.det_labels(I.E2E_BATCH, I.E2E_CLASSES, 4401)
random.seed(9)
del DRAWS[:]
out_mean, out_list, mask_cat, roi_list = net(x, labels)
crit = torch.nn.CrossEntropyLoss(label_smoothing=0.1)
loss = sum(crit(o, labels) for o in out_list)
loss.backward()
out['e2e_draws'] = np.array(DRAWS, dtype=np.float64)
out['e2e_out_mean'] = out_mean.detach().numpy()
out['e2e_out_list'] = torch.stack(out_list).detach().numpy()
out['e2e_mask_cat'] = mask_cat.detach().numpy()
for l in range(3):
    out[f'e2e_boxes_{l}'], out[f'e2e_counts_{l}'] = I.pad_rois(roi_list[l].numpy(), I.E2E_BATCH, (5, 3, 1)[l])
out['e2e_loss'] = np.float64(loss.item())
names = ['conv1.weight', 'layer2.0.conv2.weight', 'layer3.0.conv1.weight', 'layer4.0.conv3.weight', 'fpn.P5_1.conv_master.conv.weight',
         'fpn.P5_1.conv_gpb.bn.weight', 'fpn.P4_1.weight', 'fpn.P4_1.bias', 'fpn.P3_2.weight', 'fpn.P3_2.bias', 'fpn.P5_2.weight',
         'apn.A3_1.conv.weight', 'apn.A3_1.conv.bias', 'apn.A5_1.conv.weight', 'apn.A4_2.conv1.weight', 'apn.A3_2.conv2.bias',
         'cls3.3.weight', 'cls5.2.weight', 'cls4.6.bias', 'cls_concate.2.weight', 'cls_concate.3.bias']
params = dict(net.named_parameters())
out['e2e_grad_names'] = np.frombuffer(json.dumps(names).encode(), dtype=np.uint8)
for i, k in enumerate(names):
    gr = params[k].grad.flatten()
    sel = torch.from_numpy(np.random.RandomState(4410 + i).choice(gr.numel(), min(gr.numel(), 256), replace=False))
    out[f'e2e_grad_{i}_idx'], out[f'e2e_grad_{i}'] = sel.numpy(), gr[sel].numpy()
sd = net.state_dict()
for k in ('layer2.0.bn1', 'layer3.0.bn1', 'fpn.P5_1.conv_master.bn', 'cls3.2', 'cls_concate.3'):
    out[f'e2e_rm_{k}'], out[f'e2e_rv_{k}'] = sd[k + '.running_mean'].numpy(), sd[k + '.running_var'].numpy()
    out[f'e2e_nbt_{k}'] = sd[k + '.num_batches_tracked'].numpy()
print('gate ranges', [(float(mask_cat[:, l].min()), float(mask_cat[:, l].max())) for l in range(3)])
print('e2e loss', loss.item(), 'draws', DRAWS, 'counts', [out[f'e2e_counts_{l}'].tolist() for l in range(3)])

save_golden('reference_apcnn', out)
print('wrote', len(out), 'arrays')
