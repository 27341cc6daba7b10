"""Golden fixtures for MGE-CNN from the UNMODIFIED reference (model/methods/MGE_CNN/MGE.py, grad_cam.py).
Run here only:  HAWKEYE_REF=<Hawkeye checkout> python tests/golden/make_golden_mge.py -> tests/golden/reference_mge.<i>.npz
The models are built through the reference's LocalCamNet with the backbone download neutralised by oracle.ref_harness;
for the shallow models ``resnet50`` in the MGE module's namespace is swapped for the reference's own
``ResNet(Bottleneck, [1, 1, 1, 3])``.  ``get_bbox`` is wrapped to record the boxes forward computes; nothing else is
patched.  Inputs and weights come from detgen seeds and tests/mge_inputs.py, so the tests rebuild them."""
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
import mge_inputs as I  # noqa: E402

rh.load_reference()
R = sys.modules['model.methods.MGE_CNN.MGE']
GC = sys.modules['model.methods.MGE_CNN.grad_cam']
RB = sys.modules['model.backbone.resnet']

torch.set_num_threads(8)
out = {}

# ---- the full model's state layout --------------------------------------------------------------------------------------
net = R.LocalCamNet(rh.cfg(num_classes=200, box_thred=0.2, image_size=224))
out['state_keys_json'] = np.frombuffer(json.dumps([[k, list(v.shape)] for k, v in net.state_dict().items()]).encode(),
                                       dtype=np.uint8)
out['params'] = np.int64(sum(p.numel() for p in net.parameters()))
del net

# ---- get_bbox on seeded maps ----------------------------------------------------------------------------------------------
for name in I.BBOX_CASES:
    conv5, lw, rate, size = I.bbox_case(name)
    x = torch.zeros(conv5.shape[0], 3, size, size)
    _, xy = R.get_bbox(x, torch.from_numpy(conv5), torch.from_numpy(lw), rate=rate, img_size=size)
    out[f'bbox_{name}'] = np.array([[int(v) for v in r] for r in xy], dtype=np.int64)
    print('bbox', name, out[f'bbox_{name}'].tolist())

# ---- shallow models: GradCam and one train step ---------------------------------------------------------------------------
R.resnet50 = lambda pretrained=True: RB.ResNet(RB.Bottleneck, list(I.E2E_LAYERS))
net = R.LocalCamNet(rh.cfg(num_classes=I.E2E_CLASSES, box_thred=I.E2E_THRED, image_size=I.E2E_IMAGE))
net.load_state_dict(detgen.state_like(net))
c4 = torch.from_numpy(I.gradcam_input())
for tag, target in (('argmax', None), ('target', torch.tensor([3, 7]))):
    cam = GC.GradCam(model=net, feature_extractor=net.conv5_box, classifier=net.classifier, target_layer_names=['2'])
    weights = cam(c4.clone(), target)
    with torch.no_grad():
        net.eval()
        logits = net.classifier(net.pool(net.conv5_box(c4)).flatten(1))
        net.train()
    out[f'gradcam_{tag}_weights'] = weights.numpy()
    out[f'gradcam_{tag}_idx'] = (logits.argmax(1) if target is None else target).numpy()
net.zero_grad()

BOXES = []
_get_bbox = R.get_bbox


def _rec_get_bbox(*a, **k):
    input_box, xy = _get_bbox(*a, **k)
    BOXES.append([[int(v) for v in r] for r in xy])
    return input_box, xy


R.get_bbox = _rec_get_bbox
net.train()
x = detgen.det((I.E2E_BATCH, 3, I.E2E_IMAGE, I.E2E_IMAGE), 5300)
labels = detgen.det_labels(I.E2E_BATCH, I.E2E_CLASSES, 5301)
outputs = net(x)
net.zero_grad()                                   # Examples/MGE_CNN.py:48: optimizer.zero_grad() after the forward
crit = torch.nn.CrossEntropyLoss(label_smoothing=0.1)
losses = [crit(l, labels) for l in outputs['logits']]
loss = sum(losses) / len(losses)
loss.backward()
out['e2e_logits'] = torch.stack(outputs['logits']).detach().numpy()
out['e2e_pr_gate'] = outputs['pr_gate'].detach().numpy()
out['e2e_box_xy'] = np.array(BOXES, dtype=np.int64)
out['e2e_loss'] = np.float64(loss.item())
names = ['conv4.0.weight', 'conv4.6.0.conv2.weight', 'conv5.2.conv3.weight', 'conv5.0.bn1.weight', 'classifier.fc.weight',
         'classifier.fc.bias', 'conv4_box.5.0.conv1.weight', 'conv5_box.1.bn2.weight', 'classifier_box.fc.weight',
         'conv4_box_2.0.weight', 'conv5_box_2.0.conv1.weight', 'classifier_box_2.fc.bias', 'conv6.weight', 'conv6.bias',
         'conv6_1.weight', 'conv6_2.bias', 'cls_part.fc.weight', 'cls_part_1.fc.bias', 'cls_cat.fc.weight', 'cls_cat_2.fc.bias',
         'conv4_gate.0.weight', 'conv5_gate.2.conv3.weight', 'cls_gate.0.fc.weight', 'cls_gate.1.fc.weight',
         'cls_gate.1.fc.bias']
params = dict(net.named_parameters())
out['e2e_grad_names'] = np.frombuffer(json.dumps(names).encode(), dtype=np.uint8)
for i, k in enumerate(names):
    gr = params[k].grad.flatten()
    sel = torch.from_numpy(np.random.RandomState(5310 + i).choice(gr.numel(), min(gr.numel(), 256), replace=False))
    out[f'e2e_grad_{i}_idx'], out[f'e2e_grad_{i}'] = sel.numpy(), gr[sel].numpy()
out['e2e_no_grad_json'] = np.frombuffer(json.dumps(sorted(k for k, p in params.items() if p.grad is None)).encode(),
                                        dtype=np.uint8)
sd = net.state_dict()
BN = ('conv4.1', 'conv5.2.bn3', 'conv4_box.6.0.bn1', 'conv5_box_2.0.bn2', 'conv4_gate.1', 'conv5_gate.2.bn3')
out['e2e_bn_json'] = np.frombuffer(json.dumps(BN).encode(), dtype=np.uint8)
for k in BN:
    out[f'e2e_rm_{k}'], out[f'e2e_rv_{k}'] = sd[k + '.running_mean'].numpy(), sd[k + '.running_var'].numpy()
    out[f'e2e_nbt_{k}'] = sd[k + '.num_batches_tracked'].numpy()
print('e2e loss', loss.item(), 'boxes', BOXES, 'no grad', json.loads(bytes(out['e2e_no_grad_json']).decode()))

save_golden('reference_mge', out)
print('wrote', len(out), 'arrays')
