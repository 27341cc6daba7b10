"""Golden fixtures for DCL from the UNMODIFIED reference (model/methods/DCL.py, model/loss/DCL_loss.py,
dataset/transforms.py RandomSwap, dataset/dataset_DCL.py).
Run here only:  HAWKEYE_REF=<Hawkeye checkout> python tests/golden/make_golden_dcl.py  -> tests/golden/reference_dcl.<i>.npz
The reference's RandomSwap calls Image.ANTIALIAS, which Pillow 10 removed; this script alone aliases it to Image.LANCZOS
(the same filter) so that the reference can run.  Weights and trunk maps come from detgen seeds, so the fixture carries
outputs only."""
import json
import os
import random
import sys
import tempfile

import numpy as np
import torch
import torch.nn as nn
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tests'))
from conftest import save_golden  # noqa: E402
from oracle import ref_harness as rh  # noqa: E402
import detgen  # noqa: E402

rh.load_reference()
Image.ANTIALIAS = Image.LANCZOS
from model.loss.DCL_loss import DCLLoss  # noqa: E402
from model.registry import MODEL  # noqa: E402
from dataset.transforms import RandomSwap  # noqa: E402
from dataset.dataset_DCL import DCLDataset, collate_fn4train, collate_fn4val  # noqa: E402
from torchvision.transforms import transforms  # noqa: E402

torch.set_num_threads(8)
out = {}
net = MODEL.get('DCL')(rh.cfg(name='DCL', num_classes=200, cls_2=True, cls_2xmul=False))
out['state_keys_json'] = np.frombuffer(json.dumps({k: list(v.shape) for k, v in net.state_dict().items()},
                                                  sort_keys=True).encode(), dtype=np.uint8)
mul = MODEL.get('DCL')(rh.cfg(name='DCL', num_classes=200, cls_2=False, cls_2xmul=True))
out['params_cls2'] = np.int64(sum(p.numel() for p in net.parameters()))
out['params_cls2xmul'] = np.int64(sum(p.numel() for p in mul.parameters()))

# ---- the whole model end to end: detgen.state_like weights (same keys => same values in the package's DCL), train mode,
# 4 rows of 128x128 (a 4x4 trunk map, so a 4-entry mask and a 2x2 swap law), DCLLoss and its backward ----------------------
e2e = MODEL.get('DCL')(rh.cfg(name='DCL', num_classes=200, cls_2=True, cls_2xmul=False))
e2e.load_state_dict(detgen.state_like(e2e))
e2e.train()
feats = []
e2e.backbone.register_forward_hook(lambda m, i, o: feats.append(o.detach()))
x = detgen.det((4, 3, 128, 128), 560)
labels = detgen.det_labels(2, 200, 561).repeat_interleave(2)
labels_swap = torch.tensor([1, 0, 1, 0])
law = torch.tensor([[-0.5, -0.25, 0.0, 0.25], [0.25, 0.0, -0.25, -0.5]] * 2)
logits, swap_logits, mask = e2e(x)
loss = DCLLoss(rh.cfg(alpha=1.0, beta=1.0, gamma=1.0))([logits, swap_logits, mask], labels, labels_swap, law)
loss.backward()
out['e2e_feat_slice'] = feats[0][:, ::16].numpy()
out['e2e_logits'], out['e2e_swap'], out['e2e_mask'] = (t.detach().numpy() for t in (logits, swap_logits, mask))
out['e2e_labels'], out['e2e_labels_swap'], out['e2e_law'] = labels.numpy(), labels_swap.numpy(), law.numpy()
out['e2e_loss'] = np.float64(loss.item())
out['e2e_g_convmask_w'] = e2e.Convmask.weight.grad.numpy()
out['e2e_g_convmask_b'] = e2e.Convmask.bias.grad.numpy()
out['e2e_g_classifier_swap'] = e2e.classifier_swap.weight.grad.numpy()
out['e2e_g_layer4_bn3_w'] = e2e.backbone[7][2].bn3.weight.grad.numpy()
print('e2e', loss.item())
del e2e

# ---- the head with the trunk replaced by nn.Identity: input = a [4, 2048, S, S] map -------------------------------------
net.backbone = nn.Identity()
net.load_state_dict(detgen.state_like(net))
for S, seed in ((14, 501), (7, 511)):
    x = detgen.det((4, 2048, S, S), seed, positive=True).requires_grad_(True)
    logits, swap_logits, mask = net(x)
    r = [detgen.det(t.shape, seed + 1 + i) for i, t in enumerate((logits, swap_logits, mask))]
    net.zero_grad()
    ((logits * r[0]).sum() + (swap_logits * r[1]).sum() + (mask * r[2]).sum()).backward()
    out[f'head{S}_logits'], out[f'head{S}_swap'], out[f'head{S}_mask'] = (t.detach().numpy() for t in (logits, swap_logits, mask))
    out[f'head{S}_dx'] = x.grad.numpy()[:, ::16]                              # every 16th channel keeps the part small
    out[f'head{S}_dconvmask_w'], out[f'head{S}_dconvmask_b'] = net.Convmask.weight.grad.numpy(), net.Convmask.bias.grad.numpy()
    out[f'head{S}_dclassifier'] = net.classifier.weight.grad.numpy()[:, ::8]
    out[f'head{S}_dclassifier_swap'] = net.classifier_swap.weight.grad.numpy()
    print('head', S, float(logits.sum()), float(mask.sum()))


# ---- DCLLoss on seeded outputs, cls_2 and cls_2xmul ------------------------------------------------------------------
def loss_case(tag, K2, seed):
    n, K = 4, 200
    R = 2 * n
    crit = DCLLoss(rh.cfg(alpha=0.75, beta=1.25, gamma=2.0))
    logits = detgen.det((R, K), seed, 3.0).requires_grad_(True)
    swap = detgen.det((R, K2), seed + 1, 3.0).requires_grad_(True)
    mask = torch.tanh(detgen.det((R, 49), seed + 2)).requires_grad_(True)
    labels = torch.from_numpy(np.random.RandomState(seed + 3).randint(0, K, size=n)).long().repeat_interleave(2)
    if K2 == 2:
        labels_swap = torch.tensor([1, 0] * n)
    else:
        labels_swap = torch.stack([labels[::2], labels[::2] + K], 1).reshape(-1)
    law = torch.from_numpy(np.random.RandomState(seed + 4).randint(0, 49, size=(R, 49)) - 24).float() / 49
    with torch.no_grad():
        mask[0, :5] = law[0, :5]                                          # exact ties: the L1 gradient is 0 there
    loss = crit([logits, swap, mask], labels, labels_swap, law)
    loss.backward()
    for k, v in dict(logits=logits, swap=swap, mask=mask).items():
        out[f'loss_{tag}_{k}'], out[f'loss_{tag}_d{k}'] = v.detach().numpy(), v.grad.numpy()
    out[f'loss_{tag}_labels'], out[f'loss_{tag}_labels_swap'], out[f'loss_{tag}_law'] = labels.numpy(), labels_swap.numpy(), \
        law.numpy()
    out[f'loss_{tag}_value'] = np.float64(loss.item())
    print('loss', tag, loss.item())


loss_case('cls2', 2, 520)
loss_case('cls2xmul', 400, 530)
out['loss_weights'] = np.array([0.75, 1.25, 2.0])


# ---- RandomSwap on small synthetic images under a seeded `random` ------------------------------------------------------
def synthetic(w, h, seed):
    rs = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    base = np.stack([xx * 255 // max(w - 1, 1), yy * 255 // max(h - 1, 1), (xx + yy) * 127 // max(w + h - 2, 1)], -1)
    return Image.fromarray(np.clip(base + rs.randint(-30, 31, size=(h, w, 3)), 0, 255).astype(np.uint8))


for tag, (w, h, size, seed) in dict(sq=(90, 80, (7, 7), 540), rect=(61, 47, (3, 2), 541)).items():
    img = synthetic(w, h, seed)
    random.seed(seed)
    out[f'swap_{tag}_in'] = np.asarray(img)
    out[f'swap_{tag}_out'] = np.asarray(RandomSwap(size)(img))
    out[f'swap_{tag}_size'] = np.array(size)
    out[f'swap_{tag}_seed'] = np.int64(seed)

# ---- DCLDataset items and the collate functions, from PNGs in a temporary directory --------------------------------------
DATA_SEED = 550
tf = {'swap': transforms.Compose([RandomSwap((7, 7))]), 'common_aug': transforms.Compose([transforms.Resize((56, 56))]),
      'train_totensor': transforms.Compose([transforms.Resize((56, 56)), transforms.ToTensor()]),
      'val_totensor': transforms.Compose([transforms.Resize((56, 56)), transforms.ToTensor()]), 'None': None}


def u8(t):
    return (t * 255).round().clamp(0, 255).to(torch.uint8).numpy()


with tempfile.TemporaryDirectory() as root:
    lines = []
    for i in range(22):                                                  # 10 images of class 0, 12 of class 1
        label = 0 if i < 10 else 1
        name = f'c{label}/img{i:02d}.png'
        os.makedirs(os.path.join(root, f'c{label}'), exist_ok=True)
        synthetic(70 + i, 60 + (i % 5), DATA_SEED + i).save(os.path.join(root, name))
        lines.append(f'{label} {name}')
    meta = os.path.join(root, 'meta.txt')
    open(meta, 'w').write('\n'.join(lines) + '\n')
    for tag, cls_2, cls_2xmul in (('cls2', True, False), ('cls2xmul', False, True)):
        random.seed(DATA_SEED)
        ds = DCLDataset(root, meta, transforms=tf, mode='train', cls_2=cls_2, cls_2xmul=cls_2xmul)
        items = [ds[i] for i in (0, 13, 21)]
        for j, it in enumerate(items):
            out[f'ds_{tag}_{j}_img'], out[f'ds_{tag}_{j}_swap'] = u8(it[0]), u8(it[1])
            out[f'ds_{tag}_{j}_label'], out[f'ds_{tag}_{j}_label_swap'] = np.int64(it[2]), np.int64(it[3])
            out[f'ds_{tag}_{j}_law1'], out[f'ds_{tag}_{j}_law2'] = np.array(it[4]), np.array(it[5])
        imgs, lab, lab_swap, law, names = collate_fn4train(items)
        out[f'col_{tag}_imgs'], out[f'col_{tag}_labels'] = u8(imgs), lab.numpy()
        out[f'col_{tag}_labels_swap'], out[f'col_{tag}_law'] = lab_swap.numpy(), law.numpy()
        out[f'col_{tag}_names'] = np.frombuffer(json.dumps(names).encode(), dtype=np.uint8)
    random.seed(DATA_SEED + 1)
    val = DCLDataset(root, meta, transforms=tf, mode='val')
    out['val_paths'] = np.frombuffer(json.dumps(val.paths).encode(), dtype=np.uint8)
    out['val_labels'] = np.array(val.labels)
    vitems = [val[i] for i in range(len(val))]
    imgs, lab, lab_swap, law, names = collate_fn4val(vitems)
    out['val_imgs'], out['val_col_labels'], out['val_col_labels_swap'], out['val_col_law'] = \
        u8(imgs), lab.numpy(), lab_swap.numpy(), law.numpy()
    out['data_seed'] = np.int64(DATA_SEED)

save_golden('reference_dcl', out)                   # parts of under 1 MB: tests/golden/reference_dcl.<i>.npz
print('wrote', len(out), 'arrays')
