"""Golden fixtures for APINet from the UNMODIFIED reference (model/methods/APINet.py, model/loss/APINet_loss.py).
Run here only:  python tests/golden/make_golden_apinet.py  -> tests/golden/reference_apinet.<i>.npz
Weights come from detgen.state_like(module) and inputs from detgen seeds, so the fixture carries outputs only."""
import json
import os
import sys

import numpy as np
import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tests'))
from conftest import save_golden  # noqa: E402
from oracle import ref_harness as rh  # noqa: E402
import detgen  # noqa: E402

rh.load_reference()
from model.loss.APINet_loss import APINetLoss  # noqa: E402
from model.registry import MODEL  # noqa: E402

torch.set_num_threads(8)
out = {}
net = MODEL.get('APINet')(rh.cfg(name='APINet', num_classes=200))
out['state_keys_json'] = np.frombuffer(json.dumps({k: list(v.shape) for k, v in net.state_dict().items()},
                                                  sort_keys=True).encode(), dtype=np.uint8)
net.device = torch.device('cpu')


# ---- get_pairs: small-integer embeddings (every distance exact in fp32), exact ties, a single-sample class, n = 40 --------
def pairs_case(tag, emb, lab):
    intra, inter, il, el = net.get_pairs(emb, lab)
    out[f'pairs_{tag}_emb'], out[f'pairs_{tag}_labels'] = emb.numpy(), lab.numpy()
    out[f'pairs_{tag}_intra'], out[f'pairs_{tag}_inter'] = intra[:, 1].numpy(), inter[:, 1].numpy()
    out[f'pairs_{tag}_labels2'] = torch.cat([il[:, 1], el[:, 1]]).numpy()


rs = np.random.RandomState(11)
pairs_case('single', torch.from_numpy(rs.randint(-3, 4, size=(6, 8)).astype(np.float32)),
           torch.tensor([0, 0, 1, 2, 2, 2]))                              # class 1 has one sample: intra -> 0
base = rs.randint(-2, 3, size=(4, 4)).astype(np.float32)
emb = np.concatenate([base, base, base[:1] + 1]).astype(np.float32)       # rows i and i + 4 identical: exact ties everywhere
pairs_case('ties', torch.from_numpy(emb), torch.tensor([0, 1, 0, 1, 1, 0, 1, 0, 2]))
pairs_case('alldiff', torch.from_numpy(rs.randint(-3, 4, size=(5, 4)).astype(np.float32)), torch.arange(5))
pairs_case('allsame', torch.from_numpy(rs.randint(-3, 4, size=(5, 4)).astype(np.float32)), torch.zeros(5, dtype=torch.int64))
pairs_case('n40', detgen.det((40, 2048), 401, positive=True), torch.arange(10).repeat_interleave(4))

# ---- the head end to end: trunk replaced by nn.Identity (input = a [n, 2048, 7, 7] map), dropout off -------------------
net.backbone = nn.Identity()
net.drop.p = 0.0
head_state = detgen.state_like(net)
net.load_state_dict(head_state)
net.train()
n = 8
conv = detgen.det((n, 2048, 7, 7), 402, positive=True).requires_grad_(True)
lab = torch.arange(4).repeat_interleave(2)
self_logits, other_logits, l1, l2 = net(conv, lab, flag='train')
r1, r2 = detgen.det(self_logits.shape, 403), detgen.det(other_logits.shape, 404)
net.zero_grad()
((self_logits * r1).sum() + (other_logits * r2).sum()).backward()
out['head_self'], out['head_other'] = self_logits.detach().numpy(), other_logits.detach().numpy()
out['head_labels1'], out['head_labels2'] = l1.numpy(), l2.numpy()
out['head_dconv'] = conv.grad.numpy()
for k in ('map1.weight', 'map1.bias', 'map2.weight', 'map2.bias', 'fc.weight', 'fc.bias'):
    g = dict(net.named_parameters())[k].grad.numpy()
    out[f'head_g_{k}'] = g if g.size <= 65536 else g.reshape(g.shape[0], -1)[:, ::31]
with torch.no_grad():
    out['head_val'] = net(conv.detach(), flag='val').numpy()
print('head', float(self_logits.sum()), float(other_logits.sum()))

# ---- APINetLoss on seeded logits, with one pair exactly on the hinge --------------------------------------------------
# pair 3: self row has 10 equal maxima (target among them), the other row 20 -> p_self = fl(1/10), p_other = fl(1/20) and
# fl(p_self - p_other) == fl(0.05): the hinge argument is exactly 0 in fp32 wherever the softmax is exp(z - max) / sum
n, K = 4, 200
R = 4 * n
sl, ol = detgen.det((R, K), 405, 3.0), detgen.det((R, K), 406, 3.0)
l1 = torch.from_numpy(np.random.RandomState(407).randint(0, K, size=2 * n)).long()
l2 = torch.from_numpy(np.random.RandomState(408).randint(0, K, size=2 * n)).long()
y = int(l1[3])
others = [k for k in range(K) if k != y]
sl[3] = -100.0
sl[3, [y] + others[:9]] = 0.0
ol[3] = -100.0
ol[3, [y] + others[:19]] = 0.0
f = np.float32
assert f(f(1) / f(10)) - f(f(1) / f(20)) == f(0.05)
sl.requires_grad_(True)
ol.requires_grad_(True)
loss = APINetLoss(None)((sl, ol, l1, l2), None)
loss.backward()
out['loss_self'], out['loss_other'], out['loss_labels1'], out['loss_labels2'] = sl.detach().numpy(), ol.detach().numpy(), \
    l1.numpy(), l2.numpy()
out['loss_value'], out['loss_dself'], out['loss_dother'] = np.float64(loss.item()), sl.grad.numpy(), ol.grad.numpy()
out['loss_hinge_row'] = np.int64(3)
print('loss', loss.item())

save_golden('reference_apinet', out)                 # parts of under 1 MB: tests/golden/reference_apinet.<i>.npz
print('wrote', len(out), 'arrays')
