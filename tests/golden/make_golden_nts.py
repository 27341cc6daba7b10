"""Golden fixtures for NTS-Net from the UNMODIFIED reference (model/methods/NTS_Net/*, model/loss/NTS_loss.py).
Run here only:  HAWKEYE_REF=<Hawkeye checkout> python tests/golden/make_golden_nts.py  -> tests/golden/reference_nts.<i>.npz
Shims, none of which changes what the reference computes on the CPU:
- ``np.int = int`` (numpy 2 removed the alias anchors.py and NTSNet.py use);
- ``Tensor.cuda`` is the identity;
- ``model_zoo.load_url`` returns a freshly initialised reference ResNet-50 state (``resnet50(pretrained=True)`` is
  hard-coded, NTSNet.py:19);
- ``torch.cuda.FloatTensor`` is ``torch.FloatTensor`` while ranking_loss runs (NTS_loss.py:42);
- dropout is the identity for the parity run (resnet.py:148 builds a train-mode nn.Dropout on every call).
Inputs and weights come from detgen seeds and tests/nts_inputs.py, so the tests rebuild them."""
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
from oracle import nts_oracle as O  # noqa: E402
import detgen  # noqa: E402
import nts_inputs  # noqa: E402

np.int = int
rh.load_reference()
torch.Tensor.cuda = lambda self, *a, **k: self
import torch.utils.model_zoo as model_zoo  # noqa: E402
import model.methods.NTS_Net.resnet as R  # noqa: E402
model_zoo.load_url = lambda *a, **k: R.ResNet(R.Bottleneck, [3, 4, 6, 3]).state_dict()
from model.methods.NTS_Net.NTSNet import NTSNet  # noqa: E402
from model.methods.NTS_Net.anchors import generate_default_anchor_maps, hard_nms  # noqa: E402
from model.loss.NTS_loss import NTSLoss  # noqa: E402

torch.set_num_threads(8)
out = {}

# ---- the state layout, the anchors at 224 and 448, and hard_nms on the seeded score vectors --------------------------
net = NTSNet(rh.cfg(proposal_num=6, cat_num=4, image_size=224))
out['state_keys_json'] = np.frombuffer(json.dumps([[k, list(v.shape)] for k, v in net.state_dict().items()]).encode(),
                                       dtype=np.uint8)
out['params'] = np.int64(sum(p.numel() for p in net.parameters()))
for S in (224, 448):
    _, edges, _ = generate_default_anchor_maps(input_shape=(S, S))
    anchors = (edges + 224).astype(int)
    out[f'anchors_{S}'] = anchors.astype(np.int32)
    T = nts_inputs.NMS_TOPN[S]
    picks = []
    for k in range(nts_inputs.NMS_VECTORS):
        s = nts_inputs.nms_scores(anchors, k).astype(np.float64)
        cdds = np.concatenate((s.reshape(-1, 1), anchors, np.arange(len(s)).reshape(-1, 1)), axis=1)
        picks.append(hard_nms(cdds, topn=T, iou_thresh=0.25)[:, -1].astype(np.int64))
    out[f'nms_{S}'] = np.stack(picks)
    print('anchors', S, anchors.shape, 'nms', out[f'nms_{S}'].shape)

# ---- end to end: 2 images of 224x224, detgen.state_like weights, train mode, no dropout, NTSLoss and its backward ---------
torch.nn.Dropout.forward = lambda self, x: x
net.load_state_dict(detgen.state_like(net))
net.train()
x = detgen.det((2, 3, 224, 224), 3100)
labels = detgen.det_labels(2, 200, 3101)
seen = {}
net.proposal_net.register_forward_hook(lambda m, i, o: seen.__setitem__('rpn', o.detach().clone()))
net.pretrained_model.register_forward_hook(lambda m, i, o: seen.setdefault('trunk_in', []).append(i[0].detach().clone()))
raw, concat, part, idx, prob = net(x)
torch.cuda.FloatTensor = torch.FloatTensor
loss = NTSLoss(rh.cfg(proposal_num=6))([raw, concat, part, idx, prob], labels)
loss.backward()
rpn = seen['rpn'].numpy()
out['e2e_rpn_score'] = rpn
out['e2e_top_n_index'] = idx.numpy()
out['e2e_top_n_prob'] = prob.detach().numpy()
out['e2e_gap'] = np.float64(min(O.decisive_gap(rpn[n], out['anchors_224'], 6) for n in range(2)))
parts = seen['trunk_in'][1].reshape(-1)
pix = np.random.RandomState(3102).choice(parts.numel(), 4096, replace=False)
out['e2e_part_pix_idx'], out['e2e_part_pix'] = pix, parts[torch.from_numpy(pix)].numpy()
out['e2e_raw'], out['e2e_concat'], out['e2e_part'] = raw.detach().numpy(), concat.detach().numpy(), part.detach().numpy()
out['e2e_loss'] = np.float64(loss.item())
names = ['proposal_net.down1.weight', 'proposal_net.down2.weight', 'proposal_net.down3.bias', 'proposal_net.tidy1.weight',
         'proposal_net.tidy3.bias', 'concat_net.weight', 'partcls_net.bias', 'pretrained_model.fc.weight',
         'pretrained_model.layer4.2.conv3.weight', 'pretrained_model.conv1.weight']
params = dict(net.named_parameters())
out['e2e_grad_names'] = np.frombuffer(json.dumps(names).encode(), dtype=np.uint8)
for i, k in enumerate(names):
    gr = params[k].grad.flatten()
    sel = torch.from_numpy(np.random.RandomState(3110 + i).choice(gr.numel(), min(gr.numel(), 256), replace=False))
    out[f'e2e_grad_{i}_idx'], out[f'e2e_grad_{i}'] = sel.numpy(), gr[sel].numpy()
print('e2e loss', loss.item(), 'gap', out['e2e_gap'], 'idx', idx.tolist())

save_golden('reference_nts', out)
print('wrote', len(out), 'arrays')
