"""Golden fixtures for ProtoTree from the UNMODIFIED reference (model/methods/ProtoTree/, Examples/ProtoTreeNet.py).
Run here only:  HAWKEYE_REF=<Hawkeye checkout> python tests/golden/make_golden_prototree.py
    -> tests/golden/reference_prototree.<i>.npz
The iNat checkpoint the model loads is a synthetic one with the BBN layout, written to a temporary file.  The reference maps
prototype rows to branches through a set ordered by object hash (prototree.py:51), so the fixture records this process's
mapping: ``*_perm[k]`` is the prototype row of the k-th branch in pre-order, and every prototype array is stored in that
(the package's) order."""
import json
import os
import sys
import tempfile

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tests'))
from conftest import save_golden  # noqa: E402
from oracle import ref_harness as rh  # noqa: E402
import detgen  # noqa: E402

rh.load_reference()
from model.registry import MODEL  # noqa: E402
from model.methods.ProtoTree.prototree import ProtoTree  # noqa: E402

torch.set_num_threads(8)
out = {}


def perm_of(tree):
    """prototype row of each branch, branches in pre-order (node.index order)"""
    return np.array([tree._out_map[b] for b in sorted(tree.branches, key=lambda b: b.index)], dtype=np.int64)


def leaves_in_order(tree):
    return sorted(tree.leaves, key=lambda l: l.index)


def model_cfg(pretrain, height=9, **kw):
    return rh.cfg(name='ProtoTreeNet', num_classes=200, height=height, W1=1, H1=1, num_features=256,
                  backbone=dict(name='resnet50', pretrain=pretrain), **kw)


# ---- a synthetic iNat (BBN) checkpoint: module.backbone.* with cb_block / rb_block, and a classifier ---------------------
with tempfile.TemporaryDirectory() as tmp:
    from model.backbone import resnet50
    donor = resnet50(pretrained=False)
    g = torch.Generator().manual_seed(900)
    inat = {}
    for k, v in donor.state_dict().items():
        if k.startswith('fc.'):
            continue
        name = k.replace('layer4.2.', 'cb_block.') if k.startswith('layer4.2.') else k
        inat['module.backbone.' + name] = (torch.randn(v.shape, generator=g) if v.is_floating_point() else v.clone())
        if k.startswith('layer4.2.'):
            inat['module.backbone.' + k.replace('layer4.2.', 'rb_block.')] = torch.zeros_like(v)
    inat['module.classifier.weight'] = torch.randn(10, 4096, generator=g)
    path = os.path.join(tmp, 'inat.pth')
    torch.save(inat, path)
    net = MODEL.get('ProtoTreeNet')(model_cfg(path))
    renamed = net.get_inat_resnet50_weight(path)
    out['inat_keys_json'] = np.frombuffer(json.dumps(sorted(inat)).encode(), dtype=np.uint8)
    out['inat_renamed_json'] = np.frombuffer(json.dumps(sorted(renamed)).encode(), dtype=np.uint8)
    # what landed in the trunk: layer4.2's conv1 weight (from cb_block) and bn1's running mean
    out['inat_l42_conv1_slice'] = net.backbone[7][2].conv1.weight.detach()[:4, :4].numpy()
    out['inat_cb_conv1_slice'] = inat['module.backbone.cb_block.conv1.weight'][:4, :4].numpy()
    out['inat_bn1_rm'] = net.backbone[1].running_mean.detach().numpy()
out['state_keys_json'] = np.frombuffer(json.dumps([[k, list(v.shape)] for k, v in net.state_dict().items()]).encode(),
                                       dtype=np.uint8)
out['model_perm'] = perm_of(net.tree)

# ---- the whole model end to end: detgen.state_like weights (prototypes permuted into pre-order for the package), train
# mode, 2 images of 64x64 (a 2x2 trunk map), F.nll_loss(log(pred)) and its backward ------------------------------------
net.load_state_dict(detgen.state_like(net))
with torch.no_grad():
    for j, leaf in enumerate(leaves_in_order(net.tree)):
        leaf._dist_params.copy_(detgen.det((200,), 700 + j))
net.train()
x = detgen.det((2, 3, 64, 64), 701)
labels = detgen.det_labels(2, 200, 702)
feats = []
net.backbone.register_forward_hook(lambda m, i, o: feats.append(o.detach()))
pred, info = net(x)
loss = F.nll_loss(torch.log(pred), labels)
loss.backward()
perm = torch.as_tensor(out['model_perm'])
out['e2e_x'], out['e2e_labels'] = x.numpy(), labels.numpy()
out['e2e_feat_slice'] = feats[0][:, ::16].numpy()
out['e2e_pred'], out['e2e_loss'] = pred.detach().numpy(), np.float64(loss.item())
out['e2e_g_neck_slice'] = net.neck_conv[0].weight.grad[:, ::16].numpy()
out['e2e_g_protos'] = net.tree.prototype_layer.prototype_vectors.grad[perm].numpy()
out['e2e_g_layer4_bn3_w'] = net.backbone[7][2].bn3.weight.grad.numpy()
out['e2e_pa_root'] = info['pa_tensor'][0].detach().numpy()
print('e2e', loss.item())


# ---- the tree alone at height 9 on given features.  Inputs come from detgen seeds (tests rebuild them): prototypes
# 0.5 + 0.1 det(seed) (reference rows; row perm[k] is branch k's), leaf j det((200,), seed + 1 + j), features
# sigmoid(det((N, 256, S, S), seed + 2000)), labels det_labels(N, 200, seed + 2001) ---------------------------------------
def tree_case(tag, height, N, S, seed, **kw):
    t = ProtoTree(rh.cfg(num_classes=200, height=height, W1=1, H1=1, num_features=256, **kw))
    with torch.no_grad():
        t.prototype_layer.prototype_vectors.copy_(0.5 + 0.1 * detgen.det(tuple(t.prototype_layer.prototype_vectors.shape),
                                                                         seed))
        for j, leaf in enumerate(leaves_in_order(t)):
            leaf._dist_params.copy_(detgen.det((200,), seed + 1 + j))
    p = torch.as_tensor(perm_of(t))
    feat = torch.sigmoid(detgen.det((N, 256, S, S), seed + 2000)).requires_grad_(True)
    y = detgen.det_labels(N, 200, seed + 2001)
    dist = t.prototype_layer(feat)
    mind = -F.max_pool2d(-dist, kernel_size=(S, S)).view(N, -1)
    pred, info = t(feat, feat)
    loss = F.nll_loss(torch.log(pred), y)
    loss.backward()
    out[f'{tag}_perm'] = p.numpy()
    out[f'{tag}_labels'], out[f'{tag}_seed'] = y.numpy(), np.int64(seed)
    out[f'{tag}_mind'] = mind.detach()[:, p].numpy()
    branches = sorted(t.branches, key=lambda b: b.index)
    out[f'{tag}_ps'] = torch.cat([info['ps'][b.index] for b in branches], 1).detach().numpy()
    out[f'{tag}_pa'] = torch.cat([info['pa_tensor'][i] for i in range(t.size)], 1).detach().numpy()
    out[f'{tag}_pred'], out[f'{tag}_loss'] = pred.detach().numpy(), np.float64(loss.item())
    out[f'{tag}_dfeat_slice'] = feat.grad[:, ::4].numpy()
    out[f'{tag}_dprotos_slice'] = t.prototype_layer.prototype_vectors.grad[p][:, ::8].numpy()
    print(tag, loss.item())
    return t, info, pred, y


t, info, pred, y = tree_case('tree', 9, 4, 7, 710)

# one derivative-free leaf update (Examples/ProtoTreeNet.py:116-132) on tree.leaves, with a snapshot and 7 batches per epoch
num_batches = 7
leaves = leaves_in_order(t)
with torch.no_grad():
    old = {leaf: (0.3 * detgen.det((200,), 3000 + j)).abs() for j, leaf in enumerate(leaves)}
    target = torch.eye(200)[y]
    for leaf in t.leaves:
        update = torch.sum((info['pa_tensor'][leaf.index] * leaf.distribution() * target) / pred, dim=0)
        leaf._dist_params -= (old[leaf] / num_batches)
        F.relu_(leaf._dist_params)
        leaf._dist_params += update
out['upd_theta_rows'] = torch.stack([l._dist_params for l in leaves])[::4].numpy()     # theta0: 0.3 |det((200,), 3000 + j)|
out['upd_num_batches'] = np.int64(num_batches)

# dtheta with gradient-trained leaves (disable_derivative_free_leaf_optim)
t2, _, _, _ = tree_case('dfo_off', 9, 4, 7, 720, disable_derivative_free_leaf_optim=True)
out['dfo_off_dtheta_rows'] = torch.stack([l._dist_params.grad for l in leaves_in_order(t2)])[::4].numpy()

save_golden('reference_prototree', out)
print('wrote', len(out), 'arrays')
