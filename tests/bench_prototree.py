"""ProtoTree benchmark: prints one JSON line.

Times, with CUDA events, at 224x224 and batch 64 (the shipped yaml): (1) the library's step (ProtoTreeTrainer.batch_training
in its eval-mode steady state: forward, NLL, backward, Adam, leaf update), eager and with CUDA-graph replay; (2) the same
step for a stock-PyTorch restatement of the reference (torchvision ResNet-50 trunk, nn.Conv2d neck, the recursive tree of
Branch / Leaf modules with the expansion-form L2 distance, F.nll_loss, torch.optim.AdamW and the per-leaf update loop) with
TF32 allowed, after checking that both give the same outputs on the same weights; (3) the head alone (distance, routing,
loss, their backward and the leaf update) against the reference's recursive tree on the same features.  The card's name
and power limit are read in the same run.

    python tests/bench_prototree.py [--steps 20] [--warmup 5]
"""
import argparse
import json
import os
import sys

import torch
import torch.nn as nn
import torch.nn.functional as F

from benchutil import card, timed

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tests'))


class Leaf(nn.Module):
    def __init__(self, index, K):
        super().__init__()
        self.index = index
        self._dist_params = nn.Parameter(torch.zeros(K), requires_grad=False)

    def forward(self, n, attr, sims):
        d = F.softmax(self._dist_params - torch.max(self._dist_params), dim=0).view(1, -1)
        return torch.cat((d,) * n, dim=0)

    def leaves(self):
        return [self]


class Branch(nn.Module):
    """branch.py:22-57 with prototype row = rank in pre-order (the package's mapping)."""

    def __init__(self, index, rank, l, r):
        super().__init__()
        self.index, self.rank, self.l, self.r = index, rank, l, r

    def forward(self, n, attr, sims):
        pa = attr.setdefault(self.index, torch.ones(n, device=sims[0].device))
        ps = sims[self.rank].squeeze(1)
        attr[self.l.index] = (1 - ps) * pa
        attr[self.r.index] = ps * pa
        ld, rd = self.l(n, attr, sims), self.r(n, attr, sims)
        ps = ps.view(n, 1)
        return (1 - ps) * ld + ps * rd

    def leaves(self):
        return self.l.leaves() + self.r.leaves()


def build_tree(height, K):
    rank = [0]

    def rec(i, d):
        if d == height:
            return Leaf(i, K), 1
        r = rank[0]
        rank[0] += 1
        left, ls = rec(i + 1, d + 1)
        right, rs = rec(i + 1 + ls, d + 1)
        return Branch(i, r, left, right), 1 + ls + rs

    return rec(0, 0)[0]


class StockProtoTree(nn.Module):
    """The reference's ProtoTreeNet restated on stock PyTorch (ProtoTreeNet.py, prototree.py, l2conv.py)."""

    def __init__(self, height, K, D):
        super().__init__()
        import torchvision
        self.backbone = nn.Sequential(*list(torchvision.models.resnet50().children())[:-2])
        self.neck_conv = nn.Sequential(nn.Conv2d(2048, D, 1, bias=False), nn.Sigmoid())
        self.root = build_tree(height, K)
        self.prototype_vectors = nn.Parameter(torch.randn(2 ** height - 1, D, 1, 1))

    def tree(self, f):
        ones = torch.ones_like(self.prototype_vectors)
        dist = F.conv2d(f ** 2, weight=ones) + torch.sum(self.prototype_vectors ** 2, dim=(1, 2, 3)).view(-1, 1, 1) \
            - 2 * F.conv2d(f, weight=self.prototype_vectors)
        dist = torch.sqrt(torch.abs(dist) + 1e-14)
        mind = -F.max_pool2d(-dist, kernel_size=dist.shape[2:]).view(f.shape[0], -1)
        sims = torch.exp(-mind).chunk(mind.shape[1], dim=1)
        attr = {}
        out = self.root(f.shape[0], attr, sims)
        return out, attr

    def forward(self, x):
        return self.tree(self.neck_conv(self.backbone(x)))


def stock_leaf_update(tree, attr, pred, labels, old, nb, eye):
    with torch.no_grad():
        target = eye[labels]
        for leaf in tree.leaves():
            dist = F.softmax(leaf._dist_params - torch.max(leaf._dist_params), dim=0)
            update = torch.sum((attr[leaf.index].unsqueeze(1) * dist * target) / pred, dim=0)
            leaf._dist_params -= old[leaf] / nb
            F.relu_(leaf._dist_params)
            leaf._dist_params += update


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    args = ap.parse_args()
    os.environ['HAWKEYE_ALLOW_RANDOM_INIT'] = '1'
    import detgen
    from hawkeye_b200 import _lib, examples
    from hawkeye_b200.config import load_config
    from hawkeye_b200 import ops_prototree as OP
    torch.cuda.set_device(0)
    N, K, H, D = 64, 200, 9, 256
    x = detgen.det((N, 3, 224, 224), 900)
    y = detgen.det_labels(N, K, 901)
    data = {'img': x.pin_memory(), 'label': y.pin_memory()}
    res = dict(metric='prototree_step_ms', batch=N, image=224, height=H, **card())

    def trainer(graph):
        os.environ['HK_CUDA_GRAPH'] = '1' if graph else '0'
        cfg = load_config(os.path.join(REPO, 'configs', 'ProtoTreeNet.yaml'))
        cfg.model.backbone['pretrain'] = ''
        tr = examples.ProtoTreeTrainer(cfg, dataloaders={})
        tr.num_batches = 94
        tr.model.train()
        tr.on_start_epoch(None)
        tr.batch_training(data)                                   # the train-mode first batch; eval mode from here on
        return tr

    for graph in (False, True):
        tr = trainer(graph)
        res['lib_graph_ms' if graph else 'lib_eager_ms'] = timed(lambda: tr.batch_training(data), args.steps, args.warmup)
        model = tr.model
        del tr

    # ---- stock PyTorch with TF32, same weights, checked against the library's outputs first ----------------------------
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.allow_tf32 = True
    stock = StockProtoTree(H, K, D).cuda()
    ours = model.state_dict()
    with torch.no_grad():
        for (k, v), s in zip([(k, v) for k, v in ours.items() if k.startswith('backbone.')], stock.backbone.state_dict().values()):
            s.copy_(v)
        stock.neck_conv[0].weight.copy_(ours['neck_conv.0.weight'])
        stock.prototype_vectors.copy_(ours['tree.prototype_layer.prototype_vectors'])
        for leaf, th in zip(stock.root.leaves(), model.tree.leaf_params):
            leaf._dist_params.copy_(th)
    model.eval()
    stock.eval()
    xc, yc = x.cuda(), y.cuda()
    with torch.no_grad():
        p_lib, _ = model(xc)
        p_ref, _ = stock(xc)
    res['pred_rel_diff'] = ((p_lib - p_ref).norm() / p_ref.norm()).item()
    assert res['pred_rel_diff'] < 5e-2, res
    opt = torch.optim.AdamW([p for p in stock.parameters() if p.requires_grad], lr=1e-3, eps=1e-7, weight_decay=0.0)
    old = {leaf: leaf._dist_params.detach().clone() for leaf in stock.root.leaves()}
    eye = torch.eye(K, device='cuda')

    def stock_step():
        opt.zero_grad()
        pred, attr = stock(xc)
        loss = F.nll_loss(torch.log(pred), yc)
        loss.backward()
        opt.step()
        stock_leaf_update(stock.root, attr, pred.detach(), yc, old, 94, eye)
    res['stock_tf32_ms'] = timed(stock_step, args.steps, args.warmup)

    # ---- the head alone: distance + routing + loss, backward, leaf update ---------------------------------------------
    f = torch.sigmoid(detgen.det((N, D, 7, 7), 902)).cuda().requires_grad_(True)
    protos = (0.5 + 0.1 * detgen.det((2 ** H - 1, D, 1, 1), 903)).cuda().requires_grad_(True)
    theta = torch.zeros(2 ** H, K, device='cuda')
    th0 = theta.clone()

    def lib_head():
        z = f.permute(0, 2, 3, 1).reshape(N, 49, D)
        mind, _ = OP.PrototypeDistanceFn.apply(z, protos, False)
        pred, _, pa = OP.RouteFn.apply(mind, theta, H)
        loss, _ = OP.NLLFn.apply(pred, yc)
        loss.backward()
        OP.leaf_update(theta, th0, pa, pred.detach(), yc, 94)
    res['lib_head_ms'] = timed(lib_head, args.steps, args.warmup)
    stock.prototype_vectors.data.copy_(protos.detach())

    def stock_head():
        pred, attr = stock.tree(f)
        F.nll_loss(torch.log(pred), yc).backward()
        stock_leaf_update(stock.root, attr, pred.detach(), yc, old, 94, eye)
    res['stock_head_ms'] = timed(stock_head, args.steps, args.warmup)
    res['launches_per_lib_head'] = None
    _lib.reset_launch_count()
    lib_head()
    torch.cuda.synchronize()
    res['launches_per_lib_head'] = _lib.launch_count()
    res['speedup_graph_vs_stock'] = res['stock_tf32_ms'] / res['lib_graph_ms']
    res['speedup_head_vs_stock'] = res['stock_head_ms'] / res['lib_head_ms']
    print(json.dumps(res))


if __name__ == '__main__':
    main()
