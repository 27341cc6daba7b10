"""APINet train step (ResNet-101, 10 classes x 4 images at 224x224, Adam): the library's step with CUDA-graph replay off and
on, against a stock-PyTorch restatement of the reference's module and loss (model/methods/APINet.py, model/loss/APINet_loss.py;
pair mining with the reference's host round trip, TF32 allowed).  Device-event timing after a warm-up; the outputs of both
steps on the same weights and batch are compared first.  Prints one JSON line.

    python tests/bench_apinet.py [--steps 20] [--warmup 5]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn as nn

from benchutil import timed

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))


# ---- stock PyTorch restatement of the reference (same state_dict layout as the library's model) -------------------------
class Bottleneck(nn.Module):
    def __init__(self, inplanes, planes, stride=1, downsample=None):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = nn.Conv2d(planes, planes, 3, stride, 1, bias=False)
        self.bn2 = nn.BatchNorm2d(planes)
        self.conv3 = nn.Conv2d(planes, planes * 4, 1, bias=False)
        self.bn3 = nn.BatchNorm2d(planes * 4)
        self.relu = nn.ReLU(inplace=True)
        self.downsample = downsample

    def forward(self, x):
        out = self.relu(self.bn1(self.conv1(x)))
        out = self.relu(self.bn2(self.conv2(out)))
        out = self.bn3(self.conv3(out))
        return self.relu(out + (x if self.downsample is None else self.downsample(x)))


def stock_trunk(layers=(3, 4, 23, 3)):
    mods = [nn.Conv2d(3, 64, 7, 2, 3, bias=False), nn.BatchNorm2d(64), nn.ReLU(inplace=True), nn.MaxPool2d(3, 2, 1)]
    inplanes = 64
    for planes, n, stride in zip((64, 128, 256, 512), layers, (1, 2, 2, 2)):
        ds = nn.Sequential(nn.Conv2d(inplanes, planes * 4, 1, stride, bias=False), nn.BatchNorm2d(planes * 4))
        blocks = [Bottleneck(inplanes, planes, stride, ds)] + [Bottleneck(planes * 4, planes) for _ in range(1, n)]
        mods.append(nn.Sequential(*blocks))
        inplanes = planes * 4
    return nn.Sequential(*mods)


def pdist(v):
    return -2 * v.mm(torch.t(v)) + v.pow(2).sum(dim=1).view(1, -1) + v.pow(2).sum(dim=1).view(-1, 1)


class StockAPINet(nn.Module):
    def __init__(self, num_classes=200):
        super().__init__()
        self.backbone = stock_trunk()
        self.avg = nn.AvgPool2d(kernel_size=7, stride=1)
        self.map1 = nn.Linear(2048 * 2, 512)
        self.map2 = nn.Linear(512, 2048)
        self.fc = nn.Linear(2048, num_classes)
        self.drop = nn.Dropout(p=0.5)
        self.sigmoid = nn.Sigmoid()

    def get_pairs(self, embeddings, labels):                 # the reference's numpy mining, host round trip included
        d = pdist(embeddings).detach().cpu().numpy()
        labels = labels.detach().cpu().numpy().reshape(-1, 1)
        eq = labels == labels.T
        np.fill_diagonal(eq, False)
        intra = np.argmin(np.where(eq, d, np.inf), axis=1)
        np.fill_diagonal(eq, True)
        inter = np.argmin(np.where(eq, np.inf, d), axis=1)
        dev = embeddings.device
        lab = torch.from_numpy(labels.reshape(-1)).to(dev)
        return torch.from_numpy(intra).to(dev), torch.from_numpy(inter).to(dev), lab

    def forward(self, images, targets, pairs=None):
        return self.head(self.avg(self.backbone(images)).squeeze(), targets, pairs)

    def head(self, pool, targets, pairs=None):
        n = pool.size(0)
        intra, inter, lab = self.get_pairs(pool, targets) if pairs is None else pairs
        ar = torch.arange(n, device=pool.device)
        f1 = torch.cat([pool[ar], pool[ar]])
        f2 = torch.cat([pool[intra], pool[inter]])
        l1, l2 = torch.cat([lab, lab]), torch.cat([lab[intra], lab[inter]])
        m = self.map2(self.drop(self.map1(torch.cat([f1, f2], 1))))
        g1, g2 = self.sigmoid(m * f1), self.sigmoid(m * f2)
        fs = [g1 * f1 + f1, g2 * f1 + f1, g2 * f2 + f2, g1 * f2 + f2]
        s1, o1, s2, o2 = [self.fc(self.drop(t)) for t in fs]
        return torch.cat([s1, s2]), torch.cat([o1, o2]), l1, l2


class StockLoss(nn.Module):
    def __init__(self):
        super().__init__()
        self.ce = nn.CrossEntropyLoss(label_smoothing=0.1)
        self.rank = nn.MarginRankingLoss(margin=0.05)

    def forward(self, out):
        s, o, l1, l2 = out
        t = torch.cat([l1, l2])
        idx = torch.arange(s.shape[0], device=s.device)
        ss, so = torch.softmax(s, 1)[idx, t], torch.softmax(o, 1)[idx, t]
        return self.ce(torch.cat([s, o]), torch.cat([t, t])) + self.rank(ss, so, torch.ones_like(ss))


def gpu_info():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(',')]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), 'unknown'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_apinet needs a CUDA device')
    os.environ['HAWKEYE_ALLOW_RANDOM_INIT'] = '1'
    import detgen
    from hawkeye_b200 import examples
    from hawkeye_b200.config import load_config
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.allow_tf32 = True
    x = detgen.det((40, 3, 224, 224), 500).cuda()
    y = torch.arange(10).repeat_interleave(4).cuda()
    batch = {'img': x, 'label': y}
    cfg = load_config(os.path.join(ROOT, 'configs', 'APINet.yaml'))
    line = {'workload': 'APINet ResNet-101 train step, 10 classes x 4 images, 224x224, Adam', 'unit': 'ms/step'}

    # outputs first: the same weights and batch through both, dropout off
    os.environ['HK_CUDA_GRAPH'] = '0'
    tr = examples.APINetTrainer(cfg, dataloaders={})
    state = {k: v.detach().cpu().clone() for k, v in tr.model.state_dict().items()}
    stock = StockAPINet().cuda().train()
    stock.load_state_dict(state)
    tr.model.drop.p = stock.drop.p = 0.0
    with torch.no_grad():
        s_n, o_n, l1n, l2n = tr.model(x, y)
        s_s, o_s, l1s, l2s = stock(x, y)
        loss_n = tr.criterion((s_n, o_n, l1n, l2n)).item()
        loss_s = StockLoss()((s_s, o_s, l1s, l2s)).item()
        pool_n, pool_s = tr.model.pool(x), stock.avg(stock.backbone(x)).squeeze()
        # near-tied distances can pick other pairs when the trunks differ in the last bits: compare the head and the loss
        # on the pairs the library mined as well
        from hawkeye_b200.ops_apinet import mine_pairs
        idx2, _, _ = mine_pairs(pool_n, y)
        s_f, o_f, l1f, l2f = stock(x, y, pairs=(idx2[:40], idx2[40:], y))
        loss_f = StockLoss()((s_f, o_f, l1f, l2f)).item()

    def rel(a, b):
        return ((a.double() - b.double()).norm() / b.double().norm()).item()
    line['compare'] = {'pool_rel_l2': rel(pool_n, pool_s), 'pairs_equal_frac': (l2n == l2s).double().mean().item(),
                       'logits_rel_l2_same_pairs': rel(torch.cat([s_n, o_n]), torch.cat([s_f, o_f])),
                       'loss_native': loss_n, 'loss_stock_same_pairs': loss_f, 'loss_stock_own_pairs': loss_s}
    tr.model.drop.p = stock.drop.p = 0.5
    tr.model.load_state_dict({k: v.cuda() for k, v in state.items()})

    for g in tr.optimizer.param_groups:
        g['lr'] = 1e-4
    line['native_eager_ms'] = timed(lambda: tr.batch_training(batch), args.steps, args.warmup)
    del tr
    os.environ['HK_CUDA_GRAPH'] = '1'
    tg = examples.APINetTrainer(cfg, dataloaders={})
    for g in tg.optimizer.param_groups:
        g['lr'] = 1e-4
    line['native_graph_ms'] = timed(lambda: tg.batch_training(batch), args.steps, max(args.warmup, 5))
    del tg
    torch.cuda.empty_cache()

    bb = {id(p) for p in stock.backbone.parameters()}
    opt = torch.optim.Adam([{'params': stock.backbone.parameters(), 'lr': 1e-4},
                            {'params': [p for p in stock.parameters() if id(p) not in bb], 'lr': 1e-4}], weight_decay=2e-8)
    crit = StockLoss()

    def stock_step():
        loss = crit(stock(x, y))
        opt.zero_grad()
        loss.backward()
        opt.step()
        return loss
    line['stock_ms'] = timed(stock_step, args.steps, args.warmup)
    # the APINet part alone (pairs, head, fc, loss, backward to the pooled features) on a fixed pool
    pool = pool_n.detach().clone()
    import hawkeye_b200 as hb
    from hawkeye_b200.losses import APINetLoss
    head = hb.MODEL.get('APINet')(cfg.model)
    head.backbone = nn.Identity()
    head = head.cuda().train()
    pool4 = pool.view(40, 2048, 1, 1).expand(40, 2048, 7, 7).contiguous().requires_grad_(True)
    crit_n = APINetLoss(None)

    def native_head():
        crit_n(head(pool4, y)).backward()
    pool_s4 = pool.clone().requires_grad_(True)

    def stock_head():
        crit(stock.head(pool_s4, y)).backward()
    line['native_head_ms'] = timed(native_head, args.steps, args.warmup)
    line['stock_head_ms'] = timed(stock_head, args.steps, args.warmup)
    line['speedup_eager'] = line['stock_ms'] / line['native_eager_ms']
    line['speedup_graph'] = line['stock_ms'] / line['native_graph_ms']
    line['img_per_s_graph'] = 40 * 1000.0 / line['native_graph_ms']
    line['gpu'], line['power_limit'] = gpu_info()
    line['steps'], line['warmup'] = args.steps, args.warmup
    print(json.dumps(line), flush=True)


if __name__ == '__main__':
    main()
