"""CIN training benchmark: prints one JSON line.

Times, with CUDA events, random-initialised weights at the shipped config's shape (224x224, batch 20 = 4 classes x 5
images, h: 100352 -> 512): (1) the library's training step (CINTrainer.batch_training: ResNet-50 trunk, channel
interaction, classifier, CINLoss, backward, SGD over the model and h), eager and with CUDA-graph replay; (2) a stock-PyTorch
restatement of the reference's step (torchvision ResNet-50 on cuDNN with TF32, the module in torch ops, CINLoss with its
boolean indexing, torch.optim.SGD), with the host synchronisations of one of its steps counted by torch's sync debug mode;
(3) the head alone on a fixed trunk map: module, classifier, loss and backward, library and stock.  The card's name and
power limit are read in the same run.

    python tests/bench_cin.py [--steps 10] [--warmup 3] [--labels balanced|some]
"""
import argparse
import json
import os
import sys

import torch
import torch.nn as nn
import torch.nn.functional as F

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tests'))
import cin_inputs as I  # noqa: E402
from benchutil import card, count_syncs, timed  # noqa: E402


# ---- the stock-PyTorch restatement of the reference (model/methods/CIN.py, model/loss/CIN_loss.py, Examples/CIN.py) -------
class StockHead(nn.Module):
    def __init__(self, C=2048, WH=49, K=200):
        super().__init__()
        self.conv = nn.Conv2d(C, C, 3, 1, 1)
        self.fc = nn.Linear(2 * C * WH, 1)
        self.classifier = nn.Linear(C, K)

    def forward(self, x):
        B, C, H, W = x.shape
        X = x.reshape(B, C, H * W)
        w_sci = torch.softmax(-(X @ X.transpose(1, 2)) / (H * W), dim=-1)
        y = self.conv((w_sci @ X).view(B, C, H, W))
        z = y + x
        yv = y.reshape(B, -1)
        weight = torch.cat((self.fc(torch.cat((yv[:B // 2], yv[B // 2:]), 1)),
                            self.fc(torch.cat((yv[B // 2:], yv[:B // 2]), 1))), 0).view(B, 1, 1)
        w_cci = torch.abs(w_sci - weight * torch.cat((w_sci[B // 2:], w_sci[:B // 2]), 0))
        z_cci = self.conv((w_cci @ X).view(B, C, H, W)) + x
        return self.classifier(z.mean((2, 3))), z_cci.reshape(B, C, H * W)


class StockLoss(nn.Module):
    def __init__(self, alpha=2.0, beta=0.5):
        super().__init__()
        self.alpha, self.beta = alpha, beta
        self.h = nn.Linear(I.F, I.R)

    def forward(self, out, target):
        z, z_cci = out
        B = z_cci.shape[0]
        za = self.h(z_cci.reshape(B, -1))
        pair = target[:B // 2] == target[B // 2]
        l1 = F.pairwise_distance(za[:B // 2][pair], za[B // 2:][pair]).pow(2).sum()
        hinge = self.beta - F.pairwise_distance(za[:B // 2][~pair], za[B // 2:][~pair])     # computed, then overwritten
        hinge[hinge < 0] = 0
        return F.cross_entropy(z, target, label_smoothing=0.1) + self.alpha * (l1 + l1 ** 2)


def stock_step(x, y, steps, warmup):
    import torchvision
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = True
    torch.backends.cudnn.benchmark = True
    trunk = nn.Sequential(*list(torchvision.models.resnet50().children())[:-2])
    net = nn.Sequential(trunk, StockHead()).cuda().train()
    crit = StockLoss().cuda()
    opt = torch.optim.SGD([{'params': net.parameters()}, {'params': crit.parameters()}], lr=1e-4, weight_decay=2e-4)

    def step():
        loss = crit(net(x), y)
        opt.zero_grad()
        loss.backward()
        opt.step()

    ms = timed(step, steps, warmup)
    syncs = count_syncs(step)
    head_ms = stock_head(net[1], crit, steps, warmup, y)
    del net, opt, crit
    torch.cuda.empty_cache()
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    return round(ms, 3), syncs, round(head_ms, 3)


def trunk_map():
    return torch.randn(I.B, I.C, 7, 7, device='cuda').relu().requires_grad_(True)


def stock_head(head, crit, steps, warmup, y):
    f = trunk_map()

    def step():
        crit(head(f), y).backward()
        for p in list(head.parameters()) + list(crit.parameters()) + [f]:
            p.grad = None

    return timed(step, steps, warmup)


def lib_head(net, crit, steps, warmup, y):
    f = trunk_map()

    def step():
        crit(net.classifier(net.ChannelInteraction(f)), y).backward()
        for p in list(net.parameters()) + list(crit.parameters()) + [f]:
            p.grad = None

    return timed(step, steps, warmup)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--labels', default='balanced', choices=sorted(I.LABELS))
    args = ap.parse_args()
    result = dict(bench='cin', image=224, batch=I.B, labels=args.labels)
    if not torch.cuda.is_available():
        raise SystemExit('bench_cin: no CUDA device; nothing is measured without one: ' + json.dumps(result))
    os.environ['HAWKEYE_ALLOW_RANDOM_INIT'] = '1'
    from hawkeye_b200 import examples
    from hawkeye_b200.config import load_config
    result.update(card())
    cfg = load_config(os.path.join(REPO, 'configs', 'CIN.yaml'))
    x = torch.randn(I.B, 3, 224, 224, device='cuda')
    y = I.labels(args.labels).cuda()
    data = dict(img=x, label=y)
    for mode, env in (('eager', '0'), ('graph', '1')):
        os.environ['HK_CUDA_GRAPH'] = env
        tr = examples.CINTrainer(cfg, dataloaders={})
        result[f'step_ms_{mode}'] = round(timed(lambda: tr.batch_training(data), args.steps, max(args.warmup, 5)), 3)
        if mode == 'eager':
            result['host_syncs_per_step'] = count_syncs(lambda: tr.batch_training(data))
            result['head_alone_ms'] = round(lib_head(tr.model, tr.criterion, args.steps, args.warmup, y), 3)
        del tr
        torch.cuda.empty_cache()
    del os.environ['HK_CUDA_GRAPH']
    (result['stock_pytorch_step_ms'], result['stock_pytorch_host_syncs_per_step'],
     result['stock_pytorch_head_alone_ms']) = stock_step(x, y, args.steps, args.warmup)
    print(json.dumps(result))


if __name__ == '__main__':
    main()
