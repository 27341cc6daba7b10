"""CrossX training benchmark: prints one JSON line.

Times, with CUDA events, random-initialised weights at the shipped config's shape (448x448, batch 8, 200 classes, P = 2):
(1) the library's step (CrossXTrainer.batch_training: forward, CrossXLoss, backward, SGD), eager and with CUDA-graph
replay, and its host synchronisations per step; (2) a stock-PyTorch restatement of the reference's step (torchvision's
ResNet-50 trunk with the ME layers and the fusion head of model/methods/CrossX.py, cuDNN with TF32 allowed, the reference's
loss ops including its CPU correlation matrix, torch.optim.SGD), with the host synchronisations of one step counted by
torch's sync debug mode; (3) everything after the trunk blocks (layer3's last block onwards, the loss and the backward) on a
fixed layer3 map, library against stock; (4) each hk_crossx_* kernel at the step's shapes against the bytes it must move
and 3.35 TB/s.  The card's name and power limit are read in the same run.

    python tests/bench_crossx.py [--steps 20] [--warmup 5]
"""
import argparse
import json
import os
import sys

import torch
import torch.nn as nn
import torch.nn.functional as F

from benchutil import card, count_syncs, timed

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tests'))

N, P, K, GAMMA = 8, 2, 200, (0.5, 0.25, 0.5)
HBM = 3.35e12


# ---- the stock-PyTorch restatement of the reference (model/methods/CrossX.py, model/loss/CrossX_loss.py) ---------------
def _gates(C):
    return nn.ModuleList(nn.Sequential(nn.Linear(C, C // 256), nn.ReLU(inplace=True), nn.Linear(C // 256, C), nn.Sigmoid())
                         for _ in range(P))


def _me_block(blk, gates, x):
    """Bottleneck.forward with meflag: (relu(c + x), [relu(c g_i + x)])"""
    c = blk.bn3(blk.conv3(blk.relu(blk.bn2(blk.conv2(blk.relu(blk.bn1(blk.conv1(x))))))))
    y = c.mean((2, 3))
    return torch.relu(c + x), [torch.relu(c * g(y)[:, :, None, None] + x) for g in gates]


class StockCrossX(nn.Module):
    def __init__(self):
        import torchvision
        super().__init__()
        tv = torchvision.models.resnet50()
        self.trunk = nn.Sequential(tv.conv1, tv.bn1, tv.relu, tv.maxpool, tv.layer1, tv.layer2, tv.layer3[:-1])
        self.b3, self.l4, self.b4 = tv.layer3[-1], tv.layer4[:-1], tv.layer4[-1]
        self.me3, self.me4 = _gates(1024), _gates(2048)
        self.conv2 = nn.ModuleList(nn.Conv2d(2048, 1024, 1, bias=False) for _ in range(P))
        self.conv3 = nn.ModuleList(nn.Conv2d(1024, 1024, 3, padding=1, bias=False) for _ in range(P))
        self.bn3 = nn.ModuleList(nn.BatchNorm2d(1024) for _ in range(P))
        self.fc_ulti, self.fc_plty, self.fc_cmbn = nn.Linear(2048 * P, K), nn.Linear(1024 * P, K), nn.Linear(1024 * P, K)

    def head(self, x3):
        x, pl = _me_block(self.b3, self.me3, x3)
        _, ul = _me_block(self.b4, self.me4, self.l4(x))
        cm = [F.adaptive_avg_pool2d(self.bn3[i](self.conv3[i](pl[i] + F.interpolate(self.conv2[i](ul[i]), 28))), 1)
              for i in range(P)]
        pl = [F.adaptive_max_pool2d(t, 1) for t in pl]
        ul = [F.adaptive_avg_pool2d(t, 1) for t in ul]
        flat = [torch.cat(t, 1).flatten(1) for t in (ul, pl, cm)]
        return (self.fc_ulti(flat[0]), self.fc_plty(flat[1]), self.fc_cmbn(flat[2]), ul, pl, cm)

    def forward(self, x):
        return self.head(self.trunk(x))


def _regular(x, gamma):
    """RegularLoss.forward: each correlation entry written into a CPU tensor"""
    corr = torch.zeros(P, P)
    x = [t.squeeze() for t in x]
    x = [t / t.norm(dim=1, keepdim=True) for t in x]
    for i in range(P):
        for j in range(P):
            corr[i, j] = torch.mean(torch.mm(x[i], x[j].t()))
            if i == j:
                corr[i, j] = 1.0 - corr[i, j]
    return torch.mul(torch.sum(torch.triu(corr)), gamma).to(x[0].device)


def stock_loss(outputs, target):
    """CrossXLoss.__call__ with num_parts > 1"""
    xf, xp, xc, ul, pl, cm = outputs
    cls = F.cross_entropy(xf + xp + xc, target, label_smoothing=0.1)
    reg = _regular(list(cm), GAMMA[2]) + _regular(list(ul), GAMMA[0]) + _regular(list(pl), GAMMA[1])
    q = F.softmax(xf, 1)
    kl = (F.kl_div(F.log_softmax(xp, 1), q, reduction='sum') + F.kl_div(F.log_softmax(xc, 1), q, reduction='sum'))
    return reg + kl / target.size(0) + cls


def with_tf32(fn):
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = True
    torch.backends.cudnn.benchmark = True
    try:
        return fn()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False


def stock_measure(x, y, x3, steps, warmup):
    net = StockCrossX().cuda().train()
    opt = torch.optim.SGD(net.parameters(), lr=0.0025, momentum=0.9, weight_decay=2e-5)

    def step():
        loss = stock_loss(net(x), y)
        opt.zero_grad()
        loss.backward()
        opt.step()

    def head():
        stock_loss(net.head(x3), y).backward()

    out = dict(stock_pytorch_step_ms=round(timed(step, steps, warmup), 3),
               stock_pytorch_host_syncs_per_step=count_syncs(step),
               stock_pytorch_head_ms=round(timed(head, steps, warmup), 3))
    del net, opt
    torch.cuda.empty_cache()
    return out


def kernels(result):
    """each hk_crossx_* kernel at the step's shapes: device time, the bytes it must move, their share of 3.35 TB/s"""
    from hawkeye_b200 import _lib
    ps = _lib.stream_ptr
    HW, C = 28 * 28, 1024
    c, r = torch.randn(N, HW, C, device='cuda'), torch.randn(N, HW, C, device='cuda')
    m = torch.randn(N, P, C, device='cuda')
    out, parts = torch.empty_like(c), torch.empty(N, HW, P, C, device='cuda')
    dc, dr, dm = torch.empty_like(c), torch.empty_like(r), torch.empty_like(m)
    ws = torch.empty(_lib.query('hk_crossx_me_bwd_workspace_bytes', N, HW, P, C), dtype=torch.uint8, device='cuda')
    R = torch.randn(N, HW // 4, C, device='cuda')
    pmax = torch.empty(N, P, C, device='cuda')
    pidx = torch.empty(N, P, C, device='cuda', dtype=torch.int32)
    cases = (
        ('me_fwd_layer3', 4 * N * HW * C * (3 + P),                     # read c, r; write out and P parts
         lambda: _lib.call('hk_crossx_me_fwd', c, r, m, out, parts, N, HW, P, C, ps())),
        ('me_bwd_layer3', 4 * N * HW * C * (5 + P),                     # read c, r, dout, P dparts; write dc, dr
         lambda: _lib.call('hk_crossx_me_bwd', c, r, m, out, parts, dc, dr, dm, N, HW, P, C, ws, ws.numel(), ps())),
        ('fuse_fwd_part', 4 * N * C * (2 * HW + HW // 4),               # read part, R; write S
         lambda: _lib.call('hk_crossx_fuse_fwd', parts, R, c, pmax, pidx, N, 28, 28, P, C, 0, ps())),
        ('fuse_bwd_part', 4 * N * C * (2 * HW + HW // 4),               # read dS; write dpart, dR
         lambda: _lib.call('hk_crossx_fuse_bwd', c, pmax, pidx, parts, R, N, 28, 28, P, C, 0, ps())),
    )
    for name, nbytes, fn in cases:
        ms = timed(fn, 50, 5)
        result[name] = dict(ms=round(ms, 4), MB=round(nbytes / 1e6, 1), share_of_hbm=round(nbytes / HBM / (ms * 1e-3), 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    args = ap.parse_args()
    result = dict(bench='crossx', image=448, batch=N, parts=P, num_classes=K)
    if not torch.cuda.is_available():
        raise SystemExit('bench_crossx: no CUDA device; nothing is measured without one: ' + json.dumps(result))
    os.environ['HAWKEYE_ALLOW_RANDOM_INIT'] = '1'
    from hawkeye_b200 import examples
    from hawkeye_b200.config import load_config
    result.update(card())
    torch.manual_seed(0)
    x = torch.randn(N, 3, 448, 448, device='cuda')
    y = torch.randint(0, K, (N,), device='cuda')
    data = dict(img=x, label=y)
    cfg = load_config(os.path.join(REPO, 'configs', 'CrossX.yaml'))
    cfg.model['pretrained'] = False
    for mode, env in (('eager', '0'), ('graph', '1')):
        os.environ['HK_CUDA_GRAPH'] = env
        tr = examples.CrossXTrainer(cfg, dataloaders={})
        result[f'step_ms_{mode}'] = round(timed(lambda: tr.batch_training(data), args.steps, max(args.warmup, 5)), 3)
        if mode == 'eager':
            result['host_syncs_per_step'] = count_syncs(lambda: tr.batch_training(data))
            net, crit = tr.model, tr.criterion
            x3 = torch.randn(N, 28, 28, 1024, device='cuda').relu_().requires_grad_(True)

            def head():
                crit(net.head(x3), y).backward()

            result['head_ms'] = round(timed(head, args.steps, args.warmup), 3)
        del tr
        torch.cuda.empty_cache()
    del os.environ['HK_CUDA_GRAPH']
    x3 = torch.randn(N, 1024, 28, 28, device='cuda').relu_().requires_grad_(True)
    result.update(with_tf32(lambda: stock_measure(x, y, x3, args.steps, args.warmup)))
    kernels(result)
    print(json.dumps(result))


if __name__ == '__main__':
    main()
