"""S3N benchmark: prints one JSON line.

Times, with CUDA events, at batch 8, 448x448 and 200 classes: (1) the library's S3N train step (forward, MultiSmoothLoss,
backward, SGD), eager and with CUDA-graph replay of forward, loss and backward; (2) the same step for a stock-PyTorch
restatement of the reference (torchvision ResNet-50 trunk on cuDNN / cuBLAS with TF32 allowed, the reference's host peak
loop with its per-peak reads, F.grid_sample, torch.optim.SGD); (3) the sampler pipeline alone: hk_s3n_sample_maps, the grid
and the warp, forward and backward.  The card's name and power limit are read in the same run.

    python tests/bench_s3n.py [--steps 10] [--warmup 3]
"""
import argparse
import json
import os
import random
import sys

import torch
import torch.nn as nn
import torch.nn.functional as F

from benchutil import card, timed

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tests'))

N, SIZE, K = 8, 448, 200


class Cfg(dict):
    __getattr__ = dict.__getitem__


class StockS3N(nn.Module):
    """The reference's module restated on stock PyTorch (model/methods/S3N.py), p = 0."""

    def __init__(self):
        super().__init__()
        import torchvision
        self.features = nn.Sequential(*list(torchvision.models.resnet50().children())[:-2])
        from hawkeye_b200.methods.s3n import make_gaussian
        self.radius = nn.Parameter(torch.tensor([0.12]))
        self.radius_inv = nn.Parameter(torch.tensor([0.3]))
        self.filter = nn.Conv2d(1, 1, 61, bias=False)
        with torch.no_grad():
            self.filter.weight[0, 0].copy_(torch.from_numpy(make_gaussian(61, 13)))
        g = (torch.arange(91.0) - 30) / 30
        self.register_buffer('P', torch.stack([g.expand(91, -1), g[:, None].expand(-1, 91)])[None])
        self.raw_classifier = nn.Linear(2048, K)
        self.buffers_ = nn.ModuleList(nn.Sequential(nn.Conv2d(2048, 2048, 3, 2, 1, bias=False), nn.BatchNorm2d(2048),
                                                    nn.ReLU()) for _ in range(2))
        self.cls = nn.ModuleList(nn.Linear(2048, K) for _ in range(2))
        self.con_classifier = nn.Linear(3 * 2048, K)
        yy, xx = torch.meshgrid(torch.arange(31.0), torch.arange(31.0), indexing='ij')
        self.register_buffer('yy', yy)
        self.register_buffer('xx', xx)

    def grid(self, m):
        m = F.pad(m, (30,) * 4, mode='replicate')
        s0 = self.filter(m)
        sxy = self.filter((self.P * m).view(-1, 1, 91, 91)).view(-1, 2, 31, 31)
        g = torch.clamp(sxy / s0 * 2 - 1, -1, 1)
        return F.interpolate(g, size=(SIZE, SIZE), mode='bilinear', align_corners=True).permute(0, 2, 3, 1)

    def forward(self, x):
        f = self.features(x)
        pooled = f.mean((2, 3))
        agg_origin = self.raw_classifier(pooled)
        with torch.no_grad():
            crm = F.interpolate(F.conv2d(f, self.raw_classifier.weight[:, :, None, None], self.raw_classifier.bias), 31,
                                mode='bilinear', align_corners=True)
            prob, order = torch.sort(F.softmax(crm.mean((2, 3)), 1), 1, descending=True)
            gate = (prob[:, :5] * prob[:, :5].log()).sum(1)
        xs, xs_inv = [], []
        for n in range(x.shape[0]):                       # the reference's host loop: one read per decision and peak
            dm = crm[n, order[n, 0]] if gate[n] > -0.2 else crm[n, order[n, :5]].mean(0)
            dm = (dm - dm.min()) / (dm.max() - dm.min())
            _, idx = F.max_pool2d(F.pad(dm[None, None], (1,) * 4, value=float('-inf')), 3, 1, return_indices=True)
            el = torch.arange(33 * 33, device=x.device).view(33, 33)[1:-1, 1:-1]
            peaks = torch.nonzero((idx[0, 0] == el) & (dm >= dm.mean()))
            z, c = 0.09, 0.09
            for yx in peaks.tolist():
                s = dm[yx[0], yx[1]]
                d2 = (self.xx - yx[1]) ** 2 + (self.yy - yx[0]) ** 2
                z = z + s * torch.exp(-d2 / (2 * (self.radius * s.sqrt() * 31) ** 2))
                c = c + (1 / s) * torch.exp(-d2 / (2 * (self.radius_inv * s.sqrt() * 31) ** 2))
            xs.append(z + torch.zeros(31, 31, device=x.device))
            xs_inv.append(c + torch.zeros(31, 31, device=x.device))
        outs, pools = [], [pooled]
        for i, maps in enumerate((xs, xs_inv)):
            xi = F.grid_sample(x, self.grid(torch.stack(maps)[:, None]), align_corners=True)
            pi = self.buffers_[i](self.features(xi)).mean((2, 3))
            pools.append(pi)
            outs.append(self.cls[i](pi))
        return self.con_classifier(torch.cat(pools, 1)), agg_origin, outs[0], outs[1]


def stock_loss(outputs, y, r=0.85):
    loss = 0
    for i, o in enumerate(outputs):
        if i in (1, 3):
            loss = loss + F.cross_entropy(o, y, label_smoothing=(1 - r) * K / (K - 1))
        else:
            loss = loss + F.cross_entropy(o, y)
    return loss


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    os.environ.setdefault('HAWKEYE_ALLOW_RANDOM_INIT', '1')
    import hawkeye_b200 as hb
    from hawkeye_b200 import engine, ops_s3n
    from hawkeye_b200.losses import MultiSmoothLoss
    torch.manual_seed(0)
    random.seed(0)
    x = torch.randn(N, 3, SIZE, SIZE, device='cuda')
    y = torch.randint(0, K, (N,), device='cuda')
    res = dict(card(), batch=N, image=SIZE, classes=K)

    net = hb.MODEL.get('S3N')(Cfg(num_classes=K, image_size=SIZE, radius=0.12, radius_inv=0.3, base_ratio=0.09)).cuda()
    net.train()
    crit = MultiSmoothLoss(Cfg(smooth_ratio=0.85))
    flat = engine.FlatParams(None, groups=[list(net.parameters())])
    opt = engine.FusedSGD(flat, lr=1e-4, momentum=0.0, weight_decay=1e-4)
    pt = torch.zeros(1, dtype=torch.int32, device='cuda')

    def fwd_bwd():
        opt.zero_grad()
        loss = crit(net(x, pt), y)
        loss.backward()

    def lib_step():
        fwd_bwd()
        opt.step()
    res['lib_eager_ms'] = timed(lib_step, args.steps, args.warmup)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            fwd_bwd()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            fwd_bwd()
    torch.cuda.current_stream().wait_stream(s)

    def graph_step():
        graph.replay()
        opt.step()
    res['lib_graph_ms'] = timed(graph_step, args.steps, args.warmup)

    # the sampler pipeline alone, forward and backward
    feat = torch.randn(N, 14, 14, K, device='cuda')
    rnd = torch.rand(N, 961, device='cuda')
    r = torch.tensor([0.12], device='cuda', requires_grad=True)
    ri = torch.tensor([0.3], device='cuda', requires_grad=True)
    filt = net.filter.weight.detach().clone().requires_grad_(True)
    gout = torch.randn(2 * N, 3, SIZE, SIZE, device='cuda')

    def sampler():
        maps, _ = ops_s3n.sample_maps(feat, rnd, pt, r, ri, 0.09)
        out = ops_s3n.WarpFn.apply(x, ops_s3n.GridFn.apply(maps, filt))
        out.backward(gout)
    res['lib_sampler_fwd_bwd_ms'] = timed(sampler, args.steps, args.warmup)
    del graph, net, opt, flat
    torch.cuda.empty_cache()

    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.allow_tf32 = True
    stock = StockS3N().cuda().train()
    sopt = torch.optim.SGD(stock.parameters(), lr=1e-4, weight_decay=1e-4)

    def stock_step():
        sopt.zero_grad()
        stock_loss(stock(x), y).backward()
        sopt.step()
    res['stock_ms'] = timed(stock_step, args.steps, args.warmup)
    res['speedup_graph_vs_stock'] = res['stock_ms'] / res['lib_graph_ms']
    print(json.dumps(res))


if __name__ == '__main__':
    main()
