"""Interp-Parts benchmark: prints one JSON line.

Times, with CUDA events, at 448x448, batch 16 and 5 parts (the shipped yaml): (1) the library's step
(InterpPartsNetTrainer.batch_training: forward, cross-entropy + shaping loss, backward, SGD, the per-iteration cosine
schedule), eager and with CUDA-graph replay; (2) the same step for a stock-PyTorch restatement of the reference
(torchvision's Bottleneck trunk, the expansion-form grouping unit with its bmm's, nn.Conv2d / nn.BatchNorm2d heads, the
shaping loss with its per-call scipy prior, torch.optim.SGD) with TF32 allowed, after checking that both give the same
outputs on the same weights; (3) the head alone (grouping, attention, post-block, loss and their backward) on the same trunk
map; (4) each grouping pass against the traffic it needs: one read of the 51.4 MB map forward, one read and one write
backward (lower bounds).  The card's name and power limit are read in the same run.

    python tests/bench_interp_parts.py [--steps 20] [--warmup 5]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tests'))
HBM_PEAK = 3.35e12              # H100 SXM data sheet, bytes/s


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in q.split(',')]
        return dict(gpu=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:
        return dict(gpu=torch.cuda.get_device_name(), power_limit=f'not read ({e})')


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


# ---- stock-PyTorch restatement of the reference model and loss --------------------------------------------------------
class StockGrouping(nn.Module):
    def __init__(self, C, K):
        super().__init__()
        self.weight = nn.Parameter(torch.zeros(K, C, 1, 1))
        self.smooth_factor = nn.Parameter(torch.zeros(K))

    def forward(self, x):
        N, C, H, W = x.shape
        K = self.weight.shape[0]
        c = self.weight.view(1, K, C).expand(N, K, C)
        cx = torch.bmm(c, x.view(N, C, H * W)).view(N, K, H, W)
        x_sq = x.pow(2).sum(1, keepdim=True).expand(-1, K, -1, -1)
        c_sq = c.pow(2).sum(2).unsqueeze(2).unsqueeze(3).expand(-1, -1, H, W)
        beta = torch.sigmoid(self.smooth_factor)
        assign = F.softmax((2 * cx - x_sq - c_sq).clamp(max=0.0) / beta.view(1, K, 1, 1).expand(N, -1, H, W), dim=1)
        assign = assign.view(N, K, -1)
        qx = torch.bmm(assign, x.view(N, C, -1).permute(0, 2, 1))
        s = assign.sum(2, keepdim=True).expand(-1, -1, C).clamp(min=1e-5)
        out = (qx / s - c) / (beta / 2).sqrt().view(1, K, 1)
        return F.normalize(out, dim=2).permute(0, 2, 1), assign.view(N, K, H, W)


class StockIP(nn.Module):
    def __init__(self, lib):
        super().__init__()
        from torchvision.models.resnet import Bottleneck
        from hawkeye_b200.methods.interp_parts import Bottleneck1x1

        class B1(Bottleneck1x1):
            def forward(self, x):
                out = F.relu(self.bn1(self.conv1(x)))
                out = F.relu(self.bn2(self.conv2(out)))
                out = self.bn3(self.conv3(out))
                return F.relu(out + (self.downsample(x) if self.downsample is not None else x))

        def mk(src):
            if isinstance(src, nn.Sequential):
                return nn.Sequential(*[mk(m) for m in src])
            if type(src).__name__ == 'Bottleneck1x1':
                b = B1(src.conv1.in_channels, src.conv1.out_channels, 1,
                       None if src.downsample is None else nn.Sequential(nn.Conv2d(1024, 2048, 1, bias=False),
                                                                          nn.BatchNorm2d(2048)))
                return b
            if type(src).__name__ == 'Bottleneck':
                return Bottleneck(src.conv1.in_channels, src.conv1.out_channels, src.stride,
                                  None if src.downsample is None else copy_seq(src.downsample))
            return copy_mod(src)

        import copy

        def copy_mod(m):
            return copy.deepcopy(m)

        def copy_seq(m):
            return copy.deepcopy(m)

        self.conv1, self.bn1, self.relu, self.maxpool = (copy.deepcopy(m) for m in (lib.conv1, lib.bn1, lib.relu, lib.maxpool))
        self.layer1, self.layer2, self.layer3 = mk(lib.layer1), mk(lib.layer2), mk(lib.layer3)
        self.grouping = StockGrouping(1024, lib.n_parts)
        self.post_block, self.attconv = mk(lib.post_block), mk(lib.attconv)
        self.groupingbn, self.mylinear = copy.deepcopy(lib.groupingbn), copy.deepcopy(lib.mylinear)
        self.n_parts = lib.n_parts
        self.load_state_dict(lib.state_dict())

    def trunk(self, x):
        return self.layer3(self.layer2(self.layer1(self.maxpool(self.relu(self.bn1(self.conv1(x)))))))

    def head(self, x):
        region, assign = self.grouping(x)
        region = region.contiguous().unsqueeze(3)
        att = F.softmax(self.attconv(region), dim=2)
        out = (self.post_block(region) * att).contiguous().squeeze(3)
        out = F.avg_pool1d(out, self.n_parts) * self.n_parts
        out = self.groupingbn(out.contiguous().unsqueeze(3))
        return self.mylinear(out.view(out.size(0), -1)), att, assign

    def forward(self, x):
        return self.head(self.trunk(x))


def stock_shaping(assign, radius=2, std=0.4, alpha=1, beta=0.001, eps=1e-5):
    """InterpParts_loss.py:83-138, including its per-call prior on the host."""
    from scipy import stats
    from hawkeye_b200.ops_interp_parts import gaussian_taps
    N, K = assign.shape[:2]
    S = 2 * radius + 1
    w = gaussian_taps(radius, std).view(1, 1, S, S).expand(K, 1, S, S).cuda()
    occ = F.adaptive_max_pool2d(F.conv2d(assign, w, groups=K), (1, 1)).squeeze(2).squeeze(2)
    emp, _ = occ.sort(dim=0)
    grid = (torch.arange(1., 2 * N, 2.).float().cuda() / (2 * N)).cpu().numpy()
    prior = torch.tensor(stats.beta.ppf(grid, a=alpha, b=beta)).float().cuda().unsqueeze(1)
    return ((emp + eps).log() - (prior + eps).log()).abs().mean()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_interp_parts needs a CUDA device')
    os.environ.setdefault('HAWKEYE_ALLOW_RANDOM_INIT', '1')
    import detgen
    from hawkeye_b200 import _lib, examples
    from hawkeye_b200.config import load_config
    N, S, K = 16, 448, 5
    res = dict(bench='interp_parts', batch=N, image=S, parts=K, **card())
    data = {'img': detgen.det((N, 3, S, S), 3000).pin_memory(), 'label': detgen.det_labels(N, 200, 3001).pin_memory()}

    def trainer(graph):
        os.environ['HK_CUDA_GRAPH'] = '1' if graph else '0'
        cfg = load_config(os.path.join(REPO, 'configs', 'InterpPartsNet.yaml'))
        tr = examples.InterpPartsNetTrainer(cfg, dataloaders={})
        tr.model.train()
        return tr

    tr = trainer(False)
    res['lib_step_eager_ms'] = timed(lambda: tr.batch_training(data), args.steps, args.warmup)
    state = {k: v.detach().clone() for k, v in tr.model.state_dict().items()}
    lib_model = tr.model
    del tr
    trg = trainer(True)
    res['lib_step_graph_ms'] = timed(lambda: trg.batch_training(data), args.steps, max(args.warmup, 5))
    del trg

    # same outputs on the same weights (train mode: both on batch statistics), then the stock step with TF32
    lib_model.load_state_dict(state)
    stock = StockIP(lib_model).cuda().train()
    x = data['img'].cuda()
    labels = data['label'].cuda()
    _lib.set_precise(1)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    with torch.no_grad():
        a = lib_model(x)
        b = stock(x)
    _lib.set_precise(0)
    res['parity_logits_rel_l2'] = ((a[0] - b[0]).norm() / b[0].norm()).item()
    res['parity_logits_norms'] = [a[0].norm().item(), b[0].norm().item()]
    res['parity_att_rel_l2'] = ((a[1] - b[1]).norm() / b[1].norm()).item()
    res['parity_assign_max_abs'] = (a[2] - b[2]).abs().max().item()
    assert res['parity_logits_rel_l2'] < 1e-2, res
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = True
    fine = [p for n, p in stock.named_parameters() if n.split('.')[0] in ('conv1', 'bn1', 'layer1', 'layer2', 'layer3')]
    rest = [p for n, p in stock.named_parameters() if n.split('.')[0] not in ('conv1', 'bn1', 'layer1', 'layer2', 'layer3')]
    opt = torch.optim.SGD([{'params': fine, 'lr': 5e-4}, {'params': rest, 'lr': 1e-2}], weight_decay=5e-4, momentum=0.9)
    ce = nn.CrossEntropyLoss()

    def stock_step():
        logits, att, assign = stock(x)
        loss = ce(logits, labels) + 0.5 * stock_shaping(assign)
        opt.zero_grad()
        loss.backward()
        opt.step()

    res['stock_step_tf32_ms'] = timed(stock_step, args.steps, args.warmup)

    # the head alone on a fixed trunk map
    with torch.no_grad():
        feat = stock.trunk(x)
    feat_nhwc = feat.permute(0, 2, 3, 1).contiguous()
    from hawkeye_b200.losses import InterpPartsLoss
    from hawkeye_b200 import ops, ops_interp_parts as OP, ops_resnet
    crit = InterpPartsLoss(load_config(os.path.join(REPO, 'configs', 'InterpPartsNet.yaml')).train.criterion)
    m = lib_model

    def lib_head():
        f = feat_nhwc.requires_grad_(True)
        region, assign = m.grouping(f)
        region = region.view(N, K, 1, -1)
        a_ = ops_resnet.block_stack(region, m._att_blocks, True)
        p_ = ops_resnet.block_stack(region, m._post_blocks, True)
        pooled, att = OP.AttentionPoolFn.apply(a_.view(N * K, -1), p_.view(N * K, -1), m.attconv[2].weight, m.attconv[2].bias,
                                               m.attconv[3].weight, m.attconv[3].bias, m.attconv[3], True, N, K)
        out = ops_resnet.RowBatchNormFn.apply(pooled, m.groupingbn.weight, m.groupingbn.bias, m.groupingbn, True)
        logits = ops.linear(out, m.mylinear.weight, m.mylinear.bias)
        crit((logits, att.view(N, 1, K, 1), assign), labels).backward()

    def stock_head():
        f = feat.detach().requires_grad_(True)
        logits, att, assign = stock.head(f)
        (ce(logits, labels) + 0.5 * stock_shaping(assign)).backward()

    res['lib_head_ms'] = timed(lib_head, args.steps, args.warmup)
    res['stock_head_tf32_ms'] = timed(stock_head, args.steps, args.warmup)

    # each grouping pass against its required traffic
    C, H, W = 1024, feat.shape[2], feat.shape[3]
    HW = H * W
    dev = x.device
    e = lambda *s: torch.empty(*s, device=dev, dtype=torch.float32)
    assign, dist, out, qx, ssum, nrm = e(N, K, H, W), e(N, K, HW), e(N, K, C), e(N, K, C), e(N, K), e(N, K)
    ws = torch.empty(_lib.query('hk_ip_group_workspace_bytes', N, HW, K, C), device=dev, dtype=torch.uint8)
    cen, sf = m.grouping.weight.detach(), m.grouping.smooth_factor.detach()
    s = _lib.stream_ptr()
    fwd = lambda: _lib.call('hk_ip_group_fwd', feat_nhwc, cen, sf, assign, dist, out, qx, ssum, nrm, N, HW, K, C, ws,
                            ws.numel(), s)
    fwd()
    dout = torch.randn(N, K, C, device=dev)
    dx, dcen, dsf = torch.empty_like(feat_nhwc), torch.empty_like(cen), torch.empty_like(sf)
    bwd = lambda: _lib.call('hk_ip_group_bwd', feat_nhwc, cen, sf, assign, dist, qx, ssum, nrm, dout, None, None, None, None,
                            0, dx, dcen, dsf, N, H, W, K, C, ws, ws.numel(), s)
    map_bytes = feat_nhwc.numel() * 4
    res['map_MB'] = map_bytes / 1e6
    res['group_fwd_ms'] = timed(fwd, 10 * args.steps, args.warmup)
    res['group_bwd_ms'] = timed(bwd, 10 * args.steps, args.warmup)
    res['group_fwd_GBps'] = map_bytes / (res['group_fwd_ms'] * 1e-3) / 1e9
    res['group_bwd_GBps'] = 2 * map_bytes / (res['group_bwd_ms'] * 1e-3) / 1e9
    res['group_fwd_share_of_hbm_peak'] = res['group_fwd_GBps'] * 1e9 / HBM_PEAK
    res['group_bwd_share_of_hbm_peak'] = res['group_bwd_GBps'] * 1e9 / HBM_PEAK
    res['speedup_step_graph_vs_stock'] = res['stock_step_tf32_ms'] / res['lib_step_graph_ms']
    print(json.dumps({k: (float(f'{v:.4g}') if isinstance(v, float) else v) for k, v in res.items()}))


if __name__ == '__main__':
    main()
