"""DCL benchmark: prints one JSON line.

Times, with CUDA events, (1) the library's DCL train step (DCLTrainer.batch_training: forward, DCLLoss, backward, SGD) at
448x448 on 8 source images (16 rows), eager and with CUDA-graph replay; (2) the same step for a stock-PyTorch restatement of
the reference's module and loss (torchvision ResNet-50 trunk, nn.Conv2d / AvgPool2d / Linear head, CrossEntropyLoss(0.1) and
L1Loss, torch.optim.SGD) with TF32 allowed, after checking that both give the same outputs on the same weights; (3) the head
forward and backward alone, with the bytes they must move computed from the shapes (x read twice, dx written once) and
reported as a fraction of the H100 SXM's 3.35 TB/s.  The card's name and power limit are read in the same run.

    python tests/bench_dcl.py [--steps 20] [--warmup 5]
"""
import argparse
import json
import os
import sys

import torch
import torch.nn as nn

from benchutil import card, timed

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tests'))


class StockDCL(nn.Module):
    """The reference's module restated on stock PyTorch (model/methods/DCL.py)."""

    def __init__(self, K):
        super().__init__()
        import torchvision
        self.backbone = nn.Sequential(*list(torchvision.models.resnet50().children())[:-2])
        self.Convmask = nn.Conv2d(2048, 1, 1, bias=True)
        self.avgpool2 = nn.AvgPool2d(2, stride=2)
        self.avgpool = nn.AdaptiveAvgPool2d(1)
        self.classifier = nn.Linear(2048, K, bias=False)
        self.classifier_swap = nn.Linear(2048, 2, bias=False)

    def forward(self, x):
        x = self.backbone(x)
        mask = torch.tanh(self.avgpool2(self.Convmask(x))).flatten(1)
        x = self.avgpool(x).flatten(1)
        return [self.classifier(x), self.classifier_swap(x), mask]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    args = ap.parse_args()
    os.environ.setdefault('HAWKEYE_ALLOW_RANDOM_INIT', '1')
    import detgen
    from hawkeye_b200 import examples
    from hawkeye_b200.config import load_config
    from conftest import rel_l2

    n, K = 8, 200
    x = detgen.det((2 * n, 3, 448, 448), 700)
    y = detgen.det_labels(n, K, 701).repeat_interleave(2)
    ys = torch.tensor([1, 0] * n)
    law1 = [(i - 24) / 49 for i in range(49)]
    law = torch.tensor([law1, law1[::-1]] * n).float()
    res = dict(workload=f'DCL train step, ResNet-50 448x448, {n} source images ({2 * n} rows), fp32 params, TF32 MMA',
               **card())

    # ---- library: eager and graph replay --------------------------------------------------------------------------------
    cfg = load_config(os.path.join(REPO, 'configs', 'DCL.yaml'))
    xd, yd, ysd, lawd = x.cuda(), y.cuda(), ys.cuda(), law.cuda()
    batch = (xd, yd, ysd, lawd, ['n'] * n)
    state = None
    for graph in (False, True):
        os.environ['HK_CUDA_GRAPH'] = '1' if graph else '0'
        torch.manual_seed(0)
        tr = examples.DCLTrainer(cfg, dataloaders={})
        tr.model.train()
        if state is None:
            state = {k: v.detach().clone() for k, v in tr.model.state_dict().items()}
        ms = timed(lambda: tr.batch_training(batch), args.steps, args.warmup + (4 if graph else 0))
        res['hk_graph_ms' if graph else 'hk_eager_ms'] = round(ms, 3)
        del tr
    res['hk_graph_img_per_s'] = round(2 * n / res['hk_graph_ms'] * 1e3, 1)

    # ---- stock PyTorch with TF32 allowed, output-for-output check first -------------------------------------------------
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.allow_tf32 = True
    ref = StockDCL(K).cuda().train()
    ref.load_state_dict({k: v for k, v in state.items()}, strict=True)
    os.environ['HK_CUDA_GRAPH'] = '0'
    tr = examples.DCLTrainer(cfg, dataloaders={})
    tr.model.load_state_dict(state)
    tr.model.train()
    with torch.no_grad():
        ours = tr.model(xd)
        theirs = ref(xd)
    res['check_rel_l2'] = {k: float(f'{rel_l2(a.float().cpu(), b.float().cpu()):.2e}')
                           for k, a, b in zip(('logits', 'swap', 'mask'), ours, theirs)}
    del tr
    ce, l1 = nn.CrossEntropyLoss(label_smoothing=0.1), nn.L1Loss()
    opt = torch.optim.SGD([{'params': ref.backbone.parameters(), 'lr': 8e-4},
                           {'params': ref.classifier.parameters(), 'lr': 8e-3},
                           {'params': ref.classifier_swap.parameters(), 'lr': 8e-3},
                           {'params': ref.Convmask.parameters(), 'lr': 8e-3}], momentum=0.9)

    def stock_step():
        out = ref(xd)
        loss = ce(out[0], yd) + ce(out[1], ysd) + l1(out[2], lawd)
        opt.zero_grad()
        loss.backward()
        opt.step()
    res['stock_tf32_ms'] = round(timed(stock_step, args.steps, args.warmup), 3)
    res['speedup_graph_vs_stock'] = round(res['stock_tf32_ms'] / res['hk_graph_ms'], 2)
    del ref, opt

    # ---- the head alone ------------------------------------------------------------------------------------------------
    from hawkeye_b200 import _lib
    N, C, H, W = 2 * n, 2048, 14, 14
    feat = detgen.det((N, C, H, W), 702, positive=True).cuda()
    w = (detgen.det((C,), 703) * 0.02).cuda()
    b = torch.zeros(1, device='cuda')
    pooled, mask = torch.empty(N, C, device='cuda'), torch.empty(N, 49, device='cuda')
    gp, gm = torch.randn(N, C, device='cuda'), torch.randn(N, 49, device='cuda')
    dx, dw, db = torch.empty_like(feat), torch.empty(C, device='cuda'), torch.empty(1, device='cuda')
    ws = torch.empty(_lib.query('hk_dcl_head_workspace_bytes', N, C, H, W), dtype=torch.uint8, device='cuda')

    def head():
        s = _lib.stream_ptr()
        _lib.call('hk_dcl_head_fwd', feat, w, b, pooled, mask, N, C, H, W, ws, ws.numel(), s)
        _lib.call('hk_dcl_head_bwd', feat, w, mask, gp, gm, dx, dw, db, N, C, H, W, ws, ws.numel(), s)
    ms = timed(head, 10 * args.steps, args.warmup)
    nbytes = 3 * feat.numel() * 4
    res['head_fwd_bwd_us'] = round(ms * 1e3, 2)
    res['head_bytes'] = nbytes
    res['head_fraction_of_3.35TBps'] = round(nbytes / (ms * 1e-3) / 3.35e12, 3)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
