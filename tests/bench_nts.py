"""NTS-Net benchmark: prints one JSON line.

Times, with CUDA events, at 224x224 and batches 4 (the shipped yaml) and 16: (1) the library's step
(NTSNetTrainer.batch_training: forward over the images and the B x 6 part crops, NTSLoss, backward, Adam), eager and with
CUDA-graph replay; (2) the same step for a stock-PyTorch restatement of the reference (torchvision's ResNet-50 trunk,
nn.Conv2d proposal net, the scores copied to the host for a numpy greedy NMS, one F.interpolate per part, the list loss
row by row, torch.optim.Adam) with cuDNN / cuBLAS and TF32 allowed; (3) the navigator head alone at batch 16 (proposal net,
NMS, crops, ranking loss and their backward) on a fixed layer4 map.  The card's name and power limit are read in the
same run.

    python tests/bench_nts.py [--steps 20] [--warmup 5]
"""
import argparse
import copy
import json
import os
import sys

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from benchutil import card, timed

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tests'))


def host_nms(scores, anchors, topn):
    """greedy NMS on the host, vectorised over the candidates as the reference's hard_nms is"""
    order = np.argsort(-scores, kind='stable')
    a = anchors[order].astype(np.float64)
    area = (a[:, 2] - a[:, 0]) * (a[:, 3] - a[:, 1])
    alive = np.arange(len(order))
    kept = []
    while len(alive) and len(kept) < topn:
        p = alive[0]
        kept.append(order[p])
        rest = alive[1:]
        dy = np.minimum(a[rest, 2], a[p, 2]) - np.maximum(a[rest, 0], a[p, 0])
        dx = np.minimum(a[rest, 3], a[p, 3]) - np.maximum(a[rest, 1], a[p, 1])
        inter = np.where((dy < 0) | (dx < 0), 0.0, dy * dx)
        alive = rest[inter / (area[rest] + area[p] - inter) < 0.25]
    return np.array(kept, dtype=np.int64)


class StockNTS(nn.Module):
    """NTSNet.py restated on torchvision's ResNet-50 and nn.Conv2d, with its host NMS and interpolate loop."""

    def __init__(self, lib):
        super().__init__()
        import torchvision
        r = torchvision.models.resnet50()
        r.fc = nn.Linear(2048, 200)
        self.pretrained_model = r
        self.proposal_net = copy.deepcopy(lib.proposal_net)
        self.concat_net, self.partcls_net = copy.deepcopy(lib.concat_net), copy.deepcopy(lib.partcls_net)
        self.load_state_dict(lib.state_dict(), strict=False)
        self.anchors = lib.edge_anchors.cpu().numpy()
        self.topN, self.K = lib.topN, lib.CAT_NUM

    def trunk(self, x):
        r = self.pretrained_model
        f = r.layer4(r.layer3(r.layer2(r.layer1(r.maxpool(r.relu(r.bn1(r.conv1(x))))))))
        feat = F.dropout(f.mean((2, 3)), 0.5, True)
        return r.fc(feat), f, feat

    def proposal(self, f):
        p = self.proposal_net
        d1 = F.relu(p.down1(f))
        d2 = F.relu(p.down2(d1))
        d3 = F.relu(p.down3(d2))
        return torch.cat([p.tidy1(d1).flatten(1), p.tidy2(d2).flatten(1), p.tidy3(d3).flatten(1)], 1)

    def forward(self, x):
        B = x.shape[0]
        raw, f, feat = self.trunk(x)
        score = self.proposal(f.detach())
        idx_np = np.stack([host_nms(s, self.anchors, self.topN) for s in score.detach().cpu().numpy()])
        idx = torch.from_numpy(idx_np).cuda()
        prob = score.gather(1, idx)
        xp = F.pad(x, (224, 224, 224, 224))
        parts = torch.zeros(B, self.topN, 3, 224, 224, device=x.device)
        for i in range(B):
            for j in range(self.topN):
                y0, x0, y1, x1 = self.anchors[idx_np[i, j]].tolist()
                parts[i:i + 1, j] = F.interpolate(xp[i:i + 1, :, y0:y1, x0:x1], size=(224, 224), mode='bilinear',
                                                  align_corners=True)
        _, _, pf = self.trunk(parts.view(-1, 3, 224, 224).detach())
        concat = self.concat_net(torch.cat([pf.view(B, self.topN, -1)[:, :self.K].reshape(B, -1), feat], 1))
        return raw, concat, self.partcls_net(pf).view(B, self.topN, -1), idx, prob


def stock_loss(out, labels, T):
    raw, concat, part, _, prob = out
    B = labels.shape[0]
    rows = labels.repeat_interleave(T)
    lsm = F.log_softmax(part.view(B * T, -1), -1)
    L = torch.stack([-lsm[i][rows[i].item()] for i in range(B * T)]).view(B, T)      # NTS_loss.py:33-35
    rank = sum(F.relu((1 - prob[:, i:i + 1] + prob) * (L > L[:, i:i + 1]).float()).sum() for i in range(T)) / B
    ce = nn.CrossEntropyLoss(label_smoothing=0.1)
    return ce(raw, labels) + rank + ce(concat, labels) + ce(part.view(B * T, -1), rows)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_nts needs a CUDA device')
    os.environ.setdefault('HAWKEYE_ALLOW_RANDOM_INIT', '1')
    import detgen
    from hawkeye_b200 import examples, ops_nts
    from hawkeye_b200.config import load_config
    res = dict(bench='nts', image=224, proposals=6, **card())
    cfg0 = load_config(os.path.join(REPO, 'configs', 'NTSNet.yaml'))

    def trainer(graph):
        os.environ['HK_CUDA_GRAPH'] = '1' if graph else '0'
        tr = examples.NTSNetTrainer(load_config(os.path.join(REPO, 'configs', 'NTSNet.yaml')), dataloaders={})
        tr.model.train()
        return tr

    for B in (4, 16):
        data = {'img': detgen.det((B, 3, 224, 224), 3600 + B).pin_memory(),
                'label': detgen.det_labels(B, 200, 3700 + B).pin_memory()}
        tr = trainer(False)
        res[f'b{B}_lib_step_eager_ms'] = timed(lambda: tr.batch_training(data), args.steps, args.warmup)
        del tr
        trg = trainer(True)
        res[f'b{B}_lib_step_graph_ms'] = timed(lambda: trg.batch_training(data), args.steps, max(args.warmup, 5))
        lib_model = trg.model
        del trg
        torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = True
        stock = StockNTS(lib_model).cuda().train()
        opt = torch.optim.Adam(stock.parameters(), lr=cfg0.train.optimizer.lr, weight_decay=cfg0.train.optimizer.weight_decay)
        x, labels = data['img'].cuda(), data['label'].cuda()

        def stock_step():
            loss = stock_loss(stock(x), labels, 6)
            opt.zero_grad()
            loss.backward()
            opt.step()
            loss.item()                                    # Examples/NTSNet.py:48

        res[f'b{B}_stock_step_tf32_ms'] = timed(stock_step, args.steps, args.warmup)
        res[f'b{B}_speedup_graph_vs_stock'] = res[f'b{B}_stock_step_tf32_ms'] / res[f'b{B}_lib_step_graph_ms']

        if B == 16:                       # the navigator head alone on a fixed layer4 map
            with torch.no_grad():
                _, fmap, _ = stock.trunk(x)
            fnhwc = fmap.permute(0, 2, 3, 1).contiguous()
            m = lib_model
            part_logits = torch.randn(B * 6, 200, device='cuda')

            def lib_head():
                _, prob, idx, boxes = m.proposal_net(fnhwc, m.edge_anchors, 6)
                ops_nts.crop(x, boxes)
                ops_nts.RankLossFn.apply(part_logits, labels, prob).backward()

            def stock_head():
                score = stock.proposal(fmap)
                idx_np = np.stack([host_nms(s, stock.anchors, 6) for s in score.detach().cpu().numpy()])
                prob = score.gather(1, torch.from_numpy(idx_np).cuda())
                xp = F.pad(x, (224, 224, 224, 224))
                parts = torch.zeros(B, 6, 3, 224, 224, device=x.device)
                for i in range(B):
                    for j in range(6):
                        y0, x0, y1, x1 = stock.anchors[idx_np[i, j]].tolist()
                        parts[i:i + 1, j] = F.interpolate(xp[i:i + 1, :, y0:y1, x0:x1], size=(224, 224), mode='bilinear',
                                                          align_corners=True)
                rows = labels.repeat_interleave(6)
                lsm = F.log_softmax(part_logits, -1)
                L = torch.stack([-lsm[i][rows[i].item()] for i in range(B * 6)]).view(B, 6)
                rank = sum(F.relu((1 - prob[:, i:i + 1] + prob) * (L > L[:, i:i + 1]).float()).sum() for i in range(6)) / B
                rank.backward()

            res['b16_lib_head_ms'] = timed(lib_head, args.steps, args.warmup)
            res['b16_stock_head_tf32_ms'] = timed(stock_head, args.steps, args.warmup)
        del stock, opt, lib_model
        torch.cuda.empty_cache()
    print(json.dumps({k: (float(f'{v:.4g}') if isinstance(v, float) else v) for k, v in res.items()}))


if __name__ == '__main__':
    main()
