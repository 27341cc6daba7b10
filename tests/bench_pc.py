"""Pairwise Confusion / Baseline training benchmark: prints one JSON line.

Times, with CUDA events, random-initialised weights at the shipped configs' shape (224x224, batch 24, 200 classes):
(1) the library's Baseline step and PairConfusion step (Trainer.batch_training: ResNet-50 trunk, mean pool, fc, the loss,
backward, Adam), eager and with CUDA-graph replay; (2) a stock-PyTorch restatement of the reference's PairConfusion step
(torchvision ResNet-50 on cuDNN with TF32 allowed, the reference's loss ops, torch.optim.Adam over the fc and trunk groups),
with the host synchronisations of one of its steps counted by torch's sync debug mode; (3) the loss alone, forward and
backward on fixed logits, library against the reference's torch ops.  The card's name and power limit are read in the same
run.

    python tests/bench_pc.py [--steps 20] [--warmup 5]
"""
import argparse
import json
import os
import sys

import torch
import torch.nn as nn

from benchutil import card, count_syncs, timed

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tests'))

B, K, LAMBDA = 24, 200, 0.1


def stock_loss(features, labels, lambda_a=LAMBDA):
    """model/loss/pair_confusion.py in torch ops"""
    half = features.size(0) // 2
    loss = torch.norm((features[:half] - features[half:]).abs(), 2, 1)
    loss = loss * (labels[:half] != labels[half:])
    return nn.functional.cross_entropy(features, labels, label_smoothing=0.1) + lambda_a * loss.sum() / float(B)


def stock_step(x, y, steps, warmup, lr=4e-4):
    import torchvision
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = True
    torch.backends.cudnn.benchmark = True
    net = torchvision.models.resnet50(num_classes=K).cuda().train()
    fc = {id(p) for p in net.fc.parameters()}
    opt = torch.optim.Adam([{'params': net.fc.parameters(), 'lr': lr},
                            {'params': [p for p in net.parameters() if id(p) not in fc], 'lr': 0.1 * lr}],
                           weight_decay=2e-5)

    def step():
        loss = stock_loss(net(x), y)
        opt.zero_grad()
        loss.backward()
        opt.step()

    ms = timed(step, steps, warmup)
    syncs = count_syncs(step)
    del net, opt
    torch.cuda.empty_cache()
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    return round(ms, 3), syncs


def loss_alone(fn, y, steps, warmup):
    z = torch.randn(B, K, device='cuda', requires_grad=True)

    def step():
        fn(z, y).backward()
        z.grad = None

    return round(timed(step, steps, warmup), 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    args = ap.parse_args()
    result = dict(bench='pair_confusion', image=224, batch=B, num_classes=K)
    if not torch.cuda.is_available():
        raise SystemExit('bench_pc: no CUDA device; nothing is measured without one: ' + json.dumps(result))
    os.environ['HAWKEYE_ALLOW_RANDOM_INIT'] = '1'
    from hawkeye_b200 import examples
    from hawkeye_b200.cfgnode import CfgNode
    from hawkeye_b200.config import load_config
    from hawkeye_b200.losses import PairwiseConfusionLoss
    result.update(card())
    torch.manual_seed(0)
    x = torch.randn(B, 3, 224, 224, device='cuda')
    y = torch.randint(0, K, (B,), device='cuda')
    data = dict(img=x, label=y)
    for name, cls, yaml in (('baseline', examples.BaselineTrainer, 'Baseline.yaml'),
                            ('pc', examples.PCResNetTrainer, 'PC_resnet50.yaml')):
        cfg = load_config(os.path.join(REPO, 'configs', yaml))
        for mode, env in (('eager', '0'), ('graph', '1')):
            os.environ['HK_CUDA_GRAPH'] = env
            tr = cls(cfg, dataloaders={})
            result[f'{name}_step_ms_{mode}'] = round(timed(lambda: tr.batch_training(data), args.steps,
                                                           max(args.warmup, 5)), 3)
            if mode == 'eager':
                result[f'{name}_host_syncs_per_step'] = count_syncs(lambda: tr.batch_training(data))
            del tr
            torch.cuda.empty_cache()
    del os.environ['HK_CUDA_GRAPH']
    result['stock_pytorch_pc_step_ms'], result['stock_pytorch_pc_host_syncs_per_step'] = stock_step(x, y, args.steps,
                                                                                                    args.warmup)
    crit = PairwiseConfusionLoss(CfgNode(dict(lambda_a=LAMBDA)))
    result['loss_alone_ms'] = loss_alone(crit, y, args.steps, args.warmup)
    result['stock_pytorch_loss_alone_ms'] = loss_alone(stock_loss, y, args.steps, args.warmup)
    print(json.dumps(result))


if __name__ == '__main__':
    main()
