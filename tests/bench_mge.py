"""MGE-CNN benchmark: prints one JSON line.

Times, with CUDA events, random-initialised trunks, at 224x224 batch 4 (the shipped yaml) and at 448x448 batch 16:
(1) the library's training step (MGE_CNNTrainer.batch_training: four trunks, two CAM boxes and crops, MGECNNLoss, backward,
Adam), eager and with CUDA-graph replay; (2) a stock-PyTorch restatement of the reference's step (torchvision ResNet-50
trunks on cuDNN with TF32, GradCam as an autograd backward inside the forward, get_bbox's per-image loop with nonzero()
and F.interpolate), with the host synchronisations of one of its steps counted by torch's sync debug mode; (3) everything
after the trunks alone, on fixed layer3 / layer4 maps; (4) each new kernel over many launches, with the bytes it must move
computed from the shapes and the share of the H100's 3.35 TB/s of HBM bandwidth that gives.  The card's name and power
limit are read in the same run.

    python tests/bench_mge.py [--steps 10] [--warmup 3] [--sizes 224x4,448x16]
"""
import argparse
import json
import os
import sys
import warnings

import torch
import torch.nn as nn
import torch.nn.functional as F

from benchutil import card, timed

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tests'))
HBM_BYTES_PER_S = 3.35e12        # H100 SXM data sheet
K = 200


# ---- the stock-PyTorch restatement of the reference (MGE.py, grad_cam.py, Examples/MGE_CNN.py) ------------------------------
class StockMGE(nn.Module):
    def __init__(self, image_size, box_thred=0.2):
        super().__init__()
        import copy
        import torchvision
        base = torchvision.models.resnet50()
        kids = list(base.children())
        self.S, self.rate = image_size, box_thred
        self.conv4, self.conv5 = nn.Sequential(*kids[:-3]), nn.Sequential(*kids[-3])
        self.classifier = nn.Linear(2048, K)
        for b in ('_box', '_box_2', '_gate'):
            setattr(self, 'conv4' + b, copy.deepcopy(self.conv4))
            setattr(self, 'conv5' + b, copy.deepcopy(self.conv5))
        self.classifier_box, self.classifier_box_2 = nn.Linear(2048, K), nn.Linear(2048, K)
        for s in ('', '_1', '_2'):
            setattr(self, 'conv6' + s, nn.Conv2d(1024, 10 * K, 1, 1, 1))
            setattr(self, 'cls_part' + s, nn.Linear(10 * K, K))
            setattr(self, 'cls_cat' + s, nn.Linear(2048 + 10 * K, K))
        self.cls_gate = nn.Sequential(nn.Linear(2048, 512), nn.Linear(512, 3))

    def gradcam(self, c4, conv5):
        was = self.training
        self.eval()
        with torch.enable_grad():
            c4 = c4.detach().requires_grad_(True)
            c5 = conv5(c4)
            out = self.classifier(c5.mean((2, 3)))
            idx = out.argmax(-1)
            g, = torch.autograd.grad(out.gather(1, idx[:, None]).sum(), c5)
        self.train(was)
        return F.relu(g).mean((2, 3))

    def get_bbox(self, x, conv5, w):
        S = self.S
        cam = (conv5.detach() * w[:, :, None, None]).sum(1, keepdim=True)
        m = F.interpolate(cam, size=(S, S), mode='bilinear', align_corners=True).flatten(1)
        lo, hi = m.min(-1, keepdim=True)[0], m.max(-1, keepdim=True)[0]
        mask = torch.sign(torch.sign((m - lo) / (hi - lo) - self.rate) + 1).view(-1, 1, S, S)
        out = torch.zeros_like(x)
        for k in range(x.size(0)):
            ind = mask[k].nonzero()
            y1, x1 = ind.min(0)[0][-2:]
            y2, x2 = ind.max(0)[0][-2:]
            t = x[k, :, y1:y2, x1:x2] if not (x1 == x2 or y1 == y2) else x[k]
            out[k] = F.interpolate(t[None], size=(S, S), mode='bilinear', align_corners=True)[0].detach()
        return out

    def expert(self, c4, pool, s):
        p6 = F.adaptive_max_pool2d(F.relu(getattr(self, 'conv6' + s)(c4.detach())), 1).flatten(1)
        cat = torch.cat([10 * F.normalize(pool.detach(), dim=1, eps=0), 10 * F.normalize(p6.detach(), dim=1, eps=0)], 1)
        return getattr(self, 'cls_part' + s)(p6), getattr(self, 'cls_cat' + s)(cat)

    def forward(self, x):
        c4 = self.conv4(x)
        c5 = self.conv5(c4)
        pool = c5.mean((2, 3))
        out = [self.classifier(pool), *self.expert(c4, pool, '')]
        xb = self.get_bbox(x, c5, self.gradcam(c4, self.conv5))
        c4b = self.conv4_box(xb)
        c5b = self.conv5_box(c4b)
        pb = c5b.mean((2, 3))
        out += [self.classifier_box(pb), *self.expert(c4b, pb, '_1')]
        xb2 = self.get_bbox(xb, c5b, self.gradcam(c4b, self.conv5_box))
        c4b2 = self.conv4_box_2(xb2)
        pb2 = self.conv5_box_2(c4b2).mean((2, 3))
        out += [self.classifier_box_2(pb2), *self.expert(c4b2, pb2, '_2')]
        pr = F.softmax(self.cls_gate(self.conv5_gate(self.conv4_gate(x)).mean((2, 3))), 1)
        cats = torch.stack([out[2].detach(), out[5].detach(), out[8].detach()], -1)
        return out + [(cats * pr[:, None]).sum(-1)]


def stock_step(N, image, steps, warmup):
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = True
    torch.backends.cudnn.benchmark = True
    net = StockMGE(image).cuda().train()
    opt = torch.optim.Adam(net.parameters(), lr=4e-4, weight_decay=2e-5)
    crit = nn.CrossEntropyLoss(label_smoothing=0.1)
    x = torch.randn(N, 3, image, image, device='cuda')
    y = torch.randint(0, K, (N,), device='cuda')

    def step():
        logits = net(x)
        loss = sum(crit(l, y) for l in logits) / len(logits)
        opt.zero_grad()
        loss.backward()
        opt.step()

    ms = timed(step, steps, warmup)
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter('always')
        torch.cuda.set_sync_debug_mode('warn')
        try:
            step()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    syncs = sum('synchroniz' in str(m.message) for m in w)
    del net, opt
    torch.cuda.empty_cache()
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    return round(ms, 3), syncs


def bench_heads(net, N, image, steps, warmup):
    """everything after the trunks: part heads, CAM index passes' classifier, boxes, crops, gate, loss and backward on fixed
    layer3 / layer4 maps (the trunks are replaced; the eval-mode layer4 recompute is replaced too)"""
    from hawkeye_b200 import ops_resnet
    from hawkeye_b200.losses import MGECNNLoss
    from hawkeye_b200.ops import NHWCMeanFn
    h = image // 32
    c4 = torch.randn(N, 2 * h, 2 * h, 1024, device='cuda').relu()
    c5 = torch.randn(N, h, h, 2048, device='cuda').relu().requires_grad_(True)
    x = torch.randn(N, 3, image, image, device='cuda')
    labels = torch.randint(0, K, (N,), device='cuda')
    crit = MGECNNLoss()
    real_trunk, real_stack = net.trunk, ops_resnet.block_stack

    def step():
        net.trunk = lambda img, b: (c4, c5, NHWCMeanFn.apply(c5))
        ops_resnet.block_stack = lambda a, blocks, training: c5.detach()
        try:
            out = net(x)
        finally:
            net.trunk, ops_resnet.block_stack = real_trunk, real_stack
        crit(out, labels).backward()
        for p in net.parameters():
            p.grad = None

    return timed(step, steps, warmup)


def bench_kernels(N, image, steps, warmup):
    from hawkeye_b200 import ops_mge
    h = image // 32
    H, O = 2 * h, 10 * K
    res = {}

    def report(name, ms, nbytes):
        res[name] = dict(ms=round(ms, 4), bytes=nbytes, hbm_share=round(nbytes / (ms * 1e-3) / HBM_BYTES_PER_S, 3))

    x = torch.randn(N, H, H, 1024, device='cuda').relu()
    conv = nn.Conv2d(1024, O, 1, 1, 1).cuda()
    P = N * H * H
    # the GEMM's product goes through memory once (written, then read by the max): x, w, product twice, outputs
    report('part_fwd', timed(lambda: ops_mge.part(x, conv), steps, warmup), 4 * (P * 1024 + O * 1024 + 2 * P * O + 2 * N * O))
    pooled, _ = ops_mge.part(x, conv)
    g = torch.randn_like(pooled)
    report('part_bwd', timed(lambda: torch.autograd.grad(pooled, conv.weight, g, retain_graph=True), steps, warmup),
           4 * (N * O * 1024 + O * 1024 + 3 * N * O))        # one gathered row of x per (image, output), dw written once
    c5 = torch.randn(N, h, h, 2048, device='cuda').relu()
    W = torch.randn(K, 2048, device='cuda')
    logits = torch.randn(N, K, device='cuda')
    report('cam_box', timed(lambda: ops_mge.cam_box(c5, W, image, 0.2, logits=logits), steps, warmup),
           4 * (N * h * h * 2048 + N * 2048 + N * K))
    boxes = ops_mge.cam_box(c5, W, image, 0.2, logits=logits)
    img = torch.randn(N, 3, image, image, device='cuda')
    report('crop', timed(lambda: ops_mge.crop(img, boxes, image), steps, warmup), 4 * 2 * N * 3 * image * image)
    a = torch.randn(N, 2048, device='cuda')
    report('cat_l2n', timed(lambda: ops_mge.cat_l2n(a, pooled), steps, warmup), 4 * 2 * N * (2048 + O))
    hid = torch.randn(N, 512, device='cuda', requires_grad=True)
    lin = nn.Linear(512, 3).cuda()
    cats = [torch.randn(N, K, device='cuda') for _ in range(3)]
    report('gate_fwd', timed(lambda: ops_mge.GateFn.apply(hid.detach(), lin.weight.detach(), lin.bias.detach(), *cats),
                             steps, warmup), 4 * (N * 512 + 4 * N * K))
    out, _ = ops_mge.GateFn.apply(hid, lin.weight, lin.bias, *cats)
    go = torch.randn_like(out)
    report('gate_bwd', timed(lambda: torch.autograd.grad(out, (hid, lin.weight), go, retain_graph=True), steps, warmup),
           4 * (2 * N * 512 + 4 * N * K + 3 * 512))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--sizes', default='224x4,448x16')
    args = ap.parse_args()
    sizes = [tuple(int(v) for v in s.split('x')) for s in args.sizes.split(',')]
    result = dict(bench='mge_cnn', sizes=args.sizes)
    if not torch.cuda.is_available():
        raise SystemExit('bench_mge: no CUDA device; nothing is measured without one: ' + json.dumps(result))
    os.environ['HAWKEYE_ALLOW_RANDOM_INIT'] = '1'
    from hawkeye_b200 import examples
    from hawkeye_b200.config import load_config
    result.update(card())
    cfg = load_config(os.path.join(REPO, 'configs', 'MGE_CNN.yaml'))
    for image, N in sizes:
        r = result[f'{image}x{N}'] = {}
        c = cfg.clone() if hasattr(cfg, 'clone') else cfg
        data = dict(img=torch.randn(N, 3, image, image, device='cuda'), label=torch.randint(0, K, (N,), device='cuda'))
        for mode, env in (('eager', '0'), ('graph', '1')):
            os.environ['HK_CUDA_GRAPH'] = env
            tr = examples.MGE_CNNTrainer(c, dataloaders={})
            if image != tr.model.image_size:
                tr.model.image_size = image
            r[f'step_ms_{mode}'] = round(timed(lambda: tr.batch_training(data), args.steps, max(args.warmup, 5)), 3)
            net = tr.model
            del tr
        del os.environ['HK_CUDA_GRAPH']
        r['heads_alone_ms'] = round(bench_heads(net, N, image, args.steps, args.warmup), 3)
        del net
        torch.cuda.empty_cache()
        r['stock_pytorch_step_ms'], r['stock_pytorch_host_syncs_per_step'] = stock_step(N, image, args.steps, args.warmup)
        r['kernels'] = bench_kernels(N, image, max(args.steps, 30), args.warmup)
        torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == '__main__':
    main()
