"""AP-CNN benchmark: prints one JSON line.

Times, with CUDA events, at 448x448 and batch 16 (the shipped yaml), random-initialised trunk: (1) the library's training
step (APCNNTrainer.batch_training: both stages, APCNNLoss, backward, SGD), eager and with CUDA-graph replay; (2) everything
after the trunk alone on fixed layer2 / layer3 / layer4 maps (pyramid, attention, heads for both stages, ROI selection,
refinement, loss and backward); (3) each new kernel family over many launches, with the bytes it must move computed from the
shapes and the share of the H100's 3.35 TB/s of HBM bandwidth that gives (all of them are bandwidth-bound).  The card's name
and power limit are read in the same run.  A stock-PyTorch restatement of the reference is not part of this script.

    python tests/bench_apcnn.py [--steps 20] [--warmup 5] [--batch 16] [--image 448]
"""
import argparse
import json
import os
import sys

import torch

from benchutil import card, timed

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tests'))
HBM_BYTES_PER_S = 3.35e12        # H100 SXM data sheet


def kernel_bytes(N, H3, C2=512):
    """bytes each kernel family has to move at least once, from the shapes (fp32): {name: bytes}"""
    out = {}
    for l, name in enumerate(('3', '4', '5')):
        P = N * (H3 >> l) ** 2
        out[f'att_fwd_level{name}'] = 4 * P * 256                   # one read of F (gates and pooled vectors are small)
        out[f'att_bwd_level{name}'] = 4 * P * 256 * 2               # one read of F, one write of dF
    P4 = N * (H3 // 2) ** 2
    out['lateral_fwd_level3'] = 4 * (P4 * 256 + 2 * 4 * P4 * 256)    # top, lat, out
    out['lateral_bwd_level3'] = 4 * (4 * P4 * 256 + P4 * 256)        # dout, dtop
    out['refine_fwd'] = 4 * N * H3 * H3 * C2 * 2                     # at most one read of x2, one write
    out['refine_bwd'] = 4 * N * H3 * H3 * C2 * 2
    out['roi'] = 4 * N * (H3 * H3 + H3 * H3 // 4 + H3 * H3 // 16)
    return out


def bench_kernels(N, image, steps, warmup):
    from hawkeye_b200 import ops_apcnn
    H3 = image // 8
    need = kernel_bytes(N, H3)
    res = {}

    def report(name, ms):
        res[name] = dict(ms=round(ms, 4), bytes=need[name], hbm_share=round(need[name] / (ms * 1e-3) / HBM_BYTES_PER_S, 3))

    conv = torch.nn.ConvTranspose2d(256, 1, 3, 1, 1).cuda()
    gates = []
    for l, name in enumerate(('3', '4', '5')):
        h = H3 >> l
        Fm = torch.randn(N, h, h, 256, device='cuda', requires_grad=True)
        report(f'att_fwd_level{name}', timed(lambda: ops_apcnn.AttentionFn.apply(Fm.detach(), conv.weight.detach(), conv.bias.detach()),
                                             steps, warmup))
        g, pf, psf = ops_apcnn.AttentionFn.apply(Fm, conv.weight, conv.bias)
        gates.append(g.detach())
        loss = pf.sum() + psf.sum()
        both = timed(lambda: torch.autograd.grad(loss, (Fm, conv.weight), retain_graph=True), steps, warmup)
        report(f'att_bwd_level{name}', both)
    top = torch.randn(N, H3 // 2, H3 // 2, 256, device='cuda', requires_grad=True)
    lat = torch.randn(N, H3, H3, 256, device='cuda', requires_grad=True)
    report('lateral_fwd_level3', timed(lambda: ops_apcnn.LateralFn.apply(top.detach(), lat.detach()), steps, warmup))
    out = ops_apcnn.LateralFn.apply(top, lat)
    g = torch.randn_like(out)
    report('lateral_bwd_level3', timed(lambda: torch.autograd.grad(out, (top, lat), g, retain_graph=True), steps, warmup))
    win = torch.from_numpy(ops_apcnn.central_windows(H3, H3, 200))
    keep = torch.from_numpy(ops_apcnn.suppression_table()).cuda()
    report('roi', timed(lambda: ops_apcnn.roi_select(gates, win, keep, image, image), steps, warmup))
    boxes, counts = ops_apcnn.roi_select(gates, win, keep, image, image)
    x2 = torch.randn(N, H3, H3, 512, device='cuda', requires_grad=True)
    draws = torch.rand(N, 2, device='cuda')
    report('refine_fwd', timed(lambda: ops_apcnn.RefineFn.apply(x2.detach(), boxes, counts, draws), steps, warmup))
    y = ops_apcnn.RefineFn.apply(x2, boxes, counts, draws)
    gy = torch.randn_like(y)
    report('refine_bwd', timed(lambda: torch.autograd.grad(y, x2, gy, retain_graph=True), steps, warmup))
    return res


def bench_head(net, N, image, steps, warmup):
    """both stages' pyramid, attention and heads, the ROI selection, the refinement, the loss and the backward on fixed maps"""
    from hawkeye_b200 import ops_apcnn, ops_resnet
    from hawkeye_b200.losses import APCNNLoss
    H3 = image // 8
    maps = [torch.randn(N, H3 >> l, H3 >> l, 512 << l, device='cuda').relu().requires_grad_(True) for l in range(3)]
    labels = torch.randint(0, 200, (N,), device='cuda')
    crit = APCNNLoss()
    win = torch.from_numpy(ops_apcnn.central_windows(H3, H3, 200))
    real = ops_resnet.block_stack
    state = {'i': 0}

    def fixed(x, blocks, training):          # layer3 / layer4 replaced by the fixed maps: the trunk is not what is timed
        state['i'] += 1
        return maps[1] if state['i'] % 2 else maps[2]

    def step():
        ops_resnet.block_stack = fixed
        try:
            outs1, gates = net.stage(maps[0])
            boxes, counts = ops_apcnn.roi_select(gates, win, net.nms_keep, image, image)
            x2c = ops_apcnn.RefineFn.apply(maps[0], boxes, counts, torch.rand(N, 2, device='cuda'))
            outs2, _ = net.stage(x2c)
        finally:
            ops_resnet.block_stack = real
        out_list = outs1 + outs2
        crit((torch.stack(out_list).mean(0), out_list), labels).backward()
        for p in net.parameters():
            p.grad = None

    return timed(step, steps, warmup)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--batch', type=int, default=16)
    ap.add_argument('--image', type=int, default=448)
    args = ap.parse_args()
    result = dict(bench='apcnn', batch=args.batch, image=args.image, kernel_bytes=kernel_bytes(args.batch, args.image // 8))
    if not torch.cuda.is_available():
        raise SystemExit('bench_apcnn: no CUDA device; nothing is measured without one: ' + json.dumps(result))
    os.environ['HAWKEYE_ALLOW_RANDOM_INIT'] = '1'
    from hawkeye_b200 import _lib, examples
    from hawkeye_b200.config import load_config
    result.update(card())
    data = dict(img=torch.randn(args.batch, 3, args.image, args.image, device='cuda'),
                label=torch.randint(0, 200, (args.batch,), device='cuda'))
    cfg = load_config(os.path.join(REPO, 'configs', 'APCNN.yaml'))
    for mode, env in (('eager', '0'), ('graph', '1')):
        os.environ['HK_CUDA_GRAPH'] = env
        tr = examples.APCNNTrainer(cfg, dataloaders={})
        tr.on_start_epoch(None)
        result[f'step_ms_{mode}'] = round(timed(lambda: tr.batch_training(data), args.steps, max(args.warmup, 6)), 3)
        if mode == 'graph':
            result['graph_kernels'] = tr._graph['kernels']
            _lib.reset_launch_count()
        net = tr.model
        del tr
    del os.environ['HK_CUDA_GRAPH']
    result['head_alone_ms'] = round(bench_head(net, args.batch, args.image, args.steps, args.warmup), 3)
    del net
    torch.cuda.empty_cache()
    result['kernels'] = bench_kernels(args.batch, args.image, max(args.steps, 50), args.warmup)
    result['stock_pytorch_step_ms'] = 'not measured'
    print(json.dumps(result))


if __name__ == '__main__':
    main()
