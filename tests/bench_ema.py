"""Model EMA benchmark (csrc/ema.cu, engine.ModelEMA).  Prints one JSON line with:
  * the card's name, power limit and maximum SM clock;
  * hk_ema_update (with the counter's increment) over the BCNN VGG-16, ResNet-50 and ResNet-101 parameter sets, timed
    with CUDA events over many launches, against the bytes it must move at least (read the model, read and write the
    average: 12 bytes per fp32 element, 24 per int64 one) as a share of the H100 SXM's 3.35 TB/s;
  * torch's AveragedModel(use_buffers=True) with torchvision's avg_fn and its counter on the device, as torchvision's
    ExponentialMovingAverage builds it, on the same tensors: ms per update (host clock
    around a device synchronise), CUDA kernels per update (torch.profiler) and host synchronisations per update (the
    sync debug mode's warnings);
  * the BCNN VGG-16 448 train step (Trainer.batch_training, batch 32, pinned host inputs, eager as bench.py runs it)
    without the key, with torchvision's defaults (an update every 32 steps) and with an update every step, alternated
    over two rounds, each timed with CUDA events over --steps steps.

    python tests/bench_ema.py [--steps 64] [--warmup 3]
"""
import argparse
import json
import os
import sys
import time
import warnings

import torch
import torch.nn as nn

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tests'))
from benchutil import card, timed  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
B, C, S, K = 32, 3, 448, 200
MODELS = (('bcnn_vgg16', 'BCNN', dict(stage=2)), ('resnet50', 'ResNet50', {}), ('resnet101', 'ResNet101', {}))


class _Mirror(nn.Module):
    """The model's parameters and buffers on a plain module, which AveragedModel deep-copies (tests/test_gpu_ema.py)."""

    def __init__(self, model):
        super().__init__()
        self.p = nn.ParameterList([nn.Parameter(p.detach().clone(), requires_grad=p.requires_grad)
                                   for p in model.parameters()])
        for i, b in enumerate(model.buffers()):
            self.register_buffer(f'b{i}', b.detach().clone())


def averaged_model(model, d):
    """torchvision's ExponentialMovingAverage(model, device, decay): the counter on the device."""
    from torch.optim.swa_utils import AveragedModel
    return AveragedModel(model, device='cuda', avg_fn=lambda a, p, n: d * a + (1 - d) * p, use_buffers=True)


def kernels(name, arch, extra, res):
    import hawkeye_b200 as hb
    from hawkeye_b200 import _lib, engine
    from hawkeye_b200.cfgnode import CfgNode
    from hawkeye_b200.train import model_ema_decay
    torch.manual_seed(0)
    net = hb.MODEL.get(arch)(CfgNode(dict(name=arch, num_classes=K, **extra))).cuda()
    flat = engine.FlatParams(net)
    d = model_ema_decay(0.99998, 32, B, 30)
    ema = engine.ModelEMA(net, flat, d)
    nbytes = sum(3 * t.numel() * t.element_size() for t in ema.model_tensors)
    ema.update()                                                 # the copy; every timed update averages
    n0 = _lib.launch_count()
    ema.update()
    launches = _lib.launch_count() - n0
    ms = timed(ema.update, 200, 20)
    out = dict(tensors=len(list(net.parameters())) + len(list(net.buffers())), segments=ema.nseg,
               elements=sum(t.numel() for t in ema.model_tensors), mb_moved=round(nbytes / 1e6, 1),
               hk_ema_update=dict(ms=round(ms, 4), launches=launches,
                                  share_of_3_35_tb_s=round(nbytes / (ms / 1e3) / HBM_BYTES_PER_S, 3)))
    swap_ms = timed(ema.swap, 200, 20)
    out['hk_ema_swap_ms'] = round(swap_ms, 4)

    mirror = _Mirror(net)
    ref = averaged_model(mirror, d)
    ref.update_parameters(mirror)                                # the copy
    for _ in range(3):
        ref.update_parameters(mirror)
    torch.cuda.synchronize()
    n, t0 = 20, time.perf_counter()
    for _ in range(n):
        ref.update_parameters(mirror)
    torch.cuda.synchronize()
    torch_ms = (time.perf_counter() - t0) * 1e3 / n
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ref.update_parameters(mirror)
        torch.cuda.synchronize()
    kernels_per_update = sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                             and 'Memcpy' not in e.name and 'Memset' not in e.name)
    torch.cuda.set_sync_debug_mode('warn')
    try:
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter('always')
            ref.update_parameters(mirror)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    syncs = sum(1 for w in caught if 'synchroniz' in str(w.message))
    out['torch_averaged_model'] = dict(ms=round(torch_ms, 4), cuda_kernels=kernels_per_update, host_syncs=syncs)
    res[name] = out
    del net, flat, ema, mirror, ref
    torch.cuda.empty_cache()


def step_ms(ema, steps, warmup):
    from hawkeye_b200 import examples
    from hawkeye_b200.cfgnode import CfgNode
    from hawkeye_b200.config import load_config
    cfg = load_config(os.path.join(REPO, 'configs', 'BCNN_S2.yaml'))
    if ema is not None:
        cfg.train['model_ema'] = CfgNode(ema)
    torch.manual_seed(0)
    tr = examples.BCNNTrainer(cfg, dataloaders={})
    assert (tr.ema is None) == (ema is None)
    batch = {'img': torch.randn(B, C, S, S).pin_memory(), 'label': (torch.arange(B) % K).pin_memory()}
    ms = timed(lambda: tr.batch_training(batch), steps, warmup)
    del tr
    torch.cuda.empty_cache()
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=64)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_ema needs a CUDA device')
    os.environ.setdefault('HAWKEYE_ALLOW_RANDOM_INIT', '1')
    os.environ['HK_CUDA_GRAPH'] = '0'
    from hawkeye_b200 import _lib
    _lib.set_precise(0)
    res = dict(card())
    for name, arch, extra in MODELS:
        kernels(name, arch, extra, res)
    settings = {'without_key': None, 'defaults_every_32': {}, 'every_step': dict(steps=1)}
    rounds = {k: [] for k in settings}
    for _ in range(2):
        for k, ema in settings.items():
            rounds[k].append(round(step_ms(ema, args.steps, args.warmup), 3))
    res['bcnn_step_ms'] = dict(rounds, steps=args.steps, batch=B, size=S)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
