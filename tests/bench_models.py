"""Throughput of the other benchmark configs (parity-test cases, not the bench line): CBCNN VGG-16 d=8192 and
Fast MPN-COV ResNet-50 at 448x448, batch 32, one GPU: fwd + CE + bwd + SGD, device-timed."""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import hawkeye_b200 as hb
from hawkeye_b200 import engine, ops


class Cfg(dict):
    __getattr__ = dict.__getitem__


def run(name, cfg, B=32, steps=5):
    torch.manual_seed(0)
    net = hb.MODEL.get(name)(cfg).cuda().train()
    flat = engine.FlatParams(net)
    opt = engine.FusedSGD(flat, lr=1e-3, momentum=0.9, weight_decay=1e-5)
    crit = ops.CrossEntropyLS(0.1)
    x = torch.randn(B, 3, 448, 448, device='cuda')
    y = torch.randint(0, 200, (B,), device='cuda')

    def step():
        loss = crit(net(x), y)
        opt.zero_grad()
        loss.backward()
        opt.step()
        return loss
    for _ in range(3):
        loss = step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        loss = step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    return dict(model=name, batch=B, ms_per_step=ms, img_per_s=B / ms * 1e3, loss=float(loss))


out = [run('CBCNN', Cfg(name='CBCNN', stage=2, num_classes=200, input_channel=512, output_channel=8192)),
       run('MPN', Cfg(name='MPN', iter_num=5, is_sqrt=True, is_vec=True, input_dim=2048, dimension_reduction=256,
                      num_classes=200))]
print(json.dumps(out))
