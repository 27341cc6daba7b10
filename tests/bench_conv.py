"""VGG-16 3x3 convolution timing on the GPU (not a pytest file).

  python tests/bench_conv.py [--lib PATH] [--out DIR] [--min-ms 200]    per-layer CUDA-event timing of the weight
        gradient (hk_conv3x3_wgrad_acc, accumulate=1 as in training), the forward (hk_conv3x3_fwd, or _fwd_pool where a
        pool follows) and the data gradient (hk_conv3x3_dgrad) at the 12 VGG-16 layer shapes of the 448x448 batch-32
        train step
  python tests/bench_conv.py --profile-step [--lib PATH] [--out DIR]    torch.profiler kernel table over 3 bcnn_s2 train
        steps at batch 32, the trainer built as bench.py builds it

Tables are printed; --out DIR also writes the results there as JSON (and the profile table as text).  --lib loads that
libhawkeye_b200.so instead of the in-tree one (the C ABI is the header's), so two builds can be timed alternately in
separate processes.  TFLOP/s are 2*N*H*W*9*Cin*Cout over kernel time; the share of 495 TFLOP/s is against
NVIDIA's H100 SXM data-sheet dense TF32 figure, not a measured peak.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import torch  # noqa: E402

from benchutil import device_line, time_call  # noqa: E402
from fp64_refs import BATCH, VGG16_LAYERS  # noqa: E402

DATASHEET_TF32 = 495.0


def per_layer(args, out):
    from hawkeye_b200 import _lib
    _lib.set_precise(0)
    s = _lib.stream_ptr()
    dev = torch.device('cuda')
    g = torch.Generator(device=dev).manual_seed(0)
    rows, tot = [], {'wgrad': 0.0, 'fwd': 0.0, 'dgrad': 0.0}
    print(f'{"layer":8s} {"map":>4s} {"Cin":>4s} {"Cout":>4s} {"GFLOP":>7s} | '
          f'{"wgrad ms":>9s} {"TFLOP/s":>7s} {"%ds":>5s} | {"fwd ms":>8s} {"TFLOP/s":>7s} | {"dgrad ms":>8s} {"TFLOP/s":>7s}',
          flush=True)
    for name, H, cin, cout, pool in VGG16_LAYERS:
        N, W = BATCH, H
        x = torch.relu(torch.randn(N, H, W, cin, device=dev, generator=g))
        dy = torch.randn(N, H, W, cout, device=dev, generator=g)
        w = torch.randn(cout, cin, 3, 3, device=dev, generator=g) * (2.0 / (9 * cin)) ** 0.5
        b = torch.zeros(cout, device=dev)
        wf = torch.empty(9 * cout * cin, device=dev)
        wd = torch.empty(9 * cout * cin, device=dev)
        _lib.call('hk_conv3x3_pack_weights', w, wf, wd, cout, cin, s)
        dw = torch.zeros(cout, cin, 3, 3, device=dev)
        db = torch.zeros(cout, device=dev)
        nb = _lib.query('hk_conv3x3_wgrad_workspace_bytes', cin, cout)
        ws = torch.empty(nb, dtype=torch.uint8, device=dev)
        y = torch.empty(N, H, W, cout, device=dev)
        dx = torch.empty(N, H, W, cin, device=dev)
        if pool:
            p = torch.empty(N, H // 2, W // 2, cout, device=dev)
            code = torch.empty(N, H // 2, W // 2, cout, device=dev, dtype=torch.uint8)

            def fwd():
                _lib.call('hk_conv3x3_fwd_pool', x, wf, b, p, code, N, H, W, cin, cout, 0, s)
        else:
            def fwd():
                _lib.call('hk_conv3x3_fwd', x, wf, b, y, N, H, W, cin, cout, 1, s)

        def wgrad():
            _lib.call('hk_conv3x3_wgrad_acc', x, dy, dw, db, N, H, W, cin, cout, ws, nb, 1, s)

        def dgrad():
            _lib.call('hk_conv3x3_dgrad', dy, wd, x, dx, N, H, W, cin, cout, s)

        flop = 2.0 * N * H * W * 9 * cin * cout
        t = {k: time_call(f, args.min_ms) for k, f in (('wgrad', wgrad), ('fwd', fwd), ('dgrad', dgrad))}
        tf = {k: flop / (v * 1e-3) / 1e12 for k, v in t.items()}
        for k in tot:
            tot[k] += t[k]
        rows.append(dict(layer=name, N=N, H=H, W=W, Cin=cin, Cout=cout, gflop=flop / 1e9,
                         **{f'{k}_ms': t[k] for k in t}, **{f'{k}_tflops': tf[k] for k in tf},
                         wgrad_datasheet_share=tf['wgrad'] / DATASHEET_TF32))
        print(f'{name:8s} {H:4d} {cin:4d} {cout:4d} {flop / 1e9:7.1f} | {t["wgrad"]:9.3f} {tf["wgrad"]:7.1f} '
              f'{100 * tf["wgrad"] / DATASHEET_TF32:4.1f}% | {t["fwd"]:8.3f} {tf["fwd"]:7.1f} | {t["dgrad"]:8.3f} '
              f'{tf["dgrad"]:7.1f}', flush=True)
        del x, dy, w, wf, wd, dw, db, ws, y, dx
        torch.cuda.empty_cache()
    print(f'total ms: wgrad {tot["wgrad"]:.3f}  fwd {tot["fwd"]:.3f}  dgrad {tot["dgrad"]:.3f}   '
          f'(% = share of the {DATASHEET_TF32:.0f} TFLOP/s data-sheet dense TF32 rate, not a measured peak)', flush=True)
    return dict(layers=rows, total_ms=tot)


def profile_step(args, out):
    from torch.profiler import ProfilerActivity, profile
    from hawkeye_b200 import examples
    from hawkeye_b200.config import load_config
    os.environ.setdefault('HAWKEYE_ALLOW_RANDOM_INIT', '1')
    os.environ['HK_CUDA_GRAPH'] = '0'
    torch.cuda.set_device(0)
    dev = torch.device('cuda', 0)
    cfg = load_config(os.path.join(ROOT, 'configs', 'BCNN_S2.yaml'))
    torch.manual_seed(0)
    tr = examples.TRAINERS['BCNN'](cfg, dataloaders={})
    tr.model.train()
    gen = torch.Generator().manual_seed(1234)
    x = torch.randn(BATCH, 3, 448, 448, generator=gen).to(dev)
    y = torch.randint(0, 200, (BATCH,), generator=gen).to(dev)

    def step():
        o = tr.model(x)
        loss = tr.criterion(o, y)
        tr.optimizer.zero_grad()
        loss.backward()
        tr.allreduce.finish()
        tr.optimizer.step()

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    steps = 3
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        e0.record()
        for _ in range(steps):
            step()
        e1.record()
        torch.cuda.synchronize()
    step_us = e0.elapsed_time(e1) * 1e3 / steps
    agg = {}
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            a = agg.setdefault(ev.name, [0, 0.0])
            a[0] += 1
            a[1] += ev.time_range.elapsed_us()
    rows = sorted(agg.items(), key=lambda kv: -kv[1][1])
    busy = sum(v[1] for v in agg.values()) / steps
    lines = [f'{steps} bcnn_s2 train steps, batch {BATCH}, 448x448: {step_us / 1e3:.2f} ms per step (profiled, CUDA events); '
             f'kernel time {busy / 1e3:.2f} ms per step',
             f'{"calls/step":>10s} {"us/step":>11s} {"share":>6s}  kernel']
    for name, (calls, us) in rows:
        lines.append(f'{calls / steps:10.1f} {us / steps:11.1f} {100 * us / steps / step_us:5.1f}%  {name[:160]}')
    txt = '\n'.join(lines)
    print(txt, flush=True)
    if out:
        with open(os.path.join(out, 'profile_step.txt'), 'w') as f:
            f.write(txt + '\n')
    return dict(step_ms=step_us / 1e3, kernels=[dict(name=n, calls_per_step=c / steps, us_per_step=u / steps,
                                                     share=u / steps / step_us) for n, (c, u) in rows])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--profile-step', action='store_true')
    ap.add_argument('--lib', default=None, help='libhawkeye_b200.so to load instead of the in-tree build')
    ap.add_argument('--out', default=None, help='directory for the result files (default: print only)')
    ap.add_argument('--tag', default=None, help='name of the JSON result file (default: derived from the mode)')
    ap.add_argument('--min-ms', type=float, default=200.0, help='timed window per shape and kernel')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_conv: no CUDA device')
    from hawkeye_b200 import _lib
    if args.lib:
        _lib.LIB_PATH = os.path.abspath(args.lib)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
    print(device_line(), flush=True)
    print(f'library: {_lib.LIB_PATH}', flush=True)
    res = profile_step(args, args.out) if args.profile_step else per_layer(args, args.out)
    if not args.out:
        return
    res.update(device=device_line(), lib=_lib.LIB_PATH)
    tag = args.tag or ('profile_step' if args.profile_step else 'per_layer')
    with open(os.path.join(args.out, f'bench_conv_{tag}.json'), 'w') as f:
        json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
