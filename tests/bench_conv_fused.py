"""Fused backward entries of the VGG-16 3x3 convolutions against the launches they replace (not a pytest file).

  python tests/bench_conv_fused.py [--out DIR] [--min-ms 200]    CUDA-event timing, at the batch-32 train shapes, of
        conv1_2's data gradient with conv1_1's weight gradient (hk_conv3x3_dgrad_first_wgrad_acc against
        hk_conv3x3_dgrad + hk_conv3x3_first_wgrad_direct_acc), and of the data gradient of conv2_1, conv3_1 and conv4_1
        into the unpooled map (hk_conv3x3_dgrad_unpool against hk_conv3x3_dgrad + hk_maxpool2x2_bwd_idx)

The table is printed; --out DIR also writes it there as JSON.  Both sides of each row run in the in-tree build.
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


def fused(args):
    from hawkeye_b200 import _lib
    _lib.set_precise(0)
    s = _lib.stream_ptr()
    dev = torch.device('cuda')
    g = torch.Generator(device=dev).manual_seed(0)
    N, rows = BATCH, []
    print(f'{"layer":8s} {"map":>4s} {"Cin":>4s} {"Cout":>4s} | {"fused ms":>8s} {"unfused ms":>10s} {"saved":>6s}  unfused pair',
          flush=True)
    for name, H, cin, cout, _ in VGG16_LAYERS:
        W = H
        if name not in ('conv1_2', 'conv2_1', 'conv3_1', 'conv4_1'):
            continue
        dy = torch.randn(N, H, W, cout, device=dev, generator=g)
        w = torch.randn(cout, cin, 3, 3, device=dev, generator=g) * (2.0 / (9 * cin)) ** 0.5
        wf = torch.empty(9 * cout * cin, device=dev)
        wd = torch.empty(9 * cout * cin, device=dev)
        _lib.call('hk_conv3x3_pack_weights', w, wf, wd, cout, cin, s)
        dx = torch.empty(N, H, W, cin, device=dev)
        if name == 'conv1_2':
            img = torch.randn(N, 3, H, W, device=dev, generator=g)
            mask = torch.relu(torch.randn(N, H, W, cin, device=dev, generator=g))
            dw1 = torch.zeros(cin, 3, 3, 3, device=dev)
            db1 = torch.zeros(cin, device=dev)
            nbf = _lib.query('hk_conv3x3_dgrad_first_wgrad_workspace_bytes')
            nbd = _lib.query('hk_conv3x3_first_wgrad_direct_workspace_bytes')
            wsf = torch.empty(nbf, dtype=torch.uint8, device=dev)
            wsd = torch.empty(nbd, dtype=torch.uint8, device=dev)
            pair = 'hk_conv3x3_dgrad + hk_conv3x3_first_wgrad_direct_acc'

            def fused_call():
                _lib.call('hk_conv3x3_dgrad_first_wgrad_acc', dy, wd, mask, img, dw1, db1, N, H, W, cin, cout, wsf, nbf, 1,
                          s)

            def unfused_call():
                _lib.call('hk_conv3x3_dgrad', dy, wd, mask, dx, N, H, W, cin, cout, s)
                _lib.call('hk_conv3x3_first_wgrad_direct_acc', img, dx, dw1, db1, N, H, W, cin, wsd, nbd, 1, s)
        else:
            # the pool in front of this layer: its code from a real pooled map, its input twice the size
            pre = torch.relu(torch.randn(N, 2 * H, 2 * W, cin, device=dev, generator=g))
            pooled = torch.empty(N, H, W, cin, device=dev)
            code = torch.empty(N, H, W, cin, device=dev, dtype=torch.uint8)
            _lib.call('hk_maxpool2x2_fwd_idx', pre, pooled, code, N, 2 * H, 2 * W, cin, 0, s)
            del pooled
            full = pre
            pair = 'hk_conv3x3_dgrad + hk_maxpool2x2_bwd_idx'

            def fused_call():
                _lib.call('hk_conv3x3_dgrad_unpool', dy, wd, code, full, N, H, W, cin, cout, s)

            def unfused_call():
                _lib.call('hk_conv3x3_dgrad', dy, wd, None, dx, N, H, W, cin, cout, s)
                _lib.call('hk_maxpool2x2_bwd_idx', code, dx, full, N, 2 * H, 2 * W, cin, 0, s)
        tf, tu = time_call(fused_call, args.min_ms), time_call(unfused_call, args.min_ms)
        rows.append(dict(layer=name, N=N, H=H, W=W, Cin=cin, Cout=cout, fused_ms=tf, unfused_ms=tu, unfused=pair))
        print(f'{name:8s} {H:4d} {cin:4d} {cout:4d} | {tf:8.3f} {tu:10.3f} {tu - tf:6.3f}  {pair}', flush=True)
        torch.cuda.empty_cache()
    print(f'total ms: fused {sum(r["fused_ms"] for r in rows):.3f}  unfused {sum(r["unfused_ms"] for r in rows):.3f}',
          flush=True)
    return dict(layers=rows)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None, help='directory for the JSON result file (default: print only)')
    ap.add_argument('--min-ms', type=float, default=200.0, help='timed window per shape and call')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_conv_fused: no CUDA device')
    from hawkeye_b200 import _lib
    print(device_line(), flush=True)
    print(f'library: {_lib.LIB_PATH}', flush=True)
    res = fused(args)
    if not args.out:
        return
    os.makedirs(args.out, exist_ok=True)
    res.update(device=device_line(), lib=_lib.LIB_PATH)
    with open(os.path.join(args.out, 'bench_conv_fused.json'), 'w') as f:
        json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
