"""Bit-identity digests of the VGG-16 3x3 convolutions on the GPU (not a pytest file).

  python tests/digest_conv.py [--lib PATH] [--out DIR]    SHA-256 of every layer's forward output (hk_conv3x3_fwd with
        ReLU), fused pooled output and pooling code (hk_conv3x3_fwd_pool, where a pool follows) and masked data-gradient
        output (hk_conv3x3_dgrad) at the 12 layer shapes tests/bench_conv.py times, from fixed-seed inputs

--lib loads that libhawkeye_b200.so instead of the in-tree one, so two builds can be run in separate processes: when
their digests match, they compute bit-identical results at the sizes that are timed.  --out DIR also writes the full
digests there as JSON.
"""
import argparse
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import torch  # noqa: E402

from benchutil import device_line  # noqa: E402
from fp64_refs import BATCH, VGG16_LAYERS  # noqa: E402


def sha(t):
    torch.cuda.synchronize()
    return hashlib.sha256(t.contiguous().cpu().numpy().tobytes()).hexdigest()


def digests():
    from hawkeye_b200 import _lib
    _lib.set_precise(0)
    s = _lib.stream_ptr()
    dev = torch.device('cuda')
    rows = []
    for i, (name, H, cin, cout, pool) in enumerate(VGG16_LAYERS):
        N, W = BATCH, H
        g = torch.Generator(device=dev).manual_seed(1000 + i)
        x = torch.relu(torch.randn(N, H, W, cin, device=dev, generator=g))
        dy = torch.randn(N, H, W, cout, device=dev, generator=g)
        w = torch.randn(cout, cin, 3, 3, device=dev, generator=g) * (2.0 / (9 * cin)) ** 0.5
        b = torch.randn(cout, device=dev, generator=g) * 0.1
        wf = torch.empty(9 * cout * cin, device=dev)
        wd = torch.empty(9 * cout * cin, device=dev)
        _lib.call('hk_conv3x3_pack_weights', w, wf, wd, cout, cin, s)
        row = dict(layer=name)
        y = torch.empty(N, H, W, cout, device=dev)
        _lib.call('hk_conv3x3_fwd', x, wf, b, y, N, H, W, cin, cout, 1, s)
        row['fwd'] = sha(y)
        del y
        if pool:
            p = torch.empty(N, H // 2, W // 2, cout, device=dev)
            code = torch.empty(N, H // 2, W // 2, cout, device=dev, dtype=torch.uint8)
            _lib.call('hk_conv3x3_fwd_pool', x, wf, b, p, code, N, H, W, cin, cout, 0, s)
            row['pool'] = sha(p)
            row['code'] = sha(code)
            del p, code
        dx = torch.empty(N, H, W, cin, device=dev)
        _lib.call('hk_conv3x3_dgrad', dy, wd, x, dx, N, H, W, cin, cout, s)   # the ReLU mask is x > 0
        row['dgrad'] = sha(dx)
        rows.append(row)
        print(f'{name:8s} ' + ' '.join(f'{k} {v[:16]}' for k, v in row.items() if k != 'layer'), flush=True)
        del x, dy, w, wf, wd, dx
        torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--lib', default=None, help='libhawkeye_b200.so to load instead of the in-tree build')
    ap.add_argument('--out', default=None, help='directory for the JSON result file (default: print only)')
    ap.add_argument('--tag', default='digest', help='name of the JSON result file')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('digest_conv: no CUDA device')
    from hawkeye_b200 import _lib
    if args.lib:
        _lib.LIB_PATH = os.path.abspath(args.lib)
    print(device_line(), flush=True)
    print(f'library: {_lib.LIB_PATH}', flush=True)
    rows = digests()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, f'digest_conv_{args.tag}.json'), 'w') as f:
            json.dump(dict(layers=rows, device=device_line(), lib=_lib.LIB_PATH), f, indent=1)


if __name__ == '__main__':
    main()
