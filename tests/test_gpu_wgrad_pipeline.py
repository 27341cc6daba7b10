"""3x3 conv weight / bias gradient vs fp64 conv2d autograd at the edges of the weight gradient's two-deep wgmma pipeline:
CTAs that get exactly 1, 2, 3 and 4 stages on every pixel tile (prologue, drain, the stage ring wrapping while the
second fragment buffer is in flight), two accumulating calls in a row, the bias gradient summed by four producer warps
on grids of 2 and 4 ci tiles, and the ResNet 7x7 and 14x14 maps.  dw and db sit between guard regions."""
import pytest
import torch

from conftest import rel_l2
from test_gpu_wgrad_swap import _inputs, _reference, _run

pytestmark = pytest.mark.gpu


def _pick_tile(W, H):
    """pick_wgrad_tile in conv.cu"""
    tw = next((c for c in (16, 8) if W % c == 0), 8 if W <= 8 else 16)
    th = 1
    while th * 2 * tw <= 64 and H % (th * 2) == 0:
        th *= 2
    tn = 64 // (tw * th)
    if (th * tw) % 8 or (th + 2) * (tw + 2) * tn > 120:
        th, tn = 64 // tw, 1
    return tw, th, tn


def _stages_per_cta(N, H, W, cin, cout):
    """launch_wgrad in conv.cu: the pixel tile and `per`, the pixel tiles (pipeline stages) of a split-K CTA"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tw, th, tn = _pick_tile(W, H)
    total = -(-W // tw) * -(-H // th) * -(-N // tn)
    out_tiles = -(-cout // 64) * -(-cin // 64)
    ks, best = 1, -1.0
    for w in (1, 2, 3):
        k = min(max(sms * w // out_tiles, 1), total)
        ctas = k * out_tiles
        fill = ctas / (-(-ctas // sms) * sms)
        if fill > best + 1e-9:
            best, ks = fill, k
    ks = max(1, min(ks, total, 65535))
    return (tw, th, tn), -(-total // ks)


def _check(N, H, W, cin, cout, seed):
    x, dy = _inputs(N, H, W, cin, cout, seed)
    gw, gb = _reference(x, dy)
    dw, db, ok = _run(x, dy)
    ew, eb = rel_l2(dw.double(), gw), rel_l2(db.double(), gb)
    print(f'wgrad N={N} {H}x{W} {cin}->{cout}: dw {ew:.2e} db {eb:.2e}')
    assert ok and ew < 2e-3 and eb < 1e-3


# (tile, stages per CTA, N, H, W); 512 x 512 channels make 64 output tiles, so the split is 2 on a 132-SM H100
STAGE_CASES = [
    ((16, 4, 1), 1, 1, 4, 32), ((16, 4, 1), 2, 1, 8, 32), ((16, 4, 1), 3, 1, 8, 48), ((16, 4, 1), 4, 1, 16, 32),
    ((8, 8, 1), 1, 1, 16, 8), ((8, 8, 1), 2, 1, 32, 8), ((8, 8, 1), 3, 1, 16, 24), ((8, 8, 1), 4, 4, 16, 8),
    ((8, 4, 2), 1, 4, 4, 8), ((8, 4, 2), 2, 8, 4, 8), ((8, 4, 2), 3, 4, 12, 8), ((8, 4, 2), 4, 15, 4, 8),
]


@pytest.mark.parametrize('tile,stages,N,H,W', STAGE_CASES)
def test_wgrad_stages_per_cta(tile, stages, N, H, W):
    assert _stages_per_cta(N, H, W, 512, 512) == (tile, stages)
    _check(N, H, W, 512, 512, seed=N * 100 + H + W)


def test_wgrad_accumulate_twice():
    N, H, W, cin, cout = 2, 24, 32, 128, 64
    x, dy = _inputs(N, H, W, cin, cout, seed=7)
    x2, dy2 = _inputs(N, H, W, cin, cout, seed=8)
    gw, gb = _reference(x, dy)
    gw2, gb2 = _reference(x2, dy2)
    g = torch.Generator(device='cuda').manual_seed(9)
    dw0 = torch.randn(cout, cin, 3, 3, device='cuda', generator=g) * gw.abs().mean().float()
    db0 = torch.randn(cout, device='cuda', generator=g) * gb.abs().mean().float()
    dw1, db1, ok1 = _run(x, dy, dw0, db0, accumulate=True)
    dw2, db2, ok2 = _run(x2, dy2, dw1, db1, accumulate=True)
    ew = rel_l2(dw2.double(), dw0.double() + gw + gw2)
    eb = rel_l2(db2.double(), db0.double() + gb + gb2)
    print(f'wgrad accumulate twice: dw {ew:.2e} db {eb:.2e}')
    assert ok1 and ok2 and ew < 2e-3 and eb < 1e-3


@pytest.mark.parametrize('cin', [128, 256])
def test_wgrad_bias_ci_tiles(cin):
    """only the ci-tile-0 CTAs add the bias gradient; each of the four producer warps adds its own part"""
    _check(3, 16, 24, cin, 96, seed=cin)


@pytest.mark.parametrize('H,c', [(7, 512), (14, 256)])
def test_wgrad_resnet_small_maps(H, c):
    _check(8, H, H, c, c, seed=H)
