"""3x3 conv weight / bias gradient (hk_conv3x3_wgrad_acc) vs fp64 torch.nn.functional.conv2d autograd on the GPU, at the
VGG-16 448x448 layer shapes, the ResNet map sizes, partial output-channel tiles, accumulation and the 3xTF32 mode."""
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_l2

pytestmark = pytest.mark.gpu


def _wgrad(x, dy, dw, db, accumulate):
    from hawkeye_b200 import _lib
    N, H, W, cin = x.shape
    cout = dy.shape[-1]
    nb = _lib.query('hk_conv3x3_wgrad_workspace_bytes', cin, cout)
    ws = torch.empty(nb, dtype=torch.uint8, device='cuda')
    _lib.call('hk_conv3x3_wgrad_acc', x, dy, dw, db, N, H, W, cin, cout, ws, nb, int(accumulate), _lib.stream_ptr())
    torch.cuda.synchronize()


def _case(N, H, W, cin, cout, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    x = torch.relu(torch.randn(N, H, W, cin, device='cuda', generator=g))
    dy = torch.randn(N, H, W, cout, device='cuda', generator=g)
    xd = x.double().permute(0, 3, 1, 2)
    wd = torch.zeros(cout, cin, 3, 3, dtype=torch.float64, device='cuda', requires_grad=True)
    bd = torch.zeros(cout, dtype=torch.float64, device='cuda', requires_grad=True)
    y = F.conv2d(xd, wd, bd, padding=1)
    gw, gb = torch.autograd.grad(y, (wd, bd), dy.double().permute(0, 3, 1, 2))
    return x, dy, gw, gb


def _check(N, H, W, cin, cout, seed=0, tol_w=2e-3, tol_b=1e-3):
    x, dy, gw, gb = _case(N, H, W, cin, cout, seed)
    dw = torch.full((cout, cin, 3, 3), float('nan'), device='cuda')
    db = torch.full((cout,), float('nan'), device='cuda')
    _wgrad(x, dy, dw, db, accumulate=False)
    ew, eb = rel_l2(dw.double(), gw), rel_l2(db.double(), gb)
    print(f'wgrad N={N} {H}x{W} {cin}->{cout}: dw {ew:.2e} db {eb:.2e}')
    assert ew < tol_w and eb < tol_b


# every distinct VGG-16 (Cin, Cout, map) of the 448x448 network
@pytest.mark.parametrize('H,cin,cout', [(448, 64, 64), (224, 64, 128), (224, 128, 128), (112, 128, 256), (112, 256, 256),
                                        (56, 256, 512), (56, 512, 512), (28, 512, 512)])
def test_wgrad_vgg16_layers(H, cin, cout):
    _check(2, H, H, cin, cout)


def test_wgrad_conv5_batch32():
    """the batch of the train step: the split-K count of the production launch"""
    _check(32, 28, 28, 512, 512)


@pytest.mark.parametrize('cout', [96, 160])
def test_wgrad_partial_cout_tile(cout):
    _check(2, 24, 24, 64, cout)


@pytest.mark.parametrize('H,c', [(56, 64), (28, 128), (14, 256), (7, 512)])
def test_wgrad_resnet_maps(H, c):
    _check(4, H, H, c, c)


def test_wgrad_accumulate():
    N, H, W, cin, cout = 2, 32, 32, 128, 128
    x, dy, gw, gb = _case(N, H, W, cin, cout, 5)
    g = torch.Generator(device='cuda').manual_seed(6)
    dw0 = torch.randn(cout, cin, 3, 3, device='cuda', generator=g) * gw.abs().mean().float()
    db0 = torch.randn(cout, device='cuda', generator=g) * gb.abs().mean().float()
    dw, db = dw0.clone(), db0.clone()
    _wgrad(x, dy, dw, db, accumulate=True)
    ew, eb = rel_l2(dw.double(), dw0.double() + gw), rel_l2(db.double(), db0.double() + gb)
    print(f'wgrad accumulate: dw {ew:.2e} db {eb:.2e}')
    assert ew < 2e-3 and eb < 1e-3


def test_wgrad_precise():
    from hawkeye_b200 import _lib
    _lib.set_precise(1)
    try:
        _check(2, 28, 28, 128, 64, tol_w=1e-5, tol_b=1e-5)
    finally:
        _lib.set_precise(0)
