"""VGG backbone kernels (implicit-GEMM conv fwd/dgrad/wgrad, first layer, max-pool) vs torch-CPU fp64 (the
arithmetic the reference's nn.Conv2d / MaxPool2d dispatches to; oracle/hop_oracle.py:vgg_features_fwd)."""
import pytest
import torch
import torch.nn.functional as F

import detgen
from conftest import rel_l2
from kernel_check import nchw, nhwc

pytestmark = pytest.mark.gpu
TOL = 2e-3


@pytest.mark.parametrize('N,H,W,Cin,Cout', [(2, 16, 16, 64, 64), (2, 16, 32, 64, 128), (2, 24, 16, 128, 64), (1, 16, 16, 128, 256),
                                             (3, 8, 8, 128, 256), (8, 28, 28, 64, 128),
                                             (2, 12, 20, 256, 512), (1, 4, 4, 512, 512)])
def test_conv3x3_fwd_dgrad_wgrad(N, H, W, Cin, Cout):
    from hawkeye_b200 import _lib
    s = _lib.stream_ptr()
    x = detgen.det((N, Cin, H, W), 1, positive=True)
    w = detgen.det((Cout, Cin, 3, 3), 2, (2.0 / (Cout * 9)) ** 0.5)
    b = detgen.det((Cout,), 3, 0.1)
    dy = detgen.det((N, Cout, H, W), 4)
    xd, wd_ = x.double().requires_grad_(True), w.double().requires_grad_(True)
    bd = b.double().requires_grad_(True)
    y_ref = F.relu(F.conv2d(xd, wd_, bd, padding=1))
    # our dgrad/wgrad take dy wrt the *pre-activation* (ReLU mask already applied upstream)
    dpre = dy.double() * (y_ref > 0)
    gx, gw, gb = torch.autograd.grad(y_ref, (xd, wd_, bd), dy.double())

    xg, wg, bg = nhwc(x).cuda(), w.cuda(), b.cuda()
    wf = torch.empty(9 * Cout * Cin, device='cuda')
    wdg = torch.empty(9 * Cout * Cin, device='cuda')
    _lib.call('hk_conv3x3_pack_weights', wg, wf, wdg, Cout, Cin, s)
    y = torch.empty(N, H, W, Cout, device='cuda')
    _lib.call('hk_conv3x3_fwd', xg, wf, bg, y, N, H, W, Cin, Cout, 1, s)
    torch.cuda.synchronize()
    e = rel_l2(nchw(y).cpu(), y_ref.detach())
    print(f'conv fwd {N}x{H}x{W} {Cin}->{Cout}: {e:.2e}')
    assert e < TOL
    dpre_g = nhwc(dpre.float()).cuda()
    dx = torch.empty(N, H, W, Cin, device='cuda')
    _lib.call('hk_conv3x3_dgrad', dpre_g, wdg, None, dx, N, H, W, Cin, Cout, s)
    e = rel_l2(nchw(dx).cpu(), gx)
    print(f'conv dgrad: {e:.2e}')
    assert e < TOL
    # fused ReLU mask of the *previous* layer
    mask = nhwc(detgen.det((N, Cin, H, W), 9)).cuda()
    _lib.call('hk_conv3x3_dgrad', dpre_g, wdg, mask, dx, N, H, W, Cin, Cout, s)
    assert rel_l2(nchw(dx).cpu(), gx * (nchw(mask).cpu() > 0)) < TOL
    dw = torch.empty(Cout, Cin, 3, 3, device='cuda')
    db = torch.empty(Cout, device='cuda')
    nb = _lib.query('hk_conv3x3_wgrad_workspace_bytes', Cin, Cout)
    ws = torch.empty(nb, dtype=torch.uint8, device='cuda')
    _lib.call('hk_conv3x3_wgrad', xg, dpre_g, dw, db, N, H, W, Cin, Cout, ws, nb, s)
    ew, eb = rel_l2(dw.cpu(), gw), rel_l2(db.cpu(), gb)
    print(f'conv wgrad: {ew:.2e} bias {eb:.2e}', (db.cpu().double()[:4] / gb[:4]).tolist(), gb[:4].tolist())
    assert ew < TOL and eb < 1e-3   # bias grad comes out of the same tf32 MMA (ones column)


def test_first_layer_and_pool():
    from hawkeye_b200 import _lib
    s = _lib.stream_ptr()
    N, H, W, Cout = 2, 20, 12, 64
    x = detgen.det((N, 3, H, W), 1)
    w = detgen.det((Cout, 3, 3, 3), 2, 0.2)
    b = detgen.det((Cout,), 3, 0.1)
    xd, wd_, bd = x.double(), w.double().requires_grad_(True), b.double().requires_grad_(True)
    y_ref = F.relu(F.conv2d(xd, wd_, bd, padding=1))
    y = torch.empty(N, H, W, Cout, device='cuda')
    nb0 = _lib.query('hk_conv3x3_first_fwd_workspace_bytes', N, H, W, Cout)
    ws0 = torch.empty(nb0, dtype=torch.uint8, device='cuda')
    _lib.call('hk_conv3x3_first_fwd', x.cuda(), w.cuda(), b.cuda(), y, N, H, W, Cout, ws0, nb0, s)
    print('first fwd', rel_l2(nchw(y).cpu(), y_ref.detach()))
    assert rel_l2(nchw(y).cpu(), y_ref.detach()) < 1e-3   # fp32 math, tf32-rounded on store
    dy = detgen.det((N, Cout, H, W), 4).double()
    gw, gb = torch.autograd.grad(y_ref, (wd_, bd), dy)
    dpre = nhwc((dy * (y_ref > 0)).float()).cuda()
    dw = torch.empty(Cout, 3, 3, 3, device='cuda')
    db = torch.empty(Cout, device='cuda')
    nb = _lib.query('hk_conv3x3_first_wgrad_workspace_bytes', N, H, W, Cout)
    ws = torch.empty(nb, dtype=torch.uint8, device='cuda')
    _lib.call('hk_conv3x3_first_wgrad', ws0, dpre, dw, db, N, H, W, Cout, ws, nb, s)
    print('first wgrad', rel_l2(dw.cpu(), gw), rel_l2(db.cpu(), gb))
    assert rel_l2(dw.cpu(), gw) < 2e-3 and rel_l2(db.cpu(), gb) < 2e-3
    # accumulate onto what it just wrote: the same sums added once more, s + s = 2 s exactly
    dw1, db1 = dw.clone(), db.clone()
    _lib.call('hk_conv3x3_first_wgrad_acc', ws0, dpre, dw, db, N, H, W, Cout, ws, nb, 1, s)
    assert torch.equal(dw, 2 * dw1) and torch.equal(db, 2 * db1)
    # max-pool fwd (NHWC and NCHW-out) and bwd (first-max routing + ReLU mask)
    a = F.relu(detgen.det((N, 64, H, W), 7)).double().requires_grad_(True)
    p_ref = F.max_pool2d(a, 2, 2)
    g = detgen.det(p_ref.shape, 8).double()
    (ga,) = torch.autograd.grad(p_ref, a, g)
    ag = nhwc(a.detach().float()).cuda()
    out = torch.empty(N, H // 2, W // 2, 64, device='cuda')
    _lib.call('hk_maxpool2x2_fwd', ag, out, N, H, W, 64, 0, s)
    assert torch.equal(nchw(out).cpu().double(), p_ref.detach())
    out2 = torch.empty(N, 64, H // 2, W // 2, device='cuda')
    _lib.call('hk_maxpool2x2_fwd', ag, out2, N, H, W, 64, 1, s)
    assert torch.equal(out2.cpu().double(), p_ref.detach())
    dx = torch.empty_like(ag)
    _lib.call('hk_maxpool2x2_bwd', ag, nhwc(g.float()).cuda(), dx, N, H, W, 64, 0, s)
    ref = ga * (a.detach() > 0)
    assert rel_l2(nchw(dx).cpu(), ref) < 1e-6
    _lib.call('hk_maxpool2x2_bwd', ag, g.float().cuda(), dx, N, H, W, 64, 1, s)
    assert rel_l2(nchw(dx).cpu(), ref) < 1e-6


@pytest.mark.parametrize('N,H,W,Cin,Cout', [(2, 16, 32, 64, 64),     # v2 kernel, resident weights (VGG conv1_2)
                                            (1, 16, 16, 64, 128),    # v2<128>
                                            (2, 8, 16, 32, 64),      # v2<64>
                                            (2, 28, 28, 128, 256),   # generic kernel, 4x4 pixel tiles
                                            (3, 14, 14, 64, 512),    # generic kernel, 2x2 tiles, ragged batch tile
                                            (2, 56, 56, 32, 96),     # generic kernel, 8-wide tiles, Cout % 128 != 0
                                            (1, 4, 4, 32, 32)])
@pytest.mark.parametrize('nchw', [0, 1])
def test_conv_pool_fused_bit_exact(N, H, W, Cin, Cout, nchw):
    """hk_conv3x3_fwd_pool == hk_conv3x3_fwd + hk_maxpool2x2_fwd_idx, bit for bit (pooled map AND the arg-max / ReLU byte),
    on every conv kernel variant and both output layouts."""
    from hawkeye_b200 import _lib
    s = _lib.stream_ptr()
    x = torch.relu(detgen.det((N, H, W, Cin), 21)).cuda()
    w = detgen.det((Cout, Cin, 3, 3), 22, 0.1).cuda()
    b = detgen.det((Cout,), 23, 0.2).cuda()
    wf = torch.empty(9 * Cout * Cin, device='cuda')
    wd = torch.empty(9 * Cout * Cin, device='cuda')
    _lib.call('hk_conv3x3_pack_weights', w, wf, wd, Cout, Cin, s)
    y = torch.empty(N, H, W, Cout, device='cuda')
    _lib.call('hk_conv3x3_fwd', x, wf, b, y, N, H, W, Cin, Cout, 1, s)
    shape = (N, Cout, H // 2, W // 2) if nchw else (N, H // 2, W // 2, Cout)
    p_ref = torch.empty(shape, device='cuda')
    c_ref = torch.empty(N, H // 2, W // 2, Cout, device='cuda', dtype=torch.uint8)
    _lib.call('hk_maxpool2x2_fwd_idx', y, p_ref, c_ref, N, H, W, Cout, nchw, s)
    p = torch.full(shape, -7.0, device='cuda')
    c = torch.full((N, H // 2, W // 2, Cout), 255, device='cuda', dtype=torch.uint8)
    _lib.call('hk_conv3x3_fwd_pool', x, wf, b, p, c, N, H, W, Cin, Cout, nchw, s)
    torch.cuda.synchronize()
    assert torch.equal(p, p_ref)
    assert torch.equal(c, c_ref)
    # without the code byte (inference / frozen backbone)
    p2 = torch.empty(shape, device='cuda')
    _lib.call('hk_conv3x3_fwd_pool', x, wf, b, p2, None, N, H, W, Cin, Cout, nchw, s)
    assert torch.equal(p2, p_ref)
