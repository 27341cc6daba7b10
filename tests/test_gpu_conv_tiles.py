"""The halo-reuse 3x3 convolution (forward, data gradient and fused pooling) at the tile-schedule edges its epilogue
warpgroup sees: one tile, a partial 128-wide co tile, several co tiles, and more tiles than CTAs, so that the staging
tile between the MMA and epilogue warpgroups is reused; with both pixel tiles, 16 x 8 and 8 x 8 x 2 images, the latter
at batch 1 and odd batches, where the last tile's second image does not exist.  Forward and data gradient are checked
against torch-CPU fp64; the fused pooling against the unfused forward and max-pool, bit for bit."""
import pytest
import torch
import torch.nn.functional as F

import detgen
from conftest import rel_l2
from kernel_check import abi, guarded, nchw, nhwc

pytestmark = pytest.mark.gpu
TOL = 2e-3

SHAPES = [
    (1, 8, 16, 32, 64),      # a single pixel tile and a single co tile
    (2, 16, 32, 64, 96),     # Cout = 96: one partial co tile
    (1, 16, 16, 128, 512),   # four co tiles
    (9, 32, 64, 32, 64),     # BN 64, 144 tiles
    (3, 64, 128, 64, 64),    # resident 64 -> 64 weights, 192 tiles
    (3, 64, 128, 32, 256),   # BN 128, two co tiles, 384 tiles
    # maps the 8 x 8 x 2-image tile divides and the 16 x 8 tile does not (56 x 56, 24 x 40); the 28 x 28 maps stay on
    # the generic kernel, so that both sides of the choice see the same cases
    (1, 8, 8, 32, 64),       # a single tile, its second image missing
    (1, 56, 56, 32, 64),     # batch 1: every tile half filled
    (3, 56, 56, 64, 64),     # resident 64 -> 64 weights, odd batch, 98 tiles
    (2, 56, 56, 64, 96),     # Cout = 96: one partial co tile
    (5, 56, 56, 32, 256),    # BN 128, two co tiles, odd batch, 294 tiles
    (2, 24, 40, 128, 512),   # four co tiles, W != H
    (3, 28, 28, 32, 64),     # generic kernel, BN 64
    (2, 28, 28, 64, 256),    # generic kernel, BN 128
]


@pytest.mark.parametrize('N,H,W,Cin,Cout', SHAPES)
def test_conv3x3_tiles_fwd_dgrad(N, H, W, Cin, Cout):
    from hawkeye_b200 import _lib
    s = _lib.stream_ptr()
    x = detgen.det((N, Cin, H, W), 31, positive=True)
    w = detgen.det((Cout, Cin, 3, 3), 32, (2.0 / (Cout * 9)) ** 0.5)
    b = detgen.det((Cout,), 33, 0.1)
    dy = detgen.det((N, Cout, H, W), 34)
    xd = x.double().requires_grad_(True)
    y_ref = F.relu(F.conv2d(xd, w.double(), b.double(), padding=1))
    dpre = dy.double() * (y_ref > 0)
    (gx,) = torch.autograd.grad(y_ref, (xd,), dy.double())

    wf = torch.empty(9 * Cout * Cin, device='cuda')
    wd = torch.empty(9 * Cout * Cin, device='cuda')
    _lib.call('hk_conv3x3_pack_weights', w.cuda(), wf, wd, Cout, Cin, s)
    y = guarded((N, H, W, Cout))
    abi('hk_conv3x3_fwd', nhwc(x).cuda(), wf, b.cuda(), y, N, H, W, Cin, Cout, 1)
    e = rel_l2(nchw(y).cpu(), y_ref.detach())
    print(f'fwd {N}x{H}x{W} {Cin}->{Cout}: {e:.2e}')
    assert e < TOL
    dpre_g = nhwc(dpre.float()).cuda()
    for mask in (None, nhwc(detgen.det((N, Cin, H, W), 39)).cuda()):
        dx = guarded((N, H, W, Cin))
        abi('hk_conv3x3_dgrad', dpre_g, wd, mask, dx, N, H, W, Cin, Cout)
        ref = gx if mask is None else gx * (nchw(mask).cpu() > 0)
        e = rel_l2(nchw(dx).cpu(), ref)
        print(f'dgrad (mask {mask is not None}): {e:.2e}')
        assert e < TOL


@pytest.mark.parametrize('N,H,W,Cin,Cout', SHAPES)
@pytest.mark.parametrize('nchw', [0, 1])
def test_conv3x3_tiles_pool_bit_exact(N, H, W, Cin, Cout, nchw):
    from hawkeye_b200 import _lib
    if _lib.get_precise():
        pytest.skip('the fused conv + pool is single-pass TF32 only')
    s = _lib.stream_ptr()
    x = torch.relu(detgen.det((N, H, W, Cin), 41)).cuda()
    w = detgen.det((Cout, Cin, 3, 3), 42, 0.1).cuda()
    b = detgen.det((Cout,), 43, 0.2).cuda()
    wf = torch.empty(9 * Cout * Cin, device='cuda')
    wd = torch.empty(9 * Cout * Cin, device='cuda')
    _lib.call('hk_conv3x3_pack_weights', w, wf, wd, Cout, Cin, s)
    y = torch.empty(N, H, W, Cout, device='cuda')
    _lib.call('hk_conv3x3_fwd', x, wf, b, y, N, H, W, Cin, Cout, 1, s)
    shape = (N, Cout, H // 2, W // 2) if nchw else (N, H // 2, W // 2, Cout)
    p_ref = torch.empty(shape, device='cuda')
    c_ref = torch.empty(N, H // 2, W // 2, Cout, device='cuda', dtype=torch.uint8)
    _lib.call('hk_maxpool2x2_fwd_idx', y, p_ref, c_ref, N, H, W, Cout, nchw, s)
    p, c = guarded(shape), guarded((N, H // 2, W // 2, Cout), torch.uint8)
    abi('hk_conv3x3_fwd_pool', x, wf, b, p, c, N, H, W, Cin, Cout, nchw)
    assert torch.equal(p, p_ref)
    assert torch.equal(c, c_ref)
