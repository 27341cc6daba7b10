"""The halo-reuse 3x3 convolution on maps that its 8 x 8 x 2-image pixel tile divides and its 16 x 8 tile does not (56 x 56,
24 x 40): the checks of test_gpu_conv_tiles.py (forward and data gradient with and without mask against torch-CPU fp64,
fused pooling in both layouts bit for bit against the unfused pair, NaN-filled outputs and guard words) at batch 1 and
odd batches, where the last tile's second image does not exist, with a partial co tile, several co tiles and more tiles
than CTAs.  The 28 x 28 shapes stay on the generic kernel and are here so that both sides of the choice see the same
cases."""
import pytest

import test_gpu_conv_tiles as T

pytestmark = pytest.mark.gpu

SHAPES = [
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
def test_conv3x3_tiles8_fwd_dgrad(N, H, W, Cin, Cout):
    T.test_conv3x3_tiles_fwd_dgrad(N, H, W, Cin, Cout)


@pytest.mark.parametrize('N,H,W,Cin,Cout', SHAPES)
@pytest.mark.parametrize('nchw', [0, 1])
def test_conv3x3_tiles8_pool_bit_exact(N, H, W, Cin, Cout, nchw):
    T.test_conv3x3_tiles_pool_bit_exact(N, H, W, Cin, Cout, nchw)
