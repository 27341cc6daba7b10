"""3x3 conv weight gradient vs fp64 conv2d autograd at every pixel tile the kernel is specialised on and at the edges of
its pipeline: the (8, 4, 2) two-image tile with a partial last image tile, non-square maps, over-wide and over-tall
tiles, and CTAs with fewer pixel tiles than pipeline stages."""
import pytest

from test_gpu_wgrad import _check

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('N,H,W,cin,cout', [
    (3, 12, 24, 64, 64),      # (8, 4, 2): two images per tile, N odd -> the last tile holds one image
    (2, 20, 56, 128, 64),     # (8, 4, 2) on a non-square map, 3 tiles across
    (2, 16, 40, 64, 128),     # (8, 8, 1) on a non-square map
    (2, 24, 12, 64, 64),      # (16, 4, 1) over-wide: columns 12..15 of each tile are zero fill
    (2, 6, 32, 64, 64),       # (16, 4, 1) over-tall: the second tile row covers 2 of its 4 rows
])
def test_wgrad_tiles(N, H, W, cin, cout):
    _check(N, H, W, cin, cout, seed=N + H + W)


@pytest.mark.parametrize('N,H,W,cin,cout', [
    (1, 7, 7, 128, 128),      # one pixel tile: a single stage
    (1, 8, 16, 512, 512),     # one split of two pixel tiles
    (1, 8, 32, 512, 512),     # one split of four pixel tiles: the three-stage ring wraps once
])
def test_wgrad_short_pipeline(N, H, W, cin, cout):
    _check(N, H, W, cin, cout, seed=1)


def test_wgrad_precise_two_image_tile():
    from hawkeye_b200 import _lib
    _lib.set_precise(1)
    try:
        _check(3, 12, 24, 64, 96, tol_w=1e-5, tol_b=1e-5)
    finally:
        _lib.set_precise(0)
