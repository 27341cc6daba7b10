"""3x3 conv weight / bias gradient vs fp64 conv2d autograd where the 64 ci x 64 co CTA tile with X as the register operand
can go wrong: half-filled ci tiles, the kw-shifted X fragments at the four map edges, and the bias gradient summed by the
producer warp on grids with several ci tiles.  dw and db sit between guard regions that must stay untouched."""
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_l2

pytestmark = pytest.mark.gpu

GUARD = 4096
SENTINEL = 12345.0


def _guarded(n, fill):
    buf = torch.full((n + 2 * GUARD,), SENTINEL, device='cuda')
    buf[GUARD:GUARD + n] = fill
    return buf, buf[GUARD:GUARD + n]


def _guards_intact(buf):
    return bool((buf[:GUARD] == SENTINEL).all() and (buf[-GUARD:] == SENTINEL).all())


def _reference(x, dy):
    cin, cout = x.shape[-1], dy.shape[-1]
    wd = torch.zeros(cout, cin, 3, 3, dtype=torch.float64, device='cuda', requires_grad=True)
    bd = torch.zeros(cout, dtype=torch.float64, device='cuda', requires_grad=True)
    y = F.conv2d(x.double().permute(0, 3, 1, 2), wd, bd, padding=1)
    return torch.autograd.grad(y, (wd, bd), dy.double().permute(0, 3, 1, 2))


def _run(x, dy, dw0=None, db0=None, accumulate=False):
    """hk_conv3x3_wgrad_acc into guarded dw / db (starting from dw0 / db0 when accumulating); returns dw, db, guards ok"""
    from hawkeye_b200 import _lib
    N, H, W, cin = x.shape
    cout = dy.shape[-1]
    wbuf, dw = _guarded(cout * cin * 9, float('nan') if dw0 is None else dw0.reshape(-1))
    bbuf, db = _guarded(cout, float('nan') if db0 is None else db0)
    nb = _lib.query('hk_conv3x3_wgrad_workspace_bytes', cin, cout)
    ws = torch.empty(nb, dtype=torch.uint8, device='cuda')
    _lib.call('hk_conv3x3_wgrad_acc', x, dy, dw, db, N, H, W, cin, cout, ws, nb, int(accumulate), _lib.stream_ptr())
    torch.cuda.synchronize()
    return dw.view(cout, cin, 3, 3).clone(), db.clone(), _guards_intact(wbuf) and _guards_intact(bbuf)


def _inputs(N, H, W, cin, cout, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    x = torch.relu(torch.randn(N, H, W, cin, device='cuda', generator=g))
    dy = torch.randn(N, H, W, cout, device='cuda', generator=g)
    return x, dy


@pytest.mark.parametrize('cin,cout', [(96, 64), (160, 64), (96, 96), (160, 96)])
def test_wgrad_half_filled_ci_tile(cin, cout):
    """Cin = 96 and 160 leave the last 64-wide ci tile half filled (TMA zero fill, masked atomics), alone and with a
    half-filled co tile"""
    x, dy = _inputs(2, 24, 24, cin, cout, seed=cin + cout)
    gw, gb = _reference(x, dy)
    dw, db, ok = _run(x, dy)
    ew, eb = rel_l2(dw.double(), gw), rel_l2(db.double(), gb)
    print(f'wgrad {cin}->{cout}: dw {ew:.2e} db {eb:.2e}')
    assert ok and ew < 2e-3 and eb < 1e-3


@pytest.mark.parametrize('N,H,W', [(2, 13, 20), (1, 9, 30), (2, 7, 7), (3, 12, 24)])
def test_wgrad_map_edges(N, H, W):
    """X is non-zero only on the border ring of the map, so every tap's gradient comes from fragments shifted against
    the top, bottom, left and right edges; checked tap by tap.  Maps: W no multiple of the (16, 4, 1) tile (twice), an
    over-wide and over-tall (8, 8, 1) tile, and the (8, 4, 2) two-image tile with an odd batch"""
    x, dy = _inputs(N, H, W, 64, 64, seed=N * H * W)
    ring = torch.zeros(H, W, 1, device='cuda')
    ring[0], ring[-1], ring[:, 0], ring[:, -1] = 1, 1, 1, 1
    x = x * ring
    gw, _ = _reference(x, dy)
    dw, _, ok = _run(x, dy)
    assert ok
    for kh in range(3):
        for kw in range(3):
            e = rel_l2(dw[:, :, kh, kw].double(), gw[:, :, kh, kw])
            assert e < 2e-3, f'tap ({kh}, {kw}): {e:.2e}'


@pytest.mark.parametrize('accumulate', [False, True])
def test_wgrad_bias_several_ci_tiles(accumulate):
    """Cin = 192: three ci tiles per co tile, of which only the first adds the bias gradient"""
    x, dy = _inputs(2, 16, 16, 192, 128, seed=7)
    gw, gb = _reference(x, dy)
    g = torch.Generator(device='cuda').manual_seed(8)
    dw0 = torch.randn(128, 192, 3, 3, device='cuda', generator=g) if accumulate else None
    db0 = torch.randn(128, device='cuda', generator=g) if accumulate else None
    dw, db, ok = _run(x, dy, dw0, db0, accumulate)
    if accumulate:
        gw, gb = gw + dw0.double(), gb + db0.double()
    ew, eb = rel_l2(dw.double(), gw), rel_l2(db.double(), gb)
    print(f'wgrad bias accumulate={accumulate}: dw {ew:.2e} db {eb:.2e}')
    assert ok and ew < 2e-3 and eb < 1e-5
