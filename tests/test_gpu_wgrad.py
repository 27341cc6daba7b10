"""3x3 conv weight / bias gradient (hk_conv3x3_wgrad_acc) against fp64 conv2d autograd on the GPU.

Shapes: the VGG-16 448x448 layers, the ResNet map sizes, partial output-channel tiles, accumulation and the 3xTF32 mode;
every pixel tile the kernel is specialised on, with a partial last image tile, non-square maps, and over-wide and
over-tall tiles; the 64 ci x 64 co CTA tile with X as the register operand (half-filled ci tiles, the kw-shifted X
fragments at the four map edges, the bias gradient summed by the producer warp on grids of several ci tiles); and the
two-deep wgmma pipeline (CTAs with exactly 1 to 4 stages on every pixel tile, two accumulating calls in a row).

dw and db are NaN-filled (or hold the start of an accumulation) between guard words that must stay untouched.
"""
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_l2
from kernel_check import abi, guarded, precise_on, workspace  # noqa: F401  (precise_on: a fixture)

pytestmark = pytest.mark.gpu


def _inputs(N, H, W, cin, cout, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    x = torch.relu(torch.randn(N, H, W, cin, device='cuda', generator=g))
    dy = torch.randn(N, H, W, cout, device='cuda', generator=g)
    return x, dy


def _reference(x, dy):
    cin, cout = x.shape[-1], dy.shape[-1]
    wd = torch.zeros(cout, cin, 3, 3, dtype=torch.float64, device='cuda', requires_grad=True)
    bd = torch.zeros(cout, dtype=torch.float64, device='cuda', requires_grad=True)
    y = F.conv2d(x.double().permute(0, 3, 1, 2), wd, bd, padding=1)
    return torch.autograd.grad(y, (wd, bd), dy.double().permute(0, 3, 1, 2))


def _run(x, dy, dw0=None, db0=None, accumulate=False):
    """hk_conv3x3_wgrad_acc into guarded dw / db (starting from dw0 / db0 when accumulating) -> dw, db"""
    N, H, W, cin = x.shape
    cout = dy.shape[-1]
    dw, db = guarded((cout, cin, 3, 3)), guarded((cout,))
    if dw0 is not None:
        dw.copy_(dw0)
        db.copy_(db0)
    ws, nb = workspace('hk_conv3x3_wgrad_workspace_bytes', cin, cout)
    abi('hk_conv3x3_wgrad_acc', x, dy, dw, db, N, H, W, cin, cout, ws, nb, int(accumulate))
    return dw, db


def _check(N, H, W, cin, cout, seed=0, tol_w=2e-3, tol_b=1e-3):
    x, dy = _inputs(N, H, W, cin, cout, seed)
    gw, gb = _reference(x, dy)
    dw, db = _run(x, dy)
    ew, eb = rel_l2(dw.double(), gw), rel_l2(db.double(), gb)
    print(f'wgrad N={N} {H}x{W} {cin}->{cout}: dw {ew:.2e} db {eb:.2e}')
    assert ew < tol_w and eb < tol_b


# ------------------------------------------------------------------------------------------------ network shapes
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


@pytest.mark.parametrize('H,c', [(7, 512), (14, 256)])
def test_wgrad_resnet_small_maps(H, c):
    _check(8, H, H, c, c, seed=H)


def test_wgrad_accumulate():
    N, H, W, cin, cout = 2, 32, 32, 128, 128
    x, dy = _inputs(N, H, W, cin, cout, 5)
    gw, gb = _reference(x, dy)
    g = torch.Generator(device='cuda').manual_seed(6)
    dw0 = torch.randn(cout, cin, 3, 3, device='cuda', generator=g) * gw.abs().mean().float()
    db0 = torch.randn(cout, device='cuda', generator=g) * gb.abs().mean().float()
    dw, db = _run(x, dy, dw0, db0, accumulate=True)
    ew, eb = rel_l2(dw.double(), dw0.double() + gw), rel_l2(db.double(), db0.double() + gb)
    print(f'wgrad accumulate: dw {ew:.2e} db {eb:.2e}')
    assert ew < 2e-3 and eb < 1e-3


def test_wgrad_accumulate_twice():
    N, H, W, cin, cout = 2, 24, 32, 128, 64
    x, dy = _inputs(N, H, W, cin, cout, seed=7)
    x2, dy2 = _inputs(N, H, W, cin, cout, seed=8)
    gw, gb = _reference(x, dy)
    gw2, gb2 = _reference(x2, dy2)
    g = torch.Generator(device='cuda').manual_seed(9)
    dw0 = torch.randn(cout, cin, 3, 3, device='cuda', generator=g) * gw.abs().mean().float()
    db0 = torch.randn(cout, device='cuda', generator=g) * gb.abs().mean().float()
    dw1, db1 = _run(x, dy, dw0, db0, accumulate=True)
    dw2, db2 = _run(x2, dy2, dw1, db1, accumulate=True)
    ew = rel_l2(dw2.double(), dw0.double() + gw + gw2)
    eb = rel_l2(db2.double(), db0.double() + gb + gb2)
    print(f'wgrad accumulate twice: dw {ew:.2e} db {eb:.2e}')
    assert ew < 2e-3 and eb < 1e-3


def test_wgrad_precise(precise_on):
    _check(2, 28, 28, 128, 64, tol_w=1e-5, tol_b=1e-5)


# ------------------------------------------------------------------------------------------------ pixel tiles
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


def test_wgrad_precise_two_image_tile(precise_on):
    _check(3, 12, 24, 64, 96, tol_w=1e-5, tol_b=1e-5)


# ------------------------------------------------------------------------------------------------ the CTA tile
@pytest.mark.parametrize('cin,cout', [(96, 64), (160, 64), (96, 96), (160, 96)])
def test_wgrad_half_filled_ci_tile(cin, cout):
    """Cin = 96 and 160 leave the last 64-wide ci tile half filled (TMA zero fill, masked atomics), alone and with a
    half-filled co tile"""
    _check(2, 24, 24, cin, cout, seed=cin + cout)


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
    dw, _ = _run(x, dy)
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
    dw, db = _run(x, dy, dw0, db0, accumulate)
    if accumulate:
        gw, gb = gw + dw0.double(), gb + db0.double()
    ew, eb = rel_l2(dw.double(), gw), rel_l2(db.double(), gb)
    print(f'wgrad bias accumulate={accumulate}: dw {ew:.2e} db {eb:.2e}')
    assert ew < 2e-3 and eb < 1e-5


@pytest.mark.parametrize('cin', [128, 256])
def test_wgrad_bias_ci_tiles(cin):
    """only the ci-tile-0 CTAs add the bias gradient; each of the four producer warps adds its own part"""
    _check(3, 16, 24, cin, 96, seed=cin)


# ------------------------------------------------------------------------------------------------ the pipeline
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
