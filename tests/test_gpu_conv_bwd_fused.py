"""The fused backward entries of the halo-reuse 3x3 convolution:

- hk_conv3x3_dgrad_first_wgrad_acc (VGG conv1_2's data gradient with conv1_1's weight gradient in its epilogue): dw1 and
  db1 against fp64 of the weight gradient of the dx1 that hk_conv3x3_dgrad stores (the bounds of test_gpu_conv_vgg16.py),
  against hk_conv3x3_first_wgrad_direct_acc on that dx1, in both accumulate modes, and bit for bit across two calls;
- hk_conv3x3_dgrad_unpool (a data gradient stored straight into the unpooled map) bit for bit against hk_conv3x3_dgrad
  followed by hk_maxpool2x2_bwd_idx, on both pixel tiles, BN 64 and 128, several co tiles and an odd batch;
- VGGFeaturesFn, whose training backward takes both, against its path under activation capture.

Outputs are NaN-filled and followed by guard words."""
import time

import pytest
import torch

import detgen
from fp64_refs import BATCH, C_TF32_WGRAD, gen, pack, randn, wgrad_ref
from kernel_check import HK_ERR_UNSUPPORTED, abi, assert_guards, c_bound, check, guarded, nhwc, workspace

pytestmark = pytest.mark.gpu


def _first_wgrad_fused(dy, wd, mask, x, dw, db, accumulate):
    N, H, W, C = dy.shape
    ws, nb = workspace('hk_conv3x3_dgrad_first_wgrad_workspace_bytes')
    abi('hk_conv3x3_dgrad_first_wgrad_acc', dy, wd, mask, x, dw, db, N, H, W, C, C, ws, nb, int(accumulate))


@pytest.mark.parametrize('N,H,W', [(BATCH, 448, 448),   # the train step
                                   (1, 8, 16),          # one tile
                                   (3, 8, 32),          # one tile row, odd batch
                                   (3, 64, 96)])        # 144 tiles: more than CTAs, both halo buffers reused
def test_dgrad_first_wgrad(N, H, W):
    from hawkeye_b200 import _lib
    _lib.set_precise(0)
    t0 = time.time()
    s = _lib.stream_ptr()
    C = 64
    g = gen(5000 + W)
    x = detgen.tf32_rna(randn((N, 3, H, W), g))
    mask = torch.relu(randn((N, H, W, C), g))            # conv1_1's output: about half the ReLU mask is zero
    dy = detgen.tf32_rna(randn((N, H, W, C), g))
    _, wd = pack(randn((C, C, 3, 3), g, (2.0 / (9 * C)) ** 0.5))
    # dx1 as the unfused backward stores it
    dx1 = torch.empty(N, H, W, C, device='cuda')
    _lib.call('hk_conv3x3_dgrad', dy, wd, mask, dx1, N, H, W, C, C, s)
    gw, aw, gb, ab = wgrad_ref(nhwc(x), dx1, 3, C)
    names = ('co', 'ci', 'kh', 'kw')

    dw = guarded((C, 3, 3, 3))
    db = guarded((C,))
    _first_wgrad_fused(dy, wd, mask, x, dw, db, 0)
    assert_guards(dw, tag='fused dw1')
    assert_guards(db, tag='fused db1')
    rw = check(dw, gw, c_bound(aw, C_TF32_WGRAD), f'fused dw1 {N}x{H}x{W}', names=names)
    rb = check(db, gb, c_bound(ab, C_TF32_WGRAD), f'fused db1 {N}x{H}x{W}', names=('co',))

    # the unfused weight gradient of the same dx1: both are within the bound of fp64, so within twice it of each other
    nbd = _lib.query('hk_conv3x3_first_wgrad_direct_workspace_bytes')
    wsd = torch.empty(nbd, dtype=torch.uint8, device='cuda')
    dwu = torch.empty(C, 3, 3, 3, device='cuda')
    dbu = torch.empty(C, device='cuda')
    _lib.call('hk_conv3x3_first_wgrad_direct_acc', x, dx1, dwu, dbu, N, H, W, C, wsd, nbd, 0, s)
    torch.cuda.synchronize()
    check(dw, dwu, c_bound(aw, 2 * C_TF32_WGRAD), f'fused dw1 against the unfused pair {N}x{H}x{W}', names=names)
    check(db, dbu, c_bound(ab, 2 * C_TF32_WGRAD), f'fused db1 against the unfused pair {N}x{H}x{W}', names=('co',))

    # deterministic: per-CTA partials reduced in a fixed order
    dw2 = guarded((C, 3, 3, 3))
    db2 = guarded((C,))
    _first_wgrad_fused(dy, wd, mask, x, dw2, db2, 0)
    assert torch.equal(dw2.view(torch.int32), dw.view(torch.int32)) and torch.equal(db2.view(torch.int32),
                                                                                     db.view(torch.int32))

    dw0 = randn((C, 3, 3, 3), g, float(gw.abs().mean()))
    db0 = randn((C,), g, float(gb.abs().mean()))
    dw = guarded((C, 3, 3, 3))
    db = guarded((C,))
    dw.copy_(dw0)
    db.copy_(db0)
    _first_wgrad_fused(dy, wd, mask, x, dw, db, 1)
    assert_guards(dw, tag='fused dw1 accumulate')
    assert_guards(db, tag='fused db1 accumulate')
    rwa = check(dw, dw0.double() + gw, c_bound(dw0.double().abs() + aw, C_TF32_WGRAD),
                'fused dw1 accumulate', names=names)
    rba = check(db, db0.double() + gb, c_bound(db0.double().abs() + ab, C_TF32_WGRAD),
                'fused db1 accumulate', names=('co',))
    print(f'dgrad + first wgrad N={N} {H}x{W}: worst c-term share dw {rw:.3g} db {rb:.3g} accumulate dw {rwa:.3g} '
          f'db {rba:.3g}; {time.time() - t0:.1f} s', flush=True)


def test_dgrad_first_wgrad_rejects():
    from hawkeye_b200 import _lib
    s = _lib.stream_ptr()
    lib = _lib.lib()
    N, H, W, C = 1, 8, 24, 64                            # W % 16 != 0: the 16 x 8 tile does not fit
    dy = torch.zeros(N, H, W, C, device='cuda')
    wd = torch.zeros(9 * C * C, device='cuda')
    x = torch.zeros(N, 3, H, W, device='cuda')
    dw = torch.zeros(C, 3, 3, 3, device='cuda')
    nb = _lib.query('hk_conv3x3_dgrad_first_wgrad_workspace_bytes')
    ws = torch.empty(nb, dtype=torch.uint8, device='cuda')

    def call(w):
        return lib.hk_conv3x3_dgrad_first_wgrad_acc(dy.data_ptr(), wd.data_ptr(), None, x.data_ptr(), dw.data_ptr(), None,
                                                    N, H, w, C, C, ws.data_ptr(), nb, 0, s)
    _lib.set_precise(0)
    assert call(W) == HK_ERR_UNSUPPORTED
    _lib.set_precise(1)
    try:
        assert call(16) == HK_ERR_UNSUPPORTED
    finally:
        _lib.set_precise(0)


UNPOOL_SHAPES = [
    (BATCH, 224, 224, 64, 128),    # conv2_1 at the train step: BN 64, 16 x 8 tile
    (BATCH, 112, 112, 128, 256),   # conv3_1: BN 128
    (BATCH, 56, 56, 256, 512),     # conv4_1: BN 128, two co tiles, 8 x 8 x 2-image tile
    (1, 8, 16, 64, 64),            # one tile, resident 64 -> 64 weights
    (3, 8, 8, 32, 64),             # 8 x 8 x 2 tile, odd batch: the last tile's second image is empty
    (5, 16, 24, 128, 32),          # 8 x 8 x 2 tile, BN 128 one co tile, odd batch
    (2, 16, 32, 256, 64),          # BN 128, two co tiles
    (3, 8, 16, 96, 64),            # a partial 128-wide co tile, odd batch
    (9, 32, 64, 64, 32),           # 144 tiles: more than CTAs
]


@pytest.mark.parametrize('N,H,W,Cin,Cout', UNPOOL_SHAPES)
def test_dgrad_unpool_bit_exact(N, H, W, Cin, Cout):
    """H x W is the pooled map the data gradient runs at; the pool's input is 2H x 2W"""
    from hawkeye_b200 import _lib
    _lib.set_precise(0)
    s = _lib.stream_ptr()
    g = gen(6000 + H + Cin)
    # pre-pool activations with whole windows at or below zero, so that bit 2 of the code is clear in places
    pre = torch.relu(randn((N, 2 * H, 2 * W, Cin), g) - 0.8)
    pooled = torch.empty(N, H, W, Cin, device='cuda')
    code = torch.empty(N, H, W, Cin, device='cuda', dtype=torch.uint8)
    _lib.call('hk_maxpool2x2_fwd_idx', pre, pooled, code, N, 2 * H, 2 * W, Cin, 0, s)
    del pre, pooled
    dy = randn((N, H, W, Cout), g)
    _, wd = pack(randn((Cout, Cin, 3, 3), g, (2.0 / (9 * Cin)) ** 0.5))
    dx = torch.empty(N, H, W, Cin, device='cuda')
    _lib.call('hk_conv3x3_dgrad', dy, wd, None, dx, N, H, W, Cin, Cout, s)
    ref = torch.empty(N, 2 * H, 2 * W, Cin, device='cuda')
    _lib.call('hk_maxpool2x2_bwd_idx', code, dx, ref, N, 2 * H, 2 * W, Cin, 0, s)
    del dx
    out = guarded((N, 2 * H, 2 * W, Cin))
    _lib.call('hk_conv3x3_dgrad_unpool', dy, wd, code, out, N, H, W, Cin, Cout, s)
    torch.cuda.synchronize()
    assert_guards(out, tag='dgrad unpool')
    ndiff = int((out.view(torch.int32) != ref.view(torch.int32)).sum())
    assert ndiff == 0, f'dgrad unpool differs from dgrad + max-pool backward in {ndiff} of {out.numel()} elements'
    assert int((code & 4 == 0).sum()) > 0 and int((ref != 0).sum()) > 0


def test_dgrad_unpool_rejects():
    from hawkeye_b200 import _lib
    s = _lib.stream_ptr()
    lib = _lib.lib()
    N, C = 1, 32
    dy = torch.zeros(N, 12, 12, C, device='cuda')
    wd = torch.zeros(9 * C * C, device='cuda')
    code = torch.zeros(N, 12, 12, C, device='cuda', dtype=torch.uint8)
    dx = torch.zeros(N, 24, 24, C, device='cuda')

    def call(H, W):
        return lib.hk_conv3x3_dgrad_unpool(dy.data_ptr(), wd.data_ptr(), code.data_ptr(), dx.data_ptr(), N, H, W, C, C, s)
    _lib.set_precise(0)
    assert call(12, 8) == HK_ERR_UNSUPPORTED       # the halo-reuse kernel tiles multiples of 8 only
    assert call(8, 12) == HK_ERR_UNSUPPORTED
    _lib.set_precise(1)
    try:
        assert call(8, 8) == HK_ERR_UNSUPPORTED
    finally:
        _lib.set_precise(0)


def test_vgg_features_fused_backward_matches_capture_path():
    """All 26 parameter gradients of VGGFeaturesFn on the training path against the path taken under activation capture.
    At 64x64 the training backward computes conv1_1's weight gradient in conv1_2's data gradient and takes the unpooled
    data gradient at conv2_1 (32x32, 16 x 8 tile), conv3_1 (16x16) and conv4_1 (8x8, 8 x 8 x 2-image tile); conv5_1 (4x4)
    keeps the separate max-pool backward.  The capture path runs the X27 input layer and the unfused conv1_2 data
    gradient, so conv1_1's gradients sum in another order there."""
    from oracle import hop_oracle as O
    from hawkeye_b200 import _lib, ops
    _lib.set_precise(0)
    N, H = 4, 64
    state = detgen.vgg_bcnn_state(O.VGG16_D, 200, seed=100)
    params = [state[k].cuda() for k in sorted((k for k in state if k.startswith('backbone.')),
                                             key=lambda k: (int(k.split('.')[1]), k.endswith('bias')))]
    x = detgen.det((N, 3, H, H), 41).cuda()
    dfeat = detgen.det((N, 512, H // 32, H // 32), 43).cuda()

    def run(capture, accumulate):
        ps = [p.clone().requires_grad_(True) for p in params]
        if accumulate:       # .grad present: the backward adds into it, as in the trainer
            for p in ps:
                p.grad = torch.zeros_like(p)
        ops.CAPTURE = [] if capture else None
        try:
            out = ops.vgg_features(x, O.VGG16_D, ps)
        finally:
            ops.CAPTURE = None
        out.backward(dfeat)
        return out.detach(), [p.grad for p in ps]

    for accumulate in (False, True):
        out_f, g_f = run(False, accumulate)
        out_r, g_r = run(True, accumulate)
        assert torch.equal(out_f, out_r)
        assert len(g_f) == 26
        for i, (a, r) in enumerate(zip(g_f, g_r)):
            rel = float((a.double() - r.double()).norm() / r.double().norm().clamp_min(1e-30))
            assert rel < 1e-4, f'parameter {i} (accumulate {accumulate}): relative L2 difference {rel:.3g}'
