"""The VGG-16 input layer (Cin = 3) without X27 in memory: hk_conv3x3_first_fwd_direct and
hk_conv3x3_first_wgrad_direct_acc against fp64 (the bounds of test_gpu_conv_vgg16.py), the direct forward bit for bit
against the X27 forward, and VGGFeaturesFn's gradients on the direct path against the X27 path."""
import time

import pytest
import torch
import torch.nn.functional as F

import detgen
from fp64_refs import BATCH, C_TF32, C_TF32_WGRAD, CHUNK, fp32_exact, gen, randn, wgrad_ref
from kernel_check import HK_ERR_UNSUPPORTED, assert_guards, c_bound, check, guarded, nhwc, rnd_bound

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('N,H,W', [(BATCH, 448, 448),   # the train step: 50,176 pixel blocks over the CTAs
                                   (1, 2, 601),         # 1,202 pixels: partial 128-pixel tile and 32-pixel block
                                   (3, 7, 45)])         # 945 pixels: fewer blocks than CTAs, most CTAs get none
def test_first_direct(N, H, W):
    from hawkeye_b200 import _lib
    _lib.set_precise(0)
    t0 = time.time()
    s = _lib.stream_ptr()
    cout = 64
    g = gen(4000 + W)
    x = detgen.tf32_rna(randn((N, 3, H, W), g))
    w = detgen.tf32_rna(randn((cout, 3, 3, 3), g, 0.2))
    b = detgen.tf32_rna(randn((cout,), g, 0.5))
    y = guarded((N, H, W, cout))
    _lib.call('hk_conv3x3_first_fwd_direct', x, w, b, y, N, H, W, cout, s)
    torch.cuda.synchronize()
    assert_guards(y, tag='first fwd direct')
    worst = 0.0
    for n0 in range(0, N, CHUNK):
        xc = x[n0:n0 + CHUNK]
        ref = nhwc(F.relu(F.conv2d(xc.double(), w.double(), b.double(), padding=1)))
        with fp32_exact():
            absref = nhwc(F.conv2d(xc.abs(), w.abs(), b.abs(), padding=1))
        worst = max(worst, check(y[n0:n0 + CHUNK], ref, rnd_bound(absref, C_TF32),
                                 f'first fwd direct {N}x{H}x{W} [{n0}:{n0 + CHUNK}]', n0=n0))
        del ref, absref
    # same operands, same k order, same wgmma shape as the X27 GEMM: the same bits
    nb0 = _lib.query('hk_conv3x3_first_fwd_workspace_bytes', N, H, W, cout)
    ws0 = torch.empty(nb0, dtype=torch.uint8, device='cuda')
    y27 = torch.empty(N, H, W, cout, device='cuda')
    _lib.call('hk_conv3x3_first_fwd', x, w, b, y27, N, H, W, cout, ws0, nb0, s)
    torch.cuda.synchronize()
    ndiff = int((y.view(torch.int32) != y27.view(torch.int32)).sum())
    assert ndiff == 0, f'direct forward differs from the X27 forward in {ndiff} elements'
    del y, y27, ws0

    dy = detgen.tf32_rna(randn((N, H, W, cout), g))
    gw, aw, gb, ab = wgrad_ref(nhwc(x), dy, 3, cout)
    nb = _lib.query('hk_conv3x3_first_wgrad_direct_workspace_bytes')
    ws = torch.empty(nb, dtype=torch.uint8, device='cuda')
    dw = guarded((cout, 3, 3, 3))
    db = guarded((cout,))
    _lib.call('hk_conv3x3_first_wgrad_direct_acc', x, dy, dw, db, N, H, W, cout, ws, nb, 0, s)
    torch.cuda.synchronize()
    assert_guards(dw, tag='first dw direct')
    assert_guards(db, tag='first db direct')
    names = ('co', 'ci', 'kh', 'kw')
    rw = check(dw, gw, c_bound(aw, C_TF32_WGRAD), f'first wgrad direct dw {N}x{H}x{W}', names=names)
    rb = check(db, gb, c_bound(ab, C_TF32_WGRAD), f'first wgrad direct db {N}x{H}x{W}', names=('co',))
    dw0 = randn((cout, 3, 3, 3), g, float(gw.abs().mean()))
    db0 = randn((cout,), g, float(gb.abs().mean()))
    dw = guarded((cout, 3, 3, 3))
    db = guarded((cout,))
    dw.copy_(dw0)
    db.copy_(db0)
    _lib.call('hk_conv3x3_first_wgrad_direct_acc', x, dy, dw, db, N, H, W, cout, ws, nb, 1, s)
    torch.cuda.synchronize()
    assert_guards(dw, tag='first dw direct accumulate')
    assert_guards(db, tag='first db direct accumulate')
    rwa = check(dw, dw0.double() + gw, c_bound(dw0.double().abs() + aw, C_TF32_WGRAD),
                'first wgrad direct dw accumulate', names=names)
    rba = check(db, db0.double() + gb, c_bound(db0.double().abs() + ab, C_TF32_WGRAD),
                'first wgrad direct db accumulate', names=('co',))
    print(f'first layer direct N={N} {H}x{W}: worst c-term share fwd {worst:.3g} dw {rw:.3g} db {rb:.3g} accumulate dw '
          f'{rwa:.3g} db {rba:.3g}; {time.time() - t0:.1f} s', flush=True)


def test_first_direct_rejects_precise_mode():
    from hawkeye_b200 import _lib
    s = _lib.stream_ptr()
    x = torch.zeros(1, 3, 4, 4, device='cuda')
    w = torch.zeros(64, 3, 3, 3, device='cuda')
    y = torch.zeros(1, 4, 4, 64, device='cuda')
    ws = torch.empty(_lib.query('hk_conv3x3_first_wgrad_direct_workspace_bytes'), dtype=torch.uint8, device='cuda')
    lib = _lib.lib()
    _lib.set_precise(1)
    try:
        assert lib.hk_conv3x3_first_fwd_direct(x.data_ptr(), w.data_ptr(), None, y.data_ptr(), 1, 4, 4, 64, s) == \
            HK_ERR_UNSUPPORTED
        assert lib.hk_conv3x3_first_wgrad_direct_acc(x.data_ptr(), y.data_ptr(), w.data_ptr(), None, 1, 4, 4, 64,
                                                     ws.data_ptr(), ws.numel(), 0, s) == HK_ERR_UNSUPPORTED
    finally:
        _lib.set_precise(0)


def test_vgg_features_direct_first_layer_matches_x27_path():
    """All 26 parameter gradients of VGGFeaturesFn with the direct input layer (the training path) against the X27 path
    (taken under activation capture).  The forward is bit-identical; the backward differs only where the weight
    gradients sum in another order."""
    from oracle import hop_oracle as O
    from hawkeye_b200 import _lib, ops
    _lib.set_precise(0)
    N, H = 4, 64
    state = detgen.vgg_bcnn_state(O.VGG16_D, 200, seed=100)
    params = [state[k].cuda() for k in sorted((k for k in state if k.startswith('backbone.')),
                                             key=lambda k: (int(k.split('.')[1]), k.endswith('bias')))]
    x = detgen.det((N, 3, H, H), 41).cuda()
    dfeat = detgen.det((N, 512, H // 32, H // 32), 43).cuda()

    def run(capture):
        ps = [p.clone().requires_grad_(True) for p in params]
        ops.CAPTURE = [] if capture else None
        try:
            out = ops.vgg_features(x, O.VGG16_D, ps)
        finally:
            ops.CAPTURE = None
        out.backward(dfeat)
        return out.detach(), [p.grad for p in ps]

    out_d, g_d = run(False)
    out_r, g_r = run(True)
    assert torch.equal(out_d, out_r)
    assert len(g_d) == 26
    for i, (a, r) in enumerate(zip(g_d, g_r)):
        rel = float((a.double() - r.double()).norm() / r.double().norm().clamp_min(1e-30))
        assert rel < 1e-4, f'parameter {i}: relative L2 difference {rel:.3g} between the direct and the X27 path'
