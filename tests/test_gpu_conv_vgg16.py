"""Every VGG-16 3x3 convolution of the 448x448 batch-32 train step, element by element against fp64.

The inputs are TF32-representable (detgen.tf32_rna), so every tensor-core product is exact and a kernel's output may
differ from the fp64 result only by its fp32 accumulation and, where it stores TF32, one rounding on store.  That allows
one element-wise bound (kernel_check.check) three orders of magnitude tighter than a rel-L2 over a whole tensor, applied
to every output element of the batch-32 launches, where each persistent CTA cycles its ring, barriers and staging tile
hundreds of times.  The sensitivity tests show that the bound, with the constants below, rejects a kernel output that
lacks one tap of one 32-channel chunk over one 16 x 8 pixel tile, repeats one output row, or carries a bias off by 1e-3.

The fp64 references run on the GPU, 4 images at a time against the kernel's full-batch output.  The kernel each layer
takes (conv3x3_igemm_1x, TF32 mode): conv1_2 the resident v2 kernel (16 x 8 pixel tiles, 64 -> 64 weights in shared
memory); conv2_x and conv3_x v2 with 16 x 8 tiles; conv4_x v2 with 8 x 8 x 2-image tiles; conv5_x the generic kernel
(28 % 8 != 0).  The data gradient swaps Cin and Cout, so conv2_1's runs v2<64> without resident weights.
"""
import time

import pytest
import torch
import torch.nn.functional as F

import detgen
from fp64_refs import (BATCH, C_TF32, C_TF32_WGRAD, CHUNK, VGG16_LAYERS, conv_ref, dgrad_ref, fp32_exact, gen, pack,
                       randn, wgrad_ref)
from kernel_check import HK_ERR_UNSUPPORTED, Out, abi, c_bound, check, guarded, nchw, nhwc, rnd_bound, workspace

pytestmark = pytest.mark.gpu

# |out - ref| <= RND * max(|out|, |ref|) + c * absref, element-wise (kernel_check.rnd_bound).  RND: the TF32 rounding on
# store (10 explicit mantissa bits, round to nearest); c: the fp32 accumulation, relative to the same operation applied
# to |inputs| and |weights|.  Each c is at least 6x the worst (|err| - rounding term) / absref measured over every test
# below on an H100 SXM (80 GB HBM3, 700 W): forward and data gradient 1.15e-6 (conv4_2 / conv5_3 forward), weight
# gradient 4.6e-6 (conv4_3), 3xTF32 2.1e-6 (conv4_3 forward).  C_TF32 and C_TF32_WGRAD are in fp64_refs.py.
# The weight-gradient figure is for zero-mean dY, whose sums cancel.  Where dY has a per-channel mean the sums are
# coherent and the error grows with the pixels each split-K CTA accumulates: 5.4e-5 at conv5_1, batch 32 (14,336 pixels
# per CTA), with half the elements beyond 2^-16: a bias of the accumulation, not a local defect, which the tests leave
# out by using zero-mean gradients.
C_PRECISE = 2.0 ** -16        # 3xTF32, every direction
LAYERS = {name: (H, cin, cout, pool) for name, H, cin, cout, pool in VGG16_LAYERS}
LAST = VGG16_LAYERS[-1][0]    # its pool writes NCHW: the input of the pooling heads


def _fwd(x, wf, b, cout, relu=1):
    N, H, W, cin = x.shape
    y = guarded((N, H, W, cout))
    abi('hk_conv3x3_fwd', x, wf, b, y, N, H, W, cin, cout, relu)
    return y


def _wgrad(x, dy, dw, db, accumulate):
    N, H, W, cin = x.shape
    cout = dy.shape[-1]
    ws, nb = workspace('hk_conv3x3_wgrad_workspace_bytes', cin, cout)
    abi('hk_conv3x3_wgrad_acc', x, dy, dw, db, N, H, W, cin, cout, ws, nb, int(accumulate))


def _windows(t):
    """NHWC (n, H, W, C) -> (n, H/2, W/2, C, 4): the 2x2 pooling windows in scan order (0 0), (0 1), (1 0), (1 1)"""
    n, H, W, C = t.shape
    return t.reshape(n, H // 2, 2, W // 2, 2, C).permute(0, 1, 3, 5, 2, 4).reshape(n, H // 2, W // 2, C, 4)


def _unwindows(t):
    n, Ho, Wo, C, _ = t.shape
    return t.reshape(n, Ho, Wo, C, 2, 2).permute(0, 1, 4, 2, 5, 3).reshape(n, 2 * Ho, 2 * Wo, C)


def _layer_inputs(H, cin, cout, N, seed, tf32=True):
    """a ReLU activation map x (NHWC), kaiming-scaled weights and a bias; TF32-representable unless tf32 is False"""
    g = gen(seed)
    rnd = detgen.tf32_rna if tf32 else (lambda t: t)
    x = rnd(torch.relu(randn((N, H, H, cin), g)))
    w = rnd(randn((cout, cin, 3, 3), g, (2.0 / (9 * cin)) ** 0.5))
    b = randn((cout,), g, 0.5)
    return x, w, b


# ------------------------------------------------------------------------------------------------------------------
# 2. the bound rejects one-tap, one-row and one-bias defects of each kernel variant's own output
# ------------------------------------------------------------------------------------------------------------------
# a 16 x 8 pixel region of image 0 at rows 8..15, columns 0..15; tap (kh, kw) = (0, 2); input-channel chunk 32..63
R_H0, R_W0, R_TAP, R_CI0 = 8, 0, (0, 2), 32


def _tap_contribution(x, w):
    """fp64 sum over ci in the chunk of x[0, h + kh - 1, w + kw - 1, ci] * w[co, ci, kh, kw] over the region:
    (8, 16, Cout)"""
    kh, kw = R_TAP
    xp = F.pad(nchw(x[:1, :, :, R_CI0:R_CI0 + 32]).double(), (1, 1, 1, 1))[0]
    win = xp[:, R_H0 + kh:R_H0 + kh + 8, R_W0 + kw:R_W0 + kw + 16]
    return torch.einsum('cij,oc->ijo', win, w[:, R_CI0:R_CI0 + 32, kh, kw].double())


@pytest.mark.parametrize('variant,layer', [('v2 resident', 'conv1_2'), ('v2<128>', 'conv3_2'),
                                           ('v2 8-wide', 'conv4_2'), ('generic', 'conv5_2')])
def test_bound_rejects_conv_defects(variant, layer):
    """the forward without ReLU, so that each defect is an exact edit of the kernel's output: one tap of one
    32-channel chunk missing over a 16 x 8 pixel region, the region's first row repeated from the row above, one bias
    off by 1e-3"""
    H, cin, cout, _ = LAYERS[layer]
    x, w, b = _layer_inputs(H, cin, cout, 2, 700)
    b = detgen.tf32_rna(b * 4.0)             # a bias of the outputs' own size: its 1e-3 is visible beside them
    wf, _ = pack(w)
    y = _fwd(x, wf, b, cout, relu=0)
    ref, absref = conv_ref(x, w, b)
    tag = f'sensitivity {variant} ({layer})'
    check(y, ref, rnd_bound(absref, C_TF32), f'{tag} unedited')
    bad = y.clone()
    bad[0, R_H0:R_H0 + 8, R_W0:R_W0 + 16] -= _tap_contribution(x, w).float()
    with pytest.raises(AssertionError):
        check(bad, ref, rnd_bound(absref, C_TF32), f'{tag} one tap missing')
    bad = y.clone()
    bad[0, R_H0, R_W0:R_W0 + 16] = y[0, R_H0 - 1, R_W0:R_W0 + 16]
    with pytest.raises(AssertionError):
        check(bad, ref, rnd_bound(absref, C_TF32), f'{tag} row repeated')
    co = int(b.abs().argmax())
    bad = y.clone()
    bad[..., co] += 1e-3 * b[co]
    with pytest.raises(AssertionError):
        check(bad, ref, rnd_bound(absref, C_TF32), f'{tag} bias x (1 + 1e-3)')


def test_bound_rejects_wgrad_defects():
    """the weight gradient at conv5_1's shape: a 16 x 8 pixel tile's share of one tap and one 32-channel chunk, one
    repeated ci row of a 64 x 64 output tile, one channel's bias gradient off by 1e-3.  Batch 2, like the forward's: the
    bias gradient of a zero-mean dY is a cancelling sum, and over the 25,088 pixels of batch 32 its largest value is
    below 1e3 * C_TF32_WGRAD * sum |dY|, so the bound cannot see a 1e-3 error in it there."""
    H, cin, cout, _ = LAYERS['conv5_1']
    x, _, _ = _layer_inputs(H, cin, cout, 2, 710)
    g = gen(711)
    dy = detgen.tf32_rna(randn((2, H, H, cout), g))
    dw, db = guarded((cout, cin, 3, 3)), guarded((cout,))
    _wgrad(x, dy, dw, db, 0)
    gw, aw, gb, ab = wgrad_ref(x, dy, cin, cout)
    names = ('co', 'ci', 'kh', 'kw')
    tag = 'sensitivity wgrad (conv5_1)'
    check(dw, gw, c_bound(aw, C_TF32_WGRAD), f'{tag} dw unedited', names=names)
    check(db, gb, c_bound(ab, C_TF32_WGRAD), f'{tag} db unedited', names=('co',))
    kh, kw = R_TAP
    xp = F.pad(nchw(x[:1, :, :, R_CI0:R_CI0 + 32]).double(), (1, 1, 1, 1))[0]
    win = xp[:, R_H0 + kh:R_H0 + kh + 8, R_W0 + kw:R_W0 + kw + 16]
    part = torch.einsum('cij,ijo->oc', win, dy[0, R_H0:R_H0 + 8, R_W0:R_W0 + 16].double())
    bad = dw.clone()
    bad[:, R_CI0:R_CI0 + 32, kh, kw] -= part.float()
    with pytest.raises(AssertionError):
        check(bad, gw, c_bound(aw, C_TF32_WGRAD), f'{tag} one tile of one tap missing', names=names)
    bad = dw.clone()
    bad[:64, 65, kh, kw] = dw[:64, 64, kh, kw]
    with pytest.raises(AssertionError):
        check(bad, gw, c_bound(aw, C_TF32_WGRAD), f'{tag} ci row repeated', names=names)
    co = int(gb.abs().argmax())
    bad = db.clone()
    bad[co] *= 1 + 1e-3
    with pytest.raises(AssertionError):
        check(bad, gb, c_bound(ab, C_TF32_WGRAD), f'{tag} db x (1 + 1e-3)', names=('co',))


# ------------------------------------------------------------------------------------------------------------------
# 3. forward, fused pooling, pooling backward and data gradient at batch 32, single-pass TF32
# ------------------------------------------------------------------------------------------------------------------
def _check_pool(name, y, p, code, pre, absref, n0):
    """the fused pooling of chunk [n0, n0 + len(pre)) (pre: the fp64 pre-activation): pooled values within the largest
    bound of their window; arg-max
    bits equal to the fp64 first maximum where the window's top two fp64 values are more than twice that bound apart;
    the ReLU bit equal to (fp64 max > 0) where |fp64 max| exceeds it"""
    n1 = n0 + pre.shape[0]
    rr = torch.relu(pre)
    wb = _windows(rnd_bound(absref, C_TF32).total(y[n0:n1], rr)).amax(-1)
    win = _windows(rr)
    pref = win.amax(-1)
    worst = check(p[n0:n1], pref, wb, f'{name} pool [{n0}:{n1}]', n0=n0)
    c = code[n0:n1]
    top2 = win.topk(2, dim=-1).values
    sure = (top2[..., 0] - top2[..., 1]) > 2 * wb
    arg = win.argmax(-1)
    nbad = int(((c & 3).long() != arg)[sure].sum())
    assert nbad == 0, f'{name} pool [{n0}:{n1}]: {nbad} arg-max bits differ from the fp64 first maximum'
    pmax = _windows(pre).amax(-1)
    sure_r = pmax.abs() > wb
    nbad = int((((c & 4) != 0) != (pmax > 0))[sure_r].sum())
    assert nbad == 0, f'{name} pool [{n0}:{n1}]: {nbad} ReLU bits differ from fp64 max > 0'
    return worst


@pytest.mark.parametrize('name', [v[0] for v in VGG16_LAYERS])
def test_vgg16_fwd_pool_dgrad_batch32(name):
    from hawkeye_b200 import _lib
    _lib.set_precise(0)
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    H, cin, cout, pool = LAYERS[name]
    N = BATCH
    seed = 1000 + 10 * [v[0] for v in VGG16_LAYERS].index(name)
    x, w, b = _layer_inputs(H, cin, cout, N, seed)
    wf, wd = pack(w)
    y = _fwd(x, wf, b, cout)
    worst = {}
    if pool:
        to_nchw = int(name == LAST)
        Ho = H // 2
        pshape = (N, cout, Ho, Ho) if to_nchw else (N, Ho, Ho, cout)
        p, code = abi('hk_conv3x3_fwd_pool', x, wf, b, Out(pshape), Out((N, Ho, Ho, cout), torch.uint8), N, H, H, cin,
                      cout, to_nchw)
        p_unf = torch.empty(pshape, device='cuda')
        code_unf = torch.empty(N, Ho, Ho, cout, device='cuda', dtype=torch.uint8)
        abi('hk_maxpool2x2_fwd_idx', y, p_unf, code_unf, N, H, H, cout, to_nchw)
        assert torch.equal(code, code_unf), f'{name}: fused code bytes differ from hk_maxpool2x2_fwd_idx'
        del p_unf, code_unf
        p_nhwc = nhwc(p) if to_nchw else p
    for n0 in range(0, N, CHUNK):
        pre, absref = conv_ref(x[n0:n0 + CHUNK], w, b)
        r = check(y[n0:n0 + CHUNK], torch.relu(pre), rnd_bound(absref, C_TF32),
                  f'{name} fwd [{n0}:{n0 + CHUNK}]', n0=n0)
        worst['fwd'] = max(worst.get('fwd', 0.0), r)
        if pool:
            r = _check_pool(name, y, p_nhwc, code, pre, absref, n0)
            worst['pool'] = max(worst.get('pool', 0.0), r)
        del pre, absref
    del y
    if pool:
        # pooling backward on the fused codes: dy scattered to window position code & 3 where code & 4, bit for bit
        del p, p_nhwc
        g = gen(seed + 1)
        dyp = detgen.tf32_rna(randn(pshape, g))
        (dxp,) = abi('hk_maxpool2x2_bwd_idx', code, dyp, Out((N, H, H, cout)), N, H, H, cout, to_nchw)
        dyp_nhwc = nhwc(dyp) if to_nchw else dyp
        for n0 in range(0, N, CHUNK):
            c = code[n0:n0 + CHUNK]
            gv = torch.where((c & 4) != 0, dyp_nhwc[n0:n0 + CHUNK], torch.zeros((), device='cuda'))
            ref = _unwindows(torch.stack([torch.where((c & 3) == k, gv, torch.zeros((), device='cuda'))
                                          for k in range(4)], -1))
            assert torch.equal(dxp[n0:n0 + CHUNK], ref), f'{name} pool bwd [{n0}:{n0 + CHUNK}] differs from the scatter'
        del dxp, dyp, dyp_nhwc, code
    g = gen(seed + 2)
    dy = detgen.tf32_rna(randn((N, H, H, cout), g))
    for masked in (False, True):
        (dx,) = abi('hk_conv3x3_dgrad', dy, wd, x if masked else None, Out((N, H, H, cin)), N, H, H, cin, cout)
        key = 'dgrad masked' if masked else 'dgrad'
        for n0 in range(0, N, CHUNK):
            ref, absref = dgrad_ref(dy[n0:n0 + CHUNK], w)
            if masked:
                m = x[n0:n0 + CHUNK] > 0
                ref, absref = ref * m, absref * m
            r = check(dx[n0:n0 + CHUNK], ref, rnd_bound(absref, C_TF32), f'{name} {key} [{n0}:{n0 + CHUNK}]', n0=n0)
            worst[key] = max(worst.get(key, 0.0), r)
            del ref, absref
        del dx
    print(f'{name} N={N} {H}x{H} {cin}->{cout}: worst c-term share ' +
          ', '.join(f'{k} {v:.3g}' for k, v in worst.items()) +
          f'; {time.time() - t0:.1f} s, peak {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB', flush=True)


# ------------------------------------------------------------------------------------------------------------------
# 4. weight gradient at batch 32: the split-K count of the timed launch
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', [v[0] for v in VGG16_LAYERS])
def test_vgg16_wgrad_batch32(name):
    from hawkeye_b200 import _lib
    _lib.set_precise(0)
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    H, cin, cout, _ = LAYERS[name]
    N = BATCH
    seed = 2000 + 10 * [v[0] for v in VGG16_LAYERS].index(name)
    x, _, _ = _layer_inputs(H, cin, cout, N, seed)
    g = gen(seed + 1)
    dy = detgen.tf32_rna(randn((N, H, H, cout), g))
    gw, aw, gb, ab = wgrad_ref(x, dy, cin, cout)
    names = ('co', 'ci', 'kh', 'kw')
    dw, db = guarded((cout, cin, 3, 3)), guarded((cout,))
    _wgrad(x, dy, dw, db, 0)
    rw = check(dw, gw, c_bound(aw, C_TF32_WGRAD), f'{name} wgrad dw', names=names)
    rb = check(db, gb, c_bound(ab, C_TF32_WGRAD), f'{name} wgrad db', names=('co',))
    dw0 = randn((cout, cin, 3, 3), g, float(gw.abs().mean()))
    db0 = randn((cout,), g, float(gb.abs().mean()))
    dw, db = dw0.clone(), db0.clone()
    _wgrad(x, dy, dw, db, 1)
    rwa = check(dw, dw0.double() + gw, c_bound(dw0.double().abs() + aw, C_TF32_WGRAD),
                f'{name} wgrad dw accumulate', names=names)
    rba = check(db, db0.double() + gb, c_bound(db0.double().abs() + ab, C_TF32_WGRAD),
                f'{name} wgrad db accumulate', names=('co',))
    print(f'{name} N={N} wgrad: worst c-term share dw {rw:.3g} db {rb:.3g} accumulate dw {rwa:.3g} db {rba:.3g}; '
          f'{time.time() - t0:.1f} s, peak {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB', flush=True)


# ------------------------------------------------------------------------------------------------------------------
# 5. the first layer (Cin = 3): X27 patches + one GEMM forward, split-K weight gradient with db from the ones column
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('N,H,W', [(BATCH, 448, 448),   # 6,422,528 pixels: 512 splits
                                   (1, 2, 601)])        # 1,202 pixels: the largest divisor <= 592 is 2
def test_first_layer(N, H, W):
    from hawkeye_b200 import _lib
    _lib.set_precise(0)
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    cout = 64
    g = gen(3000 + W)
    x = detgen.tf32_rna(randn((N, 3, H, W), g))
    w = detgen.tf32_rna(randn((cout, 3, 3, 3), g, 0.2))
    b = detgen.tf32_rna(randn((cout,), g, 0.5))  # the bias rides in the GEMM as column 27 of W27: TF32 like the weights
    ws0, nb0 = workspace('hk_conv3x3_first_fwd_workspace_bytes', N, H, W, cout)
    (y,) = abi('hk_conv3x3_first_fwd', x, w, b, Out((N, H, W, cout)), N, H, W, cout, ws0, nb0)
    worst = 0.0
    for n0 in range(0, N, CHUNK):
        xc = x[n0:n0 + CHUNK]
        ref = nhwc(F.relu(F.conv2d(xc.double(), w.double(), b.double(), padding=1)))
        with fp32_exact():
            absref = nhwc(F.conv2d(xc.abs(), w.abs(), b.abs(), padding=1))
        worst = max(worst, check(y[n0:n0 + CHUNK], ref, rnd_bound(absref, C_TF32),
                                 f'first fwd {N}x{H}x{W} [{n0}:{n0 + CHUNK}]', n0=n0))
        del ref, absref
    del y
    dy = detgen.tf32_rna(randn((N, H, W, cout), g))
    gw, aw, gb, ab = wgrad_ref(nhwc(x), dy, 3, cout)
    ws, nb = workspace('hk_conv3x3_first_wgrad_workspace_bytes', N, H, W, cout)
    dw, db = abi('hk_conv3x3_first_wgrad', ws0, dy, Out((cout, 3, 3, 3)), Out((cout,)), N, H, W, cout, ws, nb)
    names = ('co', 'ci', 'kh', 'kw')
    rw = check(dw, gw, c_bound(aw, C_TF32_WGRAD), f'first wgrad dw {N}x{H}x{W}', names=names)
    rb = check(db, gb, c_bound(ab, C_TF32_WGRAD), f'first wgrad db {N}x{H}x{W}', names=('co',))
    dw0 = randn((cout, 3, 3, 3), g, float(gw.abs().mean()))
    db0 = randn((cout,), g, float(gb.abs().mean()))
    dw, db = dw0.clone(), db0.clone()
    abi('hk_conv3x3_first_wgrad_acc', ws0, dy, dw, db, N, H, W, cout, ws, nb, 1)
    rwa = check(dw, dw0.double() + gw, c_bound(dw0.double().abs() + aw, C_TF32_WGRAD),
                f'first wgrad dw accumulate', names=names)
    rba = check(db, db0.double() + gb, c_bound(db0.double().abs() + ab, C_TF32_WGRAD),
                f'first wgrad db accumulate', names=('co',))
    print(f'first layer N={N} {H}x{W}: worst c-term share fwd {worst:.3g} dw {rw:.3g} db {rb:.3g} accumulate dw '
          f'{rwa:.3g} db {rba:.3g}; {time.time() - t0:.1f} s', flush=True)


# ------------------------------------------------------------------------------------------------------------------
# 6. 3xTF32: arbitrary fp32 inputs, the generic kernel in three chained passes, no output rounding
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', [v[0] for v in VGG16_LAYERS])
def test_vgg16_precise(name):
    from hawkeye_b200 import _lib
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    H, cin, cout, pool = LAYERS[name]
    N = 4
    seed = 4000 + 10 * [v[0] for v in VGG16_LAYERS].index(name)
    _lib.set_precise(1)
    try:
        x, w, b = _layer_inputs(H, cin, cout, N, seed, tf32=False)
        wf, wd = pack(w)
        y = _fwd(x, wf, b, cout)
        pre, absref = conv_ref(x, w, b)
        rf = check(y, torch.relu(pre), c_bound(absref, C_PRECISE), f'{name} precise fwd')
        del y, pre, absref
        if pool:
            p = torch.empty(N, H // 2, H // 2, cout, device='cuda')
            rc = _lib.query('hk_conv3x3_fwd_pool', x, wf, b, p, None, N, H, H, cin, cout, 0, _lib.stream_ptr())
            assert rc == HK_ERR_UNSUPPORTED, f'hk_conv3x3_fwd_pool in 3xTF32 mode returned {rc}'
        g = gen(seed + 1)
        dy = randn((N, H, H, cout), g)
        (dx,) = abi('hk_conv3x3_dgrad', dy, wd, x, Out((N, H, H, cin)), N, H, H, cin, cout)
        ref, absref = dgrad_ref(dy, w)
        m = x > 0
        rd = check(dx, ref * m, c_bound(absref * m, C_PRECISE), f'{name} precise dgrad masked')
        del dx, ref, absref
        gw, aw, gb, ab = wgrad_ref(x, dy, cin, cout)
        dw, db = guarded((cout, cin, 3, 3)), guarded((cout,))
        _wgrad(x, dy, dw, db, 0)
        rw = check(dw, gw, c_bound(aw, C_PRECISE), f'{name} precise wgrad dw', names=('co', 'ci', 'kh', 'kw'))
        rb = check(db, gb, c_bound(ab, C_PRECISE), f'{name} precise wgrad db', names=('co',))
    finally:
        _lib.set_precise(0)
    print(f'{name} N={N} 3xTF32: worst c-term share fwd {rf:.3g} dgrad {rd:.3g} dw {rw:.3g} db {rb:.3g}; '
          f'{time.time() - t0:.1f} s, peak {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB', flush=True)
