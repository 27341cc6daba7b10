"""Every VGG-16 3x3 convolution of the 448x448 batch-32 train step, element by element against fp64.

The inputs are TF32-representable (detgen.tf32_rna), so every tensor-core product is exact and a kernel's output may
differ from the fp64 result only by its fp32 accumulation and, where it stores TF32, one rounding on store.  That allows
one element-wise bound (check_bound) three orders of magnitude tighter than a rel-L2 over a whole tensor, applied to
every output element of the batch-32 launches, where each persistent CTA cycles its ring, barriers and staging tile
hundreds of times.  The sensitivity tests show that the bound, with the constants below, rejects a kernel output that
lacks one tap of one 32-channel chunk over one 16 x 8 pixel tile, repeats one output row, or carries a bias off by 1e-3.

The fp64 references run on the GPU, 4 images at a time against the kernel's full-batch output.  The kernel each layer
takes (conv3x3_igemm_1x, TF32 mode): conv1_2 the resident v2 kernel (16 x 8 pixel tiles, 64 -> 64 weights in shared
memory); conv2_x and conv3_x v2 with 16 x 8 tiles; conv4_x v2 with 8 x 8 x 2-image tiles; conv5_x the generic kernel
(28 % 8 != 0).  The data gradient swaps Cin and Cout, so conv2_1's runs v2<64> without resident weights.
"""
import contextlib
import time

import pytest
import torch
import torch.nn.functional as F

import detgen
from bench_conv import BATCH, VGG16_LAYERS

pytestmark = pytest.mark.gpu

# |out - ref| <= ROUND * max(|out|, |ref|) + c * absref, element-wise (check_bound).  ROUND: the TF32 rounding on store
# (10 explicit mantissa bits, round to nearest); c: the fp32 accumulation, relative to the same operation applied to
# |inputs| and |weights|.  Each c is at least 6x the worst (|err| - rounding term) / absref measured over every test
# below on an H100 SXM (80 GB HBM3, 700 W): forward and data gradient 1.15e-6 (conv4_2 / conv5_3 forward), weight
# gradient 4.6e-6 (conv4_3), 3xTF32 2.1e-6 (conv4_3 forward).
# The weight-gradient figure is for zero-mean dY, whose sums cancel.  Where dY has a per-channel mean the sums are
# coherent and the error grows with the pixels each split-K CTA accumulates: 5.4e-5 at conv5_1, batch 32 (14,336 pixels
# per CTA), with half the elements beyond 2^-16: a bias of the accumulation, not a local defect, which the tests leave
# out by using zero-mean gradients.
ROUND = 2.0 ** -11
C_TF32 = 2.0 ** -17           # forward and data gradient (9 Cin terms per output), single-pass TF32
C_TF32_WGRAD = 2.0 ** -15     # weight and bias gradients (a sum over every pixel of the batch), single-pass TF32
C_PRECISE = 2.0 ** -16        # 3xTF32, every direction
CHUNK = 4                     # images per fp64 reference evaluation
GUARD = 12345.0
CODE_GUARD = 0xA5
HK_ERR_UNSUPPORTED = -3
LAYERS = {name: (H, cin, cout, pool) for name, H, cin, cout, pool in VGG16_LAYERS}
LAST = VGG16_LAYERS[-1][0]    # its pool writes NCHW: the input of the pooling heads


@contextlib.contextmanager
def _fp32_exact():
    """fp32 convolutions without TF32 (the scale references)"""
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cudnn.allow_tf32 = old


def _nchw(t):
    return t.permute(0, 3, 1, 2).contiguous()


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


def _guarded(shape, dtype=torch.float32, fill=float('nan'), guard=GUARD):
    """output buffer filled with `fill` (NaN: a skipped element fails the bound) followed by 64 KB of guard words"""
    n = 1
    for d in shape:
        n *= d
    extra = 65536 // torch.empty((), dtype=dtype).element_size()
    buf = torch.full((n + extra,), fill, device='cuda', dtype=dtype)
    buf[n:] = guard
    return buf[:n].view(shape), buf[n:]


def _assert_guard(g, guard=GUARD, tag=''):
    assert bool((g == guard).all()), f'{tag}: store past the end of the output'


def _tf32(t):
    return detgen.tf32_rna(t)


def _gen(seed):
    return torch.Generator(device='cuda').manual_seed(seed)


def _randn(shape, g, scale=1.0):
    return torch.randn(shape, device='cuda', generator=g) * scale


def _rounding_term(out, ref):
    return ROUND * torch.fmax(out.double().abs(), ref.double().abs())


def bound_of(out, ref, absref, c, rnd=True):
    """element-wise bound: c * absref, plus the TF32 rounding on store where the kernel rounds its output"""
    b = c * absref.double()
    return b + _rounding_term(out, ref) if rnd else b


def _worst(ratio):
    ratio = torch.nan_to_num(ratio, nan=float('inf'))
    k = int(ratio.argmax())
    return float(ratio.flatten()[k]), [int(i) for i in torch.unravel_index(torch.tensor(k), tuple(ratio.shape))]


def check_bound(out, ref, absref, c, tag, rnd=True, n0=0, bound=None, names=('image', 'h', 'w', 'channel')):
    """Assert |out - ref| <= ROUND * max(|out|, |ref|) + c * absref for every element (without the first term when
    rnd is False; `bound` replaces the whole right-hand side where given).  out, ref and absref have one shape; n0 is
    the index of out's first element along dimension 0 in the full tensor.

    Prints the worst |out - ref| / bound and the worst share of c * absref that the error beyond the rounding term
    takes: the rounding term alone can bring the first near 1 whatever c is, so the second is the margin of c.
    Returns that share; on failure reports the number of violating elements and the worst one's index (`names`)."""
    o, r = out.double(), ref.double()
    err = (o - r).abs()
    zero = torch.zeros((), dtype=err.dtype, device=err.device)
    if bound is None:
        cterm = c * absref.double()
        excess = (err - _rounding_term(o, r)).clamp_min(0) if rnd else err
        share, _ = _worst(torch.where(excess == 0, zero, excess / cterm))
        del excess
        bound = bound_of(o, r, absref, c, rnd)
    else:
        share = None
    worst, idx = _worst(torch.where(err == 0, zero, err / bound))
    share = worst if share is None else share
    idx[0] += n0
    where = ', '.join(f'{nm} {i}' for nm, i in zip(names, idx))
    print(f'{tag}: worst |err|/bound {worst:.3g} ({where}); c-term share {share:.3g}', flush=True)
    nbad = int((~(err <= bound)).sum())
    if nbad:
        j = tuple([idx[0] - n0] + idx[1:])
        raise AssertionError(f'{tag}: {nbad} of {err.numel()} elements out of bound; worst at ({where}): out '
                             f'{float(o[j]):.9g} ref {float(r[j]):.9g} bound {float(bound[j]):.3g} ratio {worst:.3g}')
    return share


def _pack(w):
    from hawkeye_b200 import _lib
    cout, cin = w.shape[:2]
    wf = torch.empty(9 * cout * cin, device='cuda')
    wd = torch.empty(9 * cout * cin, device='cuda')
    _lib.call('hk_conv3x3_pack_weights', w, wf, wd, cout, cin, _lib.stream_ptr())
    return wf, wd


def _fwd(x, wf, b, cout, relu=1):
    from hawkeye_b200 import _lib
    N, H, W, cin = x.shape
    y, g = _guarded((N, H, W, cout))
    _lib.call('hk_conv3x3_fwd', x, wf, b, y, N, H, W, cin, cout, relu, _lib.stream_ptr())
    torch.cuda.synchronize()
    _assert_guard(g, tag='fwd')
    return y


def _wgrad(x, dy, dw, db, accumulate):
    from hawkeye_b200 import _lib
    N, H, W, cin = x.shape
    cout = dy.shape[-1]
    nb = _lib.query('hk_conv3x3_wgrad_workspace_bytes', cin, cout)
    ws = torch.empty(nb, dtype=torch.uint8, device='cuda')
    _lib.call('hk_conv3x3_wgrad_acc', x, dy, dw, db, N, H, W, cin, cout, ws, nb, int(accumulate), _lib.stream_ptr())
    torch.cuda.synchronize()


def _conv_ref(x, w, b):
    """fp64 pre-activation conv2d and its fp32 scale conv2d(|x|, |w|) + |b|, NHWC, of an NHWC chunk"""
    xc = _nchw(x)
    ref = _nhwc(F.conv2d(xc.double(), w.double(), None if b is None else b.double(), padding=1))
    with _fp32_exact():
        absref = _nhwc(F.conv2d(xc.abs(), w.abs(), None if b is None else b.abs(), padding=1))
    return ref, absref


def _dgrad_ref(dy, w):
    """fp64 input gradient of conv2d(., w, padding=1) (conv_transpose2d) and its fp32 scale, NHWC"""
    dc = _nchw(dy)
    ref = _nhwc(F.conv_transpose2d(dc.double(), w.double(), padding=1))
    with _fp32_exact():
        absref = _nhwc(F.conv_transpose2d(dc.abs(), w.abs(), padding=1))
    return ref, absref


def _wgrad_ref(x, dy, cin, cout, chunk=CHUNK):
    """fp64 weight and bias gradients of conv2d(x, ., padding=1) against dy, summed chunk by chunk, and their fp32
    scales computed from |x|, |dy|"""
    gw = torch.zeros(cout, cin, 3, 3, dtype=torch.float64, device='cuda')
    aw = torch.zeros(cout, cin, 3, 3, dtype=torch.float64, device='cuda')
    gb = torch.zeros(cout, dtype=torch.float64, device='cuda')
    ab = torch.zeros(cout, dtype=torch.float64, device='cuda')
    for n0 in range(0, x.shape[0], chunk):
        xc, dc = _nchw(x[n0:n0 + chunk]), _nchw(dy[n0:n0 + chunk])
        gw += torch.nn.grad.conv2d_weight(xc.double(), gw.shape, dc.double(), padding=1)
        gb += dc.double().sum((0, 2, 3))
        with _fp32_exact():
            aw += torch.nn.grad.conv2d_weight(xc.abs(), gw.shape, dc.abs(), padding=1).double()
        ab += dc.abs().double().sum((0, 2, 3))
        del xc, dc
    return gw, aw, gb, ab


def _windows(t):
    """NHWC (n, H, W, C) -> (n, H/2, W/2, C, 4): the 2x2 pooling windows in scan order (0 0), (0 1), (1 0), (1 1)"""
    n, H, W, C = t.shape
    return t.reshape(n, H // 2, 2, W // 2, 2, C).permute(0, 1, 3, 5, 2, 4).reshape(n, H // 2, W // 2, C, 4)


def _unwindows(t):
    n, Ho, Wo, C, _ = t.shape
    return t.reshape(n, Ho, Wo, C, 2, 2).permute(0, 1, 4, 2, 5, 3).reshape(n, 2 * Ho, 2 * Wo, C)


def _layer_inputs(H, cin, cout, N, seed, tf32=True):
    """a ReLU activation map x (NHWC), kaiming-scaled weights and a bias; TF32-representable unless tf32 is False"""
    g = _gen(seed)
    rnd = _tf32 if tf32 else (lambda t: t)
    x = rnd(torch.relu(_randn((N, H, H, cin), g)))
    w = rnd(_randn((cout, cin, 3, 3), g, (2.0 / (9 * cin)) ** 0.5))
    b = _randn((cout,), g, 0.5)
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
    xp = F.pad(_nchw(x[:1, :, :, R_CI0:R_CI0 + 32]).double(), (1, 1, 1, 1))[0]
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
    b = _tf32(b * 4.0)                       # a bias of the outputs' own size: its 1e-3 is visible beside them
    wf, _ = _pack(w)
    y = _fwd(x, wf, b, cout, relu=0)
    ref, absref = _conv_ref(x, w, b)
    tag = f'sensitivity {variant} ({layer})'
    check_bound(y, ref, absref, C_TF32, f'{tag} unedited')
    bad = y.clone()
    bad[0, R_H0:R_H0 + 8, R_W0:R_W0 + 16] -= _tap_contribution(x, w).float()
    with pytest.raises(AssertionError):
        check_bound(bad, ref, absref, C_TF32, f'{tag} one tap missing')
    bad = y.clone()
    bad[0, R_H0, R_W0:R_W0 + 16] = y[0, R_H0 - 1, R_W0:R_W0 + 16]
    with pytest.raises(AssertionError):
        check_bound(bad, ref, absref, C_TF32, f'{tag} row repeated')
    co = int(b.abs().argmax())
    bad = y.clone()
    bad[..., co] += 1e-3 * b[co]
    with pytest.raises(AssertionError):
        check_bound(bad, ref, absref, C_TF32, f'{tag} bias x (1 + 1e-3)')


def test_bound_rejects_wgrad_defects():
    """the weight gradient at conv5_1's shape: a 16 x 8 pixel tile's share of one tap and one 32-channel chunk, one
    repeated ci row of a 64 x 64 output tile, one channel's bias gradient off by 1e-3.  Batch 2, like the forward's: the
    bias gradient of a zero-mean dY is a cancelling sum, and over the 25,088 pixels of batch 32 its largest value is
    below 1e3 * C_TF32_WGRAD * sum |dY|, so the bound cannot see a 1e-3 error in it there."""
    H, cin, cout, _ = LAYERS['conv5_1']
    x, _, _ = _layer_inputs(H, cin, cout, 2, 710)
    g = _gen(711)
    dy = _tf32(_randn((2, H, H, cout), g))
    dw, gd = _guarded((cout, cin, 3, 3))
    db, gdb = _guarded((cout,))
    _wgrad(x, dy, dw, db, 0)
    _assert_guard(gd, tag='dw')
    _assert_guard(gdb, tag='db')
    gw, aw, gb, ab = _wgrad_ref(x, dy, cin, cout)
    names = ('co', 'ci', 'kh', 'kw')
    tag = 'sensitivity wgrad (conv5_1)'
    check_bound(dw, gw, aw, C_TF32_WGRAD, f'{tag} dw unedited', rnd=False, names=names)
    check_bound(db, gb, ab, C_TF32_WGRAD, f'{tag} db unedited', rnd=False, names=('co',))
    kh, kw = R_TAP
    xp = F.pad(_nchw(x[:1, :, :, R_CI0:R_CI0 + 32]).double(), (1, 1, 1, 1))[0]
    win = xp[:, R_H0 + kh:R_H0 + kh + 8, R_W0 + kw:R_W0 + kw + 16]
    part = torch.einsum('cij,ijo->oc', win, dy[0, R_H0:R_H0 + 8, R_W0:R_W0 + 16].double())
    bad = dw.clone()
    bad[:, R_CI0:R_CI0 + 32, kh, kw] -= part.float()
    with pytest.raises(AssertionError):
        check_bound(bad, gw, aw, C_TF32_WGRAD, f'{tag} one tile of one tap missing', rnd=False, names=names)
    bad = dw.clone()
    bad[:64, 65, kh, kw] = dw[:64, 64, kh, kw]
    with pytest.raises(AssertionError):
        check_bound(bad, gw, aw, C_TF32_WGRAD, f'{tag} ci row repeated', rnd=False, names=names)
    co = int(gb.abs().argmax())
    bad = db.clone()
    bad[co] *= 1 + 1e-3
    with pytest.raises(AssertionError):
        check_bound(bad, gb, ab, C_TF32_WGRAD, f'{tag} db x (1 + 1e-3)', rnd=False, names=('co',))


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
    wb = _windows(bound_of(y[n0:n1], rr, absref, C_TF32)).amax(-1)
    win = _windows(rr)
    pref = win.amax(-1)
    worst = check_bound(p[n0:n1], pref, None, C_TF32, f'{name} pool [{n0}:{n1}]', n0=n0, bound=wb)
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
    s = _lib.stream_ptr()
    H, cin, cout, pool = LAYERS[name]
    N = BATCH
    seed = 1000 + 10 * [v[0] for v in VGG16_LAYERS].index(name)
    x, w, b = _layer_inputs(H, cin, cout, N, seed)
    wf, wd = _pack(w)
    y = _fwd(x, wf, b, cout)
    worst = {}
    if pool:
        nchw = int(name == LAST)
        Ho = H // 2
        pshape = (N, cout, Ho, Ho) if nchw else (N, Ho, Ho, cout)
        p, gp = _guarded(pshape)
        code, gc = _guarded((N, Ho, Ho, cout), torch.uint8, 255, CODE_GUARD)
        _lib.call('hk_conv3x3_fwd_pool', x, wf, b, p, code, N, H, H, cin, cout, nchw, s)
        p_unf = torch.empty(pshape, device='cuda')
        code_unf = torch.empty(N, Ho, Ho, cout, device='cuda', dtype=torch.uint8)
        _lib.call('hk_maxpool2x2_fwd_idx', y, p_unf, code_unf, N, H, H, cout, nchw, s)
        torch.cuda.synchronize()
        _assert_guard(gp, tag=f'{name} pooled')
        _assert_guard(gc, CODE_GUARD, tag=f'{name} code')
        assert torch.equal(code, code_unf), f'{name}: fused code bytes differ from hk_maxpool2x2_fwd_idx'
        del p_unf, code_unf
        p_nhwc = _nhwc(p) if nchw else p
    for n0 in range(0, N, CHUNK):
        pre, absref = _conv_ref(x[n0:n0 + CHUNK], w, b)
        r = check_bound(y[n0:n0 + CHUNK], torch.relu(pre), absref, C_TF32, f'{name} fwd [{n0}:{n0 + CHUNK}]', n0=n0)
        worst['fwd'] = max(worst.get('fwd', 0.0), r)
        if pool:
            r = _check_pool(name, y, p_nhwc, code, pre, absref, n0)
            worst['pool'] = max(worst.get('pool', 0.0), r)
        del pre, absref
    del y
    if pool:
        # pooling backward on the fused codes: dy scattered to window position code & 3 where code & 4, bit for bit
        del p, p_nhwc
        g = _gen(seed + 1)
        dyp = _tf32(_randn(pshape, g))
        dxp, gdx = _guarded((N, H, H, cout))
        _lib.call('hk_maxpool2x2_bwd_idx', code, dyp, dxp, N, H, H, cout, nchw, s)
        torch.cuda.synchronize()
        _assert_guard(gdx, tag=f'{name} pool bwd')
        dyp_nhwc = _nhwc(dyp) if nchw else dyp
        for n0 in range(0, N, CHUNK):
            c = code[n0:n0 + CHUNK]
            gv = torch.where((c & 4) != 0, dyp_nhwc[n0:n0 + CHUNK], torch.zeros((), device='cuda'))
            ref = _unwindows(torch.stack([torch.where((c & 3) == k, gv, torch.zeros((), device='cuda'))
                                          for k in range(4)], -1))
            assert torch.equal(dxp[n0:n0 + CHUNK], ref), f'{name} pool bwd [{n0}:{n0 + CHUNK}] differs from the scatter'
        del dxp, dyp, dyp_nhwc, code
    g = _gen(seed + 2)
    dy = _tf32(_randn((N, H, H, cout), g))
    for masked in (False, True):
        dx, gdx = _guarded((N, H, H, cin))
        _lib.call('hk_conv3x3_dgrad', dy, wd, x if masked else None, dx, N, H, H, cin, cout, s)
        torch.cuda.synchronize()
        _assert_guard(gdx, tag=f'{name} dgrad')
        key = 'dgrad masked' if masked else 'dgrad'
        for n0 in range(0, N, CHUNK):
            ref, absref = _dgrad_ref(dy[n0:n0 + CHUNK], w)
            if masked:
                m = x[n0:n0 + CHUNK] > 0
                ref, absref = ref * m, absref * m
            r = check_bound(dx[n0:n0 + CHUNK], ref, absref, C_TF32, f'{name} {key} [{n0}:{n0 + CHUNK}]', n0=n0)
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
    g = _gen(seed + 1)
    dy = _tf32(_randn((N, H, H, cout), g))
    gw, aw, gb, ab = _wgrad_ref(x, dy, cin, cout)
    names = ('co', 'ci', 'kh', 'kw')
    dw, gd = _guarded((cout, cin, 3, 3))
    db, gdb = _guarded((cout,))
    _wgrad(x, dy, dw, db, 0)
    _assert_guard(gd, tag='dw')
    _assert_guard(gdb, tag='db')
    rw = check_bound(dw, gw, aw, C_TF32_WGRAD, f'{name} wgrad dw', rnd=False, names=names)
    rb = check_bound(db, gb, ab, C_TF32_WGRAD, f'{name} wgrad db', rnd=False, names=('co',))
    dw0 = _randn((cout, cin, 3, 3), g, float(gw.abs().mean()))
    db0 = _randn((cout,), g, float(gb.abs().mean()))
    dw, db = dw0.clone(), db0.clone()
    _wgrad(x, dy, dw, db, 1)
    rwa = check_bound(dw, dw0.double() + gw, dw0.double().abs() + aw, C_TF32_WGRAD, f'{name} wgrad dw accumulate',
                      rnd=False, names=names)
    rba = check_bound(db, db0.double() + gb, db0.double().abs() + ab, C_TF32_WGRAD, f'{name} wgrad db accumulate',
                      rnd=False, names=('co',))
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
    s = _lib.stream_ptr()
    cout = 64
    g = _gen(3000 + W)
    x = _tf32(_randn((N, 3, H, W), g))
    w = _tf32(_randn((cout, 3, 3, 3), g, 0.2))
    b = _tf32(_randn((cout,), g, 0.5))      # the bias rides in the GEMM as column 27 of W27: TF32 like the weights
    nb0 = _lib.query('hk_conv3x3_first_fwd_workspace_bytes', N, H, W, cout)
    ws0 = torch.empty(nb0, dtype=torch.uint8, device='cuda')
    y, gy = _guarded((N, H, W, cout))
    _lib.call('hk_conv3x3_first_fwd', x, w, b, y, N, H, W, cout, ws0, nb0, s)
    torch.cuda.synchronize()
    _assert_guard(gy, tag='first fwd')
    worst = 0.0
    for n0 in range(0, N, CHUNK):
        xc = x[n0:n0 + CHUNK]
        ref = _nhwc(F.relu(F.conv2d(xc.double(), w.double(), b.double(), padding=1)))
        with _fp32_exact():
            absref = _nhwc(F.conv2d(xc.abs(), w.abs(), b.abs(), padding=1))
        worst = max(worst, check_bound(y[n0:n0 + CHUNK], ref, absref, C_TF32,
                                       f'first fwd {N}x{H}x{W} [{n0}:{n0 + CHUNK}]', n0=n0))
        del ref, absref
    del y
    dy = _tf32(_randn((N, H, W, cout), g))
    gw, aw, gb, ab = _wgrad_ref(_nhwc(x), dy, 3, cout)
    nb = _lib.query('hk_conv3x3_first_wgrad_workspace_bytes', N, H, W, cout)
    ws = torch.empty(nb, dtype=torch.uint8, device='cuda')
    dw, gd = _guarded((cout, 3, 3, 3))
    db, gdb = _guarded((cout,))
    _lib.call('hk_conv3x3_first_wgrad', ws0, dy, dw, db, N, H, W, cout, ws, nb, s)
    torch.cuda.synchronize()
    _assert_guard(gd, tag='first dw')
    _assert_guard(gdb, tag='first db')
    names = ('co', 'ci', 'kh', 'kw')
    rw = check_bound(dw, gw, aw, C_TF32_WGRAD, f'first wgrad dw {N}x{H}x{W}', rnd=False, names=names)
    rb = check_bound(db, gb, ab, C_TF32_WGRAD, f'first wgrad db {N}x{H}x{W}', rnd=False, names=('co',))
    dw0 = _randn((cout, 3, 3, 3), g, float(gw.abs().mean()))
    db0 = _randn((cout,), g, float(gb.abs().mean()))
    dw, db = dw0.clone(), db0.clone()
    _lib.call('hk_conv3x3_first_wgrad_acc', ws0, dy, dw, db, N, H, W, cout, ws, nb, 1, s)
    torch.cuda.synchronize()
    rwa = check_bound(dw, dw0.double() + gw, dw0.double().abs() + aw, C_TF32_WGRAD, f'first wgrad dw accumulate',
                      rnd=False, names=names)
    rba = check_bound(db, db0.double() + gb, db0.double().abs() + ab, C_TF32_WGRAD, f'first wgrad db accumulate',
                      rnd=False, names=('co',))
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
    s = _lib.stream_ptr()
    H, cin, cout, pool = LAYERS[name]
    N = 4
    seed = 4000 + 10 * [v[0] for v in VGG16_LAYERS].index(name)
    _lib.set_precise(1)
    try:
        x, w, b = _layer_inputs(H, cin, cout, N, seed, tf32=False)
        wf, wd = _pack(w)
        y = _fwd(x, wf, b, cout)
        pre, absref = _conv_ref(x, w, b)
        rf = check_bound(y, torch.relu(pre), absref, C_PRECISE, f'{name} precise fwd', rnd=False)
        del y, pre, absref
        if pool:
            p = torch.empty(N, H // 2, H // 2, cout, device='cuda')
            rc = _lib.query('hk_conv3x3_fwd_pool', x, wf, b, p, None, N, H, H, cin, cout, 0, s)
            assert rc == HK_ERR_UNSUPPORTED, f'hk_conv3x3_fwd_pool in 3xTF32 mode returned {rc}'
        g = _gen(seed + 1)
        dy = _randn((N, H, H, cout), g)
        dx, gdx = _guarded((N, H, H, cin))
        _lib.call('hk_conv3x3_dgrad', dy, wd, x, dx, N, H, H, cin, cout, s)
        torch.cuda.synchronize()
        _assert_guard(gdx, tag=f'{name} precise dgrad')
        ref, absref = _dgrad_ref(dy, w)
        m = x > 0
        rd = check_bound(dx, ref * m, absref * m, C_PRECISE, f'{name} precise dgrad masked', rnd=False)
        del dx, ref, absref
        gw, aw, gb, ab = _wgrad_ref(x, dy, cin, cout)
        dw, gd = _guarded((cout, cin, 3, 3))
        db, gdb = _guarded((cout,))
        _wgrad(x, dy, dw, db, 0)
        _assert_guard(gd, tag='dw')
        _assert_guard(gdb, tag='db')
        rw = check_bound(dw, gw, aw, C_PRECISE, f'{name} precise wgrad dw', rnd=False, names=('co', 'ci', 'kh', 'kw'))
        rb = check_bound(db, gb, ab, C_PRECISE, f'{name} precise wgrad db', rnd=False, names=('co',))
    finally:
        _lib.set_precise(0)
    print(f'{name} N={N} 3xTF32: worst c-term share fwd {rf:.3g} dgrad {rd:.3g} dw {rw:.3g} db {rb:.3g}; '
          f'{time.time() - t0:.1f} s, peak {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB', flush=True)
