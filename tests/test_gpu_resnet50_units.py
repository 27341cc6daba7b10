"""Every distinct unit of the ResNet-50 trunk, forward and backward, element by element against fp64, at the shapes the
train steps run: 448x448 batch 32 (MPN, APCNN, CrossX, DCL, NTS, MGE, ProtoTree) and 224x224 batch 24 (Baseline, Pairwise
Confusion) in TF32 mode, 448x448 batch 4 in 3xTF32 mode, and 448x448 batch 5 in eval mode.  ResNet-101's units have the
same shapes.

Each unit is driven through ops_resnet.Unit, the code the train step runs: forward(save=True), bn_backward on its record,
then Unit.backward (with an addend on the 1x1 units, so that the dgrad GEMM's fused epilogue runs at production M).  Each
stage is compared with fp64 of the same operation on the fp32 values it was given.  In TF32 mode those values are
TF32-representable (the inputs here are rounded, and the im2col, the BN outputs and dC are rounded on store), so every
tensor-core product is exact and what is left is fp32 accumulation plus, where the kernel rounds its output, one TF32
rounding (kernel_check.RND = 2^-11).  The bound of every check is |out - ref| <= RND * max(|out|, |ref|)
(where the output is rounded) + c * scale, with `scale` the same expression over absolute values:

  conv output c        scale = the same conv of |x|, |w|                                     C_CONV (C_PRECISE)
  dx                   scale = the transposed conv of |dC|, |w|, plus |addend|               C_CONV (C_PRECISE)
  dW                   scale = the weight gradient of |x|, |dC|                              C_WGRAD (C_PRECISE)
  BN output y          scale = |gamma| invstd (|c| + |mean|) + |beta| + |res|                C_BN
  dC                   scale = |gamma| invstd (|g'| + sum|g'|/P + |xhat| sum|g' xhat|/P)     C_BN
  mean, invstd         scale = sigma, invstd                                                 C_SUMS
  dbeta, dgamma        scale = sum|g'|, sum|g' xhat|                                         C_SUMS

with g' = dy masked by the forward's y > 0 and xhat = (c - mean) invstd from the kernel's own fp32 statistics.  The |mean|
term of the y scale covers the fp32 rounding of c - mean where the mean is large.  Unit allocates its outputs with
torch.empty, so every kernel is also called once more through the C ABI into NaN-filled buffers followed by guard words and
must give the Unit's bits (the 3x3 weight gradient, which adds its splits with atomics, is held to its bound instead).

The fp64 references run on the GPU, CHUNK images at a time: a 1x1 conv is one DGEMM, a k x k conv k^2 shifted DGEMMs.
"""
import time

import pytest
import torch
import torch.nn.functional as F

import detgen
from oracle.hop_oracle import RESNET50_LAYERS
from kernel_check import Bound, Out, Worst, abi, c_bound, check, rnd_bound, workspace

# Each constant is at least 4x the worst (|err| - rounding term) / scale measured over every check of this file (the
# four sweeps of test_unit) on an H100 80GB HBM3 at 700 W:
#   C_CONV     1.54e-6  tf32-448-b32 layer4.1.conv1 c (K = 2048)                  4.9x
#   C_WGRAD    3.9e-6   tf32-448-b32 layer4.0.conv2 dW (the stride-2 3x3)         7.9x
#   C_BN       1.9e-7   precise-448-b4 layer1.0.conv3 y (with its residual)       5.0x
#   C_SUMS     4.5e-6   precise-448-b4 layer4.0.downsample invstd (P = 784)       6.8x
#   C_PRECISE  1.8e-6   precise-448-b4 layer4.1.conv2 dx                          8.6x
# The invstd error is the largest of the sums: the variance is E[d^2] - E[d]^2 of the fp32 sums of d = c - c[0], which
# cancels where a channel's first value lies far from its mean.  Over the train-mode sweeps the mean is within 1.2e-6
# sigma of fp64.
C_CONV = 2.0 ** -17
C_WGRAD = 2.0 ** -15
C_BN = 2.0 ** -20
C_SUMS = 2.0 ** -15
C_PRECISE = 2.0 ** -16
# The max-pool gradient adds at most 4 fp32 terms per element: 3 roundings, within 2^-22 of sum |terms| by analysis
# (the worst measured is 0.70 of it).
CHUNK = 4
BN_EPS = 1e-5

# sweep: (image side, batch, precise, train mode)
SWEEPS = {'tf32-448-b32': (448, 32, 0, True), 'tf32-224-b24': (224, 24, 0, True),
          'precise-448-b4': (448, 4, 1, True), 'eval-448-b5': (448, 5, 0, False)}
# kind -> (kernel size, stride, padding)
GEOM = {'stem': (7, 2, 3), '1x1': (1, 1, 0), '1x1s2': (1, 2, 0), '3x3': (3, 1, 1), '3x3s2': (3, 2, 1)}


def resnet50_units(size):
    """(name, kind, input side, cin, cout, relu, residual) of the 24 distinct units of ResNet-50 on size x size images:
    the stem, then per layer block 0's conv1, conv2, downsample and conv3 (with its residual) and the later blocks' conv1
    and, where block 0's conv2 has stride 2 and so another shape, conv2"""
    units = [('stem', 'stem', size, 3, 64, True, False)]
    H, cin = size // 4, 64                     # after the stem's stride and the max-pool
    for li, (planes, blocks, stride) in enumerate(RESNET50_LAYERS):
        L, Ho, s2 = f'layer{li + 1}', H // stride, stride == 2
        units += [(f'{L}.0.conv1', '1x1', H, cin, planes, True, False),
                  (f'{L}.0.conv2', '3x3s2' if s2 else '3x3', H, planes, planes, True, False),
                  (f'{L}.0.downsample', '1x1s2' if s2 else '1x1', H, cin, 4 * planes, False, False),
                  (f'{L}.0.conv3', '1x1', Ho, planes, 4 * planes, True, True),
                  (f'{L}.1.conv1', '1x1', Ho, 4 * planes, planes, True, False)]
        if s2 and blocks > 1:
            units.append((f'{L}.1.conv2', '3x3', Ho, planes, planes, True, False))
        H, cin = Ho, 4 * planes
    return units


UNITS = {u[0]: u for u in resnet50_units(448)}


# ------------------------------------------------------------------------------------------------------------------
# 1. fp64 restatements (device-agnostic, NHWC)
# ------------------------------------------------------------------------------------------------------------------
def _taps(k, stride, Ho, Wo):
    for kh in range(k):
        for kw in range(k):
            yield kh, kw, slice(kh, kh + stride * (Ho - 1) + 1, stride), slice(kw, kw + stride * (Wo - 1) + 1, stride)


def conv_nhwc(x, w, stride, pad):
    """fp64 conv2d of an NHWC map with [Cout, Cin, k, k] weights, as k^2 shifted GEMMs -> NHWC"""
    n, H, W, _ = x.shape
    cout, _, k, _ = w.shape
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    xp, wd = F.pad(x.double(), (0, 0, pad, pad, pad, pad)), w.double()
    out = torch.zeros(n, Ho, Wo, cout, dtype=torch.float64, device=x.device)
    for kh, kw, sh, sw in _taps(k, stride, Ho, Wo):
        out += xp[:, sh, sw] @ wd[:, :, kh, kw].T
    return out


def conv_nhwc_t(dc, w, stride, pad, H, W):
    """fp64 adjoint of conv_nhwc in its input: the NHWC input gradient [n, H, W, Cin] of the output gradient dc"""
    n, Ho, Wo, _ = dc.shape
    _, cin, k, _ = w.shape
    dxp = torch.zeros(n, H + 2 * pad, W + 2 * pad, cin, dtype=torch.float64, device=dc.device)
    dd, wd = dc.double(), w.double()
    for kh, kw, sh, sw in _taps(k, stride, Ho, Wo):
        dxp[:, sh, sw] += dd @ wd[:, :, kh, kw]
    return dxp[:, pad:pad + H, pad:pad + W]


def wgrad_nhwc(x, dc, k, stride, pad):
    """fp64 weight gradient [Cout, Cin, k, k] of conv_nhwc(x, ., stride, pad) against the output gradient dc"""
    n, Ho, Wo, cout = dc.shape
    cin = x.shape[-1]
    xp, dd = F.pad(x.double(), (0, 0, pad, pad, pad, pad)), dc.double().reshape(-1, cout)
    gw = torch.empty(cout, cin, k, k, dtype=torch.float64, device=x.device)
    for kh, kw, sh, sw in _taps(k, stride, Ho, Wo):
        gw[:, :, kh, kw] = dd.T @ xp[:, sh, sw].reshape(-1, cin)
    return gw


def bn_stats_ref(c):
    """fp64 batch mean and biased variance of an NHWC map per channel"""
    cd = c.reshape(-1, c.shape[-1]).double()
    m = cd.mean(0)
    return m, (cd - m).pow(2).mean(0)


def bn_fwd_ref(c, mean, invstd, gamma, beta, res, relu):
    """fp64 of the BN (+ residual) (+ ReLU) expression on the given statistics -> (y, scale of its error)"""
    m, i, g, b = (t.double() for t in (mean, invstd, gamma, beta))
    cd = c.double()
    y = (cd - m) * i * g + b
    a = g.abs() * i * (cd.abs() + m.abs()) + b.abs()
    if res is not None:
        y, a = y + res.double(), a + res.double().abs()
    return (y.clamp_min(0) if relu else y), a


def bn_bwd_sums(c, gp, mean, invstd):
    """(dbeta, dgamma, sum|g'|, sum|g' xhat|) in fp64 from the masked output gradient g'"""
    C = c.shape[-1]
    xh = (c.double() - mean.double()) * invstd.double()
    g = gp.double()
    return tuple(t.reshape(-1, C).sum(0) for t in (g, g * xh, g.abs(), (g * xh).abs()))


def bn_bwd_ref(c, gp, gamma, mean, invstd, sums, P, frozen):
    """fp64 input gradient of BN from the masked output gradient g' -> (dC, scale of its error); ``frozen``: constant
    statistics (eval mode), dC = gamma invstd g'"""
    s = gamma.double().abs() * invstd.double()
    g = gp.double()
    if frozen:
        return gamma.double() * invstd.double() * g, s * g.abs()
    db, dg, ab, ag = sums
    xh = (c.double() - mean.double()) * invstd.double()
    dc = gamma.double() * invstd.double() * (g - db / P - xh * dg / P)
    return dc, s * (g.abs() + ab / P + xh.abs() * ag / P)


def maxpool_ref(y):
    """MaxPool2d(3, 2, 1) of an NHWC map -> (max, index 0..8 of the first maximum in scan order)"""
    n, H, W, C = y.shape
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    yp = F.pad(y, (0, 0, 1, 1, 1, 1), value=float('-inf'))
    win = torch.stack([yp[:, sh, sw] for _, _, sh, sw in _taps(3, 2, Ho, Wo)], -1)
    return win.amax(-1), win.argmax(-1)


def maxpool_bwd_ref(arg, dy, H, W):
    """fp64 scatter of dy to the recorded window positions -> (dx, sum of |terms| per element)"""
    n, Ho, Wo, C = dy.shape
    dx = torch.zeros(n, H + 2, W + 2, C, dtype=torch.float64, device=dy.device)
    ax = torch.zeros_like(dx)
    for k, (_, _, sh, sw) in enumerate(_taps(3, 2, Ho, Wo)):
        t = torch.where(arg == k, dy.double(), torch.zeros((), dtype=torch.float64, device=dy.device))
        dx[:, sh, sw] += t
        ax[:, sh, sw] += t.abs()
    return dx[:, 1:H + 1, 1:W + 1], ax[:, 1:H + 1, 1:W + 1]


# ------------------------------------------------------------------------------------------------------------------
# 2. defects the bounds must reject, as edits of an output (shared by the CPU self-tests and the GPU sensitivity tests)
# ------------------------------------------------------------------------------------------------------------------
def drop_k_slice(c, xin, w, r0, k0):
    """1x1 conv output c without the products of input channels k0..k0+31 in rows r0..r0+127 (one 128-row tile)"""
    cm = c.reshape(-1, c.shape[-1]).clone()
    part = xin.reshape(-1, xin.shape[-1])[r0:r0 + 128, k0:k0 + 32].double() @ w.reshape(w.shape[0], -1)[:, k0:k0 + 32].double().T
    cm[r0:r0 + 128] -= part.to(cm.dtype)
    return cm.view(c.shape)


def drop_tap(c, x, w, stride, h0, w0, th, tw, tap, ci0):
    """3x3 conv output c (padding 1) without tap (kh, kw) of input channels ci0..ci0+31 over the th x tw output tile at
    (h0, w0) of image 0"""
    kh, kw = tap
    xp = F.pad(x[:1].double(), (0, 0, 1, 1, 1, 1))[0]
    win = xp[kh + stride * h0:kh + stride * (h0 + th - 1) + 1:stride, kw + stride * w0:kw + stride * (w0 + tw - 1) + 1:stride,
             ci0:ci0 + 32]
    bad = c.clone()
    bad[0, h0:h0 + th, w0:w0 + tw] -= (win @ w[:, ci0:ci0 + 32, kh, kw].double().T).to(c.dtype)
    return bad


def wrong_phase_row(c, x, w, h0):
    """stride-2 3x3 conv output c with row h0 of image 0 read from input rows 2 h0 .. 2 h0 + 2 instead of 2 h0 - 1 .. 2 h0 + 1"""
    xs = F.pad(x[:1, 1:], (0, 0, 0, 0, 0, 1))
    bad = c.clone()
    bad[0, h0] = conv_nhwc(xs, w, 2, 1)[0, h0].to(c.dtype)
    return bad


def drop_stem_column(c, cols, w147, p0, col):
    """stem GEMM output c [P, Cout] without im2col column `col` over pixels p0..p0+127"""
    bad = c.reshape(-1, c.shape[-1]).clone()
    bad[p0:p0 + 128] -= (cols[p0:p0 + 128, col:col + 1].double() * w147[:, col].double()).to(bad.dtype)
    return bad.view(c.shape)


def drop_bn_block(db, dg, gp, xh, ch, nblk, j):
    """dbeta, dgamma without partial block j (of nblk over the P rows) of channel ch"""
    C = gp.shape[-1]
    g, x = gp.reshape(-1, C).double(), xh.reshape(-1, C).double()
    per = -(-g.shape[0] // nblk)
    rows = slice(j * per, (j + 1) * per)
    bdb, bdg = db.clone(), dg.clone()
    bdb[ch] -= g[rows, ch].sum().to(db.dtype)
    bdg[ch] -= (g[rows, ch] * x[rows, ch]).sum().to(dg.dtype)
    return bdb, bdg


def drop_split(dw, xin, dc, S, j):
    """matrix-form weight gradient dw [Cout, K] = dc^T xin without split j of S over the pixels"""
    K, cout = xin.shape[-1], dc.shape[-1]
    xm, dm = xin.reshape(-1, K), dc.reshape(-1, cout)
    per = xm.shape[0] // S
    rows = slice(j * per, (j + 1) * per)
    return dw - (dm[rows].double().T @ xm[rows].double()).to(dw.dtype)


def drop_rows(dw, x, g, n, r0, r1):
    """stride-1 3x3 weight gradient dw without output rows r0..r1-1 of image n"""
    gi = torch.zeros_like(g[n:n + 1])
    gi[:, r0:r1] = g[n:n + 1, r0:r1]
    return dw - wgrad_nhwc(x[n:n + 1], gi, 3, 1, 1).to(dw.dtype)


def rejected(bad, ref, absref, c, tag, rnd=False, names=('image', 'h', 'w', 'channel')):
    """assert that check rejects `bad` and that its worst violation is at least 2x the bound -> that ratio"""
    bound = Bound(c * absref.double(), rounded=rnd)
    b = bound.total(bad, ref)
    err = (bad.double() - ref.double()).abs()
    ratio = float(torch.where(err == 0, torch.zeros_like(err), err / b).max())
    with pytest.raises(AssertionError):
        check(bad, ref, bound, tag, names=names)
    print(f'{tag}: rejected, violation ratio {ratio:.3g}', flush=True)
    assert ratio >= 2, f'{tag}: violation ratio {ratio:.3g} < 2'
    return ratio


# ------------------------------------------------------------------------------------------------------------------
# 3. CPU self-tests of the restatements and of the bounds' sensitivity
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('k,stride,pad,H', [(1, 1, 0, 6), (1, 2, 0, 6), (1, 2, 0, 7), (3, 1, 1, 6), (3, 2, 1, 6),
                                            (3, 2, 1, 7), (7, 2, 3, 10)])
def test_conv_restatement_matches_autograd(k, stride, pad, H):
    g = torch.Generator().manual_seed(10 * k + H)
    x = torch.randn(2, 5, H, H + 1, generator=g, dtype=torch.float64, requires_grad=True)
    w = torch.randn(4, 5, k, k, generator=g, dtype=torch.float64, requires_grad=True)
    y = F.conv2d(x, w, stride=stride, padding=pad)
    dy = torch.randn(y.shape, generator=g, dtype=torch.float64)
    dx, dw = torch.autograd.grad(y, (x, w), dy)
    xh, dyh = x.detach().permute(0, 2, 3, 1), dy.permute(0, 2, 3, 1)
    torch.testing.assert_close(conv_nhwc(xh, w.detach(), stride, pad), y.detach().permute(0, 2, 3, 1))
    torch.testing.assert_close(conv_nhwc_t(dyh, w.detach(), stride, pad, H, H + 1), dx.permute(0, 2, 3, 1))
    torch.testing.assert_close(wgrad_nhwc(xh, dyh, k, stride, pad), dw)
    if (k, stride) == (3, 2) and H % 2 == 0:
        xs = torch.randn(2, 5, H, H, generator=g, dtype=torch.float64)
        d2 = torch.randn(2, 4, H // 2, H // 2, generator=g, dtype=torch.float64)
        ct = F.conv_transpose2d(d2, w.detach(), stride=2, padding=1, output_padding=1)
        torch.testing.assert_close(conv_nhwc_t(d2.permute(0, 2, 3, 1), w.detach(), 2, 1, H, H), ct.permute(0, 2, 3, 1))
        assert ct.shape == xs.shape


@pytest.mark.parametrize('relu,res', [(True, False), (True, True), (False, False)])
def test_bn_restatement_matches_autograd(relu, res):
    g = torch.Generator().manual_seed(20 + 2 * relu + res)
    c = (torch.randn(3, 4, 5, 8, generator=g, dtype=torch.float64) * 2 + 0.5).requires_grad_(True)
    gamma = (1 + 0.1 * torch.randn(8, generator=g, dtype=torch.float64)).requires_grad_(True)
    beta = (0.1 * torch.randn(8, generator=g, dtype=torch.float64)).requires_grad_(True)
    r = torch.randn(3, 4, 5, 8, generator=g, dtype=torch.float64).requires_grad_(True) if res else None
    dy = torch.randn(3, 4, 5, 8, generator=g, dtype=torch.float64)
    mean, var = bn_stats_ref(c.detach())
    invstd = (var + BN_EPS).rsqrt()
    for frozen in (False, True):
        z = F.batch_norm(c.permute(0, 3, 1, 2), mean if frozen else None, var if frozen else None, gamma, beta,
                         training=not frozen, eps=BN_EPS).permute(0, 2, 3, 1)
        if r is not None:
            z = z + r
        y = F.relu(z) if relu else z
        yref, _ = bn_fwd_ref(c.detach(), mean, invstd, gamma.detach(), beta.detach(),
                             None if r is None else r.detach(), relu)
        torch.testing.assert_close(yref, y.detach())
        ins = (c, gamma, beta) + ((r,) if r is not None else ())
        grads = torch.autograd.grad(y, ins, dy)
        gp = dy * (y.detach() > 0) if relu else dy
        sums = bn_bwd_sums(c.detach(), gp, mean, invstd)
        dc, _ = bn_bwd_ref(c.detach(), gp, gamma.detach(), mean, invstd, sums, c[..., 0].numel(), frozen)
        torch.testing.assert_close(dc, grads[0])
        torch.testing.assert_close(sums[1], grads[1])
        torch.testing.assert_close(sums[0], grads[2])
        if r is not None:
            torch.testing.assert_close(gp, grads[3])


def test_maxpool_restatement_matches_autograd():
    g = torch.Generator().manual_seed(30)
    y = torch.randn(2, 4, 9, 10, generator=g, dtype=torch.float64, requires_grad=True)
    p = F.max_pool2d(y, 3, 2, 1)
    dp = torch.randn(p.shape, generator=g, dtype=torch.float64)
    (dx,) = torch.autograd.grad(p, y, dp)
    val, arg = maxpool_ref(y.detach().permute(0, 2, 3, 1))
    torch.testing.assert_close(val, p.detach().permute(0, 2, 3, 1), rtol=0, atol=0)
    ref, _ = maxpool_bwd_ref(arg, dp.permute(0, 2, 3, 1), 9, 10)
    torch.testing.assert_close(ref, dx.permute(0, 2, 3, 1))
    ties = torch.zeros(1, 3, 3, 4, dtype=torch.float64)      # an all-zero window: the first position wins
    assert int(maxpool_ref(ties)[1].max()) == 4 and int(maxpool_ref(ties)[1][0, 1, 1, 0]) == 0


def _fake(ref, rnd):
    """what an exact kernel would store: fp32 of the fp64 result, TF32-rounded where the kernel rounds"""
    out = ref.float()
    return detgen.tf32_rna(out) if rnd else out


def test_cpu_bounds_reject_defects():
    """each defect of the GPU sensitivity tests, applied to exact results of synthetic data, fails its bound"""
    g = torch.Generator().manual_seed(40)
    tf = detgen.tf32_rna
    # 1x1 forward, K = 256: one 32-wide K slice of one 128-row tile
    x = tf(torch.relu(torch.randn(1, 16, 16, 256, generator=g)))
    w = tf(torch.randn(64, 256, 1, 1, generator=g) * (2 / 256) ** 0.5)
    ref, a = conv_nhwc(x, w, 1, 0), conv_nhwc(x.abs(), w.abs(), 1, 0)
    rejected(drop_k_slice(_fake(ref, False), x, w, 128, 96), ref, a, C_CONV, 'cpu 1x1 K slice')
    # 3x3 stride 2: one tap of one 32-channel chunk over an 8 x 8 tile; one row at the wrong stride phase
    x = tf(torch.relu(torch.randn(1, 32, 32, 64, generator=g)))
    w = tf(torch.randn(64, 64, 3, 3, generator=g) * (2 / 576) ** 0.5)
    ref, a = conv_nhwc(x, w, 2, 1), conv_nhwc(x.abs(), w.abs(), 2, 1)
    out = _fake(ref, True)
    rejected(drop_tap(out, x, w, 2, 8, 0, 8, 8, (0, 2), 32), ref, a, C_CONV, 'cpu 3x3s2 tap', rnd=True)
    rejected(wrong_phase_row(out, x, w, 5), ref, a, C_CONV, 'cpu 3x3s2 stride phase', rnd=True)
    # stem: one im2col column over 128 pixels
    img = tf(torch.randn(1, 3, 32, 32, generator=g))
    w7 = tf(torch.randn(64, 3, 7, 7, generator=g) * (2 / 147) ** 0.5)
    cols = F.unfold(img, 7, padding=3, stride=2)[0].T
    ih = img.permute(0, 2, 3, 1)
    ref, a = conv_nhwc(ih, w7, 2, 3), conv_nhwc(ih.abs(), w7.abs(), 2, 3)
    rejected(drop_stem_column(_fake(ref, False), cols, w7.reshape(64, 147), 64, 49 + 24), ref, a, C_CONV,
             'cpu stem column')
    # BN statistics: one channel's mean by 1e-4 sigma, one channel's invstd by 1 + 1e-4
    c = torch.randn(4, 8, 8, 16, generator=g) * 3 + 5
    m, v = bn_stats_ref(c)
    sig, inv = v.sqrt(), (v + BN_EPS).rsqrt()
    bad = m.float()
    bad[3] += 1e-4 * sig[3]
    rejected(bad, m, sig, C_SUMS, 'cpu BN mean + 1e-4 sigma', names=('channel',))
    bad = inv.float()
    bad[3] *= 1 + 1e-4
    rejected(bad, inv, inv, C_SUMS, 'cpu BN invstd x (1 + 1e-4)', names=('channel',))
    # BN backward: one partial block of one channel's sums
    mean, invstd = m.float(), inv.float()
    gp = torch.randn(c.shape, generator=g) * (c > 5)
    db, dg, ab, ag = bn_bwd_sums(c, gp, mean, invstd)
    xh = (c.double() - mean.double()) * invstd.double()
    bdb, bdg = drop_bn_block(db.float(), dg.float(), gp, xh, 5, 4, 2)
    rejected(bdb, db, ab, C_SUMS, 'cpu BN dbeta block', names=('channel',))
    rejected(bdg, dg, ag, C_SUMS, 'cpu BN dgamma block', names=('channel',))
    # matrix-form weight gradient: one of 16 splits
    dc = tf(torch.randn(1024, 64, generator=g))
    xm = tf(torch.randn(1024, 160, generator=g))
    gw, aw = dc.double().T @ xm.double(), dc.double().abs().T @ xm.double().abs()
    rejected(drop_split(gw.float(), xm, dc, 16, 5), gw, aw, C_WGRAD, 'cpu matconv split', names=('co', 'k'))
    # 3x3 weight gradient at 14 x 14: rows 12-13 of one image
    x = tf(torch.relu(torch.randn(4, 14, 14, 32, generator=g)))
    dcm = tf(torch.randn(4, 14, 14, 32, generator=g))
    gw, aw = wgrad_nhwc(x, dcm, 3, 1, 1), wgrad_nhwc(x.abs(), dcm.abs(), 3, 1, 1)
    rejected(drop_rows(gw.float(), x, dcm, 1, 12, 14), gw, aw, C_WGRAD, 'cpu 3x3 wgrad rows 12-13',
             names=('co', 'ci', 'kh', 'kw'))


# ------------------------------------------------------------------------------------------------------------------
# 4. the production path on the GPU
# ------------------------------------------------------------------------------------------------------------------
WORST = Worst()


def _chk(const, out, ref, absref, c, tag, rnd=True, **kw):
    return WORST.add(const, check(out, ref, (rnd_bound if rnd else c_bound)(absref, c), tag, **kw), tag)


def _gemm(A, B, b_mn, M, N, K, D=None):
    """the GEMM of conv1x1_fwd (B = w [N, K]) or conv1x1_dgrad (b_mn: B = w [K, N], D: the epilogue addend)"""
    (C,) = abi('hk_gemm_tf32', A, 0, K, 0, B, int(b_mn), N if b_mn else K, 0, Out((M, N)), N, 0, 0, M, N, K, 1, 1.0,
               None, 0.0, D, 0 if D is None else N, 0, 0.0 if D is None else 1.0, None, 0)
    return C


def _inputs(spec, N, seed, tf32):
    """seeded unit inputs: an image (stem, normalised) or a post-ReLU map, kaiming weights, gamma = 1 + 0.1 randn,
    beta = 0.1 randn, a residual on conv3, the output gradient dy; TF32-representable (but dy) where tf32"""
    _, kind, H, cin, cout, _, has_res = spec
    k, stride, _ = GEOM[kind]
    Ho = (H - 1) // stride + 1
    g = torch.Generator(device='cuda').manual_seed(seed)
    rnd = detgen.tf32_rna if tf32 else (lambda t: t)

    def randn(*shape):
        return torch.randn(shape, device='cuda', generator=g)
    x = rnd(randn(N, 3, H, H)) if kind == 'stem' else rnd(torch.relu(randn(N, H, H, cin)))
    w = rnd(randn(cout, cin, k, k) * (2.0 / (k * k * cin)) ** 0.5)
    gamma, beta = 1 + 0.1 * randn(cout), 0.1 * randn(cout)
    res = rnd(randn(N, Ho, Ho, cout)) if has_res else None
    return x, w, gamma, beta, res, randn(N, Ho, Ho, cout), g


def run_unit(spec, N, seed, precise=False, training=True):
    """ops_resnet.Unit on seeded inputs: forward(save=True), bn_backward on its record (twice: bit-identical), backward
    (with an addend on the 1x1 units) -> dict of inputs and outputs"""
    from hawkeye_b200 import _lib, ops_resnet
    _, kind, H, cin, cout, relu, has_res = spec
    x, w, gamma, beta, res, dy, g = _inputs(spec, N, seed, not precise)
    u = ops_resnet.Unit(kind, None, torch.nn.BatchNorm2d(cout).cuda(), relu)
    if not training:     # running statistics of the scale a trained network has: one train step with momentum 1
        u.bn.momentum = 1.0
        u.forward(x, w, gamma, beta, res, False, True)
        u.bn.momentum = 0.1
    rm0, rv0 = u.bn.running_mean.clone(), u.bn.running_var.clone()
    y, rec = u.forward(x, w, gamma, beta, res, True, training)
    if not training:
        assert torch.equal(u.bn.running_mean, rm0) and torch.equal(u.bn.running_var, rv0), 'eval forward moved the stats'
    mask_beta = beta if relu and not has_res else None
    args = (rec['c'], rec['y'], dy, gamma, mask_beta, rec['mean'], rec['invstd'], has_res, relu, not training, rec['P'],
            cout, _lib.stream_ptr())
    dc, dres, dg, db = ops_resnet.bn_backward(*args)
    again = ops_resnet.bn_backward(*args)
    assert all(a is b or torch.equal(a, b) for a, b in zip((dc, dres, dg, db), again)), 'bn_backward is not deterministic'
    addend = None
    if kind in ('1x1', '1x1s2'):
        scale = float(dc.pow(2).mean().sqrt()) * (cout * float(w.pow(2).mean())) ** 0.5
        addend = torch.randn(N, H, H, cin, device='cuda', generator=g) * scale
    dx, dres_u, dw, dg_u, db_u = u.backward(rec, dy, need_dx=kind != 'stem', addend=addend)
    torch.cuda.synchronize()
    assert torch.equal(dg_u, dg) and torch.equal(db_u, db) and (dres is None or torch.equal(dres_u, dres))
    return dict(u=u, x=x, w=w, gamma=gamma, beta=beta, res=res, dy=dy, rec=rec, y=y, c=rec['c'], mean=rec['mean'],
                invstd=rec['invstd'], dc=dc, dres=dres, dg=dg, db=db, addend=addend, dx=dx, dw=dw, rm0=rm0, rv0=rv0,
                mask=(y > 0) if relu else None, mask_beta=mask_beta)


def _nhwc_in(d, kind):
    """the unit's input as an NHWC map (the stem's NCHW image permuted)"""
    return d['x'].permute(0, 2, 3, 1) if kind == 'stem' else d['x']




def _checkabi(spec, d, tag):
    """every kernel of the unit once more through the C ABI into NaN-filled buffers followed by guard words: the Unit's
    bits -> the directly called 3x3 weight gradient (its splits add with atomics: held to its bound by the caller), or None"""
    from hawkeye_b200.ops import conv3x3_pack
    _, kind, H, cin, cout, relu, has_res = spec
    x, w, c, dc, dx, rec = d['x'], d['w'], d['c'], d['dc'], d['dx'], d['rec']
    N, P = x.shape[0], rec['P']
    # forward convolution
    if kind == 'stem':
        (x147,) = abi('hk_stem_im2col', x, Out(rec['xin'].shape), N, H, H)
        (w147,) = abi('hk_pack_stem_weights', w, Out((cout, 160)), cout)
        assert torch.equal(x147, rec['xin']), f'{tag}: im2col differs'
        assert torch.equal(_gemm(x147, w147, 0, P, cout, 160), c.view(P, cout)), f'{tag}: stem GEMM differs'
    elif kind in ('1x1', '1x1s2'):
        if kind == '1x1s2':
            (xs,) = abi('hk_subsample2', x, Out(rec['xin'].shape), N, H, H, cin)
            assert torch.equal(xs, rec['xin']) and torch.equal(xs, x[:, ::2, ::2]), f'{tag}: subsample differs'
        assert torch.equal(_gemm(rec['xin'], w, 0, P, cout, cin), c.view(P, cout)), f'{tag}: GEMM differs'
    else:
        wf, wd = conv3x3_pack(w, True)
        (cd,) = abi('hk_conv3x3_s2_fwd' if kind == '3x3s2' else 'hk_conv3x3_fwd', x, wf, None, Out(c.shape), N, H, H,
                    cin, cout, 0)
        assert torch.equal(cd, c), f'{tag}: conv differs'
    # BatchNorm forward and backward
    bn = d['u'].bn
    ws, nb = workspace('hk_bn_workspace_bytes', P, cout)
    if rec['frozen']:
        (y,) = abi('hk_bn_apply', c, d['mean'], d['invstd'], d['gamma'], d['beta'], d['res'], Out(c.shape), P, cout,
                   int(relu))
    else:
        rm, rv = d['rm0'].clone(), d['rv0'].clone()
        y, mean, invstd = abi('hk_bn_fwd', c, d['gamma'], d['beta'], d['res'], Out(c.shape), Out((cout,)),
                              Out((cout,)), rm, rv, float(bn.momentum), float(bn.eps), P, cout, int(relu), ws, nb)
        assert torch.equal(mean, d['mean']) and torch.equal(invstd, d['invstd']), f'{tag}: BN statistics differ'
        assert torch.equal(rm, bn.running_mean) and torch.equal(rv, bn.running_var), f'{tag}: running statistics differ'
    assert torch.equal(y, d['y']), f'{tag}: BN output differs'
    outs = abi('hk_bn_bwd_frozen' if rec['frozen'] else 'hk_bn_bwd_ex', c, rec['y'], d['dy'], d['gamma'],
               d['mask_beta'], d['mean'], d['invstd'], Out(c.shape), Out(c.shape) if has_res else None, Out((cout,)),
               Out((cout,)), P, cout, int(relu), ws, nb)
    want = [dc] + ([d['dres']] if has_res else []) + [d['dg'], d['db']]
    assert all(torch.equal(a, b) for a, b in zip(outs, want)), f'{tag}: BN backward differs'
    # weight and data gradients
    if kind in ('stem', '1x1', '1x1s2'):
        K = 160 if kind == 'stem' else cin
        ws, nb = workspace('hk_matconv_wgrad_workspace_bytes', P, K, cout)
        (dwm,) = abi('hk_matconv_wgrad', rec['xin'], dc, Out((cout, K)), P, K, cout, ws, nb)
        assert torch.equal(dwm[:, :d['dw'][0].numel()], d['dw'].view(cout, -1)), f'{tag}: matconv wgrad differs'
        if kind == 'stem':
            assert not bool(dwm[:, 147:].any()), f'{tag}: the zero im2col columns have a non-zero weight gradient'
            return None
        if kind == '1x1':
            assert torch.equal(_gemm(dc, w, 1, P, cin, cout, D=d['addend']), dx.view(P, cin)), f'{tag}: dgrad differs'
            return None
        dxs = _gemm(dc, w, 1, P, cin, cout)
        (up,) = abi('hk_upsample2_zero', dxs, Out(dx.shape), N, H, H, cin)
        assert torch.equal(up[:, ::2, ::2], dxs.view(N, (H + 1) // 2, (H + 1) // 2, cin)), f'{tag}: upsample differs'
        assert not bool(up[:, 1::2].any()) and not bool(up[:, :, 1::2].any()), f'{tag}: upsample odd rows not zero'
        assert torch.equal(up + d['addend'], dx), f'{tag}: stride-2 dgrad differs'
        return None
    g = dc
    if kind == '3x3s2':
        (g,) = abi('hk_upsample2_zero', dc, Out((N, H, H, cout)), N, H, H, cout)
        assert torch.equal(g[:, ::2, ::2], dc) and not bool(g[:, 1::2].any()) and not bool(g[:, :, 1::2].any()), \
            f'{tag}: zero insertion of dC differs'
    (dxd,) = abi('hk_conv3x3_dgrad', g, wd, None, Out(dx.shape), N, H, H, cin, cout)
    assert torch.equal(dxd, dx), f'{tag}: dgrad differs'
    ws, nb = workspace('hk_conv3x3_wgrad_workspace_bytes', cin, cout)
    (dwd,) = abi('hk_conv3x3_wgrad_acc', x, g, Out(w.shape), None, N, H, H, cin, cout, ws, nb, 0)
    return dwd


def _check_stats(d, tag):
    """batch mean / invstd against fp64 (the mean's error in units of sigma) and the running statistics after the step"""
    c, bn = d['c'], d['u'].bn
    m, v = bn_stats_ref(c)
    P = c.numel() // c.shape[-1]
    sig, inv = v.sqrt(), (v + bn.eps).rsqrt()
    rm = _chk('C_SUMS', d['mean'], m, sig, C_SUMS, f'{tag} mean', rnd=False, names=('channel',))
    ri = _chk('C_SUMS', d['invstd'], inv, inv, C_SUMS, f'{tag} invstd', rnd=False, names=('channel',))
    print(f'{tag}: mean error up to {rm * C_SUMS:.3g} sigma, invstd relative error up to {ri * C_SUMS:.3g}', flush=True)
    mom = torch.tensor(bn.momentum, dtype=torch.float32).double().item()      # the kernel's fp32 momentum
    unb = v * P / (P - 1)
    rm0, rv0 = d['rm0'].double(), d['rv0'].double()
    # the statistics' own bound, scaled by the momentum, plus the update's three fp32 roundings
    bm = mom * C_SUMS * sig + 2.0 ** -22 * ((1 - mom) * rm0.abs() + mom * m.abs())
    bv = mom * 2 * C_SUMS * unb + 2.0 ** -22 * ((1 - mom) * rv0.abs() + mom * unb)
    check(bn.running_mean, (1 - mom) * rm0 + mom * m, bm, f'{tag} running mean', names=('channel',))
    check(bn.running_var, (1 - mom) * rv0 + mom * unb, bv, f'{tag} running var', names=('channel',))


def _check_maxpool(y, tag, seed):
    """MaxPool2d(3, 2, 1) behind the stem: values and first-maximum positions exact, the gradient's scatter within
    2^-22 of its |terms|"""
    N, H, W, C = y.shape
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    p, am = abi('hk_maxpool3x3s2_fwd', y, Out((N, Ho, Wo, C)), Out((N, Ho, Wo, C), torch.uint8), N, H, W, C)
    dp = torch.randn(p.shape, device='cuda', generator=torch.Generator(device='cuda').manual_seed(seed))
    (dx,) = abi('hk_maxpool3x3s2_bwd', am, dp, Out(y.shape), N, H, W, C)
    ties = 0
    for n0 in range(0, N, CHUNK):
        sl = slice(n0, n0 + CHUNK)
        val, arg = maxpool_ref(y[sl])
        assert torch.equal(p[sl], val), f'{tag} maxpool [{n0}:]: values differ from the window maxima'
        assert torch.equal(am[sl].long(), arg), f'{tag} maxpool [{n0}:]: arg-max bytes differ from the first maximum'
        ties += int((val == 0).sum())
        ref, ax = maxpool_bwd_ref(arg, dp[sl], H, W)
        check(dx[sl], ref, c_bound(ax, 2.0 ** -22), f'{tag} maxpool dx [{n0}:]', n0=n0)
    print(f'{tag} maxpool: {ties / p.numel():.1%} of the windows are all zero (tied)', flush=True)


def _check_unit(sweep, spec, seed):
    size, N, precise, training = SWEEPS[sweep]
    name, kind, H, cin, cout, relu, has_res = spec
    rnd = not precise
    cc, cw = ('C_PRECISE', 'C_PRECISE') if precise else ('C_CONV', 'C_WGRAD')
    crnd = rnd and kind.startswith('3x3')     # the 3x3 convolutions store TF32, the GEMMs fp32
    tag = f'{sweep} {name}'
    d = run_unit(spec, N, seed, precise, training)
    dw3 = _checkabi(spec, d, tag)
    if training:
        _check_stats(d, tag)
    k, stride, pad = GEOM[kind]
    x, w, c, y, dc, dx = _nhwc_in(d, kind), d['w'], d['c'], d['y'], d['dc'], d['dx']
    mean, invstd, gamma, res, addend, P = d['mean'], d['invstd'], d['gamma'], d['res'], d['addend'], d['rec']['P']
    gp = torch.where(d['mask'], d['dy'], torch.zeros((), device='cuda')) if relu else d['dy']
    sums = bn_bwd_sums(c, gp, mean, invstd)
    _chk('C_SUMS', d['db'], sums[0], sums[2], C_SUMS, f'{tag} dbeta', rnd=False, names=('channel',))
    _chk('C_SUMS', d['dg'], sums[1], sums[3], C_SUMS, f'{tag} dgamma', rnd=False, names=('channel',))
    gw = aw = 0
    for n0 in range(0, N, CHUNK):
        sl = slice(n0, n0 + CHUNK)
        xs = x[sl]
        if kind == 'stem':
            cols = F.unfold(d['x'][sl], 7, padding=3, stride=2).transpose(1, 2)
            xin = d['rec']['xin'].view(N, -1, 160)[sl]
            assert torch.equal(xin[..., :147], cols) and not bool(xin[..., 147:].any()), f'{tag}: im2col [{n0}:] differs'
        ref, a = conv_nhwc(xs, w, stride, pad), conv_nhwc(xs.abs(), w.abs(), stride, pad)
        _chk(cc, c[sl], ref, a, C_PRECISE if precise else C_CONV, f'{tag} c [{n0}:]', rnd=crnd, n0=n0)
        del ref, a
        ref, a = bn_fwd_ref(c[sl], mean, invstd, gamma, d['beta'], None if res is None else res[sl], relu)
        _chk('C_BN', y[sl], ref, a, C_BN, f'{tag} y [{n0}:]', rnd=rnd, n0=n0)
        ref, a = bn_bwd_ref(c[sl], gp[sl], gamma, mean, invstd, sums, P, not training)
        _chk('C_BN', dc[sl], ref, a, C_BN, f'{tag} dC [{n0}:]', rnd=rnd, n0=n0)
        del ref, a
        if has_res:
            assert torch.equal(d['dres'][sl], gp[sl]), f'{tag}: dres [{n0}:] differs from the masked dy'
        if kind != 'stem':
            ref, a = conv_nhwc_t(dc[sl], w, stride, pad, H, H), conv_nhwc_t(dc[sl].abs(), w.abs(), stride, pad, H, H)
            if addend is not None:
                ref, a = ref + addend[sl].double(), a + addend[sl].double().abs()
            _chk(cc, dx[sl], ref, a, C_PRECISE if precise else C_CONV, f'{tag} dx [{n0}:]', rnd=crnd, n0=n0)
            del ref, a
            if kind == '1x1s2':
                assert torch.equal(dx[sl, 1::2], addend[sl, 1::2]) and torch.equal(dx[sl, :, 1::2], addend[sl, :, 1::2]), \
                    f'{tag}: dx [{n0}:] off the stride-2 grid is not the addend alone'
        gw = gw + wgrad_nhwc(xs, dc[sl], k, stride, pad)
        aw = aw + wgrad_nhwc(xs.abs(), dc[sl].abs(), k, stride, pad)
    names = ('co', 'ci', 'kh', 'kw')
    cwv = C_PRECISE if precise else C_WGRAD
    _chk(cw, d['dw'], gw, aw, cwv, f'{tag} dW', rnd=False, names=names)
    if dw3 is not None:
        _chk(cw, dw3, gw, aw, cwv, f'{tag} dW (direct call)', rnd=False, names=names)
    if kind == 'stem':
        _check_maxpool(y, tag, seed + 1)


CASES = [(s, u[0]) for s in SWEEPS for u in resnet50_units(448)]


@pytest.mark.gpu
@pytest.mark.parametrize('sweep,unit', CASES, ids=[f'{s}-{u}' for s, u in CASES])
def test_unit(sweep, unit):
    from hawkeye_b200 import _lib
    size, N, precise, _ = SWEEPS[sweep]
    spec = {u[0]: u for u in resnet50_units(size)}[unit]
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    _lib.set_precise(precise)
    try:
        _check_unit(sweep, spec, 5000 + 100 * list(SWEEPS).index(sweep) + list(UNITS).index(unit))
    finally:
        _lib.set_precise(0)
    print(f'{sweep} {unit} ({spec[1]}, N={N}, {spec[2]}x{spec[2]}, {spec[3]}->{spec[4]}): {time.time() - t0:.1f} s, peak '
          f'{torch.cuda.max_memory_allocated() / 2**30:.1f} GiB; worst c-term share so far: ' + WORST.summary(),
          flush=True)


# the dimension-reduction unit in front of the mpn step's covariance head (1x1, 2048 -> 256 at 14x14, BN, ReLU)
DR_UNIT = ('pool.conv_dr_block', '1x1', 14, 2048, 256, True, False)


@pytest.mark.gpu
def test_dr_unit_b32():
    """the dimension-reduction unit of the mpn step at 448x448 batch 32, TF32 train mode"""
    from hawkeye_b200 import _lib
    _lib.set_precise(0)
    _check_unit('tf32-448-b32', DR_UNIT, 6000)


# ------------------------------------------------------------------------------------------------------------------
# 5. the bounds reject real defects of the kernels' own outputs
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_gpu_bounds_reject_conv_defects():
    from hawkeye_b200 import _lib
    _lib.set_precise(0)
    for name in ('layer1.1.conv1', 'layer4.1.conv1'):            # K = 256 and K = 2048
        spec = UNITS[name]
        d = run_unit(spec, 2, 900)
        x, w, c = d['x'], d['w'], d['c']
        ref, a = conv_nhwc(x, w, 1, 0), conv_nhwc(x.abs(), w.abs(), 1, 0)
        check(c, ref, c_bound(a, C_CONV), f'sensitivity {name} unedited')
        rejected(drop_k_slice(c, x, w, 128, spec[3] // 2), ref, a, C_CONV,
                 f'sensitivity {name} K={spec[3]}: one 32-wide K slice of one 128-row tile left out')
    d = run_unit(UNITS['layer2.0.conv2'], 2, 901)                # 112 -> 56, 8 x 8 output tiles
    x, w, c = d['x'], d['w'], d['c']
    ref, a = conv_nhwc(x, w, 2, 1), conv_nhwc(x.abs(), w.abs(), 2, 1)
    check(c, ref, rnd_bound(a, C_CONV), 'sensitivity layer2.0.conv2 unedited')
    rejected(drop_tap(c, x, w, 2, 8, 16, 8, 8, (0, 2), 32), ref, a, C_CONV,
             'sensitivity layer2.0.conv2: tap (0, 2) of channels 32..63 left out over one 8x8 tile', rnd=True)
    rejected(wrong_phase_row(c, x, w, 9), ref, a, C_CONV, 'sensitivity layer2.0.conv2: row 9 at the wrong stride phase',
             rnd=True)
    d = run_unit(UNITS['stem'], 2, 902)
    x, w, c = _nhwc_in(d, 'stem'), d['w'], d['c']
    ref, a = conv_nhwc(x, w, 2, 3), conv_nhwc(x.abs(), w.abs(), 2, 3)
    check(c, ref, c_bound(a, C_CONV), 'sensitivity stem unedited')
    rejected(drop_stem_column(c, d['rec']['xin'], w.reshape(64, 147), 4096, 73), ref, a, C_CONV,
             'sensitivity stem: im2col column 73 left out over 128 pixels')


@pytest.mark.gpu
def test_gpu_bounds_reject_bn_defects():
    """layer4.0.conv3 at 448x448 batch 32: P = 6,272 rows of 2,048 channels in 25 partial blocks"""
    from hawkeye_b200 import _lib
    _lib.set_precise(0)
    spec = UNITS['layer4.0.conv3']
    d = run_unit(spec, 32, 903)
    c, mean, invstd, cout, P = d['c'], d['mean'], d['invstd'], spec[4], d['rec']['P']
    m, v = bn_stats_ref(c)
    sig, inv = v.sqrt(), (v + BN_EPS).rsqrt()
    ch, nm = 7, ('channel',)
    check(mean, m, c_bound(sig, C_SUMS), 'sensitivity BN mean unedited', names=nm)
    bad = mean.clone()
    bad[ch] += float(1e-4 * sig[ch])
    rejected(bad, m, sig, C_SUMS, 'sensitivity BN: one mean moved by 1e-4 sigma', names=nm)
    bad = invstd.clone()
    bad[ch] *= 1 + 1e-4
    rejected(bad, inv, inv, C_SUMS, 'sensitivity BN: one invstd x (1 + 1e-4)', names=nm)
    gp = torch.where(d['mask'], d['dy'], torch.zeros((), device='cuda'))
    db, dg, ab, ag = bn_bwd_sums(c, gp, mean, invstd)
    _, nb = workspace('hk_bn_workspace_bytes', P, cout)
    nblk = nb // (2 * cout * 4)
    assert P == 6272 and nblk == 25
    xh = (c.double() - mean.double()) * invstd.double()
    bdb, bdg = drop_bn_block(d['db'], d['dg'], gp, xh, ch, nblk, 12)
    rejected(bdb, db, ab, C_SUMS, 'sensitivity BN: one of 25 partial blocks left out of dbeta', names=nm)
    rejected(bdg, dg, ag, C_SUMS, 'sensitivity BN: one of 25 partial blocks left out of dgamma', names=nm)


def _wgrad_refs(x, dc, k, stride, pad):
    gw = aw = 0
    for n0 in range(0, x.shape[0], CHUNK):
        xs, ds = x[n0:n0 + CHUNK], dc[n0:n0 + CHUNK]
        gw = gw + wgrad_nhwc(xs, ds, k, stride, pad)
        aw = aw + wgrad_nhwc(xs.abs(), ds.abs(), k, stride, pad)
    return gw, aw


@pytest.mark.gpu
def test_gpu_bounds_reject_wgrad_defects():
    from hawkeye_b200 import _lib
    _lib.set_precise(0)
    names = ('co', 'ci', 'kh', 'kw')
    # the stem at 448x448 batch 32: hk_matconv_wgrad over P = 1,605,632 pixels in S splits
    d = run_unit(UNITS['stem'], 32, 904)
    P, dc = d['rec']['P'], d['dc']
    _, nb = workspace('hk_matconv_wgrad_workspace_bytes', P, 160, 64)
    S = nb // (64 * 160 * 4)
    assert S == 256, S
    gw, aw = _wgrad_refs(_nhwc_in(d, 'stem'), dc, 7, 2, 3)
    dw = d['dw'].view(64, 147)
    gw, aw = gw.view(64, 147), aw.view(64, 147)
    check(dw, gw, c_bound(aw, C_WGRAD), 'sensitivity stem dW unedited', names=('co', 'k'))
    rejected(drop_split(dw, d['rec']['xin'][:, :147], dc, S, 100), gw, aw, C_WGRAD,
             f'sensitivity stem dW: one split of {S} left out', names=('co', 'k'))
    # layer4's 3x3 at 14x14, batch 32: the last, partial tile row (rows 12-13) of one image
    d = run_unit(UNITS['layer4.1.conv2'], 32, 905)
    gw, aw = _wgrad_refs(d['x'], d['dc'], 3, 1, 1)
    check(d['dw'], gw, c_bound(aw, C_WGRAD), 'sensitivity layer4.1.conv2 dW unedited', names=names)
    rejected(drop_rows(d['dw'], d['x'], d['dc'], 3, 12, 14), gw, aw, C_WGRAD,
             'sensitivity layer4.1.conv2 dW: rows 12-13 of image 3 left out', names=names)
