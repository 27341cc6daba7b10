"""The OSMENet head of the osmenet train step, element by element against fp64: the OSME excitation (hk_row_mean_*,
hk_linear_* 2048 -> 128 -> 2048, hk_act_*, hk_se_gate_*), the two attention FCs over the 401408-wide gated map, the
1024 -> 200 classifier, the N-pairs term of MAMCLoss (hk_l2norm_rows_*, the 3xTF32 anchor products, hk_npair_loss), the
composed head through autograd, and the SGD step over the head's 823 M-float parameter slice.

Cases: b32_14x14 is the workload (448x448, batch 32: fc_in = 2048 x 14 x 14 = 401408, 392 K slices of 1024, n = 64
anchors); b10_7x7 is the reference config (224x224, 5 classes x 2 samples: fc_in 100352, 98 slices, n = 20);
precise_b4_14x14 runs 3xTF32 on inputs that are not tf32-representable, so the (hi, lo) split is exercised.

Every kernel is called through the C ABI into NaN-filled outputs followed by guard words, with NaN-filled workspaces of
exactly the queried size; inputs are followed by NaN.  Each stage gets its own inputs and is compared with fp64 applied
to the fp32 values it was given, on the GPU, ROWS output features at a time for the attention FCs (their 1.64 GB weight
is never copied to fp64), so that the file's peak device memory stays under 16 GiB.

Error model (u = 2^-24; PAIR = 2^-22, what a (hi, lo) tf32 pair loses; EPI = 4u, the GEMM epilogue's roundings).  A
bound is `fixed + c * scale`, fixed the analysed roundings and c a measured constant:

  row mean        (ceil(cols / 32) + 5) u sum|x| / cols + u |y| (32 lanes, a 5-level warp tree, the division)
  row mean bwd    bit-identical to the fp32 quotient dy / cols
  SE gate s, dx   8u |ref|: expf (2 ulp), 1 + e, the reciprocal and the product; g stays above 2^-126 for |m| <= 60
  SE gate dm      g(1 - g) (ceil(hw / 32) + 5) u sum|ds x| + 7u g |sum ds x| + 3u |dm|: the warp sum, g's error through
                  g(1 - g) (which is all that is left where g rounds to 1), and the two products
  ReLU            bit-exact, +0.0 where x <= 0
  linear          test_gpu_mpncov_head.linear_refs: y (S + 1) u (|x||w|^T + |b|) for the split sum, then c |x||w|^T; dx
                  c |dy||w|; dw c |dy|^T|x|; db 2^-19 sum|dy|.  In 3xTF32 mode each product adds 3 PAIR of its scale
  l2norm fwd      e_s = (ceil(D / 256) + 13) u: the squared norm (per-thread fmaf chains, warp trees, 8 warp partials);
                  inv within (e_s / 2 + 2u) |inv|, y within (e_s / 2 + 3u) |y|
  anchor GEMMs    3xTF32: fixed (3 PAIR + EPI) of the |A||B| scale (plus |t| for the addend of the second backward
                  product), then c |A||B|
  npair loss      c times the sensitivity scale: per positive pair log1p(z) + z / (1 + z) (z = E e^-p), over n; dprod:
                  the sum of the magnitudes of its positive-side and negative-side addends, over n
  l2norm bwd      inv (|y| e_s sum|y dy| + 2u (|dy| + |y s|)) + u |dx|
  SGD             buf 3u (|g| + wd |p| + m |buf_old|); p 2u |p_new| + lr (that + 2u |buf|), with the fp32 values of lr, wd
                  and momentum the kernel is given

The worst (|err| - fixed) / (c * scale) measured over every check of this file on an H100 80GB HBM3 (700 W), and the
margin of each c over it:

  C_LIN    2^-19   0.199 (b32_14x14 fcs[0] dw)   5.0x   linear products of K <= 256: every wgrad (K = B), the
                                                        expand's forward (K = 128), the squeeze's and the classifier's
                                                        dgrad (K = 128, 200), the anchor backward products (K = n)
  C_LONGK  2^-18   0.219 (b32_14x14 fcs[1] dx)   4.6x   linear products that accumulate K >= 1024 terms in one pass: the
                                                        K slices of the attention FCs and of the squeeze, the
                                                        classifier's forward, the attention FCs' dgrad (K = 1024) and
                                                        the expand's (K = 2048)
  C_GRAM   2^-15   0.159 (b32_14x14 prod)        6.3x   the anchor product F F^T (3xTF32, K = 1024)
  C_NP     2^-19   0.168 (b32_14x14 shuffled dprod) 6.0x hk_npair_loss, loss and dprod

C_LIN is test_gpu_mpncov_head's constant, measured there at K = 200.  At K = 1024 in one pass the classifier's forward
took 0.30 of it and the attention FCs' dgrad 0.44, under the 4x margin, hence C_LONGK.  F F^T has its own constant
because its diagonal is a coherent sum of 1024 positive squares: the kernel returns 0.999994 where fp64 gives 1.0 (98u
low on every anchor), the accumulated truncation of the tensor cores' fp32 accumulation: a bias, not a local defect.

The composed head (section 2) is OSME(2048, 1024, 14, 2) and nn.Linear(1024, 200) through autograd on a post-ReLU map at
batch 32, then MAMCLoss(lambda_a = 0.5): every stage bit-identical to its direct C-ABI call, x.grad within three fp32 adds
of the fp64 sum of its four contributions, and loss, logits, x_part and the 14 parameter gradients within a loose rel-L2
of an fp64 composition, printed.

The self-tests (no GPU) check that the fp64 N-pairs restatement is the oracle's, that the fp64 OSME restatement is the
reference's formula, and that the loosest bounds (TF32 mode) reject planted defects computed in fp64 and rounded to fp32:
a dropped K slice, the last slice read at its neighbour's offset, the bias added once per slice, one image missing from
db; the row mean divided by the padded width; sigmoid(-m) in the gate, dm without g(1 - g), the neighbouring row's gate;
class labels laid out with repeat instead of repeat_interleave, the anchor left out of its own positive set, EA for term
B, dF = 2 dprod F, the missing 1 / n; the l2norm backward without its projection term.
"""
import math
import os
import time

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import detgen
from conftest import rel_l2
from fp64_refs import C_LIN, classifier_inputs, linear_refs, linear_splits
from kernel_check import PAIR, U, Worst, abi, check, guarded, poisoned, workspace

EPI = 4 * U
C_LONGK = 2.0 ** -18
C_GRAM = 2.0 ** -15
C_NP = 2.0 ** -19
WORST = Worst(C_LIN=C_LIN, C_LONGK=C_LONGK, C_GRAM=C_GRAM, C_NP=C_NP)
check_c = WORST.check_c
F64 = torch.float64
ROWS = 128            # output features per fp64 reference chunk of the attention FCs
SGD_CHUNK = 1 << 25   # parameters per fp64 reference chunk of the optimizer step
RATIO = 16            # OSME_block's reduce ratio
LAMBDA_A = 0.5
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# case -> (B, C, H, P, D, classes, precise)
CASES = {
    'b32_14x14': (32, 2048, 14, 2, 1024, 200, 0),
    'b10_7x7': (10, 2048, 7, 2, 1024, 200, 0),
    'precise_b4_14x14': (4, 2048, 14, 2, 1024, 200, 1),
}
SAMPLES = {32: 4, 10: 2, 4: 2}     # BalancedBatchSampler's n_samples per class of each batch
LAYOUTS = ('class_major', 'shuffled', 'uniform200', 'one_class')


# ------------------------------------------------------------------------------------------------------------------
# 1. fp64 restatements (device-agnostic)
# ------------------------------------------------------------------------------------------------------------------
def layout_labels(B, layout, seed=0):
    """class labels of a batch: the balanced sampler's class-major n_classes x n_samples, the same shuffled, uniform draws
    over 200 classes as bench.py makes them, or one class for all"""
    if layout == 'uniform200':
        return detgen.det_labels(B, 200, seed)
    if layout == 'one_class':
        return torch.zeros(B, dtype=torch.int64)
    lab = torch.arange(B // SAMPLES[B]).repeat_interleave(SAMPLES[B])
    if layout == 'shuffled':
        lab = lab[torch.from_numpy(np.random.RandomState(seed).permutation(B))]
    return lab


def npair_sets(labels, P, repeat=False):
    """the four kinds of anchor j relative to anchor i (MAMC_loss.py:44-56), n = B P anchors of row b P + p: same attention
    and class (j = i included), same attention only, same class only, neither.  repeat: the labels laid out with repeat
    instead of repeat_interleave (a defect)"""
    cls = labels.repeat(P) if repeat else labels.repeat_interleave(P)
    part = torch.arange(P, device=labels.device).repeat(labels.numel())
    sc = cls[:, None] == cls[None, :]
    sa = part[:, None] == part[None, :]
    return sc & sa, ~sc & sa, sc & ~sa, ~sc & ~sa


def npair_from_prod(prod, labels, P, **defect):
    """the N-pairs loss of the anchor products prod [n, n]: for every anchor the three terms sum_{j in POS} log(1 +
    sum_{k in NEG} exp(prod_ik - prod_ij)), written as log1p(E_i exp(-prod_ij)) with E_i = sum_{k in NEG} exp(prod_ik),
    over n.  Defects: repeat, no_self (the anchor out of its own positive set), ea_for_b, no_inv_n."""
    n = prod.shape[0]
    s0, s1, s2, s3 = npair_sets(labels, P, defect.get('repeat', False))
    if defect.get('no_self'):
        s0 = s0 & ~torch.eye(n, dtype=torch.bool, device=prod.device)
    e, em = prod.exp(), (-prod).exp()
    EA = (e * (s1 | s2 | s3)).sum(1, keepdim=True)
    EB = (e * s3).sum(1, keepdim=True)
    total = 0.0
    for pos, E in ((s0, EA), (s1, EA if defect.get('ea_for_b') else EB), (s2, EB)):
        total = total + (torch.log1p(E * em) * pos).sum()
    return total if defect.get('no_inv_n') else total / n


def npair_scales(prod, labels, P):
    """-> (loss scale, dprod scale, dprod in closed form): the sensitivity of the loss to a relative error of each z, and
    the magnitudes of the positive-side and negative-side addends of every dprod element"""
    n = prod.shape[0]
    s0, s1, s2, s3 = npair_sets(labels, P)
    e, em = prod.exp(), (-prod).exp()
    EA = (e * (s1 | s2 | s3)).sum(1, keepdim=True)
    EB = (e * s3).sum(1, keepdim=True)
    zA, zB = EA * em, EB * em
    sl = ((torch.log1p(zA) + zA / (1 + zA)) * s0).sum() + ((torch.log1p(zB) + zB / (1 + zB)) * (s1 | s2)).sum()
    WA = (s0 * em / (1 + zA)).sum(1, keepdim=True)
    WBC = ((s1 | s2) * em / (1 + zB)).sum(1, keepdim=True)
    pos = s0 * zA / (1 + zA) + (s1 | s2) * zB / (1 + zB)
    neg = (s1 | s2 | s3) * e * WA + s3 * e * WBC
    return sl / n, (pos + neg) / n, (neg - pos) / n


def npairs64(feats, labels):
    """NPairsLoss in fp64: F.normalize of the b p rows, prod = F F^T, npair_from_prod"""
    b, p, D = feats.shape
    x = F.normalize(feats.reshape(b * p, D), p=2, dim=1)
    return npair_from_prod(x @ x.T, labels, p)


def mamc64(pred, x_part, labels, lambda_a=LAMBDA_A):
    return F.cross_entropy(pred, labels, label_smoothing=0.1) + lambda_a * npairs64(x_part, labels)


def osme_block64(x, w0, b0, w2, b2):
    """OSME_block on x [N, C, HW]: sigmoid(Linear(ReLU(Linear(mean x)))) * x, the pre-sigmoid m kept"""
    z = x.mean(-1)
    m = torch.relu(z @ w0.T + b0) @ w2.T + b2
    return torch.sigmoid(m)[:, :, None] * x, m


def l2norm_bounds(x):
    """fp64 y, inv of the fp32 rows x and their bounds"""
    xd = x.to(F64)
    nrm = xd.norm(dim=1, keepdim=True)
    e_s = (math.ceil(x.shape[1] / 256) + 13) * U
    inv = 1 / nrm.clamp_min(1e-12)
    return xd * inv, inv.squeeze(1), (e_s / 2 + 3 * U) * (xd * inv).abs(), (e_s / 2 + 2 * U) * inv.squeeze(1)


def l2norm_bwd64(y, inv, dy, projection=True):
    """dx = inv (dy - y <y, dy>) of the fp32 y, inv, dy, and its bound; without the projection term when projection is
    False (a defect)"""
    yd, dd, iv = y.to(F64), dy.to(F64), inv.to(F64)[:, None]
    s = (yd * dd).sum(1, keepdim=True)
    dx = iv * (dd - yd * s) if projection else iv * dd
    e_s = (math.ceil(y.shape[1] / 256) + 13) * U
    return dx, iv * (yd.abs() * e_s * (yd * dd).abs().sum(1, keepdim=True) + 2 * U * (dd.abs() + (yd * s).abs())) + \
        U * dx.abs()


def anchor_bwd64(dprod, xn, t=None, symmetric=True):
    """t = dprod F and dF = dprod^T F + t (the two backward products of NPairsLossFn) with their fixed bounds and
    c-scales; dF = 2 dprod F when symmetric is False (a defect)"""
    dp, xd = dprod.to(F64), xn.to(F64)
    sc = dp.abs() @ xd.abs()
    t_ref = dp @ xd
    tt = t_ref if t is None else t.to(F64)
    df = (dp.T @ xd + tt) if symmetric else 2 * t_ref
    sd = dp.abs().T @ xd.abs()
    return (t_ref, (3 * PAIR + EPI) * sc, sc), (df, (3 * PAIR + EPI) * (sd + tt.abs()), sd)


def row_mean_bound(x, cols):
    """fp64 row mean of the fp32 rows x [R, cols] and its bound"""
    xd = x.to(F64)
    ref = xd.sum(1) / cols
    return ref, (math.ceil(cols / 32) + 5) * U * xd.abs().sum(1) / cols + U * ref.abs()


def se_gate_bounds(x, m, ds, hw):
    """fp64 s, dx, dm of the fp32 x [R, hw], m [R], ds [R, hw] and their bounds"""
    xd, dd = x.to(F64), ds.to(F64)
    g = torch.sigmoid(m.to(F64))
    s, dx = g[:, None] * xd, g[:, None] * dd
    acc = (dd * xd).sum(1)
    gg = g * (1 - g)
    dm = acc * gg
    bdm = gg * (math.ceil(hw / 32) + 5) * U * (dd * xd).abs().sum(1) + 7 * U * g * acc.abs() + 3 * U * dm.abs()
    return (s, 8 * U * s.abs()), (dx, 8 * U * dx.abs()), (dm, bdm)


def sgd_bounds(p, g, buf, lr, m, wd, first):
    """oracle.hop_oracle.sgd_momentum_step in fp64 -> (p, buf) and their bounds"""
    from oracle.hop_oracle import sgd_momentum_step
    p_ref, b_ref = sgd_momentum_step(p, g, buf, lr, m, wd, first)
    eb = 3 * U * (g.abs() + wd * p.abs() + (0 if first else m * buf.abs()))
    return p_ref, b_ref, 2 * U * p_ref.abs() + lr * (eb + 2 * U * b_ref.abs()), eb


def f32(v):
    """the fp32 value of a Python float, as the C ABI hands it to a kernel"""
    return float(torch.tensor(v, dtype=torch.float32))


# ------------------------------------------------------------------------------------------------------------------
# 2. inputs and launches
# ------------------------------------------------------------------------------------------------------------------
def trunk_map(B, C, HW, seed, device='cuda'):
    """a post-ReLU map [B, C, HW] with about 60 % zeros, as ResNet's layer4 emits"""
    g = torch.Generator(device=device).manual_seed(seed)
    return torch.relu(torch.randn(B, C, HW, generator=g, device=device) - 0.25)


def operands(t, precise, seed):
    """tf32 values in TF32 mode, so that only accumulation is left; in 3xTF32 mode values with bits below tf32's set"""
    t = detgen.tf32_rna(t)
    if not precise:
        return t
    g = torch.Generator(device=t.device).manual_seed(seed)
    return t * (1 + 2.0 ** -14 * (0.25 + torch.rand(t.shape, generator=g, device=t.device)))


def fc_tiles(B, N, S, precise):
    """launch_gemm (gemm.cu) for hk_linear_fwd's split-K product: a batch of S K slices of 128 x BN tiles (BN = 128 when
    N > 64 in TF32 mode, 64 for the 3xTF32 pair kernel), n-tile fastest, then m-tile, then the slice -> tiles per slice"""
    return -(-B // 128) * -(-N // (64 if precise or N <= 64 else 128))


def run_linear(x, w, b, dy, precise):
    """hk_linear_fwd / _dgrad / _wgrad through the C ABI into poisoned buffers -> y, dx, dw, db"""
    from hawkeye_b200 import _lib
    B, Fi = x.shape
    N = w.shape[0]
    _lib.set_precise(precise)
    try:
        ws, nb = workspace('hk_linear_fwd_workspace_bytes', B, Fi, N)
        assert nb == linear_splits(Fi) * B * N * 4
        y = guarded((B, N))
        abi('hk_linear_fwd', x, w, b, y, B, Fi, N, ws, nb)
        dx = guarded((B, Fi))
        abi('hk_linear_dgrad', dy, w, dx, B, Fi, N)
        dw = guarded((N, Fi))
        db = guarded((N,))
        abi('hk_linear_wgrad', dy, x, dw, db, B, Fi, N)
    finally:
        _lib.set_precise(0)
    return y, dx, dw, db


def check_linear(tag, x, w, b, dy, out, precise):
    """every element of y, dx, dw and db against linear_refs, ROWS output features at a time (dx summed over the
    chunks); a product that accumulates 1024 or more terms in one pass (y: one K slice, dx: K = N) takes C_LONGK"""
    y, dx, dw, db = out
    S = linear_splits(x.shape[1])
    N = w.shape[0]
    ky = 'C_LONGK' if x.shape[1] // S >= 1024 else 'C_LIN'
    extra = 3 * PAIR if precise else 0.0
    dx_ref = dx_scale = None
    for r0 in range(0, N, ROWS):
        rs = slice(r0, min(r0 + ROWS, N))
        refs = linear_refs(x, w[rs], b[rs], dy[:, rs], S)
        for key, c, o, names in (('y', ky, y[:, rs], ('image', 'feature')), ('dw', 'C_LIN', dw[rs], ('feature', 'input'))):
            ref, fixed, scale = refs[key]
            check_c(c, f'{tag} {key} [features {r0}:{rs.stop}]', o, ref, fixed + extra * scale, scale, names)
        ref, fixed, _ = refs['db']
        check(db[rs], ref, fixed, f'{tag} db [{r0}:{rs.stop}]', names=('feature',))
        ref, _, scale = refs['dx']
        dx_ref = ref if dx_ref is None else dx_ref + ref
        dx_scale = scale if dx_scale is None else dx_scale + scale
        del refs, ref, scale
    check_c('C_LONGK' if N >= 1024 else 'C_LIN', f'{tag} dx (K = {N})', dx, dx_ref, extra * dx_scale, dx_scale,
            ('image', 'input'))


def _report(tag, t0):
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    print(f'{tag}: {time.time() - t0:.1f} s, peak device memory {peak:.2f} GiB; worst shares so far: ' +
          WORST.summary(), flush=True)


# ------------------------------------------------------------------------------------------------------------------
# 3. stage by stage through the C ABI
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('case', list(CASES))
def test_row_mean_and_gate(case):
    """hk_row_mean_fwd / _bwd, hk_se_gate_fwd / _bwd and hk_act_fwd / _bwd (ReLU) over the B x 2048 rows of the map"""
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    B, C, H = CASES[case][:3]
    HW, R = H * H, B * C
    x = poisoned(trunk_map(B, C, HW, 800).reshape(R, HW))
    y = guarded((R,))
    abi('hk_row_mean_fwd', x, y, R, HW, HW)
    ref, bound = row_mean_bound(x, HW)
    check(y, ref, bound, f'{case} row mean (cols {HW})', names=('row',))
    dy = poisoned(detgen.det((R,), 801).cuda())
    dx = guarded((R, HW))
    abi('hk_row_mean_bwd', dy, dx, R, HW, HW)
    assert torch.equal(dx, (dy.to(F64) / HW).float()[:, None].expand(R, HW)), 'row mean dx is not the fp32 dy / cols'
    # the gate: typical m, then channels where g saturates at both ends, and rows whose ds is zero
    m = detgen.det((R,), 802, 2.0)
    for k, v in enumerate((60.0, -60.0, 30.0, -30.0, 15.0, -15.0)):
        m[k::97] = v
    m = poisoned(m.cuda())
    ds = detgen.det((R, HW), 803, 1e-3)
    ds[7::61] = 0
    ds = poisoned(ds.cuda())
    s = guarded((R, HW))
    abi('hk_se_gate_fwd', x, m, s, R, HW)
    dxg = guarded((R, HW))
    dm = guarded((R,))
    abi('hk_se_gate_bwd', x, m, ds, dxg, dm, R, HW)
    (sr, sb), (dxr, dxb), (dmr, dmb) = se_gate_bounds(x, m, ds, HW)
    check(s, sr, sb, f'{case} gate s', names=('row', 'pos'))
    check(dxg, dxr, dxb, f'{case} gate dx', names=('row', 'pos'))
    check(dm, dmr, dmb, f'{case} gate dm', names=('row',))
    assert not bool(dm[7::61].view(torch.int32).any()) and not bool(dxg[7::61].view(torch.int32).any()), \
        'rows with ds = 0 did not get +0.0'
    # the bottleneck ReLU on [B, 128], with zeros, -0.0 and negatives
    a = detgen.det((B, C // RATIO), 804)
    a[:, ::5] = 0.0
    a[:, 1::7] = -0.0
    a = poisoned(a.cuda())
    h = guarded(a.shape)
    abi('hk_act_fwd', a, h, a.numel(), 0)
    torch.cuda.synchronize()
    da = poisoned(detgen.det(a.shape, 805).cuda())
    dh = guarded(a.shape)
    abi('hk_act_bwd', h, da, dh, a.numel(), 0)
    zero = torch.zeros((), device='cuda')
    assert torch.equal(h.view(torch.int32), torch.where(a > 0, a, zero).view(torch.int32)), 'ReLU forward'
    assert torch.equal(dh.view(torch.int32), torch.where(h > 0, da, zero).view(torch.int32)), 'ReLU backward'
    _report(case, t0)


@pytest.mark.gpu
@pytest.mark.parametrize('case', list(CASES))
def test_excitation_linears(case):
    """OSME_block's 2048 -> 128 (2 K slices) and 128 -> 2048 (one slice, bias through sum_splits) at batch B"""
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    B, C, precise = CASES[case][0], CASES[case][1], CASES[case][6]
    for name, Fi, N, seed in (('squeeze 2048->128', C, C // RATIO, 900), ('expand 128->2048', C // RATIO, C, 910)):
        g = torch.Generator(device='cuda').manual_seed(seed)
        x = torch.relu(torch.randn(B, Fi, generator=g, device='cuda'))
        w = torch.randn(N, Fi, generator=g, device='cuda') * Fi ** -0.5
        b = torch.randn(N, generator=g, device='cuda') * 0.1
        dy = torch.randn(B, N, generator=g, device='cuda') * 0.01
        assert linear_splits(Fi) == (2 if Fi == C else 1)
        x, w, dy = (operands(t, precise, seed + k) for k, t in enumerate((x, w, dy)))
        x, w, b, dy = (poisoned(t) for t in (x, w, b, dy))
        check_linear(f'{case} {name}', x, w, b, dy, run_linear(x, w, b, dy, precise), precise)
    _report(case, t0)


@pytest.mark.gpu
@pytest.mark.parametrize('case', list(CASES))
def test_attention_fc_ctas_cross_slices(case):
    """hk_linear_fwd of an attention FC: 1024-column K slices, and persistent CTAs that take tiles of several slices"""
    B, C, H, P, D, K, precise = CASES[case]
    Fi = C * H * H
    S = linear_splits(Fi)
    assert (S, Fi // S) == ({14: 392, 7: 98}[H], 1024)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    per = fc_tiles(B, D, S, precise)
    total = per * S
    grid = min(total, sms)
    ctas = [{t // per for t in range(i, total, grid)} for i in range(grid)]
    crossing = sum(len(c) > 1 for c in ctas)
    print(f'{case}: fc_in {Fi} = {S} K slices of {Fi // S}; {total} tiles ({per} per slice) on {grid} CTAs ({sms} SMs); '
          f'{crossing} CTAs take tiles of more than one slice, up to {max(map(len, ctas))} slices', flush=True)
    assert total > sms and crossing == grid


@pytest.mark.gpu
@pytest.mark.parametrize('case', list(CASES))
def test_attention_fcs(case):
    """both attention FCs at fc_in = 2048 H W: y, dx, dw (1024 x fc_in, in row blocks) and db; the last 4 columns of every
    K slice are 16x larger (classifier_inputs), so a dropped or shifted slice cannot hide"""
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    B, C, H, P, D, K, precise = CASES[case]
    Fi = C * H * H
    for i in range(P):
        x, w, b, dy, S = classifier_inputs(B, Fi, D, 700 + 10 * i, 'cuda')
        x, w, dy = (operands(t, precise, 710 + 10 * i + k) for k, t in enumerate((x, w, dy)))
        x, w, b, dy = (poisoned(t) for t in (x, w, b, dy))
        check_linear(f'{case} fcs[{i}]', x, w, b, dy, run_linear(x, w, b, dy, precise), precise)
        del x, w, b, dy
    _report(case, t0)


@pytest.mark.gpu
@pytest.mark.parametrize('case', list(CASES))
def test_classifier(case):
    """nn.Linear(1024, 200): one K slice with the bias through sum_splits; 200 is a partial n-tile of the forward, a
    partial k-block of dgrad and a partial m-tile of wgrad"""
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    B, D, K, precise = CASES[case][0], CASES[case][4], CASES[case][5], CASES[case][6]
    x, w, b, dy, S = classifier_inputs(B, D, K, 720, 'cuda')
    assert S == 1
    x, w, dy = (operands(t, precise, 721 + k) for k, t in enumerate((x, w, dy)))
    x, w, b, dy = (poisoned(t) for t in (x, w, b, dy))
    check_linear(f'{case} classifier', x, w, b, dy, run_linear(x, w, b, dy, precise), precise)
    _report(case, t0)


def run_npairs(feats, labels):
    """NPairsLossFn's launches through the C ABI: l2norm, prod = F F^T (3xTF32), hk_npair_loss, t = dprod F, dF = dprod^T
    F + t, l2norm backward -> dict of every output"""
    b, p, D = feats.shape
    n = b * p
    x = poisoned(feats.reshape(n, D))
    cls = poisoned(labels.to(torch.int32).repeat_interleave(p))
    part = poisoned(torch.arange(p, device='cuda', dtype=torch.int32).repeat(b))
    xn = guarded((n, D))
    inv = guarded((n,))
    abi('hk_l2norm_rows_fwd', x, xn, inv, n, D)
    prod = guarded((n, n))
    abi('hk_gemm_3xtf32', xn, 0, D, 0, xn, 0, D, 0, prod, n, 0, 0, n, n, D, 1, 1.0, None, 0.0, None, 0, 0, 0.0, None,
        0)
    acc = guarded((1,), dtype=F64, fill=0.0)
    dprod = guarded((n, n))
    abi('hk_npair_loss', prod, cls, part, acc, dprod, n)
    t = guarded((n, D))
    abi('hk_gemm_3xtf32', dprod, 0, n, 0, xn, 1, D, 0, t, D, 0, 0, n, D, n, 1, 1.0, None, 0.0, None, 0, 0, 0.0, None, 0)
    dxn = guarded((n, D))
    abi('hk_gemm_3xtf32', dprod, 1, n, 0, xn, 1, D, 0, dxn, D, 0, 0, n, D, n, 1, 1.0, None, 0.0, t, D, 0, 1.0, None, 0)
    dx = guarded((n, D))
    abi('hk_l2norm_rows_bwd', xn, inv, dxn, dx, n, D)
    return dict(x=x, xn=xn, inv=inv, prod=prod, loss=acc, dprod=dprod, t=t, dxn=dxn, dx=dx)


def npair_features(B, P, D, labels, seed, device='cuda'):
    """attention features with a class component, an attention component and noise, so that the anchor products spread
    over [-1, 1] as a trained head's do"""
    g = torch.Generator(device=device).manual_seed(seed)
    centre = torch.randn(int(labels.max()) + 1, D, generator=g, device=device)
    att = torch.randn(P, D, generator=g, device=device)
    noise = torch.randn(B, P, D, generator=g, device=device)
    return 0.8 * centre[labels.to(device)][:, None] + 0.5 * att[None] + 0.6 * noise


@pytest.mark.gpu
@pytest.mark.parametrize('case, layout', [('b32_14x14', lay) for lay in LAYOUTS] +
                         [('b10_7x7', 'class_major'), ('precise_b4_14x14', 'class_major')])
def test_npairs(case, layout):
    """the N-pairs term at n = B P anchors, D = 1024, stage by stage"""
    from hawkeye_b200 import _lib
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    B, C, H, P, D, K, precise = CASES[case]
    labels = layout_labels(B, layout, 930).cuda()
    tag = f'{case} {layout}'
    _lib.set_precise(precise)
    try:
        r = run_npairs(npair_features(B, P, D, labels, 931), labels)
    finally:
        _lib.set_precise(0)
    n = B * P
    y, inv, yb, ib = l2norm_bounds(r['x'])
    check(r['xn'], y, yb, f'{tag} l2norm y', names=('anchor', 'feature'))
    check(r['inv'], inv, ib, f'{tag} l2norm inv', names=('anchor',))
    xd = r['xn'].to(F64)
    sc = xd.abs() @ xd.abs().T
    check_c('C_GRAM', f'{tag} prod (K = {D})', r['prod'], xd @ xd.T, (3 * PAIR + EPI) * sc, sc, ('anchor', 'anchor'))
    prod = r['prod'].to(F64).requires_grad_(True)
    loss = npair_from_prod(prod, labels, P)
    (dprod,) = torch.autograd.grad(loss, prod)
    sl, sd, _ = npair_scales(prod.detach(), labels, P)
    check_c('C_NP', f'{tag} npair loss', r['loss'], loss.detach().reshape(1), 0 * sd[0, :1], sl.reshape(1), ('',))
    check_c('C_NP', f'{tag} npair dprod', r['dprod'], dprod, 0 * sd, sd, ('anchor', 'anchor'))
    (tr, tf, ts), (dr, df, ds) = anchor_bwd64(r['dprod'], r['xn'], r['t'])
    check_c('C_LIN', f'{tag} t = dprod F (K = {n})', r['t'], tr, tf, ts, ('anchor', 'feature'))
    check_c('C_LIN', f'{tag} dF = dprod^T F + t', r['dxn'], dr, df, ds, ('anchor', 'feature'))
    dx, bound = l2norm_bwd64(r['xn'], r['inv'], r['dxn'])
    check(r['dx'], dx, bound, f'{tag} l2norm dx', names=('anchor', 'feature'))
    _report(tag, t0)


# ------------------------------------------------------------------------------------------------------------------
# 4. the composed head through autograd
# ------------------------------------------------------------------------------------------------------------------
class _Cfg(dict):
    __getattr__ = dict.__getitem__


class _FC64(torch.autograd.Function):
    """y = s w^T + b in fp64 with the fp32 weight cast ROWS rows at a time (no fp64 copy of 1.64 GB); backward returns ds
    and keeps dy and s, from which the weight gradient is compared row block by row block"""

    @staticmethod
    def forward(ctx, s, w, b, keep):
        y = torch.cat([s @ w[r:r + ROWS].to(F64).T for r in range(0, w.shape[0], ROWS)], 1) + b.to(F64)
        ctx.save_for_backward(s)
        ctx.w, ctx.keep = w, keep
        return y

    @staticmethod
    def backward(ctx, dy):
        (s,) = ctx.saved_tensors
        ctx.keep.update(dy=dy, s=s)
        ds = sum(dy[:, r:r + ROWS] @ ctx.w[r:r + ROWS].to(F64) for r in range(0, ctx.w.shape[0], ROWS))
        return ds, None, None, None


def _gpu_osmeabi(x, blk, fc, up):
    """one attention of OSME forward and backward through direct C-ABI calls; up = the upstream gradients the autograd
    run gave (f, s, m, h, a, z) -> every forward output, input gradient and parameter gradient"""
    from hawkeye_b200 import _lib
    B, C, H, W = x.shape
    HW, R, Fi = H * W, B * C, C * H * W
    w0, b0, w2, b2 = (t.detach() for t in (blk.block[0].weight, blk.block[0].bias, blk.block[2].weight,
                                           blk.block[2].bias))
    wf, bf = fc.weight.detach(), fc.bias.detach()
    out = {}

    def lin(key, xin, w, b):
        Bn, K = xin.shape
        N = w.shape[0]
        ws, nb = workspace('hk_linear_fwd_workspace_bytes', Bn, K, N)
        y = torch.empty(Bn, N, device='cuda')
        abi('hk_linear_fwd', xin, w, b, y, Bn, K, N, ws, nb)
        out[key] = y
        return y

    def lin_bwd(key, dy, xin, w):
        Bn, K = xin.shape
        N = w.shape[0]
        dx = torch.empty(Bn, K, device='cuda')
        abi('hk_linear_dgrad', dy, w, dx, Bn, K, N)
        dw, db = torch.empty_like(w), torch.empty(N, device='cuda')
        abi('hk_linear_wgrad', dy, xin, dw, db, Bn, K, N)
        out[key] = (dx, dw, db)

    z = torch.empty(B, C, device='cuda')
    abi('hk_row_mean_fwd', x, z, R, HW, HW)
    out['z'] = z
    a = lin('a', z, w0, b0)
    h = torch.empty_like(a)
    abi('hk_act_fwd', a, h, a.numel(), 0)
    out['h'] = h
    m = lin('m', h, w2, b2)
    s = torch.empty_like(x)
    abi('hk_se_gate_fwd', x, m, s, R, HW)
    out['s'] = s
    lin('f', s.reshape(B, Fi), wf, bf)
    lin_bwd('df', up['f'], s.reshape(B, Fi), wf)
    dxg, dm = torch.empty_like(x), torch.empty_like(m)
    abi('hk_se_gate_bwd', x, m, up['s'].contiguous(), dxg, dm, R, HW)
    out['ds'] = (dxg, dm)
    lin_bwd('dm', up['m'], h, w2)
    da = torch.empty_like(a)
    abi('hk_act_bwd', h, up['h'], da, a.numel(), 0)
    out['da'] = da
    lin_bwd('da_', up['a'], z, w0)
    dxz = torch.empty(R, HW, device='cuda')
    abi('hk_row_mean_bwd', up['z'].contiguous(), dxz, R, HW, HW)
    out['dz'] = dxz.reshape(x.shape)
    return out


@pytest.mark.gpu
def test_composed_head_b32():
    """OSME(2048, 1024, 14, 2), nn.Linear(1024, 200) and MAMCLoss(lambda_a = 0.5) through autograd at batch 32 on a
    post-ReLU map, TF32 mode: every stage bit-identical to its direct C-ABI call on the same inputs, x.grad within three
    fp32 adds of the fp64 sum of its four contributions, last_correct against the fp64 argmax, and the rel-L2 of loss,
    logits, x_part and all 14 parameter gradients to an fp64 composition"""
    from hawkeye_b200 import _lib, ops, ops_cin
    from hawkeye_b200.losses import MAMCLoss
    from hawkeye_b200.methods.osme import OSME
    _lib.set_precise(0)
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    B, C, H, P, D, K, _ = CASES['b32_14x14']
    HW = H * H
    torch.manual_seed(1000)
    with torch.device('cuda'):
        osme = OSME(C, D, feature_shape=H, num_attention=P).train()
        cls = nn.Linear(D, K)
    with torch.no_grad():           # the top-1 among the batch's 8 classes, so that last_correct counts something
        cls.bias[8:] -= 10.0
    crit = MAMCLoss(_Cfg(lambda_a=LAMBDA_A))
    x = trunk_map(B, C, HW, 1001).reshape(B, C, H, H)
    labels = layout_labels(B, 'class_major').cuda()
    params = dict(list(osme.named_parameters()) + [(f'classifier.{k}', v) for k, v in cls.named_parameters()])
    assert len(params) == 14
    # the module's path: forward outputs and the input gradient
    xm = x.clone().requires_grad_(True)
    x1_m, part_m = osme(xm)
    logits_m = ops.linear(x1_m, cls.weight, cls.bias)
    loss_m = crit((logits_m, part_m), labels)
    (dx_m,) = torch.autograd.grad(loss_m, xm)
    loss_m, logits_m, part_m = loss_m.detach(), logits_m.detach(), part_m.detach()
    # the same Functions stage by stage in OSME.forward's order (both blocks, then both FCs), keeping every intermediate
    # and its gradient
    xs = x.clone().requires_grad_(True)
    st = []
    for blk in osme.blocks:
        z = ops.RowMeanFn.apply(xs.reshape(B, C, HW))
        a = ops.linear(z, blk.block[0].weight, blk.block[0].bias)
        h = ops.ActFn.apply(a, False)
        m = ops.linear(h, blk.block[2].weight, blk.block[2].bias)
        st.append(dict(z=z, a=a, h=h, m=m, s=ops_cin.SEGateFn.apply(xs, m)))
    for d, fc in zip(st, osme.fcs):
        d['f'] = ops.linear(d['s'].reshape(B, -1), fc.weight, fc.bias)
        for t in d.values():
            t.retain_grad()
    feats = [d['f'] for d in st]
    x1, x_part = sum(feats), torch.stack(feats, dim=1)
    logits = ops.linear(x1, cls.weight, cls.bias)
    for t in (x1, x_part, logits):
        t.retain_grad()
    loss = crit((logits, x_part), labels)
    loss.backward()
    assert torch.equal(loss.detach(), loss_m) and torch.equal(logits.detach(), logits_m), 'staged path differs'
    assert torch.equal(x_part.detach(), part_m) and torch.equal(xs.grad, dx_m), 'staged path differs from the module'
    with torch.no_grad():
        # the loss: cross-entropy and the N-pairs chain
        ce = guarded((1,))
        dlog = guarded((B, K))
        corr = guarded((1,), dtype=torch.int32, fill=-1, word=-7)
        abi('hk_softmax_ce_ls', logits, labels, ce, dlog, corr, B, K, 0.1, 1.0)
        np_ = run_npairs(x_part.detach(), labels)
        assert torch.equal(loss, ce[0] + LAMBDA_A * np_['loss'][0].float()), 'MAMCLoss differs from its C-ABI calls'
        assert torch.equal(logits.grad, dlog), 'the cross-entropy gradient differs from hk_softmax_ce_ls'
        assert torch.equal(x_part.grad, (np_['dx'] * LAMBDA_A).reshape(B, P, D)), 'the N-pairs gradient differs'
        assert torch.equal(crit.last_correct, corr), 'last_correct differs from hk_softmax_ce_ls'
        ws, nb = workspace('hk_linear_fwd_workspace_bytes', B, D, K)
        lo = torch.empty(B, K, device='cuda')
        abi('hk_linear_fwd', x1, cls.weight, cls.bias, lo, B, D, K, ws, nb)
        assert torch.equal(lo, logits), 'classifier forward differs from hk_linear_fwd'
        dx1, dwc, dbc = torch.empty(B, D, device='cuda'), torch.empty(K, D, device='cuda'), torch.empty(K, device='cuda')
        abi('hk_linear_dgrad', logits.grad, cls.weight, dx1, B, D, K)
        abi('hk_linear_wgrad', logits.grad, x1, dwc, dbc, B, D, K)
        assert torch.equal(dx1, x1.grad) and torch.equal(dwc, cls.weight.grad) and torch.equal(dbc, cls.bias.grad), \
            'classifier backward differs from hk_linear_dgrad / _wgrad'
        contrib = []
        for i, (blk, fc) in enumerate(zip(osme.blocks, osme.fcs)):
            d = st[i]
            assert torch.equal(d['f'].grad, x1.grad + x_part.grad[:, i]), f'attention {i}: f.grad is not the sum'
            up = {k: d[k].grad for k in ('f', 's', 'm', 'h', 'a', 'z')}
            o = _gpu_osmeabi(x, blk, fc, up)
            for k in ('z', 'a', 'h', 'm', 's', 'f'):
                assert torch.equal(o[k], d[k].detach()), f'attention {i}: forward {k} differs from its C-ABI call'
            checks = (('s', o['df'][0].reshape(B, C, H, H)), ('m', o['ds'][1]), ('h', o['dm'][0]), ('a', o['da']),
                      ('z', o['da_'][0]))
            for k, ref in checks:
                assert torch.equal(d[k].grad, ref), f'attention {i}: gradient of {k} differs from its C-ABI call'
            for (k, p), ref in zip(((f'blocks.{i}.block.0', blk.block[0]), (f'blocks.{i}.block.2', blk.block[2]),
                                    (f'fcs.{i}', fc)), (o['da_'], o['dm'], o['df'])):
                assert torch.equal(p.weight.grad, ref[1]) and torch.equal(p.bias.grad, ref[2]), \
                    f'{k}: parameter gradient differs from hk_linear_wgrad'
            contrib += [o['ds'][0], o['dz']]
            del o
        # x.grad: two gates and two row means, summed by autograd in an unspecified order
        cs = [c.to(F64) for c in contrib]
        ref = sum(cs)
        bound = 3 * U * sum(c.abs() for c in cs)
        check(xs.grad, ref, bound, 'composed x.grad (four contributions)', names=('image', 'channel', 'h', 'w'))
        del cs, ref, bound, contrib
    # the fp64 composition
    x64 = x.to(F64).reshape(B, C, HW)
    p64 = {k: v.detach().to(F64).requires_grad_(True) for k, v in params.items() if not k.startswith('fcs.')}
    keeps, f64 = [], []
    for i in range(P):
        s64, _ = osme_block64(x64, *(p64[f'blocks.{i}.block.{j}.{t}'] for j in (0, 2) for t in ('weight', 'bias')))
        keeps.append({})
        f64.append(_FC64.apply(s64.reshape(B, -1), osme.fcs[i].weight.detach(), osme.fcs[i].bias.detach(), keeps[-1]))
    part64 = torch.stack(f64, 1)
    logits64 = sum(f64) @ p64['classifier.weight'].T + p64['classifier.bias']
    loss64 = mamc64(logits64, part64, labels)
    small = list(p64)
    grads = dict(zip(small, torch.autograd.grad(loss64, [p64[k] for k in small])))
    rl = {'loss': abs(float(loss.detach()) - float(loss64.detach())) / abs(float(loss64.detach())), 'logits': rel_l2(logits, logits64),
          'x_part': rel_l2(x_part, part64)}
    for k in small:
        rl[k] = rel_l2(params[k].grad, grads[k])
    for i in range(P):
        dy, s = keeps[i]['dy'].detach(), keeps[i]['s'].detach()
        w = params[f'fcs.{i}.weight'].grad
        num = den = 0.0
        for r in range(0, D, ROWS):
            ref = dy[:, r:r + ROWS].T @ s
            num += float((w[r:r + ROWS].to(F64) - ref).norm() ** 2)
            den += float(ref.norm() ** 2)
        rl[f'fcs.{i}.weight'] = math.sqrt(num / den)
        rl[f'fcs.{i}.bias'] = rel_l2(params[f'fcs.{i}.bias'].grad, dy.sum(0))
    print('composed head B=32, rel-L2 to the fp64 composition: ' + ', '.join(f'{k} {v:.3g}' for k, v in rl.items()),
          flush=True)
    # last_correct: the fp32 logits' top-1 against the fp64 argmax, up to rows whose top two are closer than the error
    top = logits64.detach().topk(2, dim=1).values
    err = (logits.detach().to(F64) - logits64.detach()).abs().max(1).values
    ambiguous = int((top[:, 0] - top[:, 1] <= 2 * err).sum())
    c64 = int((logits64.detach().argmax(1) == labels).sum())
    print(f'last_correct {int(crit.last_correct)}, fp64 argmax {c64}, {ambiguous} ambiguous rows', flush=True)
    assert abs(int(crit.last_correct) - c64) <= ambiguous
    # measured on an H100 80GB HBM3 (700 W): loss 2.5e-6, logits 2.0e-5, x_part 7.8e-4, parameter gradients 2.8e-4 (fcs
    # weights) to 1.6e-3 (the excitation weights)
    assert rl['loss'] < 1e-4 and rl['logits'] < 1e-3 and rl['x_part'] < 1e-2
    assert max(v for k, v in rl.items() if k not in ('loss', 'logits', 'x_part')) < 2e-2
    _report('composed head', t0)


# ------------------------------------------------------------------------------------------------------------------
# 5. the optimizer step over the head group
# ------------------------------------------------------------------------------------------------------------------
def _check_sgd(tag, flat, opt, p_old, b_old, first):
    """every element of both groups' p and buf against sgd_momentum_step in fp64, SGD_CHUNK at a time"""
    worst = (0.0, '')
    for gi, ((a, b), pg) in enumerate(zip(flat.group_slices, opt.param_groups)):
        lr, m, wd = f32(pg['lr']), f32(pg['momentum']), f32(pg['weight_decay'])
        for c0 in range(a, b, SGD_CHUNK):
            c1 = min(c0 + SGD_CHUNK, b)
            p = p_old[c0:c1].cuda().to(F64)
            g = flat.grad[c0:c1].to(F64)
            bo = None if first else b_old[c0:c1].cuda().to(F64)
            p_ref, b_ref, pb, bb = sgd_bounds(p, g, bo, lr, m, wd, first)
            for what, o, ref, bound in (('p', flat.flat[c0:c1], p_ref, pb), ('buf', opt.buf[c0:c1], b_ref, bb)):
                err = (o.to(F64) - ref).abs()
                r = torch.where(err == 0, torch.zeros_like(err), err / bound)
                k = int(torch.nan_to_num(r, nan=math.inf).argmax())
                if float(r[k]) > worst[0]:
                    worst = (float(r[k]), f'group {gi} {what} element {c0 + k}')
                assert float(r[k]) <= 1, f'{tag}: group {gi} {what} element {c0 + k}: out {float(o[k]):.9g} ref ' \
                                         f'{float(ref[k]):.9g} bound {float(bound[k]):.3g}'
    print(f'{tag}: worst |err| / bound {worst[0]:.3g} ({worst[1]})', flush=True)


@pytest.mark.gpu
def test_head_sgd_steps():
    """FusedSGD over a trunk stand-in (lr x 0.1) and the head's 823 M floats (lr x 1.0) with configs/OSMENet.yaml's lr,
    momentum (none given: 0) and weight decay: the first step, one after it, one with momentum 0.9, then a direct
    hk_sgd_momentum over a slice of 4099 floats, whose last 3 run the scalar tail"""
    from hawkeye_b200 import _lib, engine
    from hawkeye_b200.config import load_config
    from hawkeye_b200.methods.osme import OSME
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    oc = load_config(os.path.join(REPO, 'configs', 'OSMENet.yaml')).train.optimizer
    lr, wd = oc.lr, oc.weight_decay
    mom = oc.momentum if 'momentum' in oc else 0.0
    torch.manual_seed(1100)
    with torch.device('cuda'):
        trunk = nn.Linear(1000, 7)
        head = nn.ModuleList([OSME(2048, 1024, feature_shape=14, num_attention=2), nn.Linear(1024, 200)])
    flat = engine.FlatParams(None, groups=[list(trunk.parameters()), list(head.parameters())])
    a, b = flat.group_slices[1]
    print(f'head group: {b - a} floats ({(b - a) * 4 / 2 ** 30:.2f} GiB)', flush=True)
    assert (b - a) * 4 > 2 ** 31 and b - a > 823_000_000
    opt = engine.FusedSGD(flat, lr=lr, momentum=mom, weight_decay=wd, group_lrs=[lr * 0.1, lr * 1.0])
    g = torch.Generator(device='cuda').manual_seed(1101)
    p_old = flat.flat.cpu()
    for step in range(3):
        flat.grad.normal_(generator=g).mul_(1e-3)
        if step == 2:
            for pg in opt.param_groups:
                pg['momentum'] = 0.9
        first = opt.first
        b_old = None if first else opt.buf.cpu()
        opt.step()
        torch.cuda.synchronize()
        _check_sgd(f'SGD step {step} (momentum {opt.param_groups[1]["momentum"]}, first {first})', flat, opt, p_old,
                   b_old, first)
        p_old = flat.flat.cpu()
    del p_old, b_old
    n, lo = 4099, b - 4100
    keep = (flat.flat[lo:lo + 4100].clone(), opt.buf[lo:lo + 4100].clone())
    lr32, wd32 = f32(lr), f32(wd)
    abi('hk_sgd_momentum', flat.flat[lo:lo + n], flat.grad[lo:lo + n], opt.buf[lo:lo + n], n, lr32, 0.9, wd32, 1.0, 0)
    p_ref, b_ref, pb, bb = sgd_bounds(keep[0][:n].to(F64), flat.grad[lo:lo + n].to(F64), keep[1][:n].to(F64), lr32,
                                      f32(0.9), wd32, False)
    check(flat.flat[lo:lo + n], p_ref, pb, 'SGD 4099 floats p', names=('element',))
    check(opt.buf[lo:lo + n], b_ref, bb, 'SGD 4099 floats buf', names=('element',))
    assert torch.equal(flat.flat[lo + n], keep[0][n]) and torch.equal(opt.buf[lo + n], keep[1][n]), \
        'hk_sgd_momentum wrote past n'
    _report('SGD', t0)


# ------------------------------------------------------------------------------------------------------------------
# 6. CPU self-tests: the restatements are the oracle's and the reference's, and the bounds reject real defects
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('B, layout', [(32, lay) for lay in LAYOUTS] + [(10, 'class_major'), (4, 'class_major')])
def test_npairs_restatement_matches_oracle(B, layout):
    from oracle import hop_oracle as O
    P, D, K = 2, 48, 200
    labels = layout_labels(B, layout, 930)
    feats = npair_features(B, P, D, labels, 20, 'cpu').to(F64)
    torch.testing.assert_close(npairs64(feats, labels), O.npairs_loss(feats, labels), rtol=1e-12, atol=0)
    pred = detgen.det((B, K), 21).to(F64)
    torch.testing.assert_close(mamc64(pred, feats, labels), O.mamc_loss(pred, feats, labels), rtol=1e-12, atol=0)
    # the closed-form dprod of npair_scales is the restatement's gradient
    xn = F.normalize(feats.reshape(B * P, D), dim=1)
    prod = (xn @ xn.T).requires_grad_(True)
    (g,) = torch.autograd.grad(npair_from_prod(prod, labels, P), prod)
    torch.testing.assert_close(npair_scales(prod.detach(), labels, P)[2], g, rtol=1e-10, atol=1e-15)


def test_osme_restatement_is_the_reference_formula():
    """osme_block64 against OSME_block's own nn.Sequential (Linear, ReLU, Linear, Sigmoid) in fp64: sigmoid(block(mean x))
    * x, then the Linear over the flattened map"""
    from hawkeye_b200.methods.osme import OSME
    torch.manual_seed(5)
    m = OSME(64, 16, feature_shape=3, num_attention=2).double()
    x = torch.relu(torch.randn(3, 64, 3, 3, dtype=F64))
    for blk, fc in zip(m.blocks, m.fcs):
        ref = blk.block(F.adaptive_avg_pool2d(x, 1).flatten(1)).view(3, 64, 1, 1) * x
        s, _ = osme_block64(x.reshape(3, 64, 9), blk.block[0].weight, blk.block[0].bias, blk.block[2].weight,
                            blk.block[2].bias)
        torch.testing.assert_close(s.reshape(x.shape), ref, rtol=1e-13, atol=0)
        torch.testing.assert_close(s.reshape(3, -1) @ fc.weight.T + fc.bias, fc(ref.reshape(3, -1)), rtol=1e-12, atol=0)


def _rejected(tag, bad, ref, bound):
    """the fp32-rounded defect violates the bound somewhere -> worst |err| / bound"""
    err = (bad.float().to(F64) - ref).abs()
    r = float(torch.where(err == 0, torch.zeros_like(err), err / bound).max())
    print(f'defect {tag}: worst |err| / bound {r:.3g}', flush=True)
    assert r > 1, f'{tag}: not rejected ({r:.3g})'


def test_bounds_reject_linear_defects():
    B, K, N = 3, 8 * 1024, 16
    x, w, b, dy, S = classifier_inputs(B, K, N, 31, 'cpu')
    assert S == 8
    refs = linear_refs(x, w, b, dy, S)
    ref, fixed, scale = refs['y']
    bound = fixed + C_LIN * scale
    xd, wd, bd = x.to(F64), w.to(F64), b.to(F64)
    Kc = K // S
    sl = [slice(s * Kc, (s + 1) * Kc) for s in range(S)]
    _rejected('linear without K slice 3', ref - xd[:, sl[3]] @ wd[:, sl[3]].T, ref, bound)
    _rejected("linear, the last slice read at its neighbour's offset",
              ref - xd[:, sl[-1]] @ wd[:, sl[-1]].T + xd[:, sl[-2]] @ wd[:, sl[-2]].T, ref, bound)
    _rejected('linear with the bias added once per slice', ref + (S - 1) * bd, ref, bound)
    ref, fixed, _ = refs['db']
    _rejected('db without image 1', ref - dy[1].to(F64), ref, fixed)


def test_bounds_reject_row_mean_and_gate_defects():
    R, HW = 64, 49
    x = trunk_map(1, R, HW, 40, 'cpu')[0]
    ref, bound = row_mean_bound(x, HW)
    _rejected('row mean divided by the padded width 52', x.to(F64).sum(1) / 52, ref, bound)
    m = detgen.det((R,), 41, 2.0)
    ds = detgen.det((R, HW), 42, 1e-3)
    (sr, sb), (dxr, dxb), (dmr, dmb) = se_gate_bounds(x, m, ds, HW)
    g = torch.sigmoid(m.to(F64))
    _rejected('gate with sigmoid(-m)', (1 - g)[:, None] * x.to(F64), sr, sb)
    _rejected('gate dx with sigmoid(-m)', (1 - g)[:, None] * ds.to(F64), dxr, dxb)
    _rejected('dm without g(1 - g)', (ds.to(F64) * x.to(F64)).sum(1), dmr, dmb)
    _rejected("gate of the neighbouring row", g.roll(-1)[:, None] * x.to(F64), sr, sb)


def test_bounds_reject_npairs_defects():
    B, P, D = 32, 2, 64
    labels = layout_labels(B, 'class_major')
    feats = npair_features(B, P, D, labels, 50, 'cpu')
    xn = F.normalize(feats.reshape(B * P, D), dim=1)
    prod = (xn.to(F64) @ xn.to(F64).T).float().to(F64).requires_grad_(True)
    loss = npair_from_prod(prod, labels, P)
    (dprod,) = torch.autograd.grad(loss, prod)
    sl, sd, _ = npair_scales(prod.detach(), labels, P)
    for defect in ('repeat', 'no_self', 'ea_for_b', 'no_inv_n'):
        p2 = prod.detach().clone().requires_grad_(True)
        bad = npair_from_prod(p2, labels, P, **{defect: True})
        (bd,) = torch.autograd.grad(bad, p2)
        _rejected(f'npair loss, {defect}', bad.detach().reshape(1), loss.detach().reshape(1), C_NP * sl.reshape(1))
        _rejected(f'npair dprod, {defect}', bd, dprod, C_NP * sd)
    dp32 = dprod.float()
    (tr, tf, ts), (dr, df, ds) = anchor_bwd64(dp32, xn)
    _rejected('dF = 2 dprod F', anchor_bwd64(dp32, xn, symmetric=False)[1][0], dr, df + C_LIN * ds)
    dxn = dr.float()
    ref, bound = l2norm_bwd64(xn, 1 / feats.reshape(B * P, D).norm(dim=1), dxn)
    _rejected('l2norm backward without its projection term',
              l2norm_bwd64(xn, 1 / feats.reshape(B * P, D).norm(dim=1), dxn, projection=False)[0], ref, bound)
