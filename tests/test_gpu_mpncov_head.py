"""The Fast MPN-COV head of the mpn train step, element by element against fp64: hk_covpool_fwd / _bwd, hk_sqrtm_fwd /
_bwd and hk_triuvec_fwd / _bwd at the batch-32, 448x448 shapes (and the 224x224 batch-8 shape of the reference config),
the classifier behind them, and the composed head through autograd.  The dimension-reduction unit in front of them is
checked with the other ResNet-50 units (test_gpu_resnet50_units.py).

Every kernel is called through the C ABI into NaN-filled outputs followed by guard words, with NaN-filled workspaces of
exactly the queried size and a NaN-filled `saved` buffer of exactly hk_sqrtm_saved_floats floats, also followed by
guard words; inputs are followed by NaN, so a read past their end poisons the result.  Each stage is compared with fp64
applied to the fp32 values that stage was given (its inputs are the previous kernel's outputs), with ref computed on the
GPU, CHUNK images at a time.

Error model (u = 2^-24; RND = 2^-11, the tf32 round-to-nearest on store; TRUNC = 2^-10, the MMA's truncation of an
operand that is not tf32; PAIR = 2^-22, what a (hi, lo) tf32 pair loses: its representation error, or the dropped lo.lo
product).  Each bound is `fixed + c * scale`, with `fixed` the analysed roundings and c a measured constant:

  covpool xc      e_s + (2u + RND) max(|out|, |ref|), e_s = (ceil(M / 32) + 7) u sum_k |x_ik| / M, the error of the
                  fp32 row mean (32 lanes, then a 5-level warp tree); RND in TF32 mode only
  covpool cov     scale S = |xc| |xc|^T / M.  fixed = (2 r + 3u) S + (e_s,i sum_k |xc_jk| + e_s,j sum_k |xc_ik|) / M:
                  r = RND + u (xc rounded on store; its products are exact) in TF32 mode, 3 PAIR in 3xTF32 mode
  covpool dx      scale (|g| + |g^T|) |xc| / M, two GEMMs, the second reading the first's raw output as its addend E.
                  fixed = (TRUNC + 4u) scale in TF32 mode (g is not tf32), (3 PAIR + 4u) scale in 3xTF32 mode
  sqrtm y, dx     a first-order error-bound matrix propagated through the recurrence (below)
  triuvec         exact; the strict lower triangle of dx is +0.0
  classifier      scale |x| |w|^T + |b| (fixed (S + 1) u scale for the split sum), |dy| |w|, |dy|^T |x|; db: 32 terms,
                  2^-19 sum |dy|.  The inputs are tf32, so only accumulation remains

Every Newton-Schulz product is mm3 (mpncov.cu): C = alpha A.B + delta I + beta D on (hi, lo) pairs.  Alongside the fp64
reference, each matrix X carries an elementwise bound E_X on |X_kernel - X_ref|, as two parts (fixed, coefficient of c):

  E_C = |alpha| (|A| E_B + E_A |B|) + |beta| E_D + (4u + PAIR) (|alpha| |A||B| + |delta| I + |beta| |D|)
        + PAIR |alpha| |A||B|  +  c |alpha| |A||B|

(4u: the epilogue's sum of the two accumulators, alpha, the diagonal and the addend; PAIR: the stored pair and the dropped
lo.lo; c: the fp32 accumulation of K = n exact tf32 products).  It starts from the trace normalisation (normA, an fp32
sum of n diagonal terms over 256 threads: e_tr = (ceil(n / 256) + 13) u relative, then 1 / normA and the product: 2u +
PAIR) and the initial split 0.5 (3I - A) (2u + PAIR), and ends with y = (hi + lo) sqrt(normA) (e_tr / 2 + 3u).  The
backward starts from P = g sqrt(normA) (e_tr / 2 + 2u + PAIR), uses the forward's Y_i, Z_i with their E_Y, E_Z, and
counts the tail kernel's fp32 work: D = (acc - dZ / 2)^T (3u), its sums gaux = sum D.x and gy = sum g.y (each (ceil(n^2 /
256) + 13) u of the sum of |terms|, per-thread fmaf chains and a block tree), the diagonal coefficient gy / (2 normA) -
gaux / normA^2 (normA's e_tr, five roundings) and D / normA (e_tr + u).  Second-order terms (E.E) are dropped; they are
below 1e-10 of the first-order ones here.

The worst (|err| - fixed) / scale measured over every check of this file on an H100 80GB HBM3 (700 W), and the margin
of each c over it:

  C_COV   2^-20   covpool fwd and bwd GEMM accumulation    0: the fixed terms alone covered every element (their
                                                           worst-case tf32 rounding and truncation); c is the
                                                           accumulation allowance they leave out
  C_NS    2^-19   one Newton-Schulz pair product           3.1e-7 = 2^-21.6 (b32_14x14_it3 sqrtm y)       6.2x
  C_LIN   2^-19   classifier fwd / dgrad / wgrad           4.3e-7 = 2^-21.2 (classifier dx)              4.4x

Of the whole bound (fixed + c * scale), the worst element took 0.80 in covpool dx, 0.48 in cov, 0.37 in sqrtm y and 0.31
in sqrtm dx; xc's bound is its rounding on store, which any element just below a rounding midpoint nearly fills (0.997).

The composed head's rel-L2 to the fp64 composition is printed and loosely bounded:
it measures how the chain amplifies the trunk's TF32 rounding, not a kernel's error.

The self-tests (no GPU) compute defects in fp64 at a small shape, round them to fp32, and check that the loosest bounds
(TF32 mode) reject each: Newton-Schulz one iteration short; one mm3 link single-pass; the backward tail without its
transpose; the diagonal coefficient with the neighbouring image's normA or without its aux term; one 128x64 output tile of
an image taken from the next image; the centring mean divided by the padded M; the covpool backward without its g^T term;
the classifier without one K slice or without the partial last k-block of every slice.
"""
import math
import time

import pytest
import torch

import detgen
from fp64_refs import C_LIN, classifier_inputs, linear_refs, linear_splits
from kernel_check import (PAIR, RND, TRUNC, U, Bound, Out, Worst, abi, c_bound, check, guarded, poisoned, rnd_bound,
                          workspace)

EPI = 4 * U
C_COV = 2.0 ** -20
C_NS = 2.0 ** -19
CHUNK = 8
F64 = torch.float64

# case -> (B, C, H, W, iterN, precise)
CASES = {
    'b32_14x14_it5': (32, 256, 14, 14, 5, 0),   # the mpn step: M = 196 < C, singular covariances; 256 pair tiles
    'b32_14x14_it3': (32, 256, 14, 14, 3, 0),
    'b8_7x7': (8, 256, 7, 7, 5, 0),             # the reference config (224x224, batch 8): M = 49 padded to 52
    'b17_14x14': (17, 256, 14, 14, 5, 0),       # 136 pair tiles: just past 132 SMs
    'b37_7x7': (37, 256, 7, 7, 2, 0),           # 296 tiles; B % 4 != 0 pads normA; iterN = 2: empty Newton-Schulz loops
    'precise_b4_14x14': (4, 256, 14, 14, 5, 1),
}
F_CLS, N_CLS = 256 * 257 // 2, 200


# ------------------------------------------------------------------------------------------------------------------
# 1. fp64 restatements (device-agnostic) with first-order error bounds
# ------------------------------------------------------------------------------------------------------------------
def pad4(v):
    return (v + 3) & ~3


def _hi(t):
    """the tf32 hi half of a value: what a single-pass product keeps of a (hi, lo) pair"""
    return detgen.tf32_rna(t.float()).to(t.dtype)


def _zero_e(t):
    return torch.zeros((2,) + tuple(t.shape), dtype=F64, device=t.device)


def covpool_fwd64(x, mean_div=None):
    """X I_hat X^T = xc xc^T / M (MPNCOV.py:107-119) -> (cov, xc [B, C, M]); mean_div replaces M in the mean (a defect)"""
    B, C, H, W = x.shape
    M = H * W
    X = x.reshape(B, C, M).to(F64)
    xc = X - X.sum(-1, keepdim=True) / (mean_div or M)
    return xc @ xc.mT / M, xc


def covpool_bwd64(xc, g, M, transpose_term=True):
    """(g + g^T) X I_hat = (g + g^T) xc / M (MPNCOV.py:121-134); without the g^T term when transpose_term is False"""
    gd = g.to(F64)
    return ((gd + gd.mT) if transpose_term else gd) @ xc.to(F64) / M


def covpool_fwd_bounds(x, precise):
    """fp64 cov and xc of the fp32 map x, and (xc's mean term e_s, cov's fixed bound, cov's c-scale S)"""
    B, C, H, W = x.shape
    M = H * W
    cov, xc = covpool_fwd64(x)
    e_s = (math.ceil(M / 32) + 7) * U * x.reshape(B, C, M).to(F64).abs().sum(-1, keepdim=True) / M
    ac = xc.abs()
    S = ac @ ac.mT / M
    r = 3 * PAIR if precise else RND + U
    t = e_s * ac.sum(-1).unsqueeze(1) / M
    return cov, xc, e_s, (2 * r + 3 * U) * S + t + t.mT, S


def covpool_bwd_bounds(xc, g, M, precise):
    """fp64 dx of the given xc [B, C, M] and g, its fixed bound and c-scale"""
    ref = covpool_bwd64(xc, g, M)
    ga = g.to(F64).abs()
    scale = (ga + ga.mT) @ xc.to(F64).abs() / M
    return ref, ((3 * PAIR if precise else TRUNC) + 4 * U) * scale, scale


class Chain:
    """hk_sqrtm_fwd / _bwd (MPNCOV.py:137-202) in fp64, product by product in mpncov.cu's order, each matrix with its
    error bound [fixed, per unit of c] (see the module docstring).  `defect` switches in the self-tests' defects:
    single=k (the k-th mm3 single-pass), no_transpose, neighbour_norm, no_aux."""

    def __init__(self, n, device, **defect):
        self.I = torch.eye(n, dtype=F64, device=device)
        self.n, self.k, self.defect = n, 0, defect

    def mm(self, A, B, alpha=1.0, diag=0.0, D=None, beta=0.0):
        (a, ea), (b, eb) = A, B
        if self.defect.get('single') == self.k:
            a, b = _hi(a), _hi(b)
        self.k += 1
        aa, ab = a.abs(), b.abs()
        mag = abs(alpha) * (aa @ ab)
        c = alpha * (a @ b) + diag * self.I
        e = abs(alpha) * (aa @ eb + ea @ ab)
        rounded = mag + abs(diag) * self.I
        if D is not None:
            c = c + beta * D[0]
            e = e + abs(beta) * D[1]
            rounded = rounded + abs(beta) * D[0].abs()
        e[0] += (EPI + PAIR) * rounded + PAIR * mag
        e[1] += mag
        return c, e

    def affine(self, A, alpha, diag):
        """affine_diag_split_kernel: alpha (hi + lo) + diag I, split into a new pair (two roundings and the split)"""
        a, ea = A
        c = alpha * a + diag * self.I
        e = abs(alpha) * ea
        e[0] += (2 * U + PAIR) * (abs(alpha) * a.abs() + abs(diag) * self.I)
        return c, e

    def fwd(self, x, iterN):
        """-> (y, E_y), saved"""
        n = self.n
        xd = x.to(F64)
        dg = xd.diagonal(dim1=1, dim2=2)
        tr = dg.sum(1)
        e_tr = (math.ceil(n / 256) + 13) * U * dg.abs().sum(1) / tr.abs()
        A = xd / tr.view(-1, 1, 1)
        EA = _zero_e(A)
        EA[0] = A.abs() * (e_tr + 2 * U + PAIR).view(-1, 1, 1)
        A = (A, EA)
        Z = [self.affine(A, -0.5, 1.5)]
        Y = [self.mm(A, Z[0])]
        for _ in range(1, iterN - 1):
            ZY = self.mm(Z[-1], Y[-1], -0.5, 1.5)
            Y.append(self.mm(Y[-1], ZY))
            Z.append(self.mm(ZY, Z[-1]))
        T = self.mm(Z[-1], Y[-1], -1.0, 3.0)
        yzy, e = self.mm(Y[-1], T, 0.5)
        s = tr.sqrt().view(-1, 1, 1)
        e[0] += (e_tr.view(-1, 1, 1) / 2 + 3 * U) * yzy.abs()
        return (yzy * s, e * s), dict(A=A, Y=Y, Z=Z, tr=tr, e_tr=e_tr)

    def bwd(self, x, y, g, sv):
        """-> (dx, E_dx); y is the forward output the kernel is given"""
        n, mm = self.n, self.mm
        A, Ys, Zs, tr, e_tr = sv['A'], sv['Y'], sv['Z'], sv['tr'], sv['e_tr']
        L = len(Ys)
        gd = g.to(F64)
        s = tr.sqrt().view(-1, 1, 1)
        EP = _zero_e(gd)
        EP[0] = gd.abs() * s * (e_tr.view(-1, 1, 1) / 2 + 2 * U + PAIR)
        P = (gd * s, EP)
        Yl, Zl = Ys[-1], Zs[-1]
        T1 = mm(Yl, Zl, -1.0, 3.0)
        U_ = mm(P, T1)
        V = mm(Zl, Yl)
        dY = mm(V, P, -0.5, D=U_, beta=0.5)
        W2 = mm(Yl, P)
        dZ = mm(W2, Yl, -0.5)
        for i in range(L - 2, -1, -1):
            Yi, Zi = Ys[i], Zs[i]
            T1 = mm(Yi, Zi, -1.0, 3.0)
            V = mm(Zi, Yi)
            U_ = mm(dY, T1)
            W2 = mm(Zi, dZ)
            acc = mm(W2, Zi, -0.5, D=U_, beta=0.5)
            dY2 = mm(V, dY, -0.5, D=acc, beta=1.0)
            U_ = mm(T1, dZ)
            W2 = mm(Yi, dY)
            acc = mm(W2, Yi, -0.5, D=U_, beta=0.5)
            dZ = mm(dZ, V, -0.5, D=acc, beta=1.0)
            dY = dY2
        E1 = self.affine(A, -1.0, 3.0)
        U_ = mm(dY, E1)
        acc = mm(A, dY, -0.5, D=U_, beta=0.5)
        # sqrtm_bwd_tail_kernel
        Dm = acc[0] - 0.5 * dZ[0]
        ED = acc[1] + 0.5 * dZ[1]
        ED[0] += 3 * U * (acc[0].abs() + 0.5 * dZ[0].abs())
        if not self.defect.get('no_transpose'):
            Dm, ED = Dm.mT, ED.mT
        xd, yd = x.to(F64), y.to(F64)
        kt = (math.ceil(n * n / 256) + 13) * U
        ga = (Dm * xd).sum((1, 2))
        Ega = (ED * xd.abs()).sum((-2, -1))
        Ega[0] += kt * (Dm.abs() * xd.abs()).sum((1, 2))
        gy = (gd * yd).sum((1, 2))
        Egy = _zero_e(gy)
        Egy[0] = kt * (gd.abs() * yd.abs()).sum((1, 2))
        na = tr.roll(-1) if self.defect.get('neighbour_norm') else tr
        aux = 0.0 if self.defect.get('no_aux') else gy / (2 * na)
        coef = aux - ga / (na * na)
        Ec = Egy / (2 * tr) + Ega / (tr * tr)
        Ec[0] += (gy.abs() / (2 * tr) * (e_tr + 3 * U) + ga.abs() / (tr * tr) * (2 * e_tr + 3 * U) +
                  U * (gy.abs() / (2 * tr) + ga.abs() / (tr * tr)))
        t3 = tr.view(-1, 1, 1)
        dx = Dm / t3 + coef.view(-1, 1, 1) * self.I
        E = ED / t3 + Ec.view(2, -1, 1, 1) * self.I
        E[0] += Dm.abs() / t3 * (e_tr.view(-1, 1, 1) + U) + U * dx.abs()
        return dx, E


def triuvec_fwd64(x):
    n = x.shape[-1]
    r, c = torch.triu_indices(n, n, device=x.device)
    return x[:, r, c].unsqueeze(-1)


def triuvec_bwd64(g, n):
    r, c = torch.triu_indices(n, n, device=g.device)
    dx = torch.zeros(g.shape[0], n, n, dtype=g.dtype, device=g.device)
    dx[:, r, c] = g.reshape(g.shape[0], -1)
    return dx


# ------------------------------------------------------------------------------------------------------------------
# 2. inputs and checks
# ------------------------------------------------------------------------------------------------------------------
def feature_map(B, C, H, W, seed):
    """post-ReLU sparse maps, as the dimension-reduction unit emits; a batch of 5 or more ends with an image scaled by
    1e-3 next to one scaled by 1e3, then an image with a single dominant channel"""
    x = torch.relu(detgen.det_uniform((B, C, H, W), seed) - 0.4)
    if B >= 5:
        x[B - 3] *= 1e-3
        x[B - 2] *= 1e3
        x[B - 1] *= 1e-2
        x[B - 1, C // 3] = 10.0 * torch.relu(detgen.det_uniform((H, W), seed + 1) - 0.4)
    return x


def upstream(B, n, seed):
    """the gradient reaching the covariance head: a triuvec vector [B, n(n+1)/2, 1]"""
    return detgen.det((B, n * (n + 1) // 2, 1), seed)


WORST = Worst(C_COV=C_COV, C_NS=C_NS, C_LIN=C_LIN)
check_c = WORST.check_c


def pair_tiles_per_cta(B, n, sms):
    """launch_gemm (gemm.cu) for a batched n x n pair product: 128 x 64 tiles, n-tile fastest, then m-tile, then the
    image; grid = min(tiles, SMs), CTA i takes tiles i, i + grid, ... -> the image of each of its tiles, per CTA"""
    per = -(-n // 128) * -(-n // 64)
    total = per * B
    grid = min(total, sms)
    return [[t // per for t in range(i, total, grid)] for i in range(grid)]


def run_head(case, seed=300):
    """covpool, sqrtm and triuvec forward and backward of `case` through the C ABI into poisoned buffers -> tensors"""
    from hawkeye_b200 import _lib
    B, C, H, W, iterN, precise = CASES[case]
    M, Mp, L = H * W, pad4(H * W), C * (C + 1) // 2
    x = poisoned(feature_map(B, C, H, W, seed).cuda())
    gv = poisoned(upstream(B, C, seed + 2).cuda())
    cov, xc = abi('hk_covpool_fwd', x, Out((B, C, C)), Out((B, C, Mp)), B, C, M, precise=precise)
    saved = guarded((int(_lib.query('hk_sqrtm_saved_floats', B, C, iterN)),))
    ws, nb = workspace('hk_sqrtm_fwd_workspace_bytes', B, C)
    (y,) = abi('hk_sqrtm_fwd', cov, Out((B, C, C)), saved, B, C, iterN, ws, nb, precise=precise)
    (v,) = abi('hk_triuvec_fwd', y, Out((B, L, 1)), B, C, precise=precise)
    (g,) = abi('hk_triuvec_bwd', gv, Out((B, C, C)), B, C, precise=precise)
    ws, nb = workspace('hk_sqrtm_bwd_workspace_bytes', B, C)
    (gx,) = abi('hk_sqrtm_bwd', cov, y, g, saved, Out((B, C, C)), B, C, iterN, ws, nb, precise=precise)
    (dx,) = abi('hk_covpool_bwd', xc, gx, Out((B, C, M)), B, C, M, precise=precise)
    return dict(x=x, gv=gv, cov=cov, xc=xc, y=y, v=v, g=g, gx=gx, dx=dx)


# ------------------------------------------------------------------------------------------------------------------
# 3. the head on the GPU
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('case', ['b32_14x14_it5', 'b17_14x14', 'b37_7x7'])
def test_pair_gemm_ctas_cross_images(case):
    """the pair GEMMs of these batches make persistent CTAs carry their k-block ring from one image to the next (b37:
    some take three tiles)"""
    B, C = CASES[case][:2]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ctas = pair_tiles_per_cta(B, C, sms)
    crossing = sum(len(set(t)) > 1 for t in ctas)
    print(f'{case}: {8 * B} pair tiles on {len(ctas)} CTAs ({sms} SMs); {crossing} CTAs cross an image boundary, '
          f'at most {max(map(len, ctas))} tiles per CTA', flush=True)
    assert crossing > 0
    if B == 37:
        assert max(map(len, ctas)) == 3


@pytest.mark.gpu
@pytest.mark.parametrize('case', list(CASES))
def test_head_stages(case):
    t0 = time.time()
    B, C, H, W, iterN, precise = CASES[case]
    M, Mp = H * W, pad4(H * W)
    d = run_head(case)
    x, xc, cov, y, g, gx, dx = d['x'], d['xc'], d['cov'], d['y'], d['g'], d['gx'], d['dx']
    assert not bool(xc[..., M:].view(torch.int32).any()), 'the pitch padding of xc is not +0.0'
    # triuvec: a gather and a scatter, bit for bit
    assert torch.equal(d['v'], triuvec_fwd64(y)), 'triuvec forward differs from the upper-triangle gather'
    assert torch.equal(g, triuvec_bwd64(d['gv'], C)), 'triuvec backward differs from the scatter'
    assert not bool(torch.tril(g, -1).view(torch.int32).any()), 'the strict lower triangle of dx is not +0.0'
    nm = ('image', 'row', 'col')
    for n0 in range(0, B, CHUNK):
        sl = slice(n0, n0 + CHUNK)
        tag = f'{case} [{n0}:{min(n0 + CHUNK, B)}]'
        ref, xc64, e_s, fixed, S = covpool_fwd_bounds(x[sl], precise)
        xo = xc[sl, :, :M]
        rb = (c_bound if precise else rnd_bound)(e_s.expand_as(xc64), 1.0).total(xo, xc64) + \
            2 * U * torch.fmax(xo.abs(), xc64.abs())
        check(xo, xc64, rb, f'{tag} covpool xc', names=('image', 'channel', 'pos'), n0=n0)
        check_c('C_COV', f'{tag} covpool cov', cov[sl], ref, fixed, S, nm)
        del ref, xc64, fixed, S
        chain = Chain(C, 'cuda')
        (yr, ey), sv = chain.fwd(cov[sl], iterN)
        check_c('C_NS', f'{tag} sqrtm y', y[sl], yr, ey[0], ey[1], nm)
        gr, eg = chain.bwd(cov[sl], y[sl], g[sl], sv)
        check_c('C_NS', f'{tag} sqrtm dx', gx[sl], gr, eg[0], eg[1], nm)
        del sv, yr, ey, gr, eg
        ref, fixed, scale = covpool_bwd_bounds(xc[sl, :, :M], gx[sl], M, precise)
        check_c('C_COV', f'{tag} covpool dx', dx[sl], ref, fixed, scale, ('image', 'channel', 'pos'))
    print(f'{case}: {time.time() - t0:.1f} s; worst shares so far: ' + WORST.summary(), flush=True)


@pytest.mark.gpu
def test_classifier_b32():
    """hk_linear_fwd / _dgrad / _wgrad at B = 32, F = 32896: 32 K slices of 1028 columns, each ending in a partial
    k-block of 4"""
    from hawkeye_b200 import _lib
    _lib.set_precise(0)
    B, F, N = 32, F_CLS, N_CLS
    x, w, b, dy, S = classifier_inputs(B, F, N, 400, 'cuda')
    assert S == 32 and F // S == 1028
    xi, wi, bi, dyi = (poisoned(t) for t in (x, w, b, dy))
    ws, nb = workspace('hk_linear_fwd_workspace_bytes', B, F, N)
    (y,) = abi('hk_linear_fwd', xi, wi, bi, Out((B, N)), B, F, N, ws, nb)
    (dx,) = abi('hk_linear_dgrad', dyi, wi, Out((B, F)), B, F, N)
    dw, db = abi('hk_linear_wgrad', dyi, xi, Out((N, F)), Out((N,)), B, F, N)
    refs = linear_refs(x, w, b, dy, S)
    for key, out, names in (('y', y, ('image', 'class')), ('dx', dx, ('image', 'feature')),
                            ('dw', dw, ('class', 'feature')), ('db', db, ('class',))):
        ref, fixed, scale = refs[key]
        if key == 'db':
            check(out, ref, fixed, 'classifier db', names=names)
        else:
            check_c('C_LIN', f'classifier {key}', out, ref, fixed, scale, names)


class _Head64(torch.autograd.Function):
    """covpool, sqrtm and triuvec in fp64 with the reference's own backward formulae (the restatements above)"""

    @staticmethod
    def forward(ctx, h, iterN):
        B, C, H, W = h.shape
        cov, xc = covpool_fwd64(h)
        chain = Chain(C, h.device)
        (y, _), sv = chain.fwd(cov, iterN)
        ctx.save_for_backward(cov, y, xc)
        ctx.sv, ctx.shape = sv, h.shape
        return triuvec_fwd64(y)

    @staticmethod
    def backward(ctx, gv):
        cov, y, xc = ctx.saved_tensors
        B, C, H, W = ctx.shape
        gc, _ = Chain(C, gv.device).bwd(cov, y, triuvec_bwd64(gv, C), ctx.sv)
        return covpool_bwd64(xc, gc, H * W).reshape(B, C, H, W), None


@pytest.mark.gpu
def test_composed_head_b32():
    """MPNCOV(5, True, True, 2048, 256) and the classifier through autograd at [32, 2048, 14, 14], train mode: every
    deterministic stage bit-identical to its C-ABI call on the same inputs, finite outputs, and the rel-L2 of the logits
    and the input gradient to the fp64 composition"""
    import torch.nn.functional as F
    from hawkeye_b200 import _lib, ops, ops_resnet
    from hawkeye_b200.methods.mpn import MPNCOV
    _lib.set_precise(0)
    torch.manual_seed(500)
    B, Cin, C, H = 32, 2048, 256, 14
    M, L = H * H, C * (C + 1) // 2
    pool = MPNCOV(5, True, True, Cin, C).cuda().train()
    g = torch.Generator(device='cuda').manual_seed(501)
    x = torch.relu(torch.randn(B, Cin, H, H, device='cuda', generator=g))
    w = torch.randn(N_CLS, L, device='cuda', generator=g) * L ** -0.5
    b = torch.randn(N_CLS, device='cuda', generator=g) * 0.01
    dlogits = detgen.tf32_rna(torch.randn(B, N_CLS, device='cuda', generator=g) * 0.01)
    # the module's path
    xm = x.clone().requires_grad_(True)
    logits_m = ops.linear(pool(xm).view(B, -1), w, b)
    (dx_m,) = torch.autograd.grad(logits_m, xm, dlogits)
    # the same Functions, stage by stage, keeping every intermediate and its gradient
    xs = x.clone().requires_grad_(True)
    h = ops.ToNCHWFn.apply(ops_resnet.unit(ops.ToNHWCFn.apply(xs), pool._dr_unit, True))
    c = ops.CovpoolLayer(h)
    s = ops.SqrtmLayer(c, 5)
    t = ops.TriuvecLayer(s)
    logits = ops.linear(t.view(B, -1), w, b)
    for z in (h, c, s, t):
        z.retain_grad()
    logits.backward(dlogits)
    assert torch.equal(logits, logits_m) and torch.equal(xs.grad, dx_m), 'the staged path differs from the module'
    with torch.no_grad():
        cov = guarded((B, C, C))
        xc = guarded((B, C, pad4(M)))
        abi('hk_covpool_fwd', h.contiguous(), cov, xc, B, C, M)
        assert torch.equal(cov, c), 'CovpoolFn forward differs from hk_covpool_fwd'
        dh = guarded((B, C, H, H))
        abi('hk_covpool_bwd', xc, c.grad.contiguous(), dh, B, C, M)
        assert torch.equal(dh, h.grad), 'CovpoolFn backward differs from hk_covpool_bwd'
        y = guarded((B, C, C))
        saved = guarded((int(_lib.query('hk_sqrtm_saved_floats', B, C, 5)),))
        ws, nb = workspace('hk_sqrtm_fwd_workspace_bytes', B, C)
        abi('hk_sqrtm_fwd', c, y, saved, B, C, 5, ws, nb)
        assert torch.equal(y, s), 'SqrtmFn forward differs from hk_sqrtm_fwd'
        gc = guarded((B, C, C))
        ws, nb = workspace('hk_sqrtm_bwd_workspace_bytes', B, C)
        abi('hk_sqrtm_bwd', c, y, s.grad.contiguous(), saved, gc, B, C, 5, ws, nb)
        assert torch.equal(gc, c.grad), 'SqrtmFn backward differs from hk_sqrtm_bwd'
        v = guarded((B, L, 1))
        abi('hk_triuvec_fwd', s, v, B, C)
        assert torch.equal(v, t), 'TriuvecFn forward differs from hk_triuvec_fwd'
        gs = guarded((B, C, C))
        abi('hk_triuvec_bwd', t.grad.contiguous(), gs, B, C)
        assert torch.equal(gs, s.grad), 'TriuvecFn backward differs from hk_triuvec_bwd'
        ws, nb = workspace('hk_linear_fwd_workspace_bytes', B, L, N_CLS)
        lo = guarded((B, N_CLS))
        abi('hk_linear_fwd', t, w, b, lo, B, L, N_CLS, ws, nb)
        assert torch.equal(lo, logits), 'LinearFn forward differs from hk_linear_fwd'
        gt = guarded((B, L))
        abi('hk_linear_dgrad', dlogits, w, gt, B, L, N_CLS)
        assert torch.equal(gt.view(B, L, 1), t.grad), 'LinearFn backward differs from hk_linear_dgrad'
    assert bool(torch.isfinite(logits).all()) and bool(torch.isfinite(xs.grad).all())
    # the fp64 composition
    conv, bn = pool.conv_dr_block[0], pool.conv_dr_block[1]
    x64 = x.to(F64).requires_grad_(True)
    h64 = torch.relu(F.batch_norm(F.conv2d(x64, conv.weight.to(F64)), None, None, bn.weight.to(F64),
                                  bn.bias.to(F64), training=True, eps=bn.eps))
    v64 = _Head64.apply(h64, 5)
    logits64 = v64.view(B, -1) @ w.to(F64).T + b.to(F64)
    (dx64,) = torch.autograd.grad(logits64, x64, dlogits.to(F64))
    logits64 = logits64.detach()
    rl = float((logits.detach().to(F64) - logits64).norm() / logits64.norm())
    rd = float((xs.grad.to(F64) - dx64).norm() / dx64.norm())
    print(f'composed head B=32: rel-L2 to fp64 logits {rl:.3g}, input gradient {rd:.3g}', flush=True)
    # measured on an H100 80GB HBM3 (700 W): 8.3e-4 and 1.5e-2
    assert rl < 1e-2 and rd < 1e-1


# ------------------------------------------------------------------------------------------------------------------
# 4. CPU self-tests: the restatements are the oracle's, and the bounds reject real defects
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('iterN', [2, 3, 5])
def test_restatement_matches_oracle(iterN):
    from oracle import hop_oracle as O
    B, C, H, W = 2, 24, 5, 5
    x = feature_map(B, C, H, W, 10 + iterN).double()
    x[1] *= 1e3
    gm = detgen.det((B, C, C), 11 + iterN).double()
    cov, xc = covpool_fwd64(x)
    torch.testing.assert_close(cov, O.covpool_fwd(x), rtol=1e-12, atol=0)
    torch.testing.assert_close(covpool_bwd64(xc, gm, H * W).reshape(x.shape), O.covpool_bwd(x, gm), rtol=1e-10,
                               atol=1e-14 * float(O.covpool_bwd(x, gm).abs().max()))
    chain = Chain(C, 'cpu')
    (y, _), sv = chain.fwd(cov, iterN)
    y_ref, saved = O.sqrtm_fwd(cov, iterN)
    torch.testing.assert_close(y, y_ref, rtol=1e-12, atol=1e-14 * float(y_ref.abs().max()))
    gx, _ = chain.bwd(cov, y, gm, sv)
    gx_ref = O.sqrtm_bwd(cov, saved, gm, iterN)
    torch.testing.assert_close(gx, gx_ref, rtol=1e-9, atol=1e-12 * float(gx_ref.abs().max()))
    gv = detgen.det((B, C * (C + 1) // 2, 1), 12).double()
    assert torch.equal(triuvec_fwd64(y), O.triuvec_fwd(y))
    assert torch.equal(triuvec_bwd64(gv, C), O.triuvec_bwd(gv, C))
    assert chain.k == 3 * (iterN - 2) + 3 + 10 * (iterN - 2) + 8     # mm3 calls of hk_sqrtm_fwd then hk_sqrtm_bwd


def _rejected(tag, bad, ref, fixed, scale, c, rnd=False):
    """the fp32-rounded defect violates fixed + c * scale (+ the tf32 rounding where the kernel rounds) -> worst ratio"""
    out = bad.float().to(F64)
    bound = fixed + Bound(c * scale.double(), rounded=rnd).total(out, ref)
    err = (out - ref).abs()
    r = float(torch.where(err == 0, torch.zeros_like(err), err / bound).max())
    print(f'defect {tag}: worst |err| / bound {r:.3g}', flush=True)
    assert r > 1, f'{tag}: not rejected ({r:.3g})'
    return r


def _small_head(iterN=5):
    """B = 3, n = 128, 7x7 maps (M = 49 padded to 52): the stage inputs as fp32, as the kernels would get them"""
    B, C, H, W = 3, 128, 7, 7
    x = feature_map(B, C, H, W, 20)
    x[1] *= 1e3
    cov = covpool_fwd64(x)[0].float()
    g = triuvec_bwd64(upstream(B, C, 21), C)
    return x, cov, g, iterN


def test_bounds_reject_sqrtm_defects():
    x, cov, g, iterN = _small_head()
    n = cov.shape[-1]
    chain = Chain(n, 'cpu')
    (y, ey), sv = chain.fwd(cov, iterN)
    nf = chain.k
    y32 = y.float()
    gr, eg = chain.bwd(cov, y32, g, sv)
    nb = chain.k - nf
    fy, sy, fg, sg = ey[0], ey[1], eg[0], eg[1]

    def fwd_bwd(it=iterN, **defect):
        ch = Chain(n, 'cpu', **defect)
        (yb, _), s2 = ch.fwd(cov, it)
        return yb, ch.bwd(cov, y32, g, s2)[0]

    short_y, short_g = fwd_bwd(iterN - 1)
    _rejected('Newton-Schulz one iteration short, y', short_y, y, fy, sy, C_NS)
    _rejected('Newton-Schulz one iteration short, dx', short_g, gr, fg, sg, C_NS)
    assert (nf, nb) == (12, 38)
    # Single-pass products that build the Newton-Schulz factor T = 0.5 (3I - Z Y) leave Y Z^-1 = (Y T)(T Z)^-1 unchanged
    # and only slow the convergence, which the later iterations make up: those links barely move y, and no bound can see
    # them.  The ones that carry A or the upstream gradient into the chain can be seen:
    _rejected('forward mm3 link 0 (Y_0 = A Z_0) single-pass, y', fwd_bwd(single=0)[0], y, fy, sy, C_NS)
    _rejected('backward mm3 link 1 (P (3I - Y Z)) single-pass, dx', fwd_bwd(single=nf + 1)[1], gr, fg, sg, C_NS)
    _rejected('backward tail without the transpose', fwd_bwd(no_transpose=True)[1], gr, fg, sg, C_NS)
    _rejected("diagonal coefficient with the next image's normA", fwd_bwd(neighbour_norm=True)[1], gr, fg, sg, C_NS)
    _rejected('diagonal coefficient without aux', fwd_bwd(no_aux=True)[1], gr, fg, sg, C_NS)
    for b in range(2):
        for what, ref, f, s in (('y', y, fy, sy), ('dx', gr, fg, sg)):
            bad = ref.clone()
            bad[b, :128, 64:128] = ref[b + 1, :128, 64:128]
            _rejected(f'{what}: one 128x64 tile of image {b} from image {b + 1}', bad, ref, f, s, C_NS)


def test_bounds_reject_covpool_defects():
    x, cov, g, _ = _small_head()
    B, C, H, W = x.shape
    M = H * W
    ref, xc64, e_s, fixed, S = covpool_fwd_bounds(x, False)
    bad_cov, bad_xc = covpool_fwd64(x, mean_div=pad4(M))
    xb = e_s + (2 * U + RND) * torch.fmax(bad_xc.float().to(F64).abs(), xc64.abs())
    _rejected('covpool xc: mean divided by the padded M', bad_xc, xc64, xb, 0 * xb, 0.0)
    _rejected('covpool cov: mean divided by the padded M', bad_cov, ref, fixed, S, C_COV)
    xc = detgen.tf32_rna(xc64.float())
    ref, fixed, scale = covpool_bwd_bounds(xc, g, M, False)
    _rejected('covpool dx without the g^T term', covpool_bwd64(xc, g, M, transpose_term=False), ref, fixed, scale, C_COV)
    bad = ref.clone()
    bad[0, :, :32] = ref[1, :, :32]
    _rejected('covpool dx: 32 columns of image 0 from image 1', bad, ref, fixed, scale, C_COV)


def test_bounds_reject_classifier_defects():
    B, F, N = 3, 8 * 1028, 8
    x, w, b, dy, S = classifier_inputs(B, F, N, 30, 'cpu')
    assert S == 8 and F // S == 1028 and linear_splits(F_CLS) == 32
    ref, fixed, scale = linear_refs(x, w, b, dy, S)['y']
    xd, wd = x.to(F64), w.to(F64)
    Kc = F // S
    sl = slice(5 * Kc, 6 * Kc)
    _rejected('classifier without K slice 5', ref - xd[:, sl] @ wd[:, sl].T, ref, fixed, scale, C_LIN)
    tail = torch.cat([torch.arange((s + 1) * Kc - 4, (s + 1) * Kc) for s in range(S)])
    _rejected('classifier without the partial k-block of every slice', ref - xd[:, tail] @ wd[:, tail].T, ref, fixed,
              scale, C_LIN)
