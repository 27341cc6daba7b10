"""The second-order pooling heads against fp64, element by element: hk_bilinear_pool_fwd / _bwd and hk_cbp_fwd / _bwd,
called through the C ABI with workspaces of exactly the queried size, in both precision modes, on padded maps (H*W % 4 != 0)
and at the batch-32 shapes of the benchmarked train steps.

Every call writes into NaN-filled outputs followed by guard words, and gets a NaN-filled workspace of exactly
*_workspace_bytes(...) bytes, also followed by guard words; inputs are followed by NaN, so a read past their end shows.
Each element must satisfy |out - ref| <= bound, with ref computed in fp64 on the CPU (oracle/hop_oracle.py and plain
torch) and the bound derived below from the arithmetic the kernels do.

Error model (u = 2^-24, the fp32 unit roundoff; inputs are post-ReLU, x >= 0, so |X| = X and every Gram entry is >= 0):

* One tensor-core GEMM entry sum_k a_k b_k, relative to sum_k |a_k b_k|:
  - TF32 mode, arbitrary fp32 operands: the MMA truncates each operand to tf32, losing less than 2^-10 of it, so each
    product is off by less than 2^-10 + 2^-10 + 2^-20 of |a_k b_k|.  An operand that is tf32-representable (rounded on
    store by its producer, or by the test) loses nothing.
  - TF32-representable operands: the 11-bit x 11-bit products are exact in fp32; only the accumulation errs.
  - Precise mode (3xTF32): a = hi + lo + e with |e| <= 2^-22 |a|; dropping lo*lo and the two representation errors cost
    at most 3 * 2^-22 |a_k b_k|, the final add of the two accumulators u; together below 2^-20.
  - Accumulation: the MMA adds the products into an fp32 accumulator k-step by k-step, truncating; modelled as at most
    two units of 2^-23 per added term, K * 2^-22 of sum |a_k b_k| over K terms (a factor of 2 to 8 above the truncation
    bias of non-negative sums, and far above their random walk).
* The other fp32 arithmetic is recursive summation (n terms: (n - 1) u of the sum of magnitudes, whatever the order,
  which covers the atomics of the sketch scatter) plus a few correctly rounded operations, counted generously.
* TF32 mode rounds y (both heads) and dx (both backwards) to tf32 on store, to nearest: 2^-11 of |out| more.  Where
  that term dominates, e.g. y close to 1/C = 2^-9 just above a power of two, the worst ratio comes close to 1 by
  construction; it exceeds 1 only if the arithmetic before the store errs beyond its own share of the bound.

Bilinear forward, y = z / ||z||, z = sqrt(G / HW + 1e-5): a Gram error of c_G G_ij moves z_ij by c_G w_ij / 2 with
w_ij = (G_ij / HW) / z_ij^2 <= 1; the closed-form norm comes from the channel sums s_p (truncated in TF32 mode, c_s =
2^-10 + C u) and sum_p s_p^2 (HW terms), so ||z|| is off by c_n wbar / 2, c_n = 2 c_s + (HW + 4) u, wbar the share of
sum G / HW in ||z||^2 (HW padded to 4 throughout).  Hence |y'_ij - y_ij| <= y_ij (c_G w_ij / 2 + dn + 8 u) with dn = c_n wbar / 2 + 3 u.

Bilinear backward, dx = alpha (S . X) + beta 1 s^T with S = (dY + dY^T) / (2 z), alpha = 1 / (n HW),
beta = -<dY, z> / (n^3 HW): S inherits z's error; the second GEMM (K = C) truncates the unrounded S in TF32 mode;
<dY, z> is an fp32 sum of 32 terms per thread and a warp tree.  The bound is k1 alpha (|S| . X) + k2 babs s with
babs = sum |dY| z / (n^3 HW), the absolute-value version of |beta| (the signed sum can cancel, its error cannot).

Compact bilinear forward: bin k of pre takes the signed Gram entries of its n_k pairs through fp32 atomics, so
|pre'_k - pre_k| <= (c_G + n_k u) sum_{(i,j) in k} G_ij.  y is checked against the fp64 signed-sqrt-and-normalise of the
kernel's own pre, which keeps the ill-conditioned square root out of the bound: only the block sums (d / 256 + 13
terms deep) and a few roundings remain.

Compact bilinear backward: pre is computed in fp64 and cast to fp32, and dx is compared with the fp64 gradient at that
same pre.  dpre_k errs by a few dozen u of dabs_k = (|g_k| + |y_k| sum_l r_l |g_l| / n) / (2 n r_k); S is rounded to tf32
in TF32 mode, so the second GEMM truncates only X.

The self-tests at the end (no GPU) compute plausible kernel defects in fp64 at these cases' shapes, round them to fp32,
and check that the loosest of these bounds (TF32 mode, arbitrary fp32 inputs) rejects each of them.
"""
import functools
import math

import numpy as np
import pytest
import torch

import detgen
from kernel_check import RND, TRUNC, U, abi, check, guarded, poisoned, store_bound, workspace, worst_ratio
from oracle import hop_oracle as O

EPS_BP = 1e-5           # BCNN.py:21
EPS_CBP = 1e-10         # CBCNN.py:132
MODES = ('tf32', 'precise')


def pad4(v):
    return (v + 3) & ~3


# ------------------------------------------------------------------------------------------------ cases and inputs
# (B, C, H, W, what it reaches); tf32=True: the batch's values are tf32-representable
BILINEAR = {
    'b32_14x14': (32, 512, 14, 14, False),            # the benchmark shape
    'b32_14x14_tf32in': (32, 512, 14, 14, True),
    'hw49_7x7': (2, 512, 7, 7, False),                # padded to 52
    'hw9_3x3': (3, 256, 3, 3, False),
    'hw1_1x1': (5, 128, 1, 1, False),                 # padded to one partial k-step
    'hw169_13x13': (2, 384, 13, 13, False),           # padded; C is three 128-row tiles
    'hw1024_32x32': (2, 128, 32, 32, False),          # the first one-row-lane channel sum
    'hw1600_40x40': (1, 128, 40, 40, False),          # more float4 columns than threads
    'hw12544_112x112': (2, 128, 112, 112, False),     # channel sums above the default 48 KB of shared memory
}
# (B, C, H, W, d, tf32)
CBP = {
    'b32_14x14_d8192': (32, 512, 14, 14, 8192, False),   # the benchmark shape
    'b32_14x14_d8192_tf32in': (32, 512, 14, 14, 8192, True),
    'hw49_7x7_d6000': (2, 512, 7, 7, 6000, False),       # the reference's 224x224 config; ldc = 49 in the backward
    'hw9_3x3_d127': (3, 512, 3, 3, 127, False),          # about 2000 pairs per bin: heavy atomic contention
    'hw1_1x1_d1000': (5, 128, 1, 1, 1000, False),        # backward: an N = 1 GEMM storing dx with ldc = 1, B read at ldb = 4
    'hw169_13x13_d8192': (2, 384, 13, 13, 8192, False),  # backward: dx stored with the odd ldc = 169 across two N tiles
}


def feature_map(B, C, H, W, tf32, seed):
    """Post-ReLU, sparse, non-negative maps, as the trunk emits.  A batch of 5 or more ends with an all-zero image, an
    image with one non-zero channel (large enough that its Gram entry dominates ||z||), and two images scaled by 1e3 and
    1e-3 next to each other; a batch of 2 to 4 ends with the one-channel image."""
    x = torch.relu(detgen.det_uniform((B, C, H, W), seed) - 0.4)
    one = torch.zeros(C, H, W)
    one[C // 3] = 30.0 * torch.relu(detgen.det_uniform((H, W), seed + 1) - 0.4)
    if B >= 5:
        x[B - 4] = 0.0
        x[B - 3] = one
        x[B - 2] *= 1e3
        x[B - 1] *= 1e-3
    elif B >= 2:
        x[B - 1] = one
    return detgen.tf32_rna(x) if tf32 else x


def bilinear_dy(B, C, seed):
    """A non-symmetric dY with a non-zero mean: a symmetric dY hides a missing transpose, a zero-mean one the rank-1 term."""
    return detgen.det((B, C * C), seed) + 0.5


# ------------------------------------------------------------------------------------------------ fp64 references
def gram_c(K, mode, trunc_a, trunc_b):
    """Relative error of one GEMM entry with respect to sum_k |a_k b_k| (see the module docstring)."""
    if mode == 'precise':
        return 2.0 ** -20 + K * 2.0 ** -22
    ta, tb = (TRUNC if trunc_a else 0.0), (TRUNC if trunc_b else 0.0)
    return ta + tb + ta * tb + K * 2.0 ** -22


def bilinear_parts(x, dy=None, hw=None, dyT='transpose', rank1=True):
    """fp64 restatement of BCNN.py:13-27 and of its gradient in the kernels' closed form.  hw, dyT and rank1 switch in the
    defects of the self-tests: the normalising H*W, how dY^T enters S ('transpose', 'dropped', 'dy' = dY read twice), and
    whether the rank-1 (beta) correction is applied."""
    B, C, H, W = x.shape
    HW = H * W
    hw = hw or HW
    X = x.reshape(B, C, HW)
    G = X @ X.transpose(1, 2)
    z = torch.sqrt(G / hw + EPS_BP)
    n = z.flatten(1).norm(dim=1).clamp_min(1e-12)
    p = {'G': G, 'z': z, 'n': n, 'y': (z / n.view(B, 1, 1)).reshape(B, C * C), 'hw': hw}
    if dy is None:
        return p
    D = dy.reshape(B, C, C)
    Dt = {'transpose': D.transpose(1, 2), 'dropped': torch.zeros_like(D), 'dy': D}[dyT]
    S = (D + Dt) / (2 * z)
    s = X.sum(dim=1)                                                  # [B, HW] channel sums
    alpha = 1.0 / (n * hw)
    beta = -(D * z).sum(dim=(1, 2)) / (n ** 3 * hw)
    dx = alpha.view(B, 1, 1) * (S @ X)
    if rank1:
        dx = dx + beta.view(B, 1, 1) * s.unsqueeze(1)
    p.update(S=S, s=s, alpha=alpha, babs=(D.abs() * z).sum(dim=(1, 2)) / (n ** 3 * hw), dx=dx.reshape(x.shape))
    return p


def bilinear_bounds(x, p, mode, tf32in):
    """Per-element bounds of y [B, C*C], inv_norm [B] and (with dy) dx [B, C, H, W], without the rounding on store."""
    assert (x >= 0).all(), 'the bound assumes post-ReLU inputs'
    B, C, H, W = x.shape
    HW, K = H * W, pad4(H * W)
    trunc_x = mode == 'tf32' and not tf32in
    cG = gram_c(K, mode, trunc_x, trunc_x)
    c_s = (TRUNC if trunc_x else 0.0) + C * U
    c_n = 2 * c_s + (K + 4) * U
    g = p['G'] / HW
    w = g / (g + EPS_BP)
    wbar = g.sum(dim=(1, 2)) / (g.sum(dim=(1, 2)) + C * C * EPS_BP)
    dn = c_n * wbar / 2 + 3 * U
    b = {'y': (p['y'].view(B, C, C) * (cG * w / 2 + dn.view(B, 1, 1) + 8 * U)).reshape(B, C * C),
         'inv_norm': (1.0 / p['n']) * (dn + 4 * U)}
    if 'S' in p:
        cG2 = gram_c(C, mode, mode == 'tf32', trunc_x)                # S is stored unrounded: the MMA truncates it
        dz = cG / 2 + 3 * U
        k1 = dz + 3 * U + cG2 + dn + 8 * U
        k2 = 3 * dn + dz + c_s + 48 * U
        X = x.reshape(B, C, HW)
        b['dx'] = ((k1 * p['alpha']).view(B, 1, 1) * (p['S'].abs() @ X) +
                   (k2 * p['babs']).view(B, 1, 1) * p['s'].unsqueeze(1)).reshape(x.shape)
    return b


def cbp_pre_bound(H, W, mode, tf32in, gabs, npairs):
    trunc_x = mode == 'tf32' and not tf32in
    return (gram_c(pad4(H * W), mode, trunc_x, trunc_x) + npairs * U) * gabs


def cbp_y_bound(y_ref, dn2):
    return y_ref.abs() * (dn2.unsqueeze(1) / 2 + 8 * U)


def cbp_dx_c(C, d, mode, tf32in):
    """Relative error of dx with respect to (Sabs . X): dpre (block sums m + 13 deep, a dozen roundings), S (one add,
    then the tf32 rounding in TF32 mode), and the second GEMM, which in TF32 mode truncates X only."""
    m = math.ceil(d / 256)
    dn = (m + 16) * U / 2 + 2 * U
    e_d = 2 * dn + (m + 16) * U + 10 * U
    cG2 = gram_c(C, mode, False, mode == 'tf32' and not tf32in)
    return e_d + 2 * U + (RND if mode == 'tf32' else 0.0) + cG2


def sketch_index(h1, h2, d):
    return torch.from_numpy((h1[:, None] + h2[None, :]) % d).reshape(-1)


def cbp_pre_parts(x, d, hashes, swap_hashes=False, drop=None):
    """fp64 pre-sqrt sketch (the oracle's Gram scatter) and the per-bin sum of |G_ij| and pair count.  swap_hashes pairs
    h2 with s1 and h1 with s2; drop = (image, i, j) leaves one pair out of its bin."""
    h1, s1, h2, s2 = hashes
    if swap_hashes:
        h1, h2 = h2, h1
    B, C, H, W = x.shape
    pre = O.cbp_presqrt_gram_scatter(x, d, (h1, s1, h2, s2))
    X = x.reshape(B, C, H * W)
    G = X @ X.transpose(1, 2)
    idx = sketch_index(h1, h2, d)
    gabs = torch.zeros(B, d, dtype=x.dtype).index_add_(1, idx, G.abs().reshape(B, -1))
    npairs = torch.bincount(idx, minlength=d).to(x.dtype)
    if drop is not None:
        b, i, j = drop
        pre[b, (h1[i] + h2[j]) % d] -= float(s1[i] * s2[j]) * G[b, i, j]
    return pre, gabs, npairs


def cbp_finalize(pre):
    """fp64 y = normalize(sign(pre) sqrt(|pre| + 1e-10)) (CBCNN.py:132-133) and the relative error of the kernel's
    fp32 block sum of the squared norm."""
    r = torch.where(pre != 0, torch.sqrt(pre.abs() + EPS_CBP), torch.zeros_like(pre))
    sig = torch.sign(pre) * r
    n2 = (r * r).sum(dim=1)
    y = sig / n2.sqrt().clamp_min(1e-12).unsqueeze(1)
    d = pre.shape[1]
    n2abs = (pre.abs() + EPS_CBP).sum(dim=1) + EPS_CBP * (pre == 0).sum(dim=1)
    dn2 = (math.ceil(d / 256) + 16) * U * n2abs / n2.clamp_min(1e-300)
    return y, dn2


def cbp_bwd_parts(x, pre32, g, hashes, d):
    """fp64 dx of CBCNN.py:96-135 at the given fp32 pre, and its absolute-value scale (Sabs . X)."""
    h1, s1, h2, s2 = hashes
    B, C, H, W = x.shape
    pre = pre32.double()
    nz = pre != 0
    r = torch.where(nz, torch.sqrt(pre.abs() + EPS_CBP), torch.ones_like(pre))
    sig = torch.where(nz, torch.sign(pre) * r, torch.zeros_like(pre))
    n = torch.sqrt((sig * sig).sum(dim=1)).clamp_min(1e-12).unsqueeze(1)
    y = sig / n
    c = (y * g).sum(dim=1, keepdim=True)
    dpre = torch.where(nz, (g - y * c) / n / (2 * r), torch.zeros_like(pre))
    cabs = (sig.abs() * g.abs()).sum(dim=1, keepdim=True) / n
    dabs = torch.where(nz, (g.abs() + y.abs() * cabs) / (2 * n * r), torch.zeros_like(pre))
    k1 = sketch_index(h1, h2, d).view(C, C)
    sgn = torch.from_numpy(s1[:, None] * s2[None, :]).double()
    dG = sgn * dpre[:, k1]                                            # [B, C, C]
    dGabs = dabs[:, k1]
    X = x.reshape(B, C, H * W)
    dx = ((dG + dG.transpose(1, 2)) @ X).reshape(x.shape)
    scale = ((dGabs + dGabs.transpose(1, 2)) @ X).reshape(x.shape)
    return dx, scale


@functools.lru_cache(maxsize=None)
def bilinear_case(name):
    B, C, H, W, tf32 = BILINEAR[name]
    x = feature_map(B, C, H, W, tf32, seed=101)
    dy = bilinear_dy(B, C, seed=102)
    D = dy.view(B, C, C)
    assert (D - D.transpose(1, 2)).abs().mean() > 0.5          # far from symmetric
    return x, dy, bilinear_parts(x.double(), dy.double())


@functools.lru_cache(maxsize=None)
def cbp_case(name):
    from hawkeye_b200 import ops
    B, C, H, W, d, tf32 = CBP[name]
    x = feature_map(B, C, H, W, tf32, seed=201)
    hashes = ops.count_sketch_hashes(C, d)
    pre, gabs, npairs = cbp_pre_parts(x.double(), d, hashes)
    g = detgen.det((B, d), 202)
    pre32 = pre.float()
    dx, dx_scale = cbp_bwd_parts(x.double(), pre32, g.double(), hashes, d)
    return x, hashes, pre, gabs, npairs, g, pre32, dx, dx_scale


# ------------------------------------------------------------------------------------------------ GPU tests
@pytest.mark.gpu
@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('case', list(BILINEAR))
def test_bilinear_pool_fwd_bwd(case, mode):
    B, C, H, W, tf32in = BILINEAR[case]
    HW = H * W
    x, dy, p = bilinear_case(case)
    xd, dyd = poisoned(x), poisoned(dy)
    y, invn = guarded((B, C, C)), guarded((B,))
    ws, nb = workspace('hk_bilinear_pool_fwd_workspace_bytes', B, C, HW)
    precise = mode == 'precise'
    abi('hk_bilinear_pool_fwd', xd, y, invn, B, C, HW, ws, nb, inputs=(xd,), precise=precise)
    dx = guarded((B, C, HW))
    wsb, nbb = workspace('hk_bilinear_pool_bwd_workspace_bytes', B, C, HW)
    abi('hk_bilinear_pool_bwd', xd, dyd, dx, B, C, HW, wsb, nbb, inputs=(xd, dyd), precise=precise)
    bd = bilinear_bounds(x.double(), p, mode, tf32in)
    tag = f'bilinear {case} {mode}'
    yk, dxk = y.cpu(), dx.cpu()
    check(yk, p['y'].view(B, C, C), store_bound(yk, bd['y'].view(B, C, C), not precise), f'{tag} y',
          names=('image', 'row', 'col'))
    check(invn, 1.0 / p['n'], bd['inv_norm'], f'{tag} inv_norm', names=('image',))
    check(dxk, p['dx'].view(B, C, HW), store_bound(dxk, bd['dx'].view(B, C, HW), not precise), f'{tag} dx',
          names=('image', 'channel', 'pos'))
    if B >= 5:                               # the all-zero image: y is 1/C (an ulp of the product in precise mode), dx 0
        z = B - 4
        yz = yk[z].double().cpu() * C
        assert (yz == 1).all() if mode == 'tf32' else ((yz - 1).abs() <= 2 * U).all(), yz
        assert (dxk[z] == 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('case', list(CBP))
def test_cbp_fwd(case, mode):
    B, C, H, W, d, tf32in = CBP[case]
    x, hashes, pre_ref, gabs, npairs, *_ = cbp_case(case)
    h1, s1, h2, s2 = [torch.from_numpy(a).cuda() for a in hashes]
    h1, h2, s1, s2 = h1.int(), h2.int(), s1.float(), s2.float()
    xd = poisoned(x)
    y, pre = guarded((B, d)), guarded((B, d))
    abi('hk_cbp_fwd', xd, h1, h2, s1, s2, y, pre, B, C, H * W, d, inputs=(xd,), precise=mode == 'precise')
    tag = f'cbp {case} {mode}'
    check(pre, pre_ref, cbp_pre_bound(H, W, mode, tf32in, gabs, npairs), f'{tag} pre', names=('image', 'bin'))
    y_ref, dn2 = cbp_finalize(pre.double().cpu())
    yk = y.cpu()
    check(yk, y_ref, store_bound(yk, cbp_y_bound(y_ref, dn2), mode == 'tf32'), f'{tag} y', names=('image', 'bin'))
    if B >= 5:                               # the all-zero image
        assert (pre[B - 4] == 0).all() and (y[B - 4] == 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('case', list(CBP))
def test_cbp_bwd(case, mode):
    B, C, H, W, d, tf32in = CBP[case]
    x, hashes, _, _, _, g, pre32, dx_ref, dx_scale = cbp_case(case)
    h1, s1, h2, s2 = [torch.from_numpy(a).cuda() for a in hashes]
    h1, h2, s1, s2 = h1.int(), h2.int(), s1.float(), s2.float()
    xd, pred, gd = poisoned(x), poisoned(pre32), poisoned(g)
    dx = guarded((B, C, H * W))
    ws, nb = workspace('hk_cbp_bwd_workspace_bytes', B, C, d)
    abi('hk_cbp_bwd', xd, pred, gd, h1, h2, s1, s2, dx, B, C, H * W, d, ws, nb, inputs=(xd, pred, gd),
        precise=mode == 'precise')
    dxk = dx.cpu()
    check(dxk, dx_ref.view(B, C, H * W),
          store_bound(dxk, cbp_dx_c(C, d, mode, tf32in) * dx_scale.view(B, C, H * W), mode == 'tf32'),
          f'cbp {case} {mode} dx', names=('image', 'channel', 'pos'))
    if B >= 5:
        assert (dxk[B - 4] == 0).all()


# ------------------------------------------------------------------------------------------------ self-tests of the bound
# Each computes a defect in fp64 at a GPU case's shape and inputs, rounds it to fp32, and checks it against the loosest
# bound of the GPU tests (TF32 mode, arbitrary fp32 inputs), rounding on store included where the kernel rounds.
def rejected(bad, ref, bound, rounded):
    """Worst err/bound ratio of the fp32-rounded defect, and where; > 1 means the GPU check would fail it."""
    out = bad.float().double()
    r, idx = worst_ratio(out, ref, store_bound(out, bound, rounded))
    return r, tuple(idx)


def loosest_bilinear(x, p):
    return bilinear_bounds(x.double(), p, 'tf32', False)


def loosest_cbp(case):
    B, C, H, W, d, _ = CBP[case]
    x, hashes, pre, gabs, npairs, g, pre32, dx_ref, dx_scale = cbp_case(case)
    return {'pre': cbp_pre_bound(H, W, 'tf32', False, gabs, npairs), 'dx': cbp_dx_c(C, d, 'tf32', False) * dx_scale}


def test_restatement_matches_oracle():
    """The defect-free restatement the self-tests perturb is the oracle's forward and gradient."""
    x, dy, p = bilinear_case('hw49_7x7')
    assert torch.allclose(p['y'], O.bilinear_pool_fwd(x.double()), rtol=1e-12, atol=0)
    assert torch.allclose(p['dx'], O.bilinear_pool_bwd(x.double(), dy.double()), rtol=1e-10, atol=1e-18)


@pytest.mark.parametrize('case', ['hw9_3x3_d127', 'hw1_1x1_d1000'])
def test_cbp_gradient_restatement_matches_autograd(case):
    """The closed-form CBP gradient the GPU tests compare with is autograd of the oracle's fp64 forward (Gram scatter,
    signed sqrt, normalise), zero bins (sign(0) = 0) and, in the 1x1 case, the all-zero image included."""
    import torch.nn.functional as F
    B, C, H, W, d, _ = CBP[case]
    x, hashes, _, _, _, g, *_ = cbp_case(case)
    xg = x.double().requires_grad_(True)
    pre = O.cbp_presqrt_gram_scatter(xg, d, hashes)
    y = F.normalize(O.Plain.signed_sqrt(pre))
    (dx_auto,) = torch.autograd.grad(y, xg, g.double())
    dx, _ = cbp_bwd_parts(x.double(), pre.detach(), g.double(), hashes, d)
    assert (pre.detach() == 0).any()
    assert torch.allclose(dx, dx_auto, rtol=1e-9, atol=1e-12 * dx_auto.abs().max().item())


@pytest.mark.parametrize('case', ['hw49_7x7', 'hw9_3x3', 'hw1_1x1', 'hw169_13x13'])
def test_bound_rejects_padded_hw_normalisation(case):
    """Normalising a padded map by the padded H*W instead of the true one, in the forward and in the backward."""
    x, dy, p = bilinear_case(case)
    bd = loosest_bilinear(x, p)
    bad = bilinear_parts(x.double(), dy.double(), hw=pad4(x.shape[2] * x.shape[3]))
    ry, _ = rejected(bad['y'], p['y'], bd['y'], True)
    rdx, _ = rejected(bad['dx'], p['dx'], bd['dx'], True)
    assert ry > 1 and rdx > 1, (ry, rdx)


@pytest.mark.parametrize('defect', ['dropped', 'dy'])
@pytest.mark.parametrize('case', ['b32_14x14', 'hw49_7x7'])
def test_bound_rejects_wrong_transpose_term(case, defect):
    """S = (dY + dY^T) / (2z) with the dY^T term dropped, or with dY read in its place (a missing transpose)."""
    x, dy, p = bilinear_case(case)
    bad = bilinear_parts(x.double(), dy.double(), dyT=defect)
    r, _ = rejected(bad['dx'], p['dx'], loosest_bilinear(x, p)['dx'], True)
    assert r > 1, r


@pytest.mark.parametrize('case', ['b32_14x14', 'hw49_7x7'])
def test_bound_rejects_missing_rank1_correction(case):
    x, dy, p = bilinear_case(case)
    bad = bilinear_parts(x.double(), dy.double(), rank1=False)
    r, _ = rejected(bad['dx'], p['dx'], loosest_bilinear(x, p)['dx'], True)
    assert r > 1, r


def test_bound_rejects_swapped_hashes():
    """h1 paired with s2 and h2 with s1 in the scatter.  Swapping both pairs, (h1, s1) <-> (h2, s2), is an exact symmetry
    of the sketch of a symmetric Gram (pair (i, j) lands where pair (j, i) did, with the same sign, and G_ij = G_ji): it
    changes nothing, so no bound can reject it, and that is asserted too."""
    case = 'b32_14x14_d8192'
    d = CBP[case][4]
    x, hashes, pre, *_ = cbp_case(case)
    h1, s1, h2, s2 = hashes
    assert torch.allclose(O.cbp_presqrt_gram_scatter(x.double(), d, (h2, s2, h1, s1)), pre, rtol=1e-12, atol=1e-9)
    bad, _, _ = cbp_pre_parts(x.double(), d, hashes, swap_hashes=True)
    r, _ = rejected(bad, pre, loosest_cbp(case)['pre'], False)
    assert r > 1, r


@pytest.mark.parametrize('case', ['b32_14x14_d8192', 'hw49_7x7_d6000'])
def test_bound_rejects_missing_pair(case):
    """One (i, j) pair left out of its bin: the largest pair of the bin with the most Gram mass, in the first image."""
    B, C, H, W, d, _ = CBP[case]
    x, hashes, pre, gabs, *_ = cbp_case(case)
    h1, s1, h2, s2 = hashes
    X = x[0].double().reshape(C, H * W)
    G = X @ X.T
    k = int(torch.argmax(gabs[0]))
    in_bin = (sketch_index(h1, h2, d) == k).view(C, C)
    i, j = np.unravel_index(int(torch.argmax(torch.where(in_bin, G, torch.zeros_like(G)))), (C, C))
    bad, _, _ = cbp_pre_parts(x.double(), d, hashes, drop=(0, int(i), int(j)))
    r, idx = rejected(bad, pre, loosest_cbp(case)['pre'], False)
    assert r > 1 and idx == (0, k), (r, idx)


@pytest.mark.parametrize('output', ['bilinear_y', 'bilinear_dx', 'cbp_pre', 'cbp_y', 'cbp_dx'])
def test_bound_rejects_output_in_neighbours_slot(output):
    """Image 0's output also written into image 1's slot (a batch-index slip), at the benchmark shapes."""
    if output.startswith('bilinear'):
        x, dy, p = bilinear_case('b32_14x14')
        key = output.split('_')[1]
        ref, bound = p[key], loosest_bilinear(x, p)[key]
    else:
        case = 'b32_14x14_d8192'
        x, hashes, pre, gabs, npairs, g, pre32, dx_ref, dx_scale = cbp_case(case)
        if output == 'cbp_y':
            ref, dn2 = cbp_finalize(pre)
            bound = cbp_y_bound(ref, dn2)
        else:
            ref, bound = (pre, loosest_cbp(case)['pre']) if output == 'cbp_pre' else (dx_ref, loosest_cbp(case)['dx'])
    bad = ref.clone()
    bad[1] = ref[0]
    r, idx = rejected(bad, ref, bound, output != 'cbp_pre')
    assert r > 1 and idx[0] == 1, (r, idx)
