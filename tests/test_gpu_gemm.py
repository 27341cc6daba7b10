"""wgmma GEMM (gemm.cu) against an fp64 CPU product of the same operands.  GPU only.

The conformance tests check every element against the standard GEMM error bound

    |C_ij - ref_ij| <= tol * mag_ij,   mag = |alpha_b| (|A|.|B|) + |diag| I + |beta_b| |D|   (fp64)

so an output that nearly cancels still counts, and one misplaced, missing or stale element fails.  Operands are stored
with a leading dimension past their logical extent and NaN in the padding, and C sits inside a guard buffer: a read
outside an operand poisons C, and every word the GEMM must not write is compared bit for bit afterwards.
"""
import pytest
import torch

import detgen

pytestmark = pytest.mark.gpu

TOL = 2e-3   # TF32 operands (10-bit mantissa), fp32 accumulate
U = 2.0 ** -23
MAJORS = [(0, 0), (1, 0), (0, 1), (1, 1)]
MODES = {'1x': (0, False), 'precise': (1, False), '3x': (0, True)}   # (hk_set_precise, hk_gemm_3xtf32)
PATTERN = 0x7FA5A5A5          # a NaN payload: guard words, and any output element the GEMM fails to write
EPI_ROUND = 2.0 ** -22        # alpha / diag / beta * D applied in fp32


# Measured on an H100 80GB HBM3 (700 W), worst err / mag over every case: 0.26 K U with tf32-representable operands
# (1.2e-7 at K = 4), 1.34e-3 single pass over fp32 operands (K = 8: the MMA truncates, it does not round), 8.2e-7 in
# 3xTF32 (K = 100).  The bounds below are the analytic ones; the measured worst sits 1.5x (single pass over fp32
# operands) to 6x below them.
def tol_exact(K):
    """one pass over tf32-representable operands: every product is exact, only the fp32 accumulation errs"""
    return K * U


def tol_1x(K):
    """one pass over arbitrary fp32 operands: the MMA also drops each operand's low 13 bits (< 2^-10 relative)"""
    return 2.0 ** -9 + 2 * K * U


def tol_3x(K):
    """3xTF32: the dropped Al.Bl product and the rounding of the lo halves (3 * 2^-22), plus two fp32 accumulators"""
    return 2.0 ** -20 + K * U


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


@pytest.mark.parametrize('a_mn,b_mn', MAJORS)
@pytest.mark.parametrize('M,N,K,batch', [(128, 128, 64, 1), (200, 300, 100, 2), (32, 200, 1024, 3), (256, 64, 40, 2)])
def test_gemm_majors(a_mn, b_mn, M, N, K, batch):
    from hawkeye_b200 import ops
    torch.manual_seed(M + N + K)
    A = torch.randn(batch, M, K, device='cuda')
    B = torch.randn(batch, K, N, device='cuda')
    ref = torch.bmm(A.double(), B.double())
    Ain = A.transpose(1, 2).contiguous() if a_mn else A            # [b,K,M] if MN-major
    Bin = B if b_mn else B.transpose(1, 2).contiguous()            # [b,K,N] if MN-major else [b,N,K]
    out = ops.gemm_tf32(Ain, Bin, a_mn=bool(a_mn), b_mn=bool(b_mn))
    torch.cuda.synchronize()
    err = _rel(out, ref)
    print(f'gemm a_mn={a_mn} b_mn={b_mn} {M}x{N}x{K} b{batch}: rel={err:.3e}')
    assert err < TOL


def test_gemm_epilogue():
    from hawkeye_b200 import ops
    torch.manual_seed(1)
    b, n = 3, 256
    A = torch.randn(b, n, n, device='cuda') / 16
    B = torch.randn(b, n, n, device='cuda') / 16
    D = torch.randn(b, n, n, device='cuda')
    av = torch.rand(b, device='cuda') + 0.5
    I = torch.eye(n, device='cuda', dtype=torch.float64)
    ref = -0.5 * av.double().view(b, 1, 1) * torch.bmm(A.double(), B.double()) + 1.5 * I + 0.25 * D.double()
    out = ops.gemm_tf32(A, B, b_mn=True, alpha=-0.5, alpha_vec=av, diag=1.5, D=D, beta=0.25)
    assert _rel(out, ref) < TOL
    out_t = ops.gemm_tf32(A, B, b_mn=True, alpha=-0.5, alpha_vec=av, diag=1.5, D=D, beta=0.25, trans_c=True)
    assert _rel(out_t, ref.transpose(1, 2)) < TOL
    # shared (2-D) B operand and row-broadcast D (ldd = 0)
    drow = torch.randn(b, 1, n, device='cuda')
    out = ops.gemm_tf32(A, B[0], b_mn=True, D=drow, beta=2.0)
    ref = torch.matmul(A.double(), B[0].double()) + 2.0 * drow.double()
    assert _rel(out, ref) < TOL


# ---------------------------------------------------------------------------------------------------- conformance
def _ld(cols):
    """a leading dimension in whole 16-byte units with at least one padding column"""
    return (cols + 4) // 4 * 4


def _store(X, ld):
    """[b, rows, cols] -> device buffer [b, rows, ld], NaN in columns cols..ld-1"""
    b, r, c = X.shape
    buf = torch.full((b, r, ld), float('nan'))
    buf[..., :c] = X
    return buf.cuda()


def _operands(M, N, K, batch, seed, exact, share=None):
    """logical A [bA, M, K] and B [bB, K, N] (a batch of 1 is shared by every product when batch > 1)"""
    A = detgen.det((1 if share == 'A' else batch, M, K), seed)
    B = detgen.det((1 if share == 'B' else batch, K, N), seed + 1)
    return (detgen.tf32_rna(A), detgen.tf32_rna(B)) if exact else (A, B)


def gemm(A, B, a_mn=0, b_mn=0, mode='1x', alpha=1.0, alpha_vec=None, diag=0.0, D=None, beta=0.0, beta_vec=None,
         relu=0, trans_c=False, ldc=None, c_off=0):
    """C = A.B through ops.gemm with the operands in the given majors; returns C as logical [batch, M, N] after checking
    that nothing outside the logical output (columns past N, the gap between batch entries, the words before and after)
    was written.  D is [bD, M, N] or a row [bD, 1, N] (ldd = 0); a batch of 1 is shared (stride 0)."""
    from hawkeye_b200 import _lib, ops
    bA, M, K = A.shape
    bB, _, N = B.shape
    batch = max(bA, bB)
    Xa = A.transpose(1, 2) if a_mn else A                 # as stored: [M][K] K-major, or [K][M] MN-major
    Xb = B if b_mn else B.transpose(1, 2)                 # [K][N] MN-major, or [N][K] K-major
    lda, ldb = _ld(Xa.shape[2]), _ld(Xb.shape[2])
    dA, dB = _store(Xa, lda), _store(Xb, ldb)
    sA = Xa.shape[1] * lda if bA > 1 else 0
    sB = Xb.shape[1] * ldb if bB > 1 else 0
    dD, ldd, sD = None, 0, 0
    if D is not None:
        ld = _ld(N)
        dD = _store(D, ld)
        ldd = 0 if D.shape[1] == 1 else ld
        sD = D.shape[1] * ld if D.shape[0] > 1 else 0
    rows, cols = (N, M) if trans_c else (M, N)
    ldc = ldc or _ld(cols)
    sC = rows * ldc + 4
    G = 64 + c_off
    total = 2 * G + batch * sC
    buf = torch.full((total,), PATTERN, dtype=torch.int32).view(torch.float32).cuda()
    av = alpha_vec.cuda() if alpha_vec is not None else None
    bv = beta_vec.cuda() if beta_vec is not None else None
    precise, exact = MODES[mode]
    _lib.set_precise(precise)
    try:
        ops.gemm(dA, a_mn, lda, sA, dB, b_mn, ldb, sB, buf[G:], ldc, sC, M, N, K, batch, alpha, av, diag, dD, ldd, sD,
                 beta, bv, relu, trans_c, exact)
        torch.cuda.synchronize()
    finally:
        _lib.set_precise(0)
    host = buf.cpu()
    idx = (G + torch.arange(batch).view(-1, 1, 1) * sC + torch.arange(rows).view(1, -1, 1) * ldc
           + torch.arange(cols).view(1, 1, -1))
    outside = torch.ones(total, dtype=torch.bool)
    outside[idx.reshape(-1)] = False
    clobbered = int((host.view(torch.int32)[outside] != PATTERN).sum())
    assert clobbered == 0, f'{clobbered} words outside the logical output were written'
    out = host[idx]
    return out.transpose(1, 2) if trans_c else out


def check(label, out, A, B, tol, alpha=1.0, alpha_vec=None, diag=0.0, D=None, beta=0.0, beta_vec=None, relu=0,
          rounded=False, **_):
    """element-wise bound against the fp64 product; returns the worst err / mag"""
    A64, B64 = A.double(), B.double()
    ref, mag = A64 @ B64, A64.abs() @ B64.abs()
    batch, M, N = ref.shape
    a = torch.full((batch, 1, 1), float(alpha), dtype=torch.float64)
    if alpha_vec is not None:
        a = a * alpha_vec.double().view(-1, 1, 1)
    ref, mag = a * ref, a.abs() * mag
    if diag:
        I = torch.eye(M, N, dtype=torch.float64)
        ref, mag = ref + diag * I, mag + abs(diag) * I
    if D is not None:
        b = torch.full((batch, 1, 1), float(beta), dtype=torch.float64)
        if beta_vec is not None:
            b = b * beta_vec.double().view(-1, 1, 1)
        ref, mag = ref + b * D.double(), mag + b.abs() * D.double().abs()
    if relu & 1:
        ref = ref.clamp_min(0)
    err = (out.double() - ref).abs()
    worst = (err / mag.clamp_min(1e-30)).max().item()
    tol = tol + EPI_ROUND + (2.0 ** -11 if rounded else 0.0)
    bound = tol * mag + 1e-30
    print(f'{label}: worst err/mag {worst:.3e} (bound {tol:.3e})')
    assert not torch.isnan(out).any(), f'{label}: NaN in C (an unwritten element or a read past an operand)'
    bad = ~(err <= bound)
    if bad.any():
        i = [int(t) for t in bad.nonzero()[0]]
        raise AssertionError(f'{label}: {int(bad.sum())} elements out of bound; first [b, m, n] = {i}: '
                             f'{out[tuple(i)].item()} vs {ref[tuple(i)].item()}')
    return worst


@pytest.mark.parametrize('M', [1, 127, 128, 129])
@pytest.mark.parametrize('a_mn,b_mn', MAJORS)
def test_gemm_shapes_and_tiles(a_mn, b_mn, M):
    """Every N around the 32-column chunk and the 64 / 128 tile widths, K from one partial k-step to four k-blocks,
    single pass over tf32-representable operands (exact products): a dropped k-step or a misplaced element is orders of
    magnitude above the bound."""
    worst = 0.0
    for N in (1, 4, 31, 32, 64, 65, 127, 128, 129):
        for K in (4, 8, 32, 33, 36, 100):
            A, B = _operands(M, N, K, 2, M + N + K, exact=True)
            out = gemm(A, B, a_mn, b_mn)
            worst = max(worst, check(f'{M}x{N}x{K} a_mn={a_mn} b_mn={b_mn}', out, A, B, tol_exact(K)))
    print(f'M={M} a_mn={a_mn} b_mn={b_mn}: worst err/mag over all N, K {worst:.3e}')


@pytest.mark.parametrize('a_mn,b_mn', MAJORS)
@pytest.mark.parametrize('M,N,K,batch', [
    (2048, 1024, 32, 3),    # 384 tiles of 128 x 128 on 132 SMs, one k-block each: 3-stage ring across tiles
    (2048, 1024, 64, 3),    # nk = 2
    (2048, 1024, 96, 3),    # nk = 3
    (2048, 1024, 160, 3),   # nk = 5: the ring wraps inside a tile
    (2048, 64, 130, 12),    # 192 tiles of 128 x 64, partial last k-block
    (896, 64, 96, 19),      # exactly 133 tiles of 128 x 64: one CTA runs two
    (896, 2400, 65, 1),     # exactly 133 tiles of 128 x 128, partial last n-tile
])
def test_gemm_persistent_tiles(a_mn, b_mn, M, N, K, batch):
    A, B = _operands(M, N, K, batch, 7 + K, exact=True)
    out = gemm(A, B, a_mn, b_mn)
    check(f'{M}x{N}x{K} b{batch} a_mn={a_mn} b_mn={b_mn}', out, A, B, tol_exact(K))


@pytest.mark.parametrize('a_mn,b_mn', MAJORS)
@pytest.mark.parametrize('M,N,K,batch', [(129, 100, 100, 2), (200, 65, 33, 3), (256, 300, 1024, 1), (127, 31, 8, 2)])
def test_gemm_single_pass_fp32_operands(a_mn, b_mn, M, N, K, batch):
    A, B = _operands(M, N, K, batch, 11 + K, exact=False)
    out = gemm(A, B, a_mn, b_mn)
    check(f'1x fp32 {M}x{N}x{K} b{batch} a_mn={a_mn} b_mn={b_mn}', out, A, B, tol_1x(K))


@pytest.mark.parametrize('mode', ['precise', '3x'])
@pytest.mark.parametrize('a_mn,b_mn', MAJORS)
@pytest.mark.parametrize('M,N,K,batch', [(1, 1, 4, 1), (127, 31, 8, 2), (200, 65, 33, 3), (129, 100, 100, 2),
                                         (2048, 256, 96, 3), (896, 64, 160, 19)])
def test_gemm_3xtf32(mode, a_mn, b_mn, M, N, K, batch):
    """3xTF32 through hk_gemm_3xtf32 and through hk_gemm_tf32 in precise mode, arbitrary fp32 operands: fp32-class
    error in all four majors (both MN-major: the double staging buffer), partial tiles, more tiles than SMs."""
    A, B = _operands(M, N, K, batch, 13 + K, exact=False)
    out = gemm(A, B, a_mn, b_mn, mode=mode)
    check(f'{mode} {M}x{N}x{K} b{batch} a_mn={a_mn} b_mn={b_mn}', out, A, B, tol_3x(K))


# name: (M, N, K, batch, a_mn, b_mn, options); 'fast*' store every chunk on the fast path, 'general*' every chunk on
# the general one, 'n_partial' and 'vecs_general' mix both (whole 32-column chunks fast, the partial last one general).
#  D = 'full' [b, M, N], 'row' [b, 1, N] (ldd = 0), 'shared' [1, M, N]
EPILOGUES = {
    'fast': (200, 256, 64, 3, 0, 0, {}),
    'fast_D_relu': (200, 256, 64, 3, 0, 1, dict(alpha=-0.5, D='full', beta=0.75, relu=1)),
    'fast_round': (200, 256, 64, 3, 1, 0, dict(relu=2)),
    'fast_D_relu_round': (200, 256, 64, 3, 1, 1, dict(D='full', beta=-0.75, relu=3)),
    'general_ldc_odd': (200, 256, 64, 3, 0, 0, dict(ldc=257, alpha=-0.5, D='full', beta=0.75, relu=1)),
    'general_c_unaligned': (200, 256, 64, 3, 1, 1, dict(c_off=1, relu=3)),
    'n_partial': (200, 100, 64, 3, 0, 1, dict(D='full', beta=-1.25, relu=1)),
    'general_diag': (200, 200, 72, 2, 1, 0, dict(alpha=-0.5, diag=1.5)),
    'general_trans_c': (200, 100, 40, 2, 0, 1, dict(trans_c=True, D='full', beta=0.5, diag=2.0, relu=1)),
    'general_trans_c_round': (129, 65, 36, 2, 1, 1, dict(trans_c=True, diag=-1.0, relu=2)),
    'general_row_D': (129, 100, 36, 3, 0, 0, dict(D='row', beta=2.0)),
    'general_row_D_full_n': (129, 128, 36, 3, 1, 0, dict(D='row', beta=2.0, relu=1)),
    'vecs_shared_D': (150, 192, 48, 3, 1, 1, dict(alpha_vec=True, beta_vec=True, D='shared', beta=0.5)),
    'vecs_general': (150, 100, 48, 3, 0, 1, dict(alpha=2.0, alpha_vec=True, beta_vec=True, D='full', beta=-0.5)),
    'shared_A': (200, 128, 64, 3, 0, 0, dict(share='A', D='full', beta=1.0)),
    'shared_B': (200, 128, 64, 3, 1, 1, dict(share='B', alpha_vec=True)),
}


@pytest.mark.parametrize('mode', list(MODES))
@pytest.mark.parametrize('name', list(EPILOGUES))
def test_gemm_epilogue_paths(name, mode):
    """The fast epilogue (plain store of whole aligned 32-column chunks) and the general one (diag, trans_c, ldc % 4,
    unaligned C, partial chunks, row-broadcast D) on the same kind of product, each against fp64, with alpha_vec,
    beta_vec, shared operands and D, and ReLU (bit 0) / tf32 rounding on store (bit 1, which 3xTF32 ignores)."""
    M, N, K, batch, a_mn, b_mn, opt = EPILOGUES[name]
    opt = dict(opt)
    exact = mode == '1x'
    A, B = _operands(M, N, K, batch, 17 + M + N, exact, share=opt.pop('share', None))
    if opt.pop('alpha_vec', False):
        opt['alpha_vec'] = detgen.det_uniform((batch,), 18) + 0.5
    if opt.pop('beta_vec', False):
        opt['beta_vec'] = detgen.det_uniform((batch,), 19) * 2 - 1.5
    kind = opt.pop('D', None)
    if kind:
        opt['D'] = detgen.det(({'full': batch, 'row': batch, 'shared': 1}[kind], 1 if kind == 'row' else M, N), 20, 4.0)
    out = gemm(A, B, a_mn, b_mn, mode=mode, **opt)
    rounded = bool(opt.get('relu', 0) & 2) and mode == '1x'
    tol = tol_exact(K) if exact else tol_3x(K)
    check(f'{name} {mode}', out, A, B, tol, rounded=rounded, **opt)
    if rounded:
        assert torch.equal(out, detgen.tf32_rna(out)), 'relu bit 1: the stored values must be tf32'
    elif opt.get('relu', 0) & 2:   # 3xTF32 clears the rounding bit: its output carries fp32 precision
        nz = out[out != 0]
        assert (nz != detgen.tf32_rna(nz)).float().mean() > 0.9


@pytest.mark.parametrize('mode', ['precise', '3x'])
@pytest.mark.parametrize('mn', [0, 1])
def test_gemm_3xtf32_aliased_gram(mode, mn):
    """A Gram product with A and B the same pointer and layout splits the operand once (2 launches instead of 3) and
    gives the bits of the same call with B passed as a separate copy."""
    from hawkeye_b200 import _lib, ops
    M, K, batch = 200, 100, 3
    S = detgen.det((batch, K, M) if mn else (batch, M, K), 23)
    ld = _ld(S.shape[2])
    dS = _store(S, ld)
    stride = S.shape[1] * ld
    precise, exact = MODES[mode]
    outs, launches = [], []
    _lib.set_precise(precise)
    try:
        for B in (dS, dS.clone()):
            C = torch.empty(batch, M, M, device='cuda')
            _lib.reset_launch_count()
            ops.gemm(dS, mn, ld, stride, B, mn, ld, stride, C, M, M * M, M, M, K, batch, exact=exact)
            torch.cuda.synchronize()
            launches.append(_lib.launch_count())
            outs.append(C.cpu())
    finally:
        _lib.set_precise(0)
    assert launches == [2, 3]
    assert torch.equal(outs[0], outs[1])
    A = S.transpose(1, 2) if mn else S
    check(f'aliased Gram {mode} mn={mn}', outs[0], A, A.transpose(1, 2), tol_3x(K))


@pytest.mark.parametrize('mode', list(MODES))
def test_gemm_deterministic(mode):
    """The plain epilogue has no atomics: two identical calls give identical bits, also across persistent tiles."""
    A, B = _operands(2048, 1024, 160, 3, 29, exact=False)
    D = detgen.det((3, 2048, 1024), 30)
    a = gemm(A, B, 1, 0, mode=mode, D=D, beta=0.5, relu=1)
    b = gemm(A, B, 1, 0, mode=mode, D=D, beta=0.5, relu=1)
    assert torch.equal(a, b)
