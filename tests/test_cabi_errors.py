"""Error convention of the C ABI (include/hawkeye_b200.h), exercised WITHOUT a GPU: argument / shape / alignment /
workspace errors are detected before anything is launched (return < 0, hk_last_error() explains), never a slow path."""
import ctypes

import pytest


@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as g
    g.build()
    from hawkeye_b200 import _lib
    return _lib.lib()


FAKE = 0x10000      # a non-null, 16-byte aligned address that must never be dereferenced on these paths


def err(lib):
    return lib.hk_last_error().decode()


def test_workspace_queries_are_pure(lib):
    a = lib.hk_bilinear_pool_fwd_workspace_bytes(32, 512, 196)
    assert a >= 32 * 4 and a == lib.hk_bilinear_pool_fwd_workspace_bytes(32, 512, 196)
    assert lib.hk_bilinear_pool_bwd_workspace_bytes(32, 512, 196) >= 32 * 512 * 512 * 4
    assert lib.hk_cbp_bwd_workspace_bytes(2, 512, 8192) == (2 * 512 * 512 + 2 * 8192) * 4
    assert lib.hk_conv3x3_wgrad_workspace_bytes(64, 64) >= 9 * 64 * 64 * 4


def test_bilinear_pool_argument_errors(lib):
    f = lib.hk_bilinear_pool_fwd
    assert f(None, FAKE, None, 2, 512, 196, FAKE, 1 << 30, None) == -1 and 'null' in err(lib)
    assert f(FAKE, FAKE, None, 2, 100, 196, FAKE, 1 << 30, None) == -3 and 'multiple of 128' in err(lib)
    # H*W % 4 != 0 is supported (zero-padded copy in the workspace): the workspace query grows accordingly
    q = lib.hk_bilinear_pool_fwd_workspace_bytes
    q.restype = ctypes.c_size_t
    assert q(2, 512, 49) > q(2, 512, 52) and f(FAKE, FAKE, None, 2, 512, 49, FAKE, q(2, 512, 52), None) == -4
    assert f(FAKE + 4, FAKE, None, 2, 512, 196, FAKE, 1 << 30, None) == -2 and 'aligned' in err(lib)
    assert f(FAKE, FAKE, None, 2, 512, 196, FAKE, 16, None) == -4 and 'workspace' in err(lib)
    assert f(FAKE, FAKE, None, 0, 512, 196, FAKE, 1 << 30, None) == -1
    b = lib.hk_bilinear_pool_bwd
    assert b(FAKE, None, FAKE, 2, 512, 196, FAKE, 1 << 40, None) == -2
    assert b(FAKE, FAKE, FAKE, 2, 512, 196, FAKE, 16, None) == -4


def test_pooling_head_errors_launch_nothing(lib):
    """hk_bilinear_pool_fwd/bwd reject a map whose channel sums exceed shared memory (H*W > 58112, and not 58112 itself),
    and hk_cbp_fwd/bwd reject C % 128, a null pointer, d <= 0 and a short workspace, before anything is launched, in both
    precision modes."""
    f, b = lib.hk_bilinear_pool_fwd, lib.hk_bilinear_pool_bwd
    cf, cb = lib.hk_cbp_fwd, lib.hk_cbp_bwd
    cbq = lib.hk_cbp_bwd_workspace_bytes

    def cbp_bwd(x=FAKE, dx=FAKE, C=512, HW=196, d=8192, ws=1 << 30):
        return cb(x, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, dx, 2, C, HW, d, FAKE, ws, None)

    for precise in (0, 1):
        lib.hk_set_precise(precise)
        lib.hk_reset_launch_count()
        try:
            for hw in (58113, 241 * 242):
                assert f(FAKE, FAKE, None, 2, 128, hw, FAKE, 1 << 40, None) == -3 and '58112' in err(lib)
                assert b(FAKE, FAKE, FAKE, 2, 128, hw, FAKE, 1 << 40, None) == -3 and '58112' in err(lib)
            for hw in (58112, 58110):        # the largest maps still pass the shape checks (a 16-byte workspace does not)
                assert f(FAKE, FAKE, None, 2, 128, hw, FAKE, 16, None) == -4 and 'workspace' in err(lib)
                assert b(FAKE, FAKE, FAKE, 2, 128, hw, FAKE, 16, None) == -4 and 'workspace' in err(lib)
            assert cf(FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, 2, 100, 196, 8192, None) == -3 and 'multiple of 128' in err(lib)
            assert cf(FAKE, FAKE, FAKE, FAKE, FAKE, None, FAKE, 2, 512, 196, 8192, None) == -1 and 'null' in err(lib)
            assert cf(None, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, 2, 512, 196, 8192, None) == -1 and 'null' in err(lib)
            assert cf(FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, 2, 512, 196, 0, None) == -1 and 'bad d' in err(lib)
            assert cbp_bwd(C=100) == -3 and 'multiple of 128' in err(lib)
            assert cbp_bwd(dx=None) == -1 and 'null' in err(lib)
            assert cbp_bwd(x=None) == -1 and 'null' in err(lib)
            for d in (0, -8192):
                assert cbp_bwd(d=d) == -1 and 'bad d' in err(lib)
            assert cbp_bwd(ws=cbq(2, 512, 8192) - 4) == -4 and 'workspace' in err(lib)
            assert cbp_bwd(HW=49, ws=cbq(2, 512, 8192) - 4) == -4 and 'workspace' in err(lib)
            assert lib.hk_launch_count() == 0
        finally:
            lib.hk_set_precise(0)


def test_conv_argument_errors(lib):
    assert lib.hk_conv3x3_fwd(None, FAKE, None, FAKE, 2, 8, 8, 64, 64, 1, None) == -1
    assert lib.hk_conv3x3_fwd(FAKE, FAKE, None, FAKE, 2, 8, 8, 48, 64, 1, None) == -3 and 'multiples of 32' in err(lib)
    assert lib.hk_conv3x3_fwd(FAKE + 8, FAKE, None, FAKE, 2, 8, 8, 64, 64, 1, None) == -2
    assert lib.hk_conv3x3_wgrad(FAKE, FAKE, FAKE, None, 2, 8, 8, 64, 64, FAKE, 16, None) == -4
    assert lib.hk_maxpool2x2_fwd(FAKE, FAKE, 2, 7, 8, 64, 0, None) == -3
    assert lib.hk_conv3x3_first_fwd(FAKE, FAKE, None, FAKE, 2, 8, 8, 300, FAKE, 1 << 30, None) == -3


def test_head_and_mpncov_argument_errors(lib):
    assert lib.hk_linear_fwd(None, FAKE, None, FAKE, 2, 64, 8, FAKE, 1 << 30, None) == -1
    assert lib.hk_linear_fwd(FAKE, FAKE, None, FAKE, 2, 63, 8, FAKE, 1 << 30, None) == -3
    assert lib.hk_softmax_ce_ls(None, FAKE, FAKE, None, None, 2, 200, ctypes.c_float(0.1), ctypes.c_float(1.0), None) == -1
    assert lib.hk_sgd_momentum(FAKE, FAKE + 4, FAKE, 64, ctypes.c_float(0.1), ctypes.c_float(0.9), ctypes.c_float(0.0),
                               ctypes.c_float(1.0), 1, None) == -2
    assert lib.hk_covpool_fwd(None, FAKE, FAKE, 2, 256, 195, None) == -1
    assert lib.hk_sqrtm_fwd(FAKE, FAKE, FAKE, 2, 256, 1, FAKE, 1 << 40, None) == -3 and 'iterN' in err(lib)


@pytest.mark.parametrize('precise', [0, 1], ids=['tf32', 'precise'])
def test_sqrtm_dim_not_multiple_of_4_launches_nothing(lib, precise):
    """hk_sqrtm_fwd and hk_sqrtm_bwd reject n % 4 != 0 (the (hi, lo) rows are TMA operands at a 16-byte pitch) at the
    entry point, before the backward's first element-wise kernel, in both precision modes."""
    lib.hk_set_precise(precise)
    lib.hk_reset_launch_count()
    try:
        for n in (6, 255, 258):
            assert lib.hk_sqrtm_fwd(FAKE, FAKE, FAKE, 2, n, 5, FAKE, 1 << 40, None) == -3 and 'multiple of 4' in err(lib)
            assert lib.hk_sqrtm_bwd(FAKE, FAKE, FAKE, FAKE, FAKE, 2, n, 5, FAKE, 1 << 40, None) == -3
            assert f'dim={n}' in err(lib) and 'multiple of 4' in err(lib)
        assert lib.hk_launch_count() == 0
    finally:
        lib.hk_set_precise(0)


@pytest.mark.parametrize('precise', [0, 1], ids=['tf32', 'precise'])
@pytest.mark.parametrize('entry', ['hk_gemm_tf32', 'hk_gemm_3xtf32'])
def test_gemm_operand_errors_before_any_allocation_or_launch(lib, entry, precise):
    """The GEMM's TMA preconditions (16-byte aligned operand base, row pitch and batch stride in 16-byte units,
    batch <= 65535) are checked before the 3xTF32 path allocates its operand halves or anything is launched, so an
    unaligned operand is rejected in both precision modes."""
    f = getattr(lib, entry)

    def call(A=FAKE, lda=64, strideA=64 * 64, B=FAKE, ldb=64, batch=2):
        return f(A, 0, lda, strideA, B, 0, ldb, 64 * 64, FAKE, 64, 64 * 64, 0, 64, 64, 64, batch, 1.0, None, 0.0, None,
                 0, 0, 0.0, None, 0, None)

    lib.hk_set_precise(precise)
    lib.hk_reset_launch_count()
    try:
        assert call(lda=5) == -2 and 'lda=5' in err(lib) and '16-byte' in err(lib)
        assert call(ldb=66) == -2 and 'ldb=66' in err(lib)
        assert call(A=FAKE + 4) == -2 and 'not 16-byte aligned' in err(lib)
        assert call(B=FAKE + 8) == -2 and 'not 16-byte aligned' in err(lib)
        assert call(strideA=64 * 64 + 2) == -2 and 'batch stride of a' in err(lib)
        assert call(batch=65536) == -3 and '65535' in err(lib)
        assert call(batch=0) == -1 and 'bad shape' in err(lib)
        assert call(A=None) == -1 and 'null' in err(lib)
        assert lib.hk_launch_count() == 0
    finally:
        lib.hk_set_precise(0)


def test_errors_are_thread_local_text(lib):
    lib.hk_bilinear_pool_fwd(FAKE, FAKE, None, 2, 100, 196, FAKE, 1 << 30, None)
    msg = err(lib)
    import threading
    seen = []
    t = threading.Thread(target=lambda: seen.append(lib.hk_last_error().decode()))
    t.start(); t.join()
    assert 'multiple of 128' in msg and seen == ['']


def test_round2_entry_points_argument_errors(lib):
    """hk_conv3x3_fwd_pool, hk_bn_bwd_ex, hk_l2norm_rows_*, hk_npair_loss: bad arguments are rejected before any launch."""
    p = lib.hk_conv3x3_fwd_pool
    assert p(FAKE, FAKE, None, None, None, 2, 8, 8, 64, 64, 0, None) == -1 and 'null output' in err(lib)
    assert p(FAKE, FAKE, None, FAKE, None, 2, 7, 8, 64, 64, 0, None) == -3 and 'even H/W' in err(lib)
    assert p(FAKE, FAKE, None, FAKE, FAKE + 8, 2, 8, 8, 64, 64, 0, None) == -3            # unaligned code buffer
    assert p(FAKE, FAKE, None, FAKE, None, 2, 8, 8, 48, 64, 0, None) == -3 and 'multiples of 32' in err(lib)
    lib.hk_set_precise(1)
    try:
        assert p(FAKE, FAKE, None, FAKE, None, 2, 8, 8, 64, 64, 0, None) == -3 and '3xTF32' in err(lib)
    finally:
        lib.hk_set_precise(0)
    b = lib.hk_bn_bwd_ex
    assert b(FAKE, None, FAKE, FAKE, None, FAKE, FAKE, FAKE, None, FAKE, FAKE, 64, 64, 1, FAKE, 1 << 30, None) == -1  # relu needs y or beta
    assert b(FAKE, None, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, None, FAKE, FAKE, 64, 62, 1, FAKE, 1 << 30, None) == -3
    assert b(FAKE, None, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, None, FAKE, FAKE, 64, 64, 1, FAKE, 16, None) == -4
    assert lib.hk_l2norm_rows_fwd(None, FAKE, FAKE, 4, 64, None) == -1
    assert lib.hk_l2norm_rows_bwd(FAKE, FAKE, None, FAKE, 4, 64, None) == -1
    assert lib.hk_npair_loss(FAKE, FAKE, FAKE, None, FAKE, 8, None) == -1
    assert lib.hk_npair_loss(FAKE, FAKE, FAKE, FAKE, FAKE, 0, None) == -1


# Calls every `int hk_*` entry point that takes a pointer with all pointers null and small positive scalars, and prints
# each one that does not reject the call with a return < 0 and a last-error text.
_NULL_POINTER_CALLS = r'''
import ctypes
from hawkeye_b200 import _lib
lib = _lib.lib()
raw_error = ctypes.CDLL(_lib.LIB_PATH).hk_last_error
raw_error.restype = ctypes.c_void_p
error_buf = raw_error()                  # this thread's last-error text; cleared before every call
for name, (res, argtypes, _) in sorted(_lib.parse_header().items()):
    if res is not ctypes.c_int or ctypes.c_void_p not in argtypes:
        continue
    args = [None if t is ctypes.c_void_p else t(0.5) if t is ctypes.c_float else t(8) for t in argtypes]
    ctypes.memset(error_buf, 0, 1)
    rc = getattr(lib, name)(*args)
    msg = lib.hk_last_error().decode()
    if rc >= 0 or not msg:
        print(f'{name}: returned {rc}, last error {msg!r}')
'''


def test_null_pointers_are_rejected_at_every_entry_point(lib):
    """The header promises that an argument error returns < 0 and launches nothing. The calls run in a child process
    that sees no GPU, so an entry point that skipped its checks fails to launch instead of touching a device."""
    import os
    import subprocess
    import sys
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    p = subprocess.run([sys.executable, '-c', _NULL_POINTER_CALLS], cwd=repo, capture_output=True, text=True,
                       env=dict(os.environ, CUDA_VISIBLE_DEVICES=''), timeout=300)
    assert p.returncode == 0, p.stderr
    assert p.stdout == '', p.stdout
