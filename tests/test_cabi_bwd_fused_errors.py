"""Host-side argument checks of the fused backward entries (hk_conv3x3_dgrad_unpool, hk_conv3x3_dgrad_first_wgrad_acc),
exercised WITHOUT a GPU: every error returns before a launch."""
import pytest

FAKE = 0x10000      # a non-null, 16-byte aligned address that must never be dereferenced on these paths


@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as g
    g.build()
    from hawkeye_b200 import _lib
    return _lib.lib()


def err(lib):
    return lib.hk_last_error().decode()


def test_dgrad_unpool_argument_errors(lib):
    f = lib.hk_conv3x3_dgrad_unpool
    assert f(None, FAKE, FAKE, FAKE, 2, 8, 8, 64, 64, None) == -1
    assert f(FAKE, None, FAKE, FAKE, 2, 8, 8, 64, 64, None) == -1
    assert f(FAKE, FAKE, None, FAKE, 2, 8, 8, 64, 64, None) == -1
    assert f(FAKE, FAKE, FAKE, None, 2, 8, 8, 64, 64, None) == -1
    assert f(FAKE, FAKE, FAKE, FAKE, 0, 8, 8, 64, 64, None) == -1
    assert f(FAKE, FAKE, FAKE, FAKE, 2, 8, 8, 48, 64, None) == -3 and 'multiples of 32' in err(lib)
    assert f(FAKE, FAKE, FAKE, FAKE, 2, 8, 8, 64, 40, None) == -3
    assert f(FAKE, FAKE, FAKE, FAKE, 2, 8, 12, 64, 64, None) == -3 and 'multiple of 8x8' in err(lib)
    assert f(FAKE, FAKE, FAKE, FAKE, 2, 4, 8, 64, 64, None) == -3
    assert f(FAKE, FAKE, FAKE, FAKE, 1, 1024, 1024, 512, 64, None) == -3 and 'too large' in err(lib)
    assert f(FAKE + 4, FAKE, FAKE, FAKE, 2, 8, 8, 64, 64, None) == -2
    assert f(FAKE, FAKE, FAKE + 4, FAKE, 2, 8, 8, 64, 64, None) == -2
    assert f(FAKE, FAKE, FAKE, FAKE + 8, 2, 8, 8, 64, 64, None) == -2


def test_dgrad_first_wgrad_argument_errors(lib):
    f = lib.hk_conv3x3_dgrad_first_wgrad_acc
    nb = lib.hk_conv3x3_dgrad_first_wgrad_workspace_bytes()
    assert nb >= 64 * 32 * 4 and nb == lib.hk_conv3x3_dgrad_first_wgrad_workspace_bytes()
    assert f(None, FAKE, FAKE, FAKE, FAKE, None, 2, 8, 16, 64, 64, FAKE, nb, 0, None) == -1
    assert f(FAKE, None, FAKE, FAKE, FAKE, None, 2, 8, 16, 64, 64, FAKE, nb, 0, None) == -1
    assert f(FAKE, FAKE, FAKE, None, FAKE, None, 2, 8, 16, 64, 64, FAKE, nb, 0, None) == -1
    assert f(FAKE, FAKE, FAKE, FAKE, None, None, 2, 8, 16, 64, 64, FAKE, nb, 0, None) == -1
    assert f(FAKE, FAKE, FAKE, FAKE, FAKE, None, 2, 0, 16, 64, 64, FAKE, nb, 0, None) == -1
    assert f(FAKE, FAKE, FAKE, FAKE, FAKE, None, 2, 8, 16, 32, 64, FAKE, nb, 0, None) == -3 and '64 only' in err(lib)
    assert f(FAKE, FAKE, FAKE, FAKE, FAKE, None, 2, 8, 16, 64, 128, FAKE, nb, 0, None) == -3
    assert f(FAKE, FAKE, FAKE, FAKE, FAKE, None, 2, 8, 24, 64, 64, FAKE, nb, 0, None) == -3 and '16x8' in err(lib)
    assert f(FAKE, FAKE, FAKE, FAKE, FAKE, None, 2, 12, 16, 64, 64, FAKE, nb, 0, None) == -3
    assert f(FAKE + 4, FAKE, FAKE, FAKE, FAKE, None, 2, 8, 16, 64, 64, FAKE, nb, 0, None) == -2
    assert f(FAKE, FAKE, FAKE + 4, FAKE, FAKE, None, 2, 8, 16, 64, 64, FAKE, nb, 0, None) == -2
    assert f(FAKE, FAKE, FAKE, FAKE, FAKE, None, 2, 8, 16, 64, 64, None, nb, 0, None) == -4
    assert f(FAKE, FAKE, FAKE, FAKE, FAKE, None, 2, 8, 16, 64, 64, FAKE, nb - 4, 1, None) == -4
    assert f(FAKE, FAKE, FAKE, FAKE, FAKE, None, 1 << 14, 1 << 12, 1 << 12, 64, 64, FAKE, nb, 0, None) == -3 and \
        'too many tiles' in err(lib)
