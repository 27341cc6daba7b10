"""Host-side argument checks of the direct first-layer entries (hk_conv3x3_first_fwd_direct,
hk_conv3x3_first_wgrad_direct_acc), exercised WITHOUT a GPU: every error returns before a launch."""
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


def test_first_fwd_direct_argument_errors(lib):
    f = lib.hk_conv3x3_first_fwd_direct
    assert f(None, FAKE, None, FAKE, 2, 8, 8, 64, None) == -1
    assert f(FAKE, None, None, FAKE, 2, 8, 8, 64, None) == -1
    assert f(FAKE, FAKE, None, None, 2, 8, 8, 64, None) == -1
    assert f(FAKE, FAKE, None, FAKE, 2, 8, 8, 32, None) == -3 and '64 only' in err(lib)
    assert f(FAKE, FAKE, None, FAKE, 0, 8, 8, 64, None) == -1
    assert f(FAKE, FAKE, None, FAKE + 4, 2, 8, 8, 64, None) == -2
    assert f(FAKE, FAKE, None, FAKE, 1 << 12, 1 << 10, 1 << 10, 64, None) == -3 and 'too many pixels' in err(lib)


def test_first_wgrad_direct_argument_errors(lib):
    f = lib.hk_conv3x3_first_wgrad_direct_acc
    nb = lib.hk_conv3x3_first_wgrad_direct_workspace_bytes()
    assert nb >= 64 * 32 * 4 and nb == lib.hk_conv3x3_first_wgrad_direct_workspace_bytes()
    assert f(None, FAKE, FAKE, None, 2, 8, 8, 64, FAKE, nb, 0, None) == -1
    assert f(FAKE, None, FAKE, None, 2, 8, 8, 64, FAKE, nb, 0, None) == -1
    assert f(FAKE, FAKE, None, None, 2, 8, 8, 64, FAKE, nb, 0, None) == -1
    assert f(FAKE, FAKE, FAKE, None, 2, 8, 8, 48, FAKE, nb, 0, None) == -3 and '64 only' in err(lib)
    assert f(FAKE, FAKE, FAKE, None, 2, 0, 8, 64, FAKE, nb, 0, None) == -1
    assert f(FAKE, FAKE, FAKE, None, 2, 8, 8, 64, None, nb, 0, None) == -4
    assert f(FAKE, FAKE, FAKE, None, 2, 8, 8, 64, FAKE, nb - 4, 1, None) == -4
    assert f(FAKE, FAKE, FAKE, None, 1 << 12, 1 << 10, 1 << 10, 64, FAKE, nb, 0, None) == -3
