"""kernel_check.check on the CPU: a non-finite output fails whatever the bound, and the bound holds at its edge."""
import math

import pytest
import torch

from kernel_check import RND, Bound, c_bound, check, rnd_bound, store_bound

C = 2.0 ** -17


def _case():
    ref = torch.linspace(-3.0, 5.0, 24, dtype=torch.float64).reshape(2, 3, 4)
    absref = ref.abs() + 1.0
    return ref, absref


def _bounds(ref, absref):
    """every form of bound a suite passes: the c term, the c term plus the rounding on store, an explicit bound plus the
    rounding on store, and an explicit bound taken whole"""
    explicit = C * absref
    return {'c': c_bound(absref, C), 'rnd': rnd_bound(absref, C), 'store': store_bound(ref.float(), explicit),
            'whole': explicit}


@pytest.mark.parametrize('form', ['c', 'rnd', 'store', 'whole'])
@pytest.mark.parametrize('value', [math.inf, -math.inf, math.nan])
def test_non_finite_output_rejected(form, value):
    ref, absref = _case()
    out = ref.float().clone()
    out[1, 2, 3] = value
    with pytest.raises(AssertionError, match='1 of 24 elements out of bound'):
        check(out, ref, _bounds(ref, absref)[form], f'{form} {value}', names=('a', 'b', 'c'))


def test_non_finite_reference_does_not_excuse_a_mismatch():
    ref, absref = _case()
    ref[0, 0, 0] = math.inf
    out = ref.float().clone()
    out[0, 0, 0] = math.nan
    with pytest.raises(AssertionError):
        check(out, ref, c_bound(absref, C), 'nan against inf')


@pytest.mark.parametrize('form', ['c', 'rnd', 'whole'])
def test_bound_edge(form):
    """an error of 0.99 times the bound passes, one of 1.01 times it fails; fp64 outputs, so the error is exact"""
    ref, absref = _case()
    bound = _bounds(ref, absref)[form]
    full = bound.total(ref, ref) if isinstance(bound, Bound) else bound
    out = ref.clone()
    out[1, 0, 2] += 0.99 * full[1, 0, 2]
    check(out, ref, bound, f'{form} 0.99')
    out[1, 0, 2] = ref[1, 0, 2] + 1.01 * full[1, 0, 2] / (1 - RND if form == 'rnd' else 1)
    with pytest.raises(AssertionError):
        check(out, ref, bound, f'{form} 1.01')


def test_reported_index_includes_n0(capsys):
    ref, absref = _case()
    out = ref.float().clone()
    out[1, 2, 3] += 1.0
    with pytest.raises(AssertionError, match=r'worst at \(image 9, h 2, w 3\)'):
        check(out, ref, c_bound(absref, C), 'n0', names=('image', 'h', 'w'), n0=8)
    assert 'n0: worst |err|/bound' in capsys.readouterr().out


def test_share_is_of_the_c_term():
    """the printed and returned share is of c * absref, beyond the rounding term where the output is rounded"""
    ref, absref = _case()
    out = ref.clone()
    out[0, 1, 1] += 0.5 * C * absref[0, 1, 1]
    assert check(out, ref, c_bound(absref, C), 'share') == pytest.approx(0.5)
    assert check(out, ref, rnd_bound(absref, C), 'share rnd') == 0.0
