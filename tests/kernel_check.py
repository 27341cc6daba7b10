"""The checking machinery of the kernel test suites: guarded and poisoned device buffers, one raw C-ABI call, one
element-wise bound check with its bound builders, the record of each suite's worst c-term shares, and the precision
fixtures.

Every output a check reads is NaN-filled (uint8: 255) between runs of guard words, so an element a kernel never writes
fails its bound and a store outside the buffer changes a guard word.  Inputs are copied between runs of NaN, so a read
past their end poisons the result; workspaces are poisoned the same way and have exactly the queried byte count.

Error model constants: U, the fp32 unit roundoff; RND, the tf32 round-to-nearest on store; TRUNC, the MMA's truncation
of an operand that is not tf32; PAIR, what a (hi, lo) tf32 pair loses (its representation error, or the dropped lo.lo
product).
"""
import math
from typing import NamedTuple, Optional

import pytest
import torch

U = 2.0 ** -24
RND = 2.0 ** -11
TRUNC = 2.0 ** -10
PAIR = 2.0 ** -22

GUARD_BYTES = 65536       # guard words on each side of a guarded buffer
GUARD = 12345.0           # the guard word of a float buffer
CODE_GUARD = 0xA5         # the guard byte of a uint8 (code, arg-max) or integer buffer
HK_ERR_UNSUPPORTED = -3   # include/hawkeye_b200.h


def nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def nchw(t):
    return t.permute(0, 3, 1, 2).contiguous()


# ------------------------------------------------------------------------------------------------ guarded buffers
class _Guards:
    """the runs of guard words on both sides of a buffer, and a copy of their bits"""

    def __init__(self, before, after):
        self.runs = (before, after)
        self.bits = tuple(r.clone() for r in self.runs)

    def intact(self):
        return all(torch.equal(r.view(torch.uint8), b.view(torch.uint8)) for r, b in zip(self.runs, self.bits))


def guarded(shape, dtype=torch.float32, fill=None, word=None):
    """A device buffer of `shape` between GUARD_BYTES of guard words on each side.  By default a float buffer is
    NaN-filled with GUARD words around it, an integer one 255-filled (all ones) with CODE_GUARD around it.  abi() and
    assert_guards() check the guards of a buffer made here."""
    shape = tuple(shape)
    n = math.prod(shape)
    g = GUARD_BYTES // torch.empty((), dtype=dtype).element_size()
    flt = dtype.is_floating_point
    buf = torch.full((g + n + g,), (GUARD if flt else CODE_GUARD) if word is None else word, dtype=dtype, device='cuda')
    body = buf[g:g + n]
    body.fill_((float('nan') if flt else -1 if dtype != torch.uint8 else 255) if fill is None else fill)
    body = body.view(shape)
    body.guards = _Guards(buf[:g], buf[g + n:])
    return body


def poisoned(t):
    """a device copy of t between runs of NaN (integers: -7, out of range as an index or a label): a read past either
    end poisons the result"""
    body = guarded(t.shape, t.dtype, word=float('nan') if t.dtype.is_floating_point else -7)
    body.copy_(t)
    return body


def workspace(query, *args):
    """a 0xFF-filled (NaN as floats) guarded workspace of exactly the byte count the entry point `query` returns for
    args -> (workspace, byte count)"""
    from hawkeye_b200 import _lib
    nb = int(_lib.query(query, *args))
    return guarded((nb,), torch.uint8), nb


def assert_guards(*ts, tag=''):
    """every tensor of ts made by guarded() or poisoned() still has its guard words"""
    for i, t in enumerate(ts):
        g = getattr(t, 'guards', None)
        assert g is None or g.intact(), f'{tag}: store outside buffer {i}'


class Out:
    """an output argument of abi(): replaced by a fresh guarded() buffer of this shape and dtype, which abi() returns"""

    def __init__(self, shape, dtype=torch.float32):
        self.shape, self.dtype = tuple(shape), dtype


def abi(name, *args, inputs=(), precise=None):
    """Call the C-ABI entry point `name` with the current stream appended and synchronise.  Each Out argument becomes a
    fresh guarded buffer; afterwards the guards of every guarded argument are checked and each tensor in `inputs` must
    be bit-unchanged.  With `precise` given the call runs in that precision mode and the previous mode is restored.
    -> the buffers made for the Out arguments, in order."""
    from hawkeye_b200 import _lib
    outs = [guarded(a.shape, a.dtype) for a in args if isinstance(a, Out)]
    it = iter(outs)
    args = [next(it) if isinstance(a, Out) else a for a in args]
    before = [t.clone() for t in inputs]
    prev = _lib.get_precise()
    if precise is not None:
        _lib.set_precise(precise)
    try:
        _lib.call(name, *args, _lib.stream_ptr())
        torch.cuda.synchronize()
    finally:
        _lib.set_precise(prev)
    assert_guards(*args, tag=name)
    for t, b in zip(inputs, before):
        assert torch.equal(t.view(torch.uint8), b.view(torch.uint8)), f'{name}: an input was modified'
    return outs


# ----------------------------------------------------------------------------------------------- the element-wise check
class Bound(NamedTuple):
    """|out - ref| <= cterm + fixed (+ RND * max(|out|, |ref|), the tf32 rounding on store, where `rounded`), element by
    element.  cterm is c times the scale of the error, whose share check() reports; with cterm None the share reported
    is that of the whole bound."""
    cterm: Optional[torch.Tensor] = None
    fixed: object = 0.0
    rounded: bool = False

    def fixed_of(self, out, ref):
        return self.fixed + rounding_term(out, ref) if self.rounded else self.fixed

    def total(self, out, ref):
        f = self.fixed_of(out, ref)
        return f if self.cterm is None else self.cterm + f


def rounding_term(out, ref):
    return RND * torch.fmax(out.double().abs(), ref.double().abs())


def c_bound(absref, c):
    """the c-term bound c * absref"""
    return Bound(c * absref.double())


def rnd_bound(absref, c):
    """c * absref plus the rounding on store RND * max(|out|, |ref|), for an output the kernel rounds to tf32"""
    return Bound(c * absref.double(), rounded=True)


def store_bound(out, bound, rounded=True):
    """an explicit bound, plus RND * |out| where the kernel rounds its output to tf32 on store"""
    return Bound(fixed=bound + RND * out.double().abs().to(bound.device) if rounded else bound)


def _worst(ratio):
    ratio = torch.nan_to_num(ratio, nan=float('inf'))
    k = int(ratio.argmax())
    return float(ratio.flatten()[k]), [int(i) for i in torch.unravel_index(torch.tensor(k), tuple(ratio.shape))]


def worst_ratio(out, ref, bound):
    """the worst |out - ref| / bound (inf where ref is finite and out is not) and its index; bound: a Bound or tensor"""
    r = ref.double()
    o = out.double().to(r.device)
    b = bound.total(o, r) if isinstance(bound, Bound) else bound
    err = (o - r).abs()
    ratio = torch.where(err == 0, torch.zeros((), dtype=err.dtype, device=err.device), err / b)
    ratio = torch.where(torch.isfinite(o) | ~torch.isfinite(r), ratio, math.inf)
    return _worst(ratio)


def check(out, ref, bound, tag, names=('image', 'h', 'w', 'channel'), n0=0):
    """Assert |out - ref| <= bound for every element, and that out is finite wherever ref is, whatever the bound.  bound
    is a Bound (from c_bound, rnd_bound, store_bound) or a tensor taken whole.  out, ref and the bound have one shape;
    n0 is the index of out's first element along dimension 0 in the full tensor.

    Prints the worst |out - ref| / bound and the worst share of the c term that the error beyond the fixed term takes
    (the fixed term alone can bring the first near 1 whatever c is, so the second is the margin of c).  Returns that
    share; on failure reports the number of violating elements and the worst one's index (`names`)."""
    r = ref.double()
    o = out.double().to(r.device)
    if not isinstance(bound, Bound):
        bound = Bound(fixed=bound)
    err = (o - r).abs()
    share = None
    if bound.cterm is not None:
        excess = (err - bound.fixed_of(o, r)).clamp_min(0)
        share, _ = _worst(torch.where(excess == 0, torch.zeros((), dtype=err.dtype, device=err.device),
                                      excess / bound.cterm))
        del excess
    b = bound.total(o, r)
    worst, idx = worst_ratio(o, r, b)
    share = worst if share is None else share
    idx[0] += n0
    where = ', '.join(f'{nm} {i}' for nm, i in zip(names, idx))
    print(f'{tag}: worst |err|/bound {worst:.3g} ({where}); c-term share {share:.3g}', flush=True)
    nbad = int((~(err <= b) | (torch.isfinite(r) & ~torch.isfinite(o))).sum())
    if nbad:
        j = tuple([idx[0] - n0] + idx[1:])
        bj = b[j] if isinstance(b, torch.Tensor) and b.dim() else b
        raise AssertionError(f'{tag}: {nbad} of {err.numel()} elements out of bound; worst at ({where}): out '
                             f'{float(o[j]):.9g} ref {float(r[j]):.9g} bound {float(bj):.3g} ratio {worst:.3g}')
    return share


class Worst(dict):
    """constant -> (the worst c-term share over the checks run so far, the tag of that check); one per suite.  consts
    names the constants check_c takes."""

    def __init__(self, **consts):
        super().__init__()
        self.consts = consts

    def add(self, const, share, tag):
        if share > self.get(const, (-1.0, ''))[0]:
            self[const] = (share, tag)
        return share

    def summary(self):
        return ', '.join(f'{k} {v:.3g} ({t})' for k, (v, t) in sorted(self.items()))

    def check_c(self, const, tag, out, ref, fixed, scale, names):
        """|out - ref| <= fixed + c * scale for every element, c the constant named const; prints and records the worst
        share of c * scale that the error beyond `fixed` takes"""
        c = self.consts[const]
        o = out.double()
        excess = ((o - ref).abs() - fixed).clamp_min(0)
        share = torch.where(excess == 0, torch.zeros_like(excess), excess / (c * scale))
        share = float(torch.nan_to_num(share, nan=math.inf).max())
        print(f'{tag}: share of {const} = 2^{math.log2(c):.0f} taken {share:.3g}', flush=True)
        self.add(const, share, tag)
        check(o, ref, fixed + c * scale, tag, names=names)
        return share


# ------------------------------------------------------------------------------------------------ precision fixtures
@pytest.fixture(params=[0, 1], ids=['tf32', 'precise'])
def precise(request):
    """the library's precision mode for the test: 0 single-pass TF32, 1 3xTF32; restored to 0 after it"""
    from hawkeye_b200 import _lib
    _lib.set_precise(request.param)
    yield request.param
    _lib.set_precise(0)


@pytest.fixture
def precise_on():
    """3xTF32 mode for the test, restored to single-pass TF32 after it"""
    from hawkeye_b200 import _lib
    _lib.set_precise(1)
    yield
    _lib.set_precise(0)
