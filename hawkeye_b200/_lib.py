"""ctypes binding of libhawkeye_b200.so — the only route from Python to the CUDA kernels.

Argument types are derived from ``include/hawkeye_b200.h`` itself, so the header is the single source
of truth for the C ABI.  There is NO fallback: if the library is missing or a call fails, we raise.
"""
import ctypes
import os
import re

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libhawkeye_b200.so')
HEADER_PATH = os.path.join(os.path.dirname(_HERE), 'include', 'hawkeye_b200.h')

_CTYPES = {
    'int': ctypes.c_int, 'float': ctypes.c_float, 'long long': ctypes.c_longlong, 'size_t': ctypes.c_size_t,
    'void': None, 'const char*': ctypes.c_char_p,
}


def _ctype(t):
    t = ' '.join(t.replace('*', ' * ').split()).replace(' *', '*')
    if t in _CTYPES:
        return _CTYPES[t]
    if t.endswith('*'):
        return ctypes.c_void_p
    raise ValueError(f'unknown C type in header: {t!r}')


def parse_header(path=HEADER_PATH):
    """-> {name: (restype, [argtypes], [argnames])} for every prototype in the header."""
    src = open(path).read()
    src = re.sub(r'/\*.*?\*/', ' ', src, flags=re.S)
    src = re.sub(r'//[^\n]*', ' ', src)
    src = re.sub(r'#[^\n]*', ' ', src)
    src = src.replace('extern "C" {', ' ')
    protos = {}
    for m in re.finditer(r'([A-Za-z_][\w\s\*]*?)\b(hk_\w+)\s*\(([^)]*)\)\s*;', src):
        ret, name, args = m.group(1).strip(), m.group(2), m.group(3).strip()
        argtypes, argnames = [], []
        if args and args != 'void':
            for a in args.split(','):
                a = a.strip()
                mm = re.match(r'(.*?)(\w+)$', a)
                argtypes.append(_ctype(mm.group(1).strip()))
                argnames.append(mm.group(2))
        protos[name] = (_ctype(ret), argtypes, argnames)
    return protos


class HawkeyeLibError(RuntimeError):
    pass


_lib = None
_protos = None


def lib():
    global _lib, _protos
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise HawkeyeLibError(
                f'{LIB_PATH} not found: build it with `python -c "import __graft_entry__ as g; g.build()"` '
                '(hawkeye_b200 has no CPU / PyTorch fallback)')
        _lib = ctypes.CDLL(LIB_PATH)
        _protos = parse_header()
        for name, (res, argtypes, _) in _protos.items():
            fn = getattr(_lib, name)  # AttributeError here == header/library mismatch, which must be loud
            fn.restype = res
            fn.argtypes = argtypes
    return _lib


def _arg(a):
    if isinstance(a, torch.Tensor):
        return a.data_ptr()
    return a


def call(name, *args):
    """Invoke an ``int hk_*`` entry point; raises with hk_last_error() on a non-zero return."""
    fn = getattr(lib(), name)
    rc = fn(*[_arg(a) for a in args])
    if rc != 0:
        msg = lib().hk_last_error().decode()
        raise HawkeyeLibError(f'{name} failed (rc={rc}): {msg}')


def query(name, *args):
    """Invoke an entry point that returns a value (workspace sizes, counters, strings)."""
    return getattr(lib(), name)(*[_arg(a) for a in args])


def stream_ptr():
    """Handle of the current CUDA stream.  Read directly rather than through torch.cuda.current_stream(), which builds a
    Stream object: this runs for every launch, and the ResNet steps are bound by host launch time."""
    return torch._C._cuda_getCurrentRawStream(torch._C._cuda_getDevice())


def set_precise(on):
    """Process-wide precision mode of the library: False = single-pass TF32 (default), True = 3xTF32 (parity runs)."""
    lib().hk_set_precise(1 if on else 0)


def get_precise():
    return bool(lib().hk_get_precise())


def launch_count():
    return int(lib().hk_launch_count())


def reset_launch_count():
    lib().hk_reset_launch_count()
