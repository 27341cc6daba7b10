"""Mixup and CutMix on the device (``hk_mix_batch``, csrc/mixup.cu).  The loader's workers make the draws
(``hawkeye_b200.data.MixupCutmixCollateFn``) and hand the batch one row of ``MIX_COLS`` doubles; the kernel applies it
to the staged fp32 batch, and ``ops.CrossEntropyLSMix`` reads the same row for the soft target.  Image i is paired with
image i - 1 (mod B), the reference's ``batch.roll(1, 0)``, so no dense [B, K] target is ever built.  The columns:

==============  ====================================================================================================
``KIND``        ``MIXUP`` (0) or ``CUTMIX`` (1)
``LAMBDA``      the Dirichlet draw: the image weight of Mixup; CutMix sizes its box from it
``BOX`` (4)     CutMix's x1, y1, x2, y2: columns [x1, x2) and rows [y1, y2) come from image i - 1 (zeros for Mixup)
``WEIGHT``      the target weight w of label i (label i - 1 gets 1 - w): lambda for Mixup, 1 - area / (W H) for CutMix
==============  ====================================================================================================
"""
import ctypes

import numpy as np
import torch

from . import _lib

KIND, LAMBDA, BOX, WEIGHT = 0, 1, 2, 6
MIX_COLS = 7
MIXUP, CUTMIX = 0, 1


def mix_row(kind, lam, box=(0, 0, 0, 0), weight=None):
    """One batch's mix row; ``weight`` defaults to ``lam`` (Mixup's target weight)."""
    row = np.zeros(MIX_COLS, np.float64)
    row[KIND], row[LAMBDA] = kind, lam
    row[BOX:BOX + 4] = box
    row[WEIGHT] = lam if weight is None else weight
    return torch.from_numpy(row)


def check_row(row, height, width):
    """Raises ValueError unless ``row`` (a host float64 row) is a mix row the kernels accept for H x W images: a known
    kind, lambda and weight in [0, 1], and a box inside the image (``hk_mix_check``)."""
    row = np.ascontiguousarray(np.asarray(row, np.float64))
    if row.shape != (MIX_COLS,):
        raise ValueError(f'a mix row has {MIX_COLS} columns, not shape {row.shape}')
    if _lib.lib().hk_mix_check(row.ctypes.data_as(ctypes.c_void_p), int(height), int(width)) != 0:
        raise ValueError(_lib.lib().hk_last_error().decode())


def mix_batch(x, mix, out=None):
    """fp32 NCHW ``x`` mixed by the device row ``mix`` into ``out`` (allocated when None): out of place, since image i
    reads image i - 1."""
    if not (x.is_cuda and mix.is_cuda) or x.dtype != torch.float32 or mix.dtype != torch.float64 or x.dim() != 4 \
            or not x.is_contiguous() or mix.numel() != MIX_COLS or not mix.is_contiguous():
        raise _lib.HawkeyeLibError('mix_batch: x must be contiguous fp32 NCHW and mix a float64 row of '
                                   f'{MIX_COLS}, both on the device')
    out = torch.empty_like(x) if out is None else out
    if out.shape != x.shape or out.dtype != torch.float32 or not out.is_contiguous() or out.data_ptr() == x.data_ptr():
        raise _lib.HawkeyeLibError('mix_batch: out must be a separate contiguous fp32 tensor of the shape of x')
    N, C, H, W = x.shape
    _lib.call('hk_mix_batch', x, mix, out, N, C, H, W, _lib.stream_ptr())
    return out
