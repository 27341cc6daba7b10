"""The default train and eval presets on the GPU (``hk_augment_*``, csrc/augment.cu): the loader's workers decode and draw
each image's parameters, and everything after the decode runs on the device in three launches per batch.

A batch travels as ``PackedImages``: the decoded RGB uint8 HWC images back to back in one buffer, the byte offset and
(H, W) of each, and one row of ``PARAM_COLS`` doubles per image with its draws.  The columns:

====================  ======================================================================================
``BOX`` (4)           source box x, y, width, height: RandomResizedCrop's crop, or the whole image (eval)
``VIRTUAL`` (2)       width, height the box is resized to (S x S, or Resize's output size)
``WINDOW`` (2)        x, y of the kept S x S window in the resized image (CenterCrop; 0 for the train crop)
``FLIP``              1 when RandomHorizontalFlip fired
``OP``, ``MAG``       TrivialAugmentWide's op index (``TA_OPS`` order) and signed magnitude, as ``_apply_op`` receives them
``MATRIX`` (6)        the inverse affine matrix PIL applies for ShearX/Y, TranslateX/Y and Rotate
``ERASE`` (4)         RandomErasing's top, left, height, width; height 0 when nothing is erased
====================  ======================================================================================
"""
import math

import numpy as np
import torch

from . import _lib

BOX, VIRTUAL, WINDOW, FLIP, OP, MAG, MATRIX, ERASE = 0, 4, 6, 8, 9, 10, 11, 17
PARAM_COLS = 21

# TrivialAugmentWide._augmentation_space order
TA_OPS = ('Identity', 'ShearX', 'ShearY', 'TranslateX', 'TranslateY', 'Rotate', 'Brightness', 'Color', 'Contrast',
          'Sharpness', 'Posterize', 'Solarize', 'AutoContrast', 'Equalize')
GEOMETRIC = ('ShearX', 'ShearY', 'TranslateX', 'TranslateY', 'Rotate')


def pil_rotate_matrix(angle, width, height):
    """The inverse matrix ``PIL.Image.rotate(angle)`` hands to its AFFINE transform (no expand, centre, translate).
    Angles PIL turns into a copy or a transpose give the identity or an exact permutation of pixel centres, which the
    bilinear transform samples without interpolation, so one path covers them."""
    angle = angle % 360.0
    if angle == 0:
        return [1.0, 0.0, 0.0, 0.0, 1.0, 0.0]
    cx, cy = width / 2, height / 2
    a = -math.radians(angle)
    m = [round(math.cos(a), 15), round(math.sin(a), 15), 0.0, round(-math.sin(a), 15), round(math.cos(a), 15), 0.0]
    m[2], m[5] = m[0] * -cx + m[1] * -cy + m[2], m[3] * -cx + m[4] * -cy + m[5]
    m[2] += cx
    m[5] += cy
    return m


def op_matrix(op_name, magnitude, width, height):
    """The inverse affine matrix of a geometric TrivialAugmentWide op on a PIL image of this size: the arguments
    ``autoaugment._apply_op`` passes to ``F.affine`` (shears about the top-left corner, translations about the centre),
    through torchvision's own ``_get_inverse_affine_matrix``; Rotate through ``F.rotate``, which is PIL's rotate."""
    from torchvision.transforms.functional import _get_inverse_affine_matrix
    if op_name == 'Rotate':
        return pil_rotate_matrix(magnitude, width, height)
    if op_name in ('ShearX', 'ShearY'):
        s = math.degrees(math.atan(magnitude))
        return _get_inverse_affine_matrix([0, 0], 0.0, [0, 0], 1.0, [s, 0.0] if op_name == 'ShearX' else [0.0, s])
    t = [int(magnitude), 0] if op_name == 'TranslateX' else [0, int(magnitude)]
    return _get_inverse_affine_matrix([width * 0.5, height * 0.5], 0.0, t, 1.0, [0.0, 0.0])


def param_row(box, virtual, window=(0, 0), flip=False, op='Identity', magnitude=0.0, size=None, erase=None):
    """One image's row of the parameter table.  ``size`` (S) is needed for the geometric ops' matrix."""
    row = np.zeros(PARAM_COLS, np.float64)
    row[BOX:BOX + 4] = box
    row[VIRTUAL:VIRTUAL + 2] = virtual
    row[WINDOW:WINDOW + 2] = window
    row[FLIP] = 1.0 if flip else 0.0
    row[OP] = TA_OPS.index(op)
    row[MAG] = magnitude
    if op in GEOMETRIC:
        row[MATRIX:MATRIX + 6] = op_matrix(op, magnitude, size, size)
    if erase is not None:
        row[ERASE:ERASE + 4] = erase
    return row


class PackedImages:
    """One batch of decoded images and their draws (see the module docstring), on the host or on the device.  ``size``
    is S, ``mean`` and ``std`` the Normalize constants.  The DataLoader pins it through ``pin_memory``.

    With ``dataset.transformer.decode: cuda`` some images may still be encoded: ``jpeg`` is then their
    ``ops_jpeg.JpegBatch``, ``data`` holds the pixel images only, as the first bytes of a device pixel buffer of
    ``pixel_bytes`` bytes, and the encoded images' offsets point past them, where the decode writes."""

    def __init__(self, data, offsets, sizes, params, size, mean, std, jpeg=None, pixel_bytes=None):
        self.data, self.offsets, self.sizes, self.params = data, offsets, sizes, params
        self.size, self.mean, self.std = int(size), tuple(mean), tuple(std)
        self.jpeg = jpeg
        self.pixel_bytes = int(data.numel() if pixel_bytes is None else pixel_bytes)

    def __len__(self):
        return self.offsets.shape[0]

    def _map(self, fn):
        return PackedImages(fn(self.data), fn(self.offsets), fn(self.sizes), fn(self.params), self.size, self.mean,
                            self.std, None if self.jpeg is None else self.jpeg._map(fn), self.pixel_bytes)

    def pin_memory(self):
        return self._map(lambda t: t.pin_memory())

    def to(self, device, non_blocking=False):
        return self._map(lambda t: t.to(device, non_blocking=non_blocking))

    def pixels(self, out=None, work=None):
        """The uint8 pixel buffer of a batch on the device with every image decoded (``ops_jpeg.decode`` into ``out``,
        with the grow-only buffers of ``work``), and the decode's status words (None without encoded images)."""
        if self.jpeg is None:
            return self.data, None
        from .ops_jpeg import decode
        out = torch.empty(self.pixel_bytes, dtype=torch.uint8, device=self.data.device) if out is None else out
        out[:self.data.numel()].copy_(self.data)
        return out, decode(self.jpeg, out, self.offsets, work=work)

    def images(self, out=None, work=None, lut=None):
        """The model's fp32 NCHW input [N, 3, S, S] of a batch on the device (``augment``).  Encoded images are decoded
        first, and a decode error raises here, naming the file."""
        data, status = self.pixels()
        if status is not None:
            from .ops_jpeg import raise_on_status
            raise_on_status(status.cpu().numpy(), self.jpeg.paths)
        return augment(data, self.offsets, self.sizes, self.params, self.size, self.mean, self.std, out, work, lut)


def pack(images, params, size, mean, std):
    """Decoded uint8 HWC arrays, or ``ops_jpeg.EncodedJPEG`` images, and their parameter rows -> ``PackedImages`` on the
    host.  The pixel images come first in the pixel buffer, the encoded ones after them."""
    from .ops_jpeg import EncodedJPEG, pack_encoded
    if not images:
        raise ValueError('pack: empty batch')
    encoded = [i for i, a in enumerate(images) if isinstance(a, EncodedJPEG)]
    plain = [i for i, a in enumerate(images) if not isinstance(a, EncodedJPEG)]
    for i in plain:
        a = images[i]
        if not isinstance(a, np.ndarray) or a.dtype != np.uint8 or a.ndim != 3 or a.shape[2] != 3:
            raise ValueError(f'pack: expected uint8 HWC RGB images, got {getattr(a, "dtype", type(a))} '
                             f'{getattr(a, "shape", "")}')
    sizes = np.array([(a.size[1], a.size[0]) if isinstance(a, EncodedJPEG) else a.shape[:2] for a in images], np.int32)
    nbytes = sizes[:, 0].astype(np.int64) * sizes[:, 1] * 3
    order = plain + encoded
    offsets = np.zeros(len(images), np.int64)
    offsets[order] = np.concatenate(([0], np.cumsum(nbytes[order])[:-1]))
    data = torch.empty(int(nbytes[plain].sum()), dtype=torch.uint8)
    buf = data.numpy()
    for i in plain:
        buf[offsets[i]:offsets[i] + nbytes[i]] = np.ascontiguousarray(images[i]).reshape(-1)
    table = np.stack(params).astype(np.float64)
    if table.shape[1] != PARAM_COLS:
        raise ValueError(f'pack: parameter rows have {table.shape[1]} columns, expected {PARAM_COLS}')
    box = table[:, BOX:BOX + 4]
    if (box[:, 2:] < 1).any() or (box[:, :2] < 0).any() or (box[:, 0] + box[:, 2] > sizes[:, 1]).any() or \
            (box[:, 1] + box[:, 3] > sizes[:, 0]).any():
        raise ValueError('pack: a source box lies outside its image')
    jpeg = pack_encoded([images[i] for i in encoded], encoded) if encoded else None
    return PackedImages(data, torch.from_numpy(offsets), torch.from_numpy(sizes), torch.from_numpy(table), size, mean, std,
                        jpeg, int(nbytes.sum()))


def augment(data, offsets, sizes, params, size, mean, std, out=None, work=None, lut=None):
    """Device tensors of a packed batch -> fp32 [N, 3, S, S]: crop-resize into ``work`` (uint8 [N, S, S, 3]), the tables
    of Contrast / AutoContrast / Equalize into ``lut`` (uint8 [N, 3, 256]), then the op, Normalize and erasing into
    ``out``.  Buffers left as None are allocated."""
    for t, dt, name in ((data, torch.uint8, 'data'), (offsets, torch.int64, 'offsets'), (sizes, torch.int32, 'sizes'),
                        (params, torch.float64, 'params')):
        if not t.is_cuda or t.dtype != dt or not t.is_contiguous():
            raise _lib.HawkeyeLibError(f'augment: {name} must be a contiguous CUDA {dt} tensor')
    N, S = offsets.shape[0], int(size)
    if sizes.shape != (N, 2) or params.shape != (N, PARAM_COLS):
        raise _lib.HawkeyeLibError(f'augment: sizes {tuple(sizes.shape)} / params {tuple(params.shape)} do not match '
                                   f'{N} images')
    dev = data.device
    work = torch.empty(N, S, S, 3, dtype=torch.uint8, device=dev) if work is None else work
    lut = torch.empty(N, 3, 256, dtype=torch.uint8, device=dev) if lut is None else lut
    out = torch.empty(N, 3, S, S, dtype=torch.float32, device=dev) if out is None else out
    if work.shape != (N, S, S, 3) or lut.shape != (N, 3, 256) or out.shape != (N, 3, S, S) or out.dtype != torch.float32:
        raise _lib.HawkeyeLibError('augment: work / lut / out have the wrong shape or type')
    stream = _lib.stream_ptr()
    _lib.call('hk_augment_crop_resize', data, offsets, sizes, params, work, N, S, stream)
    _lib.call('hk_augment_stats', work, params, lut, N, S, stream)
    _lib.call('hk_augment_apply', work, params, lut, out, N, S, *[float(m) for m in mean], *[float(s) for s in std],
              stream)
    return out
