"""JPEG decode on the GPU for the device presets (``dataset.transformer.decode: cuda``; ``hk_jpeg_*``, csrc/jpeg.cu).

A loader worker reads the file and parses its markers only (``encoded_loader``).  A JPEG the device decodes stays
encoded: its scan, with the 0xFF00 stuffing and the RSTn markers taken out, travels in the packed batch next to its
tables.  Any other image is decoded by PIL in the worker, as without the key, and travels as pixels.  The device writes
the decoded images into the same uint8 pixel buffer as those, at their own offsets, so ``hk_augment_*`` reads both
alike.  The decoded pixels equal ``np.asarray(Image.open(path).convert('RGB'))`` bit for bit.

What the device decodes: SOF0 / SOF1 frames of 8-bit samples, Huffman-coded; one scan of every component, interleaved,
in frame order; optional DRI restart intervals; one component (grey), or three that libjpeg reads as YCbCr (a JFIF
marker, an Adobe marker with transform 1, or no such marker and component ids 1, 2, 3) with luma sampling 1x1, 2x1 or
2x2 and chroma 1x1.  Quant tables of 16-bit precision are taken up to 32767.  Everything else is decoded by PIL.

The device form of a batch (``JpegBatch``), beside ``PackedImages``' pixel images:

==============  ==================================================================================================
``scan``        uint8: the unstuffed scans back to back, padded by 8 bytes
``segs``        int32 [G + 1]: byte offset in ``scan`` where each restart segment starts; the last entry is the end
``header``      int32 [J, HEADER_COLS]: one row per encoded image (the ``H_*`` columns)
``qtabs``       int32 [Q, 64]: quant tables in natural order
``htabs``       uint8 [T, HTAB_BYTES]: Huffman tables as canonical maxcode / valoffset / huffval and a 9-bit look-ahead
==============  ==================================================================================================

Image paths stay on the host (``JpegBatch.paths``) so that a decode error can name its file.
"""
import numpy as np
import torch

from . import _lib

# header columns (csrc/jpeg.cu JpegCol)
(H_IMG, H_W, H_H, H_NCOMP, H_HY, H_VY, H_MCUX, H_MCUY, H_RI, H_SEG0, H_NSEG, H_BLK0, H_PLANE0, H_Q0, H_DC0,
 H_AC0) = 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 16, 19
HEADER_COLS = 22
LOOKAHEAD_BITS = 9
HTAB_DTYPE = np.dtype([('maxcode', '<i4', 18), ('valoffset', '<i4', 18), ('huffval', 'u1', 256),
                       ('look', '<u2', 1 << LOOKAHEAD_BITS)])
HTAB_BYTES = HTAB_DTYPE.itemsize
# Bytes of scan per chunk of the parallel Huffman decode: each thread decodes one chunk, from a guessed state until
# it agrees with the state its neighbour recorded.  tests/bench_decode.py times the choices.
CHUNK_BYTES = 256

STATUS_MESSAGES = {1: 'invalid Huffman code', 2: 'the entropy-coded data ends early',
                   3: 'the segment holds data past its last block', 4: 'the restart markers do not match the frame',
                   5: 'a coefficient index beyond 63'}

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,
                   7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31,
                   39, 46, 53, 60, 61, 54, 47, 55, 62, 63])

_SOF_OTHER = {0xC2, 0xC3, 0xC5, 0xC6, 0xC7, 0xC9, 0xCA, 0xCB, 0xCD, 0xCE, 0xCF}


class EncodedJPEG:
    """One JPEG the device decodes, parsed down to its markers: ``size`` is (W, H) as PIL gives it, ``scan`` the
    unstuffed entropy-coded data and ``segs`` the offsets of its restart segments in it."""

    def __init__(self, path, size, ncomp, sampling, restart, comps, qtabs, htabs, scan, segs):
        self.path, self.size, self.ncomp, self.sampling, self.restart = path, size, ncomp, sampling, restart
        self.comps, self.qtabs, self.htabs, self.scan, self.segs = comps, qtabs, htabs, scan, segs

    def __repr__(self):
        return f'EncodedJPEG({self.path!r}, size={self.size}, ncomp={self.ncomp}, sampling={self.sampling})'


def _huffman_ok(bits, vals, dc):
    code = 0
    for length in range(1, 17):
        code += bits[length - 1]
        if code > (1 << length):
            return False
        code <<= 1
    return not (dc and any(v > 15 for v in vals))


def parse(buf, path=None):
    """JPEG bytes -> ``EncodedJPEG`` when the device decodes it, else None (the image is left to PIL)."""
    n = len(buf)
    if n < 4 or buf[0] != 0xFF or buf[1] != 0xD8:
        return None
    pos, frame, q, h, ri, jfif, adobe = 2, None, {}, {}, 0, False, None
    while True:
        if pos + 4 > n or buf[pos] != 0xFF:
            return None
        m = buf[pos + 1]
        if m == 0xFF:                                  # fill byte
            pos += 1
            continue
        if m in (0x01, 0xD8, 0xD9) or 0xD0 <= m <= 0xD7:
            return None
        ln = (buf[pos + 2] << 8) | buf[pos + 3]
        if ln < 2 or pos + 2 + ln > n:
            return None
        seg = buf[pos + 4:pos + 2 + ln]
        if m == 0xE0 and len(seg) >= 14 and seg[:5] == b'JFIF\0':
            jfif = True
        elif m == 0xEE and len(seg) >= 12 and seg[:5] == b'Adobe':
            adobe = seg[11]
        elif m in (0xC0, 0xC1):
            if frame is not None or len(seg) < 6 or seg[0] != 8:
                return None
            H, W, nf = (seg[1] << 8) | seg[2], (seg[3] << 8) | seg[4], seg[5]
            if H == 0 or W == 0 or nf not in (1, 3) or len(seg) < 6 + 3 * nf:
                return None
            frame = (W, H, [(seg[6 + 3 * i], seg[7 + 3 * i] >> 4, seg[7 + 3 * i] & 15, seg[8 + 3 * i]) for i in range(nf)])
        elif m in _SOF_OTHER:
            return None
        elif m == 0xDB:
            i = 0
            while i < len(seg):
                pq, tq = seg[i] >> 4, seg[i] & 15
                k = 128 if pq else 64
                if pq > 1 or tq > 3 or i + 1 + k > len(seg):
                    return None
                vals = np.frombuffer(bytes(seg[i + 1:i + 1 + k]), '>u2' if pq else 'u1').astype(np.int32)
                if vals.max() > 32767:
                    return None
                tab = np.zeros(64, np.int32)
                tab[ZIGZAG] = vals
                q[tq] = tab
                i += 1 + k
        elif m == 0xC4:
            i = 0
            while i < len(seg):
                tc, th = seg[i] >> 4, seg[i] & 15
                if tc > 1 or th > 3 or i + 17 > len(seg):
                    return None
                bits = bytes(seg[i + 1:i + 17])
                total = sum(bits)
                vals = bytes(seg[i + 17:i + 17 + total])
                if total > 256 or len(vals) != total or not _huffman_ok(bits, vals, tc == 0):
                    return None
                h[(tc, th)] = (bits, vals)
                i += 17 + total
        elif m == 0xDD:
            if len(seg) < 2:
                return None
            ri = (seg[0] << 8) | seg[1]
        elif m == 0xDA:
            return _scan(buf, pos + 2 + ln, seg, frame, q, h, ri, jfif, adobe, path)
        pos += 2 + ln


def _scan(buf, start, sos, frame, q, h, ri, jfif, adobe, path):
    if frame is None or len(sos) < 1:
        return None
    W, H, comps = frame
    ns = sos[0]
    if ns != len(comps) or len(sos) < 4 + 2 * ns:
        return None
    sel = [(sos[1 + 2 * i], sos[2 + 2 * i] >> 4, sos[2 + 2 * i] & 15) for i in range(ns)]
    if [s[0] for s in sel] != [c[0] for c in comps] or tuple(sos[1 + 2 * ns:4 + 2 * ns]) != (0, 63, 0):
        return None
    if len(comps) == 3:
        ids = tuple(c[0] for c in comps)
        ycc = jfif or (adobe == 1 if adobe is not None else ids == (1, 2, 3))
        if not ycc or (comps[0][1], comps[0][2]) not in ((1, 1), (2, 1), (2, 2)) or \
                any((c[1], c[2]) != (1, 1) for c in comps[1:]):
            return None
        sampling = (comps[0][1], comps[0][2])
    else:
        sampling = (1, 1)
    use = []
    for (cid, hh, vv, tq), (_, td, ta) in zip(comps, sel):
        if tq not in q or (0, td) not in h or (1, ta) not in h:
            return None
        use.append((tq, td, ta))
    d = np.frombuffer(buf, np.uint8, offset=start)
    ff = np.flatnonzero(d[:-1] == 0xFF) if len(d) > 1 else np.zeros(0, np.int64)
    nxt = d[ff + 1]
    rst = (nxt >= 0xD0) & (nxt <= 0xD7)
    marker = (nxt != 0) & ~rst
    end = len(d)
    if marker.any():
        end = int(ff[np.argmax(marker)])
        after = end
        while after < len(d) and d[after] == 0xFF:
            after += 1
        if after >= len(d) or d[after] != 0xD9:          # another scan, DNL or anything but EOI: PIL decodes it
            return None
        inside = ff < end
        ff, nxt, rst = ff[inside], nxt[inside], rst[inside]
    elif len(d) and d[-1] == 0xFF:
        end = len(d) - 1
        inside = ff < end
        ff, nxt, rst = ff[inside], nxt[inside], rst[inside]
    keep = np.ones(end, bool)
    keep[ff[nxt == 0] + 1] = False
    r = ff[rst]
    if len(r) and (ri == 0 or not np.array_equal(nxt[rst] - 0xD0, np.arange(len(r)) % 8)):
        return None
    keep[r] = False
    keep[r + 1] = False
    kept_before = np.concatenate(([0], np.cumsum(keep)))
    segs = np.concatenate(([0], kept_before[r])).astype(np.int64)
    return EncodedJPEG(path, (W, H), len(comps), sampling, ri, use, q, h, d[:end][keep], segs)


def encoded_loader(path):
    """The loader of ``dataset.transformer.decode: cuda``: the file's bytes parsed down to the markers
    (``EncodedJPEG``) when the device decodes it, otherwise the PIL image ``default_loader`` gives.  Either has
    ``.size`` = (W, H), and PIL's decompression-bomb limit applies to both."""
    from PIL import Image
    with open(path, 'rb') as f:
        buf = f.read()
    enc = parse(buf, path)
    if enc is None:
        img = Image.open(path)
        return img.convert('RGB')
    Image._decompression_bomb_check(enc.size)
    return enc


_HTAB_CACHE = {}


def huffman_table(bits, vals):
    """One DHT (16 code-length counts, symbols) -> its device record (``HTAB_DTYPE``)."""
    key = bits + vals
    t = _HTAB_CACHE.get(key)
    if t is not None:
        return t
    t = np.zeros((), HTAB_DTYPE)
    t['maxcode'][:] = -1
    code = k = 0
    for length in range(1, 17):
        cnt = bits[length - 1]
        if cnt:
            t['valoffset'][length] = k - code
            t['maxcode'][length] = code + cnt - 1
            if length <= LOOKAHEAD_BITS:
                sh = LOOKAHEAD_BITS - length
                for c in range(cnt):
                    t['look'][(code + c) << sh:(code + c + 1) << sh] = (length << 8) | vals[k + c]
        code = (code + cnt) << 1
        k += cnt
    t['maxcode'][17] = 0x7FFFFFFF
    t['huffval'][:len(vals)] = np.frombuffer(vals, np.uint8)
    if len(_HTAB_CACHE) > 4096:
        _HTAB_CACHE.clear()
    _HTAB_CACHE[key] = t
    return t


class JpegBatch:
    """The encoded images of one packed batch in the device form the module docstring describes."""

    def __init__(self, scan, segs, header, qtabs, htabs, paths, blocks, plane_bytes):
        self.scan, self.segs, self.header, self.qtabs, self.htabs = scan, segs, header, qtabs, htabs
        self.paths, self.blocks, self.plane_bytes = list(paths), int(blocks), int(plane_bytes)

    def __len__(self):
        return self.header.shape[0]

    def tensors(self):
        return ('scan', 'segs', 'header', 'qtabs', 'htabs')

    def _map(self, fn):
        return JpegBatch(*[fn(getattr(self, k)) for k in self.tensors()], self.paths, self.blocks, self.plane_bytes)


def pack_encoded(encoded, indices):
    """``EncodedJPEG`` images (batch positions ``indices``) -> ``JpegBatch`` on the host; the pixel offsets are the
    caller's."""
    qkeys, hkeys, qlist, hlist = {}, {}, [], []

    def intern(keys, lst, key, make):
        if key not in keys:
            keys[key] = len(lst)
            lst.append(make())
        return keys[key]

    header = np.zeros((len(encoded), HEADER_COLS), np.int32)
    scans, segs = [], []
    scan_off = seg_off = blk = plane = 0
    for j, (e, n) in enumerate(zip(encoded, indices)):
        W, H = e.size
        hy, vy = e.sampling
        mx, my = -(-W // (8 * hy)), -(-H // (8 * vy))
        row = header[j]
        row[[H_IMG, H_W, H_H, H_NCOMP, H_HY, H_VY, H_MCUX, H_MCUY, H_RI]] = (n, W, H, e.ncomp, hy, vy, mx, my, e.restart)
        row[[H_SEG0, H_NSEG, H_BLK0, H_PLANE0]] = (seg_off, len(e.segs), blk, plane)
        for c, (tq, td, ta) in enumerate(e.comps):
            row[H_Q0 + c] = intern(qkeys, qlist, e.qtabs[tq].tobytes(), lambda: e.qtabs[tq])
            row[H_DC0 + c] = intern(hkeys, hlist, (0,) + e.htabs[(0, td)], lambda: huffman_table(*e.htabs[(0, td)]))
            row[H_AC0 + c] = intern(hkeys, hlist, (1,) + e.htabs[(1, ta)], lambda: huffman_table(*e.htabs[(1, ta)]))
        scans.append(e.scan)
        segs.append(e.segs + scan_off)
        scan_off += len(e.scan)
        seg_off += len(e.segs)
        blk += mx * my * (hy * vy + e.ncomp - 1)
        plane += mx * my * 64 * (hy * vy + e.ncomp - 1)
    if scan_off + 8 >= 2 ** 28:
        raise ValueError('pack: the scans of one batch must stay under 256 MB')
    scan = torch.zeros(scan_off + 8, dtype=torch.uint8)
    if scan_off:
        scan.numpy()[:scan_off] = np.concatenate(scans)
    seg = torch.from_numpy(np.concatenate(segs + [np.array([scan_off])]).astype(np.int32))
    htabs = torch.from_numpy(np.stack(hlist).view(np.uint8).reshape(len(hlist), HTAB_BYTES).copy())
    return JpegBatch(scan, seg, torch.from_numpy(header), torch.from_numpy(np.stack(qlist).astype(np.int32)), htabs,
                     [e.path for e in encoded], blk, plane)


def workspace_bytes(jb, chunk_bytes):
    return int(_lib.query('hk_jpeg_workspace_bytes', len(jb), jb.segs.shape[0] - 1, jb.scan.numel(), int(chunk_bytes)))


def _buffer(work, key, n, dtype, device):
    """A view of n elements of the grow-only buffer ``work[key]``."""
    t = work.get(key)
    if t is None or t.numel() < n:
        t = work[key] = torch.empty(max(n, 1), dtype=dtype, device=device)
    return t[:n]


def decode(jb, pixels, offsets, chunk_bytes=CHUNK_BYTES, work=None):
    """Decodes the device-side ``JpegBatch`` jb into ``pixels`` (uint8) at ``offsets`` (int64 per batch image) on the
    current stream: Huffman decode, IDCT, upsampling and colour conversion.  ``work`` is a dict of grow-only buffers
    (coefficients, planes, workspace, status) kept between calls.  -> int32 status [J] on the device: 0 when image j
    decoded, else a ``STATUS_MESSAGES`` code."""
    dev = pixels.device
    for t, name in ((jb.scan, 'scan'), (jb.segs, 'segs'), (jb.header, 'header'), (jb.qtabs, 'qtabs'),
                    (jb.htabs, 'htabs'), (pixels, 'pixels'), (offsets, 'offsets')):
        if not t.is_cuda or not t.is_contiguous():
            raise _lib.HawkeyeLibError(f'jpeg decode: {name} must be a contiguous CUDA tensor')
    work = {} if work is None else work
    J, stream = len(jb), _lib.stream_ptr()
    coef = _buffer(work, 'coef', jb.blocks * 64, torch.int16, dev)
    planes = _buffer(work, 'planes', jb.plane_bytes, torch.uint8, dev)
    ws_bytes = workspace_bytes(jb, chunk_bytes)
    ws = _buffer(work, 'workspace', ws_bytes, torch.uint8, dev)
    status = _buffer(work, 'status', J, torch.int32, dev)
    _lib.call('hk_jpeg_huffman', jb.scan, jb.segs, jb.header, jb.htabs, coef, status, J, jb.segs.shape[0] - 1,
              jb.scan.numel(), int(chunk_bytes), ws, ws_bytes, stream)
    _lib.call('hk_jpeg_idct', coef, jb.header, jb.qtabs, planes, J, stream)
    _lib.call('hk_jpeg_color', planes, jb.header, offsets, pixels, J, stream)
    return status


def raise_on_status(status, paths):
    """Raises naming the first file whose status word (a host int32 array) is nonzero."""
    bad = np.flatnonzero(np.asarray(status))
    if len(bad):
        j = int(bad[0])
        code = int(status[j])
        raise RuntimeError(f'JPEG decode failed for {paths[j]}: {STATUS_MESSAGES.get(code, f"status {code}")}'
                           + (f' (and {len(bad) - 1} more images of the batch)' if len(bad) > 1 else ''))


def decode_setting(config):
    """'cuda' when a ``dataset.transformer`` config sets ``decode: cuda``, None when it has no ``decode`` key.  The key
    needs ``device: cuda``: the decoded images go straight to the device presets."""
    dec = config['decode'] if 'decode' in config else None
    if dec is None:
        return None
    if dec != 'cuda':
        raise ValueError(f"dataset.transformer.decode must be 'cuda' or absent, not {dec!r}")
    dev = config['device'] if 'device' in config else None
    if dev != 'cuda':
        raise ValueError("dataset.transformer.decode: cuda needs dataset.transformer.device: cuda")
    return dec


__all__ = ['EncodedJPEG', 'JpegBatch', 'encoded_loader', 'parse', 'pack_encoded', 'decode', 'raise_on_status',
           'decode_setting', 'CHUNK_BYTES']
