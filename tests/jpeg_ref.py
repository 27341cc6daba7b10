"""A plain restatement of the baseline JPEG decode PIL does through libjpeg-turbo, in numpy and Python: the marker parse,
a sequential Huffman decode straight from the stuffed scan, jpeg_idct_islow (jidctint.c) with its range limiting, the
fancy upsampling of jdsample.c (h2v1, h2v2) and the YCbCr -> RGB table arithmetic of jdcolor.c.  It is the oracle of
the device decoder's intermediate stages (coefficients, component planes) and of its pixels.  Slow: small images only.

Supports what the device decodes (SOF0 / SOF1, 8-bit, Huffman, one interleaved scan, DRI, grey or YCbCr with luma
sampling 1x1, 2x1 or 2x2 and 1x1 chroma); anything else raises ValueError.
"""
import numpy as np

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,
                   7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31,
                   39, 46, 53, 60, 61, 54, 47, 55, 62, 63])     # zig-zag index -> natural (row-major) index


def parse(buf):
    """-> dict of the frame, tables, restart interval and the stuffed scan bytes (from after SOS to the next non-RST
    marker)."""
    if buf[:2] != b'\xff\xd8':
        raise ValueError('not a JPEG')
    pos, q, h, out = 2, {}, {}, dict(ri=0)
    while True:
        while buf[pos] == 0xFF and buf[pos + 1] == 0xFF:
            pos += 1
        if buf[pos] != 0xFF:
            raise ValueError('marker expected')
        m = buf[pos + 1]
        ln = int.from_bytes(buf[pos + 2:pos + 4], 'big')
        seg = buf[pos + 4:pos + 2 + ln]
        if m in (0xC0, 0xC1):
            if seg[0] != 8:
                raise ValueError('not 8-bit')
            out['H'], out['W'], nf = int.from_bytes(seg[1:3], 'big'), int.from_bytes(seg[3:5], 'big'), seg[5]
            out['comps'] = [(seg[6 + 3 * i], seg[7 + 3 * i] >> 4, seg[7 + 3 * i] & 15, seg[8 + 3 * i]) for i in range(nf)]
        elif 0xC2 <= m <= 0xCF and m not in (0xC4, 0xC8, 0xCC):
            raise ValueError('not a baseline / extended sequential Huffman frame')
        elif m == 0xDB:
            i = 0
            while i < len(seg):
                pq, tq = seg[i] >> 4, seg[i] & 15
                n = 128 if pq else 64
                vals = np.frombuffer(bytes(seg[i + 1:i + 1 + n]), '>u2' if pq else 'u1').astype(np.int64)
                tab = np.zeros(64, np.int64)
                tab[ZIGZAG] = vals
                q[tq] = tab
                i += 1 + n
        elif m == 0xC4:
            i = 0
            while i < len(seg):
                tc, th = seg[i] >> 4, seg[i] & 15
                bits = list(seg[i + 1:i + 17])
                vals = list(seg[i + 17:i + 17 + sum(bits)])
                h[(tc, th)] = _code_table(bits, vals)
                i += 17 + sum(bits)
        elif m == 0xDD:
            out['ri'] = int.from_bytes(seg[0:2], 'big')
        elif m == 0xDA:
            ns = seg[0]
            out['scan'] = [(seg[1 + 2 * i], seg[2 + 2 * i] >> 4, seg[2 + 2 * i] & 15) for i in range(ns)]
            start = pos + 2 + ln
            out['q'], out['h'] = q, h
            out['data'] = (buf, start)
            return out
        elif m in (0xD9,):
            raise ValueError('no scan')
        pos += 2 + ln


def _code_table(bits, vals):
    """{(length, code): symbol} of a DHT's canonical code."""
    table, code, k = {}, 0, 0
    for length in range(1, 17):
        for _ in range(bits[length - 1]):
            table[(length, code)] = vals[k]
            code += 1
            k += 1
        code <<= 1
    return table


class _Bits:
    """MSB-first reader of the entropy-coded data: drops the 0x00 after each 0xFF, stops at a marker."""

    def __init__(self, buf, pos):
        self.buf, self.pos, self.acc, self.n = buf, pos, 0, 0

    def _fill(self):
        b = self.buf[self.pos] if self.pos < len(self.buf) else None
        if b is None:
            raise ValueError('stream ends early')
        if b == 0xFF:
            nxt = self.buf[self.pos + 1]
            if nxt != 0:
                raise ValueError('stream ends early (marker inside the data)')
            self.pos += 2
        else:
            self.pos += 1
        self.acc = (self.acc << 8) | b
        self.n += 8

    def get(self, k):
        while self.n < k:
            self._fill()
        self.n -= k
        v = (self.acc >> self.n) & ((1 << k) - 1)
        self.acc &= (1 << self.n) - 1
        return v

    def restart(self, expect):
        """Drop the buffered bits and read the RST marker ``0xFFD0 + expect``."""
        self.acc = self.n = 0
        if self.buf[self.pos] != 0xFF or self.buf[self.pos + 1] != 0xD0 + expect:
            raise ValueError('restart marker missing')
        self.pos += 2


def _symbol(bits, table):
    code = 0
    for length in range(1, 17):
        code = (code << 1) | bits.get(1)
        s = table.get((length, code))
        if s is not None:
            return s
    raise ValueError('invalid Huffman code')


def _extend(v, s):
    return v - (1 << s) + 1 if s and v < (1 << (s - 1)) else v


def layout(f):
    """-> (blocks per MCU as [(component, row, col)], MCUs across, MCUs down, luma h, luma v)."""
    comps = f['comps']
    hy, vy = comps[0][1], comps[0][2]
    if len(comps) == 1:
        hy = vy = 1
    mcu = [(0, r, c) for r in range(vy) for c in range(hy)] + [(i, 0, 0) for i in range(1, len(comps))]
    return mcu, -(-f['W'] // (8 * hy)), -(-f['H'] // (8 * vy)), hy, vy


def coefficients(f):
    """-> one int64 array [rows of blocks, cols of blocks, 64] (natural order, DC absolute) per component, in the layout
    of the whole MCUs."""
    comps = f['comps']
    if [c[0] for c in f['scan']] != [c[0] for c in comps]:
        raise ValueError('not one interleaved scan of every component in frame order')
    mcu, mx, my, hy, vy = layout(f)
    blocks = [np.zeros((my * (vy if i == 0 else 1), mx * (hy if i == 0 else 1), 64), np.int64) for i in range(len(comps))]
    dc_tab = [f['h'][(0, f['scan'][i][1])] for i in range(len(comps))]
    ac_tab = [f['h'][(1, f['scan'][i][2])] for i in range(len(comps))]
    bits = _Bits(*f['data'])
    pred = [0] * len(comps)
    ri, rst = f['ri'], 0
    for m in range(mx * my):
        if ri and m and m % ri == 0:
            bits.restart(rst)
            rst = (rst + 1) & 7
            pred = [0] * len(comps)
        mr, mc = divmod(m, mx)
        for ci, r, c in mcu:
            hh, vv = (hy, vy) if ci == 0 else (1, 1)
            blk = blocks[ci][mr * vv + r, mc * hh + c]
            s = _symbol(bits, dc_tab[ci])
            pred[ci] += _extend(bits.get(s), s)
            blk[0] = np.int16(pred[ci])
            k = 1
            while k < 64:
                rs = _symbol(bits, ac_tab[ci])
                r_, s = rs >> 4, rs & 15
                if s:
                    k += r_
                    if k > 63:
                        raise ValueError('coefficient index beyond 63')
                    blk[ZIGZAG[k]] = _extend(bits.get(s), s)
                    k += 1
                elif r_ == 15:
                    k += 16
                else:
                    break
    return blocks


CONST_BITS, PASS1_BITS = 13, 2
F = dict(f0298=2446, f0390=3196, f0541=4433, f0765=6270, f0899=7373, f1175=9633, f1501=12299, f1847=15137, f1961=16069,
         f2053=16819, f2562=20995, f3072=25172)


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _idct_1d(c0, c1, c2, c3, c4, c5, c6, c7):
    """jidctint.c's even / odd parts on int64 arrays -> the eight outputs before descaling."""
    z1 = (c2 + c6) * F['f0541']
    tmp2 = z1 + c6 * -F['f1847']
    tmp3 = z1 + c2 * F['f0765']
    tmp0 = (c0 + c4) << CONST_BITS
    tmp1 = (c0 - c4) << CONST_BITS
    t10, t13, t11, t12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    t0, t1, t2, t3 = c7, c5, c3, c1
    z1, z2, z3, z4 = t0 + t3, t1 + t2, t0 + t2, t1 + t3
    z5 = (z3 + z4) * F['f1175']
    t0, t1, t2, t3 = t0 * F['f0298'], t1 * F['f2053'], t2 * F['f3072'], t3 * F['f1501']
    z1, z2, z3, z4 = z1 * -F['f0899'], z2 * -F['f2562'], z3 * -F['f1961'], z4 * -F['f0390']
    z3 = z3 + z5
    z4 = z4 + z5
    t0, t1, t2, t3 = t0 + z1 + z3, t1 + z2 + z4, t2 + z2 + z3, t3 + z1 + z4
    return [t10 + t3, t11 + t2, t12 + t1, t13 + t0, t13 - t0, t12 - t1, t11 - t2, t10 - t3]


def idct_islow(coef, qtab):
    """jpeg_idct_islow of blocks [..., 64] (natural order) with quant table [64] -> uint8 [..., 8, 8]."""
    d = (coef.astype(np.int64) * qtab.astype(np.int64)).reshape(coef.shape[:-1] + (8, 8))
    cols = _idct_1d(*[d[..., u, :] for u in range(8)])                # pass 1 over columns: row u of coefficients
    ws = np.stack([_descale(c, CONST_BITS - PASS1_BITS) for c in cols], -2)     # [..., 8 (y), 8 (x freq)]
    rows = _idct_1d(*[ws[..., :, v] for v in range(8)])
    out = np.stack([_descale(r, CONST_BITS + PASS1_BITS + 3) for r in rows], -1)
    return np.clip((((out + 512) & 1023) - 512) + 128, 0, 255).astype(np.uint8)


def planes(f, blocks):
    """-> the uint8 component planes at whole-MCU size."""
    out = []
    for ci, b in enumerate(blocks):
        px = idct_islow(b, f['q'][f['comps'][ci][3]])                # [by, bx, 8, 8]
        out.append(px.transpose(0, 2, 1, 3).reshape(b.shape[0] * 8, b.shape[1] * 8))
    return out


def _h2v1(c, dw):
    c = c[:, :dw].astype(np.int64)
    out = np.empty((c.shape[0], 2 * dw), np.int64)
    if dw <= 2:
        return np.repeat(c, 2, axis=1)
    left = np.concatenate([c[:, :1], c[:, :-1]], 1)
    right = np.concatenate([c[:, 1:], c[:, -1:]], 1)
    out[:, 0::2] = (3 * c + left + 1) >> 2
    out[:, 1::2] = (3 * c + right + 2) >> 2
    out[:, 0], out[:, -1] = c[:, 0], c[:, -1]
    return out


def _h2v2(c, dw, dh):
    c = c[:dh, :dw].astype(np.int64)
    if dw <= 2:
        return np.repeat(np.repeat(c, 2, axis=0), 2, axis=1)
    above = np.concatenate([c[:1], c[:-1]], 0)
    below = np.concatenate([c[1:], c[-1:]], 0)
    out = np.empty((2 * dh, 2 * dw), np.int64)
    for v, far in ((0, above), (1, below)):
        cs = 3 * c + far
        left = np.concatenate([cs[:, :1], cs[:, :-1]], 1)
        right = np.concatenate([cs[:, 1:], cs[:, -1:]], 1)
        row = np.empty((dh, 2 * dw), np.int64)
        row[:, 0::2] = (3 * cs + left + 8) >> 4
        row[:, 1::2] = (3 * cs + right + 7) >> 4
        row[:, 0] = (cs[:, 0] * 4 + 8) >> 4
        row[:, -1] = (cs[:, -1] * 4 + 7) >> 4
        out[v::2] = row
    return out


def _fix(x):
    return int(x * 65536 + 0.5)


def to_rgb(f, pl):
    """Component planes -> uint8 [H, W, 3] as PIL's ``convert('RGB')`` gives it."""
    W, H = f['W'], f['H']
    y = pl[0][:H, :W].astype(np.int64)
    if len(pl) == 1:
        return np.repeat(y[..., None].astype(np.uint8), 3, axis=2)
    _, _, _, hy, vy = layout(f)
    dw, dh = -(-W // hy), -(-H // vy)
    up = []
    for c in pl[1:]:
        if hy == 1:
            u = c[:H, :W].astype(np.int64)
        elif vy == 1:
            u = _h2v1(c[:H], dw)
        else:
            u = _h2v2(c, dw, dh)
        up.append(u[:H, :W] - 128)
    cb, cr = up
    r = y + ((_fix(1.40200) * cr + 32768) >> 16)
    g = y + ((-_fix(0.34414) * cb + 32768 - _fix(0.71414) * cr) >> 16)
    b = y + ((_fix(1.77200) * cb + 32768) >> 16)
    return np.clip(np.stack([r, g, b], -1), 0, 255).astype(np.uint8)


def decode(buf):
    """JPEG bytes -> (uint8 [H, W, 3], frame dict, coefficient blocks, planes)."""
    f = parse(bytes(buf))
    blocks = coefficients(f)
    pl = planes(f, blocks)
    return to_rgb(f, pl), f, blocks, pl


# ------------------------------------------------------------------------------------------------- seeded test images
SIZES = [(1, 1), (7, 9), (17, 33), (45, 37), (61, 23)]
# Pillow save options of each supported class: every sampling, grey, qualities 10 / 75 / 100, optimised tables and
# restart intervals of one block and of one MCU row
CLASSES = {'444': dict(subsampling=0), '422': dict(subsampling=1), '420': dict(subsampling=2),
           'grey': dict(mode='L'), 'q10': dict(quality=10), 'q100': dict(quality=100, subsampling=1),
           'optimize': dict(optimize=True), 'rst_block': dict(restart_marker_blocks=1),
           'rst_row': dict(restart_marker_rows=1, subsampling=1), 'grey_rst': dict(mode='L', restart_marker_blocks=1)}
# what PIL writes that the device leaves to PIL
FALLBACKS = {'progressive': dict(progressive=True), 'cmyk': dict(mode='CMYK'), 'rgb_adobe': dict(keep_rgb=True),
             'png': dict(format='PNG')}


def random_image(w, h, seed):
    """A smooth random field with noise on top, uint8 [h, w, 3]."""
    r = np.random.RandomState(seed)
    from PIL import Image
    base = Image.fromarray(r.randint(0, 256, (max(h // 8, 2), max(w // 8, 2), 3)).astype(np.uint8))
    arr = np.asarray(base.resize((w, h), Image.BICUBIC)).astype(np.int32) + r.randint(-40, 41, (h, w, 3))
    return np.clip(arr, 0, 255).astype(np.uint8)


def write(path, w, h, seed, options):
    """Saves a seeded image with Pillow's save ``options`` (plus 'mode' and 'format'); -> path."""
    from PIL import Image
    opts = dict(options)
    mode, fmt = opts.pop('mode', 'RGB'), opts.pop('format', 'JPEG')
    im = Image.fromarray(random_image(w, h, seed))
    if mode != 'RGB':
        im = im.convert(mode)
    im.save(path, fmt, quality=opts.pop('quality', 75), **opts) if fmt == 'JPEG' else im.save(path, fmt)
    return path


def write_cases(root, classes=CLASSES, sizes=SIZES):
    """Every class at every size under ``root`` -> [(name, path)]."""
    import os
    out = []
    for c, opts in classes.items():
        for w, h in sizes:
            name = f'{c}_{w}x{h}'
            out.append((name, write(os.path.join(root, name + ('.png' if opts.get('format') == 'PNG' else '.jpg')), w, h,
                                    w * 1000 + h, opts)))
    return out
