"""The host side of the device JPEG decode (hawkeye_b200.ops_jpeg): the restatement in tests/jpeg_ref.py against PIL
bit for bit, the marker parse's classification and its unstuffing, the draws of the device presets on encoded images,
packed batches that mix encoded and pixel images, the ``dataset.transformer.decode`` key and the C-ABI error paths."""
import os

import numpy as np
import pytest
import torch
from PIL import Image

import jpeg_ref as R
from hawkeye_b200 import data, ops_augment as A, ops_jpeg as J, train

MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


@pytest.fixture(scope='module')
def cases(tmp_path_factory):
    return R.write_cases(str(tmp_path_factory.mktemp('jpeg')), dict(R.CLASSES, **R.FALLBACKS))


def _supported(cases):
    return [(n, p) for n, p in cases if not any(n.startswith(f) for f in R.FALLBACKS)]


def test_restatement_is_pil_bit_for_bit(cases):
    """Every sampling mode, grey, qualities 10 / 75 / 100, optimised tables, restarts every block and every MCU row, at
    1x1, 7x9, 17x33 and sizes that are not multiples of 8 or 16."""
    for name, path in _supported(cases):
        got = R.decode(open(path, 'rb').read())[0]
        assert np.array_equal(got, np.asarray(Image.open(path).convert('RGB'))), name


def test_parse_classifies_every_case(cases, tmp_path):
    for name, path in cases:
        img = data.encoded_loader(path)
        fallback = any(name.startswith(f) for f in R.FALLBACKS)
        assert isinstance(img, Image.Image) == fallback, name
        if fallback:
            assert np.array_equal(np.asarray(img), np.asarray(Image.open(path).convert('RGB')))
        else:
            assert img.size == Image.open(path).size and img.path == path
    buf = open(dict(cases)['420_45x37'], 'rb').read()
    assert isinstance(J.parse(buf[:len(buf) // 2]), J.EncodedJPEG)      # cut in the scan: the device reports it
    assert J.parse(buf[:200]) is None and J.parse(b'\xff\xd8') is None and J.parse(b'GIF89a') is None
    sof = buf.index(b'\xff\xc0')
    assert J.parse(buf[:sof + 4] + b'\x0c' + buf[sof + 5:]) is None      # 12-bit samples
    assert J.parse(buf[:sof + 1] + b'\xc9' + buf[sof + 2:]) is None      # arithmetic coding
    eoi = buf.rindex(b'\xff\xd9')
    assert J.parse(buf[:eoi] + b'\xff\xdc\x00\x04\x00\x25' + buf[eoi:]) is None      # DNL after the scan


def test_unstuffing_and_restart_segments(cases):
    """Re-stuffing the unstuffed scan and putting the RSTn markers back at the segment offsets gives the file's scan
    bytes, and there is one segment per restart interval."""
    for name, path in _supported(cases):
        buf = open(path, 'rb').read()
        e = J.parse(buf, path)
        W, H = e.size
        hy, vy = e.sampling
        mcus = -(-W // (8 * hy)) * -(-H // (8 * vy))
        assert len(e.segs) == (-(-mcus // e.restart) if e.restart else 1), name
        out = bytearray()
        ends = list(e.segs[1:]) + [len(e.scan)]
        for k, (a, b) in enumerate(zip(e.segs, ends)):
            if k:
                out += bytes([0xFF, 0xD0 + (k - 1) % 8])
            out += bytes(e.scan[a:b]).replace(b'\xff', b'\xff\x00')
        start = buf.index(b'\xff\xda')
        start += 2 + int.from_bytes(buf[start + 2:start + 4], 'big')
        assert buf[start:start + len(out)] == bytes(out) and buf[start + len(out):start + len(out) + 2] == b'\xff\xd9'


def test_huffman_lookahead_agrees_with_the_canonical_code(cases):
    e = J.parse(open(dict(cases)['optimize_61x23'], 'rb').read())
    for (tc, th), (bits, vals) in e.htabs.items():
        t = J.huffman_table(bits, vals)
        for (length, code), sym in R._code_table(list(bits), list(vals)).items():
            if length <= J.LOOKAHEAD_BITS:
                sh = J.LOOKAHEAD_BITS - length
                assert (t['look'][code << sh:(code + 1) << sh] == (length << 8) | sym).all()
            assert code <= t['maxcode'][length] and t['huffval'][code + t['valoffset'][length]] == sym


def test_decompression_bomb_limit(cases, monkeypatch):
    monkeypatch.setattr(Image, 'MAX_IMAGE_PIXELS', 100)
    with pytest.raises(Image.DecompressionBombError):
        data.encoded_loader(dict(cases)['420_45x37'])


def test_draws_from_the_encoded_image_equal_the_pil_draws(cases):
    train_p = data.DevicePresetTrain(224, auto_augment_policy='ta_wide', random_erase_prob=0.5)
    eval_p = data.DevicePresetEval(224, resize_size=256)
    for name, path in _supported(cases):
        for preset in (train_p, eval_p):
            for seed in range(3):
                torch.manual_seed(seed)
                a, ra = preset(data.default_loader(path))
                sa = torch.get_rng_state()
                torch.manual_seed(seed)
                e, re = preset(data.encoded_loader(path))
                assert isinstance(e, J.EncodedJPEG) and np.array_equal(ra, re), name
                assert torch.equal(sa, torch.get_rng_state())


def test_pack_mixed_batches(cases):
    paths = [dict(cases)[n] for n in ('420_45x37', 'progressive_17x33', 'grey_rst_61x23', 'cmyk_7x9', '444_1x1',
                                      'optimize_45x37')]
    preset = data.DevicePresetEval(32, resize_size=40)
    items = [{'img': preset(data.encoded_loader(p)), 'label': i} for i, p in enumerate(paths)]
    batch = preset.collate(items)
    p = batch['img']
    enc = [isinstance(it['img'][0], J.EncodedJPEG) for it in items]
    assert enc == [True, False, True, False, True, True] and len(p.jpeg) == 4
    sizes = np.array([Image.open(q).size[::-1] for q in paths])
    assert np.array_equal(p.sizes.numpy(), sizes)
    nbytes = sizes.prod(1) * 3
    assert p.data.numel() == nbytes[~np.array(enc)].sum() and p.pixel_bytes == nbytes.sum()
    order = [1, 3, 0, 2, 4, 5]                          # pixel images first, encoded ones after
    assert np.array_equal(p.offsets.numpy()[order], np.concatenate(([0], np.cumsum(nbytes[order])[:-1])))
    off = p.offsets.numpy()
    for i in (1, 3):
        px = np.asarray(Image.open(paths[i]).convert('RGB')).reshape(-1)
        assert np.array_equal(p.data.numpy()[off[i]:off[i] + px.size], px)
    h = p.jpeg.header.numpy()
    assert list(h[:, J.H_IMG]) == [0, 2, 4, 5] and list(h[:, J.H_NCOMP]) == [3, 1, 3, 3]
    assert p.jpeg.paths == [paths[i] for i in (0, 2, 4, 5)]
    assert p.jpeg.htabs.shape[1] == J.HTAB_BYTES and p.jpeg.segs[-1] == p.jpeg.scan.numel() - 8
    assert len(p.jpeg.qtabs) < 4 * 3 and len(p.jpeg.htabs) < 4 * 6          # shared tables are stored once
    moved = p.to('cpu')
    assert moved.jpeg.paths == p.jpeg.paths and moved.pixel_bytes == p.pixel_bytes
    plain = preset.collate([{'img': preset(data.default_loader(q)), 'label': i} for i, q in enumerate(paths)])['img']
    assert plain.jpeg is None and plain.pixel_bytes == plain.data.numel() == nbytes.sum()


def test_decode_key_validation():
    from hawkeye_b200.cfgnode import CfgNode
    assert train.transformer_decode(CfgNode(dict(device='cuda'))) is None
    assert train.transformer_decode(CfgNode(dict(device='cuda', decode='cuda'))) == 'cuda'
    for bad in (dict(decode='cuda'), dict(device='cuda', decode='cpu'), dict(device='cuda', decode=True)):
        with pytest.raises(ValueError):
            train.transformer_device(CfgNode(bad))
    with pytest.raises(ValueError, match='decode: cuda'):
        train.device_collate(CfgNode(dict(device='cuda', decode='cuda')), {'train': object(), 'val': object()}, 'DCL')
    assert train.dataset_loader(CfgNode(dict(device='cuda', decode='cuda'))) is data.encoded_loader
    assert train.dataset_loader(CfgNode(dict(device='cuda'))) is data.default_loader


FAKE = 0x10000


def test_cabi_errors_launch_nothing():
    import __graft_entry__ as g
    g.build()
    from hawkeye_b200 import _lib
    lib = _lib.lib()
    assert lib.hk_jpeg_header_cols() == J.HEADER_COLS
    assert lib.hk_jpeg_workspace_bytes(2, 2, 1000, 64) > 0
    for args in ((0, 2, 1000, 64), (2, 1, 1000, 64), (2, 2, -1, 64), (2, 2, 1000, 0)):
        assert lib.hk_jpeg_workspace_bytes(*args) == 0
    lib.hk_reset_launch_count()
    hf = lib.hk_jpeg_huffman
    ok = [FAKE] * 6 + [2, 2, 1000, 64, FAKE, 1 << 20, None]
    for i in range(6):
        bad = list(ok)
        bad[i] = None
        assert hf(*bad) == -1 and 'null' in lib.hk_last_error().decode()
    for i, v in ((6, 0), (7, 1), (8, 8), (8, 1 << 28), (9, 0)):
        bad = list(ok)
        bad[i] = v
        assert hf(*bad) == -1
    assert hf(*(ok[:11] + [16, None])) != 0 and 'workspace' in lib.hk_last_error().decode()
    assert hf(*([FAKE + 1] + ok[1:])) != 0
    assert lib.hk_jpeg_idct(None, FAKE, FAKE, FAKE, 2, None) == -1
    assert lib.hk_jpeg_idct(FAKE, FAKE, FAKE, FAKE, 0, None) == -1
    assert lib.hk_jpeg_color(FAKE, FAKE, None, FAKE, 2, None) == -1
    assert lib.hk_jpeg_color(FAKE, FAKE, FAKE, FAKE, 0, None) == -1
    assert lib.hk_launch_count() == 0
