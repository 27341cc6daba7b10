"""The JPEG decode on the device (hawkeye_b200.ops_jpeg, csrc/jpeg.cu) against PIL and the host restatement in
tests/jpeg_ref.py: pixels bit for bit over every supported class at several chunk sizes, coefficients and planes, mixed
batches with the key on and off, corrupt streams, a BCNN train step and the Tester fed by encoded images."""
import contextlib
import os

import numpy as np
import pytest
import torch
from PIL import Image

import bench_input
import detgen
import jpeg_ref as R
from hawkeye_b200 import data, ops_augment as A, ops_jpeg as J
from kernel_check import Out, abi
from step_check import no_host_sync

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


@pytest.fixture(scope='module')
def small(tmp_path_factory):
    return R.write_cases(str(tmp_path_factory.mktemp('small')))


@pytest.fixture(scope='module')
def cub(tmp_path_factory):
    root = str(tmp_path_factory.mktemp('cub'))
    bench_input.make_jpegs(root, 8)
    return [os.path.join(root, f'{i}.jpg') for i in range(8)]


def decode_paths(paths, chunk, work=None):
    """-> (decoded uint8 HWC images, status) of the files, all encoded, in one batch."""
    enc = [data.encoded_loader(p) for p in paths]
    assert all(isinstance(e, J.EncodedJPEG) for e in enc)
    p = A.pack(enc, [A.param_row((0, 0) + e.size, (8, 8)) for e in enc], 8, MEAN, STD).to('cuda')
    pixels = torch.zeros(p.pixel_bytes, dtype=torch.uint8, device='cuda')
    status = J.decode(p.jpeg, pixels, p.offsets, chunk_bytes=chunk, work=work)
    px, off = pixels.cpu().numpy(), p.offsets.cpu().numpy()
    return [px[o:o + e.size[0] * e.size[1] * 3].reshape(e.size[1], e.size[0], 3) for e, o in zip(enc, off)], \
        status.cpu().numpy()


def test_pixels_are_pil_bit_for_bit(small, cub):
    """Every supported class at every small size, and CUB-sized images, at chunk sizes from one byte (long
    synchronisation chains) to larger than any scan."""
    for paths, chunks in (([p for _, p in small], (1, 3, 64, J.CHUNK_BYTES, 1 << 16)),
                          (cub, (7, 64, J.CHUNK_BYTES, 1024, 1 << 20))):
        refs = [np.asarray(Image.open(p).convert('RGB')) for p in paths]
        for chunk in chunks:
            got, status = decode_paths(paths, chunk)
            assert not status.any(), (chunk, status)
            bad = [os.path.basename(p) for p, g, r in zip(paths, got, refs) if not np.array_equal(g, r)]
            assert not bad, (chunk, bad)


def test_coefficients_and_planes_equal_the_restatement(small):
    for name, path in small:
        buf = open(path, 'rb').read()
        _, f, blocks, planes = R.decode(buf)
        work = {}
        got, status = decode_paths([path], 5, work)
        assert status[0] == 0
        mcu, mx, my, hy, vy = R.layout(f)
        want = []
        for m in range(mx * my):
            mr, mc = divmod(m, mx)
            for ci, r, c in mcu:
                hh, vv = (hy, vy) if ci == 0 else (1, 1)
                want.append(blocks[ci][mr * vv + r, mc * hh + c])
        coef = work['coef'].cpu().numpy().reshape(-1, 64)
        assert np.array_equal(coef, np.array(want, np.int16)), name
        flat = work['planes'].cpu().numpy()
        off = 0
        for pl in planes:
            assert np.array_equal(flat[off:off + pl.size].reshape(pl.shape), pl), name
            off += pl.size


def _mixed_items(paths, preset, decode, seed):
    items = []
    for k, p in enumerate(paths):
        torch.manual_seed(seed + k)
        img = data.encoded_loader(p) if decode else data.default_loader(p)
        items.append({'img': preset(img), 'label': k})
    return preset.collate(items)['img']


def test_mixed_batches_equal_with_the_key_on_and_off(tmp_path, cub):
    """Supported, progressive, CMYK and PNG images in one batch: the fp32 model input is identical with and without
    the device decode, for the train and the eval preset."""
    paths = cub[:3]
    for name, opts in list(R.FALLBACKS.items()) + [('420', R.CLASSES['420']), ('rst', R.CLASSES['rst_row'])]:
        paths.append(R.write(str(tmp_path / f'{name}.{"png" if name == "png" else "jpg"}'), 300, 200, 5, opts))
    enc = [data.encoded_loader(p) for p in paths]
    assert sum(isinstance(e, J.EncodedJPEG) for e in enc) == 5
    for preset in (data.DevicePresetTrain(224, auto_augment_policy='ta_wide', random_erase_prob=0.1),
                   data.DevicePresetEval(224, resize_size=256)):
        on = _mixed_items(paths, preset, True, 11)
        off = _mixed_items(paths, preset, False, 11)
        assert on.jpeg is not None and off.jpeg is None and torch.equal(on.params, off.params)
        assert torch.equal(on.to('cuda').images(), off.to('cuda').images())


def _corrupt(tmp_path, cub):
    """-> {kind: path}: a file cut in its scan, and one with 48 one-bits (no valid code) in the middle of its scan."""
    buf = open(cub[0], 'rb').read()
    sos = buf.index(b'\xff\xda')
    cut = tmp_path / 'truncated.jpg'
    cut.write_bytes(buf[:sos + (len(buf) - sos) // 2])
    mid = sos + (len(buf) - sos) // 2
    while buf[mid - 1] == 0xFF:
        mid += 1
    bad = tmp_path / 'bad_code.jpg'
    bad.write_bytes(buf[:mid] + b'\xff\x00' * 6 + buf[mid + 6:])
    return {'truncated': str(cut), 'bad_code': str(bad)}


def test_corrupt_streams_give_a_status(tmp_path, cub):
    files = _corrupt(tmp_path, cub)
    _, status = decode_paths([cub[1], files['truncated'], cub[2], files['bad_code']], J.CHUNK_BYTES)
    assert status[0] == 0 and status[2] == 0 and status[1] != 0 and status[3] == 1, status
    enc = [data.encoded_loader(p) for p in (cub[1], files['bad_code'])]
    p = A.pack(enc, [A.param_row((0, 0) + e.size, (8, 8)) for e in enc], 8, MEAN, STD).to('cuda')
    with pytest.raises(RuntimeError, match='bad_code.jpg'):
        p.images()


def test_guarded_outputs_and_argument_errors(cub):
    """The IDCT and colour launches write their outputs and nothing around them; bad arguments launch nothing."""
    from hawkeye_b200 import _lib
    enc = [data.encoded_loader(p) for p in cub[:2]]
    p = A.pack(enc, [A.param_row((0, 0) + e.size, (8, 8)) for e in enc], 8, MEAN, STD).to('cuda')
    jb, work = p.jpeg, {}
    pixels = torch.zeros(p.pixel_bytes, dtype=torch.uint8, device='cuda')
    J.decode(jb, pixels, p.offsets, work=work)
    (planes,) = abi('hk_jpeg_idct', work['coef'], jb.header, jb.qtabs, Out((jb.plane_bytes,), torch.uint8), len(jb),
                    inputs=(work['coef'], jb.header, jb.qtabs))
    assert torch.equal(planes, work['planes'])
    (px,) = abi('hk_jpeg_color', planes, jb.header, p.offsets, Out((p.pixel_bytes,), torch.uint8), len(jb),
                inputs=(planes,))
    assert torch.equal(px, pixels)
    lib = _lib.lib()
    lib.hk_reset_launch_count()
    ws = work['workspace']
    args = [jb.scan, jb.segs, jb.header, jb.htabs, work['coef'], work['status'], 2, jb.segs.numel() - 1, jb.scan.numel(),
            64, ws, ws.numel(), None]
    for i in range(6):
        bad = list(args)
        bad[i] = None
        with pytest.raises(_lib.HawkeyeLibError, match='null'):
            _lib.call('hk_jpeg_huffman', *bad)
    for i, v in ((6, 0), (7, 1), (8, 4), (9, 0)):
        bad = list(args)
        bad[i] = v
        with pytest.raises(_lib.HawkeyeLibError):
            _lib.call('hk_jpeg_huffman', *bad)
    with pytest.raises(_lib.HawkeyeLibError, match='workspace'):
        _lib.call('hk_jpeg_huffman', *args[:10], ws, 16, None)
    with pytest.raises(_lib.HawkeyeLibError):
        _lib.call('hk_jpeg_idct', work['coef'], jb.header, jb.qtabs, planes, 0, None)
    with pytest.raises(_lib.HawkeyeLibError):
        _lib.call('hk_jpeg_color', None, jb.header, p.offsets, px, 2, None)
    assert lib.hk_launch_count() == 0


@pytest.fixture(scope='module')
def folder(tmp_path_factory):
    root = tmp_path_factory.mktemp('cubfolder')
    lines = []
    for i in range(24):
        opts = [R.CLASSES['420'], R.CLASSES['422'], R.FALLBACKS['progressive'], R.CLASSES['rst_row']][i % 4]
        R.write(str(root / f'{i}.jpg'), 500 if i % 3 else 375, 375 if i % 3 else 500, 100 + i, dict(opts, quality=90))
        lines.append(f'{(7 * i) % 200} {i}.jpg')
    for split in ('train', 'val'):
        (root / f'{split}.txt').write_text('\n'.join(lines) + '\n')
    return str(root)


def _config(root, tmp_path, decode, graph):
    from hawkeye_b200.config import load_config
    cfg = load_config(os.path.join(REPO, 'configs', 'BCNN_S2.yaml'))
    cfg.dataset.update(root_dir=root, meta_dir=root, batch_size=4, num_workers=0)
    cfg.dataset.transformer['device'] = 'cuda'
    if decode:
        cfg.dataset.transformer['decode'] = 'cuda'
    cfg.experiment['log_dir'] = str(tmp_path)
    cfg.experiment['cuda_graph'] = graph
    return cfg


def test_bcnn_train_step_with_the_device_decode(folder, tmp_path, monkeypatch):
    """Six BCNN 448 steps fed by encoded JPEGs, eager and with graph replay, and six fed by PIL-decoded ones: the staged
    images are identical in all three runs, and the steps other than the first and the capture make no host
    synchronisation."""
    from hawkeye_b200 import _lib, examples
    monkeypatch.setenv('HAWKEYE_ALLOW_RANDOM_INIT', '1')
    _lib.set_precise(0)
    seen = {}
    for decode, graph in ((True, False), (True, True), (False, False)):
        tr = examples.BCNNTrainer(_config(folder, tmp_path, decode, graph))
        assert (tr.dataloaders['train'].dataset.loader is data.encoded_loader) == decode
        torch.manual_seed(5)
        stage, images = tr.stage_inputs, []

        def spy(batch):
            out = stage(batch)
            images.append(out[0].clone())
            return out
        tr.stage_inputs = spy
        for i, batch in enumerate(tr.dataloaders['train']):
            assert (batch['img'].jpeg is not None) == decode
            with no_host_sync() if i not in (0, 2) else contextlib.nullcontext():
                tr.batch_training(batch)
        tr.check_decode()
        torch.cuda.synchronize()
        assert (tr._graph is not None) == graph and np.isfinite(tr.average_meters['loss'].avg)
        seen[(decode, graph)] = torch.stack(images).cpu()
        tr.validate()
        assert tr.average_meters['acc'].count == 24
        del tr
        torch.cuda.empty_cache()
    assert torch.equal(seen[(True, False)], seen[(True, True)])
    assert torch.equal(seen[(True, False)], seen[(False, False)])


def test_trainer_raises_naming_the_corrupt_file(tmp_path, cub, monkeypatch):
    from hawkeye_b200 import _lib, examples
    monkeypatch.setenv('HAWKEYE_ALLOW_RANDOM_INIT', '1')
    _lib.set_precise(0)
    files = _corrupt(tmp_path, cub)
    root = tmp_path / 'set'
    root.mkdir()
    names = [os.path.basename(p) for p in cub[:3]] + ['bad_code.jpg']
    for p in cub[:3] + [files['bad_code']]:
        (root / os.path.basename(p)).write_bytes(open(p, 'rb').read())
    for split in ('train', 'val'):
        (root / f'{split}.txt').write_text('\n'.join(f'{i} {n}' for i, n in enumerate(names)) + '\n')
    tr = examples.BCNNTrainer(_config(str(root), tmp_path, True, False))
    with pytest.raises(RuntimeError, match='bad_code.jpg'):
        for batch in tr.dataloaders['train']:
            tr.batch_training(batch)
        tr.check_decode()
    with pytest.raises(RuntimeError, match='bad_code.jpg'):
        tr.validate()


def test_tester_with_the_device_decode(folder, tmp_path, monkeypatch):
    from hawkeye_b200.cfgnode import CfgNode
    from hawkeye_b200.test import Tester
    from oracle.hop_oracle import VGG16_D
    monkeypatch.setenv('HAWKEYE_ALLOW_RANDOM_INIT', '1')
    path = str(tmp_path / 'best_model.pth')
    torch.save(detgen.vgg_bcnn_state(VGG16_D, 200, seed=100), path)
    acc, ims = {}, {}
    for decode in (False, True):
        tr = dict(image_size=448, resize_size=512, device='cuda')
        if decode:
            tr['decode'] = 'cuda'
        cfg = CfgNode(dict(experiment=dict(name='t', cuda=[0]), dataset=dict(root_dir=folder, meta_dir=folder, batch_size=8,
                                                                             num_workers=0, transformer=tr),
                           model=dict(name='BCNN', num_classes=200, load=path)))
        t = Tester(cfg)
        ims[decode] = torch.cat([t.to_device(b['img']) for b in t.dataloader])
        acc[decode] = t.test()
    assert torch.equal(ims[False], ims[True]) and acc[False] == acc[True]
