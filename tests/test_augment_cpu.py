"""The device presets' host side (hawkeye_b200.data.DevicePresetTrain / DevicePresetEval, hawkeye_b200.ops_augment): the
random draws against the host presets', the packing of a batch, and the loader builders with and without
``dataset.transformer.device``."""
import math
import os

import numpy as np
import pytest
import torch
from PIL import Image

from hawkeye_b200 import data, examples, ops_augment as A, train
from hawkeye_b200 import test as hb_test
from hawkeye_b200.config import load_config

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _image(w, h, seed):
    return Image.fromarray(np.random.RandomState(seed).randint(0, 256, (h, w, 3), dtype=np.uint8))


class _Spy:
    """Records what the host preset computes from its draws: the RandomResizedCrop box, whether the flip fired, the
    TrivialAugmentWide op and magnitude handed to _apply_op, and the RandomErasing rectangle."""

    def __init__(self, monkeypatch):
        from torchvision.transforms import autoaugment, functional, transforms
        self.log = {}
        get_params, apply_op, hflip, erase_params = (transforms.RandomResizedCrop.get_params, autoaugment._apply_op,
                                                     functional.hflip, transforms.RandomErasing.get_params)

        def rrc(img, scale, ratio):
            self.log['crop'] = get_params(img, scale, ratio)
            return self.log['crop']

        def op(img, name, magnitude, **kw):
            self.log['op'] = (name, magnitude)
            return apply_op(img, name, magnitude, **kw)

        def flip(img):
            self.log['flip'] = True
            return hflip(img)

        def erase(img, scale, ratio, value=None):
            out = erase_params(img, scale, ratio, value)
            self.log['erase'] = out[:4]
            return out

        monkeypatch.setattr(transforms.RandomResizedCrop, 'get_params', staticmethod(rrc))
        monkeypatch.setattr(autoaugment, '_apply_op', op)
        monkeypatch.setattr(functional, 'hflip', flip)
        monkeypatch.setattr(transforms.RandomErasing, 'get_params', staticmethod(erase))


def _fallback_box(w, h):
    """RandomResizedCrop.get_params after ten rejected draws: the centred crop of the clamped aspect ratio."""
    r = w / h
    if r < 3 / 4:
        cw, ch = w, int(round(w / (3 / 4)))
    elif r > 4 / 3:
        ch, cw = h, int(round(h * (4 / 3)))
    else:
        cw, ch = w, h
    return (h - ch) // 2, (w - cw) // 2, ch, cw


SIZES = [(500, 375), (375, 500), (64, 48), (33, 97), (400, 9), (7, 300), (45, 45), (1000, 12)]


def test_train_draws_match_the_host_preset(monkeypatch):
    """Under one seed per image, the device preset draws exactly the parameters the host preset uses, over many images,
    sizes and ops, and leaves the torch RNG in the same state."""
    S = 32
    host = data.ClassificationPresetTrain(S, auto_augment_policy='ta_wide', random_erase_prob=0.5)
    dev = data.DevicePresetTrain(S, auto_augment_policy='ta_wide', random_erase_prob=0.5)
    spy = _Spy(monkeypatch)
    ops, fallbacks, flips, erased = set(), 0, 0, 0
    for k in range(400):
        w, h = SIZES[k % len(SIZES)]
        img = _image(w, h, k)
        spy.log = {}
        torch.manual_seed(1000 + k)
        host(img)
        after_host = torch.get_rng_state()
        torch.manual_seed(1000 + k)
        arr, row = dev(img)
        assert torch.equal(torch.get_rng_state(), after_host)
        assert arr.shape == (h, w, 3) and arr.dtype == np.uint8 and np.array_equal(arr, np.asarray(img))
        i, j, ch, cw = spy.log['crop']
        assert tuple(row[A.BOX:A.BOX + 4]) == (j, i, cw, ch) and tuple(row[A.VIRTUAL:A.VIRTUAL + 2]) == (S, S)
        assert tuple(row[A.WINDOW:A.WINDOW + 2]) == (0, 0)
        fallbacks += (i, j, ch, cw) == _fallback_box(w, h)
        assert row[A.FLIP] == float(spy.log.get('flip', False))
        flips += spy.log.get('flip', False)
        name, magnitude = spy.log['op']
        ops.add(name)
        assert A.TA_OPS[int(row[A.OP])] == name and row[A.MAG] == magnitude
        if name in A.GEOMETRIC:
            assert list(row[A.MATRIX:A.MATRIX + 6]) == A.op_matrix(name, magnitude, S, S)
        e = spy.log.get('erase')
        if e is not None and e[2] < S:
            erased += 1
            assert tuple(row[A.ERASE:A.ERASE + 4]) == tuple(e)
        else:
            assert row[A.ERASE + 2] == 0
    assert ops == set(A.TA_OPS) and fallbacks >= 10 and 100 < flips < 300 and erased > 50


def test_eval_draws_no_random_number_and_follows_resize_and_center_crop():
    from torchvision.transforms import functional as F
    for (w, h), resize, S in [((500, 375), 512, 448), ((375, 500), 512, 448), ((333, 120), 64, 56), ((40, 30), 20, 32),
                              ((31, 77), [50, 20], 24)]:
        dev = data.DevicePresetEval(S, resize_size=resize)
        img = _image(w, h, 1)
        state = torch.get_rng_state()
        arr, row = dev(img)
        assert torch.equal(torch.get_rng_state(), state)
        assert tuple(row[A.BOX:A.BOX + 4]) == (0, 0, w, h) and row[A.FLIP] == 0 and row[A.OP] == 0 and row[A.ERASE + 2] == 0
        vw, vh = int(row[A.VIRTUAL]), int(row[A.VIRTUAL + 1])
        assert F.resize(img, resize).size == (vw, vh)
        # the window, on a virtual image whose pixels encode their own coordinates
        coords = np.stack(np.meshgrid(np.arange(vw), np.arange(vh)), -1).astype(np.int32) + 1
        cropped = F.center_crop(torch.from_numpy(coords).permute(2, 0, 1), [S, S]).permute(1, 2, 0).numpy()
        wx, wy = int(row[A.WINDOW]), int(row[A.WINDOW + 1])
        ys, xs = np.mgrid[0:S, 0:S]
        inside = (xs + wx >= 0) & (xs + wx < vw) & (ys + wy >= 0) & (ys + wy < vh)
        assert np.array_equal(cropped[..., 0][inside], (xs + wx + 1)[inside])
        assert np.array_equal(cropped[..., 1][inside], (ys + wy + 1)[inside]) and (cropped[~inside] == 0).all()


def test_rotate_matrix_is_pils():
    """PIL.Image.rotate's own matrix, read back from the transform call it makes."""
    seen = []
    orig = Image.Image.transform

    def spy(self, size, method, data=None, *a, **k):
        seen.append(list(data))
        return orig(self, size, method, data, *a, **k)

    img = _image(20, 20, 3)
    Image.Image.transform = spy
    try:
        for angle in (4.5, -31.5, 135.0, -90.0 + 1e-9):
            seen.clear()
            img.rotate(angle, Image.BILINEAR)
            assert seen[0] == A.pil_rotate_matrix(angle, 20, 20)
    finally:
        Image.Image.transform = orig
    assert A.pil_rotate_matrix(0.0, 20, 20) == [1.0, 0.0, 0.0, 0.0, 1.0, 0.0]
    m = A.pil_rotate_matrix(90.0, 20, 20)                  # PIL transposes: the matrix is an exact permutation
    assert m[0] == 0 and m[4] == 0 and abs(m[1]) == 1 and float(m[2]).is_integer() and float(m[5]).is_integer()


def test_presets_reject_what_they_do_not_implement():
    from torchvision.transforms.functional import InterpolationMode
    for policy in ('ra', 'imagenet'):
        with pytest.raises(ValueError, match='auto_augment_policy'):
            data.DevicePresetTrain(32, auto_augment_policy=policy)
    with pytest.raises(ValueError, match='BILINEAR'):
        data.DevicePresetTrain(32, interpolation=InterpolationMode.BICUBIC)
    with pytest.raises(ValueError, match='BILINEAR'):
        data.DevicePresetEval(32, interpolation=InterpolationMode.NEAREST)
    with pytest.raises(ValueError, match='square'):
        data.DevicePresetTrain((32, 48))
    data.DevicePresetTrain(32, auto_augment_policy=None)


def test_collate_packs_offsets_sizes_and_parameters():
    dev = data.DevicePresetTrain(16, auto_augment_policy='ta_wide', random_erase_prob=0.1, mean=(0.1, 0.2, 0.3),
                                 std=(1.0, 2.0, 3.0))
    torch.manual_seed(0)
    items = [{'img': dev(_image(w, h, i)), 'label': i, 'id': 7 * i} for i, (w, h) in enumerate(SIZES[:5])]
    b = dev.collate(items)
    p = b['img']
    assert isinstance(p, A.PackedImages) and len(p) == 5 and p.size == 16
    assert p.mean == (0.1, 0.2, 0.3) and p.std == (1.0, 2.0, 3.0)
    assert p.data.dtype == torch.uint8 and p.offsets.dtype == torch.int64 and p.sizes.dtype == torch.int32
    assert p.params.dtype == torch.float64 and p.params.shape == (5, A.PARAM_COLS)
    assert p.data.numel() == sum(w * h * 3 for w, h in SIZES[:5])
    for i, it in enumerate(items):
        arr, row = it['img']
        o = int(p.offsets[i])
        assert o == sum(w * h * 3 for w, h in SIZES[:i]) and tuple(p.sizes[i].tolist()) == arr.shape[:2]
        assert np.array_equal(p.data[o:o + arr.size].numpy().reshape(arr.shape), arr)
        assert np.array_equal(p.params[i].numpy(), row)
    assert b['label'].tolist() == list(range(5)) and b['label'].dtype == torch.int64 and b['id'].tolist() == [0, 7, 14, 21, 28]
    bad = dict(items[0], img=(items[0]['img'][0], items[0]['img'][1].copy()))
    bad['img'][1][A.BOX + 2] = 10 ** 6
    with pytest.raises(ValueError, match='outside its image'):
        dev.collate([bad])


# ---- builders --------------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def image_folder(tmp_path_factory):
    root = tmp_path_factory.mktemp('jpegs')
    lines = []
    for i in range(12):
        _image(40 + 3 * i, 30 + 2 * i, i).save(root / f'{i}.jpg', quality=90)
        lines.append(f'{i % 3} {i}.jpg')
    for split in ('train', 'val'):
        (root / f'{split}.txt').write_text('\n'.join(lines) + '\n')
    return str(root)


def _loaders(cls, yaml, root, device):
    cfg = load_config(os.path.join(REPO, 'configs', yaml))
    cfg.dataset.update(root_dir=root, meta_dir=root, batch_size=4, num_workers=0)
    cfg.dataset.transformer.update(image_size=16, resize_size=20)
    if device is not None:
        cfg.dataset.transformer['device'] = device
    t = object.__new__(cls)
    t.config, t.world, t.rank, t.samplers = cfg, 1, 0, {}
    return t, cfg, t.get_dataloader(cfg.dataset)


@pytest.mark.parametrize('cls,yaml', [(train.Trainer, 'BCNN_S2.yaml'), (examples.OSMENetTrainer, 'OSMENet.yaml'),
                                      (examples.MPNTrainer, 'MPN.yaml')])
def test_trainer_builders(image_folder, cls, yaml):
    from torch.utils.data import default_collate
    t, _, loaders = _loaders(cls, yaml, image_folder, None)
    for s, want in (('train', data.ClassificationPresetTrain), ('val', data.ClassificationPresetEval)):
        assert type(loaders[s].dataset.transform) is want and loaders[s].collate_fn is default_collate
    t, _, loaders = _loaders(cls, yaml, image_folder, 'cuda')
    for s, want in (('train', data.DevicePresetTrain), ('val', data.DevicePresetEval)):
        tf = loaders[s].dataset.transform
        assert type(tf) is want and tf.size == 16 and loaders[s].collate_fn == tf.collate
    assert loaders['val'].dataset.transform.resize_size == [20]
    batch = next(iter(loaders['val']))
    assert isinstance(batch['img'], A.PackedImages) and len(batch['img']) == 4 and batch['label'].shape == (4,)
    train_tf = loaders['train'].dataset.transform
    assert train_tf.ta is not None and train_tf.erase is not None and train_tf.erase.p == 0.1


def test_builders_reject_the_key_where_presets_are_the_method_s(image_folder):
    for cls, yaml in ((examples.APCNNTrainer, 'APCNN.yaml'), (examples.DCLTrainer, 'DCL.yaml'),
                      (examples.S3NTrainer, 'S3N.yaml')):
        with pytest.raises(ValueError, match='default presets only'):
            _loaders(cls, yaml, image_folder, 'cuda')
    with pytest.raises(ValueError, match="'cuda' or absent"):
        _loaders(train.Trainer, 'BCNN_S2.yaml', image_folder, 'gpu')


def test_tester_builder(image_folder):
    from torchvision import transforms
    from hawkeye_b200.cfgnode import CfgNode
    for device in (None, 'cuda'):
        tr = dict(image_size=16, resize_size=20)
        if device:
            tr['device'] = device
        cfg = CfgNode(dict(root_dir=image_folder, meta_dir=image_folder, batch_size=4, num_workers=0, transformer=tr))
        loader = hb_test.Tester.get_dataloader(object.__new__(hb_test.Tester), cfg)
        tf = loader.dataset.transform
        if device is None:
            assert type(tf) is transforms.Compose and [type(x).__name__ for x in tf.transforms] == [
                'Resize', 'CenterCrop', 'ToTensor', 'Normalize']
        else:
            assert type(tf) is data.DevicePresetEval and loader.collate_fn == tf.collate and tf.size == 16
            assert tf.mean == hb_test.IMAGENET_MEAN and tf.std == hb_test.IMAGENET_STD


def test_param_row_layout_matches_the_library():
    from hawkeye_b200 import _lib
    try:
        cols = _lib.query('hk_augment_params_cols')
    except _lib.HawkeyeLibError:
        pytest.skip('library not built')
    assert cols == A.PARAM_COLS == A.ERASE + 4
    assert len(A.TA_OPS) == 14 and list(data.DevicePresetTrain(8, auto_augment_policy='ta_wide').ta._augmentation_space(
        31)) == list(A.TA_OPS)
    assert math.isclose(A.op_matrix('TranslateX', 7.9, 10, 10)[2], -7.0)
