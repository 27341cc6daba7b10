"""Mixup / CutMix on the host side (hawkeye_b200.data.MixupCutmixCollateFn, hawkeye_b200.ops_mixup): the collate's draws
against the reference's MixupCutmixCollateFn, the CPU restatement of the mix and the dense target against the reference's
outputs, the C-ABI error paths of the mix entries, and which trainers take ``dataset.mixup_cutmix``.  The reference's
outputs are fixtures recorded by tests/golden/make_golden_mixup.py."""
import os
import random

import numpy as np
import pytest
import torch

import mixup_ref
from conftest import load_golden
from hawkeye_b200 import data, examples, ops, ops_augment as A, ops_mixup as M, train
from hawkeye_b200.config import load_config

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K = 10                       # the fixtures' num_classes


@pytest.fixture(scope='module')
def gold():
    return load_golden('reference_mixup')


@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as g
    g.build()
    from hawkeye_b200 import _lib
    return _lib.lib()


def _items(img, label):
    return [{'img': torch.from_numpy(img[i]), 'label': int(label[i])} for i in range(len(label))]


def test_collate_draws_what_the_reference_draws(gold, lib):
    """Over 50 seeded batches: the same kind, lambda, box and target weight as the reference's collate, images and labels
    passed through untouched, and both kinds drawn."""
    kinds = []
    for k in range(50):
        img, label = gold[f'draws.img.{k}'], gold[f'draws.label.{k}']
        random.seed(k)
        torch.manual_seed(k)
        out = data.MixupCutmixCollateFn(K)(_items(img, label))
        row = out['mix'].numpy()
        assert out['mix'].dtype == torch.float64 and row.shape == (M.MIX_COLS,)
        assert row[M.KIND] == gold['draws.kind'][k] and row[M.LAMBDA] == gold['draws.lam'][k]
        assert tuple(row[M.BOX:M.BOX + 4]) == tuple(gold['draws.box'][k]) and row[M.WEIGHT] == gold['draws.weight'][k]
        assert np.array_equal(out['img'].numpy(), img) and out['label'].dtype == torch.int64
        assert np.array_equal(out['label'].numpy(), label)
        kinds.append(int(row[M.KIND]))
    assert 10 < sum(kinds) < 40


def test_restatement_is_the_reference_bit_for_bit(gold):
    """The mix and the dense target restated from the recorded draws equal the reference's, bit for bit, on the 50
    collate batches and on every kernel case (clipped, empty and full boxes, B = 1)."""
    cases = [(gold[f'draws.img.{k}'], gold[f'draws.label.{k}'], gold[f'draws.out.{k}'], gold[f'draws.target.{k}'],
              [gold['draws.kind'][k], gold['draws.lam'][k], *gold['draws.box'][k], gold['draws.weight'][k]])
             for k in range(50)]
    cases += [tuple(gold[f'case.{n}.{f}'] for f in ('img', 'label', 'out', 'target', 'draw')) for n in gold['case.names']]
    for img, label, out, target, draw in cases:
        row = mixup_ref.row_of(draw)
        assert mixup_ref.mix_images(img, row).tobytes() == out.tobytes()
        assert mixup_ref.dense_target(label, row, K).tobytes() == target.tobytes()
    assert set(gold['case.names']) >= {'mixup', 'cutmix', 'cutmix_left_top', 'cutmix_right_bottom', 'cutmix_empty',
                                       'cutmix_full', 'mixup_b1', 'cutmix_b1'}


FAKE = 0x10000      # a non-null, 16-byte aligned address that must never be dereferenced on these paths


def test_cabi_errors_launch_nothing(lib):
    import ctypes
    assert lib.hk_mix_cols() == M.MIX_COLS
    lib.hk_reset_launch_count()
    mb, ce = lib.hk_mix_batch, lib.hk_softmax_ce_ls_mix
    assert mb(None, FAKE, FAKE, 2, 3, 8, 8, None) == -1 and 'null' in lib.hk_last_error().decode()
    assert mb(FAKE, None, FAKE + 64, 2, 3, 8, 8, None) == -1 and mb(FAKE, FAKE, None, 2, 3, 8, 8, None) == -1
    for n, c, h, w in ((0, 3, 8, 8), (2, 0, 8, 8), (2, 3, -1, 8), (2, 3, 8, 0)):
        assert mb(FAKE, FAKE, FAKE + 64, n, c, h, w, None) == -1
    assert mb(FAKE, FAKE, FAKE, 2, 3, 8, 8, None) == -1 and 'alias' in lib.hk_last_error().decode()
    assert ce(None, FAKE, FAKE, FAKE, FAKE, FAKE, 4, 8, 0.1, 1.0, None) == -1
    assert ce(FAKE, FAKE, None, FAKE, FAKE, FAKE, 4, 8, 0.1, 1.0, None) == -1
    assert ce(FAKE, FAKE, FAKE, None, FAKE, FAKE, 4, 8, 0.1, 1.0, None) == -1
    assert ce(FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, 0, 8, 0.1, 1.0, None) == -1
    assert ce(FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, 4, 0, 0.1, 1.0, None) == -1
    assert lib.hk_launch_count() == 0

    def check(row, h=24, w=40):
        r = np.ascontiguousarray(row, np.float64)
        return lib.hk_mix_check(r.ctypes.data_as(ctypes.c_void_p), h, w)

    good = [M.mix_row(M.MIXUP, 0.3).numpy(), M.mix_row(M.CUTMIX, 0.5, (0, 0, 40, 24), 0.0).numpy(),
            M.mix_row(M.CUTMIX, 1.0, (7, 3, 7, 3), 1.0).numpy()]
    assert all(check(r) == 0 for r in good)
    assert lib.hk_mix_check(None, 24, 40) == -1 and check(good[0], 0, 40) == -1 and check(good[0], 24, 0) == -1
    bad = {'box outside': (M.CUTMIX, 0.5, (0, 0, 41, 24), 0.5), 'negative corner': (M.CUTMIX, 0.5, (-1, 0, 4, 4), 0.5),
           'box below': (M.CUTMIX, 0.5, (0, 20, 4, 25), 0.5), 'reversed': (M.CUTMIX, 0.5, (5, 0, 4, 4), 0.5),
           'fractional': (M.CUTMIX, 0.5, (0.5, 0, 4, 4), 0.5), 'kind': (2, 0.5, (0, 0, 0, 0), 0.5),
           'lambda': (M.MIXUP, 1.5, (0, 0, 0, 0), 0.5), 'weight': (M.CUTMIX, 0.5, (0, 0, 4, 4), -0.1),
           'nan': (M.MIXUP, float('nan'), (0, 0, 0, 0), 0.5)}
    for name, (kind, lam, box, w) in bad.items():
        assert check(M.mix_row(kind, lam, box, w).numpy()) == -1, name
    with pytest.raises(ValueError, match='outside the 40 x 24 image'):
        M.check_row(M.mix_row(M.CUTMIX, 0.5, (0, 0, 41, 24), 0.5), 24, 40)
    assert lib.hk_launch_count() == 0


def _cfg(yaml, key=True):
    cfg = load_config(os.path.join(REPO, 'configs', yaml))
    if key:
        cfg.dataset['mixup_cutmix'] = True
    return cfg


TAKE = {'BCNN': 'BCNN_S2.yaml', 'CBCNN': 'CBCNN_S1.yaml', 'MPN': 'MPN.yaml', 'Baseline': 'Baseline.yaml'}
YAML = {'PeerLearning': 'PeerLearning_BCNN_S2.yaml', 'OSMENet': 'OSMENet.yaml', 'APINet': 'APINet.yaml', 'DCL': 'DCL.yaml',
        'ProtoTreeNet': 'ProtoTreeNet.yaml', 'InterpPartsNet': 'InterpPartsNet.yaml', 'NTSNet': 'NTSNet.yaml',
        'APCNN': 'APCNN.yaml', 'MGE_CNN': 'MGE_CNN.yaml', 'CIN': 'CIN.yaml', 'PairConfusion': 'PC_resnet50.yaml',
        'CrossX': 'CrossX.yaml', 'S3N': 'S3N.yaml'}


def test_every_trainer_outside_the_list_rejects_the_key():
    assert set(TAKE) | set(YAML) == set(examples.ALL_TRAINERS)
    for name, yaml in YAML.items():
        cls = examples.ALL_TRAINERS[name]
        with pytest.raises(ValueError, match=f'dataset.mixup_cutmix .*; {cls.__name__} has its own loss'):
            cls(_cfg(yaml))
    for name, yaml in TAKE.items():
        assert train.mixup_cutmix(_cfg(yaml).dataset, examples.ALL_TRAINERS[name])
        assert not train.mixup_cutmix(_cfg(yaml, key=False).dataset, examples.ALL_TRAINERS[name])
    assert train.mixup_cutmix(_cfg('BCNN_S2.yaml').dataset, train.Trainer)


@pytest.fixture(scope='module')
def image_folder(tmp_path_factory):
    from PIL import Image
    root = tmp_path_factory.mktemp('jpegs')
    lines = []
    for i in range(8):
        Image.fromarray(np.random.RandomState(i).randint(0, 256, (30 + 2 * i, 40 + 3 * i, 3), dtype=np.uint8)).save(
            root / f'{i}.jpg', quality=90)
        lines.append(f'{i % 3} {i}.jpg')
    for split in ('train', 'val'):
        (root / f'{split}.txt').write_text('\n'.join(lines) + '\n')
    return str(root)


def _loaders(cls, yaml, root, device, key):
    cfg = _cfg(yaml, key)
    cfg.dataset.update(root_dir=root, meta_dir=root, batch_size=4, num_workers=0)
    cfg.dataset.transformer.update(image_size=16, resize_size=20)
    if device is not None:
        cfg.dataset.transformer['device'] = device
    t = object.__new__(cls)
    t.config, t.world, t.rank, t.samplers = cfg, 1, 0, {}
    return t, t.get_dataloader(cfg.dataset)


@pytest.mark.parametrize('device', [None, 'cuda'])
def test_loaders_mix_the_training_split_only(image_folder, lib, device):
    """With the key, the training collate wraps the split's own (default_collate, or the device preset's) and adds the
    mix row; validation batches are the same as without the key, and so is every batch of a config without it."""
    from torch.utils.data import default_collate
    for cls, yaml in ((examples.BCNNTrainer, 'BCNN_S2.yaml'), (examples.MPNTrainer, 'MPN.yaml')):
        t, loaders = _loaders(cls, yaml, image_folder, device, True)
        c = loaders['train'].collate_fn
        assert isinstance(c, data.MixupCutmixCollateFn) and c.num_classes == t.config.model.num_classes
        tf = loaders['train'].dataset.transform
        if device is None:
            assert c.collate is None and loaders['val'].collate_fn is default_collate
        else:
            assert c.collate == tf.collate and loaders['val'].collate_fn == loaders['val'].dataset.transform.collate
        torch.manual_seed(0)
        random.seed(0)
        batch = next(iter(loaders['train']))
        assert batch['mix'].shape == (M.MIX_COLS,) and batch['label'].shape == (4,)
        assert isinstance(batch['img'], A.PackedImages) == (device == 'cuda')
        images, labels = t.batch_tensors(batch)
        assert images is batch['img'] and labels[0] is batch['label'] and labels[1] is batch['mix']
        assert type(t.get_criterion(t.config.train.criterion)) is ops.CrossEntropyLSMix
        val = next(iter(loaders['val']))
        assert 'mix' not in val and t.batch_tensors(val)[1] is val['label']
        t, loaders = _loaders(cls, yaml, image_folder, device, False)
        assert not isinstance(loaders['train'].collate_fn, data.MixupCutmixCollateFn)
        for s in ('train', 'val'):
            assert 'mix' not in next(iter(loaders[s]))
        assert type(t.get_criterion(t.config.train.criterion)) is ops.CrossEntropyLS


def test_collate_rejects_what_the_reference_rejects(lib):
    c = data.MixupCutmixCollateFn(K)
    with pytest.raises(TypeError, match='int64'):
        c([{'img': torch.zeros(3, 4, 4), 'label': 1.5}])
    with pytest.raises(TypeError, match='float'):
        c([{'img': torch.zeros(3, 4, 4, dtype=torch.uint8), 'label': 1}])
    with pytest.raises(ValueError):
        data.MixupCutmixCollateFn(0)
