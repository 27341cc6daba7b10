"""hawkeye_b200.data — the mirror of the reference's dataset package (dataset/dataset.py, transforms.py:14-73, sampler.py) — on a
generated image folder: item format, the deterministic eval preset, class-balanced batches; and item-for-item / batch-for-batch
equality with the reference's own classes (recorded outputs)."""
import os
import sys

import numpy as np
import pytest
import torch

from hawkeye_b200 import data as D


@pytest.fixture(scope='module')
def folder(tmp_path_factory):
    from PIL import Image
    root = tmp_path_factory.mktemp('imgs')
    rng = np.random.RandomState(0)
    lines = []
    for i in range(24):
        arr = rng.randint(0, 256, size=(40 + i, 50 + 2 * i, 3), dtype=np.uint8)
        name = f'c{i % 4}/img_{i}.png'
        os.makedirs(os.path.join(root, f'c{i % 4}'), exist_ok=True)
        Image.fromarray(arr).save(os.path.join(root, name))
        lines.append(f'{i % 4} {name}')
    meta = os.path.join(root, 'train.txt')
    open(meta, 'w').write('\n'.join(lines) + '\n')
    return str(root), meta


def test_dataset_items_and_eval_preset(folder):
    root, meta = folder
    ds = D.FGDataset(root, meta, transform=D.ClassificationPresetEval(crop_size=32, resize_size=36), return_id=True)
    assert len(ds) == 24
    it = ds[5]
    assert set(it) == {'img', 'label', 'id'} and it['id'] == 5 and int(it['label']) == 1
    assert it['img'].shape == (3, 32, 32) and it['img'].dtype == torch.float32
    assert torch.equal(ds[5]['img'], it['img'])                               # deterministic
    tr = D.FGDataset(root, meta, transform=D.ClassificationPresetTrain(crop_size=32, auto_augment_policy='ta_wide',
                                                                      random_erase_prob=0.1))
    assert tr[0]['img'].shape == (3, 32, 32)


def test_balanced_batches(folder):
    root, meta = folder
    ds = D.FGDataset(root, meta)
    np.random.seed(3)
    s = D.BalancedBatchSampler(ds, n_classes=2, n_samples=3)
    batches = list(s)
    assert len(s) == 4 and 1 <= len(batches) <= 4
    labels = np.array(ds.images['label'])
    for b in batches:
        assert len(b) == 6
        cls, cnt = np.unique(labels[b], return_counts=True)
        assert len(cls) == 2 and (cnt == 3).all()                               # what MAMCLoss needs


REFERENCE_DATA = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'reference_data.npz')


def reference_data_outputs(root, meta, rd, rt, rs):
    """What the reference's dataset classes return on the generated folder: eval items 0 / 7 / 23, one train-preset draw
    (torch / python RNG seeded 11) and the class-balanced batches (numpy RNG seeded 5).  `rd, rt, rs` are its
    dataset.dataset, dataset.transforms and dataset.sampler modules — or ours, which must give the same."""
    import random
    out = {}
    ds = rd.FGDataset(root, meta, transform=rt.ClassificationPresetEval(crop_size=32, resize_size=36))
    out['len'] = np.array(len(ds))
    for i in (0, 7, 23):
        it = ds[i]
        out[f'img_{i}'], out[f'label_{i}'] = it['img'].numpy(), np.array(int(it['label']))
    tr = rt.ClassificationPresetTrain(32, auto_augment_policy='ta_wide', random_erase_prob=0.1)
    img = D.default_loader(os.path.join(root, 'c1/img_5.png'))
    torch.manual_seed(11); random.seed(11)
    out['train_draw'] = tr(img).numpy()
    np.random.seed(5)
    out['batches'] = np.array([list(map(int, b)) for b in rs.BalancedBatchSampler(ds, 2, 3)])
    return out


def test_matches_reference_classes(folder):
    """Item-for-item / batch-for-batch equality with the reference's own classes, recorded in
    tests/golden/reference_data.npz by running reference_data_outputs on the reference's modules."""
    root, meta = folder
    want = np.load(REFERENCE_DATA)
    got = reference_data_outputs(root, meta, D, D, D)
    assert sorted(got) == sorted(want.files)
    for k in got:
        assert got[k].shape == want[k].shape and np.array_equal(got[k], want[k]), k
    assert len(got['batches']) > 0
