"""Host logic the trainers share, with no kernel run: which output of each model validation scores (``train.prediction``),
the one validation step of ``Trainer`` and ``Tester``, and the rank-sharded loaders the trainers build."""
import os

import numpy as np
import pytest
import torch
import torch.nn as nn
from torch.utils.data import RandomSampler, SequentialSampler
from torch.utils.data.distributed import DistributedSampler

from hawkeye_b200 import data, examples, test as hb_test, train
from hawkeye_b200.config import load_config
from hawkeye_b200.methods import apcnn, dcl, interp_parts, mge, nts, osme, peer_learning, prototree

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N, C = 16, 5


def _stub(cls, outputs, **attrs):
    """An instance of the registered model class ``cls`` whose forward returns ``outputs`` (its own __init__ not run)."""
    class Stub(cls):
        def __init__(self):
            nn.Module.__init__(self)
            self.__dict__.update(attrs)

        def forward(self, *args, **kwargs):
            return outputs
    return Stub()


def _logits(seed):
    return torch.randn(N, C, generator=torch.Generator().manual_seed(seed))


def _cases():
    """-> [(name, trainer class, model, outputs, what the trainer's validation scored before it was shared)]."""
    out = []
    o = (_logits(1), torch.rand(N, 2, 1024))
    out.append(('OSMENet', examples.OSMENetTrainer, _stub(osme.OSMENet, o), o, o[0]))
    for xmul in (False, True):
        o = [_logits(2), torch.randn(N, 2 * C if xmul else 2), torch.rand(N, 49)]
        scored = o[0] + o[1][:, :C] + o[1][:, C:2 * C] if xmul else o[0]
        out.append((f'DCL-cls_2xmul={xmul}', examples.DCLTrainer, _stub(dcl.DCL, o, cls_2xmul=xmul), o, scored))
    o = (_logits(3), {'pa_tensor': None, 'ps': None})
    out.append(('ProtoTreeNet', examples.ProtoTreeTrainer, _stub(prototree.ProtoTreeNet, o), o, o[0]))
    o = (_logits(4), torch.rand(N, 1, 5, 1), torch.rand(N, 5, 7, 7))
    out.append(('InterpPartsNet', examples.InterpPartsNetTrainer, _stub(interp_parts.ResNet, o), o, o[0]))
    o = [_logits(5), _logits(6), torch.randn(N, 6, C), torch.zeros(N, 6), torch.rand(N, 6)]
    out.append(('NTSNet', examples.NTSNetTrainer, _stub(nts.NTSNet, o), o, o[1]))
    o = (_logits(7), [_logits(8)] * 8, torch.rand(N, 3), [])
    out.append(('APCNN', examples.APCNNTrainer, _stub(apcnn.ResNet, o), o, o[0]))
    o = {'logits': [_logits(10 + i) for i in range(10)], 'pr_gate': torch.rand(N, 3), 'boxes': torch.zeros(2, N, 4)}
    out.append(('MGE_CNN', examples.MGE_CNNTrainer, _stub(mge.LocalCamNet, o), o, o['logits'][-1]))
    return out


CASES = _cases()
LABELS = torch.randint(0, C, (N,), generator=torch.Generator().manual_seed(0))


def _trainer(cls, model):
    t = object.__new__(cls)
    t.device, t.model, t.average_meters = torch.device('cpu'), model, {'acc': train.AverageMeter()}
    return t


def _tester(model):
    t = object.__new__(hb_test.Tester)
    t.device, t.model, t.average_meters = torch.device('cpu'), model, {'acc': train.AverageMeter()}
    return t


def _batch(cls):
    images = torch.zeros(N, 3, 8, 8)
    if cls is examples.DCLTrainer:             # collate_fn4val: (images, labels, labels_swap, swap_law, paths)
        return (images, LABELS, LABELS, torch.zeros(N, 49), ['x'] * N)
    return {'img': images, 'label': LABELS}


@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_prediction_is_what_validation_scored(case):
    _, _, model, outputs, scored = case
    pred = train.prediction(model, outputs)
    assert pred.shape == (N, C) and torch.equal(pred, scored)


def test_prediction_of_peer_learning_and_plain_models():
    heads = (_logits(20), _logits(21))
    assert train.prediction(_stub(peer_learning.PeerLearningNet, heads), heads) == heads
    logits = _logits(22)
    assert train.prediction(nn.Identity(), logits) is logits          # a model without prediction(): its outputs


@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_trainer_and_tester_validate_alike(case):
    _, cls, model, _, scored = case
    t = _trainer(cls, model)
    t.batch_validate(_batch(cls))
    tester = _tester(model)
    tester.batch_validate({'img': torch.zeros(N, 3, 8, 8), 'label': LABELS})
    want = train.accuracy(scored, LABELS)
    assert t.average_meters['acc'].avg == tester.average_meters['acc'].avg == want
    assert t.average_meters['acc'].count == tester.average_meters['acc'].count == N


def test_tester_scores_peer_learning_on_its_better_head():
    heads = (_logits(30), _logits(31))
    tester = _tester(_stub(peer_learning.PeerLearningNet, heads))
    tester.batch_validate({'img': torch.zeros(N, 3, 8, 8), 'label': LABELS})
    assert tester.average_meters['acc'].avg == max(train.accuracy(h, LABELS) for h in heads)


def test_tester_scores_osmenet_on_its_logits():
    """OSMENet's (logits, x_part [N, P, 1024]) is not a pair of heads: x_part must not be scored."""
    labels = torch.zeros(8, dtype=torch.long)                    # every label below P = 2
    o = (torch.randn(8, C, generator=torch.Generator().manual_seed(40)), torch.rand(8, 2, 1024))
    tester = _tester(_stub(osme.OSMENet, o))
    tester.batch_validate({'img': torch.zeros(8, 3, 8, 8), 'label': labels})
    acc = tester.average_meters['acc'].avg
    assert acc <= 100.0 and acc == train.accuracy(o[0], labels)


def test_tester_evaluates_dcl():
    o = [_logits(50), torch.randn(N, 2 * C), torch.rand(N, 49)]
    tester = _tester(_stub(dcl.DCL, o, cls_2xmul=True))
    tester.batch_validate({'img': torch.zeros(N, 3, 8, 8), 'label': LABELS})
    assert tester.average_meters['acc'].avg == train.accuracy(o[0] + o[1][:, :C] + o[1][:, C:], LABELS)


# ---- loaders ----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def image_folder(tmp_path_factory):
    """Two classes of ten 24 x 24 images, listed in train.txt and val.txt."""
    from PIL import Image
    root = tmp_path_factory.mktemp('images')
    rng = np.random.RandomState(0)
    lines = []
    for i in range(20):
        Image.fromarray((rng.rand(24, 24, 3) * 255).astype(np.uint8)).save(root / f'{i}.png')
        lines.append(f'{i % 2} {i}.png')
    for split in ('train', 'val'):
        (root / f'{split}.txt').write_text('\n'.join(lines) + '\n')
    return str(root)


def _loaders(cls, yaml, root, world, rank):
    cfg = load_config(os.path.join(REPO, 'configs', yaml))
    cfg.dataset.update(root_dir=root, meta_dir=root, batch_size=8, num_workers=0)
    cfg.dataset.transformer.update(image_size=16, resize_size=20)
    t = object.__new__(cls)
    t.config, t.world, t.rank, t.samplers = cfg, world, rank, {}
    return t, t.get_dataloader(cfg.dataset)


def _transform_types(t):
    return [type(x).__name__ for x in t.transforms]


LOADERS = [
    (train.Trainer, 'MPN.yaml', None,
     {'train': ['ClassificationPresetTrain'], 'val': ['ClassificationPresetEval']}),
    (examples.InterpPartsNetTrainer, 'InterpPartsNet.yaml', None,
     {'train': ['Resize', 'RandomHorizontalFlip', 'ColorJitter', 'RandomCrop', 'ToTensor', 'Normalize', 'RandomErasing'],
      'val': ['Resize', 'CenterCrop', 'ToTensor', 'Normalize']}),
    (examples.APCNNTrainer, 'APCNN.yaml', None,
     {'train': ['Resize', 'RandomCrop', 'RandomHorizontalFlip', 'TrivialAugmentWide', 'ToTensor', 'Normalize'],
      'val': ['Resize', 'CenterCrop', 'ToTensor', 'Normalize']}),
    (examples.DCLTrainer, 'DCL.yaml', {'train': data.collate_fn4train, 'val': data.collate_fn4val},
     {'train': ['Resize', 'ToTensor', 'Normalize'], 'val': ['Resize', 'ToTensor', 'Normalize']}),
]


@pytest.mark.parametrize('world,rank', [(1, 0), (2, 1)])
@pytest.mark.parametrize('cls,yaml,collate,tf', LOADERS, ids=[c[0].__name__ for c in LOADERS])
def test_rank_loaders(image_folder, cls, yaml, collate, tf, world, rank):
    from torch.utils.data import default_collate
    t, loaders = _loaders(cls, yaml, image_folder, world, rank)
    assert set(loaders) == {'train', 'val'} and set(t.samplers) == {'train', 'val'}
    for s, loader in loaders.items():
        assert loader.batch_size == 8 // world and loader.num_workers == 0 and loader.pin_memory
        assert loader.dataset is t.datasets[s]
        if world == 1:
            assert t.samplers[s] is None
            assert type(loader.sampler) is (RandomSampler if s == 'train' else SequentialSampler)
        else:
            sm = loader.sampler
            assert t.samplers[s] is sm and type(sm) is DistributedSampler
            assert (sm.num_replicas, sm.rank, sm.shuffle, sm.drop_last) == (2, 1, s == 'train', False)
        assert loader.collate_fn is (collate[s] if collate else default_collate)
        ds = loader.dataset
        if cls is examples.DCLTrainer:
            assert type(ds) is data.DCLDataset and ds.mode == s
            assert _transform_types(ds.totensor) == tf[s]
            assert _transform_types(ds.swap) == ['RandomSwap']
        elif cls is train.Trainer:
            assert type(ds) is data.FGDataset and [type(ds.transform).__name__] == tf[s]
        else:
            assert type(ds) is data.FGDataset and _transform_types(ds.transform) == tf[s]


@pytest.mark.parametrize('cls,yaml', [(c[0], c[1]) for c in LOADERS], ids=[c[0].__name__ for c in LOADERS])
def test_loaders_reject_a_batch_the_ranks_cannot_split(image_folder, cls, yaml):
    with pytest.raises(ValueError, match='batch_size=8 must be a multiple of the 3 ranks'):
        _loaders(cls, yaml, image_folder, 3, 0)
