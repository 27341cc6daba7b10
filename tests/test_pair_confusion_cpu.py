"""Pairwise Confusion and the plain ResNet classifiers without a GPU: the fp64 loss oracle against fixtures of the unmodified
reference (tests/golden/make_golden_pc.py), ResNet50 / ResNet101 against torchvision's layout and their pretrained loading,
the Baseline and PairConfusion trainers' registration, groups, schedules, transforms and loaders, and the argument errors
of hk_pc_loss and of the criterion."""
import ctypes
import os

import numpy as np
import pytest
import torch

import pc_inputs as I
from conftest import load_golden
from oracle import pc_oracle as O

G = load_golden('reference_pc')
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
os.environ['HAWKEYE_ALLOW_RANDOM_INIT'] = '1'


def _rel(a, b):
    a, b = np.asarray(a, dtype=np.float64).ravel(), np.asarray(b, dtype=np.float64).ravel()
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30)


@pytest.mark.parametrize('lam', I.LAMBDAS)
@pytest.mark.parametrize('name', I.NAMES)
def test_oracle_matches_reference_loss(name, lam):
    z, y = I.logits(name).numpy(), I.labels(name).numpy()
    loss, dz = O.pc_loss(z, y, lam)
    term, dterm, pairs = O.confusion(z, y)
    assert pairs == {'differ': 12, 'same': 0, 'mix': 6, 'identical': 12}[name]
    # the reference in fp32 on the CPU against fp64
    assert abs(loss - G[f'loss_{name}_{lam}']) <= 1e-6 * abs(G[f'loss_{name}_{lam}'])
    assert _rel(dz, G[f'dz_{name}_{lam}']) < 1e-6
    if name == 'same':
        assert term == 0.0 and not np.any(dterm)
    if name == 'identical':
        # rows 0 and B/2 are equal with different labels: the pair adds nothing and its gradient is exactly zero, no NaN
        _, dce = O.ce_ls(z, y)
        assert not np.any(dterm[[0, I.B // 2]]) and np.all(np.isfinite(G[f'dz_{name}_{lam}']))
        assert np.abs(G[f'dz_{name}_{lam}'][[0, I.B // 2]] - dce[[0, I.B // 2]]).max() < 1e-7


def test_oracle_rejects_an_odd_batch():
    with pytest.raises(ValueError):
        O.confusion(np.zeros((3, 4)), [0, 1, 2])


def _model(yaml, name=None, **over):
    import hawkeye_b200 as hb
    from hawkeye_b200.cfgnode import CfgNode
    from hawkeye_b200.config import load_config
    cfg = CfgNode(dict(load_config(os.path.join(REPO, 'configs', yaml)).model, **over))
    return hb.MODEL.get(name or cfg.name)(cfg)


@pytest.mark.parametrize('name,arch,entries', [('ResNet50', 'resnet50', 320), ('ResNet101', 'resnet101', 626)])
def test_resnet_has_torchvision_layout(name, arch, entries):
    import torchvision
    torch.manual_seed(3)
    net = _model('PC_resnet50.yaml', name)
    torch.manual_seed(3)
    tv = getattr(torchvision.models, arch)(num_classes=200)
    a, b = net.state_dict(), tv.state_dict()
    assert len(a) == entries and list(a) == list(b) and all(a[k].shape == b[k].shape for k in a)
    assert sum(p.numel() for p in net.parameters()) == sum(p.numel() for p in tv.parameters())
    # the reference's initialisers in its RNG order: the same seed gives torchvision's (= the reference's) weights
    assert all(torch.equal(a[k], b[k]) for k in a)
    tv_state = {k: torch.randn_like(v) if v.is_floating_point() else v for k, v in b.items()}
    net.load_state_dict(tv_state, strict=True)
    tv.load_state_dict(net.state_dict(), strict=True)
    again = _model('PC_resnet50.yaml', name)
    again.load_state_dict(net.state_dict(), strict=True)
    assert all(torch.equal(v, again.state_dict()[k]) for k, v in net.state_dict().items())


def test_yaml_surface():
    from hawkeye_b200.config import load_config
    base = load_config(os.path.join(REPO, 'configs', 'Baseline.yaml'))
    pc = load_config(os.path.join(REPO, 'configs', 'PC_resnet50.yaml'))
    for cfg in (base, pc):
        assert cfg.model.name == 'ResNet50' and cfg.model.num_classes == 200 and cfg.dataset.batch_size == 24
        assert cfg.train.optimizer.name == 'Adam' and cfg.train.optimizer.weight_decay == 0.00002
    assert (base.train.optimizer.lr, base.train.scheduler.T_max, base.train.scheduler.eta_min) == (0.0001, 30, 0.00001)
    assert (pc.train.optimizer.lr, pc.train.scheduler.T_max, pc.train.scheduler.warmup_epochs) == (0.0004, 60, 5)
    assert pc.train.criterion.name == 'PairwiseConfusionLoss' and pc.train.criterion.lambda_a == 0.1


@pytest.fixture
def torchvision_pth(tmp_path, monkeypatch):
    """torchvision's resnet50 state_dict (1000 classes, random values) at $HAWKEYE_RESNET50_PTH."""
    import torchvision
    torch.manual_seed(11)
    state = torchvision.models.resnet50().state_dict()
    path = str(tmp_path / 'resnet50.pth')
    torch.save(state, path)
    monkeypatch.setenv('HAWKEYE_RESNET50_PTH', path)
    return state, path


def test_pretrained_loads_trunk_and_fc_only_at_1000_classes(torchvision_pth):
    state, path = torchvision_pth
    net = _model('PC_resnet50.yaml', num_classes=1000)
    assert all(torch.equal(v, state[k]) for k, v in net.state_dict().items())          # fc included
    torch.manual_seed(12)
    net = _model('PC_resnet50.yaml')
    torch.manual_seed(12)
    fresh = _model('PC_resnet50.yaml', pretrained=False)
    sd = net.state_dict()
    assert all(torch.equal(v, state[k]) for k, v in sd.items() if not k.startswith('fc.'))
    assert torch.equal(sd['fc.weight'], fresh.fc.weight) and torch.equal(sd['fc.bias'], fresh.fc.bias)
    assert not torch.equal(fresh.conv1.weight, state['conv1.weight'])               # pretrained: False loads nothing
    from hawkeye_b200._lib import HawkeyeLibError
    del state['layer3.2.bn2.running_var']
    torch.save(state, path)
    for k in (1000, 200):
        with pytest.raises(HawkeyeLibError, match='layer3.2.bn2.running_var'):
            _model('PC_resnet50.yaml', num_classes=k)


def test_resnet_rejects_a_class_count_the_classifier_cannot_take():
    from hawkeye_b200._lib import HawkeyeLibError
    with pytest.raises(HawkeyeLibError, match='num_classes'):
        _model('PC_resnet50.yaml', num_classes=201)


def _cfg(yaml):
    from hawkeye_b200.config import load_config
    return load_config(os.path.join(REPO, 'configs', yaml))


class _Opt:
    def __init__(self, lrs):
        self.param_groups = [dict(initial_lr=lr, lr=lr) for lr in lrs]


def _check_schedule(mine, opt, ref, ours, epochs):
    for epoch in range(epochs):
        for g, r in zip(ours.param_groups, opt.param_groups):
            assert abs(g['lr'] - r['lr']) < 1e-12, epoch
        opt.step()
        ref.step()
        mine.step()


def test_trainer_registration_groups_and_schedules():
    from hawkeye_b200 import examples
    from hawkeye_b200.losses import PairwiseConfusionLoss
    assert examples.ALL_TRAINERS['Baseline'] is examples.BaselineTrainer
    assert examples.ALL_TRAINERS['PairConfusion'] is examples.PCResNetTrainer
    assert set(examples.TRAINERS) == {'BCNN', 'CBCNN', 'MPN', 'PeerLearning', 'OSMENet'}
    with pytest.raises(SystemExit, match='PairConfusion'):
        examples.main(['nope'])

    cfg = _cfg('PC_resnet50.yaml')
    tr = examples.PCResNetTrainer.__new__(examples.PCResNetTrainer)
    tr.config, tr.total_epoch, tr.model = cfg, cfg.train.epoch, _model('PC_resnet50.yaml')
    crit = tr.get_criterion(cfg.train.criterion)
    assert isinstance(crit, PairwiseConfusionLoss) and crit.lambda_a == 0.1
    (rest, m0), (fc, m1) = tr.param_groups()
    assert (m0, m1) == (0.1, 1.0)
    assert [id(p) for p in fc] == [id(tr.model.fc.weight), id(tr.model.fc.bias)]
    assert [id(p) for p in rest] == [id(p) for n, p in tr.model.named_parameters() if not n.startswith('fc.')]

    # PairConfusion: LinearLR warm-up into CosineAnnealingLR over T_max - warmup_epochs (Examples/PairConfusion.py:25-34)
    sc, lr = cfg.train.scheduler, cfg.train.optimizer.lr
    p = [torch.nn.Parameter(torch.zeros(1)) for _ in range(2)]
    opt = torch.optim.Adam([{'params': [p[0]], 'lr': lr}, {'params': [p[1]], 'lr': 0.1 * lr}])
    ref = torch.optim.lr_scheduler.SequentialLR(
        opt, [torch.optim.lr_scheduler.LinearLR(opt, start_factor=sc.lr_warmup_decay, total_iters=sc.warmup_epochs),
              torch.optim.lr_scheduler.CosineAnnealingLR(opt, T_max=sc.T_max - sc.warmup_epochs)],
        milestones=[sc.warmup_epochs])
    tr.optimizer = _Opt([lr, 0.1 * lr])
    _check_schedule(tr.get_scheduler(sc), opt, ref, tr.optimizer, cfg.train.epoch)

    # Baseline: the base Trainer's groups, criterion and CosineAnnealingLR(T_max, eta_min) (Examples/Baseline.py:30-37)
    cfg = _cfg('Baseline.yaml')
    tr = examples.BaselineTrainer.__new__(examples.BaselineTrainer)
    tr.config, tr.total_epoch, tr.model = cfg, cfg.train.epoch, _model('Baseline.yaml')
    for hook in ('get_criterion', 'get_optimizer', 'get_scheduler', 'param_groups', 'batch_training', 'get_dataloader'):
        assert getattr(examples.BaselineTrainer, hook) is getattr(examples.Trainer, hook), hook
    assert [[id(p) for p in g] for g, _ in tr.trained_groups()] == [[id(p) for p in tr.model.parameters()]]
    assert tr.get_criterion(cfg.train.criterion).label_smoothing == 0.1
    sc, lr = cfg.train.scheduler, cfg.train.optimizer.lr
    p = torch.nn.Parameter(torch.zeros(1))
    opt = torch.optim.Adam([p], lr=lr)
    ref = torch.optim.lr_scheduler.CosineAnnealingLR(opt, sc.T_max, sc.eta_min)
    tr.optimizer = _Opt([lr])
    _check_schedule(tr.get_scheduler(sc), opt, ref, tr.optimizer, cfg.train.epoch)


def test_baseline_transforms_equal_the_reference():
    from PIL import Image
    import detgen
    from hawkeye_b200 import examples
    tf = examples.BaselineTrainer.get_transformers(None, _cfg('Baseline.yaml').dataset.transformer)
    img = Image.fromarray((detgen.det_uniform((300, 260, 3), 7200).numpy() * 255).astype(np.uint8))
    for split in ('train', 'val'):
        torch.manual_seed(7201)
        t = tf[split](img)
        assert list(t.shape) == G[f'tf_{split}_shape'].tolist() == [3, 224, 224]
        assert np.array_equal(t.numpy()[:, ::8, ::8], G[f'tf_{split}_slice']), split
        assert np.abs(t.double().sum((1, 2)).numpy() - G[f'tf_{split}_sums']).max() < 1e-6 * 224 * 224, split


@pytest.fixture(scope='module')
def image_folder(tmp_path_factory):
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


def _loaders(cls, yaml, root, world, batch):
    cfg = _cfg(yaml)
    cfg.dataset.update(root_dir=root, meta_dir=root, batch_size=batch, num_workers=0)
    t = object.__new__(cls)
    t.config, t.world, t.rank, t.samplers = cfg, world, world - 1, {}
    return t.get_dataloader(cfg.dataset)


def test_pc_loaders_keep_each_rank_batch_even(image_folder):
    from hawkeye_b200 import examples
    one = _loaders(examples.PCResNetTrainer, 'PC_resnet50.yaml', image_folder, 1, 6)
    assert one['train'].batch_size == 6 and not one['train'].drop_last                # one GPU: the reference's loader
    two = _loaders(examples.PCResNetTrainer, 'PC_resnet50.yaml', image_folder, 2, 8)
    assert two['train'].batch_size == 4 and two['train'].drop_last and not two['val'].drop_last
    assert type(two['train'].sampler).__name__ == 'DistributedSampler'
    assert all(b['img'].shape[0] == 4 for b in two['train'])                         # 10 images per rank: 2 batches of 4
    assert len(two['train']) == 2
    with pytest.raises(ValueError, match='must be even'):
        _loaders(examples.PCResNetTrainer, 'PC_resnet50.yaml', image_folder, 2, 6)
    base = _loaders(examples.BaselineTrainer, 'Baseline.yaml', image_folder, 2, 6)
    assert [type(x).__name__ for x in base['train'].dataset.transform.transforms] == [
        'RandomResizedCrop', 'RandomHorizontalFlip', 'ToTensor', 'Normalize']
    assert [type(x).__name__ for x in base['val'].dataset.transform.transforms] == [
        'Resize', 'CenterCrop', 'ToTensor', 'Normalize']


def test_criterion_rejects_an_odd_batch():
    from hawkeye_b200.cfgnode import CfgNode
    from hawkeye_b200.losses import PairwiseConfusionLoss
    crit = PairwiseConfusionLoss(CfgNode({}))
    assert crit.lambda_a == 10
    with pytest.raises(ValueError, match='batch size'):
        crit(torch.zeros(3, 8), torch.zeros(3, dtype=torch.long))                   # raised before any launch


def test_hk_pc_loss_rejects_bad_arguments():
    from hawkeye_b200 import _lib
    lib = _lib.lib()
    buf = (ctypes.c_float * 64)()
    p = ctypes.addressof(buf)
    f = ctypes.c_float
    args = [p, p, p, p, p, 4, 4, f(0.1), f(10.0), f(1.0), None]
    for i in range(5):
        a = list(args)
        a[i] = None
        assert lib.hk_pc_loss(*a) == -1 and 'null' in lib.hk_last_error().decode(), i
    for B, K in ((5, 4), (3, 4), (1, 4), (0, 4), (-2, 4), (4, 0), (4, -1)):
        a = list(args)
        a[5], a[6] = B, K
        assert lib.hk_pc_loss(*a) == -1, (B, K)
    assert 'even' in lib.hk_last_error().decode()
