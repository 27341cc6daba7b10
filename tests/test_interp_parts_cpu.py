"""Interp-Parts without a GPU: the state layout and strict loads both ways, registration and the shipped yaml, the rejected
options, the fp64 oracle against fixtures of the unmodified reference (tests/golden/make_golden_interp_parts.py), the cached
Beta prior, the trainer's parameter groups and per-iteration cosine schedule, and the train transforms."""
import json
import os

import numpy as np
import pytest
import torch

import detgen
from conftest import load_golden, rel_l2
from oracle import interp_parts_oracle as O

G = load_golden('reference_interp_parts')
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _json(key):
    return json.loads(bytes(G[key]).decode())


def _net(layers=(3, 4, 23, 3), K=5):
    from hawkeye_b200.methods.interp_parts import ResNet
    return ResNet(list(layers), 200, K)


def test_state_layout_and_strict_loads():
    net = _net()
    assert [[k, list(v.shape)] for k, v in net.state_dict().items()] == _json('state_keys_json')
    assert sum(p.numel() for p in net.parameters()) == int(G['params_101'])
    sd = {k: torch.zeros(s) if not k.endswith('num_batches_tracked') else torch.tensor(0) for k, s in _json('state_keys_json')}
    net.load_state_dict(sd, strict=True)                                    # a reference checkpoint loads strictly here
    other = _net()
    other.load_state_dict(net.state_dict(), strict=True)                    # and this one's state has the same keys


def test_initialisers():
    net = _net((1, 1, 1))
    assert (net.grouping.weight >= 1e-5).all() and (net.grouping.smooth_factor == 0).all()
    for m in list(net.post_block) + list(net.attconv)[:2] + [net.layer1[0]]:
        assert (m.bn3.weight == 0).all()
    assert (net.groupingbn.weight == 1).all() and (net.groupingbn.bias == 0).all()


def test_registration_and_yaml(monkeypatch):
    monkeypatch.setenv('HAWKEYE_ALLOW_RANDOM_INIT', '1')
    from hawkeye_b200.config import load_config
    from hawkeye_b200.registry import MODEL
    import hawkeye_b200.methods  # noqa: F401
    assert 'IP_ResNet50' in MODEL and 'IP_ResNet101' in MODEL
    cfg = load_config(os.path.join(REPO, 'configs', 'InterpPartsNet.yaml'))
    net = MODEL.get(cfg.model.name)(cfg.model)
    assert net.n_parts == 5 and net.mylinear.out_features == 200
    assert sum(p.numel() for p in net.parameters()) == int(G['params_101'])
    assert cfg.dataset.batch_size == 16 and cfg.dataset.transformer.image_size == 448


def test_rejected_options():
    from hawkeye_b200 import _lib, ops_interp_parts as OP
    from hawkeye_b200.cfgnode import CfgNode
    from hawkeye_b200.losses import InterpPartsLoss
    with pytest.raises(_lib.HawkeyeLibError, match='num_parts=33'):
        _net((1, 1, 1), K=33)
    with pytest.raises(_lib.HawkeyeLibError, match='num_classes'):
        from hawkeye_b200.methods.interp_parts import ResNet
        ResNet([1, 1, 1], 201, 5)
    with pytest.raises(ValueError, match='radius'):
        InterpPartsLoss(CfgNode(dict(radius=-1)))
    with pytest.raises(_lib.HawkeyeLibError, match='radius=4'):
        OP.check_radius(4, 8, 9)
    OP.check_radius(3, 7, 9)


def test_oracle_against_fixtures():
    seed = int(G['unit_seed'])
    x, w, sf, Gw = (t.double() for t in (0.03 * detgen.det((4, 1024, 28, 28), seed), 0.03 * detgen.det((5, 1024, 1, 1), seed + 1),
                                         0.3 * detgen.det((5,), seed + 2), detgen.det((4, 1024, 5), seed + 3)))
    x.requires_grad_(True)
    w.requires_grad_(True)
    sf.requires_grad_(True)
    out, assign = O.grouping(x, w, sf)
    assert rel_l2(out.transpose(1, 2), G['unit_feats']) < 1e-5
    assert rel_l2(assign, G['unit_assign']) < 1e-5
    from hawkeye_b200.ops_interp_parts import beta_prior
    occ = O.occupancy(assign, O.gaussian(2, 0.4))
    shaping = O.shaping(occ, beta_prior(4, 1, 0.001))
    assert abs(shaping.item() - float(G['unit_shaping'])) < 1e-5 * abs(float(G['unit_shaping']))
    ((out.transpose(1, 2) * Gw).sum() + 0.5 * shaping).backward()
    assert rel_l2(x.grad[:, ::16], G['unit_dx_slice']) < 1e-3
    assert rel_l2(w.grad, G['unit_dweight']) < 1e-3
    assert rel_l2(sf.grad, G['unit_dsmooth']) < 1e-3


def test_prior_equals_reference():
    from hawkeye_b200.ops_interp_parts import beta_prior
    for i in range(5):
        n, a, b = G[f'prior_{i}_args']
        assert torch.equal(beta_prior(int(n), a, b), torch.from_numpy(G[f'prior_{i}']))


def test_prior_is_cached():
    from hawkeye_b200.cfgnode import CfgNode
    from hawkeye_b200.losses import InterpPartsLoss
    crit = InterpPartsLoss(CfgNode(dict(radius=2, std=0.4, num_parts=5, alpha=1, beta=0.001, coeff=0.5)))
    p = crit.prior(16, 'cpu')
    assert crit.prior(16, 'cpu') is p and crit.prior(8, 'cpu') is not p


def test_gaussian_taps_equal_reference_kernel():
    from hawkeye_b200.ops_interp_parts import gaussian_taps
    for r, s in ((2, 0.4), (0, 0.4), (3, 1.5)):
        assert torch.allclose(gaussian_taps(r, s).double(), O.gaussian(r, s).flatten(), rtol=1e-6, atol=1e-9)


class _Opt:
    def __init__(self, lrs):
        self.param_groups = [dict(lr=l, initial_lr=l) for l in lrs]


def test_per_iteration_cosine_matches_torch():
    from hawkeye_b200.train import _Cosine
    iters, epochs = 37, 9
    p = torch.nn.Parameter(torch.zeros(1))
    ref = torch.optim.SGD([{'params': [p], 'lr': 5e-4}, {'params': [torch.nn.Parameter(torch.zeros(1))], 'lr': 1e-2}],
                          lr=5e-4, momentum=0.9)
    sched = torch.optim.lr_scheduler.CosineAnnealingLR(ref, iters * epochs)
    opt = _Opt([5e-4, 1e-2])
    mine = _Cosine(opt, iters * epochs)
    for _ in range(iters * epochs):
        for a, b in zip(opt.param_groups, ref.param_groups):
            assert a['lr'] == pytest.approx(b['lr'], rel=1e-6, abs=1e-12)
        ref.step()
        sched.step()
        mine.step()


def test_trainer_groups():
    from hawkeye_b200.examples import ALL_TRAINERS, TRAINERS, InterpPartsNetTrainer
    assert ALL_TRAINERS['InterpPartsNet'] is InterpPartsNetTrainer and 'InterpPartsNet' not in TRAINERS
    net = _net((1, 1, 1))
    tr = InterpPartsNetTrainer.__new__(InterpPartsNetTrainer)
    tr.model = net
    (fine, m1), (scratch, m2) = tr.param_groups()
    assert (m1, m2) == (1.0, 20.0)
    names = {id(p): n for n, p in net.named_parameters()}
    assert {names[id(p)].split('.')[0] for p in fine} == {'conv1', 'bn1', 'layer1', 'layer2', 'layer3'}
    assert {names[id(p)].split('.')[0] for p in scratch} == {'grouping', 'post_block', 'attconv', 'groupingbn', 'mylinear'}
    assert len(fine) + len(scratch) == len(list(net.parameters()))


def test_train_transforms_equal_reference():
    """Examples/InterpPartsNet.py:17-34 restated with torchvision, under the same seeds."""
    from PIL import Image
    from torchvision import transforms as T
    from hawkeye_b200.cfgnode import CfgNode
    from hawkeye_b200.examples import InterpPartsNetTrainer
    cfg = CfgNode(dict(resize_size=80, image_size=64, p_erasing=0.5))
    norm = T.Normalize(mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225))
    ref = {'train': T.Compose([T.Resize(size=80), T.RandomHorizontalFlip(), T.ColorJitter(0.1), T.RandomCrop(size=64),
                               T.ToTensor(), norm, T.RandomErasing(0.5)]),
           'val': T.Compose([T.Resize(size=80), T.CenterCrop(size=64), T.ToTensor(), norm])}
    mine = InterpPartsNetTrainer.get_transformers(None, cfg)
    img = Image.fromarray((np.random.RandomState(3).rand(90, 120, 3) * 255).astype(np.uint8))
    for split in ('train', 'val'):
        for seed in range(4):
            torch.manual_seed(seed)
            a = mine[split](img)
            torch.manual_seed(seed)
            b = ref[split](img)
            assert a.shape == (3, 64, 64) and torch.equal(a, b)
