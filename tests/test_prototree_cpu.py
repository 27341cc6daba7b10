"""ProtoTree without a GPU: the 832-key state_dict layout and a strict load of the reference's keys, the iNat renaming, the
rejected options, the fp64 oracle against fixtures of the unmodified reference (tests/golden/make_golden_prototree.py), the
warm-up + cosine schedule against torch's SequentialLR, and the trainer's parameter groups."""
import json
import os

import pytest
import torch

from conftest import load_golden, rel_l2
from oracle import prototree_oracle as O
from prototree_inputs import theta0, tree_inputs

G = load_golden('reference_prototree')
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class Cfg(dict):
    __getattr__ = dict.__getitem__


def _cfg(**kw):
    base = dict(name='ProtoTreeNet', num_classes=200, height=9, W1=1, H1=1, num_features=256,
                backbone=Cfg(name='resnet50', pretrain=''))
    base.update(kw)
    return Cfg(base)


@pytest.fixture
def net(monkeypatch):
    monkeypatch.setenv('HAWKEYE_ALLOW_RANDOM_INIT', '1')
    import hawkeye_b200 as hb
    return hb.MODEL.get('ProtoTreeNet')(_cfg())


def test_state_dict_layout_and_strict_load(net):
    ref = json.loads(G['state_keys_json'].tobytes())
    ours = [[k, list(v.shape)] for k, v in net.state_dict().items()]
    assert len(ours) == 832 and ours == ref                          # same keys, shapes and order
    assert sum(k.endswith('._dist_params') for k, _ in ours) == 512
    sd = {k: torch.randn(s) if k.startswith('tree.') else v for (k, s), v in zip(ref, net.state_dict().values())}
    net.load_state_dict(sd, strict=True)
    theta = net.tree.leaf_params
    assert theta.shape == (512, 200)
    assert torch.equal(theta[0], sd['tree._root' + '.l' * 9 + '._dist_params'])
    assert torch.equal(theta[-1], sd['tree._root' + '.r' * 9 + '._dist_params'])
    assert torch.equal(net.state_dict()['tree._root.l.l.l.l.l.l.l.l.r._dist_params'], theta[1])
    assert not theta.requires_grad
    for k, v in net.state_dict().items():
        assert torch.equal(v, sd[k]), k


def test_inat_renaming(tmp_path, monkeypatch):
    monkeypatch.setenv('HAWKEYE_ALLOW_RANDOM_INIT', '1')
    from hawkeye_b200.methods import prototree
    keys = json.loads(G['inat_keys_json'].tobytes())
    sd = {k: torch.zeros(1) for k in keys}
    p = tmp_path / 'inat.pth'
    torch.save(sd, p)
    assert sorted(prototree.inat_resnet50_state(str(p))) == json.loads(G['inat_renamed_json'].tobytes())
    # through the model: cb_block lands in layer4.2 (trunk index 7), module.backbone.bn1 in trunk index 1
    from hawkeye_b200.backbone.resnet import resnet50
    donor = resnet50().state_dict()
    names = ['conv1', 'bn1', 'relu', 'maxpool', 'layer1', 'layer2', 'layer3', 'layer4']
    full = {}
    for k, v in donor.items():
        head, rest = k.split('.', 1)
        name = names[int(head)] + '.' + rest
        name = name.replace('layer4.2.', 'cb_block.')
        full['module.backbone.' + name] = torch.full_like(v, 0.25) if v.is_floating_point() else v
    full['module.backbone.rb_block.conv1.weight'] = torch.zeros(3)
    full['module.classifier.weight'] = torch.zeros(2, 2)
    torch.save(full, p)
    import hawkeye_b200 as hb
    net = hb.MODEL.get('ProtoTreeNet')(_cfg(backbone=Cfg(name='resnet50', pretrain=str(p))))
    assert (net.backbone[7][2].conv1.weight == 0.25).all() and (net.backbone[1].running_mean == 0.25).all()


def test_rejected_options(monkeypatch):
    monkeypatch.setenv('HAWKEYE_ALLOW_RANDOM_INIT', '1')
    import hawkeye_b200 as hb
    from hawkeye_b200 import _lib
    for k in ('log_probabilities', 'kontschieder_normalization', 'kontschieder_train'):
        with pytest.raises(_lib.HawkeyeLibError, match=k):
            hb.MODEL.get('ProtoTreeNet')(_cfg(**{k: True}))
    for k in ('W1', 'H1'):
        with pytest.raises(_lib.HawkeyeLibError, match='W1 x H1'):
            hb.MODEL.get('ProtoTreeNet')(_cfg(**{k: 2}))
    with pytest.raises(_lib.HawkeyeLibError, match='height=13'):
        hb.MODEL.get('ProtoTreeNet')(_cfg(height=13))
    with pytest.raises(_lib.HawkeyeLibError, match='num_classes=202'):
        hb.MODEL.get('ProtoTreeNet')(_cfg(num_classes=202))
    with pytest.raises(_lib.HawkeyeLibError, match=r'model\.backbone\.pretrain'):
        hb.MODEL.get('ProtoTreeNet')(_cfg(backbone=Cfg(name='resnet50', pretrain='/nonexistent/inat.pth')))
    net = hb.MODEL.get('ProtoTreeNet')(_cfg(height=2))
    for s in ('sample_max', 'greedy'):
        with pytest.raises(_lib.HawkeyeLibError, match=s):
            net.tree(torch.zeros(1), torch.zeros(1, 256, 1, 1), sampling_strategy=s)


def test_tree_layout_matches_reference_numbering():
    from hawkeye_b200.methods.prototree import tree_layout
    for h in (1, 2, 3, 9):
        branches, leaves, keys = tree_layout(h)
        nodes = O.layout(h)
        assert branches == [i for i, _, k, _, _ in nodes if k == 'b'] and leaves == O.leaf_indices(h)
        assert sorted(branches + leaves) == list(range(2 ** (h + 1) - 1))
    assert tree_layout(1)[2] == ['_root.l._dist_params', '_root.r._dist_params']


@pytest.mark.parametrize('tag', ['tree', 'dfo_off'])
def test_oracle_against_reference(tag):
    feat, protos, theta, labels = (t.double() if t.is_floating_point() else t for t in tree_inputs(G, tag))
    feat.requires_grad_(True)
    protos = protos.view(511, 256).requires_grad_(True)
    theta.requires_grad_(True)
    z = feat.permute(0, 2, 3, 1).reshape(4, 49, 256)
    mind, _ = O.distances(z, protos)
    pred, ps, pa = O.route(mind, theta, 9)
    loss = O.nll(pred, labels)
    loss.backward()
    # the reference forms |x|^2 + |p|^2 - 2 x.p in fp32 (l2conv.py:41-59): about 1e-6 off the direct distance, and its
    # gradients at the minimum carry that cancellation
    assert rel_l2(mind.detach(), G[f'{tag}_mind']) < 1e-5
    assert rel_l2(ps.detach(), G[f'{tag}_ps']) < 1e-5 and rel_l2(pa.detach(), G[f'{tag}_pa']) < 1e-5
    assert rel_l2(pred.detach(), G[f'{tag}_pred']) < 1e-5
    assert abs(loss.item() - float(G[f'{tag}_loss'])) < 1e-5
    assert rel_l2(feat.grad[:, ::4], G[f'{tag}_dfeat_slice']) < 1e-3
    assert rel_l2(protos.grad[:, ::8], G[f'{tag}_dprotos_slice'].reshape(511, -1)) < 1e-3
    if tag == 'dfo_off':
        assert rel_l2(theta.grad[::4], G['dfo_off_dtheta_rows']) < 1e-5


def test_oracle_leaf_update_against_reference():
    feat, protos, theta, labels = (t.double() if t.is_floating_point() else t for t in tree_inputs(G, 'tree'))
    z = feat.permute(0, 2, 3, 1).reshape(4, 49, 256)
    mind, _ = O.distances(z, protos.view(511, 256))
    pred, _, pa = O.route(mind, theta, 9)
    new = O.leaf_update(theta, theta0(512).double(), pa[:, O.leaf_indices(9)], pred, labels, int(G['upd_num_batches']))
    assert rel_l2(new[::4], G['upd_theta_rows']) < 1e-6


def test_cosine_matches_sequential_lr():
    from hawkeye_b200.config import load_config
    from hawkeye_b200.examples import _warmup_cosine
    cfg = load_config(os.path.join(REPO, 'configs', 'ProtoTreeNet.yaml'))
    sc = cfg.train.scheduler
    p = torch.nn.Parameter(torch.zeros(1))
    opt = torch.optim.AdamW([{'params': [p], 'lr': 0.01 * cfg.train.optimizer.lr},
                             {'params': [torch.nn.Parameter(torch.zeros(1))], 'lr': cfg.train.optimizer.lr}],
                            lr=cfg.train.optimizer.lr)
    ref = torch.optim.lr_scheduler.SequentialLR(
        opt, [torch.optim.lr_scheduler.LinearLR(opt, start_factor=sc.lr_warmup_decay, total_iters=sc.warmup_epochs),
              torch.optim.lr_scheduler.CosineAnnealingLR(opt, T_max=sc.T_max - sc.warmup_epochs)],
        milestones=[sc.warmup_epochs])

    class Opt:
        param_groups = [dict(initial_lr=g['initial_lr']) for g in opt.param_groups]
    ours = _warmup_cosine(Opt, sc, cfg.train.epoch)
    for e in range(cfg.train.epoch):
        for a, b in zip(Opt.param_groups, opt.param_groups):
            assert abs(a['lr'] - b['lr']) <= 1e-9 + 1e-6 * b['lr'], (e, a['lr'], b['lr'])
        opt.step()
        ref.step()
        ours.step()


def test_trainer_groups_and_learning_rates(net):
    from hawkeye_b200.examples import ProtoTreeTrainer

    class T(ProtoTreeTrainer):
        def __init__(self, model, **model_cfg):       # the group and optimizer logic only: no device, no data
            import yaml
            from hawkeye_b200.cfgnode import CfgNode
            self.config = CfgNode(yaml.safe_load(open(os.path.join(REPO, 'configs', 'ProtoTreeNet.yaml'))))
            self.config.model.update(model_cfg)
            self.model = model
    tr = T(net)
    groups = tr.param_groups()
    names = {id(p): n for n, p in net.named_parameters()}
    assert [m for _, m in groups] == [0.01, 1.0, 1.0, 1.0]
    assert all(n.startswith('backbone.') and '7.2' not in n for n in (names[id(p)] for p in groups[0][0]))
    assert {names[id(p)] for p in groups[1][0]} == {n for n in names.values() if n.startswith('backbone.7.2.')}
    assert [names[id(p)] for p in groups[2][0]] == ['neck_conv.0.weight']
    assert [names[id(p)] for p in groups[3][0]] == ['tree.prototype_layer.prototype_vectors']
    assert len(groups[0][0]) + len(groups[1][0]) == 159               # every trunk parameter trains: nothing is frozen
    tr.config.train.optimizer.lr_pi = 0.05
    tr.config.model.disable_derivative_free_leaf_optim = True
    assert groups != tr.param_groups() and tr.param_groups()[4][1] == pytest.approx(50.0)
    tr.config.model.disable_derivative_free_leaf_optim = False
    for name, wd in (('SGD', 0.0), ('AdamW', 1e-4)):
        tr.config.train.optimizer.name, tr.config.train.optimizer.weight_decay = name, wd
        with pytest.raises(ValueError, match=name):
            tr.get_optimizer(tr.config.train.optimizer)


def test_trainer_is_registered():
    from hawkeye_b200 import examples
    assert examples.ALL_TRAINERS['ProtoTreeNet'] is examples.ProtoTreeTrainer and 'ProtoTreeNet' not in examples.TRAINERS
