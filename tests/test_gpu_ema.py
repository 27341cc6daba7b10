"""Model EMA on the device (``hk_ema_update``, ``hk_ema_swap``, ``engine.ModelEMA``) and in the trainers.

The restatement everything is held to is torch's own ``AveragedModel(m, avg_fn=lambda a, p, n: d * a + (1 - d) * p,
use_buffers=True)``, torchvision's ExponentialMovingAverage, run on a plain module that mirrors the model's parameters and
buffers in the order AveragedModel iterates them.  Every comparison is bit for bit."""
import logging

import pytest
import torch
import torch.nn as nn
from torch.optim.swa_utils import AveragedModel

import detgen
from step_check import no_host_sync
from hawkeye_b200 import engine, train as T
from hawkeye_b200.cfgnode import CfgNode

pytestmark = pytest.mark.gpu


def _tensors(model):
    return list(model.parameters()) + list(model.buffers())


class _Mirror(nn.Module):
    """model.parameters() then model.buffers() as the parameters and buffers of a plain module, which AveragedModel can
    deep-copy whatever the model holds."""

    def __init__(self, model):
        super().__init__()
        self.p = nn.ParameterList([nn.Parameter(p.detach().clone(), requires_grad=p.requires_grad)
                                   for p in model.parameters()])
        for i, b in enumerate(model.buffers()):
            self.register_buffer(f'b{i}', b.detach().clone())

    @torch.no_grad()
    def load(self, tensors):
        for d, s in zip(_tensors(self), tensors, strict=True):
            d.copy_(s)


def _reference(model, d):
    mirror = _Mirror(model)
    return mirror, AveragedModel(mirror, avg_fn=lambda a, p, n: d * a + (1 - d) * p, use_buffers=True)


def _ref_update(mirror, ref, model):
    mirror.load(_tensors(model))
    ref.update_parameters(mirror)


def _averaged(ema, model):
    with ema.swapped():
        return [t.detach().clone() for t in _tensors(model)]


def _assert_matches(ema, model, ref, what=''):
    ours, theirs = _averaged(ema, model), _tensors(ref.module)
    assert len(ours) == len(theirs)
    for i, (a, b) in enumerate(zip(ours, theirs)):
        assert a.dtype == b.dtype and torch.equal(a, b), f'{what}tensor {i} {tuple(a.shape)} {a.dtype}'
    assert int(ema.n_averaged) == int(ref.n_averaged), what


class _Segments(nn.Module):
    """Flat segments of 1, 3, 4, 5, 1023 and 4097 elements, a frozen parameter, BatchNorm (running statistics and the
    int64 num_batches_tracked) and a buffer that is not 16-byte aligned."""

    def __init__(self):
        super().__init__()
        self.w = nn.ParameterList([nn.Parameter(torch.randn(n)) for n in (1, 3, 4, 5, 1023, 4097)])
        self.frozen = nn.Parameter(torch.randn(7, 5), requires_grad=False)
        self.bn = nn.BatchNorm2d(6)
        self.register_buffer('odd', torch.randn(12)[1:])


def _segments():
    torch.manual_seed(0)
    m = _Segments().cuda()
    m.odd = torch.randn(12, device='cuda')[1:]              # .cuda() made it contiguous from 0: re-offset by 4 bytes
    assert m.odd.data_ptr() % 16
    return m, engine.FlatParams(m)


@torch.no_grad()
def _perturb(m, g):
    for p in m.parameters():
        p.add_(torch.randn(p.shape, generator=g, device='cuda'))
    m.odd.add_(torch.randn(m.odd.shape, generator=g, device='cuda'))
    m.bn.train()(torch.randn(4, 6, 3, 3, generator=g, device='cuda'))         # running stats and num_batches_tracked
    m.bn.num_batches_tracked.add_(int(torch.randint(0, 1 << 30, (1,), generator=g, device='cuda')))


@pytest.mark.parametrize('d', [0.7, T.model_ema_decay(0.99998, 32, 32, 30)])
def test_update_is_averaged_model_over_six_updates(d):
    m, flat = _segments()
    ema = engine.ModelEMA(m, flat, d)
    assert ema.nseg == 6          # flat, frozen, running_mean, running_var, num_batches_tracked, odd
    mirror, ref = _reference(m, d)
    g = torch.Generator(device='cuda').manual_seed(1)
    for k in range(6):
        _perturb(m, g)
        ema.update()
        _ref_update(mirror, ref, m)
        if k == 2:                                               # a reset in the middle: the next update copies again
            ema.reset()
            ref.n_averaged.fill_(0)
        if k == 4:                                               # and the warm-up reset after an update
            _perturb(m, g)
            ema.update(reset_after=True)
            _ref_update(mirror, ref, m)
            ref.n_averaged.fill_(0)
        _assert_matches(ema, m, ref, f'update {k}: ')


def test_update_over_the_bcnn_parameter_set():
    import hawkeye_b200 as hb
    torch.manual_seed(0)
    net = hb.MODEL.get('BCNN')(CfgNode(dict(name='BCNN', stage=2, num_classes=200))).cuda()
    flat = engine.FlatParams(net)
    assert flat.numel > 60_000_000
    d = T.model_ema_decay(0.99998, 32, 32, 30)
    ema = engine.ModelEMA(net, flat, d)
    mirror, ref = _reference(net, d)
    ema.update()                                                  # the copy
    _ref_update(mirror, ref, net)
    with torch.no_grad():
        flat.flat.add_(torch.randn_like(flat.flat), alpha=1e-3)
    ema.update()                                                  # the average
    _ref_update(mirror, ref, net)
    _assert_matches(ema, net, ref)


def _bits(t):
    return t.detach().view(torch.int32).clone() if t.dtype == torch.float32 else t.detach().clone()


def test_two_swaps_restore_every_bit():
    m, flat = _segments()
    ema = engine.ModelEMA(m, flat, 0.9)
    g = torch.Generator(device='cuda').manual_seed(2)
    ema.update()
    _perturb(m, g)
    ema.update()
    _perturb(m, g)
    with torch.no_grad():                                         # a NaN payload and a negative zero survive as bits
        m.w[4].view(torch.int32)[:2] = torch.tensor([0x7fc00123, -2 ** 31], dtype=torch.int32, device='cuda')
        ema.averages[0].view(torch.int32)[3] = 0x7f800001
    before = [_bits(t) for t in ema.model_tensors], [_bits(t) for t in ema.averages]
    ema.swap()
    for a, b in zip(ema.model_tensors, before[1]):
        assert torch.equal(_bits(a), b)
    for a, b in zip(ema.averages, before[0]):
        assert torch.equal(_bits(a), b)
    ema.swap()
    for now, then in zip((ema.model_tensors, ema.averages), before):
        for a, b in zip(now, then):
            assert torch.equal(_bits(a), b)


# ---------------------------------------------------------------------------------------------------- the trainers
def _trainer(monkeypatch, tmp_path, yaml='Baseline.yaml', name='Baseline', *, ema=None, graph=False, dataloaders=None,
             train=None, scheduler=None, experiment=None, model=None):
    """examples.ALL_TRAINERS[name] on configs/<yaml> with train.model_ema = ``ema``, random initialisation allowed, graph
    replay on or off and its log directory under tmp_path.  The other arguments replace entries of those sections."""
    import os
    from hawkeye_b200 import examples
    from hawkeye_b200.config import load_config
    monkeypatch.setenv('HAWKEYE_ALLOW_RANDOM_INIT', '1')
    monkeypatch.setenv('HK_CUDA_GRAPH', '1' if graph else '0')
    cfg = load_config(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'configs', yaml))
    cfg.experiment['log_dir'] = str(tmp_path)
    cfg.train['model_ema'] = CfgNode(dict(decay=0.99, steps=1) if ema is None else ema)
    for section, kv in ((cfg.train, train), (cfg.train.scheduler, scheduler), (cfg.experiment, experiment),
                        (cfg.model, model)):
        for k, v in (kv or {}).items():
            section[k] = v
    torch.manual_seed(0)
    tr = examples.ALL_TRAINERS[name](cfg, dataloaders={} if dataloaders is None else dataloaders)
    tr.model.train()
    return tr


def _batch(seed, n=8, classes=200):
    return dict(img=detgen.det((n, 3, 224, 224), seed).cuda(), label=detgen.det_labels(n, classes, seed + 1).cuda())


def test_baseline_training_follows_torchvisions_schedule(monkeypatch, tmp_path):
    """Two epochs of five batches, warm-up epochs 1, an update every 2 batches: the model after every optimizer step, fed
    to AveragedModel on torchvision's schedule (updates at batches 0, 2 and 4 of each epoch, the counter reset after each
    update of epoch 0), gives the trainer's average bit for bit."""
    loaders = {'train': [_batch(9000 + 2 * i) for i in range(5)], 'val': [_batch(9100)]}
    tr = _trainer(monkeypatch, tmp_path, ema=dict(decay=0.99, steps=2), train=dict(epoch=2),
                  scheduler=dict(warmup_epochs=1), dataloaders=loaders)
    assert tr.ema_steps == 2 and tr.ema_warmup == 1
    d = T.model_ema_decay(0.99, 2, 24, 2)
    assert tr.ema.decay == d and 0 < d < 1
    mirror, ref = _reference(tr.model, d)
    snaps, after = [], tr.after_optimizer_step

    def record():
        after()
        snaps.append((tr.epoch, tr.epoch_batch, [t.detach().clone() for t in _tensors(tr.model)]))
    tr.after_optimizer_step = record
    tr.train()
    assert [(e, i) for e, i, _ in snaps] == [(e, i) for e in range(2) for i in range(5)]
    for epoch, i, tensors in snaps:
        if i % 2 == 0:
            mirror.load(tensors)
            ref.update_parameters(mirror)
            if epoch < 1:
                ref.n_averaged.fill_(0)
    assert int(ref.n_averaged) == 3                    # epoch 1: the copy at batch 0, then batches 2 and 4
    _assert_matches(tr.ema, tr.model, ref)
    assert tr.acc_ema is not None and 0 <= tr.acc_ema <= 100


def test_prototree_average_includes_the_leaf_update(monkeypatch, tmp_path):
    """Derivative-free leaves: the average taken after a step holds that step's leaf update."""
    tr = _trainer(monkeypatch, tmp_path, 'ProtoTreeNet.yaml', 'ProtoTreeNet', ema=dict(decay=0.9, steps=1),
                  model=dict(backbone=CfgNode(dict(name='resnet50', pretrain=''))))
    tr.num_batches = 10
    tr.ema_warmup = 0                 # the yaml's 5 warm-up epochs would reset the counter after every update of epoch 0
    leaves = tr.model.tree.leaf_params
    assert not leaves.requires_grad
    d = tr.ema.decay
    tr.on_start_epoch(None)
    seen = []
    for k in range(2):
        before = leaves.detach().clone()
        tr.batch_training(_batch(9200 + 2 * k, n=16))
        assert not torch.equal(leaves, before)
        seen.append(leaves.detach().clone())
    expected = d * seen[0] + (1 - d) * seen[1]
    sd = tr.ema.state_dict()
    keys = ['module.tree.' + k for k in tr.model.tree._leaf_keys]
    assert all(k in sd for k in keys) and 'module.tree.leaf_params' not in sd
    assert torch.equal(torch.stack([sd[k] for k in keys]), expected.cpu())
    assert int(sd['n_averaged']) == 2


def test_ema_step_has_no_host_sync(monkeypatch, tmp_path):
    tr = _trainer(monkeypatch, tmp_path)
    for k in range(2):                                              # warm-up: workspaces, first-call attributes
        tr.batch_training(_batch(9300 + 2 * k))
    batch = _batch(9310)
    torch.cuda.synchronize()
    with no_host_sync():
        tr.batch_training(batch)                                    # the fourth read-back slot of eight: no wrap
    assert int(tr.ema.n_averaged) == 3


def test_graph_replay_after_ema_validation(monkeypatch, tmp_path):
    """With cuda_graph the step is captured; an EMA validation then leaves the model's weights and buffers bit for bit as
    they were, and the replayed step gives the eager step's loss from the same state."""
    tr = _trainer(monkeypatch, tmp_path, graph=True, dataloaders={'val': [_batch(9400)]})
    batches = [_batch(9410 + 2 * i) for i in range(4)]
    for b in batches:
        tr.batch_training(b)
    assert tr._graph is not None
    state = {k: v.detach().clone() for k, v in tr.model.state_dict().items()}
    flat = tr.flat.flat.clone()
    acc = tr.validate_ema()
    assert 0 <= acc <= 100 and tr.model.training
    for k, v in tr.model.state_dict().items():
        assert torch.equal(_bits(v), _bits(state[k])), k
    assert torch.equal(_bits(tr.flat.flat), _bits(flat))
    x, y = batches[0]['img'], batches[0]['label']
    replayed = float(tr._graph_step(x, y)[1].item())
    tr.model.load_state_dict(state)                                # the replay's forward moved the BN running stats
    eager = float(tr.eager_step(x, y)[1].item())
    assert replayed == eager


def test_acc_ema_is_the_testers_accuracy_on_best_model_ema(monkeypatch, tmp_path):
    from hawkeye_b200.test import Tester
    val = [_batch(9500, classes=4)]
    tr = _trainer(monkeypatch, tmp_path, train=dict(epoch=6), model=dict(num_classes=4),
                  dataloaders={'train': [_batch(9510, classes=4)], 'val': val})
    tr.train()
    path = tmp_path / tr.config.experiment.name / 'best_model_ema.pth'
    assert path.exists()
    saved, now = torch.load(path), tr.ema.model_state_dict()
    assert list(saved) == list(now) and all(torch.equal(saved[k], now[k]) for k in now)
    cfg = CfgNode(dict(experiment=dict(name='t', cuda=[0]), dataset=dict(batch_size=8, num_workers=0,
                                                                         transformer=dict(resize_size=256, image_size=224)),
                       model=dict(name='ResNet50', num_classes=4, load=str(path))))
    assert Tester(cfg, dataloader=val).test() == tr.acc_ema
    # labels half right for the average: both score 50 %
    with tr.ema.swapped(), torch.no_grad():
        pred = tr.model.eval()(val[0]['img']).argmax(1)
    tr.model.train()
    val[0]['label'] = torch.where(torch.arange(8, device='cuda') % 2 == 0, pred, (pred + 1) % 4)
    assert tr.validate_ema() == 50.0 and Tester(cfg, dataloader=val).test() == 50.0


def test_resume_restores_the_average_and_its_counter(monkeypatch, tmp_path, caplog):
    tr = _trainer(monkeypatch, tmp_path)
    for k in range(3):
        tr.batch_training(_batch(9600 + 2 * k))
    path = tr.save_checkpoint()
    want = tr.ema.state_dict()
    assert int(want['n_averaged']) == 3 and list(torch.load(path)['model_ema']) == list(want)
    back = _trainer(monkeypatch, tmp_path, experiment=dict(resume=path))
    got = back.ema.state_dict()
    assert list(got) == list(want) and all(torch.equal(got[k], want[k]) for k in want)
    # a checkpoint without the average: it starts from the restored weights with the counter at 0
    ck = torch.load(path)
    del ck['model_ema']
    with caplog.at_level(logging.WARNING, logger='hawkeye_b200'):
        back.restore_checkpoint(ck, path)
    assert 'no model_ema' in caplog.text
    got = back.ema.state_dict()
    assert int(got['n_averaged']) == 0
    assert all(torch.equal(got['module.' + k], v) for k, v in ck['model'].items())
