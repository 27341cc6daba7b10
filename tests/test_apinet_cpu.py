"""APINet on CPU: the registry model against the reference's state_dict layout, APINetTrainer's learning-rate sequence against
torch's own schedulers with the reference's backbone freeze, the numpy dropout hash, and the fp64 oracle against the fixtures
of the unmodified reference (tests/golden/make_golden_apinet.py)."""
import json
import os

import numpy as np
import torch

from conftest import load_golden, rel_l2
from oracle import apinet_oracle as A

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = load_golden('reference_apinet')


def _ref_layout():
    return json.loads(bytes(G['state_keys_json']).decode())


def _net(monkeypatch):
    monkeypatch.setenv('HAWKEYE_ALLOW_RANDOM_INIT', '1')
    import hawkeye_b200 as hb
    from hawkeye_b200.config import load_config
    cfg = load_config(os.path.join(REPO, 'configs', 'APINet.yaml'))
    return hb.MODEL.get(cfg.model.name)(cfg.model), cfg


def test_yaml_builds_apinet_with_reference_layout(monkeypatch):
    net, cfg = _net(monkeypatch)
    ref = _ref_layout()
    assert {k: list(v.shape) for k, v in net.state_dict().items()} == ref
    n_ref = sum(int(np.prod(s)) for k, s in ref.items() if not k.endswith(('running_mean', 'running_var', 'num_batches_tracked')))
    assert sum(p.numel() for p in net.parameters()) == n_ref
    for attr in ('backbone', 'avg', 'map1', 'map2', 'fc', 'drop', 'sigmoid'):
        assert hasattr(net, attr)
    assert net.drop.p == 0.5 and cfg.dataset.n_classes * cfg.dataset.n_samples == 40
    sd = {k: torch.full(s, 0.25) if not k.endswith('num_batches_tracked') else torch.tensor(3) for k, s in ref.items()}
    net.load_state_dict(sd, strict=True)                                    # a reference checkpoint loads as is
    assert torch.equal(net.fc.weight, torch.full((200, 2048), 0.25))


def test_apinet_rejects_num_classes_off_the_tma_pitch(monkeypatch):
    import pytest
    import hawkeye_b200 as hb
    monkeypatch.setenv('HAWKEYE_ALLOW_RANDOM_INIT', '1')

    class Cfg(dict):
        __getattr__ = dict.__getitem__
    with pytest.raises(hb._lib.HawkeyeLibError):
        hb.MODEL.get('APINet')(Cfg(name='APINet', num_classes=202))


def test_apinet_trainer_lr_follows_torch_with_frozen_backbone(monkeypatch):
    """Examples/APINet.py: Adam over (backbone, rest) at config.lr, SequentialLR(LinearLR, CosineAnnealingLR), and
    on_start_epoch setting group 0's lr to 0 at epoch 0 (a no-op re-assignment at epoch 8)."""
    from hawkeye_b200 import examples
    from hawkeye_b200.config import load_config
    cfg = load_config(os.path.join(REPO, 'configs', 'APINet.yaml'))
    sc, lr = cfg.train.scheduler, cfg.train.optimizer.lr
    ps = [torch.nn.Parameter(torch.zeros(1)) for _ in range(2)]
    opt = torch.optim.Adam([dict(params=[ps[0]], lr=lr), dict(params=[ps[1]], lr=lr)], weight_decay=2e-8)
    sch = torch.optim.lr_scheduler.SequentialLR(
        opt, schedulers=[torch.optim.lr_scheduler.LinearLR(opt, start_factor=sc.lr_warmup_decay, total_iters=sc.warmup_epochs),
                         torch.optim.lr_scheduler.CosineAnnealingLR(opt, T_max=sc.T_max - sc.warmup_epochs)],
        milestones=[sc.warmup_epochs])

    class FakeOpt:
        param_groups = [dict(lr=lr, initial_lr=lr), dict(lr=lr, initial_lr=lr)]
    t = object.__new__(examples.APINetTrainer)
    t.optimizer, t.total_epoch = FakeOpt(), cfg.train.epoch
    ours = t.get_scheduler(sc)
    for epoch in range(20):
        if epoch == 0:                                                      # Examples/APINet.py:86-93
            opt.param_groups[0]['lr'] = 0
        elif epoch == 8:
            opt.param_groups[0]['lr'] = opt.param_groups[0]['lr']
        want = [g['lr'] for g in opt.param_groups]
        got = [g['lr'] for g in t.optimizer.param_groups]
        assert np.allclose(got, want, rtol=1e-12, atol=0), (epoch, got, want)
        assert (got[0] == 0) == (want[0] == 0)
        opt.step()
        sch.step()
        ours.step()


def test_apinet_trainer_groups_and_cli(monkeypatch):
    from hawkeye_b200 import examples
    net, cfg = _net(monkeypatch)
    t = object.__new__(examples.APINetTrainer)
    t.model = net
    groups = t.param_groups()
    assert [m for _, m in groups] == [1.0, 1.0]
    assert sum(p.numel() for p in groups[0][0]) == sum(p.numel() for p in net.backbone.parameters())
    assert sum(p.numel() for g, _ in groups for p in g) == sum(p.numel() for p in net.parameters())
    assert t.meter_counts(40) == (320, 160)                                 # Examples/APINet.py:74-77
    assert examples.ALL_TRAINERS['APINet'] is examples.APINetTrainer
    assert type(t.get_criterion(cfg.train.criterion)).__name__ == 'APINetLoss'


def test_dropout_hash_keep_fraction_and_calls():
    n, p = 10 ** 6, 0.5
    k0 = A.dropout_keep(1234, 0, (n,), p)
    sigma = (p * (1 - p) / n) ** 0.5
    assert abs(k0.mean() - 0.5) < 4 * sigma
    k1 = A.dropout_keep(1234, 1, (n,), p)
    k2 = A.dropout_keep(1235, 0, (n,), p)
    assert 0.45 < (k0 != k1).mean() < 0.55 and 0.45 < (k0 != k2).mean() < 0.55
    assert np.array_equal(k0, A.dropout_keep(1234, 0, (n,), p))
    assert A.dropout_keep(1234, 0, (1000,), 0.0).all()
    assert abs(A.dropout_keep(99, 3, (n,), 0.25).mean() - 0.75) < 4 * (0.1875 / n) ** 0.5


def test_oracle_pairs_match_reference_get_pairs():
    for tag in ('single', 'ties', 'alldiff', 'allsame', 'n40'):
        intra, inter, _ = A.apinet_pairs(G[f'pairs_{tag}_emb'], G[f'pairs_{tag}_labels'])
        assert np.array_equal(intra, G[f'pairs_{tag}_intra']), tag
        assert np.array_equal(inter, G[f'pairs_{tag}_inter']), tag
    assert G['pairs_single_intra'][2] == 0 and G['pairs_alldiff_intra'].tolist() == [0] * 5
    assert G['pairs_allsame_inter'].tolist() == [0] * 5


def test_oracle_head_and_loss_match_reference():
    import detgen
    import torch.nn as nn
    n = 8
    st = {k: torch.as_tensor(v) for k, v in detgen.state_like(nn.ModuleDict(dict(
        map1=nn.Linear(4096, 512), map2=nn.Linear(512, 2048), fc=nn.Linear(2048, 200)))).items()}
    conv = detgen.det((n, 2048, 7, 7), 402, positive=True).double().requires_grad_(True)
    pool = conv.reshape(n, 2048, 49).mean(2)
    lab = torch.arange(4).repeat_interleave(2)
    intra, inter, _ = A.apinet_pairs(pool.detach(), lab)
    _, logits = A.apinet_head(pool, intra, inter, st)
    assert rel_l2(logits[:4 * n].detach(), G['head_self']) < 1e-5 and rel_l2(logits[4 * n:].detach(), G['head_other']) < 1e-5
    r = torch.cat([detgen.det((4 * n, 200), 403), detgen.det((4 * n, 200), 404)]).double()
    (logits * r).sum().backward()
    assert rel_l2(conv.grad, G['head_dconv']) < 1e-5
    z = torch.cat([torch.as_tensor(G['loss_self']), torch.as_tensor(G['loss_other'])]).double().requires_grad_(True)
    l1, l2 = torch.as_tensor(G['loss_labels1']), torch.as_tensor(G['loss_labels2'])
    loss = A.apinet_loss(z, torch.cat([l1, l2, l1, l2]))
    loss.backward()
    assert abs(loss.item() - float(G['loss_value'])) < 1e-5 * abs(float(G['loss_value']))
    R = z.shape[0] // 2
    assert rel_l2(z.grad[:R], G['loss_dself']) < 1e-5 and rel_l2(z.grad[R:], G['loss_dother']) < 1e-5
