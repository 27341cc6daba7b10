"""CIN's training path without a GPU: the fp64 loss oracle against fixtures of the unmodified reference's CINLoss
(tests/golden/make_golden_cin_loss.py) on three label orders, the yaml, the criterion's parameters and checks, the trainer's
groups and schedule, and the new C entries' argument errors."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

import cin_inputs as I
from conftest import load_golden
from oracle import cin_oracle as O

G = load_golden('reference_cin_loss')
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
os.environ['HAWKEYE_ALLOW_RANDOM_INIT'] = '1'


def _rel(a, b):
    a, b = np.asarray(a, dtype=np.float64).ravel(), np.asarray(b, dtype=np.float64).ravel()
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30)


@pytest.fixture(scope='module')
def weights():
    st = I.h_state()
    return st['h.weight'].numpy(), st['h.bias'].numpy()


@pytest.mark.parametrize('name,pairs', [('balanced', 0), ('some', 4), ('allsame', 10)])
def test_oracle_matches_reference_loss(name, pairs, weights):
    w, _ = weights
    target = I.LABELS[name]
    z, zc = I.logits().numpy(), I.z_cci().numpy()
    loss, dz, dzc, dw, db = O.cin_loss(z, zc, target, w, I.ALPHA)
    term, l1, n, *_ = O.contrastive(zc, target, w, I.ALPHA)
    assert n == pairs == int(O.pair_mask(target).sum())
    # the reference in fp32 on the CPU against fp64: ~1e-7 relative, larger where the pair differences cancel
    assert abs(loss - G[f'{name}_loss']) <= 1e-5 * abs(G[f'{name}_loss'])
    assert abs((G[f'{name}_loss'] - G[f'{name}_ce']) - I.ALPHA * (l1 + l1 * l1)) <= 1e-5 * abs(G[f'{name}_loss'])
    assert _rel(dz, G[f'{name}_dz']) < 1e-5
    assert not np.any(db) and np.abs(G[f'{name}_db']).max() <= 1e-5 * max(np.abs(G[f'{name}_dw_rowsums']).max(), 1e-30)
    if pairs == 0:
        # no pair: the contrastive term and every gradient it sends are exactly zero, in the reference too (zeros, not None)
        assert term == 0.0 and not np.any(dzc) and not np.any(dw)
        for k in ('dzc_slice', 'dzc_sums', 'dw_slice', 'dw_rowsums', 'db'):
            assert not np.any(G[f'{name}_{k}']), k
        return
    assert _rel(dzc[:, ::64, ::7], G[f'{name}_dzc_slice']) < 1e-5
    assert _rel(dzc.sum((1, 2)), G[f'{name}_dzc_sums']) < 1e-4          # sums of +-dd rows: partly cancelling
    assert _rel(dw[::16, ::389], G[f'{name}_dw_slice']) < 1e-5
    assert _rel(dw.sum(1), G[f'{name}_dw_rowsums']) < 1e-5


def test_pair_mask_compares_against_one_label():
    assert O.pair_mask([0, 1, 0, 2, 0, 1]).tolist() == [False, False, False]         # target[3] = 2
    assert O.pair_mask([0, 0, 1, 0, 1, 1]).tolist() == [True, True, False]          # not element by element: [F, T, F]
    assert O.pair_mask(np.repeat(np.arange(3), 6)).sum() == 3                       # 3 x 6: target[9] = 1, pairs 6, 7, 8


def test_yaml_builds_cin_and_criterion():
    import hawkeye_b200 as hb
    from hawkeye_b200.config import load_config
    from hawkeye_b200.losses import CINLoss
    cfg = load_config(os.path.join(REPO, 'configs', 'CIN.yaml'))
    assert cfg.model.name == 'CIN' and cfg.dataset.n_classes * cfg.dataset.n_samples == 20
    assert cfg.train.optimizer.name == 'SGD' and 'momentum' not in cfg.train.optimizer
    net = hb.MODEL.get('CIN')(cfg.model)
    ref = json.loads(bytes(load_golden('reference_cin')['cin_state_keys_json']).decode())
    ref_params = sum(int(np.prod(s)) for k, s in ref.items()
                     if not k.endswith(('running_mean', 'running_var', 'num_batches_tracked')))
    assert sum(p.numel() for p in net.parameters()) == ref_params
    c = cfg.train.criterion
    crit = CINLoss(c)
    assert (crit.alpha, crit.beta, crit.channel, crit.feature_size, crit.r_channel) == (2.0, 0.5, 2048, 49, 512)
    assert list(crit.state_dict()) == ['h.weight', 'h.bias']
    assert sum(p.numel() for p in crit.parameters()) == 100352 * 512 + 512
    assert not crit.h.bias.any() and abs(crit.h.weight.std().item() / (2.0 / 100352) ** 0.5 - 1) < 0.01   # kaiming_normal_


def test_criterion_rejects_bad_sizes():
    from hawkeye_b200.cfgnode import CfgNode
    from hawkeye_b200.losses import CINLoss
    with pytest.raises(ValueError, match='r_channel'):
        CINLoss(CfgNode(dict(channel=8, feature_size=4, r_channel=6)))
    crit = CINLoss(CfgNode(dict(channel=8, feature_size=49, r_channel=4)))
    with pytest.raises(ValueError, match='feature_size'):                         # a 448x448 input: 14x14, not 7x7
        crit((torch.zeros(2, 4), torch.zeros(2, 8, 196)), torch.zeros(2, dtype=torch.long))


def test_trainer_registration_groups_and_schedule():
    from hawkeye_b200 import examples
    from hawkeye_b200.config import load_config
    from hawkeye_b200.losses import CINLoss
    assert examples.ALL_TRAINERS['CIN'] is examples.CINTrainer
    assert set(examples.TRAINERS) == {'BCNN', 'CBCNN', 'MPN', 'PeerLearning', 'OSMENet'}
    with pytest.raises(SystemExit, match='CIN'):
        examples.main(['nope'])
    from hawkeye_b200.cfgnode import CfgNode
    cfg = load_config(os.path.join(REPO, 'configs', 'CIN.yaml'))
    tr =examples.CINTrainer.__new__(examples.CINTrainer)
    tr.config, tr.total_epoch = cfg, cfg.train.epoch
    tr.model = torch.nn.Linear(8, 4)
    tr.criterion = CINLoss(CfgNode(dict(channel=2, feature_size=4, r_channel=4)))
    (mp, m0), (cp, m1) = tr.param_groups()
    assert (m0, m1) == (1.0, 1.0)
    assert [id(p) for p in mp] == [id(p) for p in tr.model.parameters()]
    assert [id(p) for p in cp] == [id(tr.criterion.h.weight), id(tr.criterion.h.bias)]

    sc = cfg.train.scheduler
    p = torch.nn.Parameter(torch.zeros(1))
    opt = torch.optim.SGD([p], lr=cfg.train.optimizer.lr)
    ref = torch.optim.lr_scheduler.SequentialLR(
        opt, [torch.optim.lr_scheduler.LinearLR(opt, start_factor=sc.lr_warmup_decay, total_iters=sc.warmup_epochs),
              torch.optim.lr_scheduler.CosineAnnealingLR(opt, T_max=sc.T_max - sc.warmup_epochs)],
        milestones=[sc.warmup_epochs])

    class _Opt:
        param_groups = [dict(initial_lr=cfg.train.optimizer.lr, lr=cfg.train.optimizer.lr)]

    tr.optimizer = _Opt()
    mine = tr.get_scheduler(sc)
    for epoch in range(cfg.train.epoch):
        assert abs(_Opt.param_groups[0]['lr'] - opt.param_groups[0]['lr']) < 1e-12, epoch
        opt.step()
        ref.step()
        mine.step()


def test_c_entries_reject_bad_arguments():
    from hawkeye_b200 import _lib
    lib = _lib.lib()
    buf = (ctypes.c_float * 64)()
    p = ctypes.addressof(buf)
    a = ctypes.c_float(2.0)
    assert lib.hk_cin_contrastive_loss(None, p, p, p, 4, 4, a, None) == -1
    assert lib.hk_cin_contrastive_loss(p, None, p, p, 4, 4, a, None) == -1
    assert lib.hk_cin_contrastive_loss(p, p, None, p, 4, 4, a, None) == -1
    assert lib.hk_cin_contrastive_loss(p, p, p, None, 4, 4, a, None) == -1
    assert lib.hk_cin_contrastive_loss(p, p, p, p, 5, 4, a, None) == -1
    assert 'even' in lib.hk_last_error().decode()
    assert lib.hk_cin_contrastive_loss(p, p, p, p, 0, 4, a, None) == -1
    assert lib.hk_cin_contrastive_loss(p, p, p, p, 4, 0, a, None) == -1
    assert lib.hk_cin_pair_diff_fwd(None, p, 4, 4, None) == -1 and lib.hk_cin_pair_diff_fwd(p, p, 3, 4, None) == -1
    assert lib.hk_cin_pair_diff_bwd(p, None, 4, 4, None) == -1 and lib.hk_cin_pair_diff_bwd(p, p, 7, 4, None) == -1
