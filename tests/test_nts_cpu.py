"""NTS-Net without a GPU: the state layout and strict loads, the anchors and the survivor bound, the fp64 oracle's NMS, crop
and loss against the unmodified reference (fixtures from tests/golden/make_golden_nts.py, and torch's own interpolate), the
rejected options, the shipped yaml, the trainer's schedule against torch's SequentialLR, and the C entries' argument
errors (nothing launched)."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import nts_inputs
from conftest import load_golden
from oracle import nts_oracle as O

G = load_golden('reference_nts')
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cfg(**kw):
    from hawkeye_b200.cfgnode import CfgNode
    return CfgNode(dict(dict(proposal_num=6, cat_num=4, image_size=224), **kw))


def _net(monkeypatch, **kw):
    monkeypatch.setenv('HAWKEYE_ALLOW_RANDOM_INIT', '1')
    from hawkeye_b200.methods.nts import NTSNet
    return NTSNet(_cfg(**kw))


def test_state_layout_and_strict_loads(monkeypatch):
    net = _net(monkeypatch)
    keys = json.loads(bytes(G['state_keys_json']).decode())
    assert len(keys) == 336
    assert [[k, list(v.shape)] for k, v in net.state_dict().items()] == keys
    assert sum(p.numel() for p in net.parameters()) == int(G['params'])
    sd = {k: torch.zeros(s) if not k.endswith('num_batches_tracked') else torch.tensor(0) for k, s in keys}
    net.load_state_dict(sd, strict=True)
    assert net.pretrained_model.drop.p == 0.5 and net.edge_anchors.dtype == torch.int32


@pytest.mark.parametrize('size,A,bound', [(224, 426, 8), (448, 1614, 26)])
def test_anchors_and_survivor_bound(size, A, bound):
    from hawkeye_b200.methods.nts import edge_anchors, survivor_bound
    a = edge_anchors(size)
    assert a.shape == (A, 4) and np.array_equal(a, G[f'anchors_{size}'])
    assert survivor_bound(a) == bound


@pytest.mark.parametrize('size', [224, 448])
def test_oracle_nms_equals_hard_nms(size):
    anchors = G[f'anchors_{size}']
    T = nts_inputs.NMS_TOPN[size]
    assert len(nts_inputs.quarter_pairs(anchors)) == {224: 336, 448: 1456}[size]
    picks = G[f'nms_{size}']
    assert picks.shape == (nts_inputs.NMS_VECTORS, T)
    for k in range(nts_inputs.NMS_VECTORS):
        s = nts_inputs.nms_scores(anchors, k)
        assert len(np.unique(s)) == len(s)
        assert np.array_equal(O.hard_nms(s, anchors, T), picks[k]), k


def test_quarter_pairs_reach_the_top():
    anchors = G['anchors_224']
    pairs = {tuple(p) for p in nts_inputs.quarter_pairs(anchors)}
    s = nts_inputs.nms_scores(anchors, 1)
    top = np.argsort(-s)[:2]
    assert tuple(top) in pairs
    assert top[1] not in O.hard_nms(s, anchors, 8)            # IoU exactly 0.25 suppresses


def test_oracle_crop_equals_pad_and_interpolate():
    from hawkeye_b200.methods.nts import edge_anchors
    anchors = edge_anchors(224)
    rs = np.random.RandomState(5)
    x = torch.from_numpy(rs.standard_normal((2, 3, 224, 224)))
    boxes = anchors[rs.choice(len(anchors), (2, 3))]
    xp = F.pad(x, (224, 224, 224, 224))
    ref = torch.stack([F.interpolate(xp[n:n + 1, :, y0:y1, x0:x1], size=(224, 224), mode='bilinear', align_corners=True)[0]
                       for n in range(2) for y0, x0, y1, x1 in boxes[n].tolist()])
    assert (O.crop(x, boxes) - ref).abs().max() < 1e-12


def test_oracle_loss_equals_reference_restated():
    rs = np.random.RandomState(6)
    B, T = 3, 6
    raw, concat = (torch.from_numpy(rs.standard_normal((B, 200))) for _ in range(2))
    part = torch.from_numpy(rs.standard_normal((B, T, 200)))
    prob = torch.from_numpy(rs.standard_normal((B, T)))
    labels = torch.from_numpy(rs.randint(0, 200, B))
    # NTS_loss.py restated with torch, row by row as the reference loops
    rows = labels.unsqueeze(1).repeat(1, T).view(-1)
    lsm = F.log_softmax(part.view(B * T, -1), -1)
    L = torch.stack([-lsm[i][rows[i]] for i in range(B * T)]).view(B, T)
    rank = torch.zeros(1, dtype=torch.float64)
    for i in range(T):
        rank += F.relu((1 - prob[:, i:i + 1] + prob) * (L > L[:, i:i + 1]).double()).sum()
    ce = torch.nn.CrossEntropyLoss(label_smoothing=0.1)
    ref = ce(raw, labels) + rank / B + ce(concat, labels) + ce(part.view(B * T, -1), rows)
    assert abs(O.nts_loss(raw, concat, part, prob, labels).item() - ref.item()) < 1e-10


def test_rejected_options(monkeypatch):
    with pytest.raises(ValueError, match='proposal_num=9'):
        _net(monkeypatch, proposal_num=9)
    _net(monkeypatch, proposal_num=8)
    with pytest.raises(ValueError, match='image_size=200'):
        _net(monkeypatch, image_size=200)
    with pytest.raises(ValueError, match='cat_num=7'):
        _net(monkeypatch, cat_num=7)


def test_registration_and_yaml(monkeypatch):
    from hawkeye_b200.config import load_config
    from hawkeye_b200.registry import MODEL, install_into
    import hawkeye_b200.methods  # noqa: F401
    cfg = load_config(os.path.join(REPO, 'configs', 'NTSNet.yaml'))
    assert cfg.model.proposal_num == 6 and cfg.model.cat_num == 4 and cfg.dataset.batch_size == 4
    monkeypatch.setenv('HAWKEYE_ALLOW_RANDOM_INIT', '1')
    net = MODEL.get(cfg.model.name)(cfg.model)
    assert net.pretrained_model.fc.out_features == 200
    assert install_into({}, names=('NTSNet',))['NTSNet'] is MODEL['NTSNet']


def test_trainer_schedule_matches_sequential_lr():
    from hawkeye_b200.config import load_config
    from hawkeye_b200.examples import ALL_TRAINERS, TRAINERS, NTSNetTrainer
    assert ALL_TRAINERS['NTSNet'] is NTSNetTrainer and 'NTSNet' not in TRAINERS
    cfg = load_config(os.path.join(REPO, 'configs', 'NTSNet.yaml'))
    sc = cfg.train.scheduler
    p = torch.nn.Parameter(torch.zeros(1))
    opt = torch.optim.Adam([p], lr=cfg.train.optimizer.lr)
    ref = torch.optim.lr_scheduler.SequentialLR(
        opt, [torch.optim.lr_scheduler.LinearLR(opt, start_factor=sc.lr_warmup_decay, total_iters=sc.warmup_epochs),
              torch.optim.lr_scheduler.CosineAnnealingLR(opt, T_max=sc.T_max - sc.warmup_epochs)],
        milestones=[sc.warmup_epochs])

    class _Opt:
        param_groups = [dict(initial_lr=cfg.train.optimizer.lr, lr=cfg.train.optimizer.lr)]

    tr = NTSNetTrainer.__new__(NTSNetTrainer)
    tr.optimizer, tr.total_epoch = _Opt(), cfg.train.epoch
    mine = tr.get_scheduler(sc)
    for epoch in range(cfg.train.epoch):
        assert abs(_Opt.param_groups[0]['lr'] - opt.param_groups[0]['lr']) < 1e-12, epoch
        opt.step()
        ref.step()
        mine.step()


def test_c_entries_reject_bad_arguments():
    from hawkeye_b200 import _lib
    lib = _lib.lib()
    n0 = _lib.launch_count()
    p = 16                                     # any non-null, 16-byte aligned address: nothing may be launched
    assert lib.hk_nts_num_anchors(7, 7) == 426 and lib.hk_nts_num_anchors(14, 14) == 1614
    assert lib.hk_nts_score_fwd(None, p, p, p, p, p, p, p, p, p, 2, 7, 7, 4, 4, 2, 2, 128, None) < 0
    assert lib.hk_nts_score_fwd(p, p, p, p, p, p, p, p, p, p, 2, 7, 7, 3, 4, 2, 2, 128, None) < 0      # not a ceil chain
    assert lib.hk_nts_score_bwd(p, p, p, p, p, p, p, p, None, p, p, p, p, p, p, p, p, 2, 6, 7, 7, 4, 4, 2, 2, 128,
                                None) < 0
    assert lib.hk_nts_nms(p, None, p, p, p, 2, 426, 6, None) < 0
    assert lib.hk_nts_nms(p, p, p, p, p, 2, 4096, 6, None) < 0                                        # too many anchors
    assert lib.hk_nts_nms(p, p, p, p, p, 2, 426, 427, None) < 0
    assert lib.hk_nts_nms(p, 20, p, p, p, 2, 426, 6, None) < 0                                        # misaligned anchors
    assert lib.hk_nts_crop(None, p, p, 2, 6, 3, 224, 224, 224, 224, None) < 0
    assert lib.hk_nts_crop(p, p, p, 2, 6, 3, 224, 224, -1, 224, None) < 0
    assert lib.hk_nts_rank_loss(p, p, p, None, p, 2, 6, 200, None) < 0
    assert lib.hk_nts_rank_loss(p, p, p, p, p, 2, 0, 200, None) < 0
    assert _lib.launch_count() == n0
