"""MGE-CNN without a GPU: the state layout against the reference's (strict load, 1302 entries, 108,521,155 parameters), the
get_params split, the trainer's groups and schedule, the yaml, the oracle's closed-form Grad-CAM weights and boxes against
fixtures of the unmodified reference (tests/golden/make_golden_mge.py), and the new C entries' argument errors."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

import detgen
import mge_inputs as I
from conftest import load_golden
from oracle import mge_oracle as O

G = load_golden('reference_mge')
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
os.environ['HAWKEYE_ALLOW_RANDOM_INIT'] = '1'


def _cfg(**kw):
    from hawkeye_b200.cfgnode import CfgNode
    return CfgNode(dict(dict(name='MGE_CNN', num_classes=200, image_size=224, box_thred=0.2), **kw))


def _shallow():
    from hawkeye_b200.methods.mge import LocalCamNet
    return LocalCamNet(_cfg(num_classes=I.E2E_CLASSES, image_size=I.E2E_IMAGE, box_thred=I.E2E_THRED), layers=I.E2E_LAYERS)


@pytest.fixture(scope='module')
def full():
    import hawkeye_b200 as hb
    return hb.MODEL.get('MGE_CNN')(_cfg())


def test_state_dict_layout_matches_reference_and_loads_strictly(full):
    ref = json.loads(bytes(G['state_keys_json']).decode())
    mine = [[k, list(v.shape)] for k, v in full.state_dict().items()]
    assert mine == ref and len(mine) == 1302
    assert sum(p.numel() for p in full.parameters()) == int(G['params']) == 108_521_155
    full.load_state_dict({k: torch.zeros(s) for k, s in ref}, strict=True)
    assert tuple(full.conv6.weight.shape) == (2000, 1024, 1, 1) and full.conv6.padding == (1, 1)


def test_trunks_start_identical(full):
    sd = _shallow().state_dict()
    for b in ('_box', '_box_2', '_gate'):
        for m in ('conv4', 'conv5'):
            for k, v in sd.items():
                if k.startswith(m + '.'):
                    assert torch.equal(v, sd[m + b + k[len(m):]]), (b, k)


def test_get_params_split(full):
    ext = full.get_params('extractor')
    assert full.get_params('extract') is not None
    trunks = {id(p) for b in ('', '_box', '_box_2', '_gate') for m in ('conv4', 'conv5')
              for p in getattr(full, m + b).parameters()}
    assert {id(p) for p in ext} == trunks and len(ext) == len(trunks)
    cls = list(full.get_params('classifier'))
    assert {id(p) for p in cls} == {id(p) for p in full.parameters()} - trunks
    ids = {id(p) for p in cls}
    for m in (full.cls_cat_a, full.conv6, full.conv6_1, full.conv6_2, full.cls_gate, full.classifier_box_2):
        assert all(id(p) in ids for p in m.parameters())


def test_registry_builds_from_yaml_and_rejects_sizes():
    import hawkeye_b200 as hb
    from hawkeye_b200.config import load_config
    cfg = load_config(os.path.join(REPO, 'configs', 'MGE_CNN.yaml'))
    assert cfg.model.name == 'MGE_CNN' and cfg.model.num_classes == 200 and cfg.model.image_size == 224
    assert cfg.model.box_thred == 0.2 and cfg.dataset.batch_size == 4
    assert cfg.train.optimizer.lr == 0.0004 and cfg.train.optimizer.weight_decay == 0.00002
    assert 'MGE_CNN' in hb.MODEL
    from hawkeye_b200.methods.mge import LocalCamNet
    with pytest.raises(ValueError):
        LocalCamNet(_cfg(image_size=200), layers=I.E2E_LAYERS)
    with pytest.raises(Exception):
        LocalCamNet(_cfg(num_classes=10), layers=I.E2E_LAYERS)
    net = _shallow()
    with pytest.raises(ValueError):
        net(torch.zeros(1, 3, 96, 96))


def test_trainer_groups_and_schedule():
    from hawkeye_b200.config import load_config
    from hawkeye_b200.examples import ALL_TRAINERS, TRAINERS, MGE_CNNTrainer
    assert ALL_TRAINERS['MGE_CNN'] is MGE_CNNTrainer and 'MGE_CNN' not in TRAINERS
    cfg = load_config(os.path.join(REPO, 'configs', 'MGE_CNN.yaml'))
    net = _shallow()
    tr = MGE_CNNTrainer.__new__(MGE_CNNTrainer)
    tr.model, tr.config = net, cfg
    (cls, m0), (ext, m1) = tr.param_groups()
    assert (m0, m1) == (1.0, 0.1)
    assert {id(p) for p in ext} == {id(p) for p in net.get_params('extractor')}
    unused = {id(p) for p in net.cls_cat_a.parameters()}
    assert {id(p) for p in cls} == {id(p) for p in net.get_params('classifier')} - unused and len(unused) == 2
    tr2 = MGE_CNNTrainer.__new__(MGE_CNNTrainer)
    tr2.model = net
    tr2.config = _cfg(name='x')
    tr2.config = type('C', (), {'train': type('T', (), {'optimizer': _cfg(lr=1.0, lr_rate=0.25)})})()
    assert tr2.param_groups()[1][1] == 0.25

    sc = cfg.train.scheduler
    p = torch.nn.Parameter(torch.zeros(1))
    opt = torch.optim.Adam([p], lr=cfg.train.optimizer.lr)
    ref = torch.optim.lr_scheduler.SequentialLR(
        opt, [torch.optim.lr_scheduler.LinearLR(opt, start_factor=sc.lr_warmup_decay, total_iters=sc.warmup_epochs),
              torch.optim.lr_scheduler.CosineAnnealingLR(opt, T_max=sc.T_max - sc.warmup_epochs)],
        milestones=[sc.warmup_epochs])

    class _Opt:
        param_groups = [dict(initial_lr=cfg.train.optimizer.lr, lr=cfg.train.optimizer.lr)]

    tr.optimizer, tr.total_epoch = _Opt(), cfg.train.epoch
    mine = tr.get_scheduler(sc)
    for epoch in range(cfg.train.epoch):
        assert abs(_Opt.param_groups[0]['lr'] - opt.param_groups[0]['lr']) < 1e-12, epoch
        opt.step()
        ref.step()
        mine.step()


def test_gradcam_closed_form_matches_reference():
    net = _shallow()
    net.load_state_dict(detgen.state_like(net))
    W = net.classifier.fc.weight.detach().numpy()
    for tag in ('argmax', 'target'):
        want = G[f'gradcam_{tag}_weights']
        got = O.gradcam_weights(W, G[f'gradcam_{tag}_idx'], 16)
        assert want.shape == got.shape == (2, 2048)
        assert np.abs(got - want).max() < 1e-9 and (want > 0).any()
    assert G['gradcam_target_idx'].tolist() == [3, 7]


@pytest.mark.parametrize('name', sorted(I.BBOX_CASES))
def test_box_oracle_matches_reference(name):
    conv5, lw, rate, size = I.bbox_case(name)
    got = O.cam_box(conv5, lw, rate, size)
    want = np.array([I.crop_box(xy, size) for xy in G[f'bbox_{name}']])
    if name in I.EXACT_CASES:
        assert np.array_equal(got, want)
    else:
        assert np.abs(got - want).max() <= 1


def test_box_fallbacks_and_nan_case():
    assert G['bbox_const224'].tolist() == [[0, 223, 0, 223]] * 2                 # NaN CAM: every pixel, last row dropped
    assert G['bbox_peak224'].tolist() == [[82, 141, 82, 141]]
    assert I.crop_box(G['bbox_row224'][0], 224) == (0, 0, 224, 224)              # one row: the whole image
    assert I.crop_box(G['bbox_col448'][0], 448) == (0, 0, 448, 448)              # one column
    assert tuple(O.cam_box(*I.bbox_case('const224')[:3], 224)[0]) == (0, 0, 223, 223)


def test_part_head_and_gate_oracles_against_torch():
    rs = np.random.RandomState(3)
    x = rs.standard_normal((2, 3, 4, 8))
    w, b = rs.standard_normal((12, 8)), rs.standard_normal(12)
    w[0], b[0] = 0.0, 2.0                                                    # channel 0: the border ties the interior and wins
    pooled, pos = O.part_head(x, w, b)
    xt = torch.from_numpy(x).permute(0, 3, 1, 2).requires_grad_(False)
    wt, bt = torch.from_numpy(w).view(12, 8, 1, 1).requires_grad_(True), torch.from_numpy(b).requires_grad_(True)
    ref = torch.nn.functional.adaptive_max_pool2d(torch.relu(torch.nn.functional.conv2d(xt, wt, bt, padding=1)), 1).flatten(1)
    assert np.abs(pooled - ref.detach().numpy()).max() < 1e-12 and (pos[:, 0] == -1).all()
    g = rs.standard_normal(pooled.shape)
    ref.backward(torch.from_numpy(g))
    dw, db = O.part_head_bwd(x, pos, pooled, g)
    assert np.abs(dw - wt.grad.view(12, 8).numpy()).max() < 1e-10 and np.abs(db - bt.grad.numpy()).max() < 1e-10
    h, w2, b2 = rs.standard_normal((3, 16)), rs.standard_normal((3, 16)), rs.standard_normal(3)
    cats = [rs.standard_normal((3, 8)) for _ in range(3)]
    out, pr = O.gate(h, w2, b2, cats)
    ht, w2t, b2t = (torch.from_numpy(t).requires_grad_(True) for t in (h, w2, b2))
    prt = torch.softmax(ht @ w2t.T + b2t, 1)
    outt = (torch.stack([torch.from_numpy(c) for c in cats], -1) * prt[:, None]).sum(-1)
    assert np.abs(out - outt.detach().numpy()).max() < 1e-12
    dout = rs.standard_normal(out.shape)
    outt.backward(torch.from_numpy(dout))
    _, dh, dw2, db2 = O.gate_bwd(h, w2, pr, cats, dout)
    for a, t in ((dh, ht), (dw2, w2t), (db2, b2t)):
        assert np.abs(a - t.grad.numpy()).max() < 1e-12


def test_c_entries_reject_bad_arguments():
    from hawkeye_b200 import _lib
    lib = _lib.lib()
    buf = (ctypes.c_float * 64)()
    p = ctypes.addressof(buf)
    assert lib.hk_mge_part_fwd(None, p, p, p, p, 1, 2, 2, 4, 4, p, 1 << 20, None) == -1
    assert lib.hk_mge_part_fwd(p, p, p, p, p, 1, 2, 2, 6, 4, p, 1 << 20, None) == -3
    assert lib.hk_mge_part_fwd(p, p, p, p, p, 1, 2, 2, 4, 4, p, 8, None) == -4
    assert lib.hk_mge_part_fwd(p, p, p, p, p, 0, 2, 2, 4, 4, p, 1 << 20, None) == -1
    assert lib.hk_mge_part_workspace_bytes(2, 3, 3, 8) == 2 * 9 * 8 * 4 and lib.hk_mge_part_workspace_bytes(0, 3, 3, 8) == 0
    assert lib.hk_mge_part_bwd(p, p, p, p, None, p, 1, 2, 2, 4, 4, None) == -1
    assert lib.hk_mge_part_bwd(p, p, p, p, p, p, 1, 0, 2, 4, 4, None) == -1
    assert lib.hk_mge_cam_box(None, None, p, p, p, 1, 4, 8, 7, 7, 224, ctypes.c_float(0.2), None) == -1
    assert lib.hk_mge_cam_box(p, None, p, p, p, 1, 4, 8, 7, 7, 1, ctypes.c_float(0.2), None) == -1
    assert lib.hk_mge_cam_box(p, None, p, p, p, 1, 4, 12288, 7, 7, 224, ctypes.c_float(0.2), None) == -3
    assert lib.hk_mge_cat_l2n(p, None, p, 1, 4, 4, ctypes.c_float(10.0), None) == -1
    assert lib.hk_mge_cat_l2n(p, p, p, 1, 0, 4, ctypes.c_float(10.0), None) == -1
    assert lib.hk_mge_gate_fwd(p, p, p, p, p, None, p, p, 1, 4, 4, None) == -1
    assert lib.hk_mge_gate_fwd(p, p, p, p, p, p, p, p, 1, 0, 4, None) == -1
    assert lib.hk_mge_gate_bwd(p, p, p, p, p, p, p, None, None, None, None, None, 1, 4, 4, None) == -1
    assert lib.hk_mge_gate_bwd(p, p, p, p, p, p, p, None, p, None, p, None, 1, 4, 4, None) == -1
