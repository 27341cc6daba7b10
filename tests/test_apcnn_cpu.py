"""AP-CNN without a GPU: the state layout against the reference's (strict load both ways), the suppression-offset table
and the ROI oracle against fixtures of the unmodified reference's get_att_roi / nms_pytorch (tests/golden/make_golden_apcnn.py),
the tie rule, the refinement oracle against the fixture and against F.interpolate, the pooled form of the attended maps, the
trainer's groups and schedule, the yaml, the rejected input sizes and the new C entries' argument errors."""
import ctypes
import json
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import apcnn_inputs as I
import detgen
from conftest import load_golden
from oracle import apcnn_oracle as O

G = load_golden('reference_apcnn')
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
os.environ['HAWKEYE_ALLOW_RANDOM_INIT'] = '1'


def _model(nc=200):
    from hawkeye_b200.methods.apcnn import resnet50
    return resnet50(nc)


def test_state_dict_layout_matches_reference_and_loads_strictly():
    ref = json.loads(bytes(G['state_keys_json']).decode())
    net = _model()
    mine = [[k, list(v.shape)] for k, v in net.state_dict().items()]
    assert mine == ref
    assert sum(p.numel() for p in net.parameters()) == int(G['params'])
    sd = {k: torch.zeros(s) for k, s in ref}
    net.load_state_dict(sd, strict=True)
    other = _model()
    other.load_state_dict(net.state_dict(), strict=True)
    assert tuple(net.apn.A3_1.conv.weight.shape) == (256, 1, 3, 3)
    assert net.fpn.P5_1.conv_master.bn.momentum == 0.01 and net.cls3[2].momentum == 0.1
    assert net.cls3[3].out_features == 512 and _model(12).cls3[3].out_features == 256


def test_registry_builds_from_yaml():
    import hawkeye_b200 as hb
    from hawkeye_b200.config import load_config
    cfg = load_config(os.path.join(REPO, 'configs', 'APCNN.yaml'))
    assert cfg.model.name == 'APCNN' and cfg.model.num_classes == 200 and cfg.dataset.batch_size == 16
    assert cfg.train.optimizer.lr == 0.0005 and cfg.train.optimizer.weight_decay == 0.0005 and cfg.train.epoch == 100
    net = hb.MODEL.get('APCNN')(cfg.model)
    assert len(net.state_dict()) == len(json.loads(bytes(G['state_keys_json']).decode()))


def test_suppression_table_matches_reference_nms_arithmetic():
    from hawkeye_b200 import ops_apcnn
    t = ops_apcnn.suppression_table()
    assert t.shape == (3, 15, 15) and t.dtype == np.uint8
    for l in range(3):
        for i in range(15):
            for j in range(15):
                assert bool(t[l, i, j]) == O.nms_keep(O.SIZES[l], O.STRIDES[l], i - 7, j - 7)
    # power-of-two sizes: no offset sits on the threshold (20 inter == union has no solution)
    for l in range(3):
        for dy in range(8):
            for dx in range(8):
                w, h = O.SIZES[l] - dx * O.STRIDES[l], O.SIZES[l] - dy * O.STRIDES[l]
                assert 20 * w * h != 2 * O.SIZES[l] ** 2 - w * h


@pytest.mark.parametrize('nc', [200, 12])
def test_roi_oracle_matches_reference(nc):
    boxes, counts = O.roi_select(I.gates(nc), nc, I.ROI_IMAGE, I.ROI_IMAGE)
    for l in range(3):
        assert np.array_equal(counts[:, l], G[f'roi_{nc}_counts_{l}'])
        assert np.array_equal(boxes[:, O.OFFSETS[l]:O.OFFSETS[l] + O.TOPK[l]], G[f'roi_{nc}_boxes_{l}'])
    assert counts[0, 0] < 5 and counts[1, 0] < 5           # the fixture includes images with fewer boxes than topk


def test_roi_tie_goes_to_highest_index():
    g = np.full((28, 28), 0.5, dtype=np.float32)
    boxes, n = O.roi_level(g, 0, 200, 224, 224)
    assert n == 5
    assert tuple(boxes[0]) == (21 * 8 - 32, 21 * 8 - 32, 21 * 8 + 32, 21 * 8 + 32)    # the last cell of the 5..22 window


def test_central_windows_and_rejected_sizes():
    from hawkeye_b200 import ops_apcnn
    assert ops_apcnn.central_windows(56, 56, 200).tolist() == [[11, 44, 11, 44], [5, 22, 5, 22], [2, 11, 2, 11]]
    net = _model(12)
    for h, w in ((100, 96), (96, 0), (32, 32)):
        with pytest.raises(ValueError):
            net.check_input(h, w)
    net.check_input(96, 128)


def _draws(rec, counts):
    """the reference's recorded (random(), randint) -> the op's [N, 2] fractions"""
    d = np.zeros((len(rec), 2), dtype=np.float32)
    for n, (u, ind) in enumerate(rec):
        lv = 0 if u < 0.3 else (1 if u < 0.6 else -1)
        d[n] = (u, (ind + 0.5) / counts[n, lv] if lv >= 0 else 0.0)
    return d


def _roi_200():
    boxes = np.concatenate([G[f'roi_200_boxes_{l}'] for l in range(3)], axis=1)
    counts = np.stack([G[f'roi_200_counts_{l}'] for l in range(3)], axis=1)
    return boxes, counts


def test_refine_oracle_matches_reference():
    boxes, counts = _roi_200()
    x = detgen.det((I.ROI_BATCH, 8, 28, 28), 4100).double().numpy()
    y = O.refine(x, boxes, counts, _draws(G['refine_draws'], counts))
    assert np.abs(y - G['refine_train_y']).max() < 1e-5
    y = O.refine(x, boxes, counts, None)
    assert np.abs(y - G['refine_eval_y']).max() < 1e-5
    n = 3
    r = np.concatenate([boxes[n, O.OFFSETS[l]:O.OFFSETS[l] + counts[n, l]] for l in range(3)]) / 8
    X1, Y1, X2, Y2 = int(r[:, 0].min()), int(r[:, 1].min()), int(r[:, 2].max()), int(r[:, 3].max())
    ref = F.interpolate(torch.from_numpy(x[n:n + 1, :, Y1:Y2, X1:X2]), (28, 28), mode='bilinear', align_corners=False)
    assert (torch.from_numpy(y[n:n + 1]) - ref).abs().max() < 1e-5


def test_pooled_form_of_attended_maps():
    rs = np.random.RandomState(1)
    Fm, gate, ch = rs.standard_normal((2, 16, 5, 7)), rs.random_sample((2, 1, 5, 7)), rs.random_sample((2, 16, 1, 1))
    a, b = O.attended_pool(Fm, gate, ch)
    assert np.abs(a - b).max() < 1e-12
    top, lat = rs.standard_normal((1, 2, 2, 3)), rs.standard_normal((1, 2, 4, 6))
    ref = F.interpolate(torch.from_numpy(top), scale_factor=2) + torch.from_numpy(lat)
    assert np.array_equal(O.lateral(top, lat), ref.numpy())


def test_trainer_groups_and_schedule():
    from hawkeye_b200.examples import ALL_TRAINERS, TRAINERS, APCNNTrainer, _EpochCosine
    assert 'APCNN' in ALL_TRAINERS and 'APCNN' not in TRAINERS

    class T(APCNNTrainer):
        def __init__(self, m):
            self.model = m

    net = _model(12)
    (early, m0), (late, m1) = T(net).param_groups()
    kids = list(net.children())
    assert (m0, m1) == (0.1, 1.0)
    assert {id(p) for p in early} == {id(p) for c in kids[:7] for p in c.parameters()}
    assert {id(p) for p in late} == {id(p) for c in kids[7:] for p in c.parameters()}

    class Opt:
        param_groups = [dict(lr=5e-5, initial_lr=5e-5), dict(lr=5e-4, initial_lr=5e-4)]

    s = _EpochCosine(Opt, 100)
    for e in range(205):
        s.set_epoch(e)
        want = float(5e-4 / 2 * (np.cos(np.pi * (e % 100) / 100) + 1))
        assert math.isclose(Opt.param_groups[1]['lr'], want, rel_tol=1e-12, abs_tol=1e-18)
        assert math.isclose(Opt.param_groups[0]['lr'], want / 10, rel_tol=1e-12, abs_tol=1e-18)


def test_apcnn_and_act_entries_reject_bad_arguments():
    from hawkeye_b200 import _lib
    lib = _lib.lib()
    buf = (ctypes.c_float * 64)()
    p = ctypes.addressof(buf)
    assert lib.hk_apcnn_lateral_fwd(None, p, p, 1, 1, 1, 4, None) == -1
    assert lib.hk_apcnn_lateral_fwd(p, p, p, 1, 1, 1, 3, None) == -1
    assert lib.hk_apcnn_lateral_bwd(p, None, 1, 1, 1, 4, None) == -1
    assert lib.hk_apcnn_bcast(None, None, p, 1, 1, 4, 1.0, None) == -1
    assert lib.hk_apcnn_pool(p, p, 1, 1, 128, 1.0, p, 4096, None) == -1
    assert lib.hk_apcnn_pool(p, p, 1, 1, 256, 1.0, p, 8, None) == -4
    assert lib.hk_apcnn_att_fwd(p, p, p, p, p, p, 1, 2, 2, 128, p, 1 << 20, None) == -3
    assert lib.hk_apcnn_att_fwd(p, p, p, p, p, p, 1, 2, 2, 256, p, 8, None) == -4
    assert lib.hk_apcnn_att_bwd(p, p, p, None, None, p, p, p, 1, 2, 2, 256, p, 1 << 20, None) == -1
    assert lib.hk_apcnn_roi(p, p, p, p, p, p, p, 1, 6, 8, 64, 64, None) == -1
    win = (ctypes.c_int * 12)(*([1, 1, 0, 2] * 3))
    assert lib.hk_apcnn_roi(p, p, p, ctypes.addressof(win), p, p, p, 1, 8, 8, 64, 64, None) == -1
    assert b'central window' in lib.hk_last_error()
    assert lib.hk_apcnn_refine_fwd(p, p, p, None, p, None, 1, 2, 2, 4, None) == -1
    assert lib.hk_apcnn_refine_bwd(p, p, p, 1, 2, 2, 6, None) == -1
    assert lib.hk_act_fwd(p, p, 0, 1, None) == -1
    assert lib.hk_act_bwd(p, None, p, 4, 1, None) == -1
    assert lib.hk_apcnn_mix_fwd(p, p, p, p, None, 1, 4, None) == -1
    assert lib.hk_apcnn_mix_bwd(p, p, p, p, p, p, 0, 4, None) == -1
    assert lib.hk_apcnn_mask_cat(p, p, p, p, 1, 6, 8, None) == -1
    assert lib.hk_apcnn_att_workspace_bytes(0, 1, 1) == 0 and lib.hk_apcnn_pool_workspace_bytes(1, 64, 256) == 1024
