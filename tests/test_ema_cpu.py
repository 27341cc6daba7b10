"""Model EMA on the host side: the ``train.model_ema`` setting, torchvision's decay adjustment, the AveragedModel
state-dict layout (ProtoTree's nested leaf keys included), the construction-time checks of ``engine.ModelEMA`` and the
C-ABI error paths of the EMA entries, none of which needs a device."""
import copy
import ctypes
import glob
import os

import pytest
import torch
import torch.nn as nn
from torch.optim.swa_utils import AveragedModel

from hawkeye_b200 import engine, train
from hawkeye_b200.cfgnode import CfgNode
from hawkeye_b200.config import load_config

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ERR_ARG, ERR_ALIGN = -1, -2


@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as g
    g.build()
    from hawkeye_b200 import _lib
    return _lib.lib()


def _train(**ema):
    return CfgNode(dict(epoch=30, model_ema=ema if ema else None))


def test_setting_defaults_and_absence():
    assert train.model_ema_setting(CfgNode(dict(epoch=30))) is None
    assert train.model_ema_setting(_train()) == (0.99998, 32)
    assert train.model_ema_setting(CfgNode(dict(model_ema={}))) == (0.99998, 32)
    assert train.model_ema_setting(_train(decay=0.999)) == (0.999, 32)
    assert train.model_ema_setting(_train(steps=4)) == (0.99998, 4)
    assert train.model_ema_setting(_train(decay=0.5, steps=1)) == (0.5, 1)


def test_shipped_configs_have_no_ema():
    for path in sorted(glob.glob(os.path.join(REPO, 'configs', '*.yaml'))):
        assert train.model_ema_setting(load_config(path).train) is None, path


@pytest.mark.parametrize('value', [0, 1, 1.5, -0.1, 0.0, 1.0, True, '0.9', float('nan')])
def test_bad_decay_names_the_key(value):
    with pytest.raises(ValueError, match=r'train\.model_ema\.decay'):
        train.model_ema_setting(_train(decay=value))


@pytest.mark.parametrize('value', [0, -3, 2.0, 1.5, True, '32', None])
def test_bad_steps_names_the_key(value):
    with pytest.raises(ValueError, match=r'train\.model_ema\.steps'):
        train.model_ema_setting(CfgNode(dict(model_ema=dict(steps=value))))


def test_bad_mapping_and_unknown_keys():
    with pytest.raises(ValueError, match=r'train\.model_ema'):
        train.model_ema_setting(CfgNode(dict(model_ema=0.999)))
    with pytest.raises(ValueError, match='unknown keys'):
        train.model_ema_setting(_train(decay=0.9, step=3))


def _torchvision_decay(decay, steps, batch_size, epochs, world_size=1):
    """references/classification/train.py, as written there."""
    adjust = world_size * batch_size * steps / epochs
    alpha = 1.0 - decay
    alpha = min(1.0, alpha * adjust)
    return 1.0 - alpha


@pytest.mark.parametrize('decay', [0.99998, 0.9999, 0.999, 0.9])
def test_decay_is_torchvisions_formula(decay):
    clamped = 0
    for batch in (1, 8, 24, 32, 96, 256):
        for steps in (1, 2, 32, 100):
            for epochs in (1, 2, 30, 100, 600):
                d = train.model_ema_decay(decay, steps, batch, epochs)
                assert d == _torchvision_decay(decay, steps, batch, epochs)
                assert 0.0 <= d < 1.0
                clamped += d == 0.0
    assert clamped > 0 or decay > 0.9999      # the grid reaches the clamp at alpha = 1 for the smaller decays
    assert train.model_ema_decay(0.9, 32, 256, 1) == 0.0


def test_global_batch_stands_for_world_times_rank_batch():
    """dataset.batch_size is the global batch: 4 ranks of 8 images adjust as one rank of 32."""
    assert train.model_ema_decay(0.99998, 32, 32, 30) == _torchvision_decay(0.99998, 32, 8, 30, world_size=4)


class _Net(nn.Module):
    def __init__(self):
        super().__init__()
        self.conv = nn.Conv2d(3, 4, 3)
        self.bn = nn.BatchNorm2d(4)
        self.fc = nn.Linear(4, 5)
        self.frozen = nn.Parameter(torch.randn(3), requires_grad=False)


def test_state_dict_layout_is_averaged_models():
    net = _Net()
    ref = AveragedModel(copy.deepcopy(net), use_buffers=True).state_dict()
    ours = engine.averaged_state(torch.zeros((), dtype=torch.int64), net.state_dict())
    assert list(ours) == list(ref)
    assert all(ours[k].shape == ref[k].shape and ours[k].dtype == ref[k].dtype for k in ref)
    assert list(engine.averaged_model_state(ours)) == list(net.state_dict())


def test_state_dict_layout_keeps_prototree_leaf_keys():
    from hawkeye_b200.methods.prototree import ProtoTree
    tree = ProtoTree(CfgNode(dict(height=3, num_classes=6, num_features=8)))
    ref = AveragedModel(copy.deepcopy(tree), use_buffers=True).state_dict()
    ours = engine.averaged_state(torch.zeros((), dtype=torch.int64), tree.state_dict())
    assert list(ours) == list(ref)
    leaves = [k for k in ours if k.endswith('._dist_params')]
    assert len(leaves) == 8 and 'module._root.l.l.l._dist_params' in leaves and 'module.leaf_params' not in ours
    # and back: the model's load hook restacks the nested keys
    other = ProtoTree(CfgNode(dict(height=3, num_classes=6, num_features=8)))
    other.load_state_dict(engine.averaged_model_state(ours))
    assert torch.equal(other.leaf_params, tree.leaf_params)


def test_construction_rejects_other_dtypes_by_name(lib):
    net = _Net()
    net.register_buffer('scale', torch.ones(3, dtype=torch.float64))
    flat = engine.FlatParams(net)
    with pytest.raises(ValueError, match='scale is torch.float64'):
        engine.ModelEMA(net, flat, 0.99)
    net = _Net().half()
    with pytest.raises(ValueError, match='is torch.float16'):
        engine.ModelEMA(net, engine.FlatParams(net), 0.99)


def test_construction_table_covers_flat_frozen_and_buffers(lib):
    net = _Net()
    flat = engine.FlatParams(net)
    ema = engine.ModelEMA(net, flat, 0.99)
    # the flat buffer, the frozen parameter, BN's running mean, running var and num_batches_tracked
    assert ema.nseg == 5
    t = ema.table
    assert t[0, 0] == flat.flat.data_ptr() and t[0, 2] == flat.numel and t[0, 3] == 0
    assert t[1, 0] == net.frozen.data_ptr() and t[1, 2] == 3
    assert [int(k) for k in t[:, 3]] == [0, 0, 0, 0, 1]
    assert [int(c) for c in t[:, 4]] == [0, 1, 2, 3, 4] and ema.chunks == 5
    assert ema.n_averaged.dtype == torch.int64 and int(ema.n_averaged) == 0
    with pytest.raises(ValueError, match='decay'):
        engine.ModelEMA(net, flat, 1.5)


def _table(rows):
    t = torch.zeros(len(rows), engine.EMA_COLS, dtype=torch.int64)
    for i, r in enumerate(rows):
        t[i, :4] = torch.tensor(r)
    return t


def _plan(lib, t, nseg=None):
    return lib.hk_ema_plan(ctypes.c_void_p(t.data_ptr()), t.shape[0] if nseg is None else nseg)


def test_plan_checks_and_chunks(lib):
    assert lib.hk_ema_cols() == engine.EMA_COLS
    good = [(4096, 8192, 4097, 0), (64, 128, 1, 1), (256, 512, 8192, 0)]
    t = _table(good)
    assert _plan(lib, t) == 2 + 1 + 2
    assert [int(c) for c in t[:, 4]] == [0, 2, 3]
    assert lib.hk_ema_plan(None, 3) == ERR_ARG
    assert _plan(lib, t, 0) == ERR_ARG
    for bad, code in (((0, 64, 4, 0), ERR_ARG), ((64, 0, 4, 0), ERR_ARG), ((64, 64, 4, 0), ERR_ARG),
                      ((64, 128, 0, 0), ERR_ARG), ((64, 128, -1, 0), ERR_ARG), ((64, 128, 4, 2), ERR_ARG),
                      ((66, 128, 4, 0), ERR_ALIGN), ((68, 128, 4, 1), ERR_ALIGN), ((64, 132, 4, 1), ERR_ALIGN)):
        assert _plan(lib, _table(good[:1] + [bad])) == code, bad


def test_update_and_swap_reject_bad_arguments(lib):
    t = _table([(4096, 8192, 4, 0)])
    assert _plan(lib, t) == 1
    tp, cnt, s = ctypes.c_void_p(t.data_ptr()), ctypes.c_void_p(64), None
    up, sw = lib.hk_ema_update, lib.hk_ema_swap
    assert up(None, 1, 1, cnt, 0.9, 0.1, 0, s) == ERR_ARG
    assert up(tp, 1, 1, None, 0.9, 0.1, 0, s) == ERR_ARG
    assert up(tp, 0, 1, cnt, 0.9, 0.1, 0, s) == ERR_ARG
    assert up(tp, 1, 0, cnt, 0.9, 0.1, 0, s) == ERR_ARG
    assert up(tp, 1, 2 ** 31, cnt, 0.9, 0.1, 0, s) == ERR_ARG
    assert up(tp, 1, 1, cnt, 1.5, 0.1, 0, s) == ERR_ARG
    assert up(tp, 1, 1, cnt, 0.9, -0.1, 0, s) == ERR_ARG
    assert up(tp, 1, 1, cnt, float('nan'), 0.1, 0, s) == ERR_ARG
    assert sw(None, 1, 1, s) == ERR_ARG
    assert sw(tp, -1, 1, s) == ERR_ARG
    assert sw(tp, 1, 0, s) == ERR_ARG
    assert b'hk_ema_swap' in lib.hk_last_error()
