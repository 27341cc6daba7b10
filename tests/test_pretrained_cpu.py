"""The pretrained-checkpoint loader (hawkeye_b200.utils.load_pretrained) through every model that calls it, without a GPU:
a torchvision-layout file loads bit-exactly into the trunk and leaves every other tensor as the seeded construction made
it, a file that lacks a trunk tensor is rejected by name, and a missing file warns once unless random initialisation is
allowed.  ProtoTree's iNat checkpoint only borrows the renaming."""
import logging
import os
import re

import pytest
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BODY = ('conv1', 'bn1', 'layer1', 'layer2', 'layer3', 'layer4')
TORCHVISION_FC = {'fc.weight': torch.zeros(1000, 2048), 'fc.bias': torch.zeros(1000)}


def _model(yaml, name=None):
    from hawkeye_b200.config import load_config
    from hawkeye_b200.registry import MODEL
    import hawkeye_b200.methods  # noqa: F401
    cfg = load_config(os.path.join(REPO, 'configs', yaml)).model
    return lambda: MODEL.get(name or cfg.name)(cfg)


def _backbone(name):
    from hawkeye_b200.registry import BACKBONE
    import hawkeye_b200.backbone  # noqa: F401
    return lambda: BACKBONE[name](pretrained=True)


def _trunk_index(k):
    """ResNetTrunk key -> torchvision's (``4.0.conv1.weight`` -> ``layer1.0.conv1.weight``)"""
    from hawkeye_b200.backbone.resnet import RESNET_NAMES
    head, _, rest = k.partition('.')
    return RESNET_NAMES[int(head)] + '.' + rest


def _under(prefix, heads):
    """model key -> torchvision's for the keys under ``prefix`` whose first name is one of ``heads``, else None"""
    def key(k):
        if k.startswith(prefix) and k[len(prefix):].partition('.')[0] in heads:
            return k[len(prefix):]
        return None
    return key


# name -> (build with pretrained=True, checkpoint variable, model key -> checkpoint key or None, what torchvision's file
# holds besides: never loaded)
CASES = {
    'resnet50': (_backbone('resnet50'), 'HAWKEYE_RESNET50_PTH', _trunk_index, TORCHVISION_FC),
    'resnet101': (_backbone('resnet101'), 'HAWKEYE_RESNET101_PTH', _trunk_index, TORCHVISION_FC),
    'vgg16': (_backbone('vgg16'), 'HAWKEYE_VGG16_PTH', lambda k: 'features.' + k, {'classifier.6.bias': torch.zeros(1000)}),
    'NTSNet': (_model('NTSNet.yaml'), 'HAWKEYE_RESNET50_PTH', _under('pretrained_model.', BODY), TORCHVISION_FC),
    'APCNN': (_model('APCNN.yaml'), 'HAWKEYE_RESNET50_PTH', _under('', BODY), TORCHVISION_FC),
    'IP_ResNet50': (_model('InterpPartsNet.yaml', 'IP_ResNet50'), 'HAWKEYE_RESNET50_PTH', _under('', BODY[:5]),
                    dict(TORCHVISION_FC, **{'layer4.0.conv1.weight': torch.zeros(512, 1024, 1, 1)})),
    'IP_ResNet101': (_model('InterpPartsNet.yaml', 'IP_ResNet101'), 'HAWKEYE_RESNET101_PTH', _under('', BODY[:5]),
                     dict(TORCHVISION_FC, **{'layer4.0.conv1.weight': torch.zeros(512, 1024, 1, 1)})),
}


def _reference(name, monkeypatch):
    """(the state of the seeded model built without a checkpoint, a torchvision-layout file of random tensors for it)"""
    build, env, key, extra = CASES[name]
    monkeypatch.setenv('HAWKEYE_ALLOW_RANDOM_INIT', '1')
    monkeypatch.delenv(env, raising=False)
    torch.manual_seed(0)
    net = build()
    state = {k: v.clone() for k, v in net.state_dict().items()}
    g = torch.Generator().manual_seed(1)
    ckpt = {key(k): (torch.randn(v.shape, generator=g) if v.is_floating_point() else torch.full_like(v, 7))
            for k, v in state.items() if key(k) is not None}
    assert len(ckpt) > 10
    return state, dict(ckpt, **extra)


@pytest.mark.parametrize('name', list(CASES))
def test_file_loads_into_the_trunk_only(name, monkeypatch, tmp_path):
    build, env, key, _ = CASES[name]
    state, ckpt = _reference(name, monkeypatch)
    torch.save(ckpt, tmp_path / 'tv.pth')
    monkeypatch.setenv(env, str(tmp_path / 'tv.pth'))
    torch.manual_seed(0)
    got = build().state_dict()
    assert list(got) == list(state)
    for k, v in got.items():
        want = state[k] if key(k) is None else ckpt[key(k)]
        assert v.shape == state[k].shape and torch.equal(v, want), k


@pytest.mark.parametrize('name', list(CASES))
def test_incomplete_file_is_rejected(name, monkeypatch, tmp_path):
    from hawkeye_b200._lib import HawkeyeLibError
    build, env, _, _ = CASES[name]
    _, ckpt = _reference(name, monkeypatch)
    weights = [k for k in ckpt if k.endswith('.weight') and k not in CASES[name][3]]
    gone = weights[len(weights) // 2]
    del ckpt[gone]
    torch.save(ckpt, tmp_path / 'partial.pth')
    monkeypatch.setenv(env, str(tmp_path / 'partial.pth'))
    with pytest.raises(HawkeyeLibError, match=re.escape(env) + '.*' + re.escape(repr(gone))):
        build()


@pytest.mark.parametrize('name', list(CASES))
def test_missing_file_warns_once(name, monkeypatch, tmp_path, caplog):
    build, env, _, _ = CASES[name]
    monkeypatch.setenv(env, str(tmp_path / 'absent.pth'))
    monkeypatch.delenv('HAWKEYE_ALLOW_RANDOM_INIT', raising=False)
    with caplog.at_level(logging.WARNING, logger='hawkeye_b200'):
        build()
    assert len(caplog.records) == 1 and env in caplog.records[0].getMessage()
    caplog.clear()
    monkeypatch.setenv('HAWKEYE_ALLOW_RANDOM_INIT', '1')
    with caplog.at_level(logging.WARNING, logger='hawkeye_b200'):
        build()
    assert not caplog.records


def test_prototree_inat_trunk_lands_in_the_trunk(monkeypatch, tmp_path):
    """iNat layout: ``module.backbone.<name>`` for the trunk, ``cb_block`` for layer4.2, plus tensors that are dropped."""
    from hawkeye_b200.backbone.resnet import ResNetTrunk
    from hawkeye_b200.cfgnode import CfgNode
    from hawkeye_b200.config import load_config
    from hawkeye_b200.registry import MODEL
    import hawkeye_b200.methods  # noqa: F401
    monkeypatch.setenv('HAWKEYE_ALLOW_RANDOM_INIT', '1')
    g = torch.Generator().manual_seed(2)
    trunk = {k: torch.randn(v.shape, generator=g) if v.is_floating_point() else torch.full_like(v, 7)
             for k, v in ResNetTrunk().state_dict().items()}
    inat = {}
    for k, v in trunk.items():
        name = _trunk_index(k)
        inat['module.backbone.' + ('cb_block' + name[len('layer4.2'):] if name.startswith('layer4.2.') else name)] = v
    inat['module.backbone.rb_block.conv1.weight'] = torch.zeros(512, 2048, 1, 1)
    inat['module.classifier.weight'] = torch.zeros(4, 4)
    torch.save(inat, tmp_path / 'inat.pth')
    cfg = CfgNode(load_config(os.path.join(REPO, 'configs', 'ProtoTreeNet.yaml')).model.to_dict())
    cfg.backbone.pretrain = str(tmp_path / 'inat.pth')
    got = MODEL.get('ProtoTreeNet')(cfg).backbone.state_dict()
    assert list(got) == list(trunk)
    for k, v in got.items():
        assert torch.equal(v, trunk[k]), k
