"""CIN registry surface on CPU: state_dict keys / shapes identical to the reference's MODEL['CIN']."""
import json
import os

import numpy as np

from conftest import load_golden  # noqa: E402

G = load_golden('reference_cin')


class Cfg(dict):
    __getattr__ = dict.__getitem__


def test_cin_state_dict_matches_reference(monkeypatch):
    monkeypatch.setenv('HAWKEYE_ALLOW_RANDOM_INIT', '1')
    import hawkeye_b200 as hb
    net = hb.MODEL.get('CIN')(Cfg(name='CIN', num_classes=200))
    ref = json.loads(bytes(G['cin_state_keys_json']).decode())
    assert {k: list(v.shape) for k, v in net.state_dict().items()} == ref
    big = hb.MODEL.get('CIN')(Cfg(name='CIN', num_classes=200, spatial_size=(14, 14)))       # 448x448 inputs
    assert big.ChannelInteraction.fc.in_features == 2 * 2048 * 196


def test_osmenet_state_dict_matches_reference(monkeypatch):
    monkeypatch.setenv('HAWKEYE_ALLOW_RANDOM_INIT', '1')
    import hawkeye_b200 as hb
    net = hb.MODEL.get('OSMENet')(Cfg(name='OSMENet', num_attention=2, num_classes=200))
    ref = json.loads(bytes(G['osme_state_keys_json']).decode())
    assert {k: list(v.shape) for k, v in net.state_dict().items()} == ref          # ResNet-101 trunk + OSME + classifier
