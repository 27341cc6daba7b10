"""Checkpoint wire format against the reference's (reference train.py:369-395, test.py:64-76): a .pth with the exact
state_dict layout the UNMODIFIED reference writes — key order, shapes and dtypes recorded from it in
tests/golden/reference_checkpoint_layout.json — loads into the native classes key for key, plain and DataParallel-prefixed,
and the file hawkeye_b200.Trainer.save_model's code path writes has that same layout, so the reference loads it strictly."""
import json
import os
import sys

import pytest
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
LAYOUT = json.load(open(os.path.join(REPO, 'tests', 'golden', 'reference_checkpoint_layout.json')))


class Cfg(dict):
    __getattr__ = dict.__getitem__


@pytest.mark.parametrize('name,kw', [('BCNN', dict(stage=2, num_classes=200)),
                                     ('MPN', dict(iter_num=5, is_sqrt=True, is_vec=True, input_dim=2048,
                                                  dimension_reduction=256, num_classes=200))])
def test_reference_checkpoint_round_trip(name, kw, tmp_path, monkeypatch):
    monkeypatch.setenv('HAWKEYE_ALLOW_RANDOM_INIT', '1')
    import hawkeye_b200 as hb
    from hawkeye_b200.utils import load_state_dict
    g = torch.Generator().manual_seed(1)
    ref = {}                                                                  # what the reference's train.py:375 saves
    for k, shape, dtype in LAYOUT[name]:
        dt = getattr(torch, dtype)
        ref[k] = torch.randn(shape, generator=g).to(dt) if dt.is_floating_point else torch.randint(0, 7, shape, generator=g).to(dt)
    path = str(tmp_path / f'{name}_epoch_1.pth')
    torch.save(ref, path)
    ours = hb.MODEL.get(name)(Cfg(name=name, **kw))
    load_state_dict(ours, torch.load(path, map_location='cpu'))               # hawkeye_b200.test.Tester.get_model
    b = ours.state_dict()
    assert list(ref.keys()) == list(b.keys())
    assert all(torch.equal(ref[k], b[k]) for k in ref)
    # DataParallel-prefixed files (the reference saves self.model.state_dict() of the wrapped module, train.py:375)
    torch.save({'module.' + k: v for k, v in ref.items()}, path)
    ours2 = hb.MODEL.get(name)(Cfg(name=name, **kw))
    load_state_dict(ours2, torch.load(path, map_location='cpu'))
    assert all(torch.equal(ref[k], ours2.state_dict()[k]) for k in ref)
    # and back: our file has the reference's layout (its strict load_state_dict, test.py:74-75, checks keys and shapes)
    torch.save({k: v.detach().cpu().clone() for k, v in ours.state_dict().items()}, path)     # Trainer.save_model
    mine = torch.load(path, map_location='cpu')
    assert [[k, list(v.shape), str(v.dtype).replace('torch.', '')] for k, v in mine.items()] == LAYOUT[name]
    assert all(torch.equal(ref[k], mine[k]) for k in ref)
