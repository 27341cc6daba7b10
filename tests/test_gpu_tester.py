"""Evaluation entry point: hawkeye_b200.test.Tester over a synthetic loader, fp32 and uint8 batches."""
import os

import pytest
import torch

import detgen
from conftest import rel_l2

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_normalize_u8_matches_torchvision_arithmetic():
    from hawkeye_b200.test import normalize_u8, IMAGENET_MEAN, IMAGENET_STD
    g = torch.Generator().manual_seed(3)
    u8 = torch.randint(0, 256, (3, 37, 41, 3), generator=g, dtype=torch.uint8)
    ref = (u8.permute(0, 3, 1, 2).float() / 255.0 - torch.tensor(IMAGENET_MEAN).view(1, 3, 1, 1)) / torch.tensor(IMAGENET_STD).view(1, 3, 1, 1)
    out = normalize_u8(u8.cuda())
    assert out.shape == (3, 3, 37, 41) and rel_l2(out.cpu(), ref) < 1e-6


def test_tester_runs_checkpoint_and_reports_accuracy(tmp_path, monkeypatch):
    import hawkeye_b200 as hb
    from hawkeye_b200.cfgnode import CfgNode
    from hawkeye_b200.test import Tester, normalize_u8
    from oracle.hop_oracle import VGG16_D
    monkeypatch.setenv('HAWKEYE_ALLOW_RANDOM_INIT', '1')
    path = str(tmp_path / 'best_model.pth')
    torch.save({'module.' + k: v for k, v in detgen.vgg_bcnn_state(VGG16_D, 200, seed=100).items()}, path)   # DataParallel-style keys
    cfg = CfgNode(dict(experiment=dict(name='t', cuda=[0]), dataset=dict(batch_size=4, num_workers=0,
                                                                         transformer=dict(resize_size=128, image_size=128)),
                       model=dict(name='BCNN', num_classes=200, load=path)))
    g = torch.Generator().manual_seed(5)
    u8 = [torch.randint(0, 256, (4, 128, 128, 3), generator=g, dtype=torch.uint8) for _ in range(2)]
    # labels = the model's own predictions for the first batch, something else for the second: accuracy must be 50 %
    t = Tester(cfg, dataloader=[])
    with torch.no_grad():
        pred0 = t.model.eval()(normalize_u8(u8[0].cuda())).argmax(1).cpu()
        pred1 = t.model(normalize_u8(u8[1].cuda())).argmax(1).cpu()
    loader = [{'img': u8[0], 'label': pred0}, {'img': u8[1], 'label': (pred1 + 1) % 200}]
    t = Tester(cfg, dataloader=loader)
    assert abs(t.test() - 50.0) < 1e-6
    # the fp32 route (what the reference's loader yields) gives the same logits
    f32 = normalize_u8(u8[0].cuda())
    t2 = Tester(cfg, dataloader=[{'img': f32.cpu(), 'label': pred0}])
    assert abs(t2.test() - 100.0) < 1e-6
