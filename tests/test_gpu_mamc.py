"""MAMC / N-pairs loss kernels (hk_l2norm_rows_*, hk_npair_loss, 3xTF32 GEMMs) against reference-generated fixtures
(tests/golden/make_golden_cin.py imports model/loss/MAMC_loss.py) and the fp64 oracle at a realistic size."""
import os

import numpy as np
import pytest
import torch

from conftest import load_golden, rel_l2

pytestmark = pytest.mark.gpu
G = load_golden('reference_cin')


@pytest.mark.parametrize('tag', ['npair_b8_p2', 'npair_b12_p3', 'npair_b6_p2_allsame', 'npair_b4_p2_alldiff'])
def test_npairs_vs_reference(tag):
    from hawkeye_b200.losses import NPairsLoss
    f = torch.from_numpy(G[f'{tag}_feats']).cuda().requires_grad_(True)
    lab = torch.from_numpy(G[f'{tag}_labels']).cuda()
    loss = NPairsLoss()(f, lab)
    loss.backward()
    ref = float(G[f'{tag}_loss'])
    e = rel_l2(f.grad.cpu(), G[f'{tag}_dfeats'])
    print(f'{tag}: loss {loss.item():.6f} vs {ref:.6f}; grad rel {e:.2e}')
    assert abs(loss.item() - ref) < 1e-4 * max(1.0, abs(ref)) and e < 1e-3


def test_mamc_vs_reference():
    from hawkeye_b200.losses import MAMCLoss

    class Cfg(dict):
        __getattr__ = dict.__getitem__
    crit = MAMCLoss(Cfg(lambda_a=0.5, use_mamc=True))
    pred = torch.from_numpy(G['mamc_pred']).cuda().requires_grad_(True)
    parts = torch.from_numpy(G['mamc_parts']).cuda().requires_grad_(True)
    loss = crit((pred, parts), torch.from_numpy(G['mamc_labels']).cuda())
    loss.backward()
    assert abs(loss.item() - float(G['mamc_loss'])) < 1e-4
    assert rel_l2(pred.grad.cpu(), G['mamc_dpred']) < 5e-4 and rel_l2(parts.grad.cpu(), G['mamc_dparts']) < 1e-3
    assert int(crit.last_correct.item()) == int((pred.argmax(1).cpu() == torch.from_numpy(G['mamc_labels'])).sum())


def test_npairs_osme_size_vs_oracle():
    """OSMENet's own shape: 16 samples x 2 attentions x 1024 features, 4 classes x 4 samples (BalancedBatchSampler)."""
    import detgen
    from hawkeye_b200.losses import NPairsLoss
    from oracle import hop_oracle as O
    f = detgen.det((16, 2, 1024), 77)
    lab = torch.arange(16) // 4
    fd = f.double().requires_grad_(True)
    ref = O.npairs_loss(fd, lab)
    ref.backward()
    fg = f.cuda().requires_grad_(True)
    loss = NPairsLoss()(fg, lab.cuda())
    loss.backward()
    e = rel_l2(fg.grad.cpu(), fd.grad)
    print(f'npairs 16x2x1024: loss {loss.item():.6f} vs {ref.item():.6f}; grad rel {e:.2e}')
    assert abs(loss.item() - ref.item()) < 1e-4 and e < 1e-3


def test_osmenet_train_step(monkeypatch):
    """Examples/OSMENet.py:60-76 end to end on the library: ResNet-101 trunk -> OSME -> (logits, attention features) ->
    MAMCLoss -> backward -> SGD step through OSMENetTrainer.batch_training, on a class-balanced batch.  Checks that the loss is
    what the fp64 oracle computes from the model's own outputs, that every parameter received a finite gradient step and that a
    few steps on the same batch drive the loss down."""
    import detgen
    from hawkeye_b200.config import load_config
    from hawkeye_b200.examples import OSMENetTrainer
    from oracle import hop_oracle as O
    monkeypatch.setenv('HAWKEYE_ALLOW_RANDOM_INIT', '1')
    cfg = load_config(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'configs', 'OSMENet.yaml'))
    cfg.model['feature_shape'] = 4                   # 128x128 inputs -> 4x4 trunk output
    cfg.train.optimizer['lr'] = 0.01
    tr = OSMENetTrainer(cfg, dataloaders={})
    tr.model.train()
    x = detgen.det((8, 3, 128, 128), 301)
    y = (torch.arange(8) // 2).to(torch.int64)        # 4 classes x 2 samples
    with torch.no_grad():
        pred, parts = tr.model(x.cuda())
    ref = O.mamc_loss(pred.double().cpu(), parts.double().cpu(), y).item()
    before = [p.detach().clone() for p in tr.model.parameters()]
    losses = [tr.batch_training({'img': x.pin_memory(), 'label': y.pin_memory()}).item() for _ in range(4)]
    torch.cuda.synchronize()
    print('osmenet losses', losses, 'oracle on the first forward', ref)
    # train-mode BN uses batch statistics in both passes; the no_grad forward above also updated running stats only
    assert abs(losses[0] - ref) < 2e-3 * max(1.0, abs(ref))
    assert all(torch.isfinite(p).all() for p in tr.model.parameters())
    moved = sum(int(not torch.equal(a, b.detach())) for a, b in zip(before, tr.model.parameters()))
    assert moved == len(before)
    assert losses[-1] < losses[0]
