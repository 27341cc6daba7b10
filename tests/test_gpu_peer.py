"""PeerLearningNet on the GPU: the two-model train step of Examples/PeerLearning.py:82-91 through
PeerLearningTrainer.batch_training against fixtures from the UNMODIFIED reference (tests/golden/make_golden_peer.py), and the
bilinear-pool kernel under concurrent streams (no co-residency assumption, VERDICT r1 weak #11)."""
import os

import numpy as np
import pytest
import torch

import detgen
from conftest import rel_l2

pytestmark = pytest.mark.gpu
G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'reference_peer.npz'))
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize('stage', [1, 2])
def test_peer_learning_train_step_matches_reference(stage, monkeypatch):
    from hawkeye_b200.config import load_config
    from hawkeye_b200.train import PeerLearningTrainer
    from oracle.hop_oracle import VGG16_D
    monkeypatch.setenv('HAWKEYE_ALLOW_RANDOM_INIT', '1')
    cfg = load_config(os.path.join(REPO, 'configs', f'PeerLearning_BCNN_S{stage}.yaml'))
    tr = PeerLearningTrainer(cfg, dataloaders={})
    net = tr.model
    st1 = detgen.vgg_bcnn_state(VGG16_D, 200, seed=100)
    st2 = dict(st1)
    st2['classifier.weight'] = detgen.det((200, 512 * 512), 7001, (2.0 / (512 * 512)) ** 0.5)
    st2['classifier.bias'] = detgen.det((200,), 7002, 0.01)
    net.base_model.load_state_dict(st1)
    net.base_model2.load_state_dict(st2)
    net.train()
    tr.epoch = len(tr.rate_scheduler) - 1                      # drop rate 0.35, as in the fixture
    assert abs(float(tr.rate_scheduler[tr.epoch]) - 0.35) < 1e-12
    x, y = detgen.det((4, 3, 128, 128), 81), detgen.det_labels(4, 200, 82)
    # the step itself (forward of both networks, co-teaching loss, two backwards, optimizer) ...
    before = net.base_model.classifier.bias.detach().clone()
    loss1, loss2 = tr.batch_training({'img': x.pin_memory(), 'label': y.pin_memory()})
    torch.cuda.synchronize()
    t = f'peer_step_s{stage}'
    assert abs(loss1.item() - G[t + '_loss'][0]) < 2e-4 and abs(loss2.item() - G[t + '_loss'][1]) < 2e-4
    assert not torch.equal(before, net.base_model.classifier.bias.detach())          # the optimizer stepped
    # ... and its pieces against the reference: logits of both networks and the head gradients (weights re-loaded, since
    # the step above already updated them)
    net.base_model.load_state_dict(st1)
    net.base_model2.load_state_dict(st2)
    l1, l2 = net(x.cuda())
    e1, e2 = rel_l2(l1.detach().cpu(), G[t + '_logits1']), rel_l2(l2.detach().cpu(), G[t + '_logits2'])
    v1, v2 = tr.criterion(l1, l2, y.cuda(), drop_rate=0.35)
    tr.optimizer.zero_grad()
    v1.backward()
    v2.backward()
    g = {'g1_classifier.bias': net.base_model.classifier.bias.grad, 'g2_classifier.bias': net.base_model2.classifier.bias.grad,
         'g1_classifier.weight_slice': net.base_model.classifier.weight.grad[:, ::4099],
         'g2_classifier.weight_slice': net.base_model2.classifier.weight.grad[:, ::4099]}
    errs = {k: rel_l2(v.cpu(), G[f'{t}_{k}']) for k, v in g.items()}
    print(f'peer stage {stage}: logits {e1:.2e} {e2:.2e} losses {v1.item():.6f} {v2.item():.6f}', {k: f'{v:.1e}' for k, v in errs.items()})
    assert e1 < 1e-3 and e2 < 1e-3 and max(errs.values()) < 2e-3
    if stage == 1:
        assert net._backbones_identical()                       # one backbone pass serves both heads
        assert all(p.grad is None for p in net.base_model.backbone.parameters())


def test_bilinear_pool_under_concurrent_streams():
    """Three streams at once — two running hk_bilinear_pool_fwd, one saturating the SMs with other kernels — so the CTAs of
    a pooling launch are NOT all co-resident.  Results must be exact and nothing may hang (bounded-wait norm exchange)."""
    from hawkeye_b200 import ops
    from oracle import hop_oracle as O
    xs = [torch.relu(detgen.det_uniform((48, 512, 14, 14), 5 + i) - 0.3) for i in range(2)]
    refs = [O.bilinear_pool_fwd(x.double()) for x in xs]
    xg = [x.cuda() for x in xs]
    a = torch.randn(8192, 8192, device='cuda')
    streams = [torch.cuda.Stream() for _ in range(3)]
    outs = [[], []]
    torch.cuda.synchronize()
    for rep in range(6):
        with torch.cuda.stream(streams[2]):
            for _ in range(4):
                a = torch.mm(a, a) * 1e-4
        for i in range(2):
            with torch.cuda.stream(streams[i]):
                outs[i].append(ops.bilinear_pool(xg[i]))
    torch.cuda.synchronize()
    for i in range(2):
        for y in outs[i]:
            worst = max(rel_l2(y[b].cpu(), refs[i][b]) for b in range(0, 48, 7))
            assert worst < 1e-3, worst
