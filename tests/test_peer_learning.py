"""PeerLearningNet against fixtures generated from the unmodified reference
(tests/golden/make_golden_peer.py): registry surface / state_dict, and the co-teaching loss with its gradients."""
import json
import os

import numpy as np
import pytest
import torch

import detgen

G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'reference_peer.npz'))


class Cfg(dict):
    __getattr__ = dict.__getitem__


def test_registry_builds_peer_net_with_reference_state_dict():
    import hawkeye_b200 as hb
    net = hb.MODEL.get('PeerLearningNet')(Cfg(name='PeerLearningNet', base_model=Cfg(name='BCNN', stage=1, num_classes=200),
                                              drop_rate=0.35, T_k=10))
    ref = json.loads(bytes(G['peer_state_keys_json']).decode())
    ours = {k: list(v.shape) for k, v in net.state_dict().items()}
    assert ours == ref                                               # base_model.* / base_model2.*: 56 tensors, same shapes
    trainable = sorted(k for k, p in net.named_parameters() if p.requires_grad)
    assert trainable == sorted(s.decode() for s in G['peer_trainable_s1'])
    # the second classifier is re-initialised (PeerLearningNet.py:15), the backbones are copies
    assert not torch.equal(net.base_model.classifier.weight, net.base_model2.classifier.weight)
    assert torch.equal(net.base_model.backbone[0].weight, net.base_model2.backbone[0].weight)
    assert net.base_model.backbone[0].weight.data_ptr() != net.base_model2.backbone[0].weight.data_ptr()


@pytest.mark.parametrize('tag', ['mixed', 'mixed_b', 'all_agree', 'all_disagree', 'drop0'])
def test_peer_learning_loss_matches_reference(tag):
    from hawkeye_b200.losses import peer_learning_loss
    N, K, s1, s2, s3, dr = G[f'peer_{tag}_meta']
    N, K = int(N), int(K)
    l1 = detgen.det((N, K), int(s1), 2.0).requires_grad_(True)
    l2 = torch.from_numpy(G[f'peer_{tag}_l2in']).clone().requires_grad_(True)
    y = detgen.det_labels(N, K, int(s3))
    v1, v2 = peer_learning_loss(l1, l2, y, float(dr))
    assert abs(v1.item() - G[f'peer_{tag}_loss'][0]) < 1e-6 and abs(v2.item() - G[f'peer_{tag}_loss'][1]) < 1e-6
    g1, = torch.autograd.grad(v1, l1)
    g2, = torch.autograd.grad(v2, l2)
    assert np.allclose(g1.numpy(), G[f'peer_{tag}_g1'], rtol=1e-5, atol=1e-7)
    assert np.allclose(g2.numpy(), G[f'peer_{tag}_g2'], rtol=1e-5, atol=1e-7)
