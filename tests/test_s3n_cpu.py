"""S3N without a GPU: the fp64 oracle of the sampler (oracle/s3n_oracle.py) against the reference's own fixtures for p = 0, 1
and 2 (tests/golden/make_golden_s3n.py), the state_dict surface, the trainer's parameter groups and p schedule, the label
smoothing that MultiSmoothLoss maps onto hk_softmax_ce_ls, and the shipped config."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import load_golden
from hawkeye_b200.methods.s3n import make_gaussian
from oracle import s3n_oracle as O

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFG = dict(num_classes=200, image_size=128, radius=0.12, radius_inv=0.3, base_ratio=0.09)


class Cfg(dict):
    __getattr__ = dict.__getitem__


def draws_at_positions(g, N):
    """The reference's per-peak random.uniform draws placed at their peaks' positions ([N, 961], 2 elsewhere: never drawn)."""
    d = np.full((N, 31 * 31), 2.0)
    d[g['draw_image'], g['draw_pos']] = g['draw_value']
    return d


def oracle_maps(g, p):
    N = g['crm'].shape[0]
    dms, _, _ = O.decision_maps(O.interpolate_maps(g['crm']))
    r, ri = torch.tensor([0.12], dtype=torch.float64), torch.tensor([0.3], dtype=torch.float64)
    xs, xs_inv, recs = O.sampling_maps(dms, p, r, ri, 0.09, draws_at_positions(g, N) if p == 1 else None)
    return dms, xs, xs_inv, recs


@pytest.mark.parametrize('p', [0, 1, 2])
def test_oracle_sampler_matches_reference(p):
    g = load_golden(f'reference_s3n.{p}')
    N = g['crm'].shape[0]
    dms, xs, xs_inv, recs = oracle_maps(g, p)
    np.testing.assert_allclose(dms.reshape(N, -1).numpy(), g['dm'], rtol=0, atol=1e-5)
    for n in range(N):
        ref = g[f'peaks_{n}']
        assert recs[n][0].tolist() == (ref[:, 0] * 31 + ref[:, 1]).tolist()
    np.testing.assert_allclose(xs.detach().numpy(), g['xs'], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(xs_inv.detach().numpy(), g['xs_inv'], rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize('p', [0, 1, 2])
def test_oracle_grid_and_warp_match_reference(p):
    """From the reference's own sampling maps: the grids (every 4th row and column) and the sampled images."""
    import detgen
    g = load_golden(f'reference_s3n.{p}')
    N = g['xs'].shape[0]
    coarse = O.coarse_grid(np.concatenate([g['xs'], g['xs_inv']]), torch.from_numpy(make_gaussian(61, fwhm=13)).float())
    fine = O.fine_grid(coarse, 128)
    np.testing.assert_allclose(fine[:N, ::4, ::4].numpy(), g['grid_zoom'], rtol=0, atol=2e-5)
    np.testing.assert_allclose(fine[N:, ::4, ::4].numpy(), g['grid_inv'], rtol=0, atol=2e-5)
    x = detgen.det((N, 3, 128, 128), 5100)
    sampled = O.warp(x, coarse).reshape(-1)[torch.from_numpy(g['sampled_idx'])]
    # the reference's fp32 grid rounds at ~1e-5 of [-1, 1], ~1e-3 pixel at 128: on a noise image that moves a sample ~1e-3
    np.testing.assert_allclose(sampled.numpy(), g['sampled'], rtol=0, atol=5e-3)


def test_multi_smooth_loss_eps_mapping():
    """hk_softmax_ce_ls's target (1 - eps) onehot + eps / K equals the reference's smoothed target at eps = (1-r)K/(K-1)."""
    from hawkeye_b200.losses import smooth_ratio_eps
    K, r = 200, 0.85
    z = torch.randn(6, K, dtype=torch.float64, generator=torch.Generator().manual_seed(1))
    y = torch.tensor([0, 5, 199, 17, 17, 3])
    eps = smooth_ratio_eps(r, K)
    ls = F.cross_entropy(z, y, label_smoothing=eps)
    logp = F.log_softmax(z, 1)
    m = torch.zeros_like(z).scatter_(1, y[:, None], 1)
    ref = -(logp * (r * m + (1 - r) * (1 - m) / (K - 1))).sum(1).mean()
    assert abs(ls.item() - ref.item()) < 1e-12
    outs = tuple(torch.randn(6, K, dtype=torch.float64, generator=torch.Generator().manual_seed(i)) for i in range(4))
    total = sum(F.cross_entropy(o, y, label_smoothing=eps if i in (1, 3) else 0.0) for i, o in enumerate(outs))
    assert abs(total.item() - O.multi_smooth_loss(outs, y, r).item()) < 1e-12


def test_state_dict_keys_match_reference_and_load_strictly():
    import hawkeye_b200 as hb
    g = load_golden('reference_s3n.0')
    ref_keys = json.loads(bytes(g['state_keys_json']).decode())
    net = hb.MODEL.get('S3N')(Cfg(CFG))
    sd = net.state_dict()
    assert list(sd.keys()) == ref_keys
    assert any(k.startswith('backbone.fc.') for k in sd) and 'features.7.2.conv3.weight' in sd
    assert {'radius.scale', 'radius_inv.scale', 'filter.weight', 'map_origin.weight', 'map_origin.bias'} <= set(sd)
    other = hb.MODEL.get('S3N')(Cfg(CFG))
    other.load_state_dict({k: v.clone() + 1 if v.is_floating_point() else v for k, v in sd.items()}, strict=True)
    assert torch.equal(other.features[0].weight, other.backbone.conv1.weight)       # one module under two names
    assert not isinstance(net.P_basis, torch.nn.Parameter) and 'P_basis' not in sd
    assert torch.allclose(net.filter.weight[0, 0], torch.from_numpy(make_gaussian(61, 13)).float())


def test_image_size_must_allow_the_stride2_buffer():
    import hawkeye_b200 as hb
    with pytest.raises(ValueError, match='multiple of 64'):
        hb.MODEL.get('S3N')(Cfg(CFG, image_size=224))


def test_trainer_parameter_groups():
    """Four groups: the classifiers at lr, radius at 1e-5 lr, filter at 1e-5 lr, everything else (radius_inv included) at
    0.1 lr (Examples/S3N.py:37-56)."""
    import hawkeye_b200 as hb
    from hawkeye_b200.examples import S3NTrainer
    net = hb.MODEL.get('S3N')(Cfg(CFG))

    class T:
        get_model_module = lambda self: net          # noqa: E731
    groups = S3NTrainer.param_groups(T())
    assert [m for _, m in groups] == [1.0, 1e-5, 1e-5, 0.1]
    names = {id(p): n for n, p in net.named_parameters()}
    cls, rad, filt, rest = ([names[id(p)] for p in g] for g, _ in groups)
    assert sorted(cls) == sorted(n for n in names.values() if 'classifier' in n) and len(cls) == 8
    assert rad == ['radius.scale'] and filt == ['filter.weight']
    assert 'radius_inv.scale' in rest and 'backbone.conv1.weight' in rest
    never = {'backbone.fc.weight', 'backbone.fc.bias', 'map_origin.weight', 'map_origin.bias'}
    assert not never & set(rest) and len(cls) + len(rad) + len(filt) + len(rest) + 4 == len(list(net.parameters()))
    assert S3NTrainer.early_group(T()) == 0


def test_early_group_is_reached_by_the_loss():
    """The early all-reduce group (the classifiers) launches once every one of its parameters has a gradient: each must be
    reached by the loss.  The four classifiers, applied to pooled features as the model applies them, under the reference's
    MultiSmoothLoss in fp64; the whole model's trained parameters are checked on the device (test_gpu_s3n)."""
    import hawkeye_b200 as hb
    from hawkeye_b200.examples import S3NTrainer
    net = hb.MODEL.get('S3N')(Cfg(CFG)).double()

    class T:
        get_model_module = lambda self: net          # noqa: E731
    early = S3NTrainer.param_groups(T())[S3NTrainer.early_group(T())][0]
    pools = [torch.randn(2, 2048, dtype=torch.float64) for _ in range(3)]
    outs = (net.con_classifier(torch.cat(pools, 1)), net.raw_classifier(pools[0]), net.sampler_classifier(pools[1]),
            net.sampler_classifier1(pools[2]))
    O.multi_smooth_loss(outs, torch.tensor([1, 2]), 0.85).backward()
    assert len(early) == 8 and all(p.grad is not None and p.grad.abs().max() > 0 for p in early)


def test_p_schedule():
    from hawkeye_b200.examples import ALL_TRAINERS, S3NTrainer
    assert ALL_TRAINERS['S3N'] is S3NTrainer
    assert [S3NTrainer.train_p(e) for e in (0, 19, 20, 99)] == [0, 0, 1, 1]
    assert [S3NTrainer.val_p(e) for e in (0, 19, 20, 99)] == [1, 1, 2, 2]


def test_config_loads_and_builds():
    import hawkeye_b200 as hb
    from hawkeye_b200.config import load_config
    cfg = load_config(os.path.join(REPO, 'configs', 'S3N.yaml'))
    assert cfg.model.name == 'S3N' and cfg.train.criterion.smooth_ratio == 0.85
    assert (cfg.model.radius, cfg.model.radius_inv, cfg.model.base_ratio) == (0.12, 0.3, 0.09)
    assert (cfg.train.scheduler.T_max, cfg.train.scheduler.eta_min) == (100, 1e-6)
    net = hb.MODEL.get(cfg.model.name)(cfg.model)
    assert net.input_size_net == 448 and net.base_ratio == 0.09
