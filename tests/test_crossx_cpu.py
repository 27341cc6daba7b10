"""CrossX on the CPU: the fp64 oracle against fixtures of the unmodified reference (tests/golden/make_golden_crossx.py),
the model's state_dict layout and parameter count, configs/CrossX.yaml, the MultiStep schedule, the trainer's transforms
and its registration."""
import json
import os

import numpy as np
import pytest
import torch

import crossx_inputs as I
import detgen
from conftest import load_golden, rel_l2
from oracle import crossx_oracle as O

G = load_golden('reference_crossx')
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize('P,N', I.LOSS_CASES)
def test_oracle_loss_against_reference(P, N):
    inputs = I.loss_inputs(P, N)
    loss, grads = O.loss(*inputs, I.GAMMA)
    ref = float(G[f'loss_{P}_{N}'])
    assert abs(loss - ref) <= 1e-7 * abs(ref)          # the reference stores its correlation matrix in float32
    for name, g in zip(('xf', 'xp', 'xc', 'fu', 'fp', 'fc'), grads):
        assert rel_l2(g, G[f'd{name}_{P}_{N}']) < 1e-6, name


def test_oracle_closed_form_regulariser_gradient():
    """dL/ds_i = gamma / N^2 (sum_{j != i} s_j - 2 s_i), the same for every row of part i."""
    f = detgen.det((4, 3, 16), 8800, positive=True).double().requires_grad_(True)
    reg, s = O._corr_reg(f, 0.5)
    (ds,) = torch.autograd.grad(reg, f)
    xhat = f.detach() / f.detach().norm(dim=2, keepdim=True)
    want_ds = 0.5 / 16 * (s.sum(0, keepdim=True) - 3 * s)
    proj = want_ds[None] - xhat * (xhat * want_ds[None]).sum(2, keepdim=True)
    assert torch.allclose(ds, proj / f.detach().norm(dim=2, keepdim=True), rtol=1e-10, atol=1e-12)


def _cfg(**kw):
    from hawkeye_b200.cfgnode import CfgNode
    return CfgNode(dict(kw))


@pytest.mark.parametrize('P', [1, 2, 3])
def test_state_dict_layout_and_parameter_count(P):
    import hawkeye_b200 as hb
    net = hb.MODEL.get('CrossX')(_cfg(num_parts=P, num_classes=I.K, pretrained=False))
    layout = json.loads(bytes(G['layout']).decode())[str(P)]
    assert [[k, list(v.shape)] for k, v in net.state_dict().items()] == layout
    assert len(layout) == {1: 320, 2: 354, 3: 369}[P]
    if P == 2:
        assert sum(p.numel() for p in net.parameters()) == 48_307_888


def test_config_builds_the_model_and_checks_parts():
    import hawkeye_b200 as hb
    from hawkeye_b200._lib import HawkeyeLibError
    from hawkeye_b200.config import load_config
    cfg = load_config(os.path.join(REPO, 'configs', 'CrossX.yaml'))
    cfg.model['pretrained'] = False
    net = hb.MODEL.get(cfg.model.name)(cfg.model)
    assert net.nparts == 2 and net.fc_plty.in_features == 2048 and net.fc_ulti.in_features == 4096
    assert cfg.train.criterion.num_parts == 2 and list(cfg.train.criterion.gamma) == [0.5, 0.25, 0.5]
    with pytest.raises(HawkeyeLibError):
        hb.MODEL.get('CrossX')(_cfg(num_parts=4, pretrained=False))


def test_multistep_matches_torch():
    from hawkeye_b200.train import _MultiStep

    class Opt:
        param_groups = [dict(initial_lr=0.0025), dict(initial_lr=0.01)]

    opt = Opt()
    ours = _MultiStep(opt, [15, 25], 0.1)
    p = torch.nn.Parameter(torch.zeros(1))
    ref_opt = torch.optim.SGD([p], lr=0.0025)
    ref = torch.optim.lr_scheduler.MultiStepLR(ref_opt, milestones=[15, 25], gamma=0.1)
    for _ in range(40):
        assert abs(opt.param_groups[0]['lr'] - ref_opt.param_groups[0]['lr']) < 1e-15
        ours.step()
        ref_opt.step()
        ref.step()
    assert abs(opt.param_groups[1]['lr'] - 0.01 * 0.01) < 1e-15


def test_transforms_match_reference():
    from PIL import Image
    from hawkeye_b200.examples import CrossXTrainer
    tf = CrossXTrainer.get_transformers(None, None)
    img = Image.fromarray((detgen.det_uniform((500, 700, 3), 8200).numpy() * 255).astype(np.uint8))
    for split in ('train', 'val'):
        torch.manual_seed(8201)
        t = tf[split](img)
        assert list(t.shape) == list(G[f'tf_{split}_shape'])
        assert np.array_equal(t.numpy()[:, ::16, ::16], G[f'tf_{split}_slice'])
        assert np.allclose(t.double().sum((1, 2)).numpy(), G[f'tf_{split}_sums'], rtol=1e-12)


def test_trainer_registration():
    from hawkeye_b200 import examples
    assert examples.ALL_TRAINERS['CrossX'] is examples.CrossXTrainer
    assert 'CrossX' not in examples.TRAINERS
    with pytest.raises(SystemExit, match='CrossX'):
        examples.main(['nope'])
