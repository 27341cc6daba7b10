"""LR schedules of the hot-path methods vs torch's own schedulers, which the reference uses:
LinearLR warm-up -> CosineAnnealingLR via SequentialLR (Examples/CBCNN.py:35-45, Examples/MPN.py:20-30),
CosineAnnealingLR(T_max, eta_min) (train.py:217-218), ReduceLROnPlateau(mode='max', factor=0.1, patience=3, threshold=1e-4)
(Examples/BCNN.py:42-48).  Ours drive the fused optimizers' param_groups; the LR sequences must be identical."""
import numpy as np
import torch

from hawkeye_b200.train import _Cosine, _Plateau


class FakeOpt:
    def __init__(self, lrs):
        self.param_groups = [dict(lr=l, initial_lr=l) for l in lrs]


def _torch_opt(lrs):
    ps = [torch.nn.Parameter(torch.zeros(1)) for _ in lrs]
    return torch.optim.SGD([dict(params=[p], lr=l) for p, l in zip(ps, lrs)], lr=0.1)


def test_warmup_cosine_equals_sequential_lr():
    lrs, T, warm, decay = [0.01, 0.002, 0.05], 100, 5, 0.01
    opt = _torch_opt(lrs)
    sch = torch.optim.lr_scheduler.SequentialLR(
        opt, schedulers=[torch.optim.lr_scheduler.LinearLR(opt, start_factor=decay, total_iters=warm),
                         torch.optim.lr_scheduler.CosineAnnealingLR(opt, T_max=T - warm)], milestones=[warm])
    o = FakeOpt(lrs)
    s = _Cosine(o, T, 0.0, warm, decay)
    for _ in range(60):
        assert np.allclose([g['lr'] for g in o.param_groups], [g['lr'] for g in opt.param_groups], rtol=1e-12, atol=0)
        opt.step(); sch.step(); s.step()


def test_plain_cosine_equals_cosine_annealing_lr():
    opt = _torch_opt([0.01])
    sch = torch.optim.lr_scheduler.CosineAnnealingLR(opt, T_max=20, eta_min=1e-5)
    o = FakeOpt([0.01])
    s = _Cosine(o, 20, 1e-5, 0, 0.01)
    for _ in range(20):
        assert abs(o.param_groups[0]['lr'] - opt.param_groups[0]['lr']) <= 1e-15
        opt.step(); sch.step(); s.step()


def test_plateau_equals_reduce_lr_on_plateau():
    opt = _torch_opt([1.0])
    sch = torch.optim.lr_scheduler.ReduceLROnPlateau(opt, mode='max', factor=0.1, patience=3, threshold=1e-4)
    o = FakeOpt([1.0])
    s = _Plateau(o, 'max', 0.1, 3, 1e-4)
    for acc in [10, 20, 20.001, 19, 18, 20, 20, 21, 21, 21, 21, 21, 21, 22, 1, 1, 1, 1, 1, 1, 1, 1, 1]:
        sch.step(acc); s.step(acc)
        assert o.param_groups[0]['lr'] == opt.param_groups[0]['lr']
    sd = s.state_dict()
    s2 = _Plateau(FakeOpt([1.0]))
    s2.load_state_dict(sd)
    assert s2.state_dict() == sd
