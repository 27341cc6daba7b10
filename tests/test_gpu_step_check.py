"""tests/step_check.py can fail: a step whose draw is not re-seeded does not replay like the eager step, and a host
synchronisation inside no_host_sync() raises."""
import pytest
import torch

from step_check import no_host_sync, replay_against_eager

pytestmark = pytest.mark.gpu


class Scale(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.w = torch.nn.Parameter(torch.linspace(0.5, 1.5, 4096, device='cuda'))


def _noisy_step(m, x):
    def step():
        m.zero_grad()
        y = m.w * x * torch.rand_like(x)
        loss = y.square().sum()
        loss.backward()
        return [y, loss]
    return step


def test_replay_against_eager_fails_an_unseeded_draw():
    m, x = Scale(), torch.linspace(-1.0, 1.0, 4096, device='cuda')
    with pytest.raises(AssertionError, match='output 0'):
        replay_against_eager(_noisy_step(m, x), m, m.parameters(), grad_bound=0)
    replay_against_eager(_noisy_step(m, x), m, m.parameters(), grad_bound=0, seed=5)     # re-seeded: the same draws


def test_no_host_sync_raises_on_item():
    x = torch.ones(8, device='cuda')
    with pytest.raises(RuntimeError, match='synchroniz'):
        with no_host_sync():
            x.sum().item()
    assert torch.cuda.get_sync_debug_mode() == 0
