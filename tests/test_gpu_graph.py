"""CUDA-graph replay of the train step (Trainer cuda_graph mode) must train exactly like the eager step."""
import pytest

import detgen
from step_check import eager_and_graph_losses, make_trainer

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('cfg_name,trainer', [('BCNN_S2.yaml', 'BCNN'), ('MPN.yaml', 'MPN')])
def test_graph_replay_matches_eager(cfg_name, trainer, monkeypatch):
    size = 128
    batches = [{'img': detgen.det((4, 3, size, size), 200 + i).cuda(), 'label': detgen.det_labels(4, 200, 300 + i).cuda()}
               for i in range(7)]
    (eager, _), (replayed, _) = eager_and_graph_losses(
        lambda graph: make_trainer(monkeypatch, trainer, cfg_name, graph=graph), batches)    # steps 4.. are replays
    print(trainer, eager, replayed)
    for a, b in zip(eager, replayed):
        assert abs(a - b) < 2e-3 * max(1.0, abs(a)), (eager, replayed)
