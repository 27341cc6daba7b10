"""The checks the method tests make of a training step: it does not synchronise with the host, a captured step replays
like the eager step, and a trainer captures and replays its own step, alone and against an eager run of the same trainer.

Everything a check captures runs on one side stream, warm-up steps included: autograd binds a parameter's gradient
accumulation to the stream of its first backward, and a capture cannot wait on another stream.  Environment variables
are set through pytest's monkeypatch only, so nothing outlives the test that set it.
"""
import contextlib
import copy
import os

import numpy as np
import pytest
import torch

from conftest import rel_l2

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@contextlib.contextmanager
def no_host_sync():
    """Any host synchronisation inside the block raises (torch's sync debug mode); the mode is off again after it."""
    torch.cuda.set_sync_debug_mode('error')
    try:
        yield
    finally:
        torch.cuda.set_sync_debug_mode(0)


@contextlib.contextmanager
def side_stream():
    """Runs the block on a new stream that starts after the caller's work; the caller's stream then waits for it."""
    cur = torch.cuda.current_stream()
    s = torch.cuda.Stream()
    s.wait_stream(cur)
    with torch.cuda.stream(s):
        yield s
    cur.wait_stream(s)


def capture(fn):
    """-> (graph, outputs): fn() captured into a CUDA graph on the current stream, a side stream (side_stream()).  The
    outputs are static: every replay rewrites them."""
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=torch.cuda.current_stream()):
        out = fn()
    return graph, out


def replay_against_eager(step, module, params, *, grad_bound, seed=None, warmup=2):
    """One step run eagerly and replayed from a capture, from the same state.

    step() zeroes the gradients, runs forward, loss and backward, and returns the list of tensors to compare.  After
    `warmup` steps, module's state_dict is restored before the eager step, before the capture and before the replay;
    with `seed` the CUDA generator is re-seeded before the eager step and before the replay.  Asserts that the returned
    tensors are bit-equal and that each of params' gradients is within grad_bound relative L2 of the eager one (0:
    bit-equal).  -> (eager outputs, replayed outputs)"""
    params = list(params)
    with side_stream():
        for _ in range(warmup):
            step()
        state = {k: v.clone() for k, v in module.state_dict().items()}

        def from_state(fn):
            module.load_state_dict(state)
            if seed is not None:
                torch.cuda.manual_seed(seed)
            return fn()
        eager = [t.detach().clone() for t in from_state(step)]
        eager_g = [p.grad.clone() for p in params]
        module.load_state_dict(state)
        graph, out = capture(step)
        from_state(graph.replay)
    replayed = [t.detach() for t in out]
    assert len(replayed) == len(eager)
    for i, (a, b) in enumerate(zip(replayed, eager)):
        assert torch.equal(a, b), f'output {i}: the replay differs from the eager step'
    for i, (p, e) in enumerate(zip(params, eager_g)):
        if grad_bound == 0:
            assert torch.equal(p.grad, e), f'parameter {i}: the replayed gradient differs from the eager one'
        else:
            err = rel_l2(p.grad, e)
            assert err < grad_bound, f'parameter {i}: the replayed gradient is {err:.2e} from the eager one'
    return eager, replayed


def make_trainer(monkeypatch, name, yaml, *, graph, experiment=None, dataloaders=None, **model):
    """-> examples.ALL_TRAINERS[name] on configs/<yaml>, in train mode, with random initialisation allowed and graph
    replay on or off.  `experiment` and `model` replace entries of those sections of the config."""
    from hawkeye_b200 import examples
    from hawkeye_b200.config import load_config
    monkeypatch.setenv('HAWKEYE_ALLOW_RANDOM_INIT', '1')
    monkeypatch.setenv('HK_CUDA_GRAPH', '1' if graph else '0')
    cfg = load_config(os.path.join(REPO, 'configs', yaml))
    for k, v in (experiment or {}).items():
        cfg.experiment[k] = v
    for k, v in model.items():
        cfg.model[k] = v
    tr = examples.ALL_TRAINERS[name](cfg, dataloaders={} if dataloaders is None else dataloaders)
    tr.model.train()
    return tr


@pytest.fixture
def random_init(monkeypatch):
    """Models built without a pretrained checkpoint keep their random initialisation without a warning."""
    monkeypatch.setenv('HAWKEYE_ALLOW_RANDOM_INIT', '1')


def eager_and_graph_losses(build, batches, *, frozen_groups=()):
    """Trains one epoch on `batches` twice from one state_dict: build(graph) -> a trainer, built after
    torch.manual_seed(0), first eager, then with graph replay, which loads the eager trainer's initial state.  The
    optimizer groups in frozen_groups are held at lr 0 (they still run forward and backward).  -> (per-step losses,
    final model state) of the eager run and of the graph run"""
    runs, state0 = [], None
    for graph in (False, True):
        torch.manual_seed(0)
        tr = build(graph)
        if state0 is None:
            state0 = copy.deepcopy(tr.model.state_dict())
        else:
            tr.model.load_state_dict(state0)
        for i in frozen_groups:
            g = tr.optimizer.param_groups[i]
            g['lr'] = g['initial_lr'] = 0.0                # initial_lr too: a per-step schedule recomputes lr from it
        tr.on_start_epoch(None)
        losses = [float(tr.batch_training(b).item()) for b in batches]     # a replay rewrites the graph's loss tensor
        assert (tr._graph is not None) == graph
        runs.append((losses, {k: v.detach().clone() for k, v in tr.model.state_dict().items()}))
        del tr
    return runs


def assert_trainer_replays(tr, batches):
    """Trains tr, built with graph replay on, one epoch on `batches`: the step was captured with library kernels in it,
    and the meters are finite and in range."""
    tr.on_start_epoch(None)
    for b in batches:
        tr.batch_training(b)
    assert tr._graph is not None and tr._graph['kernels'] > 0
    assert np.isfinite(tr.average_meters['loss'].avg) and 0 <= tr.average_meters['acc'].avg <= 100
