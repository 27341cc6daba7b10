"""Interp-Parts on the device: each hk_ip_* kernel against the fp64 oracle (oracle/interp_parts_oracle.py) with K in {1, 5, 32},
C = 1024, odd maps and N from 1 to 16 (dsmooth and the blur / argmax path of the shaping gradient included), the occupancy
argmax on a planted tie, bitwise repeatability, the full model against fixtures of the unmodified reference
(tests/golden/make_golden_interp_parts.py), the 448x448 batch-16 train step (no host synchronisation, CUDA-graph replay
bit-identical to eager), the shaping term split over two emulated ranks, Tester on the model's triple, and error paths."""
import copy
import json
import os

import numpy as np
import pytest
import torch

import detgen
from conftest import load_golden, rel_l2
from oracle import interp_parts_oracle as O

pytestmark = pytest.mark.gpu
G = load_golden('reference_interp_parts')
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(params=[0, 1], ids=['tf32', 'precise'])
def precise(request):
    from hawkeye_b200 import _lib
    _lib.set_precise(request.param)
    yield request.param
    _lib.set_precise(0)


def _unit_inputs(N, C, H, W, K, seed):
    return (0.03 * detgen.det((N, C, H, W), seed), 0.03 * detgen.det((K, C, 1, 1), seed + 1), 0.3 * detgen.det((K,), seed + 2),
            detgen.det((N, K, C), seed + 3))


def _lib_unit(x, w, sf, Gw, radius, std, coeff=0.5):
    """the library's grouping, occupancy and shaping loss, with the backward of (out . G) + coeff shaping"""
    from hawkeye_b200 import ops_interp_parts as OP
    xn = x.permute(0, 2, 3, 1).contiguous().cuda().requires_grad_(True)
    w, sf = w.cuda().requires_grad_(True), sf.cuda().requires_grad_(True)
    out, assign = OP.grouping(xn, w, sf)
    occ, argmax = OP.occupancy(assign, OP.gaussian_taps(radius, std).cuda(), radius)
    prior = OP.beta_prior(x.shape[0], 1, 0.001).cuda()
    shaping = OP.ShapingLossFn.apply(occ, occ.detach(), prior, 0, 1, OP.SHAPING_EPS)
    ((out * Gw.cuda()).sum() + coeff * shaping).backward()
    return (dict(out=out, assign=assign, occ=occ, argmax=argmax, shaping=shaping),
            dict(x=xn.grad.permute(0, 3, 1, 2), w=w.grad, sf=sf.grad))


def _oracle_unit(x, w, sf, Gw, radius, std, coeff=0.5):
    from hawkeye_b200.ops_interp_parts import beta_prior
    x, w, sf = (t.double().requires_grad_(True) for t in (x, w, sf))
    out, assign = O.grouping(x, w, sf)
    occ = O.occupancy(assign, O.gaussian(radius, std))
    shaping = O.shaping(occ, beta_prior(x.shape[0], 1, 0.001))
    ((out * Gw.double()).sum() + coeff * shaping).backward()
    return dict(out=out, assign=assign, occ=occ, shaping=shaping), dict(x=x.grad, w=w.grad, sf=sf.grad)


@pytest.mark.parametrize('N,H,W,K,radius', [(1, 7, 9, 1, 2), (4, 28, 28, 5, 2), (3, 7, 9, 32, 1), (16, 7, 9, 5, 0),
                                            (2, 28, 28, 32, 2)])
def test_grouping_and_shaping_against_oracle(precise, N, H, W, K, radius):
    args = _unit_inputs(N, 1024, H, W, K, 1600 + N + K)
    val, grad = _lib_unit(*args, radius, 0.4)
    ov, og = _oracle_unit(*args, radius, 0.4)
    assert rel_l2(val['assign'].cpu(), ov['assign'].detach()) < 1e-5
    assert rel_l2(val['out'].cpu(), ov['out'].detach()) < (1e-5 if precise else 2e-3)
    assert rel_l2(val['occ'].cpu(), ov['occ'].detach()) < 1e-5
    assert abs(val['shaping'].item() - ov['shaping'].item()) < 1e-5 * max(1.0, abs(ov['shaping'].item()))
    for k in ('x', 'w', 'sf'):
        _close(grad[k], og[k], 1e-4, k)


def _close(got, ref, tol, name):
    """relative L2 within tol; a reference that vanishes (dsmooth with one part: the softmax over one part is constant and
    F.normalize removes the scale sqrt(beta / 2)) is met to 1e-6 absolute"""
    got, ref = got.detach().cpu().double(), ref.detach().double()
    assert (got - ref).norm() <= tol * ref.norm() + 1e-6, (name, (got - ref).norm().item(), ref.norm().item())


def test_shaping_gradient_reaches_the_blur_window():
    """Only the shaping term, at radius 2: the gradient of assign lies on the 5x5 window under each blurred maximum, and its
    dsmooth is nonzero; both against the oracle."""
    args = list(_unit_inputs(4, 1024, 11, 13, 5, 1700))
    args[3] = torch.zeros_like(args[3])
    val, grad = _lib_unit(*args, 2, 0.4)
    ov, og = _oracle_unit(*args, 2, 0.4)
    assert grad['sf'].abs().max() > 0
    for k in ('x', 'w', 'sf'):
        _close(grad[k], og[k], 1e-4, k)


def test_occupancy_planted_tie():
    from hawkeye_b200 import ops_interp_parts as OP
    a = torch.zeros(2, 3, 9, 10)
    a[0, 0, 2, 3] = a[0, 0, 6, 7] = 1.0              # two equal maxima: the first in row-major order wins
    a[1, 2, 4, 4] = a[1, 2, 4, 2] = 0.5
    occ, am = OP.occupancy(a.cuda(), OP.gaussian_taps(1, 0.4).cuda(), 1)
    Wo = 10 - 2
    assert am[0, 0].item() == (2 - 1) * Wo + (3 - 1)
    assert am[1, 2].item() == (4 - 1) * Wo + (2 - 1)
    assert am[0, 1].item() == 0                      # an all-zero map: position 0
    assert rel_l2(occ.cpu(), O.occupancy(a.double(), O.gaussian(1, 0.4))) < 1e-6


def test_shaping_loss_ranks_ties_and_zero_sign():
    from hawkeye_b200 import ops_interp_parts as OP
    occ = torch.tensor([[0.5, 0.2], [0.5, 0.9], [0.1, 0.2], [0.7, 0.3]])
    prior = OP.beta_prior(4, 1, 0.001)
    prior[1] = 0.5                                   # the second-ranked 0.5 meets its prior exactly: sign(0) = 0
    o = occ.cuda().requires_grad_(True)
    loss = OP.ShapingLossFn.apply(o, o.detach(), prior.cuda(), 0, 1, OP.SHAPING_EPS)
    loss.backward()
    od = occ.double().requires_grad_(True)
    ref = O.shaping(od, prior)
    ref.backward()
    assert abs(loss.item() - ref.item()) < 1e-6
    assert o.grad[0, 0].item() == 0.0 or o.grad[1, 0].item() == 0.0
    assert rel_l2(o.grad.cpu()[:, 1], od.grad[:, 1]) < 1e-6


def _att_inputs(N, K, seed, C=1024, D=2048):
    return (detgen.det((N * K, C), seed), detgen.det((N * K, D), seed + 1), 0.05 * detgen.det((1, C, 1, 1), seed + 2),
            0.1 * detgen.det((1,), seed + 3), 1 + 0.1 * detgen.det((1,), seed + 4), 0.1 * detgen.det((1,), seed + 5),
            detgen.det((N, D), seed + 6), detgen.det((N, K), seed + 7))


@pytest.mark.parametrize('training', [True, False], ids=['train', 'eval'])
@pytest.mark.parametrize('N,K', [(1, 5), (16, 5), (4, 32), (3, 1)])
def test_attention_against_oracle(N, K, training):
    from hawkeye_b200 import ops_interp_parts as OP
    if training and N * K < 2:
        pytest.skip('BatchNorm in train mode needs two values')
    f, post, w, b, gm, bt, Gp, Ga = _att_inputs(N, K, 1800 + N + K)
    bn = torch.nn.BatchNorm2d(1).cuda()
    bn.running_mean.fill_(0.05)
    bn.running_var.fill_(1.3)
    rm0, rv0 = bn.running_mean.double().cpu(), bn.running_var.double().cpu()
    ts = [t.cuda().requires_grad_(True) for t in (f, post, w, b, gm, bt)]
    pooled, att = OP.AttentionPoolFn.apply(*ts, bn, training, N, K)
    ((pooled * Gp.cuda()).sum() + (att * Ga.cuda()).sum()).backward()
    ds = [t.double().requires_grad_(True) for t in (f, post, w, b, gm, bt)]
    op, oa, (rm, rv) = O.attention_pool(*ds, rm0, rv0, training, N, K)
    ((op * Gp.double()).sum() + (oa * Ga.double()).sum()).backward()
    assert rel_l2(pooled.cpu(), op.detach()) < 1e-5
    assert rel_l2(att.cpu(), oa.detach()) < 1e-5
    assert rel_l2(bn.running_mean.cpu(), rm) < 1e-6 and rel_l2(bn.running_var.cpu(), rv) < 1e-6
    for t, d, name in zip(ts, ds, ('f', 'post', 'w', 'b', 'gamma', 'beta')):
        if d.grad.abs().max() > 1e-9:
            assert rel_l2(t.grad.cpu(), d.grad) < 1e-4, name


def test_bitwise_repeatable():
    args = _unit_inputs(8, 1024, 28, 28, 5, 1900)
    a, ga = _lib_unit(*args, 2, 0.4)
    b, gb = _lib_unit(*args, 2, 0.4)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    for k in ga:
        assert torch.equal(ga[k], gb[k]), k


def _shallow_net():
    from hawkeye_b200.methods.interp_parts import ResNet
    net = ResNet([1, 1, 1], 200, 5)
    net.load_state_dict(detgen.state_like(net))
    return net.cuda().train()


def test_model_against_reference_fixture(precise):
    from hawkeye_b200.cfgnode import CfgNode
    from hawkeye_b200.losses import InterpPartsLoss
    net = _shallow_net()
    x = detgen.det((4, 3, 128, 128), 1510).cuda()
    labels = detgen.det_labels(4, 200, 1511).cuda()
    logits, att, assign = net(x)
    assert att.shape == (4, 1, 5, 1) and assign.shape == (4, 5, 8, 8)
    crit = InterpPartsLoss(CfgNode(dict(radius=2, std=0.4, num_parts=5, alpha=1, beta=0.001, coeff=0.5)))
    loss = crit((logits, att, assign), labels)
    loss.backward()
    tol = 1e-4 if precise else 5e-2
    assert rel_l2(logits.detach().cpu(), G['e2e_logits']) < tol
    assert rel_l2(att.detach().cpu(), G['e2e_att']) < tol
    assert rel_l2(assign.detach().cpu(), G['e2e_assign']) < tol
    assert abs(loss.item() - float(G['e2e_loss'])) < tol * abs(float(G['e2e_loss']))
    assert rel_l2(net.attconv[3].running_var.cpu(), G['e2e_running_var_att']) < tol
    if not precise:
        return                       # TF32: the random-init train-mode trunk's drift reaches the gradients (see README)
    params = dict(net.named_parameters())
    for i, k in enumerate(json.loads(bytes(G['e2e_grad_names']).decode())):
        got = params[k].grad.flatten().cpu()[torch.from_numpy(G[f'e2e_grad_{i}_idx'])]
        # sanity bounds: the reference sums its distances as 2 c.x - |x|^2 - |c|^2 in fp32, which cancels on trunk features
        # of this size.  attconv.2.bias feeds a train-mode BatchNorm: its gradient is 0 up to rounding in both
        _close(got, torch.from_numpy(G[f'e2e_grad_{i}']), 5e-2, k)


def test_two_rank_shaping_equals_one_rank():
    """The shaping term as two ranks run it: each holds half the batch, gathers both halves' occupancies, and takes the
    gradient of its rows times the world size; the gradient all-reduce then averages.  That equals the one-rank gradient."""
    from hawkeye_b200 import ops_interp_parts as OP
    occ = torch.rand(16, 5, generator=torch.Generator().manual_seed(3)).cuda()
    prior = OP.beta_prior(16, 1, 0.001).cuda()
    one = occ.clone().requires_grad_(True)
    OP.ShapingLossFn.apply(one, one.detach(), prior, 0, 1, OP.SHAPING_EPS).backward()
    halves = [occ[:8].clone().requires_grad_(True), occ[8:].clone().requires_grad_(True)]
    losses = [OP.ShapingLossFn.apply(h, occ, prior, 8 * r, 2, OP.SHAPING_EPS) for r, h in enumerate(halves)]
    for l in losses:
        l.backward()
    assert losses[0].item() == losses[1].item()
    avg = torch.cat([h.grad for h in halves]) / 2          # what GradAllReduce's averaging leaves of each rank's own rows
    assert torch.allclose(avg, one.grad, rtol=1e-6, atol=0)


def _trainer(monkeypatch, graph=False):
    from hawkeye_b200 import examples
    from hawkeye_b200.config import load_config
    monkeypatch.setenv('HAWKEYE_ALLOW_RANDOM_INIT', '1')
    monkeypatch.setenv('HK_CUDA_GRAPH', '1' if graph else '0')
    cfg = load_config(os.path.join(REPO, 'configs', 'InterpPartsNet.yaml'))
    tr = examples.InterpPartsNetTrainer(cfg, dataloaders={})
    tr.model.train()
    return tr


def _batch(n, seed):
    return {'img': detgen.det((n, 3, 448, 448), seed).pin_memory(), 'label': detgen.det_labels(n, 200, seed + 1).pin_memory()}


def test_train_step_448_no_sync(monkeypatch):
    tr = _trainer(monkeypatch)
    data = _batch(16, 2000)
    lr0 = tr.optimizer.param_groups[1]['lr']
    losses = [float(tr.batch_training(data).item())]
    assert tr.optimizer.param_groups[1]['lr'] < lr0             # the cosine schedule stepped after the batch
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')                      # no host synchronisation inside the step
    try:
        for _ in range(4):
            losses.append(tr.batch_training(data))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    losses[1:] = [float(v.item()) for v in losses[1:]]
    print('interp-parts 448 losses', losses)
    assert all(np.isfinite(losses))
    assert all(torch.isfinite(p).all() for p in tr.model.parameters())
    for m in tr.average_meters.values():
        assert m.avg >= 0 and m.count == 5 * 16


def test_graph_replay_matches_eager(monkeypatch):
    """Six steps with and without the graph.  The trunk (conv1, bn1, layer1-3) is held at lr 0, as the other methods' graph
    tests hold theirs: it still runs forward and backward, and the head, trained by the SGD step under the per-iteration
    schedule, and the losses must then be the same bits."""
    data = _batch(16, 2010)
    out, state0 = {}, None
    for graph in (False, True):
        torch.manual_seed(0)
        tr = _trainer(monkeypatch, graph=graph)
        if state0 is None:
            state0 = copy.deepcopy(tr.model.state_dict())
        else:
            tr.model.load_state_dict(state0)
        tr.optimizer.param_groups[0]['initial_lr'] = tr.optimizer.param_groups[0]['lr'] = 0.0
        losses = [float(tr.batch_training(data).item()) for _ in range(6)]
        out[graph] = (losses, {k: v.detach().clone() for k, v in tr.model.state_dict().items()})
        if graph:
            assert tr._graph is not None
        del tr
    print('interp-parts graph', out[False][0], out[True][0])
    assert out[False][0] == out[True][0]
    for k in out[False][1]:
        assert torch.equal(out[False][1][k], out[True][1][k]), k


def test_tester_reads_logits(monkeypatch):
    from hawkeye_b200.test import Tester
    net = _shallow_net().eval()
    t = Tester.__new__(Tester)
    t.model, t.device = net, torch.device('cuda')
    from hawkeye_b200.test import AverageMeter
    t.average_meters = {'acc': AverageMeter()}
    x = detgen.det((4, 3, 128, 128), 1510)
    with torch.no_grad():
        logits, _, _ = net(x.cuda())
    labels = logits.argmax(1).cpu()
    with torch.no_grad():
        t.batch_validate({'img': x, 'label': labels})
    assert t.average_meters['acc'].avg == 100.0


def test_errors():
    from hawkeye_b200 import _lib, ops_interp_parts as OP
    x = torch.zeros(2, 7, 9, 1024, device='cuda')
    with pytest.raises(_lib.HawkeyeLibError, match='num_parts=33'):
        OP.grouping(x, torch.zeros(33, 1024, 1, 1, device='cuda'), torch.zeros(33, device='cuda'))
    with pytest.raises(_lib.HawkeyeLibError, match='not an NHWC'):
        OP.grouping(x, torch.zeros(5, 512, 1, 1, device='cuda'), torch.zeros(5, device='cuda'))
    with pytest.raises(_lib.HawkeyeLibError, match='K=33'):
        _lib.call('hk_ip_group_fwd', x, x, x, x, x, x, x, x, x, 2, 63, 33, 1024, x, x.numel() * 4, _lib.stream_ptr())
    with pytest.raises(_lib.HawkeyeLibError, match='C=1022'):
        _lib.call('hk_ip_group_fwd', x, x, x, x, x, x, x, x, x, 2, 63, 5, 1022, x, x.numel() * 4, _lib.stream_ptr())
    with pytest.raises(_lib.HawkeyeLibError, match='null pointer'):
        _lib.call('hk_ip_occupancy', None, x, x, x, 2, 5, 7, 9, 1, _lib.stream_ptr())
    with pytest.raises(_lib.HawkeyeLibError, match='radius=4'):
        OP.occupancy(torch.zeros(2, 5, 7, 9, device='cuda'), OP.gaussian_taps(4, 0.4).cuda(), 4)
    with pytest.raises(_lib.HawkeyeLibError, match='radius=4'):
        _lib.call('hk_ip_occupancy', x, x, x, x, 2, 5, 7, 9, 4, _lib.stream_ptr())
    with pytest.raises(_lib.HawkeyeLibError, match='more than one'):
        bn = torch.nn.BatchNorm2d(1).cuda()
        OP.AttentionPoolFn.apply(torch.zeros(1, 1024, device='cuda'), torch.zeros(1, 2048, device='cuda'),
                                 torch.zeros(1, 1024, 1, 1, device='cuda'), torch.zeros(1, device='cuda'),
                                 bn.weight, bn.bias, bn, True, 1, 1)
    with pytest.raises(_lib.HawkeyeLibError, match='grouping unit'):
        OP.occupancy(torch.zeros(2, 5, 7, 9, device='cuda', requires_grad=True), OP.gaussian_taps(1, 0.4).cuda(), 1)
