"""APINet on the device: pair mining against the reference's get_pairs and the fp64 oracle, the deterministic pair
gather / scatter, the gate and dropout kernels against the oracle fed the numpy-regenerated masks, the head and the loss
against fixtures of the unmodified reference (tests/golden/make_golden_apinet.py), the 224x224 train step (no host
synchronisation, frozen backbone in the warm-up), CUDA-graph replay and evaluation through Tester."""
import numpy as np
import pytest
import torch
import torch.nn as nn

import detgen
from conftest import load_golden, rel_l2
from oracle import apinet_oracle as A
from step_check import eager_and_graph_losses, make_trainer, no_host_sync

pytestmark = pytest.mark.gpu
G = load_golden('reference_apinet')


def _s():
    from hawkeye_b200 import _lib
    return _lib.stream_ptr()


def test_pairs_match_reference_get_pairs():
    from hawkeye_b200.ops_apinet import mine_pairs
    for tag in ('single', 'ties', 'alldiff', 'allsame', 'n40'):
        emb, lab = torch.as_tensor(G[f'pairs_{tag}_emb']), torch.as_tensor(G[f'pairs_{tag}_labels'])
        n = emb.shape[0]
        idx2, l1, l2 = mine_pairs(emb.cuda(), lab.cuda())
        idx2 = idx2.cpu().numpy()
        assert np.array_equal(idx2[:n], G[f'pairs_{tag}_intra']), (tag, idx2[:n], G[f'pairs_{tag}_intra'])
        assert np.array_equal(idx2[n:], G[f'pairs_{tag}_inter']), (tag, idx2[n:], G[f'pairs_{tag}_inter'])
        assert np.array_equal(l2.cpu().numpy(), G[f'pairs_{tag}_labels2']), tag
        assert torch.equal(l1.cpu(), torch.cat([lab, lab]))


def test_pairs_n40_against_fp64_oracle():
    from hawkeye_b200.ops_apinet import mine_pairs
    pool = detgen.det((40, 2048), 410, positive=True)
    lab = torch.arange(10).repeat_interleave(4)
    intra, inter, d = A.apinet_pairs(pool, lab)
    idx2 = mine_pairs(pool.cuda(), lab.cuda())[0].cpu().numpy()
    L = lab.numpy()
    checked = 0
    for i in range(40):
        for got, want, cand in ((idx2[i], intra[i], (L == L[i]) & (np.arange(40) != i)), (idx2[40 + i], inter[i], L != L[i])):
            v = np.sort(d[i][cand])
            if v[1] - v[0] > 1e-4 * abs(v[0]):
                assert got == want, (i, got, want)
                checked += 1
            else:
                assert cand[got] and d[i, got] - v[0] <= 1e-4 * abs(v[0])
    assert checked > 60


def test_gather_scatter_deterministic():
    from hawkeye_b200 import _lib
    n, D = 40, 2048
    pool = detgen.det((n, D), 411).cuda()
    g = np.random.RandomState(412)
    idx2 = torch.from_numpy(np.concatenate([g.randint(0, 3, n), g.randint(0, 2, n)]).astype(np.int64)).cuda()   # heavy duplication
    mutual = torch.empty(2 * n, 2 * D, device='cuda')
    _lib.call('hk_apinet_gather', pool, idx2, mutual, n, D, _s())
    idx1 = torch.cat([torch.arange(n), torch.arange(n)]).cuda()
    assert torch.equal(mutual, torch.cat([pool[idx1], pool[idx2]], 1))
    dm = detgen.det((2 * n, 2 * D), 413).cuda()
    outs = []
    for _ in range(2):
        dpool = torch.empty(n, D, device='cuda')
        _lib.call('hk_apinet_scatter', dm, idx2, dpool, n, D, _s())
        outs.append(dpool)
    assert torch.equal(outs[0], outs[1])
    ref = torch.zeros(n, D, dtype=torch.float64)
    dmd = dm.double().cpu()
    ref.index_add_(0, idx1.cpu(), dmd[:, :D])
    ref.index_add_(0, idx2.cpu(), dmd[:, D:])
    assert (outs[0].double().cpu() - ref).abs().max().item() <= 1e-6 * ref.abs().max().item()
    assert rel_l2(outs[0].cpu(), ref) < 1e-6


def _gate_oracle(m, mutual, seed, p):
    D = m.shape[1]
    m, f1, f2 = m.double().cpu(), mutual[:, :D].double().cpu(), mutual[:, D:].double().cpu()
    masks = [torch.from_numpy(A.dropout_keep(seed, 1 + k, tuple(m.shape), p)).double() for k in range(4)] if p > 0 else None
    sc = 1.0 / (1.0 - p)
    g1, g2 = torch.sigmoid(m * f1), torch.sigmoid(m * f2)
    o = [g1 * f1 + f1, g2 * f1 + f1, g2 * f2 + f2, g1 * f2 + f2]                      # f1s, f1o, f2s, f2o
    if masks is not None:
        o = [t * mk * sc for t, mk in zip(o, masks)]
    return torch.cat([o[0], o[2], o[1], o[3]])


def _gate(m, mutual, p, seed_t, dout=None):
    from hawkeye_b200 import _lib
    R, D = m.shape
    out = torch.empty(4 * R, D, device='cuda')
    _lib.call('hk_apinet_gate_fwd', m, mutual, out, R, D, float(p), seed_t, 1, _s())
    if dout is None:
        return out
    dm, dmut = torch.empty_like(m), torch.empty_like(mutual)
    _lib.call('hk_apinet_gate_bwd', m, mutual, dout, dm, dmut, R, D, float(p), seed_t, 1, _s())
    return out, dm, dmut


def test_gate_and_dropout_against_oracle_masks():
    from hawkeye_b200 import _lib
    R, D, p = 16, 512, 0.5
    m, mutual = detgen.det((R, D), 414).cuda(), detgen.det((R, 2 * D), 415).cuda()
    dout = detgen.det((4 * R, D), 416).cuda()
    seed = 0x1234_5678_9abc
    seed_t = torch.tensor([seed], dtype=torch.int64, device='cuda')
    out, dm, dmut = _gate(m, mutual, p, seed_t, dout)
    md, mutd = m.double().cpu().requires_grad_(True), mutual.double().cpu().requires_grad_(True)
    ref = _gate_oracle(md, mutd, seed, p)
    (ref * dout.double().cpu()).sum().backward()
    assert rel_l2(out.cpu(), ref.detach()) < 1e-5
    assert rel_l2(dm.cpu(), md.grad) < 1e-5 and rel_l2(dmut.cpu(), mutd.grad) < 1e-5
    # the same seed gives the same masks, a new one different masks
    assert torch.equal(_gate(m, mutual, p, seed_t), out)
    other = _gate(m, mutual, p, seed_t + 1)
    assert 0.3 < ((other == 0) != (out == 0)).float().mean().item() < 0.7
    # p = 0 (and eval mode, which passes p = 0): no dropout at all
    assert rel_l2(_gate(m, mutual, 0.0, None).cpu(), _gate_oracle(m, mutual, seed, 0.0)) < 1e-6
    # standalone dropout: exactly x * keep * 2, the backward recomputes the same mask
    x = detgen.det((R, 512), 417).cuda()
    y, dx = torch.empty_like(x), torch.empty_like(x)
    _lib.call('hk_dropout_fwd', x, y, x.numel(), p, seed_t, 0, _s())
    _lib.call('hk_dropout_bwd', x, dx, x.numel(), p, seed_t, 0, _s())
    keep = torch.from_numpy(A.dropout_keep(seed, 0, tuple(x.shape), p)).cuda()
    assert torch.equal(y, torch.where(keep, x * 2, torch.zeros_like(x))) and torch.equal(dx, y)
    _lib.call('hk_dropout_fwd', x, y, x.numel(), 0.0, None, 0, _s())
    assert torch.equal(y, x)


def _head_net(monkeypatch):
    import hawkeye_b200 as hb
    monkeypatch.setenv('HAWKEYE_ALLOW_RANDOM_INIT', '1')

    class Cfg(dict):
        __getattr__ = dict.__getitem__
    net = hb.MODEL.get('APINet')(Cfg(name='APINet', num_classes=200))
    net.backbone = nn.Identity()                  # the fixture feeds a [n, 2048, 7, 7] trunk map
    net.load_state_dict(detgen.state_like(net))
    net.drop.p = 0.0
    return net.cuda().train()


@pytest.mark.parametrize('precise', [0, 1])
def test_head_matches_reference(precise, monkeypatch):
    from hawkeye_b200 import _lib
    net = _head_net(monkeypatch)
    n = 8
    conv = detgen.det((n, 2048, 7, 7), 402, positive=True).cuda().requires_grad_(True)
    lab = torch.arange(4).repeat_interleave(2).cuda()
    _lib.set_precise(precise)
    try:
        s, o, l1, l2 = net(conv, lab)
        r1, r2 = detgen.det(s.shape, 403).cuda(), detgen.det(o.shape, 404).cuda()
        ((s * r1).sum() + (o * r2).sum()).backward()
        with torch.no_grad():
            val = net(conv.detach(), flag='val')
            val2 = net(conv.detach())
    finally:
        _lib.set_precise(0)
    assert np.array_equal(l1.cpu().numpy(), G['head_labels1']) and np.array_equal(l2.cpu().numpy(), G['head_labels2'])
    errs = {'self': rel_l2(s.detach().cpu(), G['head_self']), 'other': rel_l2(o.detach().cpu(), G['head_other']),
            'val': rel_l2(val.cpu(), G['head_val']), 'dconv': rel_l2(conv.grad.cpu(), G['head_dconv'])}
    for k, p in net.named_parameters():
        g = p.grad.cpu()
        errs[k] = rel_l2(g if g.numel() <= 65536 else g.reshape(g.shape[0], -1)[:, ::31], G[f'head_g_{k}'])
    print(f'apinet head precise={precise}', {k: f'{v:.1e}' for k, v in errs.items()})
    assert torch.equal(val, val2)
    fwd = max(errs['self'], errs['other'], errs['val'])
    bwd = max(v for k, v in errs.items() if k not in ('self', 'other', 'val'))
    assert fwd < (1e-3 if not precise else 1e-4) and bwd < (3e-3 if not precise else 1e-4)


@pytest.mark.parametrize('precise', [1, 0])
def test_loss_matches_reference(precise):
    from hawkeye_b200 import _lib
    from hawkeye_b200.losses import APINetLoss
    z = torch.cat([torch.as_tensor(G['loss_self']), torch.as_tensor(G['loss_other'])]).cuda().requires_grad_(True)
    R = z.shape[0] // 2
    l1, l2 = torch.as_tensor(G['loss_labels1']).cuda(), torch.as_tensor(G['loss_labels2']).cuda()
    crit = APINetLoss(None)
    _lib.set_precise(precise)
    try:
        loss = crit((z[:R], z[R:], l1, l2), None)
        loss.backward()
    finally:
        _lib.set_precise(0)
    want = float(G['loss_value'])
    ds, do = z.grad[:R].cpu(), z.grad[R:].cpu()
    h = int(G['loss_hinge_row'])
    e = {'loss': abs(loss.item() - want) / abs(want), 'dself': rel_l2(ds, G['loss_dself']), 'dother': rel_l2(do, G['loss_dother']),
         'hinge': max(rel_l2(ds[h], G['loss_dself'][h]), rel_l2(do[h], G['loss_dother'][h]))}
    print(f'apinet loss precise={precise}', {k: f'{v:.1e}' for k, v in e.items()})
    tol = 1e-5 if precise else 1e-3                       # default mode: dlogits are rounded to tf32 (2^-11) on store
    assert e['loss'] < 1e-5 and max(e['dself'], e['dother'], e['hinge']) < tol
    targets = torch.cat([l1, l2, l1, l2])
    assert int(crit.last_correct.item()) == int((z.detach().argmax(1) == targets).sum().item())


def _trainer(monkeypatch, graph=False, p=0.5):
    tr = make_trainer(monkeypatch, 'APINet', 'APINet.yaml', graph=graph)
    tr.model.drop.p = p
    return tr


def test_train_step_224(monkeypatch):
    tr = _trainer(monkeypatch, p=0.0)
    x = detgen.det((40, 3, 224, 224), 420).cuda()
    y = torch.arange(10).repeat_interleave(4).cuda()          # 10 classes x 4 samples
    with torch.no_grad():
        s, o, l1, l2 = tr.model(x, y)
    ref = A.apinet_loss(torch.cat([s, o]).double().cpu(), torch.cat([l1, l2, l1, l2]).cpu()).item()
    backbone = [p.detach().clone() for p in tr.model.backbone.parameters()]
    ids = {id(p) for p in tr.model.backbone.parameters()}
    head = [(p, p.detach().clone()) for p in tr.model.parameters() if id(p) not in ids]
    assert tr.optimizer.param_groups[0]['lr'] == 0.0            # epoch 0: backbone frozen through lr = 0
    losses = [float(tr.batch_training({'img': x, 'label': y}).item())]
    torch.cuda.synchronize()
    assert abs(losses[0] - ref) < 1e-4 * max(1.0, abs(ref)), (losses[0], ref)
    assert all(torch.equal(a, b.detach()) for a, b in zip(backbone, tr.model.backbone.parameters()))
    assert all(not torch.equal(b, p.detach()) for p, b in head)
    for g in tr.optimizer.param_groups:                         # after the warm-up: everything trains
        g['lr'] = 1e-4
    tr.model.drop.p = 0.5
    with no_host_sync():
        for _ in range(3):
            losses.append(tr.batch_training({'img': x, 'label': y}))
    losses[1:] = [float(v.item()) for v in losses[1:]]
    print('apinet 224 losses', losses, 'oracle', ref)
    assert all(not torch.equal(a, b.detach()) for a, b in zip(backbone, tr.model.backbone.parameters()))
    assert all(torch.isfinite(p).all() for p in tr.model.parameters())
    assert losses[-1] < losses[0]


def test_graph_replay_matches_eager(monkeypatch):
    x = detgen.det((8, 3, 224, 224), 421).cuda()
    y = torch.arange(4).repeat_interleave(2).cuda()

    def build(graph):
        tr = _trainer(monkeypatch, graph=graph, p=0.0)
        tr.optimizer.param_groups[1]['lr'] = 1e-4     # a warm-up epoch: backbone frozen (lr 0), the head trains
        return tr
    (eager, _), (replayed, _) = eager_and_graph_losses(build, [{'img': x, 'label': y}] * 6)
    print('apinet graph', eager, replayed)
    for a, b in zip(eager, replayed):
        assert abs(a - b) <= 1e-5 * abs(a), (eager, replayed)
    # p = 0.5 inside the graph: the seed is drawn on the device, so two replays draw different masks
    tr = _trainer(monkeypatch, graph=True, p=0.5)
    for g in tr.optimizer.param_groups:
        g['lr'] = 0.0
    outs = []
    for _ in range(6):
        tr.batch_training({'img': x, 'label': y})
        outs.append(tr._graph['out'][0].clone() if tr._graph is not None else None)
    assert outs[-1] is not None and outs[-2] is not None and not torch.equal(outs[-1], outs[-2])


def test_tester_evaluates_apinet_checkpoint(tmp_path, monkeypatch):
    import hawkeye_b200 as hb
    from hawkeye_b200.cfgnode import CfgNode
    from hawkeye_b200.test import Tester
    monkeypatch.setenv('HAWKEYE_ALLOW_RANDOM_INIT', '1')

    class Cfg(dict):
        __getattr__ = dict.__getitem__
    net = hb.MODEL.get('APINet')(Cfg(name='APINet', num_classes=200))
    path = str(tmp_path / 'best_model.pth')
    torch.save(detgen.state_like(net), path)
    cfg = CfgNode(dict(experiment=dict(name='t', cuda=[0]), dataset=dict(batch_size=4, num_workers=0,
                                                                         transformer=dict(resize_size=256, image_size=224)),
                       model=dict(name='APINet', num_classes=200, load=path)))
    x = detgen.det((4, 3, 224, 224), 422)
    t = Tester(cfg, dataloader=[])
    with torch.no_grad():
        pred = t.model.eval()(x.cuda()).argmax(1).cpu()
    t = Tester(cfg, dataloader=[{'img': x, 'label': pred}, {'img': x, 'label': (pred + 1) % 200}])
    assert abs(t.test() - 50.0) < 1e-6
