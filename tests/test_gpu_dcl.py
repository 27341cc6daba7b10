"""DCL on the device: the head kernels against the fp64 oracle (and their run-to-run determinism), the loss kernel against
fixtures of the unmodified reference (tests/golden/make_golden_dcl.py) and fp64 autograd, the loss on row slices of the
stacked classifier output, the full model against the reference's end-to-end fixture, the 448x448 train step from DCLTrainer (no host synchronisation), CUDA-graph replay,
and the host-side errors."""
import pytest
import torch

import detgen
from conftest import load_golden, rel_l2
from oracle import dcl_oracle as D
from kernel_check import precise  # noqa: F401  (a fixture)
from step_check import eager_and_graph_losses, make_trainer, no_host_sync

pytestmark = pytest.mark.gpu
G = load_golden('reference_dcl')


@pytest.mark.parametrize('N', [2, 16])
@pytest.mark.parametrize('S', [14, 7])
def test_head_against_oracle(N, S, precise):
    from hawkeye_b200 import ops_dcl
    x = detgen.det((N, 2048, S, S), 600 + N + S, positive=True).cuda().requires_grad_(True)
    w = (detgen.det((1, 2048, 1, 1), 601) * 0.02).cuda().requires_grad_(True)
    b = torch.tensor([0.1], device='cuda', requires_grad=True)
    pooled, mask = ops_dcl.DCLHeadFn.apply(x, w, b)
    xd, wd, bd = (t.detach().cpu().double().requires_grad_(True) for t in (x, w, b))
    rp, rm = D.head(xd, wd, bd)
    assert mask.shape == (N, (S // 2) ** 2)
    assert rel_l2(mask.detach().cpu(), rp.new_tensor(rm.detach())) < 1e-5
    tol = 1e-5 if precise else 2 ** -10                    # default mode: pooled is rounded to tf32 on store
    assert (pooled.detach().cpu().double() - rp.detach()).abs().max() <= tol * rp.detach().abs().max()
    gp, gm = detgen.det((N, 2048), 602).cuda(), detgen.det(mask.shape, 603).cuda()
    grads = []
    for _ in range(2):
        x.grad = w.grad = b.grad = None
        pooled, mask = ops_dcl.DCLHeadFn.apply(x, w, b)
        torch.autograd.backward([pooled, mask], [gp, gm])
        grads.append((x.grad.clone(), w.grad.clone(), b.grad.clone()))
    torch.autograd.backward([rp, rm], [gp.cpu().double(), gm.cpu().double()])
    for got, ref, name in zip(grads[0], (xd.grad, wd.grad, bd.grad), ('dx', 'dw', 'db')):
        assert rel_l2(got.cpu(), ref) < 1e-5, name
    assert torch.equal(grads[0][1], grads[1][1]) and torch.equal(grads[0][2], grads[1][2])   # fixed-order sums


@pytest.mark.parametrize('tag', ['cls2', 'cls2xmul'])
def test_loss_against_reference(tag, precise):
    from hawkeye_b200.losses import DCLLoss
    alpha, beta, gamma = G['loss_weights'].tolist()

    class Cfg(dict):
        __getattr__ = dict.__getitem__
    crit = DCLLoss(Cfg(alpha=alpha, beta=beta, gamma=gamma))
    t = {k: torch.as_tensor(G[f'loss_{tag}_{k}']).cuda().requires_grad_(True) for k in ('logits', 'swap', 'mask')}
    labels = torch.as_tensor(G[f'loss_{tag}_labels']).cuda()
    labels_swap = torch.as_tensor(G[f'loss_{tag}_labels_swap']).cuda()
    law = torch.as_tensor(G[f'loss_{tag}_law']).cuda()
    loss = crit([t['logits'], t['swap'], t['mask']], labels, labels_swap, law)
    loss.backward()
    ref = float(G[f'loss_{tag}_value'])
    assert abs(loss.item() - ref) < 1e-5 * abs(ref)
    d = {k: torch.as_tensor(G[f'loss_{tag}_{k}']).double().requires_grad_(True) for k in ('logits', 'swap', 'mask')}
    D.loss(d['logits'], d['swap'], d['mask'], labels.cpu(), labels_swap.cpu(), law.cpu(), alpha, beta, gamma).backward()
    tol = 1e-5 if precise else 1e-3                       # default mode: dlogits are rounded to tf32 (2^-11) on store
    for k in ('logits', 'swap'):
        assert rel_l2(t[k].grad.cpu(), d[k].grad) < tol, k
        assert rel_l2(t[k].grad.cpu(), G[f'loss_{tag}_d{k}']) < tol, k
    assert rel_l2(t['mask'].grad.cpu(), d['mask'].grad) < 1e-6 and (t['mask'].grad[0, :5] == 0).all()
    host = D.top1(G[f'loss_{tag}_logits'], G[f'loss_{tag}_swap'], labels.cpu(), tag == 'cls2xmul')
    assert int(crit.last_correct.item()) == host


def test_loss_many_rows():
    from hawkeye_b200 import ops_dcl
    R, K, Q = 4100, 200, 49
    z = detgen.det((R, 204), 610, 2.0).cuda()
    y = torch.randint(0, K, (R,), device='cuda')
    ys = torch.arange(R, device='cuda') % 2
    m, law = torch.tanh(detgen.det((R, Q), 611)).cuda(), (detgen.det((R, Q), 612) * 0.3).cuda()
    zd = z[:, :K + 2].cpu().double().requires_grad_(True)
    md = m.cpu().double().requires_grad_(True)
    loss, correct = ops_dcl.DCLLossFn.apply(z.requires_grad_(True), K, 2, y, ys, m.requires_grad_(True), law, 1.0, 1.0, 1.0,
                                            False)
    loss.backward()
    ref = D.loss(zd[:, :K], zd[:, K:], md, y.cpu(), ys.cpu(), law.cpu())
    ref.backward()
    assert abs(loss.item() - ref.item()) < 1e-5 * ref.item()
    assert rel_l2(z.grad[:, :K + 2].cpu(), zd.grad) < 1e-3 and (z.grad[:, K + 2:] == 0).all()
    assert rel_l2(m.grad.cpu(), md.grad) < 1e-6
    assert int(correct.item()) == D.top1(z[:, :K].detach().cpu(), None, y.cpu(), False)


def _trainer(monkeypatch, graph=False, **model):
    return make_trainer(monkeypatch, 'DCL', 'DCL.yaml', graph=graph, **model)


def _batch(n, seed, K=200, cls_2xmul=False):
    x = detgen.det((2 * n, 3, 448, 448), seed)
    y = detgen.det_labels(n, K, seed + 1).repeat_interleave(2)
    if cls_2xmul:
        ys = torch.stack([y[::2], y[::2] + K], 1).reshape(-1)
    else:
        ys = torch.tensor([1, 0] * n)
    law1 = [(i - 24) / 49 for i in range(49)]
    law = torch.tensor([law1, law1[::-1]] * n).float()
    return x, y, ys, law


def test_full_model_matches_reference(monkeypatch):
    """The package's DCL on the reference's end-to-end fixture (detgen.state_like weights, train mode, 4 rows of 128x128,
    DCLLoss, backward).  Tight bounds on the head and classifiers given the trunk's own output; sanity bounds end to end,
    where the random-weight train-mode ResNet-50 amplifies TF32 rounding (the bounds of test_mpn_model_matches_reference;
    see the README)."""
    from hawkeye_b200.losses import DCLLoss

    class Cfg(dict):
        __getattr__ = dict.__getitem__
    monkeypatch.setenv('HAWKEYE_ALLOW_RANDOM_INIT', '1')
    import hawkeye_b200 as hb
    net = hb.MODEL.get('DCL')(Cfg(name='DCL', num_classes=200, cls_2=True, cls_2xmul=False))
    net.load_state_dict(detgen.state_like(net))
    net = net.cuda().train()
    feats = []
    net.backbone.register_forward_hook(lambda m, i, o: feats.append(o.detach()))
    x = detgen.det((4, 3, 128, 128), 560).cuda()
    logits, swap, mask = net(x)
    assert logits.shape == (4, 200) and swap.shape == (4, 2) and mask.shape == (4, 4)
    loss = DCLLoss(Cfg(alpha=1.0, beta=1.0, gamma=1.0))([logits, swap, mask], torch.as_tensor(G['e2e_labels']).cuda(),
                                                         torch.as_tensor(G['e2e_labels_swap']).cuda(),
                                                         torch.as_tensor(G['e2e_law']).cuda())
    loss.backward()
    # the head, the classifiers and the loss in fp64 on the trunk's own output, with gradients of the head's parameters
    feat = feats[0].cpu()
    ref = {k: p.detach().cpu().double().requires_grad_(True) for k, p in
           (('w', net.Convmask.weight), ('b', net.Convmask.bias), ('wc', net.classifier.weight),
            ('ws', net.classifier_swap.weight))}
    pooled, rm = D.head(feat, ref['w'], ref['b'])
    rl, rs = D.classifiers(pooled, ref['wc'], ref['ws'])
    D.loss(rl, rs, rm, G['e2e_labels'], G['e2e_labels_swap'], G['e2e_law']).backward()
    head = dict(mask=rel_l2(mask.detach().cpu(), rm.detach()), logits=rel_l2(logits.detach().cpu(), rl.detach()),
                swap=rel_l2(swap.detach().cpu(), rs.detach()),
                g_convmask_w=rel_l2(net.Convmask.weight.grad.cpu(), ref['w'].grad),
                g_convmask_b=rel_l2(net.Convmask.bias.grad.cpu(), ref['b'].grad),
                g_classifier=rel_l2(net.classifier.weight.grad.cpu(), ref['wc'].grad),
                g_classifier_swap=rel_l2(net.classifier_swap.weight.grad.cpu(), ref['ws'].grad))
    e2e = dict(feat=rel_l2(feat[:, ::16], G['e2e_feat_slice']), logits=rel_l2(logits.detach().cpu(), G['e2e_logits']),
               swap=rel_l2(swap.detach().cpu(), G['e2e_swap']), mask=rel_l2(mask.detach().cpu(), G['e2e_mask']),
               g_classifier_swap=rel_l2(net.classifier_swap.weight.grad.cpu(), G['e2e_g_classifier_swap']),
               g_convmask_w=rel_l2(net.Convmask.weight.grad.cpu(), G['e2e_g_convmask_w']),
               g_l4_bn3_w=rel_l2(net.backbone[7][2].bn3.weight.grad.cpu(), G['e2e_g_layer4_bn3_w']))
    flips = int(((mask.detach().cpu() > torch.as_tensor(G['e2e_law'])) !=
                 (torch.as_tensor(G['e2e_mask']) > torch.as_tensor(G['e2e_law']))).sum())
    print(f'dcl e2e: loss {loss.item():.6f} vs {float(G["e2e_loss"]):.6f}, L1 sign flips {flips}',
          {k: f'{v:.1e}' for k, v in head.items()}, {k: f'{v:.1e}' for k, v in e2e.items()})
    assert head['mask'] < 1e-5 and head['logits'] < 3e-3 and head['swap'] < 3e-3
    assert head['g_convmask_w'] < 1e-4 and head['g_convmask_b'] < 1e-4
    assert head['g_classifier'] < 3e-3 and head['g_classifier_swap'] < 3e-3
    # End to end: sanity bounds on what varies continuously with the trunk's drift.  The Convmask and trunk gradients
    # carry sign(mask - law), a step that the drift can flip where the mask is near the law (the 16 entries here come within
    # 0.04 of it), so those two are printed, not bounded; the bound above checks them on the trunk's own output.
    assert e2e['feat'] < 0.2 and e2e['logits'] < 0.2 and e2e['swap'] < 0.2 and e2e['mask'] < 0.2
    assert abs(loss.item() - float(G['e2e_loss'])) < 2e-2 * abs(float(G['e2e_loss']))
    assert e2e['g_classifier_swap'] < 0.2
    assert all(torch.isfinite(p.grad).all() for p in net.parameters())


@pytest.mark.parametrize('rows', ['sources', 'first_half'])
def test_loss_on_row_slices_of_the_stacked_output(rows):
    """DCLLoss on a row slice of DCL's outputs (the source images only, or the first half of the batch) takes exactly those
    rows: loss and gradient against the fp64 oracle, and no gradient on the rows left out."""
    from hawkeye_b200 import ops_dcl
    from hawkeye_b200.losses import DCLLoss

    class Cfg(dict):
        __getattr__ = dict.__getitem__
    R, K = 8, 200
    pooled = detgen.det((R, 2048), 660, positive=True).cuda().requires_grad_(True)
    w, w2 = (detgen.det((K, 2048), 661) * 0.02).cuda(), (detgen.det((2, 2048), 662) * 0.02).cuda()
    stacked = ops_dcl.StackedClassifierFn.apply(pooled, w, w2)
    mask = torch.tanh(detgen.det((R, 49), 663)).cuda().requires_grad_(True)
    sel = slice(None, None, 2) if rows == 'sources' else slice(0, R // 2)
    out = [stacked[:, :K][sel], stacked[:, K:K + 2][sel], mask[sel]]
    y = detgen.det_labels(R // 2, K, 664).cuda()
    ys = torch.tensor([1, 0] * (R // 4), device='cuda')
    law = (detgen.det((R // 2, 49), 665) * 0.3).cuda()
    loss = DCLLoss(Cfg(alpha=1.0, beta=1.0, gamma=1.0))(out, y, ys, law)
    loss.backward()
    # the oracle loss on the same rows of the kernel's own logits (the GEMM's TF32 rounding is not what is tested here);
    # d pooled = d logits . [W; W2] in fp64
    zd = stacked.detach()[:, :K + 2].cpu().double().requires_grad_(True)
    md = mask.detach().cpu().double().requires_grad_(True)
    ref = D.loss(zd[sel, :K], zd[sel, K:], md[sel], y.cpu(), ys.cpu(), law.cpu())
    ref.backward()
    dpooled = zd.grad[:, :K] @ w.cpu().double() + zd.grad[:, K:] @ w2.cpu().double()
    assert abs(loss.item() - ref.item()) < 1e-5 * ref.item()
    assert rel_l2(pooled.grad.cpu(), dpooled) < 3e-3 and rel_l2(mask.grad.cpu(), md.grad) < 1e-6
    left_out = torch.ones(R, dtype=torch.bool)
    left_out[sel] = False
    assert (pooled.grad[left_out.cuda()] == 0).all() and (mask.grad[left_out.cuda()] == 0).all()


def test_train_step_448(monkeypatch):
    tr = _trainer(monkeypatch)
    x, y, ys, law = _batch(4, 630)
    data = (x.pin_memory(), y.pin_memory(), ys.pin_memory(), law.pin_memory(), ['n'] * 4)
    with torch.no_grad():
        logits, swap, mask = tr.model(x.cuda())
    ref = D.loss(logits.cpu().double(), swap.cpu().double(), mask.cpu().double(), y, ys, law).item()
    losses = [float(tr.batch_training(data).item())]
    torch.cuda.synchronize()
    assert abs(losses[0] - ref) < 1e-4 * max(1.0, abs(ref)), (losses[0], ref)
    with no_host_sync():
        for _ in range(5):
            losses.append(tr.batch_training(data))
    losses[1:] = [float(v.item()) for v in losses[1:]]
    print('dcl 448 losses', losses, 'oracle', ref)
    assert all(torch.isfinite(p).all() for p in tr.model.parameters())
    assert losses[-1] < losses[0]
    for m in tr.average_meters.values():                        # avg drains the asynchronous read-backs
        assert m.avg >= 0 and m.count == 6 * 8


@pytest.mark.parametrize('cls_2xmul', [False, True])
def test_graph_replay_matches_eager(monkeypatch, cls_2xmul):
    """The trunk is held at lr 0 (it still runs forward and backward): its weight update is not bit-identical from run to
    run, eager against eager, so training it would measure that rather than the replay.  Every DCL kernel of the step is
    bit-reproducible, so replay and eager agree to 1e-5."""
    x, y, ys, law = _batch(2, 640, cls_2xmul=cls_2xmul)
    data = (x, y, ys, law, ['n'] * 2)
    (eager, _), (replayed, _) = eager_and_graph_losses(
        lambda graph: _trainer(monkeypatch, graph=graph, cls_2=not cls_2xmul, cls_2xmul=cls_2xmul), [data] * 6,
        frozen_groups=(0,))
    print('dcl graph', cls_2xmul, eager, replayed)
    for a, b in zip(eager, replayed):
        assert abs(a - b) <= 1e-5 * abs(a), (eager, replayed)


def test_errors(monkeypatch):
    from hawkeye_b200 import _lib
    tr = _trainer(monkeypatch)
    x = detgen.det((2, 3, 224, 224), 650).cuda()
    out = tr.model(x)
    assert out[2].shape == (2, 9)                                # AvgPool2d(2) drops the last row / column of the 7x7 map
    law = torch.zeros(2, 49, device='cuda')
    with pytest.raises(_lib.HawkeyeLibError, match=r'448x448.*swap_num \[7, 7\]'):
        tr.criterion(out, torch.zeros(2, dtype=torch.int64, device='cuda'), torch.tensor([1, 0], device='cuda'), law)
    with pytest.raises(_lib.HawkeyeLibError, match='cls_2'):
        _trainer(monkeypatch, cls_2=False, cls_2xmul=False)
    from hawkeye_b200 import ops_dcl
    feat = torch.zeros(2, 2048, 7, 7, device='cuda')
    with pytest.raises(_lib.HawkeyeLibError, match='got 1024'):
        ops_dcl.DCLHeadFn.apply(feat, torch.zeros(1024, device='cuda'), torch.zeros(1, device='cuda'))
    with pytest.raises(_lib.HawkeyeLibError, match='got 2\\)'):
        ops_dcl.DCLHeadFn.apply(feat, torch.zeros(2048, device='cuda'), torch.zeros(2, device='cuda'))
