"""ProtoTree on the device: each hk_prototree_* kernel against the fp64 oracle (oracle/prototree_oracle.py) in both precision
modes, argmin ties, heights 1 to 10 and odd shapes, bitwise repeatability, the tree against fixtures of the unmodified
reference (tests/golden/make_golden_prototree.py), backward through eval-mode BatchNorm unit by unit and on a shallow
trunk, the full model on the reference's weights, and the 224x224 batch-64 train step (no host synchronisation, CUDA-graph
replay bit-identical to eager on the eval-mode steps)."""
import copy
import os

import pytest
import torch

import detgen
from conftest import load_golden, rel_l2
from oracle import prototree_oracle as O
from prototree_inputs import theta0, tree_inputs

pytestmark = pytest.mark.gpu
G = load_golden('reference_prototree')
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(params=[0, 1], ids=['tf32', 'precise'])
def precise(request):
    from hawkeye_b200 import _lib
    _lib.set_precise(request.param)
    yield request.param
    _lib.set_precise(0)


def _head(z, protos, theta, labels, height):
    """the library's distance, routing and NLL with their backward -> (values, gradients)"""
    from hawkeye_b200 import ops_prototree as OP
    z, protos, theta = (t.cuda().requires_grad_(True) for t in (z, protos, theta))
    mind, argmin = OP.PrototypeDistanceFn.apply(z, protos, False)
    pred, ps, pa = OP.RouteFn.apply(mind, theta, height)
    loss, correct = OP.NLLFn.apply(pred, labels.cuda())
    loss.backward()
    return (dict(mind=mind, argmin=argmin, pred=pred, ps=ps, pa=pa, loss=loss, correct=correct),
            dict(z=z.grad, protos=protos.grad, theta=theta.grad))


def _oracle(z, protos, theta, labels, height):
    z, protos, theta = (t.double().requires_grad_(True) for t in (z, protos, theta))
    mind, argmin = O.distances(z, protos)
    pred, ps, pa = O.route(mind, theta, height)
    loss = O.nll(pred, labels)
    loss.backward()
    return dict(mind=mind, argmin=argmin, pred=pred, ps=ps, pa=pa, loss=loss), dict(z=z.grad, protos=protos.grad,
                                                                                      theta=theta.grad)


# fp32 against fp64: the distances are sums of D = 256 squares (relative error ~ sqrt(D) 2^-24); every other quantity is a
# product of <= 12 routing factors or a 200-term softmax; 1e-5 leaves a margin of ~10x on all of them.  The gradients
# divide by the distance and go through the same products: 1e-4.
TOL_F, TOL_G = 1e-5, 1e-4


@pytest.mark.parametrize('height,N,HW,K', [(1, 1, 1, 3), (2, 3, 49, 7), (5, 4, 70, 200), (9, 4, 49, 200), (10, 2, 9, 13)])
def test_kernels_against_oracle(height, N, HW, K, precise):
    P, L, D = 2 ** height - 1, 2 ** height, 256
    z = torch.sigmoid(detgen.det((N, HW, D), 800 + height))
    protos = 0.5 + 0.1 * detgen.det((P, D), 801 + height)
    theta = detgen.det((L, K), 802 + height)
    labels = detgen.det_labels(N, K, 803 + height)
    got, g = _head(z, protos, theta, labels, height)
    ref, r = _oracle(z, protos, theta, labels, height)
    assert torch.equal(got['argmin'].cpu().long(), ref['argmin'])
    for k in ('mind', 'pred', 'ps', 'pa'):
        assert rel_l2(got[k].detach().cpu(), ref[k].detach()) < TOL_F, k
    assert abs(got['loss'].item() - ref['loss'].item()) < TOL_F * abs(ref['loss'].item())
    assert int(got['correct'].item()) == int((ref['pred'].argmax(1) == labels).sum())
    for k in ('z', 'protos', 'theta'):
        assert rel_l2(g[k].cpu(), r[k]) < TOL_G, k


def test_argmin_ties_take_the_first_position():
    """Equal distances at several positions: the first in row-major order wins, as max_pool2d of -d picks it."""
    from hawkeye_b200 import ops_prototree as OP
    z = torch.rand(2, 16, 256)
    z[:, 9] = z[:, 3]
    z[:, 12] = z[:, 3]
    protos = z[:, 3].clone()                                    # every position 3, 9, 12 is at distance 0 (d = 1e-7)
    mind, argmin = OP.PrototypeDistanceFn.apply(z.cuda(), protos.cuda(), False)
    assert argmin[0, 0].item() == 3 and argmin[1, 1].item() == 3


def test_many_rows_and_repeatability():
    height, N, HW, K = 9, 4096, 4, 200
    P, L = 2 ** height - 1, 2 ** height
    z = torch.sigmoid(detgen.det((N, HW, 256), 810)).cuda()
    protos = (0.5 + 0.1 * detgen.det((P, 256), 811)).cuda()
    theta = detgen.det((L, K), 812).cuda()
    labels = torch.randint(0, K, (N,)).cuda()
    runs = [_head(z, protos, theta, labels, height) for _ in range(2)]
    for a, b in zip(runs[0][1].values(), runs[1][1].values()):
        assert torch.equal(a, b)                                # fixed-order sums: the same bits on every run
    assert torch.equal(runs[0][0]['loss'], runs[1][0]['loss'])
    rows = slice(0, 64)
    ref, _ = _oracle(z[rows].cpu(), protos.cpu(), theta.cpu(), labels[rows].cpu(), height)
    assert rel_l2(runs[0][0]['pred'][rows].detach().cpu(), ref['pred'].detach()) < TOL_F


def test_leaf_update_against_reference_and_oracle():
    from hawkeye_b200 import ops_prototree as OP
    feat, protos, theta, labels = tree_inputs(G, 'tree')
    z = feat.permute(0, 2, 3, 1).reshape(4, 49, 256)
    got, _ = _head(z, protos.view(511, 256), theta, labels, 9)
    th = theta.cuda().contiguous()
    th0 = theta0(512).cuda()
    OP.leaf_update(th, th0, got['pa'], got['pred'].detach(), labels.cuda(), int(G['upd_num_batches']))
    assert rel_l2(th[::4].cpu(), G['upd_theta_rows']) < 1e-5
    ref, _ = _oracle(z, protos.view(511, 256), theta, labels, 9)
    want = O.leaf_update(theta.double(), th0.cpu().double(), ref['pa'][:, O.leaf_indices(9)].detach(), ref['pred'].detach(),
                         labels, int(G['upd_num_batches']))
    assert rel_l2(th.cpu(), want) < 1e-5


@pytest.mark.parametrize('height,K', [(1, 3), (5, 13), (10, 7)])
def test_leaf_update_other_shapes(height, K):
    """The leaf update at other heights and at K not a multiple of 4, against the oracle; and split as two data-parallel
    ranks would run it: each half of the batch sums its own update, the sums are added (the all-reduce), and the result
    matches the update of the whole batch."""
    from hawkeye_b200 import _lib, ops_prototree as OP
    N, HW, P, L = 6, 9, 2 ** height - 1, 2 ** height
    z = torch.sigmoid(detgen.det((N, HW, 256), 870 + height))
    protos = 0.5 + 0.1 * detgen.det((P, 256), 871 + height)
    theta = detgen.det((L, K), 872 + height)
    labels = detgen.det_labels(N, K, 873 + height)
    labels[1] = -100                                            # an ignored row: no update from it
    th0 = detgen.det((L, K), 874 + height).abs().cuda()
    got, _ = _head(z, protos, theta, labels, height)
    pa, pred, y = got['pa'], got['pred'].detach(), labels.cuda()
    whole = theta.cuda().contiguous()
    OP.leaf_update(whole, th0, pa, pred, y, 7)
    ref, _ = _oracle(z, protos, theta, labels.clamp_min(0), height)
    keep = (labels >= 0).double()[:, None]
    want = O.leaf_update(theta.double(), th0.cpu().double(), ref['pa'][:, O.leaf_indices(height)].detach() * keep,
                         ref['pred'].detach(), labels.clamp_min(0), 7)
    assert rel_l2(whole.cpu(), want) < 1e-5
    half = slice(N // 2, N)
    other = torch.empty_like(whole)
    _lib.call('hk_prototree_leaf_update_sum', theta.cuda(), pa[half].contiguous(), pred[half].contiguous(),
              y[half].contiguous(), other, N - N // 2, height, K, _lib.stream_ptr())
    split = theta.cuda().contiguous()
    lo = slice(0, N // 2)
    OP.leaf_update(split, th0, pa[lo].contiguous(), pred[lo].contiguous(), y[lo].contiguous(), 7,
                   reduce=lambda u: u.add_(other))
    assert rel_l2(split.cpu(), want) < 1e-5


def test_nll_ignores_rows_as_torch_does(precise):
    """Rows labelled -100 (F.nll_loss's ignore_index) leave the mean: loss and gradient against F.nll_loss in fp64."""
    import torch.nn.functional as F
    from hawkeye_b200 import ops_prototree as OP
    pred = torch.softmax(detgen.det((9, 13), 880), 1)
    labels = detgen.det_labels(9, 13, 881)
    labels[[2, 5]] = -100
    p = pred.cuda().requires_grad_(True)
    loss, correct = OP.NLLFn.apply(p, labels.cuda())
    loss.backward()
    pd = pred.double().requires_grad_(True)
    ref = F.nll_loss(torch.log(pd), labels)
    ref.backward()
    assert abs(loss.item() - ref.item()) < 1e-6 * abs(ref.item())
    assert rel_l2(p.grad.cpu(), pd.grad) < 1e-6
    keep = labels >= 0
    assert int(correct.item()) == int((pred.argmax(1)[keep] == labels[keep]).sum())


@pytest.mark.parametrize('tag', ['tree', 'dfo_off'])
def test_tree_against_reference(tag, monkeypatch):
    """The package's ProtoTree (tree only) on the reference's fixture, through ProtoTree.forward with NCHW features."""
    import hawkeye_b200 as hb
    monkeypatch.setenv('HAWKEYE_ALLOW_RANDOM_INIT', '1')

    class Cfg(dict):
        __getattr__ = dict.__getitem__
    feat, protos, theta, labels = tree_inputs(G, tag)
    net = hb.MODEL.get('ProtoTreeNet')(Cfg(name='ProtoTreeNet', num_classes=200, height=9, W1=1, H1=1, num_features=256,
                                           disable_derivative_free_leaf_optim=tag == 'dfo_off'))
    tree = net.tree.cuda()
    with torch.no_grad():
        tree.prototype_layer.prototype_vectors.copy_(protos)
        tree.leaf_params.copy_(theta)
    f = feat.cuda().requires_grad_(True)
    pred, info = tree(f, f)
    from hawkeye_b200.losses import ProtoTreeLoss
    loss = ProtoTreeLoss()((pred, info), labels.cuda())
    loss.backward()
    assert rel_l2(pred.detach().cpu(), G[f'{tag}_pred']) < 1e-5
    assert abs(loss.item() - float(G[f'{tag}_loss'])) < 1e-5
    pa = torch.cat([info['pa_tensor'][i] for i in range(1023)], 1)
    assert rel_l2(pa.cpu(), G[f'{tag}_pa']) < 1e-5
    assert rel_l2(torch.cat([info['ps'][i] for i in sorted(info['ps'])], 1).cpu(), G[f'{tag}_ps']) < 1e-5
    # the reference's fp32 |x|^2 + |p|^2 - 2 x.p gradients carry its cancellation at the minimum (test_prototree_cpu)
    assert rel_l2(f.grad[:, ::4].cpu(), G[f'{tag}_dfeat_slice']) < 1e-3
    assert rel_l2(tree.prototype_layer.prototype_vectors.grad[:, ::8].cpu(), G[f'{tag}_dprotos_slice']) < 1e-3
    if tag == 'dfo_off':
        assert rel_l2(tree.leaf_params.grad[::4].cpu(), G['dfo_off_dtheta_rows']) < 1e-5


# ---- backward through eval-mode BatchNorm ------------------------------------------------------------------------------
@pytest.mark.parametrize('relu,res', [(0, 0), (1, 0), (0, 1), (1, 1)])
def test_bn_backward_frozen_statistics(relu, res, precise):
    """hk_bn_bwd_frozen against fp64 autograd of F.batch_norm(training=False), on the ReLU mask of the library's forward;
    the running statistics are not touched."""
    import torch.nn.functional as F
    from hawkeye_b200 import _lib
    from hawkeye_b200.ops import _ws
    P, C = 3 * 49, 64
    x = detgen.det((P, C), 820, 2.0).cuda() + 0.5
    gamma, beta = (1 + 0.2 * detgen.det((C,), 821)).cuda(), (0.1 * detgen.det((C,), 822)).cuda()
    rm, rv = (0.3 * detgen.det((C,), 823)).cuda(), (1 + detgen.det((C,), 824).abs()).cuda()
    rm0, rv0 = rm.clone(), rv.clone()
    r = detgen.det((P, C), 825).cuda() if res else None
    invstd = torch.rsqrt(rv + 1e-5)
    y = torch.empty_like(x)
    s = _lib.stream_ptr()
    _lib.call('hk_bn_apply', x, rm, invstd, gamma, beta, r, y, P, C, relu, s)
    dy = detgen.det((P, C), 826).cuda()
    dx, dres = torch.empty_like(x), (torch.empty_like(x) if res else None)
    dg, db = torch.empty(C, device='cuda'), torch.empty(C, device='cuda')
    ws = _ws(_lib.query('hk_bn_workspace_bytes', P, C), x.device)
    mask_beta = beta if (relu and not res) else None
    _lib.call('hk_bn_bwd_frozen', x, y, dy, gamma, mask_beta, rm, invstd, dx, dres, dg, db, P, C, relu, ws, ws.numel(), s)
    xd, gd, bd = (t.cpu().double().requires_grad_(True) for t in (x, gamma, beta))
    out = F.batch_norm(xd, rm.cpu().double(), rv.cpu().double(), gd, bd, training=False, eps=1e-5)
    if res:
        out = out + r.cpu().double()
    mask = (y.cpu() > 0).double() if relu else 1.0
    (out * mask * dy.cpu().double()).sum().backward()
    tol = 1e-5 if precise else 2 ** -10                   # default mode: dx is rounded to tf32 (operand of the next MMA)
    assert rel_l2(dx.cpu(), xd.grad) < tol and rel_l2(dg.cpu(), gd.grad) < 1e-5 and rel_l2(db.cpu(), bd.grad) < 1e-5
    if res:
        assert torch.equal(dres.cpu(), (dy.cpu() * (y.cpu() > 0)) if relu else dy.cpu())
    assert torch.equal(rm, rm0) and torch.equal(rv, rv0)


def test_shallow_trunk_eval_mode_backward(precise):
    """ResNetTrunkFn with training=False and gradients: every parameter gradient against fp64 autograd of the same trunk in
    eval mode (the trunk gives the image no gradient), and the running statistics untouched."""
    import torch.nn as nn
    from hawkeye_b200.backbone.resnet import ResNetTrunk
    torch.manual_seed(830)
    trunk = ResNetTrunk((1, 1, 1, 1))
    with torch.no_grad():
        for m in trunk.modules():
            if isinstance(m, nn.BatchNorm2d):
                m.running_mean.normal_(0, 0.1)
                m.running_var.uniform_(0.5, 2.0)
                m.weight.uniform_(0.5, 1.5)
                m.bias.normal_(0, 0.1)
    ref = copy.deepcopy(trunk).double().eval()
    trunk = trunk.cuda().eval()
    stats0 = {k: v.clone() for k, v in trunk.state_dict().items() if 'running' in k}
    x = detgen.det((2, 3, 96, 96), 831).cuda()
    out = trunk(x)
    g = detgen.det(tuple(out.shape), 832).cuda()
    (out * g).sum().backward()
    # the fp64 reference: the torch modules of the same trunk (ResNetTrunk's children are plain torch modules)
    h = x.cpu().double()
    for i, m in enumerate(ref):
        if i < 4:
            h = m(h)
        else:
            for blk in m:
                idt = h if blk.downsample is None else blk.downsample(h)
                o = blk.relu(blk.bn1(blk.conv1(h)))
                o = blk.relu(blk.bn2(blk.conv2(o)))
                h = blk.relu(blk.bn3(blk.conv3(o)) + idt)
    (h * g.cpu().double()).sum().backward()
    feat = rel_l2(out.detach().cpu(), h.detach())
    errs = {n: rel_l2(p.grad.cpu(), q.grad) for (n, p), (_, q) in zip(trunk.named_parameters(), ref.named_parameters())}
    worst = max(errs, key=errs.get)
    print(f'eval-mode trunk precise={precise}: features {feat:.2e}, worst gradient {worst} {errs[worst]:.2e}')
    # The fp64 reference runs its own forward, not the library's tape, so a ReLU decision that rounding flips near zero
    # moves a gradient, and the random running statistics leave the activations unnormalised: these bounds are looser than
    # the tape-replay bounds of test_gpu_resnet_backward.py (measured on an H100 80GB HBM3 at 400 W: features 1.7e-3 / 1.1e-5,
    # worst gradient 6.3e-2 (stem) / 6.7e-4 in the default / 3xTF32 mode).  test_bn_backward_frozen_statistics is the tight
    # check of the kernel itself.
    assert feat < (1e-4 if precise else 1e-2) and errs[worst] < (3e-3 if precise else 0.15) and len(errs) == 51
    for k, v in trunk.state_dict().items():
        if 'running' in k:
            assert torch.equal(v, stats0[k]), k


# ---- the full model --------------------------------------------------------------------------------------------------
def _model_cfg(**kw):
    class Cfg(dict):
        __getattr__ = dict.__getitem__
    base = dict(name='ProtoTreeNet', num_classes=200, height=9, W1=1, H1=1, num_features=256)
    base.update(kw)
    return Cfg(base)


def test_full_model_matches_reference(monkeypatch):
    """The reference's end-to-end fixture (detgen.state_like weights, prototypes in the package's order, train mode, two
    64x64 images, nll_loss backward).  Tight bounds on the neck and tree given the trunk's own output; sanity bounds end to
    end, where the random-weight train-mode ResNet-50 amplifies TF32 rounding (as for DCL)."""
    import hawkeye_b200 as hb
    from hawkeye_b200.losses import ProtoTreeLoss
    monkeypatch.setenv('HAWKEYE_ALLOW_RANDOM_INIT', '1')
    net = hb.MODEL.get('ProtoTreeNet')(_model_cfg())
    sd = detgen.state_like(net)
    perm = torch.as_tensor(G['model_perm'])
    sd['tree.prototype_layer.prototype_vectors'] = sd['tree.prototype_layer.prototype_vectors'][perm]
    for j in range(512):
        key = 'tree._root.' + '.'.join('lr'[(j >> (8 - b)) & 1] for b in range(9)) + '._dist_params'
        sd[key] = detgen.det((200,), 700 + j)
    net.load_state_dict(sd)
    net = net.cuda().train()
    feats = []
    net.backbone.register_forward_hook(lambda m, i, o: feats.append(o.detach()))
    pred, info = net(torch.as_tensor(G['e2e_x']).cuda())
    loss = ProtoTreeLoss()((pred, info), torch.as_tensor(G['e2e_labels']).cuda())
    loss.backward()
    # neck + tree + loss in fp64 on the trunk's own output
    feat = feats[0].cpu().double()
    w = net.neck_conv[0].weight.detach().cpu().double().requires_grad_(True)
    pr = net.tree.prototype_layer.prototype_vectors.detach().cpu().double().view(511, 256).requires_grad_(True)
    z = torch.sigmoid(torch.einsum('nchw,dc->nhwd', feat, w.view(256, -1))).reshape(feat.shape[0], -1, 256)
    mind, _ = O.distances(z, pr)
    rp, _, _ = O.route(mind, net.tree.leaf_params.detach().cpu().double(), 9)
    O.nll(rp, G['e2e_labels']).backward()
    head = dict(pred=rel_l2(pred.detach().cpu(), rp.detach()), g_neck=rel_l2(net.neck_conv[0].weight.grad.cpu(), w.grad),
                g_protos=rel_l2(net.tree.prototype_layer.prototype_vectors.grad.cpu().view(511, 256), pr.grad))
    e2e = dict(feat=rel_l2(feats[0][:, ::16].cpu(), G['e2e_feat_slice']), pred=rel_l2(pred.detach().cpu(), G['e2e_pred']),
               g_neck=rel_l2(net.neck_conv[0].weight.grad[:, ::16].cpu(), G['e2e_g_neck_slice']),
               g_protos=rel_l2(net.tree.prototype_layer.prototype_vectors.grad.cpu(), G['e2e_g_protos']),
               g_l4_bn3_w=rel_l2(net.backbone[7][2].bn3.weight.grad.cpu(), G['e2e_g_layer4_bn3_w']))
    print(f'prototree e2e: loss {loss.item():.6f} vs {float(G["e2e_loss"]):.6f}', {k: f'{v:.1e}' for k, v in head.items()},
          {k: f'{v:.1e}' for k, v in e2e.items()})
    # the neck GEMM runs in TF32 (the pre-activation is ~2^-11 off), the rest in fp32
    assert head['pred'] < 1e-3 and head['g_neck'] < 3e-3 and head['g_protos'] < 3e-3
    assert e2e['feat'] < 0.2 and e2e['pred'] < 0.2 and abs(loss.item() - float(G['e2e_loss'])) < 2e-2 * float(G['e2e_loss'])
    assert all(torch.isfinite(p.grad).all() for p in net.parameters() if p.grad is not None)


def _trainer(monkeypatch, graph=False, **model):
    from hawkeye_b200 import examples
    from hawkeye_b200.config import load_config
    monkeypatch.setenv('HAWKEYE_ALLOW_RANDOM_INIT', '1')
    monkeypatch.setenv('HK_CUDA_GRAPH', '1' if graph else '0')
    cfg = load_config(os.path.join(REPO, 'configs', 'ProtoTreeNet.yaml'))
    cfg.model.backbone['pretrain'] = ''                      # no iNat checkpoint here: the trunk keeps its random init
    for k, v in model.items():
        cfg.model[k] = v
    tr = examples.ProtoTreeTrainer(cfg, dataloaders={})
    tr.num_batches = 10
    tr.model.train()
    return tr


def _batch(n, seed):
    return {'img': detgen.det((n, 3, 224, 224), seed).pin_memory(), 'label': detgen.det_labels(n, 200, seed + 1).pin_memory()}


def test_train_step_224_no_sync(monkeypatch):
    tr = _trainer(monkeypatch)
    data = _batch(64, 840)
    tr.on_start_epoch(None)
    theta0 = tr.model.tree.leaf_params.detach().clone()
    losses = [float(tr.batch_training(data).item())]
    assert not tr.model.training                             # eval() after the first leaf update, as the reference
    assert not torch.equal(tr.model.tree.leaf_params, theta0)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')                  # no host synchronisation inside the step
    try:
        for _ in range(4):
            losses.append(tr.batch_training(data))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    losses[1:] = [float(v.item()) for v in losses[1:]]
    print('prototree 224 losses', losses)
    assert all(torch.isfinite(torch.tensor(losses)))          # a random-init trunk: the loss need not fall in 5 steps
    assert all(torch.isfinite(p).all() for p in tr.model.parameters())
    for m in tr.average_meters.values():
        assert m.avg >= 0 and m.count == 5 * 64


def test_graph_replay_matches_eager_on_eval_steps(monkeypatch):
    """224x224, batch 64.  First batch eager in train mode, then eval-mode steps; with the graph they replay.  The trunk, neck and prototypes
    are held at lr 0 (they still run forward and backward): the leaves, updated by the deterministic leaf-update kernel, and
    the losses must then be the same bits with and without the graph."""
    data = _batch(64, 850)
    out, state0 = {}, None
    for graph in (False, True):
        torch.manual_seed(0)
        tr = _trainer(monkeypatch, graph=graph)
        if state0 is None:
            state0 = copy.deepcopy(tr.model.state_dict())
        else:
            tr.model.load_state_dict(state0)
        for g in tr.optimizer.param_groups:
            g['lr'] = 0.0
        tr.on_start_epoch(None)
        losses = [float(tr.batch_training(data).item()) for _ in range(7)]    # a replay overwrites the graph's loss tensor
        out[graph] = (losses, tr.model.tree.leaf_params.detach().clone())
        if graph:
            assert tr._graph is not None
        del tr
    print('prototree graph', out[False][0], out[True][0])
    assert out[False][0] == out[True][0]
    assert torch.equal(out[False][1], out[True][1])


def test_errors():
    from hawkeye_b200 import _lib, ops_prototree as OP
    z = torch.zeros(2, 4, 256, device='cuda')
    with pytest.raises(_lib.HawkeyeLibError, match='prototypes'):
        OP.PrototypeDistanceFn.apply(z, torch.zeros(7, 128, device='cuda'), False)
    with pytest.raises(_lib.HawkeyeLibError, match='height=13'):
        OP.RouteFn.apply(torch.zeros(2, 8191, device='cuda'), torch.zeros(8192, 4, device='cuda'), 13)
    with pytest.raises(_lib.HawkeyeLibError, match='needs 7 distances'):
        OP.RouteFn.apply(torch.zeros(2, 6, device='cuda'), torch.zeros(8, 4, device='cuda'), 3)
    with pytest.raises(_lib.HawkeyeLibError, match='height=13'):
        _lib.call('hk_prototree_route_fwd', z, z, z, z, z, z, 2, 13, 4, _lib.stream_ptr())


def test_tester_reads_pred_of_pred_info(tmp_path, monkeypatch):
    """Tester on ProtoTreeNet's (pred, info) output: the accuracy is that of pred."""
    from hawkeye_b200.test import Tester
    from hawkeye_b200.config import load_config
    import hawkeye_b200 as hb
    monkeypatch.setenv('HAWKEYE_ALLOW_RANDOM_INIT', '1')
    cfg = load_config(os.path.join(REPO, 'configs', 'ProtoTreeNet.yaml'))
    cfg.model.backbone['pretrain'] = ''
    net = hb.MODEL.get('ProtoTreeNet')(cfg.model)
    path = tmp_path / 'ptn.pth'
    torch.save(net.state_dict(), path)
    cfg.model['load'] = str(path)
    x = detgen.det((4, 3, 224, 224), 860)
    with torch.no_grad():
        pred, _ = net.cuda().eval()(x.cuda())
    y = pred.argmax(1).cpu()
    y[0] = (y[0] + 1) % 200
    t = Tester(cfg, dataloader=[{'img': x, 'label': y}])
    assert t.test() == 75.0
