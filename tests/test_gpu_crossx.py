"""CrossX on the device: the hk_crossx_* kernels against the fp64 oracle (oracle/crossx_oracle.py) in both precision
modes, the loss against fixtures of the unmodified reference (tests/golden/make_golden_crossx.py), a two-rank split of the
regularisers, the 1024 -> 1024 3x3 convolution of the fusion head against fp64, the model's train- and eval-mode step
against the reference's fp64 run, and the CrossX trainer: no host synchronisation, CUDA-graph replay, and save_model read
back by the Tester."""
import numpy as np
import pytest
import torch

import crossx_inputs as I
import detgen
from conftest import load_golden, rel_l2
from oracle import crossx_oracle as O
from kernel_check import precise  # noqa: F401  (a fixture)
from step_check import make_trainer, no_host_sync, random_init, replay_against_eager  # noqa: F401

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures('random_init')]
G = load_golden('reference_crossx')

# fp32 elementwise kernels: a few ulps; the logit gradients are rounded to tf32 in the default mode
TOL = 1e-5
DX_TOL = {0: 5e-4, 1: 1e-5}
TRUNK_TOL_PRECISE = 2e-4


def _call(name, *args):
    from hawkeye_b200 import _lib
    _lib.call(name, *args, _lib.stream_ptr())


@pytest.mark.parametrize('precise', [0, 1], indirect=True)
@pytest.mark.parametrize('shape', [(2, 28 * 28, 1024, True), (2, 14 * 14, 2048, False)])
@pytest.mark.parametrize('P', [2, 3])
def test_me_against_fp64(P, shape, precise):
    from hawkeye_b200 import _lib
    N, HW, C, main = shape
    c, r = detgen.det((N, HW, C), 8300), detgen.det((N, HW, C), 8301)
    m = detgen.det((N, P, C), 8302, 2.0)
    dout, dparts = detgen.det((N, HW, C), 8303), detgen.det((N, HW, P, C), 8304)
    out_r, parts_r, dc_r, dr_r, dm_r = O.me(c, r, m, dout if main else None, dparts)
    cg, rg, mg = c.cuda(), r.cuda(), m.cuda()
    out = torch.full((N, HW, C), float('nan'), device='cuda') if main else None
    parts = torch.full((N, HW, P, C), float('nan'), device='cuda')
    _call('hk_crossx_me_fwd', cg, rg, mg, out, parts, N, HW, P, C)
    if main:
        assert rel_l2(out.cpu(), out_r) < TOL
    assert rel_l2(parts.cpu(), parts_r) < TOL
    dc, dr = torch.empty_like(cg), torch.empty_like(rg)
    dm = torch.empty_like(mg)
    ws = torch.empty(_lib.query('hk_crossx_me_bwd_workspace_bytes', N, HW, P, C), dtype=torch.uint8, device='cuda')
    _call('hk_crossx_me_bwd', cg, rg, mg, dout.cuda() if main else None, dparts.cuda(), dc, dr, dm, N, HW, P, C, ws,
          ws.numel())
    for got, ref in ((dc, dc_r), (dr, dr_r), (dm, dm_r)):
        assert rel_l2(got.cpu(), ref) < TOL
    dm2 = torch.empty_like(mg)
    _call('hk_crossx_me_bwd', cg, rg, mg, dout.cuda() if main else None, dparts.cuda(), dc, dr, dm2, N, HW, P, C, ws,
          ws.numel())
    assert torch.equal(dm, dm2)


def _bn_ref(x, bn, w, b, training):
    """BatchNorm2d of the NCHW x with the weight w, bias b, and the batch statistics or bn's running ones, in x's dtype"""
    if training:
        mean, var = x.mean((0, 2, 3)), x.var((0, 2, 3), unbiased=False)
    else:
        mean, var = bn.running_mean.to(x.dtype), bn.running_var.to(x.dtype)
    sh = (1, -1, 1, 1)
    return (x - mean.view(sh)) / torch.sqrt(var.view(sh) + bn.eps) * w.view(sh) + b.view(sh)


@pytest.mark.parametrize('precise', [1], indirect=True)
@pytest.mark.parametrize('training', [True, False])
def test_excitation_block_against_fp64(training, precise):
    """ops_crossx.excite on layer3's last block (P = 2, batch 2) against an fp64 autograd restatement of the reference's
    Bottleneck with its MELayer: the squeeze mean_hw(c) feeds the gates, so dc carries dz / HW, and the residual's
    gradient joins conv1's data gradient."""
    from hawkeye_b200 import ops, ops_crossx, ops_resnet
    from hawkeye_b200.backbone.resnet import Bottleneck
    from hawkeye_b200.methods.crossx import MELayer
    import torch.nn.functional as F
    torch.manual_seed(8900)
    blk = Bottleneck(1024, 256)
    blk.me = MELayer(1024, reduction=256, nparts=2)
    blk.load_state_dict(detgen.state_like(blk, seed=8901))
    for bn in (blk.bn1, blk.bn2, blk.bn3):
        bn.running_mean.copy_(detgen.det((bn.num_features,), 8902, 0.1))
        bn.running_var.copy_(1.0 + detgen.det((bn.num_features,), 8903, 0.1).abs())
    blk = blk.cuda()
    x = detgen.det((2, 28, 28, 1024), 8904, positive=True)
    dout, dparts = detgen.det((2, 28, 28, 1024), 8905), detgen.det((2, 28, 28, 2, 1024), 8906)
    u1, u2, _, _ = ops_resnet.block_units(blk)
    units = (u1, u2, ops_resnet.Unit('1x1', blk.conv3, blk.bn3, False))
    xg = x.cuda().requires_grad_(True)
    ops.CAPTURE = []
    try:
        out, parts = ops_crossx.excite(xg, units, list(blk.me.parts), True, training)
        masks = [(t[1] > 0).cpu().permute(0, 3, 1, 2) for t in ops.CAPTURE if t[0] == 'relu']
    finally:
        ops.CAPTURE = None
    assert len(masks) == 2
    masks += [(out > 0).cpu().permute(0, 3, 1, 2)] + [(parts[..., i, :] > 0).cpu().permute(0, 3, 1, 2) for i in range(2)]
    torch.autograd.backward((out, parts), (dout.cuda(), dparts.cuda()))
    names = [n for n, _ in blk.named_parameters()]
    got = [xg.grad.cpu()] + [p.grad.cpu() for p in blk.parameters()]

    # fp64 on the ReLU branch the library's forward took: a mask that flips between fp32 and fp64 moves a gradient by a
    # whole dy element, which is not an error of the kernels (tests/matched.py does the same for the VGG path)
    bns = {n: getattr(blk, n).cpu() for n in ('bn1', 'bn2', 'bn3')}
    ps = {n: p.detach().cpu().double().requires_grad_(True) for n, p in blk.named_parameters()}
    x64 = x.double().permute(0, 3, 1, 2).requires_grad_(True)

    def bn(t, n):
        return _bn_ref(t, bns[n], ps[n + '.weight'], ps[n + '.bias'], training)

    a = bn(F.conv2d(x64, ps['conv1.weight']), 'bn1') * masks[0]
    a = bn(F.conv2d(a, ps['conv2.weight'], padding=1), 'bn2') * masks[1]
    c = bn(F.conv2d(a, ps['conv3.weight']), 'bn3')
    z = c.mean((2, 3))
    o64 = (c + x64) * masks[2]
    obj = (o64 * dout.double().permute(0, 3, 1, 2)).sum()
    for i in range(2):
        h = F.relu(F.linear(z, ps[f'me.parts.{i}.0.weight'], ps[f'me.parts.{i}.0.bias']))
        g = torch.sigmoid(F.linear(h, ps[f'me.parts.{i}.2.weight'], ps[f'me.parts.{i}.2.bias']))
        obj = obj + ((c * g[:, :, None, None] + x64) * masks[3 + i] * dparts[:, :, :, i].double().permute(0, 3, 1, 2)).sum()
    ref = list(torch.autograd.grad(obj, [x64] + [ps[n] for n in names]))
    ref[0] = ref[0].permute(0, 2, 3, 1)
    assert rel_l2(out.cpu(), o64.detach().permute(0, 2, 3, 1)) < TRUNK_TOL_PRECISE
    errs = {n: rel_l2(gg, r) for n, gg, r in zip(['x'] + names, got, ref)}
    print('excite rel-L2 vs fp64 on the library\'s branch:', {n: f'{e:.2e}' for n, e in errs.items()})
    assert all(e < TRUNK_TOL_PRECISE for e in errs.values()), errs


@pytest.mark.parametrize('P', [2, 3])
def test_fuse_against_fp64_with_ties(P):
    N, H, W, C = 2, 28, 28, 1024
    parts = detgen.det((N, H * W, P, C), 8400)
    parts[:, :, :, :64] = 0.0                                   # all-zero channels: the max ties everywhere
    parts[0, 100, :, 70] = parts[0, 500, :, 70] = 9.0          # a two-way tie
    R = detgen.det((N, H * W // 4, C), 8401)
    dS, dmax = detgen.det((N, H * W, C), 8402), detgen.det((N, P, C), 8403)
    pg = parts.cuda()
    pmax = torch.empty(N, P, C, device='cuda')
    pidx = torch.empty(N, P, C, device='cuda', dtype=torch.int32)
    dparts = torch.full_like(pg, float('nan'))
    for p in range(P):
        S = torch.empty(N, H * W, C, device='cuda')
        _call('hk_crossx_fuse_fwd', pg, R.cuda(), S, pmax, pidx, N, H, W, P, C, p)
        S_r, mx_r, idx_r = O.fuse(parts, R, p, H, W)
        assert rel_l2(S.cpu(), S_r) < TOL
        assert torch.equal(pmax[:, p].cpu().double(), mx_r)
        assert torch.equal(pidx[:, p].cpu().long(), idx_r)
        assert (pidx[:, p, :64] == 0).all() and pidx[0, p, 70].item() == 100
        dR = torch.empty(N, H * W // 4, C, device='cuda')
        _call('hk_crossx_fuse_bwd', dS.cuda(), dmax.cuda(), pidx, dparts, dR, N, H, W, P, C, p)
        dp_r, dR_r = O.fuse_bwd(dS, dmax[:, p], idx_r, H, W)
        assert rel_l2(dparts[:, :, p].cpu(), dp_r) < TOL and rel_l2(dR.cpu(), dR_r) < TOL


def _loss(P, inputs, world=1, reduce_s=None):
    from hawkeye_b200.ops_crossx import CrossXLossFn
    xs = [t.cuda().requires_grad_(True) for t in inputs[:6]]
    loss, correct = CrossXLossFn.apply(*xs, inputs[6].cuda(), 0.1, I.GAMMA, world, reduce_s)
    loss.backward()
    return loss.item(), [t.grad.cpu() for t in xs], correct.item()


@pytest.mark.parametrize('precise', [0, 1], indirect=True)
@pytest.mark.parametrize('P,N', I.LOSS_CASES)
def test_loss_against_reference(P, N, precise):
    inputs = I.loss_inputs(P, N)
    loss, grads, correct = _loss(P, inputs)
    ref = float(G[f'loss_{P}_{N}'])
    assert abs(loss - ref) <= 1e-5 * abs(ref)
    ol, og = O.loss(*inputs, I.GAMMA)
    assert abs(ol - ref) <= 1e-7 * abs(ref)          # the reference stores its correlation matrix in float32
    for name, got, o in zip(('xf', 'xp', 'xc', 'fu', 'fp', 'fc'), grads, og):
        tol = DX_TOL[precise] if name[0] == 'x' else TOL
        assert rel_l2(got, G[f'd{name}_{P}_{N}']) < tol, name
        assert rel_l2(got, o) < tol, name
    assert correct == int(((inputs[0] + inputs[1] + inputs[2]).argmax(1) == inputs[6]).sum())
    again = _loss(P, inputs)
    assert again[0] == loss and all(torch.equal(a, b) for a, b in zip(again[1], grads))


def test_loss_zero_row_and_two_rank_split():
    """An all-zero feature row: finite loss, zero gradient.  Two halves of a batch, each with the other half's batch sums
    added to its own (the all-reduce) and the world scale, sum to the full batch's regulariser gradient."""
    P, N = 2, 8
    inputs = list(I.loss_inputs(P, N))
    inputs[4] = inputs[4].clone()
    inputs[4][3, 1] = 0.0
    _, grads, _ = _loss(P, inputs)
    assert all(torch.isfinite(g).all() for g in grads) and (grads[4][3, 1] == 0).all()
    full = _loss(P, inputs)[1]
    halves = [[t[:N // 2] for t in inputs], [t[N // 2:] for t in inputs]]
    sums = [torch.cat([O.batch_sums(h[3 + g]).flatten() for g in range(3)]).float() for h in halves]
    total = (sums[0] + sums[1]).cuda()
    for i, h in enumerate(halves):
        _, g, _ = _loss(P, h, world=2, reduce_s=lambda s: s.copy_(total))
        for j in range(3, 6):                                  # regulariser gradients: world x the global batch's share
            ref = full[j][i * N // 2:(i + 1) * N // 2] * 2
            assert rel_l2(g[j], ref) < 1e-4, (i, j)


@pytest.mark.parametrize('precise', [0, 1], indirect=True)
def test_conv3x3_1024_against_fp64(precise):
    from hawkeye_b200 import ops
    N, H, W, C = 8, 28, 28, 1024
    x = detgen.tf32_rna(detgen.det((N, H, W, C), 8500))
    w = detgen.tf32_rna(detgen.det((C, C, 3, 3), 8501, (2.0 / (9 * C)) ** 0.5))
    dy = detgen.tf32_rna(detgen.det((N, H, W, C), 8502))
    xg, wg = x.cuda().requires_grad_(True), w.cuda().requires_grad_(True)
    y = ops.Conv3x3Fn.apply(xg, wg, None)
    y.backward(dy.cuda())
    x64, w64 = x.cuda().double().permute(0, 3, 1, 2).requires_grad_(True), w.cuda().double().requires_grad_(True)
    y64 = torch.nn.functional.conv2d(x64, w64, padding=1)
    y64.backward(dy.cuda().double().permute(0, 3, 1, 2))
    tol = 1e-3 if precise == 0 else 5e-5            # 3xTF32: measured 2.1e-5 on the forward (K = 9216)
    assert rel_l2(y.permute(0, 3, 1, 2).double(), y64.detach()) < tol
    assert rel_l2(xg.grad.permute(0, 3, 1, 2).double(), x64.grad) < tol
    assert rel_l2(wg.grad.double(), w64.grad) < tol


def _net(P=2):
    import hawkeye_b200 as hb
    from hawkeye_b200.cfgnode import CfgNode
    net = hb.MODEL.get('CrossX')(CfgNode(dict(num_parts=P, num_classes=I.K, pretrained=False)))
    net.load_state_dict(detgen.state_like(net, seed=81))
    return net.cuda()


def _grads(net):
    out = {}
    for n in ('fc_ulti', 'fc_plty', 'fc_cmbn'):
        out[f'{n}_w_slice'] = getattr(net, n).weight.grad.cpu()[:, ::32]
        out[f'{n}_b'] = getattr(net, n).bias.grad.cpu()
    for blk in ('layer3', 'layer4'):
        me = getattr(net, blk)[-1].me.parts
        for i in range(2):
            out[f'{blk}_me{i}_0_w'] = me[i][0].weight.grad.cpu()[:, ::8]
            out[f'{blk}_me{i}_2_b'] = me[i][2].bias.grad.cpu()
    out['conv3_1_w_slice'] = net.conv3_1.weight.grad.cpu()[::16, ::16]
    out['conv2_1_w_slice'] = net.conv2_1.weight.grad.cpu()[::16, ::16]
    out['conv1_w'] = net.conv1.weight.grad.cpu()
    return out


@pytest.mark.parametrize('precise', [1], indirect=True)
def test_crossx_against_reference(precise):
    """The fixture's BatchNorms have momentum 1: the eval step normalises with the train step's batch statistics."""
    from hawkeye_b200.cfgnode import CfgNode
    from hawkeye_b200.losses import CrossXLoss
    net = _net()
    for m in net.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.momentum = I.NET_BN_MOMENTUM
    crit = CrossXLoss(CfgNode(dict(num_parts=2, gamma=list(I.GAMMA))))
    x, y = I.net_image().cuda(), I.net_labels().cuda()
    for mode in ('train', 'eval'):
        net.train(mode == 'train')
        net.zero_grad()
        outs = net(x)
        loss = crit(outs, y)
        loss.backward()
        got = dict(xf=outs[0].detach().cpu(), xp=outs[1].detach().cpu(), xc=outs[2].detach().cpu(), **_grads(net))
        errs = {k: rel_l2(v, G[f'net64_{mode}_{k}']) for k, v in got.items()}
        ref_errs = {k: rel_l2(G[f'net_{mode}_{k}'], G[f'net64_{mode}_{k}']) for k in got}
        ref_loss = float(G[f'net64_{mode}_loss'])
        errs['loss'] = abs(loss.item() - ref_loss) / abs(ref_loss)
        ref_errs['loss'] = abs(float(G[f'net_{mode}_loss']) - ref_loss) / abs(ref_loss)
        print(f'CrossX {mode} rel-L2 vs fp64, library / reference fp32:',
              {k: f'{errs[k]:.2e} / {ref_errs[k]:.2e}' for k in errs})
        for k in errs:
            assert errs[k] < max(TRUNK_TOL_PRECISE, 2 * ref_errs[k]), (mode, k, errs[k], ref_errs[k])
    for k in ('running_mean', 'running_var'):
        assert rel_l2(getattr(net.bn3_1, k).cpu(), G[f'net64_bn3_1_{k}']) < TRUNK_TOL_PRECISE


@pytest.mark.parametrize('precise', [1], indirect=True)
def test_p1_p3_logits_and_input_check(precise):
    from hawkeye_b200._lib import HawkeyeLibError
    x = I.net_image().cuda()
    with torch.no_grad():
        assert rel_l2(_net(1).eval()(x).cpu(), G['p1_logits']) < 1e-3
        o = _net(3).eval()(x)
        for i, n in enumerate(('xf', 'xp', 'xc')):
            assert rel_l2(o[i].cpu(), G[f'p3_{n}']) < 1e-3
        with pytest.raises(HawkeyeLibError):
            _net(2)(torch.zeros(1, 3, 480, 480, device='cuda'))


def _batch(seed, n=8):
    return dict(img=detgen.det((n, 3, 448, 448), seed).cuda(), label=detgen.det_labels(n, 200, seed + 1).cuda())


def test_trainer_step_no_sync_and_tester(tmp_path, monkeypatch):
    from hawkeye_b200.cfgnode import CfgNode
    from hawkeye_b200.test import Tester
    x = detgen.det((4, 3, 448, 448), 8600)
    val = [{'img': x, 'label': torch.zeros(4, dtype=torch.int64)}]
    tr = make_trainer(monkeypatch, 'CrossX', 'CrossX.yaml', graph=False, experiment=dict(log_dir=str(tmp_path)),
                      dataloaders={'val': val}, pretrained=False)
    tr.batch_training(_batch(8610))
    batch = _batch(8612)
    torch.cuda.synchronize()
    w0 = tr.model.fc_cmbn.weight.detach().clone()
    with no_host_sync():
        tr.batch_training(batch)
    assert not torch.equal(tr.model.fc_cmbn.weight, w0)
    assert np.isfinite(tr.average_meters['loss'].avg) and 0 <= tr.average_meters['acc'].avg <= 100
    with torch.no_grad():
        pred = tr.model.prediction(tr.model.eval()(x.cuda())).argmax(1).cpu()
    tr.model.train()
    val[0]['label'] = torch.where(torch.arange(4) % 2 == 0, pred, (pred + 1) % 200)
    tr.validate()
    acc = tr.average_meters['acc'].avg
    assert abs(acc - 50.0) < 1e-6
    path = tr.save_model('best_model.pth')
    cfg = CfgNode(dict(experiment=dict(name='t', cuda=[0]), dataset=dict(batch_size=4, num_workers=0,
                                                                         transformer=dict(resize_size=600, image_size=448)),
                       model=dict(name='CrossX', num_parts=2, num_classes=200, pretrained=False, load=path)))
    assert Tester(cfg, dataloader=val).test() == acc


def test_graph_replay_equals_eager():
    from hawkeye_b200.cfgnode import CfgNode
    from hawkeye_b200.losses import CrossXLoss
    net = _net().train()
    crit = CrossXLoss(CfgNode(dict(num_parts=2, gamma=list(I.GAMMA))))
    b = _batch(8700, 4)
    x, labels = b['img'], b['label']

    def step():
        net.zero_grad()
        out = net(x)
        loss = crit(out, labels)
        loss.backward()
        return [out[0], loss, crit.last_correct]
    # the 3x3 weight gradients add their tiles with atomics
    replay_against_eager(step, net, net.parameters(), grad_bound=1e-5)
