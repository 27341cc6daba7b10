"""MGE-CNN on the device: the part head, the CAM boxes, the concatenation and the gate against the fp64 / float32 numpy
oracle at the 224 and 448 map sizes, the boxes index-exact on fixtures of the unmodified reference
(tests/golden/make_golden_mge.py), bitwise repeatability, the shallow model in precise mode against the end-to-end fixture,
and the behaviour of a step: one BatchNorm update per trunk, no host synchronisation, an eval mode without the layer4
recompute, CUDA-graph replay and the trainer."""
import json

import numpy as np
import pytest
import torch

import detgen
import mge_inputs as I
from conftest import load_golden, rel_l2
from oracle import mge_oracle as O
from kernel_check import precise_on  # noqa: F401  (a fixture)
from step_check import assert_trainer_replays, make_trainer, no_host_sync, random_init, replay_against_eager  # noqa: F401

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures('random_init')]
G = load_golden('reference_mge')


def _cfg(**kw):
    from hawkeye_b200.cfgnode import CfgNode
    return CfgNode(dict(dict(name='MGE_CNN', num_classes=200, image_size=224, box_thred=0.2), **kw))


@pytest.mark.parametrize('N,H', [(1, 14), (3, 14), (1, 28), (5, 28)])
def test_part_head_against_fp64(N, H, precise_on):
    from hawkeye_b200 import ops_mge
    torch.manual_seed(N * H)
    O_ = 40
    x = torch.randn(N, H, H, 1024, device='cuda')
    x[..., 0] = 1.0                            # a constant feature
    conv = torch.nn.Conv2d(1024, O_, 1, 1, 1).cuda()
    with torch.no_grad():
        conv.weight[0].zero_()
        conv.bias[0] = 0.5                     # the border ties every interior pixel and wins
        conv.weight[1].zero_()
        conv.weight[1, 0] = -1.0
        conv.bias[1] = 0.5                     # the border wins outright: every interior pixel is 0.5 - 1
        conv.weight[2].zero_()
        conv.bias[2] = -1.0                    # everything is below zero: pooled 0, no gradient
    pooled, pos = ops_mge.part(x, conv)
    g = torch.randn_like(pooled)
    pooled.backward(g)
    xn = x.cpu().double().numpy()
    w64, b64 = conv.weight.detach().view(O_, -1).cpu().double().numpy(), conv.bias.detach().cpu().double().numpy()
    want, wpos = O.part_head(xn, w64, b64)
    assert np.abs(pooled.detach().cpu().numpy() - want).max() < 1e-4 * max(1.0, np.abs(want).max())
    assert np.array_equal(pos.cpu().numpy(), wpos)
    assert (pos[:, :3] == -1).all() and (pooled[:, 2] == 0).all()
    dw, db = O.part_head_bwd(xn, wpos, want, g.cpu().double().numpy())
    assert rel_l2(conv.weight.grad.view(O_, -1).cpu(), dw) < 1e-5 and rel_l2(conv.bias.grad.cpu(), db) < 1e-6
    assert (conv.weight.grad[:3] == 0).all() and conv.bias.grad[2] == 0
    p2, q2 = ops_mge.part(x, conv)
    assert torch.equal(pooled, p2) and torch.equal(pos, q2)
    gw = conv.weight.grad.clone()
    conv.weight.grad = None
    p2.backward(g)
    assert torch.equal(gw, conv.weight.grad)


def _cam_inputs(name):
    conv5, lw, rate, size = I.bbox_case(name)
    N, C, h, w = conv5.shape
    W = torch.from_numpy(lw * np.float32(h * w)).cuda()             # relu(W[n]) / hw is lw[n] again (exactly for powers of 2)
    feat = torch.from_numpy(conv5).permute(0, 2, 3, 1).contiguous().cuda()
    return feat, W, rate, size, conv5, lw


@pytest.mark.parametrize('name', sorted(I.BBOX_CASES))
def test_cam_box_against_reference_fixture(name):
    from hawkeye_b200 import ops_mge
    feat, W, rate, size, conv5, lw = _cam_inputs(name)
    N = feat.shape[0]
    want = np.array([I.crop_box(xy, size) for xy in G[f'bbox_{name}']])
    by_target = ops_mge.cam_box(feat, W, size, rate, targets=torch.arange(N, device='cuda'))
    logits = torch.eye(N, device='cuda') * 3 - 1                                # argmax n on row n
    by_argmax = ops_mge.cam_box(feat, W, size, rate, logits=logits)
    assert torch.equal(by_target, by_argmax)
    got = by_target.cpu().numpy()
    if name in I.EXACT_CASES:
        assert np.array_equal(got, want)
    else:
        assert np.abs(got - want).max() <= 1
    assert np.array_equal(got, O.cam_box(conv5, lw, rate, size)) or name not in I.EXACT_CASES
    assert torch.equal(by_target, ops_mge.cam_box(feat, W, size, rate, targets=torch.arange(N, device='cuda')))


@pytest.mark.parametrize('N,size', [(1, 224), (7, 224), (1, 448), (5, 448)])
def test_cam_box_random_maps_and_crop(N, size):
    from hawkeye_b200 import ops_mge
    rs = np.random.RandomState(N + size)
    h = size // 32
    conv5 = (np.abs(rs.standard_normal((N, 2048, h, h))) * (rs.random_sample((N, 2048, h, h)) < 0.2)).astype(np.float32)
    W = rs.standard_normal((200, 2048)).astype(np.float32)
    logits = rs.standard_normal((N, 200)).astype(np.float32)
    feat = torch.from_numpy(conv5).permute(0, 2, 3, 1).contiguous().cuda()
    boxes = ops_mge.cam_box(feat, torch.from_numpy(W).cuda(), size, 0.4, logits=torch.from_numpy(logits).cuda())
    want = O.cam_box(conv5, O.gradcam_weights(W, logits.argmax(1), h * h), 0.4, size)
    assert np.abs(boxes.cpu().numpy() - want).max() <= 1
    img = torch.randn(N, 3, size, size, device='cuda')
    out = ops_mge.crop(img, boxes, size)
    for n in range(N):
        y0, x0, y1, x1 = boxes[n].tolist()
        ref = torch.nn.functional.interpolate(img[n:n + 1, :, y0:y1, x0:x1], size=(size, size), mode='bilinear',
                                              align_corners=True)
        assert (out[n:n + 1] - ref).abs().max() < 1e-5


def test_cat_and_gate_against_fp64():
    from hawkeye_b200 import ops_mge
    torch.manual_seed(5)
    a, b = torch.randn(5, 2048, device='cuda'), torch.relu(torch.randn(5, 120, device='cuda'))
    got = ops_mge.cat_l2n(a, b)
    assert (got.double().cpu() - torch.from_numpy(O.cat_l2n(a.cpu().numpy(), b.cpu().numpy()))).abs().max() < 3e-3
    h = torch.randn(5, 512, device='cuda', requires_grad=True)
    lin = torch.nn.Linear(512, 3).cuda()
    cats = [torch.randn(5, 12, device='cuda', requires_grad=True) for _ in range(3)]
    out, pr = ops_mge.GateFn.apply(h, lin.weight, lin.bias, *cats)
    dout = torch.randn_like(out)
    out.backward(dout)
    c64 = [c.detach().cpu().numpy() for c in cats]
    wout, wpr = O.gate(h.detach().cpu().numpy(), lin.weight.detach().cpu().numpy(), lin.bias.detach().cpu().numpy(), c64)
    assert np.abs(out.detach().cpu().numpy() - wout).max() < 1e-4 and np.abs(pr.detach().cpu().numpy() - wpr).max() < 1e-5
    _, dh, dw2, db2 = O.gate_bwd(h.detach().cpu().numpy(), lin.weight.detach().cpu().numpy(), wpr, c64,
                                 dout.cpu().numpy())
    assert rel_l2(h.grad.cpu(), dh) < 1e-5 and rel_l2(lin.weight.grad.cpu(), dw2) < 1e-5 and rel_l2(lin.bias.grad.cpu(), db2) < 1e-5
    assert all(c.grad is None for c in cats)
    o2, p2 = ops_mge.GateFn.apply(h.detach(), lin.weight.detach(), lin.bias.detach(), *cats)
    assert torch.equal(o2, out) and torch.equal(p2, pr)


def _shallow():
    from hawkeye_b200.methods.mge import LocalCamNet
    net = LocalCamNet(_cfg(num_classes=I.E2E_CLASSES, image_size=I.E2E_IMAGE, box_thred=I.E2E_THRED), layers=I.E2E_LAYERS)
    net.load_state_dict(detgen.state_like(net))
    return net.cuda().train()


def _e2e_inputs():
    x = detgen.det((I.E2E_BATCH, 3, I.E2E_IMAGE, I.E2E_IMAGE), 5300).cuda()
    labels = detgen.det_labels(I.E2E_BATCH, I.E2E_CLASSES, 5301).cuda()
    return x, labels


def test_model_against_fixture(precise_on):
    """Tolerances as for AP-CNN: fp32 here (3xTF32 products) against the reference's fp32 CPU run; the trunks' gradients
    pass through batch-statistics BatchNorm over 4 images and drift the most."""
    from hawkeye_b200.losses import MGECNNLoss
    net = _shallow()
    x, labels = _e2e_inputs()
    out = net(x)
    loss = MGECNNLoss()(out, labels)
    loss.backward()
    xy = G['e2e_box_xy']
    for s in range(2):
        want = np.array([I.crop_box(r, I.E2E_IMAGE) for r in xy[s]])
        assert np.array_equal(out['boxes'][s].cpu().numpy(), want), s
    assert rel_l2(torch.stack(out['logits']).detach().cpu(), G['e2e_logits']) < 1e-3
    for i in range(10):
        assert rel_l2(out['logits'][i].detach().cpu(), G['e2e_logits'][i]) < 1e-3, i
    assert rel_l2(out['pr_gate'].detach().cpu(), G['e2e_pr_gate']) < 1e-3
    assert abs(loss.item() - float(G['e2e_loss'])) < 1e-3 * float(G['e2e_loss'])
    params = dict(net.named_parameters())
    for i, k in enumerate(json.loads(bytes(G['e2e_grad_names']).decode())):
        got = params[k].grad.flatten()[torch.from_numpy(G[f'e2e_grad_{i}_idx']).cuda()].cpu()
        assert rel_l2(got, G[f'e2e_grad_{i}']) < (3e-2 if k.startswith('conv4') or k.startswith('conv5') else 1e-2), k
    assert sorted(k for k, p in params.items() if p.grad is None) == json.loads(bytes(G['e2e_no_grad_json']).decode())
    sd = net.state_dict()
    for k in json.loads(bytes(G['e2e_bn_json']).decode()):
        assert int(sd[k + '.num_batches_tracked']) == int(G[f'e2e_nbt_{k}']) == 1
        assert rel_l2(sd[k + '.running_mean'].cpu(), G[f'e2e_rm_{k}']) < 1e-3, k
        assert rel_l2(sd[k + '.running_var'].cpu(), G[f'e2e_rv_{k}']) < 1e-3, k


def _nbt(net):
    return [int(getattr(net, 'conv4' + b)[1].num_batches_tracked) for b in ('', '_box', '_box_2', '_gate')] + \
           [int(getattr(net, 'conv5' + b)[-1].bn3.num_batches_tracked) for b in ('', '_box', '_box_2', '_gate')]


@pytest.mark.parametrize('size,batch', [(224, 4), (448, 16)])
def test_train_step_no_sync(size, batch):
    import hawkeye_b200 as hb
    from hawkeye_b200.losses import MGECNNLoss
    net, crit = hb.MODEL.get('MGE_CNN')(_cfg(image_size=size)).cuda().train(), MGECNNLoss()
    x = detgen.det((batch, 3, size, size), 5400).cuda()
    labels = detgen.det_labels(batch, 200, 5401).cuda()
    crit(net(x), labels).backward()                                  # warm-up: workspaces, first-call attributes
    torch.cuda.synchronize()
    before = _nbt(net)
    with no_host_sync():
        out = net(x)
        loss = crit(out, labels)
        loss.backward()
    assert _nbt(net) == [b + 1 for b in before] and before == [1] * 8
    assert torch.isfinite(loss).item() and crit.last_correct.dtype == torch.int32
    assert len(out['logits']) == 10 and tuple(out['boxes'].shape) == (2, batch, 4) and tuple(out['pr_gate'].shape) == (batch, 3)
    assert net.cls_cat_a.fc.weight.grad is None


def test_eval_is_deterministic_without_recompute(monkeypatch):
    from hawkeye_b200 import ops_resnet
    from hawkeye_b200.methods import mge
    net = _shallow()
    x, labels = _e2e_inputs()
    calls = []
    real = ops_resnet.block_stack
    monkeypatch.setattr(mge.ops_resnet, 'block_stack', lambda *a: calls.append(a[2]) or real(*a))
    with torch.no_grad():
        net(x)
        assert calls == [True, False, True, False, True, True]           # four trunks, two eval-mode recomputes
        del calls[:]
        net.eval()
        a, b = net(x), net(x)
        assert calls == [False] * 8
    for u, v in zip(a['logits'] + [a['boxes']], b['logits'] + [b['boxes']]):
        assert torch.equal(u, v)
    with torch.no_grad():                                                # with targets no index pass runs at all
        net.train()
        del calls[:]
        net(x, labels)
        assert calls == [True] * 4


def test_graph_replay_equals_eager():
    from hawkeye_b200.losses import MGECNNLoss
    net, crit = _shallow(), MGECNNLoss()
    x, labels = _e2e_inputs()
    params = [p for p in net.parameters() if p is not net.cls_cat_a.fc.weight and p is not net.cls_cat_a.fc.bias]

    def step():
        net.zero_grad()
        out = net(x)
        loss = crit(out, labels)
        loss.backward()
        return out['logits'] + [loss, out['boxes']]
    # the 3x3 weight gradients add their tiles with atomics
    replay_against_eager(step, net, params, grad_bound=1e-5)


def test_trainer_captures_and_replays(monkeypatch):
    data = dict(img=detgen.det((4, 3, 224, 224), 5500).cuda(), label=detgen.det_labels(4, 200, 5501).cuda())
    tr = make_trainer(monkeypatch, 'MGE_CNN', 'MGE_CNN.yaml', graph=True)
    w0 = tr.model.cls_cat_a.fc.weight.detach().clone()
    assert_trainer_replays(tr, [data] * 6)
    assert [g['lr'] for g in tr.optimizer.param_groups] == pytest.approx([0.0004 * 0.01, 0.0004 * 0.1 * 0.01])
    assert torch.equal(tr.model.cls_cat_a.fc.weight, w0)                 # never trained, never decayed
