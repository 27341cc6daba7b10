"""AP-CNN on the device: every new kernel forward and backward against fp64 / the numpy oracle at odd and even maps, the ROI
selection index-exact on fixtures of the unmodified reference (tests/golden/make_golden_apcnn.py) and on a planted tie, the
refinement against the fixture with the reference's draws replayed, the attention against the reference's materialised
A3..A5, bitwise repeatability, the full model in precise mode against the end-to-end fixture, and the behaviour of a step:
two BatchNorm updates, gradient into layer2 from stage II, no host synchronisation, CUDA-graph replay, the trainer."""
import json

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import apcnn_inputs as I
import detgen
from conftest import load_golden, rel_l2
from oracle import apcnn_oracle as O
from kernel_check import nhwc, precise_on  # noqa: F401  (a fixture)
from step_check import (assert_trainer_replays, capture, make_trainer, no_host_sync, random_init,  # noqa: F401
                        replay_against_eager, side_stream)

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures('random_init')]
G = load_golden('reference_apcnn')


def _draws(rec, counts):
    d = np.zeros((len(rec), 2), dtype=np.float32)
    for n, (u, ind) in enumerate(rec):
        lv = 0 if u < 0.3 else (1 if u < 0.6 else -1)
        d[n] = (u, (ind + 0.5) / counts[n, lv] if lv >= 0 else 0.0)
    return torch.from_numpy(d).cuda()


def _fixture_rois(prefix):
    boxes = np.concatenate([G[f'{prefix}_boxes_{l}'] for l in range(3)], axis=1)
    counts = np.stack([G[f'{prefix}_counts_{l}'] for l in range(3)], axis=1).astype(np.int32)
    return boxes, counts


def _select(gates, nc, image):
    from hawkeye_b200 import ops_apcnn
    win = torch.from_numpy(ops_apcnn.central_windows(image // 8, image // 8, nc))
    keep = torch.from_numpy(ops_apcnn.suppression_table()).cuda()
    return ops_apcnn.roi_select([torch.from_numpy(g).cuda() for g in gates], win, keep, image, image)


@pytest.mark.parametrize('N,h,w,C', [(1, 1, 1, 4), (2, 3, 5, 256), (16, 7, 7, 256)])
def test_lateral_mean_bcast(N, h, w, C):
    from hawkeye_b200 import ops, ops_apcnn
    torch.manual_seed(N + h)
    top = torch.randn(N, h, w, C, device='cuda', requires_grad=True)
    lat = torch.randn(N, 2 * h, 2 * w, C, device='cuda', requires_grad=True)
    out = ops_apcnn.LateralFn.apply(top, lat)
    ref = O.lateral(top.detach().permute(0, 3, 1, 2).cpu().numpy(), lat.detach().permute(0, 3, 1, 2).cpu().numpy())
    assert np.array_equal(out.detach().permute(0, 3, 1, 2).cpu().numpy(), ref)
    g = torch.randn_like(out)
    out.backward(g)
    want = g.double().view(N, h, 2, w, 2, C).sum((2, 4))
    assert (top.grad.double() - want).abs().max() < 1e-5 and torch.equal(lat.grad, g)
    if C % 256 == 0:
        x = torch.randn(N, 2 * h, 2 * w, C, device='cuda', requires_grad=True)
        b = torch.randn(N, C, device='cuda', requires_grad=True)
        y = ops_apcnn.BcastAddFn.apply(x, b) * 1.0
        p = ops.NHWCMeanFn.apply(y)
        assert (p.double() - (x.double() + b.double()[:, None, None]).mean((1, 2))).abs().max() < 1e-5
        p.backward(torch.ones_like(p))
        assert (x.grad - 1.0 / (4 * h * w)).abs().max() < 1e-6 and (b.grad - 1.0).abs().max() < 1e-5


@pytest.mark.parametrize('N,H,W', [(1, 1, 1), (2, 5, 7), (3, 12, 12), (16, 14, 14)])
def test_attention_fwd_bwd_against_fp64(N, H, W):
    from hawkeye_b200 import ops_apcnn
    torch.manual_seed(N * H + W)
    Fm = torch.randn(N, H, W, 256, device='cuda', requires_grad=True)
    conv = torch.nn.ConvTranspose2d(256, 1, 3, 1, 1).cuda()
    gate, pf, psf = ops_apcnn.AttentionFn.apply(Fm, conv.weight, conv.bias)
    gp, gs = torch.randn_like(pf), torch.randn_like(psf)
    ((pf * gp).sum() + (psf * gs).sum()).backward()
    c64 = torch.nn.ConvTranspose2d(256, 1, 3, 1, 1).cuda().double()
    c64.load_state_dict({k: v.double() for k, v in conv.state_dict().items()})
    F64 = Fm.detach().double().permute(0, 3, 1, 2).requires_grad_(True)
    s = torch.sigmoid(c64(F64))
    m, sf = F64.mean((2, 3)), (s * F64).mean((2, 3))
    ((m * gp.double()).sum() + (sf * gs.double()).sum()).backward()
    assert (gate.double() - s[:, 0]).abs().max() < 1e-5                    # fp32 sums of 2304 products
    assert rel_l2(pf, m) < 1e-5 and rel_l2(psf, sf) < 1e-5
    assert rel_l2(Fm.grad, F64.grad.permute(0, 2, 3, 1)) < 1e-4
    assert rel_l2(conv.weight.grad, c64.weight.grad) < 1e-4 and rel_l2(conv.bias.grad, c64.bias.grad) < 1e-4
    g2, pf2, psf2 = ops_apcnn.AttentionFn.apply(Fm.detach(), conv.weight.detach(), conv.bias.detach())
    assert torch.equal(gate, g2) and torch.equal(pf, pf2) and torch.equal(psf, psf2)


def test_attention_against_reference_fixture():
    """PyramidAttentions of the unmodified reference: gates, mean_hw A_l (materialised there), dF and the gate's gradients."""
    from hawkeye_b200.methods.apcnn import PyramidAttentions
    apn = PyramidAttentions(256)
    apn.load_state_dict(detgen.state_like(apn, seed=11))
    apn.cuda()
    Fs = [nhwc(detgen.det((3, 256, s, s), 4200 + s).cuda()).requires_grad_(True) for s in (12, 6, 3)]
    gates, pm, v = apn(Fs)
    Gv = torch.stack([detgen.det((3, 256), 4300 + i) for i in range(3)]).cuda()
    (v * Gv).sum().backward()
    for i in range(3):
        assert (gates[i].cpu() - torch.from_numpy(G[f'att_gate_{i}'])[:, 0]).abs().max() < 1e-5
        assert rel_l2(v[i].detach().cpu(), G[f'att_pool_{i}']) < 1e-4      # the channel gate's linears run in TF32
        assert rel_l2(Fs[i].grad.permute(0, 3, 1, 2).cpu(), G[f'att_dF_{i}']) < 2e-3
    assert rel_l2(apn.A3_1.conv.weight.grad.cpu(), G['att_dw_0']) < 1e-4
    assert rel_l2(apn.A3_1.conv.bias.grad.cpu(), G['att_db_0']) < 1e-4


@pytest.mark.parametrize('nc', [200, 12])
def test_roi_matches_reference_fixture(nc):
    boxes, counts = _select(I.gates(nc), nc, I.ROI_IMAGE)
    want_b, want_c = _fixture_rois(f'roi_{nc}')
    assert np.array_equal(counts.cpu().numpy(), want_c)
    assert np.array_equal(boxes.cpu().numpy(), want_b)
    b2, c2 = _select(I.gates(nc), nc, I.ROI_IMAGE)
    assert torch.equal(boxes, b2) and torch.equal(counts, c2)


@pytest.mark.parametrize('N,image', [(1, 96), (5, 224), (16, 448)])
def test_roi_matches_oracle_with_ties(N, image):
    rs = np.random.RandomState(N)
    gates = []
    for l in range(3):
        h = image // (8 << l)
        g = (rs.randint(1, 9, size=(N, h, h)) / 16.0).astype(np.float32)       # eight distinct values: ties everywhere
        gates.append(g)
    gates[0][0] = 0.5                                                          # a flat map
    boxes, counts = _select(gates, 200, image)
    want_b, want_c = O.roi_select(gates, 200, image, image)
    assert np.array_equal(counts.cpu().numpy(), want_c) and np.array_equal(boxes.cpu().numpy(), want_b)


def test_refine_matches_reference_fixture():
    from hawkeye_b200 import ops_apcnn
    boxes, counts = _fixture_rois('roi_200')
    b, c = torch.from_numpy(boxes).cuda(), torch.from_numpy(counts).cuda()
    Gw = nhwc(detgen.det((I.ROI_BATCH, 8, 28, 28), 4101).cuda())
    for mode, draws in (('train', _draws(G['refine_draws'], counts)), ('eval', None)):
        x = nhwc(detgen.det((I.ROI_BATCH, 8, 28, 28), 4100).cuda()).requires_grad_(True)
        y = ops_apcnn.RefineFn.apply(x, b, c, draws)
        (y * Gw).sum().backward()
        assert (y.detach().permute(0, 3, 1, 2).cpu() - torch.from_numpy(G[f'refine_{mode}_y'])).abs().max() < 5e-5      # fp32 on both sides; values of a few units times a rescale of up to ~2
        assert (x.grad.permute(0, 3, 1, 2).cpu() - torch.from_numpy(G[f'refine_{mode}_dx'])).abs().max() < 5e-5      # fp32 on both sides; values of a few units times a rescale of up to ~2
        y2 = ops_apcnn.RefineFn.apply(x.detach(), b, c, draws)
        assert torch.equal(y.detach(), y2)


@pytest.mark.parametrize('N,H,C', [(2, 12, 4), (3, 28, 64), (16, 56, 512)])
def test_refine_fwd_bwd_against_interpolate(N, H, C):
    from hawkeye_b200 import ops_apcnn
    rs = np.random.RandomState(H)
    gates = [rs.random_sample((N, H >> l, H >> l)).astype(np.float32) for l in range(3)]
    boxes, counts = _select(gates, 12, 8 * H)
    draws = torch.from_numpy(rs.random_sample((N, 2)).astype(np.float32)).cuda()
    x = torch.randn(N, H, H, C, device='cuda', requires_grad=True)
    y = ops_apcnn.RefineFn.apply(x, boxes, counts, draws)
    g = torch.randn_like(y)
    y.backward(g)
    want = O.refine(x.detach().double().permute(0, 3, 1, 2).cpu().numpy()[:, :4], boxes.cpu().numpy(), counts.cpu().numpy(),
                    draws.cpu().numpy())
    assert np.abs(y.detach().permute(0, 3, 1, 2).cpu().numpy()[:, :4] - want).max() < 1e-4
    # the map is linear in x: <y, g> == <x, dx>
    lhs, rhs = (y.detach().double() * g.double()).sum().item(), (x.detach().double() * x.grad.double()).sum().item()
    assert abs(lhs - rhs) < 1e-4 * max(1.0, abs(lhs))
    x.grad = None
    ops_apcnn.RefineFn.apply(x, boxes, counts, draws).backward(g)
    dx1 = x.grad.clone()
    x.grad = None
    ops_apcnn.RefineFn.apply(x, boxes, counts, draws).backward(g)
    assert torch.equal(dx1, x.grad)


def test_act_and_mix_against_torch():
    from hawkeye_b200 import ops, ops_apcnn
    torch.manual_seed(3)
    x = torch.randn(16, 512, device='cuda', requires_grad=True)
    for elu in (False, True):
        x.grad = None
        y = ops.ActFn.apply(x, elu)
        g = torch.randn_like(y)
        y.backward(g)
        x64 = x.detach().double().requires_grad_(True)
        r = F.elu(x64) if elu else F.relu(x64)
        r.backward(g.double())
        assert (y.double() - r).abs().max() < 1e-6 and (x.grad.double() - x64.grad).abs().max() < 1e-6
    z, pm, psf = (torch.randn(3, 5, 256, device='cuda', requires_grad=True) for _ in range(3))
    v = ops_apcnn.MixFn.apply(z, pm, psf)
    g = torch.randn_like(v)
    v.backward(g)
    z64, pm64, psf64 = (t.detach().double().requires_grad_(True) for t in (z, pm, psf))
    c3 = torch.sigmoid(z64[0])
    c4 = (torch.sigmoid(z64[1]) + c3) / 2
    c5 = (torch.sigmoid(z64[2]) + c4) / 2
    r = psf64 + torch.stack([c3, c4, c5]) * pm64
    r.backward(g.double())
    assert (v.double() - r).abs().max() < 1e-5
    for a, b in ((z, z64), (pm, pm64), (psf, psf64)):
        assert (a.grad.double() - b.grad).abs().max() < 1e-5


def _shallow(nc=I.E2E_CLASSES):
    from hawkeye_b200.methods.apcnn import ResNet
    net = ResNet(nc, (1, 1, 1, 1))
    net.load_state_dict(I.e2e_state(net))
    return net.cuda().train()


def _e2e_step(net, zero_stage2=False):
    from hawkeye_b200.losses import APCNNLoss
    x = detgen.det((I.E2E_BATCH, 3, I.E2E_IMAGE, I.E2E_IMAGE), 4400).cuda()
    labels = detgen.det_labels(I.E2E_BATCH, I.E2E_CLASSES, 4401).cuda()
    _, counts = _fixture_rois('e2e')
    out = net(x, labels, draws=_draws(G['e2e_draws'], counts))
    if zero_stage2:
        out = (out[0], out[1][:4] + [o.detach() for o in out[1][4:]], out[2], out[3])
    loss = APCNNLoss()(out, labels)
    loss.backward()
    return out, loss


def test_model_against_fixture(precise_on):
    """Tolerances as for DCL and NTS-Net: fp32 here (3xTF32 products) against the reference's fp32 CPU run; the trunk's
    gradients pass through two stages of batch-statistics BatchNorm over 4 images and drift the most."""
    net = _shallow()
    (out_mean, out_list, mask_cat, roi_list), loss = _e2e_step(net)
    assert (mask_cat.cpu() - torch.from_numpy(G['e2e_mask_cat'])).abs().max() < 1e-4
    for l in range(3):
        assert np.array_equal(roi_list[l][1].cpu().numpy(), G[f'e2e_counts_{l}'])
        assert np.array_equal(roi_list[l][0].cpu().numpy(), G[f'e2e_boxes_{l}'])
    assert rel_l2(torch.stack(out_list).detach().cpu(), G['e2e_out_list']) < 1e-3
    assert rel_l2(out_mean.detach().cpu(), G['e2e_out_mean']) < 1e-3
    assert abs(loss.item() - float(G['e2e_loss'])) < 1e-3 * float(G['e2e_loss'])
    params = dict(net.named_parameters())
    for i, k in enumerate(json.loads(bytes(G['e2e_grad_names']).decode())):
        got = params[k].grad.flatten()[torch.from_numpy(G[f'e2e_grad_{i}_idx']).cuda()].cpu()
        assert rel_l2(got, G[f'e2e_grad_{i}']) < (3e-2 if k.split('.')[0] in ('conv1', 'layer2', 'layer3', 'layer4') else 1e-2), k
    sd = net.state_dict()
    for k in ('layer2.0.bn1', 'layer3.0.bn1', 'fpn.P5_1.conv_master.bn', 'cls3.2', 'cls_concate.3'):
        assert int(sd[k + '.num_batches_tracked']) == int(G[f'e2e_nbt_{k}']) == (1 if k.startswith('layer2') else 2)
        assert rel_l2(sd[k + '.running_mean'].cpu(), G[f'e2e_rm_{k}']) < 1e-3, k
        assert rel_l2(sd[k + '.running_var'].cpu(), G[f'e2e_rv_{k}']) < 1e-3, k


def test_layer2_receives_gradient_from_stage_two(precise_on):
    a = _shallow()
    _e2e_step(a)
    b = _shallow()
    _e2e_step(b, zero_stage2=True)
    ga, gb = a.layer2[0].conv2.weight.grad, b.layer2[0].conv2.weight.grad
    assert rel_l2(ga, gb) > 1e-2
    from hawkeye_b200 import ops_apcnn
    roi = ops_apcnn.roi_to_reference(*_select(I.gates(200), 200, I.ROI_IMAGE))
    assert [tuple(r.shape) for r in roi] == [(int(G[f'roi_200_counts_{l}'].sum()), 5) for l in range(3)]


def _full():
    from hawkeye_b200.cfgnode import CfgNode
    from hawkeye_b200.methods.apcnn import APCNN
    return APCNN(CfgNode(dict(name='APCNN', num_classes=200))).cuda().train()


def test_train_step_448_batch_16_no_sync():
    from hawkeye_b200.losses import APCNNLoss
    net, crit = _full(), APCNNLoss()
    x = detgen.det((16, 3, 448, 448), 4500).cuda()
    labels = detgen.det_labels(16, 200, 4501).cuda()
    crit(net(x, labels), labels).backward()                          # warm-up: workspaces, first-call attributes
    torch.cuda.synchronize()
    before = net.cls3[2].num_batches_tracked.item()
    with no_host_sync():
        out = net(x, labels)
        loss = crit(out, labels)
        loss.backward()
    assert net.cls3[2].num_batches_tracked.item() == before + 2 and net.layer4[2].bn3.num_batches_tracked.item() == before + 2
    assert net.fpn.P5_1.conv_gpb.bn.num_batches_tracked.item() == before + 2 and net.bn1.num_batches_tracked.item() == 2
    assert torch.isfinite(loss).item() and crit.last_correct.dtype == torch.int32
    assert tuple(out[2].shape) == (16, 3, 56, 56) and len(out[1]) == 8 and out[3][0][0].shape == (16, 5, 4)
    net.eval()
    with torch.no_grad():
        a, b = net(x)[0], net(x)[0]
    assert torch.equal(a, b)                                          # eval mode: no drop block, no draws


def test_graph_replay_equals_eager_and_draws_afresh():
    from hawkeye_b200.losses import APCNNLoss
    net, crit = _shallow(), APCNNLoss()
    x = detgen.det((I.E2E_BATCH, 3, I.E2E_IMAGE, I.E2E_IMAGE), 4400).cuda()
    labels = detgen.det_labels(I.E2E_BATCH, I.E2E_CLASSES, 4401).cuda()
    _, counts = _fixture_rois('e2e')
    fixed = _draws(G['e2e_draws'], counts)

    def step():
        net.zero_grad()
        out = net(x, labels, draws=fixed)
        loss = crit(out, labels)
        loss.backward()
        return out[1] + [loss, out[3][0][0]]
    # the 3x3 weight gradients add their tiles with atomics
    replay_against_eager(step, net, net.parameters(), grad_bound=1e-5)
    # without explicit draws the captured torch.rand draws afresh on every replay: the stage-II logits change
    seen = set()
    with side_stream(), torch.no_grad():
        graph, free = capture(lambda: net(x, labels))
        for _ in range(6):
            graph.replay()
            seen.add(tuple(free[1][4].flatten()[:4].tolist()))
    assert len(seen) > 1


def test_trainer_captures_and_replays(monkeypatch):
    data = dict(img=detgen.det((4, 3, 224, 224), 4600).cuda(), label=detgen.det_labels(4, 200, 4601).cuda())
    tr = make_trainer(monkeypatch, 'APCNN', 'APCNN.yaml', graph=True)
    assert_trainer_replays(tr, [data] * 6)
    assert [g['lr'] for g in tr.optimizer.param_groups] == pytest.approx([0.0005 / 10, 0.0005])
