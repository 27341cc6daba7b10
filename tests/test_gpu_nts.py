"""NTS-Net on the device: hk_nts_nms index-exact against the fp64 oracle (seeded and fixture scores, IoU-0.25 pairs at the
top, B from 1 to 64, both image sizes), hk_nts_crop against F.interpolate on the same device, the proposal head and the
ranking loss forward and backward against fp64, the full model in precise mode against fixtures of the unmodified reference
(tests/golden/make_golden_nts.py), and the behaviour of a step: dropout in eval mode, two BatchNorm updates per step, no host
synchronisation, CUDA-graph replay equal to the eager step, and the trainer's captured steps."""
import json

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import detgen
import nts_inputs
from conftest import load_golden, rel_l2
from oracle import nts_oracle as O
from kernel_check import precise_on  # noqa: F401  (a fixture)
from step_check import assert_trainer_replays, make_trainer, no_host_sync, random_init, replay_against_eager  # noqa: F401

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures('random_init')]
G = load_golden('reference_nts')


def _net(seed_state=True, **kw):
    from hawkeye_b200.cfgnode import CfgNode
    from hawkeye_b200.methods.nts import NTSNet
    net = NTSNet(CfgNode(dict(dict(proposal_num=6, cat_num=4, image_size=224), **kw)))
    if seed_state:
        net.load_state_dict(detgen.state_like(net))
    return net.cuda()


@pytest.mark.parametrize('size', [224, 448])
@pytest.mark.parametrize('B', [1, 5, 64])
def test_nms_matches_oracle(size, B):
    from hawkeye_b200 import ops_nts
    anchors = G[f'anchors_{size}']
    T = nts_inputs.NMS_TOPN[size]
    ks = [(B * 7 + i) % nts_inputs.NMS_VECTORS for i in range(B)]
    scores = torch.from_numpy(np.stack([nts_inputs.nms_scores(anchors, k) for k in ks])).cuda()
    idx, prob, boxes = ops_nts.nms(scores, torch.from_numpy(anchors).cuda(), T)
    want = np.stack([G[f'nms_{size}'][k] for k in ks])
    assert np.array_equal(idx.cpu().numpy(), want)
    assert torch.equal(prob, scores.gather(1, idx))
    assert np.array_equal(boxes.cpu().numpy(), anchors[want])


def test_nms_on_fixture_scores_and_ties():
    from hawkeye_b200 import ops_nts
    anchors = torch.from_numpy(G['anchors_224']).cuda()
    rpn = torch.from_numpy(G['e2e_rpn_score']).cuda()
    idx, _, _ = ops_nts.nms(rpn, anchors, 6)
    assert np.array_equal(idx.cpu().numpy(), G['e2e_top_n_index'])
    flat = torch.zeros(2, 426, device='cuda')                       # all equal: the lower index goes first
    idx, _, _ = ops_nts.nms(flat, anchors, 8)
    for n in range(2):
        assert np.array_equal(idx[n].cpu().numpy(), O.hard_nms(np.zeros(426), G['anchors_224'], 8))


@pytest.mark.parametrize('B,T', [(1, 1), (3, 6), (16, 6)])
def test_crop_matches_interpolate(B, T):
    from hawkeye_b200 import ops_nts
    from hawkeye_b200.methods.nts import edge_anchors
    anchors = edge_anchors(224)
    rs = np.random.RandomState(B * 10 + T)
    x = torch.from_numpy(rs.standard_normal((B, 3, 224, 224)).astype(np.float32)).cuda()
    boxes = torch.from_numpy(anchors[rs.choice(len(anchors), (B, T))]).cuda()
    out = ops_nts.crop(x, boxes)
    xp = F.pad(x, (224, 224, 224, 224))
    b = boxes.cpu().tolist()
    ref = torch.cat([F.interpolate(xp[n:n + 1, :, y0:y1, x0:x1], size=(224, 224), mode='bilinear', align_corners=True)
                     for n in range(B) for y0, x0, y1, x1 in b[n]])
    assert (out - ref).abs().max().item() < 1e-6


@pytest.mark.parametrize('B,H', [(1, 7), (4, 7), (3, 14)])
def test_proposal_head_fwd_bwd(precise_on, B, H):
    from hawkeye_b200.methods.nts import ProposalNet, edge_anchors
    torch.manual_seed(B + H)
    pn = ProposalNet().cuda()
    x = (0.5 * torch.randn(B, H, H, 2048, device='cuda')).relu()
    anchors = torch.from_numpy(edge_anchors(32 * H)).cuda()
    score, prob, idx, _ = pn(x, anchors, 6)
    names = ['down1', 'down2', 'down3', 'tidy1', 'tidy2', 'tidy3']
    p64 = {n: (getattr(pn, n).weight.detach().double().cpu().requires_grad_(True),
               getattr(pn, n).bias.detach().double().cpu().requires_grad_(True)) for n in names}
    ref = O.proposal_scores(x.permute(0, 3, 1, 2).double().cpu(), p64)
    assert rel_l2(score.cpu(), ref.detach()) < 1e-4      # fp32 sums of 18432 and 1152 terms with cancellation
    Gw = torch.randn(B, 6, device='cuda')
    (prob * Gw).sum().backward()
    (ref.gather(1, idx.cpu()) * Gw.double().cpu()).sum().backward()
    for n in names:
        for mine, want in ((getattr(pn, n).weight.grad, p64[n][0].grad), (getattr(pn, n).bias.grad, p64[n][1].grad)):
            assert rel_l2(mine.cpu(), want) < 1e-3, n


@pytest.mark.parametrize('B,T', [(1, 6), (4, 6), (64, 26)])
def test_rank_loss_fwd_bwd(B, T):
    from hawkeye_b200.ops_nts import RankLossFn
    torch.manual_seed(B * T)
    logits = torch.randn(B * T, 200, device='cuda')
    labels = torch.randint(0, 200, (B,), device='cuda')
    prob = (0.5 * torch.randn(B, T, device='cuda')).requires_grad_(True)
    loss = RankLossFn.apply(logits, labels, prob)
    loss.backward()
    p64 = prob.detach().double().cpu().requires_grad_(True)
    L = O.list_loss(logits.cpu(), labels.cpu().repeat_interleave(T)).view(B, T)
    ref = O.ranking_loss(p64, L)
    ref.backward()
    assert abs(loss.item() - ref.item()) <= 1e-5 * max(1.0, abs(ref.item()))
    assert (prob.grad.cpu().double() - p64.grad).abs().max() < 1e-6


def test_model_against_fixture(precise_on):
    from hawkeye_b200.losses import NTSLoss
    from hawkeye_b200.cfgnode import CfgNode
    net = _net()
    net.pretrained_model.drop.p = 0.0
    net.train()
    seen = {}
    net.proposal_net.register_forward_hook(lambda m, i, o: seen.__setitem__('rpn', o[0].detach().clone()))
    net.pretrained_model.register_forward_hook(lambda m, i, o: seen.setdefault('trunk_in', []).append(i[0].detach()))
    x = detgen.det((2, 3, 224, 224), 3100).cuda()
    labels = detgen.det_labels(2, 200, 3101).cuda()
    out = net(x)
    loss = NTSLoss(CfgNode(dict(proposal_num=6)))(out, labels)
    loss.backward()
    raw, concat, part, idx, prob = out
    rpn_err = (seen['rpn'].cpu().double() - torch.from_numpy(G['e2e_rpn_score']).double()).abs().max().item()
    assert rel_l2(seen['rpn'].cpu(), G['e2e_rpn_score']) < 1e-3           # fp32 here and in the reference's CPU run
    assert 2 * rpn_err < float(G['e2e_gap'])                 # the recorded gap decides the picks: they must be equal
    assert np.array_equal(idx.cpu().numpy(), G['e2e_top_n_index'])
    assert rel_l2(prob.detach().cpu(), G['e2e_top_n_prob']) < 1e-3
    parts = seen['trunk_in'][1].reshape(-1)
    assert (parts[torch.from_numpy(G['e2e_part_pix_idx']).cuda()].cpu() - torch.from_numpy(G['e2e_part_pix'])).abs().max() < 1e-5
    for got, key in ((raw, 'e2e_raw'), (concat, 'e2e_concat'), (part, 'e2e_part')):
        assert rel_l2(got.detach().cpu(), G[key]) < 1e-3, key
    assert abs(loss.item() - float(G['e2e_loss'])) < 1e-3 * abs(float(G['e2e_loss']))
    params = dict(net.named_parameters())
    for i, k in enumerate(json.loads(bytes(G['e2e_grad_names']).decode())):
        got = params[k].grad.flatten()[torch.from_numpy(G[f'e2e_grad_{i}_idx']).cuda()].cpu()
        trunk = k.startswith('pretrained_model.') and not k.startswith('pretrained_model.fc')
        assert rel_l2(got, G[f'e2e_grad_{i}']) < (3e-2 if trunk else 5e-3), k     # the trunk's gradients drift the most


def test_dropout_applies_in_eval_mode():
    net = _net()
    net.eval()
    x = detgen.det((2, 3, 224, 224), 3200).cuda()
    with torch.no_grad():
        torch.manual_seed(1)
        a = net(x)[0]
        torch.manual_seed(2)
        b = net(x)[0]
        net.pretrained_model.drop.p = 0.0
        c, d = net(x)[0], net(x)[0]
    assert not torch.equal(a, b)
    assert torch.equal(c, d)


def test_train_step_no_sync_two_bn_updates():
    from hawkeye_b200.cfgnode import CfgNode
    from hawkeye_b200.losses import NTSLoss
    net = _net()
    net.train()
    crit = NTSLoss(CfgNode(dict(proposal_num=6)))
    x = detgen.det((4, 3, 224, 224), 3300).cuda()
    labels = detgen.det_labels(4, 200, 3301).cuda()
    crit(net(x), labels).backward()                                  # warm-up: workspaces, first-call attributes
    torch.cuda.synchronize()
    before = net.pretrained_model.bn1.num_batches_tracked.item()
    with no_host_sync():
        loss = crit(net(x), labels)
        loss.backward()
    assert net.pretrained_model.bn1.num_batches_tracked.item() == before + 2
    assert net.pretrained_model.layer4[2].bn3.num_batches_tracked.item() == before + 2
    assert torch.isfinite(loss).item() and crit.last_correct.dtype == torch.int32


def test_graph_replay_equals_eager():
    from hawkeye_b200.cfgnode import CfgNode
    from hawkeye_b200.losses import NTSLoss
    net = _net()
    net.train()
    crit = NTSLoss(CfgNode(dict(proposal_num=6)))
    x = detgen.det((4, 3, 224, 224), 3400).cuda()
    labels = detgen.det_labels(4, 200, 3401).cuda()

    def step():
        net.zero_grad()
        out = net(x)
        loss = crit(out, labels)
        loss.backward()
        return [out[0], out[1], out[2], out[4], loss, out[3]]
    # dropout draws: the same seed for both; the 3x3 weight gradients add their tiles with atomics
    replay_against_eager(step, net, net.parameters(), grad_bound=1e-5, seed=77)


def test_trainer_captures_and_replays(monkeypatch):
    data = dict(img=detgen.det((4, 3, 224, 224), 3500).cuda(), label=detgen.det_labels(4, 200, 3501).cuda())
    assert_trainer_replays(make_trainer(monkeypatch, 'NTSNet', 'NTSNet.yaml', graph=True), [data] * 6)
