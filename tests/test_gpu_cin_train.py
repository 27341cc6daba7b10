"""CIN's training path on the device: CINLoss against fixtures of the unmodified reference at the shape the shipped config
trains (tests/golden/make_golden_cin_loss.py) in both precision modes, a near-cancelling pair against the fp64 oracle, the
channel-interaction module's train-mode backward at batch 20, C = 2048, 7x7, and the trainer: a step without host
synchronisation, CUDA-graph replay, the zero-pair weight decay of h, checkpoints and the Tester."""
import numpy as np
import pytest
import torch

import cin_inputs as I
import detgen
from conftest import load_golden, rel_l2
from oracle import cin_oracle as O
from step_check import assert_trainer_replays, make_trainer, no_host_sync, random_init, replay_against_eager  # noqa: F401

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures('random_init')]
G = load_golden('reference_cin_loss')


def _criterion():
    from hawkeye_b200.cfgnode import CfgNode
    from hawkeye_b200.losses import CINLoss
    crit = CINLoss(CfgNode(dict(alpha=I.ALPHA, beta=0.5, channel=I.C, feature_size=I.WH, r_channel=I.R)))
    crit.load_state_dict(I.h_state())
    return crit.cuda()


@pytest.fixture(scope='module')
def crit():
    return _criterion()


def _run(crit, z, zc, target, precise):
    from hawkeye_b200 import _lib
    z, zc = z.cuda().requires_grad_(True), zc.cuda().requires_grad_(True)
    crit.zero_grad()
    _lib.set_precise(precise)
    try:
        loss = crit((z, zc), target.cuda())
        loss.backward()
    finally:
        _lib.set_precise(0)
    return loss.item(), z.grad.cpu(), zc.grad.cpu(), crit.h.weight.grad.cpu(), crit.h.bias.grad.cpu()


@pytest.mark.parametrize('precise', [0, 1])
@pytest.mark.parametrize('name', ['balanced', 'some', 'allsame'])
def test_loss_against_reference(crit, name, precise):
    loss, dz, dzc, dw, db = _run(crit, I.logits(), I.z_cci(), I.labels(name), precise)
    ref = float(G[f'{name}_loss'])
    # TF32: P = D W^T is one 100352-long single-pass TF32 dot per entry, a few 1e-4 relative, and the loss is dominated by
    # L1^2, proportional to |P|^4: four times P's error, 1.0e-3 and 1.3e-3 measured on an H100.  The gradients carry
    # P's error once.  3xTF32 is fp32-class; the reference's own fp32 dots differ from it by ~1e-5.
    tol, tol_g = (5e-3, 3e-3) if not precise else (2e-5, 2e-5)
    print(name, f'precise={precise}', f'loss {loss:.6f} ref {ref:.6f}')
    assert abs(loss - ref) <= tol * abs(ref)
    # the cross-entropy alone, no GEMM; its kernel rounds the logit gradient to TF32 in the default mode
    assert rel_l2(dz, G[f'{name}_dz']) < (5e-4 if not precise else 1e-5)
    assert not db.any()                                                  # the bias cancels: exactly zero, but present
    if name == 'balanced':
        assert not dzc.any() and not dw.any()
        assert abs(loss - float(G['balanced_ce'])) <= 1e-5 * abs(ref)
        return
    assert rel_l2(dzc[:, ::64, ::7], G[f'{name}_dzc_slice']) < tol_g
    assert rel_l2(dzc.double().sum((1, 2)), G[f'{name}_dzc_sums']) < 10 * tol_g   # sums of +-dd rows: partly cancelling
    assert rel_l2(dw[::16, ::389], G[f'{name}_dw_slice']) < tol_g
    assert rel_l2(dw.double().sum(1), G[f'{name}_dw_rowsums']) < tol_g


@pytest.mark.parametrize('precise', [0, 1])
def test_near_cancelling_pairs_against_fp64(crit, precise):
    """b = a + small noise, with the noise a thousandth of the rows: projecting the rows separately in TF32 would leave an
    error of about half the difference; projecting the difference keeps TF32's 2^-11 of it."""
    zc = I.z_cci() * 1000.0
    zc[I.B // 2:] = zc[:I.B // 2] + detgen.det((I.B // 2, I.C, I.WH), 6020, I.SCALE)
    z, target = I.logits(), I.labels('allsame')
    loss, _, dzc, dw, _ = _run(crit, z, zc, target, precise)
    st = I.h_state()
    ref_loss, _, ref_dzc, ref_dw, _ = O.cin_loss(z.numpy(), zc.numpy(), target.numpy(), st['h.weight'].numpy(), I.ALPHA)
    ce, _ = O.ce_ls(z.numpy(), target.numpy())
    # the same budget as the fixture comparison (1.1e-3 measured in TF32 on an H100): the error is relative to the
    # difference, not to the rows
    tol = 5e-3 if not precise else 2e-5
    print(f'near-cancelling precise={precise}: term {loss - ce:.6e} ref {ref_loss - ce:.6e}')
    assert ref_loss - ce > 5 * ce
    assert abs(loss - ref_loss) <= tol * (ref_loss - ce)
    assert rel_l2(dzc, ref_dzc) < tol and rel_l2(dw, ref_dw) < tol


@pytest.mark.parametrize('precise', [0, 1])
def test_module_train_backward_full_size(precise):
    from hawkeye_b200 import _lib
    from hawkeye_b200.methods.cin import ChannelInteractionModule
    m = ChannelInteractionModule(in_channel=I.C, spatial_size=(7, 7))
    m.load_state_dict(detgen.state_like(m))
    m = m.cuda().train()
    x = detgen.det((I.B, I.C, 7, 7), 6010, positive=True).cuda().requires_grad_(True)
    _lib.set_precise(precise)
    try:
        z, zc = m(x)
        ((z * detgen.det(z.shape, 6011).cuda()).sum() + (zc * detgen.det(zc.shape, 6012).cuda()).sum()).backward()
    finally:
        _lib.set_precise(0)
    z, zc = z.detach().cpu(), zc.detach().cpu()
    errs = {'z': rel_l2(z[:, ::16, ::5], G['module_z_slice']), 'zcci': rel_l2(zc[:, ::16, ::5], G['module_zcci_slice']),
            'z_sums': rel_l2(z.double().sum((1, 2)), G['module_z_sums']),
            'zcci_sums': rel_l2(zc.double().sum((1, 2)), G['module_zcci_sums']),
            'dx': rel_l2(x.grad.cpu()[:, ::16], G['module_dx_slice']),
            'dx_sums': rel_l2(x.grad.cpu().double().sum((1, 2, 3)), G['module_dx_sums']),
            'conv.weight': rel_l2(m.conv.weight.grad.cpu()[::16, ::16], G['module_g_conv.weight_slice']),
            'conv.bias': rel_l2(m.conv.bias.grad.cpu(), G['module_g_conv.bias']),
            'fc.weight': rel_l2(m.fc.weight.grad.cpu()[:, ::97], G['module_g_fc.weight_slice']),
            'fc.bias': rel_l2(m.fc.bias.grad.cpu(), G['module_g_fc.bias'])}
    print(f'module B=20 C=2048 7x7 precise={precise}', {k: f'{v:.1e}' for k, v in errs.items()})
    # the forward as test_gpu_cin.py: three chained single-pass TF32 products.  The fc gradients are sums over 20 rows
    # weighted by d_weight[b], itself a 4M-term sum (C x C) whose terms largely cancel, so at C = 2048 they carry several
    # times the error they do at C <= 256: 6e-3 (TF32) and 2.8e-4 (3xTF32) measured on an H100 against the fp32 reference.
    tol_f, tol_b = (3e-3, 1.2e-2) if not precise else (1e-4, 6e-4)
    assert max(errs[k] for k in ('z', 'zcci', 'z_sums', 'zcci_sums')) < tol_f
    assert max(errs[k] for k in ('dx', 'dx_sums', 'conv.weight', 'conv.bias', 'fc.weight', 'fc.bias')) < tol_b


def _trainer(monkeypatch, graph=False, **experiment):
    return make_trainer(monkeypatch, 'CIN', 'CIN.yaml', graph=graph, experiment=experiment)


def _batch(name, seed=6100):
    return dict(img=detgen.det((I.B, 3, 224, 224), seed).cuda(), label=I.labels(name).cuda())


def test_trainer_step_no_sync_and_h_updates(tmp_path, monkeypatch):
    tr = _trainer(monkeypatch, log_dir=str(tmp_path))
    assert tr.optimizer.param_groups[1]['params'] == [tr.criterion.h.weight, tr.criterion.h.bias]
    lr, wd = tr.optimizer.param_groups[1]['lr'], tr.optimizer.param_groups[1]['weight_decay']
    assert tr.optimizer.defaults['momentum'] == 0.0 and wd == 0.0002
    tr.batch_training(_batch('balanced'))                               # warm-up: workspaces, first-call attributes
    batch = _batch('balanced', 6101)
    torch.cuda.synchronize()
    h0 = tr.criterion.h.weight.detach().clone()
    with no_host_sync():
        tr.batch_training(batch)
    for p in list(tr.model.parameters()) + list(tr.criterion.parameters()):
        assert p.grad is not None
    assert not tr.criterion.h.weight.grad.any() and not tr.criterion.h.bias.grad.any()
    # no pair on the 4 x 5 order: h changes by the weight decay alone
    h1 = tr.criterion.h.weight.detach().clone()
    assert torch.allclose(h1, h0 * (1 - lr * wd), rtol=1e-6, atol=0)
    tr.batch_training(_batch('some', 6102))
    torch.cuda.synchronize()
    assert tr.criterion.h.weight.grad.abs().sum().item() > 0
    moved = (tr.criterion.h.weight.detach() - h1 * (1 - lr * wd)).abs().max().item()
    assert moved > 1e-5 * h1.abs().max().item()                        # a hundred times the rounding of the decay
    assert np.isfinite(tr.average_meters['loss'].avg) and 0 <= tr.average_meters['acc'].avg <= 100

    # checkpoint: h restored with the model; without 'criterion' the fresh h stays, with a warning
    path = tr.save_checkpoint()
    saved = tr.criterion.h.weight.detach().clone()
    tr2 = _trainer(monkeypatch, log_dir=str(tmp_path), resume=path)
    assert torch.equal(tr2.criterion.h.weight, saved) and tr2.start_epoch == tr.epoch
    assert tr2.criterion.h.weight.data_ptr() >= tr2.flat.flat.data_ptr()       # still a view of the flat buffer
    ck = torch.load(path, map_location='cpu')
    del ck['criterion']
    path2 = str(tmp_path / 'no_criterion.pth')
    torch.save(ck, path2)
    tr3 = _trainer(monkeypatch, log_dir=str(tmp_path), resume=path2)
    assert not torch.equal(tr3.criterion.h.weight.cpu(), saved.cpu())

    # the Tester scores the model save_model writes (the reference's format: the model alone)
    model_path = tr.save_model('best_model.pth')
    assert set(torch.load(model_path, map_location='cpu')) == set(tr.model.state_dict())
    from hawkeye_b200.cfgnode import CfgNode
    from hawkeye_b200.test import Tester
    cfg = CfgNode(dict(experiment=dict(name='t', cuda=[0]), dataset=dict(batch_size=4, num_workers=0,
                                                                         transformer=dict(resize_size=256, image_size=224)),
                       model=dict(name='CIN', num_classes=200, load=model_path)))
    x = detgen.det((4, 3, 224, 224), 6103)
    t = Tester(cfg, dataloader=[])
    with torch.no_grad():
        pred = t.model.eval()(x.cuda()).argmax(1).cpu()
    assert abs(Tester(cfg, dataloader=[{'img': x, 'label': pred}]).test() - 100.0) < 1e-6


def test_graph_replay_equals_eager():
    import hawkeye_b200 as hb
    from hawkeye_b200.cfgnode import CfgNode
    net = hb.MODEL.get('CIN')(CfgNode(dict(name='CIN', num_classes=200))).cuda().train()
    crit = _criterion()
    x, labels = detgen.det((I.B, 3, 224, 224), 6200).cuda(), I.labels('some').cuda()

    def step():
        net.zero_grad()
        crit.zero_grad()
        out = net(x)
        loss = crit(out, labels)
        loss.backward()
        return [out[0], loss]
    # the 3x3 weight gradients add their tiles with atomics
    replay_against_eager(step, net, list(net.parameters()) + list(crit.parameters()), grad_bound=1e-5)
    assert all(p.grad is not None for p in crit.parameters())           # h.bias too, though its gradient is zero
    assert crit.h.weight.grad.abs().sum() > 0


def test_trainer_captures_and_replays(tmp_path, monkeypatch):
    tr = _trainer(monkeypatch, graph=True, log_dir=str(tmp_path))
    assert_trainer_replays(tr, [_batch('balanced', 6300 + i) for i in range(5)])
