"""ResNet-50 trunk support kernels and the full MPN model vs torch-CPU fp64 / reference fixtures."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import detgen
from conftest import rel_l2
from kernel_check import nchw, nhwc

pytestmark = pytest.mark.gpu


# (N, H, W, C, relu, residual, k): the channels' means sit at k x their spread.  P = N*H*W pixels are summed in
# min(ceil(P / 256), 592) blocks: 1 block up to P = 256; 2 at P = 300; 32 at 8192; 98 at 25088 (the stem at 224x224, batch 2:
# the finalize loops over more than 32 partial rows); the 592 cap at 401408 (layer1 at 448x448, batch 32).
BN_CASES = [(4, 6, 6, 64, 1, 0, 0), (2, 4, 4, 256, 1, 1, 0), (3, 5, 7, 128, 0, 0, 0), (2, 2, 2, 2048, 1, 1, 0),
            (3, 10, 10, 12, 1, 0, 0), (3, 10, 10, 12, 0, 1, 100),
            (2, 64, 64, 2048, 1, 0, 10), (2, 64, 64, 2048, 0, 0, 100),
            (2, 112, 112, 64, 1, 0, 0), (2, 112, 112, 64, 1, 1, 10), (2, 112, 112, 64, 1, 0, 100),
            (32, 112, 112, 4, 1, 0, 100), (32, 112, 112, 64, 1, 0, 10), (32, 112, 112, 12, 0, 1, 0)]


@pytest.mark.parametrize('N,H,W,C,relu,res,k', BN_CASES,
                         ids=['-'.join(map(str, c[:6])) + (f'-mean{c[6]}sigma' if c[6] else '') for c in BN_CASES])
def test_batchnorm_train(N, H, W, C, relu, res, k):
    from hawkeye_b200 import _lib
    s = _lib.stream_ptr()
    sigma = 0.5 + detgen.det((C,), 6, positive=True)               # per-channel spread
    x = (detgen.det((N, C, H, W), 1) + k) * sigma.view(1, C, 1, 1)
    gamma, beta = 1 + detgen.det((C,), 2, 0.1), detgen.det((C,), 3, 0.1)
    r = detgen.det((N, C, H, W), 4) if res else None
    dy = detgen.det((N, C, H, W), 5)
    xd, gd, bd = x.double().requires_grad_(True), gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    rd = r.double().requires_grad_(True) if res else None
    rm, rv = torch.zeros(C, dtype=torch.float64), torch.ones(C, dtype=torch.float64)
    y_ref = F.batch_norm(xd, rm, rv, gd, bd, training=True, momentum=0.1, eps=1e-5)
    if res:
        y_ref = y_ref + rd
    P = N * H * W
    xg, y = nhwc(x).cuda(), torch.empty(N, H, W, C, device='cuda')
    mean, invstd = torch.empty(C, device='cuda'), torch.empty(C, device='cuda')
    rmg, rvg = torch.zeros(C, device='cuda'), torch.ones(C, device='cuda')
    nb = _lib.query('hk_bn_workspace_bytes', P, C)
    ws = torch.empty(nb, dtype=torch.uint8, device='cuda')
    rg = nhwc(r).cuda() if res else None
    _lib.call('hk_bn_fwd', xg, gamma.cuda(), beta.cuda(), rg, y, mean, invstd, rmg, rvg, 0.1, 1e-5, P, C, relu, ws, nb, s)
    # the statistics at fp32 accuracy whatever the offset; a mean near 0 has no relative scale of its own, so its error is
    # taken in units of the channel's spread (which is what it shifts xhat = (x - mean) * invstd by)
    xd64 = xd.detach()
    m_ref, v_ref = xd64.mean(dim=(0, 2, 3)), xd64.var(dim=(0, 2, 3), unbiased=False)
    sd = v_ref.sqrt()
    errs = {'mean': ((mean.cpu().double() - m_ref).abs() / sd).max().item(),
            'invstd': (invstd.cpu().double() * (v_ref + 1e-5).sqrt() - 1).abs().max().item(),
            'running_mean': ((rmg.cpu().double() - rm).abs() / sd).max().item(),
            'running_var': ((rvg.cpu().double() - rv).abs() / rv).max().item()}
    print(f'bn P={P} C={C} mean={k} sigma:', {n: f'{e:.1e}' for n, e in errs.items()})
    assert max(errs.values()) < 1e-5, errs
    assert rel_l2(nchw(y).cpu(), (F.relu(y_ref) if relu else y_ref).detach()) < 5e-4          # tf32-rounded on store
    # the gradients on the ReLU branch this forward took: at a mean of 100 sigma, the fp32 mean itself is off by up to
    # 6e-6 sigma, which flips the few outputs that close to zero, each an O(1) change of one dx element
    if relu:
        y_ref = y_ref * (nchw(y) > 0).cpu().double()
    grads = torch.autograd.grad(y_ref, [xd, gd, bd] + ([rd] if res else []), dy.double())
    dx, dres = torch.empty_like(xg), (torch.empty_like(xg) if res else None)
    dg, db = torch.empty(C, device='cuda'), torch.empty(C, device='cuda')
    _lib.call('hk_bn_bwd', xg, y, nhwc(dy).cuda(), gamma.cuda(), mean, invstd, dx, dres, dg, db, P, C, relu, ws, nb, s)
    assert rel_l2(nchw(dx).cpu(), grads[0]) < 2e-3
    assert rel_l2(dg.cpu(), grads[1]) < 2e-3 and rel_l2(db.cpu(), grads[2]) < 2e-3
    if res:
        assert rel_l2(nchw(dres).cpu(), grads[3]) < 1e-6
    if relu and not res:
        # hk_bn_bwd_ex: the ReLU mask re-evaluated from x (y not read, passed as null) must give the same bits
        dx2, dg2, db2 = torch.empty_like(xg), torch.empty(C, device='cuda'), torch.empty(C, device='cuda')
        _lib.call('hk_bn_bwd_ex', xg, None, nhwc(dy).cuda(), gamma.cuda(), beta.cuda(), mean, invstd, dx2, None, dg2, db2, P, C,
                  relu, ws, nb, s)
        assert torch.equal(dx2, dx) and torch.equal(dg2, dg) and torch.equal(db2, db)


@pytest.mark.parametrize('precision', [0, 1])
@pytest.mark.parametrize('relu,res', [(0, 0), (1, 0), (0, 1), (1, 1)])
def test_bn_apply_eval(relu, res, precision):
    """eval-mode BatchNorm (hk_bn_apply on running statistics, the Tester path of every ResNet model) against fp64
    F.batch_norm(training=False): the output is tf32-rounded for the next MMA in default mode, fp32 in precise mode."""
    from hawkeye_b200 import _lib
    N, H, W, C = 2, 14, 14, 256
    x = detgen.det((N, C, H, W), 11, 2.0) + 0.5
    rmean, rvar = detgen.det((C,), 12, 0.5), 0.25 + detgen.det((C,), 13, positive=True)
    gamma, beta = 1 + detgen.det((C,), 14, 0.1), detgen.det((C,), 15, 0.1)
    r = detgen.det((N, C, H, W), 16) if res else None
    y_ref = F.batch_norm(x.double(), rmean.double(), rvar.double(), gamma.double(), beta.double(), training=False, eps=1e-5)
    if res:
        y_ref = y_ref + r.double()
    if relu:
        y_ref = F.relu(y_ref)
    invstd = torch.rsqrt(rvar.cuda() + 1e-5)
    y = torch.empty(N, H, W, C, device='cuda')
    _lib.set_precise(precision)
    try:
        _lib.call('hk_bn_apply', nhwc(x).cuda(), rmean.cuda(), invstd, gamma.cuda(), beta.cuda(),
                  nhwc(r).cuda() if res else None, y, N * H * W, C, relu, _lib.stream_ptr())
    finally:
        _lib.set_precise(0)
    e = rel_l2(nchw(y).cpu(), y_ref)
    print('bn apply', relu, res, precision, e)
    assert e < (5e-4 if not precision else 1e-6)
    if relu:
        assert (y >= 0).all()


@pytest.mark.parametrize('N,H,W,C', [(2, 7, 9, 12), (3, 9, 7, 64), (2, 112, 112, 64)])
def test_maxpool3x3_s2_edges(N, H, W, C):
    """odd map sizes (the last window hangs over the bottom / right edge) and the stem's 112x112x64 output; post-ReLU
    inputs put exact-zero ties in the windows, which go to the first maximum in scan order, as in PyTorch."""
    from hawkeye_b200 import _lib
    s = _lib.stream_ptr()
    a = F.relu(detgen.det((N, C, H, W), 17)).double().requires_grad_(True)
    p_ref = F.max_pool2d(a, 3, 2, 1)
    g = detgen.det(p_ref.shape, 18).double()
    (ga,) = torch.autograd.grad(p_ref, a, g)
    Ho, Wo = p_ref.shape[2], p_ref.shape[3]
    out = torch.empty(N, Ho, Wo, C, device='cuda')
    am = torch.empty(N, Ho, Wo, C, device='cuda', dtype=torch.uint8)
    _lib.call('hk_maxpool3x3s2_fwd', nhwc(a.detach().float()).cuda(), out, am, N, H, W, C, s)
    assert torch.equal(nchw(out).cpu().double(), p_ref.detach())
    dx = torch.empty(N, H, W, C, device='cuda')
    _lib.call('hk_maxpool3x3s2_bwd', am, nhwc(g.float()).cuda(), dx, N, H, W, C, s)
    assert rel_l2(nchw(dx).cpu(), ga) < 1e-6


def test_maxpool3x3_s2_and_stride_helpers():
    from hawkeye_b200 import _lib
    s = _lib.stream_ptr()
    N, H, W, C = 2, 12, 10, 64
    a = F.relu(detgen.det((N, C, H, W), 7)).double().requires_grad_(True)
    p_ref = F.max_pool2d(a, 3, 2, 1)
    g = detgen.det(p_ref.shape, 8).double()
    (ga,) = torch.autograd.grad(p_ref, a, g)
    ag = nhwc(a.detach().float()).cuda()
    Ho, Wo = p_ref.shape[2], p_ref.shape[3]
    out = torch.empty(N, Ho, Wo, C, device='cuda')
    am = torch.empty(N, Ho, Wo, C, device='cuda', dtype=torch.uint8)
    _lib.call('hk_maxpool3x3s2_fwd', ag, out, am, N, H, W, C, s)
    assert torch.equal(nchw(out).cpu().double(), p_ref.detach())
    dx = torch.empty_like(ag)
    _lib.call('hk_maxpool3x3s2_bwd', am, nhwc(g.float()).cuda(), dx, N, H, W, C, s)
    assert rel_l2(nchw(dx).cpu(), ga) < 1e-6
    sub = torch.empty(N, H // 2, W // 2, C, device='cuda')
    _lib.call('hk_subsample2', ag, sub, N, H, W, C, s)
    assert torch.equal(sub.cpu(), ag.cpu()[:, ::2, ::2])
    up = torch.empty_like(ag)
    _lib.call('hk_upsample2_zero', sub, up, N, H, W, C, s)
    ref = torch.zeros_like(ag.cpu())
    ref[:, ::2, ::2] = sub.cpu()
    assert torch.equal(up.cpu(), ref)


@pytest.mark.parametrize('N,H,W,Cin,Cout', [(2, 16, 16, 64, 64), (4, 28, 28, 128, 128), (2, 8, 8, 256, 256)])
def test_conv3x3_stride2_fwd(N, H, W, Cin, Cout):
    from hawkeye_b200 import _lib
    s = _lib.stream_ptr()
    x = detgen.det((N, Cin, H, W), 1)
    w = detgen.det((Cout, Cin, 3, 3), 2, (2.0 / (Cout * 9)) ** 0.5)
    y_ref = F.conv2d(x.double(), w.double(), stride=2, padding=1)
    wf = torch.empty(9 * Cout * Cin, device='cuda')
    _lib.call('hk_conv3x3_pack_weights', w.cuda(), wf, None, Cout, Cin, s)
    y = torch.empty(N, H // 2, W // 2, Cout, device='cuda')
    _lib.call('hk_conv3x3_s2_fwd', nhwc(x).cuda(), wf, None, y, N, H, W, Cin, Cout, 0, s)
    e = rel_l2(nchw(y).cpu(), y_ref)
    print('conv s2', e)
    assert e < 2e-3


def test_conv3x3_wgrad_14x14_and_7x7():
    """maps whose width is not a multiple of 4 use an over-wide wgrad tile (TMA zero fill)."""
    from hawkeye_b200 import _lib
    s = _lib.stream_ptr()
    for (N, H, W, Cin, Cout) in ((3, 14, 14, 64, 128), (2, 7, 7, 128, 64)):
        x = detgen.det((N, Cin, H, W), 1, positive=True).double()
        w = detgen.det((Cout, Cin, 3, 3), 2, 0.05).double().requires_grad_(True)
        dy = detgen.det((N, Cout, H, W), 4).double()
        (gw,) = torch.autograd.grad(F.conv2d(x, w, padding=1), w, dy)
        dw = torch.empty(Cout, Cin, 3, 3, device='cuda')
        nb = _lib.query('hk_conv3x3_wgrad_workspace_bytes', Cin, Cout)
        ws = torch.empty(nb, dtype=torch.uint8, device='cuda')
        _lib.call('hk_conv3x3_wgrad', nhwc(x.float()).cuda(), nhwc(dy.float()).cuda(), dw, None, N, H, W, Cin, Cout, ws, nb, s)
        e = rel_l2(dw.cpu(), gw)
        print('wgrad', H, W, e)
        assert e < 2e-3


@pytest.mark.parametrize('P,K,Cout', [(100, 64, 128),      # one K split: the GEMM writes dw directly
                                      (1568, 64, 128),     # 16 splits and their reduction
                                      (2048, 160, 64)])    # the stem's im2col width
def test_matconv_wgrad(P, K, Cout):
    from hawkeye_b200 import _lib
    s = _lib.stream_ptr()
    x = detgen.det((P, K), 1)
    dy = detgen.det((P, Cout), 2)
    dw = torch.empty(Cout, K, device='cuda')
    nb = _lib.query('hk_matconv_wgrad_workspace_bytes', P, K, Cout)
    ws = torch.empty(nb, dtype=torch.uint8, device='cuda')
    _lib.call('hk_matconv_wgrad', x.cuda(), dy.cuda(), dw, P, K, Cout, ws, nb, s)
    e = rel_l2(dw.cpu(), dy.double().t() @ x.double())
    print('matconv wgrad', P, K, Cout, e)
    assert e < 2e-3


def _mpn_and_state():
    import hawkeye_b200 as hb

    class Cfg(dict):
        __getattr__ = dict.__getitem__
    net = hb.MODEL.get('MPN')(Cfg(name='MPN', iter_num=5, is_sqrt=True, is_vec=True, input_dim=2048,
                                  dimension_reduction=256, num_classes=200))
    st = detgen.state_like(net)
    net.load_state_dict(st)
    return net.cuda().train(), st


def test_resnet_units_vs_oracle():
    """Every conv+BN(+residual)+ReLU unit of the trunk, fed the ORACLE's input for that unit, matches the oracle's
    output to TF32 accuracy (<= 2e-3).  (End to end, a random-weight train-mode ResNet-50 amplifies any perturbation
    by ~1.3x per bottleneck — 5e-4 of TF32 rounding at layer1 is 8e-2 after 16 blocks — so parity is asserted per unit.)"""
    from hawkeye_b200 import _lib
    from oracle import hop_oracle as O
    torch.set_num_threads(16)
    net, st = _mpn_and_state()
    std = {k: v.double() for k, v in st.items()}
    plan = net.backbone._plan
    x = detgen.det((4, 3, 128, 128), 51)

    def dev(t):
        return t.float().permute(0, 2, 3, 1).contiguous().cuda()

    def rel(a, b):
        return rel_l2(a.permute(0, 3, 1, 2).cpu(), b)
    P = lambda u: list(u.params())
    y, _ = plan.stem.forward(x.cuda(), *P(plan.stem), None, False, True)
    ocur = F.relu(O._bn_train(F.conv2d(x.double(), std['backbone.0.weight'], stride=2, padding=3), std, 'backbone.1'))
    worst = rel(y, ocur)
    ocur = F.max_pool2d(ocur, 3, 2, 1)
    bi = 0
    for li, (planes, blocks, stride) in enumerate(O.RESNET50_LAYERS):
        for b in range(blocks):
            u1, u2, u3, ds = plan.blocks[bi]
            bi += 1
            pre, sb = f'backbone.{4 + li}.{b}', (stride if b == 0 else 1)
            o1 = F.relu(O._bn_train(F.conv2d(ocur, std[pre + '.conv1.weight']), std, pre + '.bn1'))
            o2 = F.relu(O._bn_train(F.conv2d(o1, std[pre + '.conv2.weight'], stride=sb, padding=1), std, pre + '.bn2'))
            oid = ocur
            if ds is not None:
                oid = O._bn_train(F.conv2d(ocur, std[pre + '.downsample.0.weight'], stride=sb), std, pre + '.downsample.1')
            o3 = F.relu(O._bn_train(F.conv2d(o2, std[pre + '.conv3.weight']), std, pre + '.bn3') + oid)
            a1, _ = u1.forward(dev(ocur), *P(u1), None, False, True)
            a2, _ = u2.forward(dev(o1), *P(u2), None, False, True)
            errs = [rel(a1, o1), rel(a2, o2)]
            idn = dev(oid)
            if ds is not None:
                idn_ours, _ = ds.forward(dev(ocur), *P(ds), None, False, True)
                errs.append(rel(idn_ours, oid))
            out, _ = u3.forward(dev(o2), *P(u3), idn, False, True)
            errs.append(rel(out, o3))
            worst = max(worst, max(errs))
            assert max(errs) < 2e-3, (pre, errs)
            ocur = o3
    print('resnet units worst rel', worst)


def test_mpn_model_matches_reference():
    from hawkeye_b200 import ops
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'reference_mpn.npz'))
    net, _ = _mpn_and_state()
    x = detgen.det((4, 3, 128, 128), 51).cuda()
    labels = detgen.det_labels(4, 200, 52).cuda()
    feat = net.backbone(x)
    ef = rel_l2(feat.detach().cpu()[:, ::16], g['feat_slice'])
    logits = net(x)
    loss = ops.CrossEntropyLS(0.1)(logits, labels)
    loss.backward()
    el = rel_l2(logits.detach().cpu(), g['logits'])
    errs = {'cls_b': rel_l2(net.classifier.bias.grad.cpu(), g['g_classifier_bias']),
            'dr_conv': rel_l2(net.pool.conv_dr_block[0].weight.grad.cpu()[:, ::8, 0, 0], g['g_dr_conv']),
            'l4_bn3_w': rel_l2(net.backbone[7][2].bn3.weight.grad.cpu(), g['g_layer4_bn3_w']),
            'stem_w': rel_l2(net.backbone[0].weight.grad.cpu(), g['g_stem_w'])}
    print(f'mpn: feat {ef:.2e} logits {el:.2e} loss {loss.item():.6f} vs {float(g["loss"]):.6f}', {k: f'{v:.1e}' for k, v in errs.items()})
    # end-to-end drift of a random-weight train-mode ResNet-50 under TF32 (see test_resnet_units_vs_oracle): sanity bounds
    assert ef < 0.2 and el < 0.2 and abs(loss.item() - float(g['loss'])) < 2e-2
    assert errs['cls_b'] < 5e-3 and all(torch.isfinite(p.grad).all() for p in net.parameters())
    assert int(net.backbone[1].num_batches_tracked) == 2
