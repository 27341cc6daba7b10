"""S3N on the device: each hk_s3n_* kernel and hk_stem_dgrad against fp64 (oracle/s3n_oracle.py, conv_transpose2d) at the
workload's shapes (448x448, batch 8, 200 classes, both decision-map branches) and at the fixture shapes, the sampler on the
reference's own class response maps against its fixtures for p = 0, 1, 2, the sampler chain's gradients, the trunk's image
gradient against torchvision's ResNet-50 in fp64, the full model against the reference's fixtures (radius, radius_inv and
filter from the model's own image gradient), the reference checkpoint in eval mode, CUDA-graph replay across p = 0, 1, 2,
and one S3NTrainer epoch with no host synchronisation in the step.  Precise mode unless stated."""
import contextlib
import json

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import detgen
from conftest import load_golden, rel_l2
from oracle import s3n_oracle as O
from kernel_check import precise_on  # noqa: F401  (a fixture)
from step_check import capture, make_trainer, no_host_sync, side_stream

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures('precise_on')]
GG = 31 * 31
CFG = dict(num_classes=200, image_size=128, radius=0.12, radius_inv=0.3, base_ratio=0.09)
SAMPLER_PARAMS = ('radius.scale', 'radius_inv.scale', 'filter.weight')


class Cfg(dict):
    __getattr__ = dict.__getitem__


def gaussian_filter():
    from hawkeye_b200.methods.s3n import make_gaussian
    return torch.from_numpy(make_gaussian(61, 13)).float().reshape(1, 1, 61, 61)


def run_sampler(crm_nhwc, p, rnd, radius=0.12, radius_inv=0.3):
    from hawkeye_b200 import ops_s3n
    r = torch.tensor([radius], device='cuda', requires_grad=True)
    ri = torch.tensor([radius_inv], device='cuda', requires_grad=True)
    pt = torch.tensor([p], device='cuda', dtype=torch.int32)
    maps, rec = ops_s3n.sample_maps(crm_nhwc.cuda(), rnd.cuda(), pt, r, ri, 0.09)
    return maps, rec, r, ri


def workload_maps(N, K, seed):
    """N class response maps of a 14x14 layer4 map (NHWC): every other image scaled by 20, so that the spatial means' softmax
    is nearly flat on half the images (gate > -0.2: the top-1 map decides) and spread over a few classes on the others
    (gate <= -0.2: the mean of the top-5 maps decides)."""
    crm = detgen.det((N, 14, 14, K), seed) * torch.tensor([1.0, 20.0] * (N // 2)).view(N, 1, 1, 1)
    _, _, gate = O.decision_maps(O.interpolate_maps(crm.permute(0, 3, 1, 2)))
    assert (gate > -0.2).any() and (gate <= -0.2).any()
    return crm


def oracle_sampler(crm_nchw, p, draws, radius=0.12, radius_inv=0.3):
    dms, _, _ = O.decision_maps(O.interpolate_maps(crm_nchw))
    r = torch.tensor([radius], dtype=torch.float64, requires_grad=True)
    ri = torch.tensor([radius_inv], dtype=torch.float64, requires_grad=True)
    xs, xs_inv, recs = O.sampling_maps(dms, p, r, ri, 0.09, draws)
    return xs, xs_inv, recs, r, ri


def check_peaks(rec, recs):
    peaks, scores, counts = (t.cpu() for t in rec)
    for n, (pos, score, zoom, inv) in enumerate(recs):
        c = int(counts[n])
        assert (peaks[n, :c] & 0xffff).tolist() == pos.tolist()
        flags = (peaks[n, :c] >> 16).tolist()
        assert flags == [int(z) | 2 * int(i) for z, i in zip(zoom, inv)]
        assert torch.allclose(scores[n, :c].double(), score, rtol=0, atol=1e-5)


@pytest.mark.parametrize('p', [0, 1, 2])
def test_sample_maps_against_oracle_at_448(p):
    """Batch 8, a 14x14 layer4 map, 200 classes, both decision-map branches: peaks, their assignment, both maps and
    dradius, dradius_inv."""
    N, K = 8, 200
    crm = workload_maps(N, K, 7000 + p)
    rnd = torch.rand(N, GG, generator=torch.Generator().manual_seed(7010 + p))
    maps, rec, r, ri = run_sampler(crm, p, rnd)
    xs, xs_inv, recs, rd, rid = oracle_sampler(crm.permute(0, 3, 1, 2), p, rnd.double().numpy())
    check_peaks(rec, recs)
    ref = torch.cat([xs, xs_inv])
    assert (maps.detach().cpu().reshape(2 * N, GG).double() - ref.detach()).abs().max() < 1e-5 * ref.detach().abs().max()
    g = detgen.det((2 * N, 31, 31), 7020 + p).cuda()
    maps.backward(g)
    ref.backward(g.cpu().double().reshape(2 * N, GG))
    for got, want in ((r.grad, rd.grad), (ri.grad, rid.grad)):
        assert abs(got.item() - want.item()) <= 1e-4 * max(abs(want.item()), 1e-3)


@pytest.mark.parametrize('p', [0, 1, 2])
def test_sample_maps_on_reference_maps(p):
    """The reference's own class response maps (its fixtures, 128x128 images): the same peaks, xs and xs_inv to fp32
    rounding; for p = 1 the reference's draws are placed at their peaks' positions."""
    g = load_golden(f'reference_s3n.{p}')
    crm = torch.from_numpy(g['crm'])
    N = crm.shape[0]
    rnd = torch.full((N, GG), 2.0)
    if p == 1:
        rnd[torch.from_numpy(g['draw_image']), torch.from_numpy(g['draw_pos'])] = torch.from_numpy(g['draw_value']).float()
    maps, rec, _, _ = run_sampler(crm.permute(0, 2, 3, 1).contiguous(), p, rnd)
    peaks, _, counts = (t.cpu() for t in rec)
    for n in range(N):
        ref = g[f'peaks_{n}']
        assert (peaks[n, :int(counts[n])] & 0xffff).tolist() == (ref[:, 0] * 31 + ref[:, 1]).tolist()
    m = maps.detach().cpu().reshape(2 * N, GG).numpy()
    np.testing.assert_allclose(m[:N], g['xs'], rtol=2e-6, atol=2e-6)
    np.testing.assert_allclose(m[N:], g['xs_inv'], rtol=2e-6, atol=2e-6)


@pytest.mark.parametrize('B', [4, 16])
def test_grid_against_oracle(B):
    from hawkeye_b200 import ops_s3n
    maps = (0.09 + detgen.det((B, 31, 31), 7100 + B).abs()).cuda().requires_grad_(True)
    filt = (gaussian_filter() * (1 + 0.1 * detgen.det((1, 1, 61, 61), 7101))).cuda().requires_grad_(True)
    grid = ops_s3n.GridFn.apply(maps, filt)
    md, fd = maps.detach().cpu().double().requires_grad_(True), filt.detach().cpu().double().requires_grad_(True)
    ref = O.coarse_grid(md, fd[0, 0])
    assert (grid.detach().cpu().double() - ref.detach()).abs().max() < 1e-5
    g = detgen.det((B, 31, 31, 2), 7102).cuda()
    grid.backward(g)
    ref.backward(g.cpu().double())
    assert rel_l2(maps.grad.cpu(), md.grad) < 1e-5
    assert rel_l2(filt.grad.cpu(), fd.grad) < 1e-5


def clean_affine_grid(B, size, seed):
    """A coarse grid whose upsampled sample coordinates all stay >= 1e-4 from an integer (the grid gradient of bilinear
    sampling jumps there): per image an affine map x -> a x + c, searched from ``seed``."""
    rng = np.random.RandomState(seed)
    lin = np.linspace(-1, 1, 31)
    out = np.zeros((B, 31, 31, 2))
    o = np.arange(size) * (30.0 / (size - 1)) / 30.0 * 2 - 1       # the fine positions in [-1, 1]
    for b in range(B):
        for comp in range(2):
            while True:
                a, c = rng.uniform(0.5, 0.95), rng.uniform(-0.05, 0.05)
                coords = ((a * o + c) + 1) / 2 * (size - 1)
                if np.abs(coords - np.round(coords)).min() > 2e-4:
                    break
            v = a * lin + c
            out[b, :, :, comp] = v[None, :] if comp == 0 else v[:, None]
    return torch.from_numpy(out).float()


@pytest.mark.parametrize('N,size', [(8, 448), (2, 128)])
def test_warp_against_oracle(N, size):
    from hawkeye_b200 import ops_s3n
    x = detgen.det((N, 3, size, size), 7200 + N)
    grid = clean_affine_grid(2 * N, size, 7201).cuda().requires_grad_(True)
    out = ops_s3n.WarpFn.apply(x.cuda(), grid)
    gd = grid.detach().cpu().double().requires_grad_(True)
    ref = O.warp(x, gd)
    # the fp32 upsampled grid is exact to ~6e-8 of [-1, 1], ~1e-5 pixel at 448: on a noise image up to ~1e-4 per sample
    assert (out.detach().cpu().double() - ref.detach()).abs().max() < 1e-3
    g = detgen.det(out.shape, 7202).cuda()
    out.backward(g)
    ref.backward(g.cpu().double())
    assert rel_l2(grid.grad.cpu(), gd.grad) < 1e-4


@pytest.mark.parametrize('p', [0, 1, 2])
def test_sampler_chain_gradients(p):
    """The sampler, the grid and the warp composed at 448x448, batch 8, 200 classes, from a fixed gradient at the sampled
    images: the coarse grid's gradient against fp64 autograd through the oracle's warp at the kernels' own grid, and from
    that gradient dradius, dradius_inv and dfilter through the oracle's maps and grid.  (Each stage starts from the device's
    values: the warp's grid gradient jumps where a sample coordinate crosses an integer, which the clamp at +-1 makes
    common, so an fp64 grid a rounding away would land on the other side.)"""
    from hawkeye_b200 import ops_s3n
    N, K = 8, 200
    crm = workload_maps(N, K, 7600 + p)
    rnd = torch.rand(N, GG, generator=torch.Generator().manual_seed(7610 + p))
    x = detgen.det((N, 3, 448, 448), 7620)
    gout = detgen.det((2 * N, 3, 448, 448), 7621)
    maps, _, r, ri = run_sampler(crm, p, rnd)
    filt = gaussian_filter().cuda().requires_grad_(True)
    grid = ops_s3n.GridFn.apply(maps, filt)
    grid.retain_grad()
    ops_s3n.WarpFn.apply(x.cuda(), grid).backward(gout.cuda())
    gd = grid.detach().cpu().double().requires_grad_(True)
    O.warp(x, gd).backward(gout.double())
    assert rel_l2(grid.grad.cpu(), gd.grad) < 1e-2         # the fp32 upsample of a grid clamped at 1 may land at 447 - 2e-5
    xs, xs_inv, _, rd, rid = oracle_sampler(crm.permute(0, 3, 1, 2), p, rnd.double().numpy())
    fd = gaussian_filter().double().requires_grad_(True)
    O.coarse_grid(torch.cat([xs, xs_inv]), fd[0, 0]).backward(grid.grad.cpu().double())
    for got, want in ((r.grad, rd.grad), (ri.grad, rid.grad)):
        assert abs(got.item() - want.item()) <= 1e-3 * abs(want.item()) + 1e-6
    # the clamp passes a grid position's gradient only inside [-1, 1]: positions a rounding away from a bound may differ
    assert rel_l2(filt.grad.cpu(), fd.grad) < 3e-2


def test_stem_dgrad_against_conv_transpose():
    from hawkeye_b200 import _lib
    N, H = 8, 448
    Ho = H // 2
    dc = detgen.det((N, Ho, Ho, 64), 7300).cuda()
    w = detgen.det((64, 3, 7, 7), 7301, 0.05).cuda()
    dx = torch.empty(N, 3, H, H, device='cuda')
    _lib.call('hk_stem_dgrad', dc, w, dx, N, H, H, _lib.stream_ptr())
    ref = F.conv_transpose2d(dc.cpu().double().permute(0, 3, 1, 2), w.cpu().double(), stride=2, padding=3,
                             output_padding=1)
    assert ref.shape == dx.shape
    assert (dx.cpu().double() - ref).abs().max() < 1e-5 * ref.abs().max()


def test_trunk_image_gradient_against_fp64():
    """ResNetTrunkFn's gradient at its input image (the stem's BatchNorm and ReLU backward, then hk_stem_dgrad, after the
    max-pool and every block) against fp64 autograd through torchvision's ResNet-50 with the same weights, train mode,
    two 128x128 images."""
    import torchvision
    from hawkeye_b200 import ops_resnet
    net = fixture_model()
    x = detgen.det((2, 3, 128, 128), 7350).cuda().requires_grad_(True)
    net.zero_grad()
    y = ops_resnet.resnet_trunk(x, net._plan, True)                        # NHWC [2, 4, 4, 2048]
    g = detgen.det(tuple(y.shape), 7351).cuda()
    y.backward(g)
    tv = torchvision.models.resnet50()
    tv.load_state_dict({k: v.cpu() for k, v in net.backbone.state_dict().items()})
    tv = tv.double().train()
    xd = x.detach().cpu().double().requires_grad_(True)
    yd = torch.nn.Sequential(*list(tv.children())[:-2])(xd)
    assert rel_l2(y.detach().cpu().permute(0, 3, 1, 2), yd.detach()) < 5e-4     # 3xTF32 products through 53 convs
    yd.backward(g.cpu().double().permute(0, 3, 1, 2))
    # dx and conv1's weight gradient are both read from the stem's dc: a dc taken at the wrong point (before the BN or ReLU
    # backward, or in another layout) would leave dw right and dx wrong.  Both carry the drift the train-mode backward
    # through 16 blocks accumulates at this size, so dx is held to the error of dw.
    e_dx = rel_l2(x.grad.cpu(), xd.grad)
    e_dw = rel_l2(net.backbone.conv1.weight.grad.cpu(), tv.conv1.weight.grad)
    print('trunk image gradient: rel dx', e_dx, 'rel dconv1', e_dw)
    assert e_dw < 0.1 and e_dx < 2 * e_dw + 1e-3


def fixture_model():
    import hawkeye_b200 as hb
    net = hb.MODEL.get('S3N')(Cfg(CFG))
    state = detgen.state_like(net)
    for k in ('radius.scale', 'radius_inv.scale', 'filter.weight'):
        state[k] = net.state_dict()[k].clone()
    net.load_state_dict(state)
    return net.cuda().train()


@pytest.mark.parametrize('p', [0, 2])
def test_model_against_reference_fixture(p):
    """The reference's end-to-end run (train mode): the raw branch, the class response maps, the two sampling maps, the four
    outputs, the loss and the sampled gradients.  p = 1 draws on the device and is
    covered at the sampler.  The sampled images feed a randomly initialised trunk with BatchNorm over 2 x 2 maps of two
    images, which moves its output by ~1e3 times a relative change of its input: the maps agree to ~1e-5 (the class
    response maps' own drift), the zoom and complementary branches' outputs to a few percent, and the gradients that flow
    through them to tens of percent.  So radius, radius_inv and filter are checked downstream of the model's own sampled
    images: from the gradient the trunk returns there to the three parameters, against fp64 autograd."""
    from hawkeye_b200 import ops_s3n
    from hawkeye_b200.losses import MultiSmoothLoss
    g = load_golden(f'reference_s3n.{p}')
    net = fixture_model()
    x = detgen.det((2, 3, 128, 128), 5100).cuda()
    labels = torch.from_numpy(g['labels']).cuda()
    seen, orig, grid_apply, warp_apply = {}, ops_s3n.sample_maps, ops_s3n.GridFn.apply, ops_s3n.WarpFn.apply

    def record(crm, rnd, *a):
        maps, rec = orig(crm, rnd, *a)
        seen['crm'], seen['rnd'], seen['maps'] = crm.detach().cpu(), rnd.cpu(), maps.detach().cpu().reshape(4, -1)
        return maps, rec

    def keep(name, fn):
        def apply(*a):
            out = fn(*a)
            out.retain_grad()
            seen[name] = out
            return out
        return apply
    monkey = pytest.MonkeyPatch()
    monkey.setattr(ops_s3n, 'sample_maps', record)
    monkey.setattr(ops_s3n.GridFn, 'apply', keep('grid', grid_apply))
    monkey.setattr(ops_s3n.WarpFn, 'apply', keep('sampled', warp_apply))
    try:
        outputs = net(x, p)
    finally:
        monkey.undo()
    loss = MultiSmoothLoss(Cfg(smooth_ratio=0.85))(outputs, labels)
    loss.backward()
    assert rel_l2(seen['crm'].permute(0, 3, 1, 2), torch.from_numpy(g['crm'])) < 1e-3
    assert rel_l2(seen['maps'][:2], torch.from_numpy(g['xs'])) < 1e-4
    assert rel_l2(seen['maps'][2:], torch.from_numpy(g['xs_inv'])) < 1e-4
    assert rel_l2(outputs[1].detach().cpu(), torch.from_numpy(g['agg_origin'])) < 1e-3
    for name, o in zip(('aggregation', 'agg_sampler', 'agg_sampler1'), (outputs[0], outputs[2], outputs[3])):
        assert rel_l2(o.detach().cpu(), torch.from_numpy(g[name])) < 0.1, name
    assert abs(loss.item() - float(g['loss'])) < 1e-2 * abs(float(g['loss']))
    params = dict(net.named_parameters())
    # radius, radius_inv and filter from the model's own gradient at the sampled images (the trunk's image gradient,
    # test_trunk_image_gradient_against_fp64): the grid gradient through the oracle's warp at the model's grid, then fp64
    # autograd through the oracle's sampler on the model's class response maps and draws
    gd = seen['grid'].detach().cpu().double().requires_grad_(True)
    O.warp(x.cpu(), gd).backward(seen['sampled'].grad.cpu().double())
    assert rel_l2(seen['grid'].grad.cpu(), gd.grad) < 3e-2          # jumps at integer sample coordinates, as in the chain
    xs, xs_inv, _, rd, rid = oracle_sampler(seen['crm'].permute(0, 3, 1, 2), p, seen['rnd'].double().numpy())
    fd = gaussian_filter().double().requires_grad_(True)
    O.coarse_grid(torch.cat([xs, xs_inv]), fd[0, 0]).backward(seen['grid'].grad.cpu().double())
    for k, want in (('radius.scale', rd.grad), ('radius_inv.scale', rid.grad)):
        assert abs(params[k].grad.item() - want.item()) <= 1e-3 * abs(want.item()) + 1e-6, k
    assert rel_l2(params['filter.weight'].grad.cpu(), fd.grad) < 3e-2
    for i, k in enumerate(json.loads(bytes(g['grad_names']).decode())):
        if k in SAMPLER_PARAMS:
            continue
        got = params[k].grad.flatten()[torch.from_numpy(g[f'grad_{i}_idx']).cuda()].cpu()
        want = torch.from_numpy(g[f'grad_{i}'])
        assert (rel_l2(got, want) < 0.5) if want.abs().max() > 0 else got.abs().max() == 0, (k, rel_l2(got, want))


def test_reference_checkpoint_eval_outputs():
    """The reference's checkpoint (its state_dict of the fixture run, rebuilt from the same seeds) loads strictly, and the
    eval-mode outputs at p = 2 (running statistics as loaded, no draws) match the reference's."""
    import hawkeye_b200 as hb
    g = load_golden('reference_s3n.2')
    ref_net = fixture_model()
    ck = {k: v.detach().cpu().clone() for k, v in ref_net.state_dict().items()}
    assert list(ck) == json.loads(bytes(g['state_keys_json']).decode())
    net = hb.MODEL.get('S3N')(Cfg(CFG))
    net.load_state_dict(ck, strict=True)
    net = net.cuda().eval()
    with torch.no_grad():
        out = net(detgen.det((2, 3, 128, 128), 5100).cuda(), 2)
    errs = {name: rel_l2(o.cpu(), torch.from_numpy(g['eval_' + name]))
            for name, o in zip(('aggregation', 'agg_origin', 'agg_sampler', 'agg_sampler1'), out)}
    # the raw branch directly; the sampled branches move with their inputs as in test_model_against_reference_fixture
    assert errs['agg_origin'] < 1e-3 and max(errs.values()) < 0.1, errs


def test_graph_replay_matches_eager_across_p(monkeypatch):
    """One capture of forward, loss and backward (default TF32 mode, as the trainer replays it) serves p = 0, 1 and 2: the
    replay gives the eager step's outputs, loss and sampler gradients bit for bit.  Eager and replay use the same draws:
    the sampler reads them from one static buffer (a replay otherwise draws anew, as it should in training)."""
    from hawkeye_b200 import _lib, ops_s3n
    from hawkeye_b200.losses import MultiSmoothLoss
    _lib.set_precise(0)
    draws = torch.rand(2, GG, device='cuda', generator=torch.Generator('cuda').manual_seed(7501))
    orig = ops_s3n.sample_maps
    monkeypatch.setattr(ops_s3n, 'sample_maps', lambda crm, rnd, *a: orig(crm, draws, *a))
    net = fixture_model()
    crit = MultiSmoothLoss(Cfg(smooth_ratio=0.85))
    x = detgen.det((2, 3, 128, 128), 7500).cuda()
    labels = torch.tensor([3, 7], device='cuda')
    pt = torch.zeros(1, dtype=torch.int32, device='cuda')
    params = list(net.parameters())
    watched = (net.radius.scale, net.radius_inv.scale, net.filter.weight)

    def step():
        for q in params:
            q.grad = None
        out = net(x, pt)
        loss = crit(out, labels)
        loss.backward()
        return out, loss, [q.grad for q in watched]

    with side_stream() as s:
        for _ in range(2):
            step()
        state = {k: v.clone() for k, v in net.state_dict().items()}
        graph, (g_out, g_loss, g_grads) = capture(step)
        for p in (0, 1, 2):
            net.load_state_dict(state)
            pt.fill_(p)
            e_out, e_loss, e_grads = step()
            e_grads = [t.clone() for t in e_grads]
            net.load_state_dict(state)
            pt.fill_(p)
            graph.replay()
            s.synchronize()
            for a, b in zip(e_out, g_out):
                assert torch.equal(a, b)
            assert torch.equal(e_loss, g_loss)
            for a, b in zip(e_grads, g_grads):
                assert torch.equal(a, b)


def test_trainer_epoch_no_sync(tmp_path, monkeypatch):
    """One S3NTrainer epoch of six synthetic 448x448 batches with ``cuda_graph: true``: two eager steps, the capture, then
    replays, with the epoch moved to 20 before the last step so that p changes from 0 to 1 under replay.  The steps other
    than the capture run with no host synchronisation; every parameter the optimizer owns gets a gradient, the classifiers
    move, and validation (p = 2 from epoch 20) scores aggregation."""
    batches = [dict(img=detgen.det((4, 3, 448, 448), 7700 + i).pin_memory(),
                    label=detgen.det_labels(4, 200, 7710 + i).pin_memory()) for i in range(6)]
    val = [dict(img=detgen.det((4, 3, 448, 448), 7720), label=torch.zeros(4, dtype=torch.int64))]
    from hawkeye_b200 import _lib
    _lib.set_precise(0)
    tr = make_trainer(monkeypatch, 'S3N', 'S3N.yaml', graph=True, experiment=dict(log_dir=str(tmp_path)),
                      dataloaders={'train': batches, 'val': val})
    assert [g['lr'] for g in tr.optimizer.param_groups] == pytest.approx([0.005, 5e-8, 5e-8, 5e-4])
    w0 = tr.model.con_classifier.weight.detach().clone()
    tr.epoch = 0
    for i, data in enumerate(batches):
        if i == 5:
            tr.epoch = 20
        with no_host_sync() if i not in (0, 2) else contextlib.nullcontext():   # step 3 captures after its eager run
            tr.batch_training(data)
        if i == 1:                                   # p = 0: every peak feeds both maps, so every gradient is non-zero
            for g in tr.flat.groups:
                for q in g:
                    assert torch.isfinite(q.grad).all() and q.grad.abs().max() > 0
    assert tr._graph is not None and int(tr.p_train.item()) == 1
    assert not torch.equal(tr.model.con_classifier.weight, w0)
    assert np.isfinite(tr.average_meters['loss'].avg) and 0 <= tr.average_meters['acc'].avg <= 100
    tr.validate()
    assert 0 <= tr.average_meters['acc'].avg <= 100 and tr.average_meters['acc'].count == 4
