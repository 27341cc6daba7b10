"""Mixup / CutMix on the device (csrc/mixup.cu): hk_mix_batch bit for bit against the reference's fixtures, the soft-target
cross-entropy against an fp64 CrossEntropyLoss(label_smoothing=0.1) on the dense target, its top-1 count with ties, its
agreement with hk_softmax_ce_ls at w = 1, and the BCNN train step with ``dataset.mixup_cutmix`` under the host and the
device presets: graph replay against eager, no host synchronisation, and the device-preset batch mixed on the device
against the host preset mixed by the CPU restatement."""
import contextlib
import os
import random

import numpy as np
import pytest
import torch

import mixup_ref
from conftest import load_golden
from kernel_check import U, Bound, Out, abi, check
from hawkeye_b200 import data, ops_mixup as M
from step_check import no_host_sync

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def gold():
    return load_golden('reference_mixup')


def test_mix_batch_is_the_reference_bit_for_bit(gold):
    """Every fixture: Mixup, CutMix clipped at each border, an empty and a full box, B = 1, and the 50 collate batches
    (odd sizes: the scalar path; the 24 x 40 cases: the vector path).  The input is left unchanged."""
    batches = [(gold[f'case.{n}.img'], gold[f'case.{n}.draw'], gold[f'case.{n}.out'], n) for n in gold['case.names']]
    batches += [(gold[f'draws.img.{k}'], [gold['draws.kind'][k], gold['draws.lam'][k], *gold['draws.box'][k],
                                          gold['draws.weight'][k]], gold[f'draws.out.{k}'], f'draws {k}') for k in range(50)]
    for img, draw, want, name in batches:
        x = torch.from_numpy(img).cuda()
        row = torch.from_numpy(mixup_ref.row_of(draw)).cuda()
        (y,) = abi('hk_mix_batch', x, row, Out(x.shape), *x.shape, inputs=(x, row))
        assert y.cpu().numpy().tobytes() == want.tobytes(), name
        assert torch.equal(M.mix_batch(x, row), y)


B, K, EPS = 32, 200, 0.1
# The fp32 softmax of a row is off by at most about (2 |z - lse| + |max z| + K + 4) U relatively, some 250 U at these
# logits (|z| < 20); the worst measured on an H100 is 13 U on dlogits and 1.4 U on the loss, and C_CE sits about 5x
# above it.
C_CE = 64 * U


def _logits(seed):
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(B, K, generator=g) * 3
    labels = torch.randint(0, K, (B,), generator=g)
    labels[5] = labels[4]                      # a row whose partner has its own label
    return z, labels


def _fp64(z, labels, row):
    """loss, dlogits of CrossEntropyLoss(label_smoothing) on the reference's fp32 dense target, in fp64"""
    t = torch.from_numpy(mixup_ref.dense_target(labels.numpy(), row, K)).double()
    zd = z.double().requires_grad_()
    loss = torch.nn.functional.cross_entropy(zd, t, label_smoothing=EPS)
    loss.backward()
    return loss.detach(), zd.grad, t


ROWS = {'mixup': M.mix_row(M.MIXUP, 0.7321), 'cutmix': M.mix_row(M.CUTMIX, 0.41, (3, 5, 30, 20), 0.59),
        'tie': M.mix_row(M.MIXUP, 0.5), 'w0': M.mix_row(M.CUTMIX, 0.0, (0, 0, 40, 24), 0.0),
        'w1': M.mix_row(M.CUTMIX, 1.0, (7, 7, 7, 7), 1.0)}


@pytest.mark.parametrize('precise', [0, 1])
@pytest.mark.parametrize('name', list(ROWS))
def test_ce_mix_against_fp64(name, precise):
    """Loss and dlogits element by element against fp64: C_CE (p + target) / B on dlogits, plus the tf32 rounding on
    store in the default mode, and C_CE (max |lse| + loss) on the loss."""
    z, labels = _logits(1)
    row = ROWS[name].numpy()
    ref_loss, ref_d, t = _fp64(z, labels, row)
    zc, lc, mc = z.cuda(), labels.cuda(), torch.from_numpy(row).cuda()
    loss, dl, corr = abi('hk_softmax_ce_ls_mix', zc, lc, mc, Out((1,)), Out((B, K)), Out((1,), torch.int32), B, K, EPS,
                         1.0, inputs=(zc, lc, mc), precise=precise)
    p = torch.softmax(z.double(), 1)
    scale = (p + (1 - EPS) * t + EPS / K) / B
    check(dl.cpu(), ref_d, Bound(C_CE * scale, rounded=not precise), f'dlogits {name}', names=('row', 'class'))
    lse = torch.logsumexp(z.double(), 1).abs().max()
    check(loss.cpu(), ref_loss.reshape(1), Bound(C_CE * (lse + ref_loss.abs()).reshape(1)), f'loss {name}',
          names=('loss',))
    want = (torch.from_numpy(np.asarray(t, np.float32)).max(1)[1] == z.argmax(1)).sum()
    assert int(corr) == int(want)


def test_correct_follows_the_target_argmax_with_ties():
    """Logits whose top-1 is the current label, the rolled label or neither, under weights above, below and at 1/2: a
    row counts when its top-1 is the heavier label, and on a tie the lower class index — target.max(1)[1]."""
    labels = torch.tensor([3, 9, 1, 1, 7, 2, 8, 0])
    n = len(labels)
    prev = labels.roll(1)
    for w in (0.8, 0.2, 0.5):
        row = M.mix_row(M.MIXUP, w).numpy()
        target = torch.from_numpy(mixup_ref.dense_target(labels.numpy(), row, 12))
        for pick in ('cur', 'prev', 'other'):
            z = torch.zeros(n, 12)
            top = {'cur': labels, 'prev': prev, 'other': torch.full_like(labels, 11)}[pick]
            z[torch.arange(n), top] = 1.0
            zc = z.cuda()
            (_, _, corr) = abi('hk_softmax_ce_ls_mix', zc, labels.cuda(), torch.from_numpy(row).cuda(), Out((1,)),
                               Out((n, 12)), Out((1,), torch.int32), n, 12, EPS, 1.0)
            want = int((target.max(1)[1] == z.argmax(1)).sum())
            assert int(corr) == want, (w, pick)
    # the tie rule itself: weights 1/2 on labels 3 and 9 -> class 3; a top-1 at 9 does not count
    row = M.mix_row(M.MIXUP, 0.5).cuda()
    z = torch.zeros(2, 12)
    z[0, 9], z[1, 3] = 1.0, 1.0
    lab = torch.tensor([3, 9]).cuda()
    (_, _, corr) = abi('hk_softmax_ce_ls_mix', z.cuda(), lab, row, Out((1,)), Out((2, 12)), Out((1,), torch.int32), 2,
                       12, EPS, 1.0)
    assert int(corr) == 1            # row 0: target {3, 9} -> 3, top-1 9; row 1: target {9, 3} -> 3, top-1 3


@pytest.mark.parametrize('precise', [0, 1])
def test_weight_one_is_the_one_hot_loss(precise):
    """At w = 1 the soft target is the one-hot target of hk_softmax_ce_ls: the same loss, dlogits and count within the
    fp64 bound of test_ce_mix_against_fp64."""
    z, labels = _logits(2)
    zc, lc = z.cuda(), labels.cuda()
    row = ROWS['w1'].cuda()
    a = abi('hk_softmax_ce_ls_mix', zc, lc, row, Out((1,)), Out((B, K)), Out((1,), torch.int32), B, K, EPS, 1.0,
            precise=precise)
    b = abi('hk_softmax_ce_ls', zc, lc, Out((1,)), Out((B, K)), Out((1,), torch.int32), B, K, EPS, 1.0, precise=precise)
    _, _, t = _fp64(z, labels, ROWS['w1'].numpy())
    scale = (torch.softmax(z.double(), 1) + (1 - EPS) * t + EPS / K) / B
    check(a[1].cpu(), b[1].cpu().double(), Bound(C_CE * scale, rounded=not precise), 'dlogits w=1',
          names=('row', 'class'))
    lse = torch.logsumexp(z.double(), 1).abs().max()
    check(a[0].cpu(), b[0].cpu().double(), Bound(C_CE * (lse + b[0].cpu().double().abs())), 'loss w=1',
          names=('loss',))
    assert int(a[2]) == int(b[2])


def test_ce_mix_module_backward_and_last_correct():
    from hawkeye_b200 import ops
    z, labels = _logits(3)
    zc = z.cuda().requires_grad_()
    row = ROWS['cutmix'].cuda()
    crit = ops.CrossEntropyLSMix(EPS)
    loss = crit(zc, labels.cuda(), row)
    (loss * 2).backward()
    _, dl, _ = abi('hk_softmax_ce_ls_mix', zc.detach(), labels.cuda(), row, Out((1,)), Out((B, K)), Out((1,), torch.int32),
                   B, K, EPS, 1.0)
    assert torch.equal(zc.grad, dl * 2) and crit.last_correct.shape == (1,)


# ---- the train step ----------------------------------------------------------------------------------------------------
def write_jpeg(path, w, h, seed, quality=90):
    """A smooth random field with noise on top, saved as JPEG; -> the decoded RGB image (what the loader sees)."""
    from PIL import Image
    r = np.random.RandomState(seed)
    base = Image.fromarray(r.randint(0, 256, (max(h // 24, 2), max(w // 24, 2), 3)).astype(np.uint8))
    arr = np.asarray(base.resize((w, h), Image.BICUBIC)).astype(np.int32) + r.randint(-24, 25, (h, w, 3))
    Image.fromarray(np.clip(arr, 0, 255).astype(np.uint8)).save(path, quality=quality)
    return data.default_loader(path)


def _pinned(batch):
    return {k: (v.pin_memory() if hasattr(v, 'pin_memory') else v) for k, v in batch.items()}


def _jpegs(tmp_path):
    return [write_jpeg(str(tmp_path / f'{i}.jpg'), 500 if i % 3 else 375, 375 if i % 3 else 500, seed=300 + i)
            for i in range(16)]


def _batches(images, labels, S=448):
    """Four batches of four images under both presets, each batch drawn from one seed: the per-image draws and then the
    collate's, identical under both presets."""
    host = data.ClassificationPresetTrain(S, auto_augment_policy='ta_wide', random_erase_prob=0.1)
    dev = data.DevicePresetTrain(S, auto_augment_policy='ta_wide', random_erase_prob=0.1)
    mh, md = data.MixupCutmixCollateFn(200), data.MixupCutmixCollateFn(200, dev.collate)
    out = {'host': [], 'cuda': []}
    for b in range(4):
        for kind, tf, coll in (('host', host, mh), ('cuda', dev, md)):
            torch.manual_seed(40 + b)
            random.seed(40 + b)
            out[kind].append(_pinned(coll([{'img': tf(images[4 * b + i]), 'label': int(labels[4 * b + i])}
                                           for i in range(4)])))
        assert torch.equal(out['host'][-1]['mix'], out['cuda'][-1]['mix'])
    kinds = {int(x['mix'][M.KIND]) for x in out['host']}
    return out, kinds


def _trainer(monkeypatch, graph):
    from hawkeye_b200 import examples
    from hawkeye_b200.config import load_config
    monkeypatch.setenv('HAWKEYE_ALLOW_RANDOM_INIT', '1')
    monkeypatch.setenv('HK_CUDA_GRAPH', '1' if graph else '0')
    cfg = load_config(os.path.join(REPO, 'configs', 'BCNN_S2.yaml'))
    cfg.dataset['mixup_cutmix'] = True
    return examples.BCNNTrainer(cfg, dataloaders={})


def test_bcnn_step_with_mixup_cutmix(tmp_path, monkeypatch):
    """Eight BCNN 448 steps (four host-preset batches, then the same four under the device presets), eager and with graph
    replay from one state.  The staged images are the restatement of the host batch bit for bit (host presets) and
    within the device presets' bound of it (device presets); replay gives the eager images bit for bit and the eager
    losses within 2e-3; every step but the first and the capture raises nothing under sync debug mode 'error'."""
    from hawkeye_b200 import _lib, ops
    _lib.set_precise(0)
    images = _jpegs(tmp_path)
    batches, kinds = _batches(images, [(7 * i) % 200 for i in range(16)])
    seq = batches['host'] + batches['cuda']
    runs, state0 = {}, None
    for graph in (False, True):
        torch.manual_seed(0)
        tr = _trainer(monkeypatch, graph)
        assert tr.mixing and type(tr.criterion) is ops.CrossEntropyLSMix
        if state0 is None:
            state0 = {k: v.detach().clone() for k, v in tr.model.state_dict().items()}
        else:
            tr.model.load_state_dict(state0)
        stage, staged, losses = tr.stage_inputs, [], []

        def spy(batch):
            out = stage(batch)
            staged.append(out[0].clone())
            return out
        tr.stage_inputs = spy
        for i, b in enumerate(seq):
            with no_host_sync() if i not in (0, 2) else contextlib.nullcontext():
                losses.append(tr.batch_training(b).detach().clone())
        torch.cuda.synchronize()
        assert (tr._graph is not None) == graph and np.isfinite(tr.average_meters['loss'].avg)
        assert 0 <= tr.average_meters['acc'].avg <= 100
        runs[graph] = (torch.stack(staged).cpu(), [float(x) for x in losses])
        del tr
        torch.cuda.empty_cache()
    (ie, le), (ig, lg) = runs[False], runs[True]
    assert torch.equal(ie, ig)
    assert all(abs(a - b) < 2e-3 * max(1.0, abs(a)) for a, b in zip(le, lg)), (le, lg)
    for k, b in enumerate(batches['host']):
        want = mixup_ref.mix_images(b['img'].numpy(), b['mix'].numpy())
        assert ie[k].numpy().tobytes() == want.tobytes()
        diff = (ie[4 + k] - torch.from_numpy(want)).abs().max()
        # the device presets are within 4e-6 of the host presets (test_gpu_augment); a convex mix of two such images
        # keeps that, plus the fp32 rounding of the mix itself (a few ulp of values below 3)
        print(f'batch {k} (kind {int(b["mix"][M.KIND])}): device-preset mix against host restatement max |diff| {diff:.3e}')
        assert diff < 4e-6 + 8 * 2.0 ** -23 * 3
    print(f'kinds drawn: {sorted(kinds)}; losses eager {le}')
