"""The device presets (hawkeye_b200.ops_augment, csrc/augment.cu) against the host presets on the same uint8 images and
the same draws: the crop-resize bit for bit against PIL, every TrivialAugmentWide op at every magnitude bin and sign, the
erasing rectangle, the whole train and eval presets, a BCNN train step fed by the device presets (eager and graph
replay, no host synchronisation) and the Tester with both presets.  The images are synthetic JPEGs drawn from a seed."""
import contextlib
import os

import numpy as np
import pytest
import torch
from PIL import Image

import detgen
from conftest import rel_l2
from hawkeye_b200 import data, ops_augment as A
from step_check import no_host_sync

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
LSB = 1.0 / 255.0 / min(STD)          # one uint8 step in normalised units, for the channel with the smallest std


def write_jpeg(path, w, h, seed, quality=90):
    """A smooth random field with noise on top, saved as JPEG; -> the decoded RGB image (what the loader sees)."""
    r = np.random.RandomState(seed)
    base = Image.fromarray(r.randint(0, 256, (max(h // 24, 2), max(w // 24, 2), 3)).astype(np.uint8))
    arr = np.asarray(base.resize((w, h), Image.BICUBIC)).astype(np.int32) + r.randint(-24, 25, (h, w, 3))
    Image.fromarray(np.clip(arr, 0, 255).astype(np.uint8)).save(path, quality=quality)
    return data.default_loader(path)


def run(images, rows, S, chunk=64):
    """-> (uint8 crop-resize output [N, S, S, 3], fp32 model input [N, 3, S, S]) on the host."""
    works, outs = [], []
    for c in range(0, len(images), chunk):
        p = A.pack([np.asarray(i) for i in images[c:c + chunk]], rows[c:c + chunk], S, MEAN, STD).to('cuda')
        work = torch.empty(len(p), S, S, 3, dtype=torch.uint8, device='cuda')
        out = p.images(work=work)
        works.append(work.cpu())
        outs.append(out.cpu())
    return torch.cat(works).numpy(), torch.cat(outs)


def to_u8(out):
    """The uint8 image behind a normalised fp32 output (exact: one step is 70x the arithmetic's error)."""
    m, s = torch.tensor(MEAN).view(1, 3, 1, 1), torch.tensor(STD).view(1, 3, 1, 1)
    return torch.round((out * s + m) * 255).clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1).numpy()


@pytest.fixture(scope='module')
def jpegs(tmp_path_factory):
    root = tmp_path_factory.mktemp('jpegs')
    sizes = [(500, 375), (375, 500), (500, 333), (333, 500), (500, 500), (420, 300), (1000, 96), (64, 700)]
    return [write_jpeg(str(root / f'{i}.jpg'), *sizes[i % len(sizes)], seed=i) for i in range(16)]


def test_crop_resize_is_pil_bit_for_bit(jpegs):
    """RandomResizedCrop's crop + resize and Resize + CenterCrop against torchvision on the PIL image, with and without
    the flip: downscales, upscales, extreme aspect ratios, 1-pixel boxes."""
    from torchvision.transforms import functional as F
    from torchvision.transforms.functional import InterpolationMode
    img = jpegs[0]                                          # 500 x 375
    tall = jpegs[7]                                         # 64 x 700
    cases = []                                              # (name, image, row, PIL reference)
    for name, im, (x, y, w, h), S in [('whole down', img, (0, 0, 500, 375), 448), ('whole down 64', img, (0, 0, 500, 375), 64),
                                      ('up', img, (37, 51, 45, 38), 448), ('mixed', img, (3, 0, 480, 20), 448),
                                      ('1px wide', img, (100, 10, 1, 300), 448), ('1px high', img, (10, 100, 400, 1), 448),
                                      ('1x1', img, (499, 374, 1, 1), 448), ('same width', img, (0, 5, 448, 300), 448),
                                      ('same size', img, (20, 30, 64, 64), 64), ('tall', tall, (0, 0, 64, 700), 448),
                                      ('strong down', tall, (0, 0, 64, 700), 16)]:
        ref = np.asarray(F.resized_crop(im, y, x, h, w, [S, S], InterpolationMode.BILINEAR))
        for flip in (False, True):
            cases.append((f'{name}{" flip" if flip else ""}', im, S, A.param_row((x, y, w, h), (S, S), flip=flip),
                          ref[:, ::-1] if flip else ref))
    for name, im, resize, S in [('eval 512/448', img, 512, 448), ('eval tall', jpegs[1], 512, 448),
                                ('eval down', img, 64, 56), ('eval pad', img, 40, 56), ('eval 1000x96', jpegs[6], 512, 448)]:
        row = data.DevicePresetEval(S, resize_size=resize).draw(im)
        cases.append((name, im, S, row, np.asarray(F.center_crop(F.resize(im, resize), S))))
    worst = []
    for name, im, S, row, ref in cases:
        work, _ = run([im], [row], S)
        d = np.abs(work[0].astype(int) - ref.astype(int))
        worst.append((int(d.max()), int((d > 0).sum()), name))
    print('crop-resize vs PIL, (max |diff|, differing values, case):', sorted(worst, reverse=True)[:3])
    assert all(w[0] == 0 for w in worst), worst


def _bases(jpegs):
    """448 x 448 uint8 images: a natural one, a low-contrast one and one with a handful of levels (ImageOps edge cases)."""
    nat = np.asarray(jpegs[0].resize((448, 448), Image.BILINEAR))
    low = (60 + nat.astype(np.int32) * 60 // 255).astype(np.uint8)
    few = (nat // 64 * 64).astype(np.uint8)
    few[..., 2] = 17                                        # a constant channel: AutoContrast / Equalize leave it alone
    return [Image.fromarray(a) for a in (nat, low, few)]


def test_every_trivial_augment_op_at_every_bin_and_sign(jpegs):
    """Each op of TrivialAugmentWide at each of its 31 magnitudes (and both signs where it has one) against torchvision's
    PIL implementation on the same uint8 448 image.  The bounds are 1 LSB everywhere for the photometric ops and 99.9 % of
    the values within 1 LSB for the geometric ones; the kernels follow PIL's arithmetic, so every op is held to
    identical results."""
    from torchvision.transforms import autoaugment
    from torchvision.transforms.functional import InterpolationMode
    space = autoaugment.TrivialAugmentWide()._augmentation_space(31)
    bases = _bases(jpegs)
    cases = []
    for name, (mags, signed) in space.items():
        values = [float(m) for m in mags.reshape(-1)] if mags.ndim > 0 else [0.0]
        for v in values:
            for sign in ((1.0, -1.0) if signed else (1.0,)):
                for b, im in enumerate(bases):
                    if b and name in A.GEOMETRIC and v not in (values[-1], values[len(values) // 2]):
                        continue                            # geometry does not depend on the content: fewer cases
                    cases.append((name, v * sign, b, im))
    report = {}
    for c in range(0, len(cases), 64):
        chunk = cases[c:c + 64]
        rows = [A.param_row((0, 0, 448, 448), (448, 448), op=n, magnitude=m, size=448) for n, m, _, _ in chunk]
        got = to_u8(run([im for _, _, _, im in chunk], rows, 448)[1])
        for k, (name, m, b, im) in enumerate(chunk):
            ref = np.asarray(autoaugment._apply_op(im, name, m, InterpolationMode.BILINEAR, None)).astype(int)
            d = np.abs(got[k].astype(int) - ref)
            r = report.setdefault(name, [0, 1.0, 0])
            r[0] = max(r[0], int(d.max()))
            r[1] = min(r[1], float((d <= 1).mean()))
            r[2] += int((d > 0).sum())
    for name, (mx, within, ndiff) in report.items():
        print(f'{name:13s} max |diff| {mx:3d}  worst fraction within 1 LSB {within:.6f}  differing values {ndiff}')
    for name, (mx, within, _) in report.items():       # the bounds; the arithmetic is PIL's, and the result identical
        assert (within >= 0.999) if name in A.GEOMETRIC else (mx <= 1), (name, mx, within)
        assert mx == 0, (name, mx)


def test_erasing_rectangle_and_value_are_exact(jpegs):
    from hawkeye_b200.test import normalize_u8
    S = 64
    rects = [(0, 0, 5, 7), (60, 50, 4, 14), (10, 0, 1, 64), (0, 33, 64, 1), (20, 21, 22, 23), None]
    rows = [A.param_row((0, 0, 500, 375), (S, S), erase=r) for r in rects]
    work, out = run([jpegs[0]] * len(rects), rows, S)
    plain = normalize_u8(torch.from_numpy(work).cuda()).cpu()
    for k, r in enumerate(rects):
        mask = torch.zeros(S, S, dtype=torch.bool)
        if r is not None:
            i, j, h, w = r
            mask[i:i + h, j:j + w] = True
        assert (out[k][:, mask] == 0).all() and not (plain[k][:, mask] == 0).any()
        assert torch.equal(out[k][:, ~mask], plain[k][:, ~mask])


def _preset_pairs(jpegs, host, dev, seeds):
    hs, imgs, rows = [], [], []
    for k, im in enumerate(jpegs):
        for s in seeds:
            torch.manual_seed(1000 * s + k)
            hs.append(host(im))
            torch.manual_seed(1000 * s + k)
            a, row = dev(im)
            imgs.append(a)
            rows.append(row)
    _, out = run(imgs, rows, dev.size)
    return torch.stack(hs), out, rows


def test_whole_presets_host_against_device(jpegs):
    """The train preset (RandomResizedCrop, flip, TrivialAugmentWide, Normalize, RandomErasing(0.1)) and the eval preset
    (Resize(512), CenterCrop(448)), host against device on the same images and draws."""
    host = data.ClassificationPresetTrain(448, auto_augment_policy='ta_wide', random_erase_prob=0.1)
    dev = data.DevicePresetTrain(448, auto_augment_policy='ta_wide', random_erase_prob=0.1)
    h, d, rows = _preset_pairs(jpegs, host, dev, range(4))
    diff = (h - d).abs()
    geo = torch.tensor([A.TA_OPS[int(r[A.OP])] in A.GEOMETRIC for r in rows])
    print(f'train preset: {len(rows)} images, max |diff| {diff.max():.3e}, mean {diff.mean():.3e}; non-geometric ops max '
          f'{diff[~geo].max():.3e}; values beyond 1 LSB {(diff > LSB * 1.001).float().mean():.2e}')
    assert diff[~geo].max() <= LSB * 1.001
    assert (diff[geo] > LSB * 1.001).float().mean() < 1e-3 and diff.mean() < 1e-3
    assert diff.max() < 4e-6                   # PIL-identical uint8 images: only the rounding of /255 and Normalize
    host = data.ClassificationPresetEval(448, resize_size=512)
    dev = data.DevicePresetEval(448, resize_size=512)
    h, d, _ = _preset_pairs(jpegs, host, dev, [0])
    diff = (h - d).abs()
    print(f'eval preset: max |diff| {diff.max():.3e}, mean {diff.mean():.3e}')
    assert diff.max() < 4e-6


def test_train_geometry_on_a_marked_corner(tmp_path):
    """A grey image with a red top-left corner: host and device agree on where the corner lands (crop and flip)."""
    arr = np.full((375, 500, 3), 128, np.uint8)
    arr[:80, :80] = (250, 10, 10)
    Image.fromarray(arr).save(tmp_path / 'c.png')
    im = data.default_loader(str(tmp_path / 'c.png'))
    host = data.ClassificationPresetTrain(448)
    dev = data.DevicePresetTrain(448)
    h, d, rows = _preset_pairs([im], host, dev, range(24))
    red_h, red_d = h[:, 0] > 1.5, d[:, 0] > 1.5
    assert torch.equal(red_h, red_d) and (h - d).abs().max() < 4e-6
    seen = red_d.flatten(1).any(1)
    flips = torch.tensor([r[A.FLIP] == 1 for r in rows])
    assert (seen & flips).any() and (seen & ~flips).any()
    for k in torch.nonzero(seen).flatten().tolist():           # a flipped crop puts the corner on the right
        cols = torch.nonzero(red_d[k].any(0)).flatten()
        assert (cols[-1] == 447) if flips[k] else (cols[0] == 0)


@pytest.fixture(scope='module')
def folder(tmp_path_factory):
    root = tmp_path_factory.mktemp('cub')
    lines = []
    for i in range(24):
        write_jpeg(str(root / f'{i}.jpg'), 500 if i % 3 else 375, 375 if i % 3 else 500, seed=100 + i)
        lines.append(f'{(7 * i) % 200} {i}.jpg')
    for split in ('train', 'val'):
        (root / f'{split}.txt').write_text('\n'.join(lines) + '\n')
    return str(root)


def _config(root, tmp_path, device, graph):
    from hawkeye_b200.config import load_config
    cfg = load_config(os.path.join(REPO, 'configs', 'BCNN_S2.yaml'))
    cfg.dataset.update(root_dir=root, meta_dir=root, batch_size=4, num_workers=0)
    if device:
        cfg.dataset.transformer['device'] = device
    cfg.experiment['log_dir'] = str(tmp_path)
    cfg.experiment['cuda_graph'] = graph
    return cfg


def test_bcnn_train_step_with_the_device_presets(folder, tmp_path, monkeypatch):
    """Six BCNN 448 steps fed by the device presets, eager and with graph replay.  The same seed gives the same images
    bit for bit in both runs; the steps other than the first and the capture run with no host synchronisation."""
    from hawkeye_b200 import _lib, examples
    monkeypatch.setenv('HAWKEYE_ALLOW_RANDOM_INIT', '1')
    _lib.set_precise(0)
    seen = {}
    for graph in (False, True):
        tr = examples.BCNNTrainer(_config(folder, tmp_path, 'cuda', graph))
        assert type(tr.dataloaders['train'].dataset.transform) is data.DevicePresetTrain
        torch.manual_seed(5)
        stage, images = tr.stage_inputs, []

        def spy(batch):
            out = stage(batch)
            images.append(out[0].clone())
            return out
        tr.stage_inputs = spy
        w0 = tr.model.classifier.weight.detach().clone()
        for i, batch in enumerate(tr.dataloaders['train']):
            assert isinstance(batch['img'], A.PackedImages) and batch['img'].data.is_pinned()
            with no_host_sync() if i not in (0, 2) else contextlib.nullcontext():
                tr.batch_training(batch)
        torch.cuda.synchronize()
        assert len(images) == 6 and all(x.shape == (4, 3, 448, 448) for x in images)
        assert (tr._graph is not None) == graph and np.isfinite(tr.average_meters['loss'].avg)
        assert not torch.equal(tr.model.classifier.weight, w0)
        seen[graph] = torch.stack(images).cpu()
        tr.validate()
        assert tr.average_meters['acc'].count == 24
        del tr
        torch.cuda.empty_cache()
    assert torch.equal(seen[False], seen[True])
    assert seen[False].abs().sum() > 0


def test_tester_with_both_presets(folder, tmp_path, monkeypatch):
    """The eval preset has no draw and no op: with a PIL-exact resize the two image batches differ by the rounding of /255
    and Normalize only.  Reports the logits' relative L2 and both accuracies."""
    from hawkeye_b200.cfgnode import CfgNode
    from hawkeye_b200.test import Tester
    from oracle.hop_oracle import VGG16_D
    monkeypatch.setenv('HAWKEYE_ALLOW_RANDOM_INIT', '1')
    path = str(tmp_path / 'best_model.pth')
    torch.save(detgen.vgg_bcnn_state(VGG16_D, 200, seed=100), path)
    testers = {}
    for device in (None, 'cuda'):
        tr = dict(image_size=448, resize_size=512)
        if device:
            tr['device'] = device
        cfg = CfgNode(dict(experiment=dict(name='t', cuda=[0]), dataset=dict(root_dir=folder, meta_dir=folder, batch_size=8,
                                                                             num_workers=0, transformer=tr),
                           model=dict(name='BCNN', num_classes=200, load=path)))
        testers[device] = Tester(cfg)
    ims, logits = {}, {}
    for device, t in testers.items():
        t.model.eval()
        ims[device], logits[device] = [], []
        with torch.no_grad():
            for batch in t.dataloader:
                x = t.to_device(batch['img'])
                ims[device].append(x)
                logits[device].append(t.model(x))
    a, b = torch.cat(ims[None]), torch.cat(ims['cuda'])
    rl = rel_l2(torch.cat(logits['cuda']).cpu(), torch.cat(logits[None]).cpu())
    acc = {d: t.test() for d, t in testers.items()}
    print(f'tester: images max |diff| {(a - b).abs().max():.3e}; logits rel L2 {rl:.3e}; accuracy host {acc[None]:.2f} '
          f'device {acc["cuda"]:.2f}')
    assert (a - b).abs().max() < 4e-6 and rl < 1e-3
