"""Golden fixtures for Mixup / CutMix from the UNMODIFIED reference (dataset/collate_fn.py MixupCutmixCollateFn,
dataset/transforms.py RandomMixup / RandomCutmix).
Run here only:  HAWKEYE_REF=<Hawkeye checkout> python tests/golden/make_golden_mixup.py  -> tests/golden/reference_mixup.<i>.npz

What each call drew and computed is read back without changing it: ``torch._sample_dirichlet`` is wrapped to record
lambda, and the locals of RandomMixup.forward / RandomCutmix.forward are read when it returns (the box x1, y1, x2, y2 and
the final ``lambda_param``, which is the target weight).

- ``draws``: 50 batches through ``MixupCutmixCollateFn(10)``, each after ``random.seed(k); torch.manual_seed(k)``, of
  1 to 5 random images of 3 x H x W (H, W in 4..15): inputs, the mixed images, the dense targets and the draws.
- ``cases``: 3 x 24 x 40 batches for the device kernel.  ``mixup`` and ``cutmix`` are seeded collate calls that drew that
  kind; the others call RandomCutmix / RandomMixup (p = 1) with ``torch._sample_dirichlet`` and ``torch.randint``
  returning chosen values, so the box lands where the case needs it: clipped at the left and top, clipped at the right
  and bottom, empty (lambda = 1), the whole image (lambda = 0), and B = 1 for both kinds (an image rolls onto itself)."""
import os
import random
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tests'))
from conftest import save_golden  # noqa: E402
from oracle import ref_harness as rh  # noqa: E402

root = rh.find_reference_root()
if root is None:
    raise SystemExit('reference tree not found (set $HAWKEYE_REF)')
sys.path.insert(0, root)
from dataset.collate_fn import MixupCutmixCollateFn  # noqa: E402
from dataset.transforms import RandomCutmix, RandomMixup  # noqa: E402

K = 10
CASE_SHAPE = (3, 24, 40)
seen = {}
_dirichlet = torch._sample_dirichlet


def rec_dirichlet(t, *a, **k):
    out = _dirichlet(t, *a, **k)
    seen['lam'] = float(out[0])
    return out


def profiler(frame, event, arg):
    code = frame.f_code
    if event == 'return' and code.co_name == 'forward' and code in (RandomMixup.forward.__code__,
                                                                     RandomCutmix.forward.__code__):
        loc = frame.f_locals
        seen['kind'] = 0 if code is RandomMixup.forward.__code__ else 1
        seen['box'] = [loc[k] for k in ('x1', 'y1', 'x2', 'y2')] if seen['kind'] == 1 else [0, 0, 0, 0]
        seen['weight'] = float(loc['lambda_param'])


def run(fn, img, label):
    seen.clear()
    torch._sample_dirichlet = rec_dirichlet
    sys.setprofile(profiler)
    try:
        out = fn(img, label)
    finally:
        sys.setprofile(None)
        torch._sample_dirichlet = _dirichlet
    return out, dict(seen)


def collate(img, label):
    return MixupCutmixCollateFn(K)([{'img': img[i], 'label': int(label[i])} for i in range(len(label))])


def direct(cls, alpha, lam, rx=0, ry=0):
    def fn(img, label):
        orig_d, orig_r = torch._sample_dirichlet, torch.randint
        picks = iter([rx, ry])
        torch._sample_dirichlet = lambda t, *a, **k: (seen.update(lam=lam), torch.tensor([lam, 1.0 - lam]))[1]
        torch.randint = lambda n, size, *a, **k: torch.tensor([next(picks)])
        try:
            return cls(num_classes=K, p=1.0, alpha=alpha)({'img': img, 'label': label})
        finally:
            torch._sample_dirichlet, torch.randint = orig_d, orig_r
    return fn


def inputs(rs, B, C, H, W):
    return (torch.from_numpy(rs.standard_normal((B, C, H, W)).astype(np.float32)),
            torch.from_numpy(rs.randint(0, K, B).astype(np.int64)))


arrays = {}
meta = {k: [] for k in ('kind', 'lam', 'box', 'weight')}
rs = np.random.RandomState(0)
for k in range(50):
    B, H, W = rs.randint(1, 6), rs.randint(4, 16), rs.randint(4, 16)
    img, label = inputs(rs, B, 3, H, W)
    random.seed(k)
    torch.manual_seed(k)
    out, d = run(collate, img, label)
    arrays.update({f'draws.img.{k}': img.numpy(), f'draws.label.{k}': label.numpy(),
                   f'draws.out.{k}': out['img'].numpy(), f'draws.target.{k}': out['label'].numpy()})
    for f in meta:
        meta[f].append(d[f])
for f, v in meta.items():
    arrays[f'draws.{f}'] = np.array(v)

C, H, W = CASE_SHAPE
names = []


def case(name, B, fn, want):
    img, label = inputs(rs, B, C, H, W)
    out, d = run(fn, img, label)
    assert want(d), (name, d)
    names.append(name)
    arrays.update({f'case.{name}.img': img.numpy(), f'case.{name}.label': label.numpy(),
                   f'case.{name}.out': out['img'].numpy(), f'case.{name}.target': out['label'].numpy(),
                   f'case.{name}.draw': np.array([d['kind'], d['lam'], *d['box'], d['weight']], np.float64)})


def seeded(kind):
    def fn(img, label):
        for s in range(1000):
            random.seed(s)
            if random.choices([0, 1])[0] == kind:
                break
        random.seed(s)
        torch.manual_seed(s)
        return collate(img, label)
    return fn


case('mixup', 4, seeded(0), lambda d: d['kind'] == 0 and 0 < d['lam'] < 1)
case('cutmix', 4, seeded(1), lambda d: d['kind'] == 1 and d['box'][0] < d['box'][2] and d['box'][1] < d['box'][3])
case('cutmix_left_top', 4, direct(RandomCutmix, 1.0, 0.3, 2, 1), lambda d: d['box'][:2] == [0, 0] and
     d['box'][2] < W and d['box'][3] < H)
case('cutmix_right_bottom', 4, direct(RandomCutmix, 1.0, 0.3, W - 2, H - 1), lambda d: d['box'][2:] == [W, H] and
     d['box'][0] > 0 and d['box'][1] > 0)
case('cutmix_empty', 4, direct(RandomCutmix, 1.0, 1.0, 17, 9), lambda d: d['box'][0] == d['box'][2] and d['weight'] == 1)
case('cutmix_full', 4, direct(RandomCutmix, 1.0, 0.0, W // 2, H // 2), lambda d: d['box'] == [0, 0, W, H] and
     d['weight'] == 0)
case('mixup_b1', 1, direct(RandomMixup, 0.2, 0.37), lambda d: d['kind'] == 0)
case('cutmix_b1', 1, direct(RandomCutmix, 1.0, 0.5, 11, 7), lambda d: d['kind'] == 1 and d['box'][0] < d['box'][2])
arrays['case.names'] = np.array(names)
save_golden('reference_mixup', arrays)
print('wrote', len(names), 'cases and 50 batches of draws')
