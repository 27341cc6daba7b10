"""Input-pipeline benchmark: the host presets (PIL and torch-CPU, image by image in the loader's workers) against the device
presets (the workers decode and draw; hawkeye_b200.ops_augment runs the rest on the GPU).  Prints one JSON line.

On a seeded set of CUB-sized JPEGs (500x375 and the like) written to a temporary directory, it reports:
  * the card's name and power limit, and the host's core count;
  * loader throughput in img/s, host presets against device presets, at num_workers 0, 4 and all cores.  Each loader is
    drained into the device (the host preset's fp32 batch copied, the device preset's batch copied and augmented), timed
    on the host clock from its first batch to a device synchronise after its last, so worker start-up is not counted;
  * the device presets' kernels per batch of 32 at 448 (train and eval), timed with CUDA events, and the bytes they move
    at least (each source box read once, the uint8 intermediate written and read back, the fp32 output written) over
    that time as a share of the H100 SXM's 3.35 TB/s;
  * BCNN VGG-16 448 train throughput (Trainer.batch_training, batch 32) fed by each loader at num_workers 0 and all
    cores, timed with CUDA events around the steps, against the same step on a batch already in device memory.

    python tests/bench_input.py [--images 160] [--batches 5]
"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

import numpy as np
import torch

from benchutil import card, timed

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tests'))

S, RESIZE, BATCH = 448, 512, 32
HBM_BYTES_PER_S = 3.35e12


def make_jpegs(root, n, seed=0):
    """n seeded JPEGs of typical CUB sizes: a smooth random field with noise on top; labels over 200 classes."""
    from PIL import Image
    r = np.random.RandomState(seed)
    sizes = [(500, 375), (375, 500), (500, 333), (500, 400), (400, 500)]
    lines = []
    for i in range(n):
        w, h = sizes[i % len(sizes)]
        base = Image.fromarray(r.randint(0, 256, (h // 24, w // 24, 3)).astype(np.uint8))
        arr = np.asarray(base.resize((w, h), Image.BICUBIC)).astype(np.int32) + r.randint(-24, 25, (h, w, 3))
        Image.fromarray(np.clip(arr, 0, 255).astype(np.uint8)).save(os.path.join(root, f'{i}.jpg'), quality=90)
        lines.append(f'{i % 200} {i}.jpg')
    for split in ('train', 'val'):
        with open(os.path.join(root, f'{split}.txt'), 'w') as f:
            f.write('\n'.join(lines) + '\n')


def presets(kind):
    from hawkeye_b200 import data
    if kind == 'host':
        return data.ClassificationPresetTrain(S, auto_augment_policy='ta_wide', random_erase_prob=0.1), None
    p = data.DevicePresetTrain(S, auto_augment_policy='ta_wide', random_erase_prob=0.1)
    return p, p.collate


def loader(root, kind, workers, batches):
    """A loader of `batches` batches drawn with replacement from the JPEG set."""
    from torch.utils.data import DataLoader, RandomSampler
    from hawkeye_b200.data import FGDataset
    tf, collate = presets(kind)
    ds = FGDataset(root, os.path.join(root, 'train.txt'), transform=tf)
    return DataLoader(ds, BATCH, num_workers=workers, pin_memory=True, collate_fn=collate, drop_last=True,
                      sampler=RandomSampler(ds, replacement=True, num_samples=batches * BATCH))


def to_device(img):
    from hawkeye_b200.ops_augment import PackedImages
    if isinstance(img, PackedImages):
        return img.to('cuda', non_blocking=True).images()
    return img.to('cuda', non_blocking=True)


def drain(root, kind, workers, batches, step=None):
    """-> (img/s on the host clock, img/s on device events) of the batches after the first: each goes to the device (and
    through `step` when given).  With many workers the run is long enough for each to deliver several batches."""
    batches = min(max(batches, 3 * workers), 200)
    it = iter(loader(root, kind, workers, batches + 1))
    b = next(it)
    step(b) if step else to_device(b['img'])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    n = 0
    for _ in range(batches):
        b = next(it)
        step(b) if step else to_device(b['img'])
        n += BATCH
    e.record()
    torch.cuda.synchronize()
    host_s = time.perf_counter() - t0
    del it
    return n / host_s, n / (a.elapsed_time(e) / 1e3)


def kernel_time(root, kind):
    """-> (ms per batch of 32, minimum bytes moved, {kernel: ms}) of the device preset's kernels."""
    from hawkeye_b200 import data, ops_augment as A
    from hawkeye_b200.data import FGDataset
    tf = (data.DevicePresetTrain(S, auto_augment_policy='ta_wide', random_erase_prob=0.1) if kind == 'train' else
          data.DevicePresetEval(S, resize_size=RESIZE))
    ds = FGDataset(root, os.path.join(root, 'train.txt'), transform=tf)
    torch.manual_seed(0)
    p = tf.collate([ds[i] for i in range(BATCH)])['img'].to('cuda')
    work = torch.empty(BATCH, S, S, 3, dtype=torch.uint8, device='cuda')
    lut = torch.empty(BATCH, 3, 256, dtype=torch.uint8, device='cuda')
    out = torch.empty(BATCH, 3, S, S, device='cuda')
    ms = timed(lambda: p.images(out, work, lut), 50, 5)
    from hawkeye_b200 import _lib
    N, stream = len(p), lambda: _lib.stream_ptr()
    each = {
        'crop_resize': timed(lambda: _lib.call('hk_augment_crop_resize', p.data, p.offsets, p.sizes, p.params, work, N, S,
                                               stream()), 50, 5),
        'stats': timed(lambda: _lib.call('hk_augment_stats', work, p.params, lut, N, S, stream()), 50, 5),
        'apply': timed(lambda: _lib.call('hk_augment_apply', work, p.params, lut, out, N, S, *p.mean, *p.std, stream()),
                       50, 5)}
    rows = p.params.cpu().numpy()
    box = rows[:, A.BOX + 2] * rows[:, A.BOX + 3] * 3
    if kind == 'eval':      # only the rows the window needs are read: the box scaled by the window's share
        box = box * np.minimum(1.0, S * S / (rows[:, A.VIRTUAL] * rows[:, A.VIRTUAL + 1]))
    stats = np.isin(rows[:, A.OP], [A.TA_OPS.index(o) for o in ('Contrast', 'AutoContrast', 'Equalize')])
    inter = S * S * 3
    nbytes = float(box.sum() + BATCH * inter * 2 + stats.sum() * inter + BATCH * inter * 4)
    return ms, nbytes, {k: round(v, 4) for k, v in each.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--images', type=int, default=160)
    ap.add_argument('--batches', type=int, default=5, help='timed batches per loader measurement (after one untimed)')
    args = ap.parse_args()
    os.environ.setdefault('HAWKEYE_ALLOW_RANDOM_INIT', '1')
    cores = os.cpu_count() or 1
    if hasattr(os, 'sched_getaffinity'):
        cores = len(os.sched_getaffinity(0))
    torch.set_num_threads(1)              # the loader's main process, as in training: workers do the host work
    res = dict(card(), host_cores=cores, images=args.images, batch=BATCH, size=S)
    root = tempfile.mkdtemp(prefix='bench_input_')
    try:
        run(args, cores, root, res)
    finally:
        shutil.rmtree(root, ignore_errors=True)
    print(json.dumps(res))


def run(args, cores, root, res):
    make_jpegs(root, args.images)
    workers = sorted({0, min(4, cores), cores})
    res['loader_img_s'] = {}
    for kind in ('host', 'device'):
        for w in workers:
            res['loader_img_s'][f'{kind}_w{w}'] = round(drain(root, kind, w, args.batches)[0], 1)
    res['kernels'] = {}
    for kind in ('train', 'eval'):
        ms, nbytes, each = kernel_time(root, kind)
        res['kernels'][kind] = dict(ms_per_batch=round(ms, 4), ms_per_kernel=each, mb_moved=round(nbytes / 1e6, 1),
                                    share_of_3_35_tb_s=round(nbytes / (ms / 1e3) / HBM_BYTES_PER_S, 3))
    from hawkeye_b200 import _lib, examples
    from hawkeye_b200.config import load_config
    _lib.set_precise(0)
    cfg = load_config(os.path.join(REPO, 'configs', 'BCNN_S2.yaml'))
    cfg.dataset.update(root_dir=root, meta_dir=root, batch_size=BATCH, num_workers=0)
    cfg.dataset.transformer['device'] = 'cuda'
    cfg.experiment['log_dir'] = os.path.join(root, 'log')
    tr = examples.BCNNTrainer(cfg)
    resident = next(iter(loader(root, 'host', 0, 1)))
    resident = {'img': resident['img'].cuda(), 'label': resident['label'].cuda()}
    step_ms = timed(lambda: tr.batch_training(resident), 10, 3)
    res['bcnn_train_img_s'] = {'resident_inputs': round(BATCH / (step_ms / 1e3), 1)}
    for kind in ('host', 'device'):
        for w in sorted({0, cores}):
            res['bcnn_train_img_s'][f'{kind}_w{w}'] = round(drain(root, kind, w, args.batches, tr.batch_training)[1], 1)


if __name__ == '__main__':
    main()
