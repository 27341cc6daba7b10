"""JPEG decode benchmark: the device presets with the decode in the loader's workers (PIL) against the decode on the
device (``dataset.transformer.decode: cuda``, hawkeye_b200.ops_jpeg).  Prints one JSON line.

On the seeded CUB-sized JPEGs of tests/bench_input.make_jpegs (500x375 and the like, quality 90, 4:2:0), written to a
temporary directory, it reports:
  * the card's name and power limit, and the host's core count;
  * a worker's time per image on this host's CPU: PIL's decode, ``np.asarray`` and the draws, against reading the file,
    parsing its markers (the 0xFF00 unstuffing and the restart search included, timed on their own too) and the draws;
  * loader throughput in img/s, device presets with and without the key, at num_workers 0, 4 and all cores (each batch
    copied to the device and turned into the model input, timed from the first batch to a synchronise after the last);
  * each decode kernel's time per batch of 32 by CUDA events, at several chunk sizes for the Huffman pass, and the
    bytes each moves at least over that time as a share of the H100 SXM's 3.35 TB/s;
  * host-to-device bytes per batch with and without the key;
  * BCNN VGG-16 448 train throughput (Trainer.batch_training, batch 32) fed by each loader at num_workers 0 and all
    cores, timed with CUDA events, next to the same step on a batch already in device memory.

    python tests/bench_decode.py [--images 160] [--batches 5]
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

S, BATCH = 448, 32
HBM_BYTES_PER_S = 3.35e12


def per_image_ms(fn, paths, reps=3):
    t0 = time.perf_counter()
    for _ in range(reps):
        for p in paths:
            fn(p)
    return (time.perf_counter() - t0) / (reps * len(paths)) * 1e3


def worker_times(paths):
    from hawkeye_b200 import data, ops_jpeg as J
    pre = data.DevicePresetTrain(S, auto_augment_policy='ta_wide', random_erase_prob=0.1)
    bufs = {p: open(p, 'rb').read() for p in paths}
    return dict(pil_decode_asarray_draw=per_image_ms(lambda p: pre(data.default_loader(p)), paths),
                encoded_read_parse_draw=per_image_ms(lambda p: pre(data.encoded_loader(p)), paths),
                parse_only=per_image_ms(lambda p: J.parse(bufs[p], p), paths),
                unstuff_and_restarts=per_image_ms(lambda p: unstuff_only(bufs[p]), paths))


def unstuff_only(buf):
    """The numpy part of the parse on its own: find the 0xFF bytes of the scan, drop the stuffing, locate RSTn."""
    start = buf.index(b'\xff\xda')
    start += 2 + int.from_bytes(buf[start + 2:start + 4], 'big')
    d = np.frombuffer(buf, np.uint8, offset=start)
    ff = np.flatnonzero(d[:-1] == 0xFF)
    nxt = d[ff + 1]
    keep = np.ones(len(d), bool)
    keep[ff[nxt == 0] + 1] = False
    return d[keep]


def loader(root, decode, workers, batches):
    from torch.utils.data import DataLoader, RandomSampler
    from hawkeye_b200 import data
    tf = data.DevicePresetTrain(S, auto_augment_policy='ta_wide', random_erase_prob=0.1)
    ds = data.FGDataset(root, os.path.join(root, 'train.txt'), transform=tf,
                        loader=data.encoded_loader if decode else data.default_loader)
    return DataLoader(ds, BATCH, num_workers=workers, pin_memory=True, collate_fn=tf.collate, drop_last=True,
                      sampler=RandomSampler(ds, replacement=True, num_samples=batches * BATCH))


def drain(root, decode, workers, batches, step=None):
    """-> img/s (host clock, device events) of the batches after the first, each taken to the model input (or through
    `step`)."""
    batches = min(max(batches, 3 * workers), 200)
    it = iter(loader(root, decode, workers, batches + 1))
    go = step or (lambda b: b['img'].to('cuda', non_blocking=True).images())
    go(next(it))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(batches):
        go(next(it))
    e.record()
    torch.cuda.synchronize()
    host_s = time.perf_counter() - t0
    n = batches * BATCH
    del it
    return n / host_s, n / (a.elapsed_time(e) / 1e3)


def kernels(root):
    from hawkeye_b200 import _lib, data, ops_jpeg as J
    tf = data.DevicePresetTrain(S, auto_augment_policy='ta_wide', random_erase_prob=0.1)
    ds = data.FGDataset(root, os.path.join(root, 'train.txt'), transform=tf, loader=data.encoded_loader)
    ds_plain = data.FGDataset(root, os.path.join(root, 'train.txt'), transform=tf)
    torch.manual_seed(0)
    host = tf.collate([ds[i] for i in range(BATCH)])['img']
    plain = tf.collate([ds_plain[i] for i in range(BATCH)])['img']
    jb_host = host.jpeg
    h2d = {'with_key': sum(getattr(jb_host, k).numel() * getattr(jb_host, k).element_size() for k in jb_host.tensors())
           + host.data.numel() + host.params.numel() * 8 + host.offsets.numel() * 8 + host.sizes.numel() * 4,
           'without_key': plain.data.numel() + plain.params.numel() * 8 + plain.offsets.numel() * 8 +
           plain.sizes.numel() * 4}
    p = host.to('cuda')
    jb = p.jpeg
    pixels = torch.empty(p.pixel_bytes, dtype=torch.uint8, device='cuda')
    work = {}
    status = J.decode(jb, pixels, p.offsets, work=work)
    assert not status.cpu().numpy().any()
    G, stream = jb.segs.numel() - 1, _lib.stream_ptr
    out = {}
    for chunk in (64, 128, 256, 512, 1024):
        ws = torch.empty(J.workspace_bytes(jb, chunk), dtype=torch.uint8, device='cuda')
        out[f'huffman_ms_chunk{chunk}'] = round(timed(lambda: _lib.call(
            'hk_jpeg_huffman', jb.scan, jb.segs, jb.header, jb.htabs, work['coef'], work['status'], len(jb), G,
            jb.scan.numel(), chunk, ws, ws.numel(), stream()), 20, 3), 4)
    out['idct_ms'] = round(timed(lambda: _lib.call('hk_jpeg_idct', work['coef'], jb.header, jb.qtabs, work['planes'],
                                                   len(jb), stream()), 50, 5), 4)
    out['color_ms'] = round(timed(lambda: _lib.call('hk_jpeg_color', work['planes'], jb.header, p.offsets, pixels,
                                                    len(jb), stream()), 50, 5), 4)
    out['decode_ms'] = round(timed(lambda: J.decode(jb, pixels, p.offsets, work=work), 20, 3), 4)
    scan = jb.scan.numel()
    coef_b = work['coef'].numel() * 2
    plane_b = work['planes'].numel()
    rgb = p.pixel_bytes - p.data.numel()
    # bytes each kernel must move at least: the scan read and the coefficients written; the coefficients read and the
    # planes written; the planes read and the RGB written
    mb = {'huffman': scan + coef_b, 'idct': coef_b + plane_b, 'color': plane_b + rgb}
    out['mb_moved'] = {k: round(v / 1e6, 2) for k, v in mb.items()}
    t = {'huffman': out[f'huffman_ms_chunk{J.CHUNK_BYTES}'], 'idct': out['idct_ms'], 'color': out['color_ms']}
    out['share_of_3_35_tb_s'] = {k: round(mb[k] / (t[k] / 1e3) / HBM_BYTES_PER_S, 3) for k in mb}
    return out, {k: round(v / 1e6, 3) for k, v in h2d.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--images', type=int, default=160)
    ap.add_argument('--batches', type=int, default=5, help='timed batches per loader measurement (after one untimed)')
    args = ap.parse_args()
    os.environ.setdefault('HAWKEYE_ALLOW_RANDOM_INIT', '1')
    if not torch.cuda.is_available():
        raise SystemExit('bench_decode.py needs a CUDA device')
    cores = len(os.sched_getaffinity(0)) if hasattr(os, 'sched_getaffinity') else (os.cpu_count() or 1)
    torch.set_num_threads(1)
    res = dict(card(), host_cores=cores, images=args.images, batch=BATCH, size=S)
    root = tempfile.mkdtemp(prefix='bench_decode_')
    try:
        run(args, cores, root, res)
    finally:
        shutil.rmtree(root, ignore_errors=True)
    print(json.dumps(res))


def run(args, cores, root, res):
    from bench_input import make_jpegs
    make_jpegs(root, args.images)
    paths = [os.path.join(root, f'{i}.jpg') for i in range(min(args.images, 40))]
    res['worker_ms_per_image'] = {k: round(v, 3) for k, v in worker_times(paths).items()}
    res['kernels_per_batch'], res['h2d_mb_per_batch'] = kernels(root)
    workers = sorted({0, min(4, cores), cores})
    res['loader_img_s'] = {}
    for w in workers:
        for decode in (False, True):
            res['loader_img_s'][f'{"device_decode" if decode else "pil_decode"}_w{w}'] = \
                round(drain(root, decode, w, args.batches)[0], 1)
    from hawkeye_b200 import _lib, examples
    from hawkeye_b200.config import load_config
    _lib.set_precise(0)
    res['bcnn_train_img_s'] = {}
    for decode in (False, True):
        cfg = load_config(os.path.join(REPO, 'configs', 'BCNN_S2.yaml'))
        cfg.dataset.update(root_dir=root, meta_dir=root, batch_size=BATCH, num_workers=0)
        cfg.dataset.transformer['device'] = 'cuda'
        if decode:
            cfg.dataset.transformer['decode'] = 'cuda'
        cfg.experiment['log_dir'] = os.path.join(root, 'log')
        tr = examples.BCNNTrainer(cfg)
        if not decode:
            x = torch.randn(BATCH, 3, S, S, device='cuda')
            y = torch.randint(0, 200, (BATCH,), device='cuda')
            step_ms = timed(lambda: tr.batch_training({'img': x, 'label': y}), 10, 3)
            res['bcnn_train_img_s']['resident_inputs'] = round(BATCH / (step_ms / 1e3), 1)
        for w in sorted({0, cores}):
            res['bcnn_train_img_s'][f'{"device_decode" if decode else "pil_decode"}_w{w}'] = \
                round(drain(root, decode, w, args.batches, tr.batch_training)[1], 1)
        tr.check_decode()
        del tr
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
