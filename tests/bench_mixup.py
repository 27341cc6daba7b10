"""Mixup / CutMix benchmark (csrc/mixup.cu).  Prints one JSON line with:
  * the card's name and power limit;
  * hk_mix_batch on a 32 x 3 x 448 x 448 fp32 batch, Mixup and CutMix, timed with CUDA events over many launches, and the
    bytes it must move at least (one read and one write of the batch, 154 MB) over that time as a share of the H100
    SXM's 3.35 TB/s;
  * hk_softmax_ce_ls_mix at B = 32, K = 200, next to hk_softmax_ce_ls on the same logits;
  * the BCNN VGG-16 448 train step (Trainer.batch_training, batch 32, pinned host inputs, eager as bench.py runs it)
    with and without ``dataset.mixup_cutmix``, two alternating rounds of each, timed with CUDA events.

    python tests/bench_mixup.py [--steps 20] [--warmup 3]
"""
import argparse
import json
import os
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tests'))
from benchutil import card, timed  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
B, C, S, K = 32, 3, 448, 200


def kernels(res):
    from hawkeye_b200 import _lib, ops_mixup as M
    _lib.set_precise(0)
    g = torch.Generator(device='cuda').manual_seed(0)
    x = torch.randn(B, C, S, S, device='cuda', generator=g)
    y = torch.empty_like(x)
    nbytes = 2.0 * x.numel() * 4
    res['mix_batch'] = {}
    for name, row in (('mixup', M.mix_row(M.MIXUP, 0.3)), ('cutmix', M.mix_row(M.CUTMIX, 0.5, (90, 120, 300, 330),
                                                                                      0.5))):
        row = row.cuda()
        ms = timed(lambda: M.mix_batch(x, row, out=y), 200, 20)
        res['mix_batch'][name] = dict(ms=round(ms, 4), mb_moved=round(nbytes / 1e6, 1),
                                      share_of_3_35_tb_s=round(nbytes / (ms / 1e3) / HBM_BYTES_PER_S, 3))
    z = torch.randn(B, K, device='cuda', generator=g)
    labels = torch.randint(0, K, (B,), device='cuda', generator=g)
    row = M.mix_row(M.MIXUP, 0.3).cuda()
    loss = torch.empty(1, device='cuda')
    dl = torch.empty_like(z)
    corr = torch.empty(1, dtype=torch.int32, device='cuda')

    def mix_ce():
        _lib.call('hk_softmax_ce_ls_mix', z, labels, row, loss, dl, corr, B, K, 0.1, 1.0, _lib.stream_ptr())

    def ce():
        _lib.call('hk_softmax_ce_ls', z, labels, loss, dl, corr, B, K, 0.1, 1.0, _lib.stream_ptr())
    res['loss_ms'] = dict(softmax_ce_ls_mix=round(timed(mix_ce, 500, 50), 4), softmax_ce_ls=round(timed(ce, 500, 50), 4))


def step_ms(key, steps, warmup):
    from hawkeye_b200 import data, examples
    from hawkeye_b200.config import load_config
    cfg = load_config(os.path.join(REPO, 'configs', 'BCNN_S2.yaml'))
    if key:
        cfg.dataset['mixup_cutmix'] = True
    torch.manual_seed(0)
    tr = examples.BCNNTrainer(cfg, dataloaders={})
    items = [{'img': torch.randn(C, S, S), 'label': i % K} for i in range(B)]
    batch = data.MixupCutmixCollateFn(K)(items) if key else torch.utils.data.default_collate(items)
    batch = {k: v.pin_memory() for k, v in batch.items()}
    ms = timed(lambda: tr.batch_training(batch), steps, warmup)
    assert tr.mixing == key
    del tr
    torch.cuda.empty_cache()
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_mixup needs a CUDA device')
    os.environ.setdefault('HAWKEYE_ALLOW_RANDOM_INIT', '1')
    os.environ['HK_CUDA_GRAPH'] = '0'
    res = dict(card(), batch=B, size=S, classes=K)
    kernels(res)
    rounds = {'without_key': [], 'with_key': []}
    for _ in range(2):
        for key in (False, True):
            rounds['with_key' if key else 'without_key'].append(round(step_ms(key, args.steps, args.warmup), 3))
    res['bcnn_step_ms'] = rounds
    base = min(rounds['without_key'])
    res['mix_share_of_step'] = round((res['mix_batch']['mixup']['ms'] + res['loss_ms']['softmax_ce_ls_mix'] -
                                      res['loss_ms']['softmax_ce_ls']) / base, 5)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
