"""Evaluation entry point with the reference's surface (test.py:14-147): ``python -m hawkeye_b200.test --config <yaml>``
builds ``MODEL.get(config.model.name)``, loads ``config.model.load`` (a plain state_dict .pth — the format the reference's
``Trainer.save_model`` writes, train.py:369-376, with or without a DataParallel ``module.`` prefix), runs the validation split
without gradients and reports top-1 accuracy.  Template methods keep the reference's names so subclasses port verbatim.

Differences that are the point of this package: the model runs the native kernels on ONE CUDA device (there is no CPU path),
and images may arrive as uint8 HWC batches — ``ToTensor + Normalize`` then run fused on the GPU (`hk_normalize_u8`), a quarter
of the host-to-device bytes of the reference's float pipeline."""
import logging
import os

import torch

from . import _lib
from .config import setup_config
from .registry import MODEL
from .utils import load_state_dict

IMAGENET_MEAN, IMAGENET_STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)      # test.py:84, dataset/transforms.py:18-19


def accuracy(output, target, topk=1):
    """utils/utils.py accuracy(): top-k hit rate in percent."""
    with torch.no_grad():
        _, pred = output.topk(topk, 1, True, True)
        return (pred.eq(target.view(-1, 1)).any(dim=1).float().sum() * (100.0 / target.size(0))).item()


def normalize_u8(images_u8, mean=IMAGENET_MEAN, std=IMAGENET_STD):
    """uint8 [N,H,W,3] (HWC, as decoded) on the GPU -> float32 [N,3,H,W] = (x/255 - mean)/std   (ToTensor + Normalize)."""
    if not images_u8.is_cuda or images_u8.dtype != torch.uint8 or images_u8.dim() != 4 or images_u8.shape[-1] != 3:
        raise _lib.HawkeyeLibError('normalize_u8 expects a CUDA uint8 tensor [N,H,W,3]')
    x = images_u8.contiguous()
    N, H, W, _ = x.shape
    out = torch.empty(N, 3, H, W, device=x.device, dtype=torch.float32)
    _lib.call('hk_normalize_u8', x, out, N, H, W, float(mean[0]), float(mean[1]), float(mean[2]), float(std[0]), float(std[1]),
              float(std[2]), _lib.stream_ptr())
    return out


class AverageMeter:
    def __init__(self):
        self.sum, self.count = 0.0, 0

    def update(self, val, n=1):
        self.sum += val * n
        self.count += n

    @property
    def avg(self):
        return self.sum / max(self.count, 1)


class Tester:
    def __init__(self, config=None, dataloader=None):
        self.config = config if config is not None else setup_config()
        self.logger = logging.getLogger('hawkeye_b200')
        if not torch.cuda.is_available():
            raise RuntimeError('hawkeye_b200 needs a CUDA device (no CPU fallback)')
        cuda = self.config.experiment.cuda if isinstance(self.config.experiment.cuda, list) else []
        self.device = torch.device('cuda', cuda[0] if cuda else 0)
        torch.cuda.set_device(self.device)
        self.dataloader = dataloader if dataloader is not None else self.get_dataloader(self.config.dataset)
        self.model = self.to_device(self.get_model(self.config.model))
        self.average_meters = {'acc': AverageMeter()}

    def get_model(self, config):
        model = MODEL.get(config.name)(config)                                                   # test.py:68-69
        assert 'load' in config and config.load != '', 'There is no valid `load` in config[model.load]!'   # test.py:71
        load_state_dict(model, torch.load(config.load, map_location='cpu'))
        return model

    def get_dataloader(self, config):
        try:
            from dataset.dataset import FGDataset               # the reference package, when run inside a Hawkeye checkout
        except Exception:
            from .data import FGDataset                         # its mirror otherwise
        from torch.utils.data import DataLoader
        from torchvision import transforms
        t = config.transformer
        tf = transforms.Compose([transforms.Resize(size=t.resize_size), transforms.CenterCrop(size=t.image_size),
                                 transforms.ToTensor(), transforms.Normalize(mean=IMAGENET_MEAN, std=IMAGENET_STD)])
        ds = FGDataset(config.root_dir, os.path.join(config.meta_dir, 'val.txt'), transform=tf)   # test.py:91-93
        return DataLoader(ds, config.batch_size, num_workers=config.num_workers, pin_memory=True, shuffle=False)

    def to_device(self, m, parallel=False):
        return m.to(self.device, non_blocking=True) if isinstance(m, torch.Tensor) else m.to(self.device)

    def get_model_module(self, model=None):
        return self.model if model is None else model

    def test(self):
        self.validate()
        acc = self.average_meters['acc'].avg
        self.logger.info(f'acc: {acc:.2f}')                                                      # test.py:141-144
        return acc

    def validate(self):
        self.model.train(False)
        with torch.no_grad():
            for data in self.dataloader:
                self.batch_validate(data)

    def batch_validate(self, data):
        images, labels = self.to_device(data['img']), self.to_device(data['label'])
        if images.dtype == torch.uint8:                          # HWC uint8 batches: ToTensor + Normalize on the GPU
            images = normalize_u8(images)
        logits = self.model(images)
        if isinstance(logits, tuple) and isinstance(logits[1], dict):   # ProtoTreeNet returns (pred, info)
            logits = logits[0]
        if isinstance(logits, tuple) and len(logits) == 3 and logits[1].dim() == 4:   # Interp-Parts: (logits, att, assign)
            logits = logits[0]
        if isinstance(logits, list) and len(logits) == 5:        # NTSNet's five outputs: accuracy on concat_logits
            logits = logits[1]
        if isinstance(logits, tuple):                            # PeerLearningNet returns both heads (PeerLearning.py:94-101)
            self.average_meters['acc'].update(max(accuracy(l, labels, 1) for l in logits), images.size(0))
        else:
            self.average_meters['acc'].update(accuracy(logits, labels, 1), images.size(0))


if __name__ == '__main__':
    logging.basicConfig(level=logging.INFO, format='[%(asctime)s] %(message)s')
    Tester().test()
