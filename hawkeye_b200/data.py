"""Host side of the input pipeline with the reference's surface: ``FGDataset`` (dataset/dataset.py:22-64),
the train / eval transform presets (dataset/transforms.py:14-73) and the class-balanced batch sampler OSMENet trains with
(dataset/sampler.py:5-38).  JPEG decode and the PIL augmentations stay on the host exactly as in the reference — this is
Python plumbing, not a kernel path; the tensor part of the eval preset (``ToTensor + Normalize``) can run on the GPU instead
(``hawkeye_b200.test.normalize_u8``).  Used by ``Trainer.get_dataloader`` when the reference's ``dataset`` package is not
importable, so the package also trains outside a Hawkeye checkout.
"""
import os

import numpy as np
import torch
from torch.utils.data.sampler import BatchSampler


def default_loader(path):
    """dataset.py:16-19"""
    from PIL import Image
    img = Image.open(path)
    return img.convert('RGB')


def webfg_loader(path):
    """dataset.py:8-13: open through a file object (no ResourceWarning on large crawled sets)"""
    from PIL import Image
    with open(path, 'rb') as f:
        img = Image.open(f)
        return img.convert('RGB')


class FGDataset(torch.utils.data.Dataset):
    """``meta_path``: one ``<label> <relative path>`` (or comma-separated) line per image; items are ``{'img', 'label'[, 'id']}``."""

    def __init__(self, root, meta_path, transform=None, return_id=False, loader=default_loader):
        import pandas as pd
        self.root = root
        try:
            self.images = pd.read_csv(meta_path, sep=' ', names=['label', 'path'])          # dataset.py:27-30
        except Exception:
            self.images = pd.read_csv(meta_path, sep=',', names=['label', 'path'])
        self.transform, self.return_id, self.loader = transform, return_id, loader

    def __getitem__(self, index):
        item = self.images.iloc[index]
        img = self.loader(os.path.join(self.root, item['path']))
        if self.transform is not None:
            img = self.transform(img)
        data = {'img': img, 'label': item['label']}
        if self.return_id:
            data['id'] = index
        return data

    def __len__(self):
        return len(self.images)


class ClassificationPresetTrain:
    """transforms.py:14-49: RandomResizedCrop -> flip -> (auto-augment) -> PILToTensor -> float -> Normalize -> (RandomErasing)."""

    def __init__(self, crop_size, mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225), interpolation=None, hflip_prob=0.5,
                 auto_augment_policy=None, random_erase_prob=0.0):
        from torchvision.transforms import autoaugment, transforms
        from torchvision.transforms.functional import InterpolationMode
        interpolation = InterpolationMode.BILINEAR if interpolation is None else interpolation
        trans = [transforms.RandomResizedCrop(crop_size, interpolation=interpolation)]
        if hflip_prob > 0:
            trans.append(transforms.RandomHorizontalFlip(hflip_prob))
        if auto_augment_policy is not None:
            if auto_augment_policy == 'ra':
                trans.append(autoaugment.RandAugment(interpolation=interpolation))
            elif auto_augment_policy == 'ta_wide':
                trans.append(autoaugment.TrivialAugmentWide(interpolation=interpolation))
            else:
                trans.append(autoaugment.AutoAugment(policy=autoaugment.AutoAugmentPolicy(auto_augment_policy),
                                                     interpolation=interpolation))
        trans += [transforms.PILToTensor(), transforms.ConvertImageDtype(torch.float), transforms.Normalize(mean=mean, std=std)]
        if random_erase_prob > 0:
            trans.append(transforms.RandomErasing(p=random_erase_prob))
        self.transforms = transforms.Compose(trans)

    def __call__(self, img):
        return self.transforms(img)


class ClassificationPresetEval:
    """transforms.py:52-73: Resize -> CenterCrop -> PILToTensor -> float -> Normalize."""

    def __init__(self, crop_size, resize_size=256, mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225), interpolation=None):
        from torchvision.transforms import transforms
        from torchvision.transforms.functional import InterpolationMode
        interpolation = InterpolationMode.BILINEAR if interpolation is None else interpolation
        self.transforms = transforms.Compose([
            transforms.Resize(resize_size, interpolation=interpolation), transforms.CenterCrop(crop_size),
            transforms.PILToTensor(), transforms.ConvertImageDtype(torch.float), transforms.Normalize(mean=mean, std=std)])

    def __call__(self, img):
        return self.transforms(img)


class BalancedBatchSampler(BatchSampler):
    """sampler.py:5-38: every batch holds ``n_classes`` classes drawn without replacement and ``n_samples`` images of each —
    the batches MAMCLoss needs (every anchor has same-class partners).  Uses numpy's global RNG in the reference's call order
    (one shuffle per class at construction, one ``choice`` per batch, a reshuffle when a class runs out), so a seeded run
    draws the same batches as the reference."""

    def __init__(self, dataset, n_classes, n_samples):
        self.labels = np.array(dataset.images['label'])
        self.labels_set = list(set(self.labels))
        self.label_to_indices = {label: np.where(self.labels == label)[0] for label in self.labels_set}
        for label in self.labels_set:
            np.random.shuffle(self.label_to_indices[label])
        self.used_label_indices_count = {label: 0 for label in self.labels_set}
        self.count = 0
        self.n_classes, self.n_samples = n_classes, n_samples
        self.dataset = dataset
        self.batch_size = n_samples * n_classes

    def __iter__(self):
        self.count = 0
        while self.count + self.batch_size < len(self.dataset):
            classes = np.random.choice(self.labels_set, self.n_classes, replace=False)
            indices = []
            for c in classes:
                used = self.used_label_indices_count[c]
                indices.extend(self.label_to_indices[c][used:used + self.n_samples])
                self.used_label_indices_count[c] += self.n_samples
                if self.used_label_indices_count[c] + self.n_samples > len(self.label_to_indices[c]):
                    np.random.shuffle(self.label_to_indices[c])
                    self.used_label_indices_count[c] = 0
            yield indices
            self.count += self.n_classes * self.n_samples

    def __len__(self):
        return len(self.dataset) // self.batch_size
