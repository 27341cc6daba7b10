"""Host side of the input pipeline with the reference's surface: ``FGDataset`` (dataset/dataset.py:22-64),
the train / eval transform presets (dataset/transforms.py:14-73) and the class-balanced batch sampler OSMENet trains with
(dataset/sampler.py:5-38).  JPEG decode and the PIL augmentations stay on the host exactly as in the reference — this is
Python plumbing, not a kernel path; the tensor part of the eval preset (``ToTensor + Normalize``) can run on the GPU instead
(``hawkeye_b200.test.normalize_u8``).  Used by ``Trainer.get_dataloader`` when the reference's ``dataset`` package is not
importable, so the package also trains outside a Hawkeye checkout.

``DevicePresetTrain`` / ``DevicePresetEval`` are the two default presets with everything after the decode on the GPU
(``hawkeye_b200.ops_augment``), selected by ``dataset.transformer.device: cuda``.  With ``decode: cuda`` as well, the
loader is ``encoded_loader`` and the JPEGs the device decodes travel encoded (``hawkeye_b200.ops_jpeg``).
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


def encoded_loader(path):
    """The loader of ``dataset.transformer.decode: cuda`` (``hawkeye_b200.ops_jpeg.encoded_loader``): an
    ``EncodedJPEG`` for a JPEG the device decodes, the PIL image of ``default_loader`` for any other file."""
    from .ops_jpeg import encoded_loader as load
    return load(path)


def _image_like(img):
    """What torchvision's get_params reads the size of: the PIL image itself, or a [3, H, W] meta tensor standing in
    for an encoded JPEG (no pixels are needed to draw)."""
    from .ops_jpeg import EncodedJPEG
    if isinstance(img, EncodedJPEG):
        return torch.empty(3, img.size[1], img.size[0], device='meta')
    return img


def _pixels(img):
    """A device preset's image: an encoded JPEG as it is, a PIL image as its uint8 HWC array."""
    from .ops_jpeg import EncodedJPEG
    return img if isinstance(img, EncodedJPEG) else np.asarray(img, dtype=np.uint8)


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


def _bilinear_only(interpolation):
    from torchvision.transforms.functional import InterpolationMode
    if interpolation not in (None, InterpolationMode.BILINEAR):
        raise ValueError(f'the device presets resize with BILINEAR only, not {interpolation}')
    return InterpolationMode.BILINEAR


def _square(crop_size):
    size = (crop_size, crop_size) if isinstance(crop_size, int) else tuple(crop_size)
    if len(size) == 1:
        size = (size[0], size[0])
    if size[0] != size[1]:
        raise ValueError(f'the device presets produce square images, not {size}')
    return int(size[0])


class DevicePresetTrain:
    """``ClassificationPresetTrain`` with everything after the decode on the GPU (``hawkeye_b200.ops_augment``).  Called on a
    decoded PIL image in a loader worker, it makes the host preset's random draws — the same torchvision calls, in the same
    order, on the same torch RNG — and returns ``(uint8 HWC array, parameter row)``; ``collate`` packs a batch of them.
    A seeded worker therefore draws the same parameters for an image under either preset and leaves the RNG in the same
    state.  Only ``auto_augment_policy`` None or 'ta_wide' and BILINEAR interpolation are supported."""

    def __init__(self, crop_size, mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225), interpolation=None, hflip_prob=0.5,
                 auto_augment_policy=None, random_erase_prob=0.0):
        from torchvision.transforms import autoaugment, transforms
        if auto_augment_policy not in (None, 'ta_wide'):
            raise ValueError(f"the device train preset supports auto_augment_policy None or 'ta_wide', not "
                             f"{auto_augment_policy!r}")
        interpolation = _bilinear_only(interpolation)
        self.size, self.mean, self.std, self.hflip_prob = _square(crop_size), tuple(mean), tuple(std), hflip_prob
        self.crop = transforms.RandomResizedCrop(crop_size, interpolation=interpolation)
        self.ta = autoaugment.TrivialAugmentWide(interpolation=interpolation) if auto_augment_policy else None
        self.erase = transforms.RandomErasing(p=random_erase_prob) if random_erase_prob > 0 else None

    def draw(self, img):
        """-> the parameter row of one PIL image (or ``EncodedJPEG``), drawn as the host preset draws it."""
        from .ops_augment import param_row
        S = self.size
        i, j, h, w = self.crop.get_params(_image_like(img), self.crop.scale, self.crop.ratio)
        flip = self.hflip_prob > 0 and bool(torch.rand(1) < self.hflip_prob)
        op, magnitude = 'Identity', 0.0
        if self.ta is not None:                          # TrivialAugmentWide.forward's draws
            op_meta = self.ta._augmentation_space(self.ta.num_magnitude_bins)
            op = list(op_meta.keys())[int(torch.randint(len(op_meta), (1,)).item())]
            magnitudes, signed = op_meta[op]
            magnitude = (float(magnitudes[torch.randint(len(magnitudes), (1,), dtype=torch.long)].item())
                         if magnitudes.ndim > 0 else 0.0)
            if signed and torch.randint(2, (1,)):
                magnitude *= -1.0
        erase = None
        if self.erase is not None and torch.rand(1) < self.erase.p:   # RandomErasing.forward on a [3, S, S] image
            ei, ej, eh, ew, _ = self.erase.get_params(torch.empty(3, S, S, device='meta'), scale=self.erase.scale,
                                                      ratio=self.erase.ratio, value=[float(self.erase.value)])
            if eh < S:                                   # otherwise get_params gave up: the image is left as it is
                erase = (ei, ej, eh, ew)
        return param_row((j, i, w, h), (S, S), (0, 0), flip, op, magnitude, S, erase)

    def __call__(self, img):
        return _pixels(img), self.draw(img)

    def collate(self, batch):
        return collate_packed(batch, self.size, self.mean, self.std)


class DevicePresetEval:
    """``ClassificationPresetEval`` (Resize, CenterCrop, ToTensor, Normalize) with everything after the decode on the GPU:
    the image is resized with PIL's arithmetic and the centred window kept, in one pass.  No random draw."""

    def __init__(self, crop_size, resize_size=256, mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225), interpolation=None):
        _bilinear_only(interpolation)
        self.size, self.mean, self.std = _square(crop_size), tuple(mean), tuple(std)
        self.resize_size = [resize_size] if isinstance(resize_size, int) else list(resize_size)

    def draw(self, img):
        from torchvision.transforms.functional import _compute_resized_output_size
        from .ops_augment import param_row
        W, H = img.size
        vh, vw = _compute_resized_output_size((H, W), self.resize_size, None)      # F.resize's output size
        S = self.size
        # F.center_crop: pad to the crop if the image is smaller, then the offset int(round((size - S) / 2))
        pad_l, pad_t = ((S - vw) // 2 if S > vw else 0), ((S - vh) // 2 if S > vh else 0)
        left = int(round((max(vw, S) - S) / 2.0)) - pad_l
        top = int(round((max(vh, S) - S) / 2.0)) - pad_t
        return param_row((0, 0, W, H), (vw, vh), (left, top))

    def __call__(self, img):
        return _pixels(img), self.draw(img)

    def collate(self, batch):
        return collate_packed(batch, self.size, self.mean, self.std)


def collate_packed(batch, size, mean, std):
    """FGDataset items whose 'img' is a device preset's (uint8 array, parameter row) -> {'img': PackedImages, 'label'
    [, 'id']}: the images back to back in one uint8 buffer (pinned by the DataLoader) with their offset, size and
    parameter tables."""
    from .ops_augment import pack
    out = {'img': pack([b['img'][0] for b in batch], [b['img'][1] for b in batch], size, mean, std),
           'label': torch.as_tensor(np.array([b['label'] for b in batch])).long()}
    if 'id' in batch[0]:
        out['id'] = torch.as_tensor([b['id'] for b in batch])
    return out


class MixupCutmixCollateFn:
    """dataset/collate_fn.py: one of RandomMixup(p=1.0, alpha=0.2) and RandomCutmix(p=1.0, alpha=1.0) per batch
    (dataset/transforms.py:76-231), picked with torchvision's RandomChoice.  The draws are the reference's own calls in
    its order, on the worker's RNGs: ``random.choices``, ``torch.rand(1)`` (drawn although p = 1 never skips),
    ``torch._sample_dirichlet`` and, for CutMix, ``torch.randint(W)`` then ``torch.randint(H)``.

    The images are not mixed here.  The batch of ``collate`` (``default_collate``, or a device preset's ``collate`` for
    ``PackedImages``) gains ``'mix'``: the float64 row of ``hawkeye_b200.ops_mixup`` with the kind, lambda, the CutMix box
    and the target weight, which ``Trainer.stage_inputs`` applies on the device.  ``'label'`` stays int64 [B]: the target
    of row i is w onehot(label i) + (1 - w) onehot(label i - 1 mod B), the reference's rolled dense target."""

    def __init__(self, num_classes, collate=None):
        if num_classes <= 0:
            raise ValueError('MixupCutmixCollateFn: num_classes must be positive')
        self.num_classes, self.collate = int(num_classes), collate
        self.alphas = (0.2, 1.0)           # RandomMixup, RandomCutmix

    def draw(self, height, width):
        """-> the mix row of one batch of H x W images, drawn as the reference's collate draws it."""
        import math
        import random
        from .ops_mixup import CUTMIX, MIXUP, check_row, mix_row
        kind = random.choices((MIXUP, CUTMIX))[0]                     # transforms.RandomChoice.__call__
        torch.rand(1)                                                 # the p = 1.0 test: never skips, still a draw
        alpha = self.alphas[kind]
        lam = float(torch._sample_dirichlet(torch.tensor([alpha, alpha]))[0])
        if kind == MIXUP:
            row = mix_row(MIXUP, lam)
        else:                                                         # transforms.py:211-226
            r_x, r_y = int(torch.randint(width, (1,))), int(torch.randint(height, (1,)))
            r = 0.5 * math.sqrt(1.0 - lam)
            r_w_half, r_h_half = int(r * width), int(r * height)
            x1, y1 = max(r_x - r_w_half, 0), max(r_y - r_h_half, 0)
            x2, y2 = min(r_x + r_w_half, width), min(r_y + r_h_half, height)
            row = mix_row(CUTMIX, lam, (x1, y1, x2, y2), float(1.0 - (x2 - x1) * (y2 - y1) / (width * height)))
        check_row(row, height, width)
        return row

    def __call__(self, batch):
        from torch.utils.data import default_collate
        from .ops_augment import PackedImages
        data = (self.collate or default_collate)(batch)
        img, label = data['img'], data['label']
        if label.ndim != 1 or label.dtype != torch.int64:
            raise TypeError(f'MixupCutmixCollateFn: labels must be int64 [B], not {label.dtype} {tuple(label.shape)}')
        if isinstance(img, PackedImages):
            height = width = img.size
        else:
            if img.ndim != 4 or not img.is_floating_point():
                raise TypeError(f'MixupCutmixCollateFn: images must be a float [B, C, H, W] batch, not {img.dtype} '
                                f'{tuple(img.shape)}')
            height, width = img.shape[-2:]
        data['mix'] = self.draw(int(height), int(width))
        return data


def _grid_cells(image, cols, rows):
    """The ``cols x rows`` grid of crops of a PIL image, row by row; cell edges at int(size / count * i)."""
    width, height = image.size
    xs = [int(width / cols * i) for i in range(cols + 1)]
    ys = [int(height / rows * j) for j in range(rows + 1)]
    return [image.crop((xs[i], ys[j], min(xs[i + 1], width), min(ys[j + 1], height)))
            for j in range(rows) for i in range(cols)]


def _swap_last_two(seq):
    """Shuffle the last two entries of ``seq`` in place with ``random.shuffle`` (one draw from Python's ``random``)."""
    import random
    if len(seq) >= 2:
        pair = seq[-2:]
        random.shuffle(pair)
        seq[-2:] = pair


class RandomSwap:
    """DCL's jigsaw (dataset/transforms.py RandomSwap): crop 10 px off every border, cut the rest into a ``size[0] x
    size[1]`` grid (columns x rows), and swap neighbours within a range of 2 — after each cell is placed in its row the last
    two cells of that row may swap, and after each cell once at least two rows are complete the last two complete rows may
    swap — then paste every cell, resized with Lanczos, into a canvas and resize it back to the input size.  The draws from
    Python's ``random`` come in the reference's order, so a seeded run gives the reference's images.  The reference names
    the filter ``Image.ANTIALIAS``, which Pillow 10 removed; ``Image.LANCZOS`` is the same filter."""

    def __init__(self, size):
        import numbers
        if isinstance(size, numbers.Number):
            size = (int(size), int(size))
        if len(size) != 2:
            raise ValueError('RandomSwap: give one size or two, (columns, rows)')
        self.size = size

    def __repr__(self):
        return f'{self.__class__.__name__}(size={self.size})'

    def __call__(self, img):
        from PIL import Image
        cols, rows = self.size
        full_w, full_h = img.size
        img = img.crop((10, 10, full_w - 10, full_h - 10))
        cells = _grid_cells(img, cols, rows)
        done, row = [], []
        for cell in cells:
            row.append(cell)
            _swap_last_two(row)
            if len(row) == cols:
                done.append(row)
                row = []
            _swap_last_two(done)
        order = [c for r in done for c in r]
        width, height = img.size
        iw, ih = int(width / cols), int(height / rows)
        canvas = Image.new('RGB', (iw * cols, ih * rows))
        for i, cell in enumerate(order):
            canvas.paste(cell.resize((iw, ih), Image.LANCZOS), ((i % cols) * iw, (i // cols) * ih))
        return canvas.resize((full_w, full_h))


def _sample_tenth_per_class(paths, labels):
    """A random tenth of every class (rounded down) in the order classes first appear: the reference's validation subset,
    drawn with Python's ``random.sample``."""
    import random
    by_class = {}
    for p, y in zip(paths, labels):
        by_class.setdefault(y, []).append(p)
    out_paths, out_labels = [], []
    for y, ps in by_class.items():
        pick = random.sample(list(range(len(ps))), len(ps) // 10)
        out_paths += [ps[i] for i in pick]
        out_labels += [y] * len(pick)
    return out_paths, out_labels


class DCLDataset(torch.utils.data.Dataset):
    """dataset/dataset_DCL.py: items of DCL's jigsaw training.  ``transforms`` is the dict of Examples/DCL.py:19-51
    ('swap', 'common_aug', '<mode>_totensor').

    train: (image, shuffled image, label, label_swap, swap_law1, swap_law2, path); swap_law1 is the identity law
    (i - n // 2) / n over the n = swap_size[0] x swap_size[1] cells; swap_law2 gives, for every cell of the shuffled image,
    the law of the unshuffled cell whose summed per-band mean is nearest (the first on ties).  label_swap is -1 under cls_2
    (the collate turns it into 1, 0) and label + num_classes under cls_2xmul only.
    val: (image, label, label, swap_law1, swap_law1, path) over a random tenth of every class, and ``common_aug`` is
    applied as in training — both as in the reference.  test: (image, label, path)."""

    def __init__(self, root, meta_path, transforms=None, swap_size=(7, 7), mode='train', cls_2=True, cls_2xmul=False):
        import pandas as pd
        self.root = root
        meta = pd.read_csv(meta_path, sep=' ', names=['label', 'path'])
        self.paths, self.labels = meta['path'].tolist(), meta['label'].tolist()
        if mode == 'val':
            self.paths, self.labels = _sample_tenth_per_class(self.paths, self.labels)
        self.use_cls_2, self.use_cls_mul = cls_2, cls_2xmul
        self.num_classes = len(set(self.labels))
        self.swap_size, self.mode = list(swap_size), mode
        self.common_aug, self.swap = transforms['common_aug'], transforms['swap']
        self.totensor = transforms[mode + '_totensor']

    def __len__(self):
        return len(self.paths)

    def __getitem__(self, item):
        from PIL import ImageStat
        img = webfg_loader(os.path.join(self.root, self.paths[item]))
        label = self.labels[item]
        if self.mode == 'test':
            return self.totensor(img), label, self.paths[item]
        if self.common_aug is not None:
            img = self.common_aug(img)
        n = self.swap_size[0] * self.swap_size[1]
        law1 = [(i - n // 2) / n for i in range(n)]
        if self.mode != 'train':
            return self.totensor(img), label, label, law1, list(law1), self.paths[item]
        swapped = self.swap(img)
        ref = [sum(ImageStat.Stat(c).mean) for c in _grid_cells(img, *self.swap_size)]
        law2 = []
        for s in (sum(ImageStat.Stat(c).mean) for c in _grid_cells(swapped, *self.swap_size)):
            dist = [abs(s - r) for r in ref]
            law2.append((dist.index(min(dist)) - n // 2) / n)
        label_swap = -1 if self.use_cls_2 else (label + self.num_classes if self.use_cls_mul else None)
        return self.totensor(img), self.totensor(swapped), label, label_swap, law1, law2, self.paths[item]


def collate_fn4train(batch):
    """Interleaves every image with its shuffled copy: -> (images [2n, ...], labels [2n], labels_swap [2n] (1, 0 per pair
    under cls_2, else label, label_swap), swap_law [2n, cells], paths [n])."""
    imgs, labels, labels_swap, law, names = [], [], [], [], []
    for s in batch:
        imgs += [s[0], s[1]]
        labels += [s[2], s[2]]
        labels_swap += [1, 0] if s[3] == -1 else [s[2], s[3]]
        law += [s[4], s[5]]
        names.append(s[-1])
    return (torch.stack(imgs, 0), torch.from_numpy(np.array(labels)).long(), torch.from_numpy(np.array(labels_swap)).long(),
            torch.from_numpy(np.array(law)).float(), names)


def collate_fn4val(batch):
    """-> (images [n, ...], labels [n], labels_swap [n] (= labels), swap_law [n, cells], paths [n])."""
    imgs = torch.stack([s[0] for s in batch], 0)
    labels = torch.from_numpy(np.array([s[1] for s in batch])).long()
    labels_swap = torch.from_numpy(np.array([1 if s[3] == -1 else s[2] for s in batch])).long()
    law = torch.from_numpy(np.array([s[3] for s in batch])).float()
    return imgs, labels, labels_swap, law, [s[-1] for s in batch]


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
