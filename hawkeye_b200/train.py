"""``Trainer`` with the reference's template-method surface (train.py:37-435) for the hot-path methods.

Same hooks (``get_model / get_criterion / get_optimizer / get_scheduler / to_device / batch_training /
batch_validate / save_model / save_checkpoint / load_checkpoint / on_*``) and the same yaml schema, so the
reference's ``Examples/{BCNN,CBCNN,MPN}.py`` subclasses port by changing one import.  Differences, all at the
edges: data-parallelism is one process per GPU + NCCL gradient all-reduce instead of
``nn.DataParallel`` (train.py:220-228); the criterion / optimizer are the fused CUDA kernels; ``verbose=`` is not
passed to ReduceLROnPlateau; a missing ``resize_size`` defaults to image_size/0.875; ``train()`` re-raises.
The JPEG input pipeline (dataset/*) is out of scope: pass ``dataloaders=`` or run inside a Hawkeye checkout
whose ``dataset`` package is importable.
"""
import logging
import os

import torch

from . import engine, ops
from .config import setup_config
from .ops_augment import PackedImages, augment
from .ops_mixup import mix_batch
from .registry import MODEL
from .utils import load_state_dict


class AverageMeter:
    """utils/utils.py:10-26 semantics.  ``update_async`` takes a value that is still on its way from the device (a pinned
    host scalar + the CUDA event of its copy) so the training loop never blocks on a read-back; ``avg`` drains them."""

    def __init__(self):
        self.reset()

    def reset(self):
        self.sum, self.count, self._pending = 0.0, 0, []

    def update(self, val, n=1):
        self.sum += val * n
        self.count += n

    def update_async(self, host_buf, index, scale, n, event):
        self._pending.append((host_buf, index, scale, n, event))
        self.drain_ready()

    def drain_ready(self):
        while self._pending and self._pending[0][4].query():       # fold in whatever has already landed
            self._fold(self._pending.pop(0))

    def _fold(self, item):
        host_buf, index, scale, n, _ = item
        self.update(float(host_buf[index]) * scale, n)

    @property
    def avg(self):
        while self._pending:
            item = self._pending.pop(0)
            item[4].synchronize()
            self._fold(item)
        return self.sum / self.count if self.count else 0.0


def accuracy(output, target, topk=1):
    """top-k accuracy in percent (utils/utils.py:52-66)."""
    with torch.no_grad():
        _, pred = output.topk(topk, 1, True, True)
        correct = pred.eq(target.view(-1, 1)).any(dim=1).float().sum()
        return (correct * (100.0 / target.size(0))).item()


def _as_tuple(labels):
    """The criterion's target arguments: one labels tensor, or the tuple a multi-target ``batch_tensors`` gives."""
    return labels if isinstance(labels, tuple) else (labels,)


def prediction(model, outputs):
    """The part of a model's ``outputs`` that validation scores: ``model.prediction(outputs)`` for a model whose forward
    returns more than its logits, the outputs themselves otherwise (so models of the reference's registry still work)."""
    return model.prediction(outputs) if hasattr(model, 'prediction') else outputs


def transformer_device(config):
    """'cuda' when a ``dataset.transformer`` config asks for the device presets (``device: cuda``), None when it has no
    ``device`` key (the host presets).  Also checks ``decode`` (``transformer_decode``)."""
    device = config['device'] if 'device' in config else None
    if device not in (None, 'cuda'):
        raise ValueError(f"dataset.transformer.device must be 'cuda' or absent, not {device!r}")
    transformer_decode(config)
    return device


def transformer_decode(config):
    """'cuda' when a ``dataset.transformer`` config sets ``decode: cuda`` (the JPEGs the device decodes travel encoded,
    ``hawkeye_b200.ops_jpeg``), None when it has no ``decode`` key.  Valid only with ``device: cuda``."""
    from .ops_jpeg import decode_setting
    return decode_setting(config)


def dataset_loader(config):
    """The image loader ``FGDataset`` is given: ``encoded_loader`` under ``decode: cuda``, else the default."""
    from .data import default_loader, encoded_loader
    return encoded_loader if transformer_decode(config) == 'cuda' else default_loader


def device_collate(config, transforms, who):
    """{split: collate function} of the device presets in ``transforms`` when the transformer config asks for them, None
    otherwise.  A trainer that builds its own presets keeps them on the host, so the key is an error there."""
    if transformer_device(config) is None:
        return None
    if not all(hasattr(t, 'collate') for t in transforms.values()):
        key = 'device: cuda and decode: cuda cover' if transformer_decode(config) else 'device: cuda covers'
        raise ValueError(f'dataset.transformer.{key} the default presets only; {who} builds its own, which run on the '
                         'host')
    return {s: t.collate for s, t in transforms.items()}


def mixup_cutmix(config, trainer_cls):
    """True when the ``dataset`` config sets ``mixup_cutmix: true``: the training batches are mixed by the reference's
    ``MixupCutmixCollateFn(model.num_classes)`` and the criterion is ``ops.CrossEntropyLSMix``.  Only trainers whose
    criterion is the base Trainer's cross-entropy on one logits tensor learn from the soft target; any other trainer
    (one that overrides ``get_criterion``) is an error, not a quiet fall-back to hard labels."""
    on = bool(config['mixup_cutmix']) if 'mixup_cutmix' in config else False
    if on and trainer_cls.get_criterion is not Trainer.get_criterion:
        raise ValueError(f'dataset.mixup_cutmix covers the trainers whose criterion is the base cross-entropy on one '
                         f'logits tensor; {trainer_cls.__name__} has its own loss')
    return on


def warmup_cosine_args(config, total_epoch):
    """-> (T_max, warmup_epochs, lr_warmup_decay) of a scheduler config, each with its default."""
    return (config['T_max'] if 'T_max' in config else total_epoch,
            config['warmup_epochs'] if 'warmup_epochs' in config else 0,
            config['lr_warmup_decay'] if 'lr_warmup_decay' in config else 0.01)


EMA_DEFAULTS = dict(decay=0.99998, steps=32)       # torchvision's --model-ema-decay and --model-ema-steps


def model_ema_setting(config):
    """-> (decay, steps) of a ``train`` config's ``model_ema`` key, each with torchvision's default, or None without the
    key: the weights' exponential moving average is on exactly when ``train.model_ema`` is present.  A ``decay`` outside
    (0, 1) or a ``steps`` that is not an integer >= 1 raises ValueError naming the key."""
    if 'model_ema' not in config:
        return None
    c = config['model_ema'] if config['model_ema'] is not None else {}
    if not isinstance(c, dict):
        raise ValueError(f'train.model_ema must be a mapping with decay and steps, or empty, not {c!r}')
    unknown = sorted(set(c) - set(EMA_DEFAULTS))
    if unknown:
        raise ValueError(f'train.model_ema has unknown keys {unknown} (decay, steps)')
    decay = c['decay'] if 'decay' in c else EMA_DEFAULTS['decay']
    steps = c['steps'] if 'steps' in c else EMA_DEFAULTS['steps']
    if isinstance(decay, bool) or not isinstance(decay, (int, float)) or not 0 < decay < 1:
        raise ValueError(f'train.model_ema.decay must lie in (0, 1), not {decay!r}')
    if isinstance(steps, bool) or not isinstance(steps, int) or steps < 1:
        raise ValueError(f'train.model_ema.steps must be an integer >= 1, not {steps!r}')
    return float(decay), steps


def model_ema_decay(decay, steps, batch_size, epochs):
    """The decay an update applies, torchvision's references/classification/train.py: the configured decay is per image
    over the whole run, adjusted to one update every ``steps`` batches of ``batch_size`` (the global batch) images,
    ``alpha = min(1, (1 - decay) * batch_size * steps / epochs)``, decay ``1 - alpha``."""
    adjust = batch_size * steps / epochs
    alpha = min(1.0, (1.0 - decay) * adjust)
    return 1.0 - alpha


class Trainer:
    def __init__(self, config=None, dataloaders=None):
        self.config = config if config is not None else setup_config()
        self.mixing = mixup_cutmix(self.config.dataset, type(self))
        self.epoch = 0
        self.start_epoch = 0
        self.total_epoch = self.config.train.epoch
        self.log_root = os.path.join(self.config.experiment.log_dir, self.config.experiment.name)
        self.logger = logging.getLogger('hawkeye_b200')
        self.rank, self.local_rank, self.world = engine.init_distributed()
        cuda = self.config.experiment.cuda if isinstance(self.config.experiment.cuda, list) else []
        if not torch.cuda.is_available():
            raise RuntimeError('hawkeye_b200 needs a CUDA device (no CPU fallback)')
        self.device = torch.device('cuda', self.local_rank if self.world > 1 else (cuda[0] if cuda else 0))
        torch.cuda.set_device(self.device)
        if 'seed' in self.config.experiment and self.config.experiment.seed is not None:
            torch.manual_seed(self.config.experiment.seed)
        self.samplers = {}
        # user-supplied dataloaders must already be rank-sharded when world > 1 (e.g. built with a DistributedSampler)
        self.dataloaders = dataloaders if dataloaders is not None else self.get_dataloader(self.config.dataset)
        self.model = self.get_model(self.config.model)
        self.model = self.to_device(self.model, parallel=True)
        self.criterion = self.get_criterion(self.config.train.criterion)
        self.flat = self.flatten_parameters()
        self.allreduce = engine.GradAllReduce(self.flat, early_group=self.early_group(), world=self.world)
        self.optimizer = self.get_optimizer(self.config.train.optimizer)
        self.optimizer.grad_scale = 1.0 / self.world
        self.scheduler = self.get_scheduler(self.config.train.scheduler)
        self.ema_steps, self.ema_warmup, self.acc_ema, self.epoch_batch = 0, 0, None, 0
        self.ema = self.get_model_ema(self.config.train)
        self.average_meters = {'acc': AverageMeter(), 'loss': AverageMeter()}
        self.copy_stream = torch.cuda.Stream(device=self.device)    # input H2D overlaps the previous step's compute
        self._in_ring = {}
        self._readback = [torch.zeros(2, dtype=torch.float32).pin_memory() for _ in range(8)]
        self._readback_ev = [None] * 8
        self._readback_i = 0
        if 'resume' in self.config.experiment and self.config.experiment.resume:
            self.load_checkpoint(self.config.experiment.resume)

    # ---- builders (override like the reference's Examples do) -------------------------------------------
    def get_model(self, config):
        model = MODEL.get(config.name)(config)                      # train.py:161-162
        if 'load' in config and config.load != '':
            load_state_dict(model, torch.load(config.load, map_location='cpu'))
        return model

    def get_transformers(self, config):
        """{'train', 'val'} transforms of the ``dataset.transformer`` config.  With ``device: cuda`` these are the device
        presets of ``hawkeye_b200.data``: the workers decode and draw, and ``stage_inputs`` runs the rest on the GPU."""
        resize = config['resize_size'] if 'resize_size' in config else int(config['image_size'] / 0.875)
        if transformer_device(config) == 'cuda':
            from .data import DevicePresetTrain, DevicePresetEval
            return {'train': DevicePresetTrain(crop_size=config['image_size'], auto_augment_policy='ta_wide',
                                               random_erase_prob=0.1),
                    'val': DevicePresetEval(crop_size=config['image_size'], resize_size=resize)}
        try:        # inside a Hawkeye checkout: the reference's own classes; otherwise the mirror in hawkeye_b200.data
            from dataset.transforms import ClassificationPresetTrain, ClassificationPresetEval
        except Exception:
            from .data import ClassificationPresetTrain, ClassificationPresetEval
        return {'train': ClassificationPresetTrain(crop_size=config['image_size'], auto_augment_policy='ta_wide',
                                                   random_erase_prob=0.1),
                'val': ClassificationPresetEval(crop_size=config['image_size'], resize_size=resize)}

    def get_dataloader(self, config):
        try:
            from dataset.dataset import FGDataset
        except Exception:
            from .data import FGDataset
        tf = self.get_transformers(config.transformer)
        collate = device_collate(config.transformer, tf, type(self).__name__)
        if mixup_cutmix(config, type(self)):           # the training batches only: validation is never mixed
            from .data import MixupCutmixCollateFn
            collate = dict(collate or {}, train=MixupCutmixCollateFn(self.config.model.num_classes,
                                                                     (collate or {}).get('train')))
        kw = {'loader': dataset_loader(config.transformer)} if transformer_decode(config.transformer) else {}
        return self.rank_loaders(config, {s: FGDataset(config.root_dir, os.path.join(config.meta_dir, s + '.txt'),
                                                       transform=tf[s], **kw) for s in ('train', 'val')},
                                 collate_fn=collate)

    def rank_loaders(self, config, datasets, collate_fn=None):
        """{'train', 'val'} loaders of this rank over ``datasets``; ``collate_fn`` maps a split to its collate function.

        One process per GPU replaces nn.DataParallel (train.py:220-228), which SPLITS config.batch_size across the visible
        GPUs: batch_size stays the GLOBAL batch, each rank draws batch_size / world images from its own shard of the
        training set (DistributedSampler, reshuffled per epoch in train()); validation is sharded the same way and the
        accuracy meters are reduced over ranks in validate()."""
        from torch.utils.data import DataLoader
        if config.batch_size % self.world != 0:
            raise ValueError(f'dataset.batch_size={config.batch_size} must be a multiple of the {self.world} ranks')
        self.datasets, self.samplers, loaders = datasets, {}, {}
        for s in ('train', 'val'):
            sampler = None
            if self.world > 1:
                from torch.utils.data.distributed import DistributedSampler
                sampler = DistributedSampler(datasets[s], num_replicas=self.world, rank=self.rank, shuffle=s == 'train',
                                             drop_last=False)
            self.samplers[s] = sampler
            loaders[s] = DataLoader(datasets[s], config.batch_size // self.world, num_workers=config.num_workers,
                                    pin_memory=True, sampler=sampler, shuffle=(s == 'train' and sampler is None),
                                    collate_fn=(collate_fn or {}).get(s))
        return loaders

    def get_criterion(self, config):
        if mixup_cutmix(self.config.dataset, type(self)):          # the soft target of dataset/collate_fn.py's batches
            return ops.CrossEntropyLSMix(label_smoothing=0.1)
        return ops.CrossEntropyLS(label_smoothing=0.1)              # train.py:211-212

    def param_groups(self):
        """[(params, lr_multiplier)] — contiguous slices of the flat buffer; the first group listed as ``early`` by
        ``early_group`` is all-reduced while the rest of backward still runs."""
        m = self.get_model_module()
        head = list(m.classifier.parameters()) if hasattr(m, 'classifier') else []
        ids = {id(p) for p in head}
        rest = [p for p in m.parameters() if id(p) not in ids]
        return [(rest, 1.0), (head, 1.0)]

    def trained_groups(self):
        """The (params, lr_multiplier) pairs of ``param_groups`` that have a trainable parameter: the flat buffer's groups."""
        return [(g, m) for g, m in self.param_groups() if any(p.requires_grad for p in g)]

    def early_group(self):
        n = len(self.trained_groups())
        return n - 1 if n > 1 else None

    def flatten_parameters(self):
        return engine.FlatParams(None, groups=[g for g, _ in self.trained_groups()])

    def get_optimizer(self, config):
        name = config.name if 'name' in config else 'Adam'
        lrs = [config.lr * m for _, m in self.trained_groups()]
        wd = config.weight_decay if 'weight_decay' in config else 0.0
        if name == 'SGD':
            return engine.FusedSGD(self.flat, lr=config.lr, momentum=config.momentum if 'momentum' in config else 0.0,
                                   weight_decay=wd, group_lrs=lrs)
        return engine.FusedAdam(self.flat, lr=config.lr, weight_decay=wd, group_lrs=lrs)   # train.py:214-215

    def get_scheduler(self, config):
        name = config.name if 'name' in config else ''
        if name == 'ReduceLROnPlateau':                              # Examples/BCNN.py:42-44 (without verbose=)
            return _Plateau(self.optimizer, mode='max', factor=0.1, patience=3, threshold=1e-4)
        T_max, warmup_epochs, warmup_decay = warmup_cosine_args(config, self.total_epoch)
        return _Cosine(self.optimizer, T_max, config.eta_min if 'eta_min' in config else 0.0, warmup_epochs, warmup_decay)

    def get_model_ema(self, config):
        """The ``engine.ModelEMA`` of the model with ``train.model_ema`` (torchvision's ``--model-ema``), None without it.
        Sets the update interval ``ema_steps`` and ``ema_warmup``, the epochs after whose updates the counter resets."""
        setting = model_ema_setting(config)
        if setting is None:
            return None
        decay, self.ema_steps = setting
        sc = config.scheduler if 'scheduler' in config else {}
        self.ema_warmup = sc['warmup_epochs'] if 'warmup_epochs' in sc else 0
        return engine.ModelEMA(self.get_model_module(), self.flat,
                               model_ema_decay(decay, self.ema_steps, self.config.dataset.batch_size, self.total_epoch))

    def to_device(self, m, parallel=False):
        """A tensor or module on the trainer's device; a packed batch of the device presets becomes its model input."""
        if isinstance(m, PackedImages):
            return m.to(self.device, non_blocking=True).images()
        return m.to(self.device, non_blocking=True) if isinstance(m, torch.Tensor) else m.to(self.device)

    def get_model_module(self, model=None):
        return self.model if model is None else model

    # ---- the hot step (train.py:310-325) ------------------------------------------------------------------------
    def batch_tensors(self, data):
        """-> (images, labels): the tensors of one loader batch the step uses.  ``labels`` is one tensor for the dict
        batches of FGDataset; a method whose criterion takes several targets returns their tuple, which reaches the
        criterion as ``criterion(outputs, *labels)``.  A batch mixed by ``MixupCutmixCollateFn`` gives (labels, mix), which
        ``ops.CrossEntropyLSMix`` takes."""
        if 'mix' in data:
            return data['img'], (data['label'], data['mix'])
        return data['img'], data['label']

    def stage_inputs(self, data):
        """Host -> device copy of one batch on the copy stream (asynchronous for pinned host tensors) into a ring of three
        preallocated device buffers per batch shape — no allocator traffic in the step.  The compute stream waits for the
        copy in-stream, and the copy stream waits (device-side) until the step that last used the slot has finished, so the
        copy of step n+1 overlaps the kernels of step n whenever the host runs ahead.  Returns (images, labels, slot);
        labels is a tuple when ``batch_tensors`` gives one, each target with its own buffer in the slot.  A mixed batch
        (``dataset.mixup_cutmix``) is mixed on the compute stream after the copy (``mix_staged``)."""
        img, lab = self.batch_tensors(data)
        labs = lab if isinstance(lab, tuple) else (lab,)
        if isinstance(img, PackedImages):
            return self.stage_packed(img, lab, labs)
        if img.is_cuda and all(t.is_cuda for t in labs):
            return self.mix_staged(img, lab, None), lab, None
        key = (tuple(img.shape), img.dtype) + tuple((tuple(t.shape), t.dtype) for t in labs)
        ring = self._in_ring.get(key)
        if ring is None:
            ring = self._in_ring[key] = dict(i=0, slots=[dict(img=torch.empty(img.shape, dtype=img.dtype, device=self.device),
                                                               lab=[torch.empty(t.shape, dtype=t.dtype, device=self.device)
                                                                    for t in labs],
                                                               free=None) for _ in range(3)])
        slot = ring['slots'][ring['i'] % 3]
        ring['i'] += 1
        cur = torch.cuda.current_stream()
        with torch.cuda.stream(self.copy_stream):
            if slot['free'] is not None:
                self.copy_stream.wait_event(slot['free'])
            slot['img'].copy_(img, non_blocking=True)
            for d, t in zip(slot['lab'], labs):
                d.copy_(t, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record()
        cur.wait_event(ev)
        lab = tuple(slot['lab']) if isinstance(lab, tuple) else slot['lab'][0]
        return self.mix_staged(slot['img'], lab, slot), lab, slot

    def stage_packed(self, packed, lab, labs):
        """``stage_inputs`` of a packed batch of the device presets: the packed images and their tables are copied on the
        copy stream into a ring slot whose byte buffer grows to the largest batch seen, then the augment kernels write
        the slot's fp32 image buffer on the compute stream.  A graph-replayed step copies from that buffer into its static
        input afterwards, as it does for any staged batch.

        A batch with encoded JPEGs (``dataset.transformer.decode: cuda``) also has its scans and tables copied, into
        grow-only buffers of the slot, and is decoded on the compute stream into the slot's pixel buffer before the
        augment kernels.  The decode's status words come back asynchronously and are checked when the slot is next
        used (or by ``check_decode``): a failed decode raises, naming the file."""
        N, S = len(packed), packed.size
        key = ('packed', N, S) + tuple((tuple(t.shape), t.dtype) for t in labs)
        ring = self._in_ring.get(key)
        dev = self.device
        if ring is None:
            ring = self._in_ring[key] = dict(i=0, slots=[dict(
                src=torch.empty(0, dtype=torch.uint8, device=dev),
                offsets=torch.empty(N, dtype=torch.int64, device=dev), sizes=torch.empty(N, 2, dtype=torch.int32, device=dev),
                params=torch.empty(packed.params.shape, dtype=torch.float64, device=dev),
                work=torch.empty(N, S, S, 3, dtype=torch.uint8, device=dev),
                lut=torch.empty(N, 3, 256, dtype=torch.uint8, device=dev),
                img=torch.empty(N, 3, S, S, dtype=torch.float32, device=dev),
                lab=[torch.empty(t.shape, dtype=t.dtype, device=dev) for t in labs], free=None) for _ in range(3)])
        slot = ring['slots'][ring['i'] % 3]
        ring['i'] += 1
        self.check_decode(slot)
        cur = torch.cuda.current_stream()
        nbytes = packed.pixel_bytes
        grown = slot['src'].numel() < nbytes
        if grown:       # allocated on the compute stream: the copy stream must not write it before that stream's earlier work
            slot['src'] = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        jpeg = packed.jpeg
        if jpeg is not None:
            jbufs = slot.setdefault('jpeg', {})
            for k in jpeg.tensors():
                t = getattr(jpeg, k)
                if k not in jbufs or jbufs[k].numel() < t.numel():
                    jbufs[k] = torch.empty(t.numel(), dtype=t.dtype, device=dev)
                    grown = True
        if grown:
            self.copy_stream.wait_stream(cur)
        with torch.cuda.stream(self.copy_stream):
            if slot['free'] is not None:
                self.copy_stream.wait_event(slot['free'])
            slot['src'][:packed.data.numel()].copy_(packed.data, non_blocking=True)
            for k in ('offsets', 'sizes', 'params'):
                slot[k].copy_(getattr(packed, k), non_blocking=True)
            if jpeg is not None:
                dev_jpeg = jpeg._map(lambda t: t)
                for k in jpeg.tensors():
                    t = getattr(jpeg, k)
                    d = jbufs[k][:t.numel()].view(t.shape)
                    d.copy_(t, non_blocking=True)
                    setattr(dev_jpeg, k, d)
            for d, t in zip(slot['lab'], labs):
                d.copy_(t, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record()
        cur.wait_event(ev)
        if jpeg is not None:
            self.decode_staged(slot, dev_jpeg)
        augment(slot['src'], slot['offsets'], slot['sizes'], slot['params'], S, packed.mean, packed.std, out=slot['img'],
                work=slot['work'], lut=slot['lut'])
        lab = tuple(slot['lab']) if isinstance(lab, tuple) else slot['lab'][0]
        return self.mix_staged(slot['img'], lab, slot), lab, slot

    def decode_staged(self, slot, jpeg):
        """Decodes the slot's encoded JPEGs into its pixel buffer on the compute stream and starts the copy of their
        status words to the host; ``check_decode`` reads them."""
        from .ops_jpeg import decode
        work = slot.setdefault('jpeg_work', {})
        status = decode(jpeg, slot['src'], slot['offsets'], work=work)
        J = len(jpeg)
        host = slot.get('status_host')
        if host is None or host.numel() < J:
            host = slot['status_host'] = torch.empty(J, dtype=torch.int32).pin_memory()
        host[:J].copy_(status, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        slot['decode'] = (ev, J, jpeg.paths)

    def check_decode(self, slot=None):
        """Raises, naming the file, when a decode whose status is pending in ``slot`` (every slot when None) failed.  By
        the time a slot comes round again its decode has long finished, so the wait is a formality."""
        slots = [slot] if slot is not None else [s for r in self._in_ring.values() for s in r['slots']]
        for s in slots:
            pending = s.get('decode')
            if pending is None:
                continue
            s['decode'] = None
            ev, J, paths = pending
            if not ev.query():
                ev.synchronize()
            from .ops_jpeg import raise_on_status
            raise_on_status(s['status_host'][:J].numpy(), paths)

    def mix_staged(self, images, labels, slot):
        """The staged images of a batch ``MixupCutmixCollateFn`` mixed (labels = (labels, mix row)): ``hk_mix_batch`` on
        the compute stream, after the copy (and the augment kernels), into the slot's own buffer — out of place, with no
        allocation once the slot has one and no host read of the draws.  Any other batch is returned as it is."""
        if not (self.mixing and isinstance(labels, tuple)):
            return images
        if slot is None:
            return mix_batch(images, labels[1])
        if slot.get('mixed') is None:
            slot['mixed'] = torch.empty_like(images)
        return mix_batch(images, labels[1], out=slot['mixed'])

    # ---- CUDA-graph replay of forward + loss + backward (+ gradient all-reduce) ----------------------------------------
    # A ResNet-50 step is ~1500 short launches issued from Python: the host, not the GPU, sets the step time.  With
    # ``experiment.cuda_graph: true`` (or $HK_CUDA_GRAPH=1) the step is captured once — after three eager warm-up steps, for
    # one batch shape — and replayed from a static input buffer; the optimizer stays outside the graph (its learning rate
    # and Adam's bias corrections are launch arguments that change from step to step).
    def _graph_wanted(self):
        if getattr(self, '_graph_mode', None) is None:
            env = os.environ.get('HK_CUDA_GRAPH')
            exp = self.config.experiment
            self._graph_mode = (env == '1') if env is not None else bool(exp.cuda_graph if 'cuda_graph' in exp else False)
            self._graph, self._graph_steps = None, 0
        return self._graph_mode

    def _graph_step(self, images, labels):
        """-> (outputs, loss) of this batch.  Eager for the first three calls, then capture, then replay.

        Everything — warm-up steps included — runs on ONE dedicated non-default stream: autograd binds each parameter's
        AccumulateGrad node to the stream of its first use, and a node bound to the legacy default stream cannot be joined from
        a capturing stream.  The caller's stream is ordered before and after (wait_stream), so callers see no difference."""
        if getattr(self, '_graph_stream', None) is None:
            self._graph_stream = torch.cuda.Stream(device=self.device)
        cur, gs = torch.cuda.current_stream(), self._graph_stream
        gs.wait_stream(cur)
        with torch.cuda.stream(gs):
            out = self._graph_step_on_stream(images, labels, gs)
        cur.wait_stream(gs)
        return out

    def _graph_step_on_stream(self, images, labels, gs):
        targets = _as_tuple(labels)
        key = (tuple(images.shape),) + tuple(tuple(t.shape) for t in targets)
        if self._graph is not None and self._graph['key'] != key:
            self._graph = None                                         # another batch shape (last batch of an epoch): eager
            self._graph_steps = -1
        if self._graph is None:
            outputs, loss = self.eager_step(images, labels)
            if self._graph_steps >= 0:
                self._graph_steps += 1
            if self._graph_steps == 3:
                g = dict(key=key, img=torch.empty_like(images), lab=[torch.empty_like(t) for t in targets],
                         graph=torch.cuda.CUDAGraph())
                static = tuple(g['lab']) if isinstance(labels, tuple) else g['lab'][0]
                gs.synchronize()
                from . import _lib
                n0 = _lib.launch_count()
                with torch.cuda.graph(g['graph'], stream=gs):
                    g['out'] = self.forward_model(g['img'], static)
                    g['loss'] = self.criterion(g['out'], *g['lab'])
                    g['correct'] = getattr(self.criterion, 'last_correct', None)
                    self.optimizer.zero_grad()
                    g['loss'].backward()
                    self.allreduce.finish()
                g['kernels'] = _lib.launch_count() - n0        # library kernels recorded in the graph (replayed every step)
                self._graph = g
            return outputs, loss
        g = self._graph
        g['img'].copy_(images, non_blocking=True)
        for d, t in zip(g['lab'], targets):
            d.copy_(t, non_blocking=True)
        g['graph'].replay()
        if g['correct'] is not None:
            self.criterion.last_correct = g['correct']
        return g['out'], g['loss']

    def eager_step(self, images, labels):
        """-> (outputs, loss) of forward, criterion, zero_grad, backward and the gradient all-reduce, launched from Python."""
        outputs = self.forward_model(images, labels)
        loss = self.criterion(outputs, *_as_tuple(labels))
        self.optimizer.zero_grad()
        loss.backward()
        self.allreduce.finish()
        return outputs, loss

    @staticmethod
    def release_inputs(slot):
        """Lets the next copy into ``slot`` (from ``stage_inputs``) start once the work enqueued so far has finished."""
        if slot is not None:
            slot['free'] = torch.cuda.Event()
            slot['free'].record()

    def batch_training(self, data):
        """train.py:310-325: forward, CE(label_smoothing), zero_grad, backward, (grad all-reduce), step, meters.
        No host synchronisation: loss and top-1 count are copied back asynchronously every step (8 bytes into pinned
        memory) and folded into the meters when they have landed."""
        images, labels, slot = self.stage_inputs(data)
        outputs, loss = self._graph_step(images, labels) if self._graph_wanted() else self.eager_step(images, labels)
        self.optimizer.step()
        self.after_optimizer_step()
        self.update_ema()
        self.release_inputs(slot)
        n = images.size(0)
        correct = getattr(self.criterion, 'last_correct', None)
        if correct is None:                                           # a user-supplied criterion: reference behaviour
            self.average_meters['acc'].update(accuracy(prediction(self.get_model_module(), outputs),
                                                       _as_tuple(labels)[0], 1), n)
            self.average_meters['loss'].update(loss.item(), n)
            return loss
        n_acc, n_loss = self.meter_counts(n)
        slot = self._readback_i % len(self._readback)
        self._readback_i += 1
        buf = self._readback[slot]
        if self._readback_ev[slot] is not None:
            self._readback_ev[slot].synchronize()      # back-pressure: never more than 8 steps of read-backs in flight
            for m in self.average_meters.values():
                m.drain_ready()
        with torch.no_grad():
            dev = torch.stack((loss.detach().float(), correct[0].float()))
        buf.copy_(dev, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self._readback_ev[slot] = ev
        self.average_meters['loss'].update_async(buf, 0, 1.0, n_loss, ev)
        self.average_meters['acc'].update_async(buf, 1, 100.0 / n_acc, n_acc, ev)
        return loss

    def after_optimizer_step(self):
        """Work of the step that follows the optimizer, still before the step's input slot is released (it may read the
        step's labels).  ProtoTree's leaf update goes here."""

    def update_ema(self):
        """After the optimizer step (and ``after_optimizer_step``) of batch ``epoch_batch`` of the epoch: torchvision's
        train_one_epoch updates the average when the index is a multiple of ``ema_steps``, and resets its counter after
        an update in a warm-up epoch.  All of it on the device; nothing when the trainer has no EMA."""
        if self.ema is not None and self.epoch_batch % self.ema_steps == 0:
            self.ema.update(reset_after=self.epoch < self.ema_warmup)
        self.epoch_batch += 1

    def forward_model(self, images, labels):
        """The model call of the training step (eager and graph-captured alike).  Methods whose forward takes the labels
        (APINet mines its pairs from them) override this."""
        return self.model(images)

    def meter_counts(self, n):
        """-> (samples behind the top-1 count, samples behind the loss) of a batch of n images."""
        return n, n

    def batch_validate(self, data):
        images, labels = self.batch_tensors(data)
        images, labels = self.to_device(images), self.to_device(_as_tuple(labels)[0])
        with torch.no_grad():
            outputs = self.model(images)
        self.average_meters['acc'].update(accuracy(prediction(self.get_model_module(), outputs), labels, 1),
                                          images.size(0))

    def validate(self):
        self.model.train(False)
        for m in self.average_meters.values():
            m.reset()
        for data in self.dataloaders['val']:
            self.batch_validate(data)
        if self.world > 1:                      # every rank saw its own shard: reduce (sum, count) of each meter over ranks
            import torch.distributed as dist
            for m in self.average_meters.values():
                t = torch.tensor([m.sum, m.count], dtype=torch.float64, device=self.device)
                dist.all_reduce(t)
                m.sum, m.count = t[0].item(), int(t[1].item())
        self.model.train(True)

    def validate_ema(self):
        """-> top-1 accuracy of the averaged weights: ``validate()`` with them swapped in, on meters of its own, so the
        model's meters keep the model's results.  Also kept as ``acc_ema``."""
        meters = self.average_meters
        self.average_meters = {k: AverageMeter() for k in meters}
        try:
            with self.ema.swapped():
                self.validate()
                self.acc_ema = self.average_meters['acc'].avg
        finally:
            self.average_meters = meters
        return self.acc_ema

    def train(self):
        cfg = self.config.train
        self.model.train()
        best = best_ema = None
        for epoch in range(self.start_epoch, self.total_epoch):
            self.epoch = epoch
            self.epoch_batch = 0
            for m in self.average_meters.values():
                m.reset()
            self.on_start_epoch(None)
            if self.samplers.get('train') is not None:
                self.samplers['train'].set_epoch(epoch)
            for data in self.dataloaders['train']:
                self.on_start_forward(None)
                self.batch_training(data)
                self.on_end_forward(None)
            self.check_decode()
            self.validate()
            val_acc = self.average_meters['acc'].avg
            is_best = epoch >= 5 and (best is None or val_acc > best)      # train.py:284-288
            best = val_acc if best is None else max(best, val_acc)
            self.do_scheduler_step()
            is_best_ema = False
            if self.ema is not None:
                acc_ema = self.validate_ema()
                self.logger.info('epoch %d: acc %.4f acc_ema %.4f', epoch, val_acc, acc_ema)
                is_best_ema = epoch >= 5 and (best_ema is None or acc_ema > best_ema)
                best_ema = acc_ema if best_ema is None else max(best_ema, acc_ema)
            if self.rank == 0:
                if epoch != 0 and (epoch + 1) % cfg.save_frequence == 0:
                    self.save_model()
                if is_best:
                    self.save_model('best_model.pth')
                if is_best_ema:
                    self.save_model('best_model_ema.pth', self.ema.model_state_dict())
            self.on_end_epoch(None)

    def do_scheduler_step(self):
        if isinstance(self.scheduler, _Plateau):
            self.scheduler.step(self.average_meters['acc'].avg)
        else:
            self.scheduler.step()

    # ---- checkpoints (train.py:369-395).  save_model writes the reference's format exactly (a plain model state_dict
    # .pth; reference-trained files load through load_state_dict and vice versa).  save_checkpoint keeps the reference's
    # top-level layout {'epoch','model','optimizer','scheduler'} with an identical 'model' part, but the optimizer /
    # scheduler parts are the fused optimizers' own state (flat momentum / Adam moments), not torch.optim's: a reference
    # checkpoint resumes here with its model weights only (load_checkpoint says so instead of failing). -----------------
    def save_model(self, name=None, state=None):
        """Writes ``state`` (the model's state_dict when None) as a plain state_dict .pth."""
        os.makedirs(self.log_root, exist_ok=True)
        path = os.path.join(self.log_root, name or f'{self.config.model.name}_epoch_{self.epoch + 1}.pth')
        state = self.model.state_dict() if state is None else state
        torch.save({k: v.detach().cpu().clone() for k, v in state.items()}, path)
        return path

    def save_checkpoint(self):
        os.makedirs(self.log_root, exist_ok=True)
        path = os.path.join(self.log_root, f'checkpoint_epoch_{self.epoch}.pth')
        torch.save(self.checkpoint_state(), path)
        return path

    def checkpoint_state(self):
        """-> the dict save_checkpoint writes; a trainer with trained state outside the model adds its own keys.  With
        ``train.model_ema`` it holds ``model_ema``, the average in ``AveragedModel.state_dict()``'s layout."""
        ck = {'epoch': self.epoch, 'model': {k: v.detach().cpu().clone() for k, v in self.model.state_dict().items()},
              'optimizer': self.optimizer.state_dict(), 'scheduler': self.scheduler.state_dict()}
        if self.ema is not None:
            ck['model_ema'] = self.ema.state_dict()
        return ck

    def load_checkpoint(self, path):
        self.restore_checkpoint(torch.load(path, map_location='cpu'), path)

    def restore_checkpoint(self, ck, path):
        """Restores the loaded checkpoint ``ck`` (read from ``path``)."""
        self.start_epoch = ck['epoch']
        load_state_dict(self.model, ck['model'])
        opt = ck.get('optimizer', {})
        if isinstance(opt, dict) and ('buf' in opt or 'm' in opt):
            self.optimizer.load_state_dict(opt)
            self.scheduler.load_state_dict(ck['scheduler'])
        else:
            self.logger.warning('checkpoint %s carries torch.optim state (a reference checkpoint): model weights and epoch '
                                'restored, optimizer / scheduler state re-initialised', path)
        if self.ema is None:
            return
        if 'model_ema' in ck:
            self.ema.load_state_dict(ck['model_ema'])
        else:
            self.logger.warning('checkpoint %s has no model_ema: the average starts from the restored weights', path)
            model = {k: v.detach().clone() for k, v in self.get_model_module().state_dict().items()}
            self.ema.load_state_dict(engine.averaged_state(torch.zeros((), dtype=torch.int64), model))

    def on_start_epoch(self, config):
        pass

    def on_end_epoch(self, config):
        pass

    def on_start_forward(self, config):
        pass

    def on_end_forward(self, config):
        pass


class PeerLearningTrainer(Trainer):
    """Examples/PeerLearning.py:17-111 on this Trainer: PeerLearningNet (two base models) + the co-teaching loss with the
    drop-rate ramp of Eqn.(2) (0 -> ``model.drop_rate`` over the first ``model.T_k`` epochs).  Model and loss are parity-tested
    against the reference on CPU (tests/test_peer_learning.py); each base model is the registry's native BCNN / CBCNN / MPN."""

    def __init__(self, config=None, dataloaders=None):
        super().__init__(config, dataloaders)
        import numpy as np
        mc = self.config.model
        self.rate_scheduler = np.ones(self.total_epoch) * mc.drop_rate                  # Examples/PeerLearning.py:21-24
        self.rate_scheduler[:mc.T_k] = np.linspace(0, mc.drop_rate, mc.T_k)[:self.total_epoch]
        self.average_meters = {k: AverageMeter() for k in ('acc', 'acc1', 'acc2', 'loss1', 'loss2')}

    def get_criterion(self, config):
        from .losses import peer_learning_loss
        return peer_learning_loss

    def batch_training(self, data):
        images, labels, slot = self.stage_inputs(data)
        logits1, logits2 = self.model(images)
        loss1, loss2 = self.criterion(logits1, logits2, labels, drop_rate=float(self.rate_scheduler[self.epoch]))
        self.optimizer.zero_grad()
        loss1.backward()
        loss2.backward()
        self.allreduce.finish()
        self.optimizer.step()
        self.update_ema()
        self.release_inputs(slot)
        n = images.size(0)
        acc1, acc2 = accuracy(logits1, labels, 1), accuracy(logits2, labels, 1)
        for k, v in (('acc', max(acc1, acc2)), ('acc1', acc1), ('acc2', acc2), ('loss1', loss1.item()), ('loss2', loss2.item())):
            self.average_meters[k].update(v, n)
        return loss1, loss2

    def batch_validate(self, data):
        images, labels = self.to_device(data['img']), self.to_device(data['label'])
        with torch.no_grad():
            logits1, logits2 = self.model(images)
        acc1, acc2 = accuracy(logits1, labels, 1), accuracy(logits2, labels, 1)
        for k, v in (('acc', max(acc1, acc2)), ('acc1', acc1), ('acc2', acc2)):
            self.average_meters[k].update(v, images.size(0))


class _Plateau:
    """ReduceLROnPlateau(mode='max') over FusedSGD/FusedAdam param_groups (Examples/BCNN.py:42-48)."""

    def __init__(self, opt, mode='max', factor=0.1, patience=3, threshold=1e-4):
        self.opt, self.factor, self.patience, self.threshold = opt, factor, patience, threshold
        self.best, self.bad = None, 0

    def step(self, metric):
        if self.best is None or metric > self.best * (1 + self.threshold):
            self.best, self.bad = metric, 0
        else:
            self.bad += 1
            if self.bad > self.patience:
                for g in self.opt.param_groups:
                    g['lr'] *= self.factor
                self.bad = 0

    def state_dict(self):
        return dict(best=self.best, bad=self.bad)

    def load_state_dict(self, sd):
        self.best, self.bad = sd['best'], sd['bad']


class _Step:
    """StepLR(step_size, gamma) over FusedSGD/FusedAdam param_groups, stepped once per epoch (Examples/DCL.py:89-90):
    lr = initial_lr * gamma ** (epoch // step_size)."""

    def __init__(self, opt, step_size, gamma=0.1):
        self.opt, self.step_size, self.gamma, self.e = opt, step_size, gamma, 0
        self._apply()

    def _apply(self):
        for g in self.opt.param_groups:
            g['lr'] = g['initial_lr'] * self.gamma ** (self.e // self.step_size)

    def step(self):
        self.e += 1
        self._apply()

    def state_dict(self):
        return dict(e=self.e)

    def load_state_dict(self, sd):
        self.e = sd['e']
        self._apply()


class _MultiStep:
    """MultiStepLR(milestones, gamma) over FusedSGD/FusedAdam param_groups, stepped once per epoch (Examples/CrossX.py:41-42):
    lr = initial_lr * gamma ** (the number of milestones <= epoch)."""

    def __init__(self, opt, milestones, gamma=0.1):
        self.opt, self.milestones, self.gamma, self.e = opt, sorted(int(m) for m in milestones), gamma, 0
        self._apply()

    def _apply(self):
        k = sum(1 for m in self.milestones if m <= self.e)
        for g in self.opt.param_groups:
            g['lr'] = g['initial_lr'] * self.gamma ** k

    def step(self):
        self.e += 1
        self._apply()

    def state_dict(self):
        return dict(e=self.e)

    def load_state_dict(self, sd):
        self.e = sd['e']
        self._apply()


class _Cosine:
    """LinearLR warm-up -> CosineAnnealingLR (Examples/CBCNN.py:35-45, Examples/MPN.py:20-30; train.py:217-218)."""

    def __init__(self, opt, T_max, eta_min=0.0, warmup_epochs=0, warmup_decay=0.01):
        import math
        self.opt, self.T, self.eta, self.w, self.d, self.e, self.math = opt, T_max, eta_min, warmup_epochs, warmup_decay, 0, math
        self._apply()

    def _apply(self):
        for g in self.opt.param_groups:
            base = g['initial_lr']
            if self.e < self.w:
                f = self.d + (1 - self.d) * self.e / max(self.w, 1)
                g['lr'] = base * f
            else:
                t = self.e - self.w
                g['lr'] = self.eta + (base - self.eta) * (1 + self.math.cos(self.math.pi * t / max(self.T - self.w, 1))) / 2

    def step(self):
        self.e += 1
        self._apply()

    def state_dict(self):
        return dict(e=self.e)

    def load_state_dict(self, sd):
        self.e = sd['e']
        self._apply()
