"""Trainer subclasses of the hot-path methods with the reference's Examples/ surface:
``python -m hawkeye_b200.examples {BCNN,CBCNN,MPN,PeerLearning,OSMENet,APINet,DCL,ProtoTreeNet,InterpPartsNet,NTSNet,APCNN,MGE_CNN,
CIN,Baseline,PairConfusion}
--config <yaml>`` replaces
``python Examples/<Method>.py --config <yaml>`` (same yaml files; one process per GPU under torchrun instead of nn.DataParallel).
Baseline and PairConfusion train the plain ResNet-50 classifier (configs/Baseline.yaml, configs/PC_resnet50.yaml).

Only what the reference's Examples override is overridden here: which parameters train, with which learning rates, and
which LR schedule — the step itself is ``Trainer.batch_training``.
"""
import os
import sys

from .train import PeerLearningTrainer, Trainer, _Cosine, _Plateau, _Step, warmup_cosine_args


def _warmup_cosine(opt, config, total_epoch):
    T_max, warmup_epochs, warmup_decay = warmup_cosine_args(config, total_epoch)
    return _Cosine(opt, T_max, 0.0, warmup_epochs, warmup_decay)


def _momentum_sgd(trainer, config):
    """SGD with momentum 0.9 and the yaml's weight_decay over the trained groups (Examples/InterpPartsNet.py,
    Examples/APCNN.py)."""
    from . import engine
    return engine.FusedSGD(trainer.flat, lr=config.lr, momentum=0.9,
                           weight_decay=config.weight_decay if 'weight_decay' in config else 0.0,
                           group_lrs=[config.lr * m for _, m in trainer.trained_groups()])


def _balanced_loaders(trainer, config):
    """The reference's class-balanced training loader (dataset/sampler.py BalancedBatchSampler: n_classes x n_samples images
    per batch, Examples/OSMENet.py:17-30, Examples/APINet.py:17-29) next to the base Trainer's validation loader."""
    import numpy as np
    from torch.utils.data import DataLoader
    loaders = Trainer.get_dataloader(trainer, config)            # datasets, transforms, validation loader
    try:
        from dataset.sampler import BalancedBatchSampler
    except Exception:
        from .data import BalancedBatchSampler
    if trainer.world > 1:                                        # one process per GPU: each rank draws its own balanced batches
        np.random.seed((trainer.config.experiment.seed if 'seed' in trainer.config.experiment else 0) + trainer.rank)
    sampler = BalancedBatchSampler(trainer.datasets['train'], config.n_classes, config.n_samples)
    loaders['train'] = DataLoader(trainer.datasets['train'], num_workers=config.num_workers, pin_memory=True,
                                  batch_sampler=sampler)
    return loaders


class BCNNTrainer(Trainer):
    """Examples/BCNN.py:10-48: SGD over the classifier (stage 1: the model freezes its backbone, BCNN.py:45-47) or over all
    parameters (stage 2); ReduceLROnPlateau(max, 0.1, patience 3, threshold 1e-4) on the validation accuracy, always."""

    def get_scheduler(self, config):
        return _Plateau(self.optimizer, mode='max', factor=0.1, patience=3, threshold=1e-4)


class CBCNNTrainer(Trainer):
    """Examples/CBCNN.py:10-45: in stage 1 the *trainer* freezes the backbone (:13-15) and optimises the classifier only;
    SGD; linear warm-up into cosine annealing."""

    def get_model(self, config):
        model = super().get_model(config)
        if config.stage == 1:
            for p in model.backbone.parameters():
                p.requires_grad = False
        return model

    def get_scheduler(self, config):
        return _warmup_cosine(self.optimizer, config, self.total_epoch)


class MPNTrainer(Trainer):
    """Examples/MPN.py:9-30: Adam with three parameter groups — classifier lr, pooling head (DR conv + BN) lr, backbone
    0.2 x lr — and weight decay; linear warm-up into cosine annealing."""

    def param_groups(self):
        m = self.get_model_module()
        return [(list(m.backbone.parameters()), 0.2), (list(m.pool.parameters()), 1.0),
                (list(m.classifier.parameters()), 1.0)]

    def get_scheduler(self, config):
        return _warmup_cosine(self.optimizer, config, self.total_epoch)


class OSMENetTrainer(Trainer):
    """Examples/OSMENet.py:10-80: the model returns (logits, per-attention features); criterion = MAMCLoss (cross-entropy +
    lambda_a x N-pairs over the attention features); SGD with the backbone at 0.1 x lr; linear warm-up into cosine annealing.
    The reference draws class-balanced batches (dataset/sampler.py BalancedBatchSampler: n_classes x n_samples) so that every
    anchor has same-class partners; with a user-supplied dataloader that is the caller's business, as in the reference."""

    def get_dataloader(self, config):
        """Examples/OSMENet.py:17-30: the training loader draws class-balanced batches (n_classes x n_samples images)."""
        return _balanced_loaders(self, config)

    def get_criterion(self, config):
        from .losses import MAMCLoss
        return MAMCLoss(config)

    def param_groups(self):
        m = self.get_model_module()
        backbone = {id(p) for p in m.backbone.parameters()}
        return [(list(m.backbone.parameters()), 0.1), ([p for p in m.parameters() if id(p) not in backbone], 1.0)]

    def get_scheduler(self, config):
        return _warmup_cosine(self.optimizer, config, self.total_epoch)

    # batch_training is the base Trainer's: it hands the model's (pred, x_part) pair to the criterion as is, and MAMCLoss exposes
    # the top-1 count of its cross-entropy kernel (last_correct), so the step has no host synchronisation either.


class _FrozenWarmupCosine(_Cosine):
    """_Cosine with the first ``frozen`` parameter groups at lr 0 until the warm-up ends.  That is what the reference's
    Examples/APINet.py gets from torch: on_start_epoch sets group 0's lr to 0 at epoch 0, LinearLR's multiplicative warm-up
    keeps it there, and at the milestone SequentialLR restarts CosineAnnealingLR from the initial lr, where both groups meet."""

    def __init__(self, opt, T_max, eta_min=0.0, warmup_epochs=0, warmup_decay=0.01, frozen=1):
        self.frozen = frozen
        super().__init__(opt, T_max, eta_min, warmup_epochs, warmup_decay)

    def _apply(self):
        super()._apply()
        if self.e < self.w:
            for g in self.opt.param_groups[:self.frozen]:
                g['lr'] = 0.0


class APINetTrainer(Trainer):
    """Examples/APINet.py: class-balanced batches (n_classes x n_samples images); the model takes the labels and returns
    (self_logits, other_logits, labels1, labels2); criterion = APINetLoss (cross-entropy + margin ranking); Adam with two
    groups — backbone and the rest — at config.lr; linear warm-up into cosine annealing, with the backbone frozen through lr = 0
    (not requires_grad, so Adam's moments and the BN running statistics evolve as in the reference) for the warm-up epochs.
    The meters count 8n logit rows for the accuracy and 4n for the loss, as Examples/APINet.py:74-77 does."""

    def get_dataloader(self, config):
        return _balanced_loaders(self, config)

    def get_criterion(self, config):
        from .losses import APINetLoss
        return APINetLoss(config)

    def param_groups(self):
        m = self.get_model_module()
        backbone = {id(p) for p in m.backbone.parameters()}
        return [(list(m.backbone.parameters()), 1.0), ([p for p in m.parameters() if id(p) not in backbone], 1.0)]

    def get_scheduler(self, config):
        T_max, warmup_epochs, warmup_decay = warmup_cosine_args(config, self.total_epoch)
        return _FrozenWarmupCosine(self.optimizer, T_max, 0.0, warmup_epochs, warmup_decay)

    def forward_model(self, images, labels):
        return self.model(images, labels, flag='train')

    def meter_counts(self, n):
        return 8 * n, 4 * n


class DCLTrainer(Trainer):
    """Examples/DCL.py: every source image and its jigsaw-shuffled copy are interleaved into one batch of 2n rows; the model
    returns [logits, swap_logits, mask]; criterion = DCLLoss(labels, labels_swap, swap_law); SGD with momentum and no weight
    decay (Examples/DCL.py:82-87 passes none, whatever the yaml says) with the trunk at lr and classifier, classifier_swap
    and Convmask at lr_ratio x lr; StepLR(step_size, gamma) once per epoch.  The meters count the 2n rows, as
    Examples/DCL.py:116-117 does.

    The dataset's swap law is taken on the same ``swap_num`` grid the jigsaw uses.  The reference's Examples/DCL.py passes no
    swap_size, so its law is always 7x7; with the default swap_num [7, 7] the two are identical, and with any other grid
    the reference's law would not describe the shuffled cells.

    The data path is always the mirror in hawkeye_b200.data (RandomSwap, DCLDataset, collate_fn4train / collate_fn4val),
    even inside a Hawkeye checkout: the reference's RandomSwap calls ``Image.ANTIALIAS``, which Pillow 10 removed, so its
    own transform no longer runs."""

    def get_transformers(self, config):
        """Examples/DCL.py:19-51, with its defaults 512, 448 and [7, 7]."""
        from torchvision.transforms import transforms
        from .data import RandomSwap
        resize = config.resize_size if 'resize_size' in config else 512
        crop = config.image_size if 'image_size' in config else 448
        swap = config.swap_num if 'swap_num' in config else [7, 7]
        norm = transforms.Normalize([0.485, 0.456, 0.406], [0.229, 0.224, 0.225])
        to_tensor = transforms.Compose([transforms.Resize((crop, crop)), transforms.ToTensor(), norm])
        return {
            'swap': transforms.Compose([RandomSwap((swap[0], swap[1]))]),
            'common_aug': transforms.Compose([transforms.Resize((resize, resize)), transforms.RandomRotation(degrees=15),
                                              transforms.RandomCrop((crop, crop)), transforms.RandomHorizontalFlip()]),
            'train_totensor': to_tensor,
            'val_totensor': to_tensor,
            'test_totensor': transforms.Compose([transforms.Resize((resize, resize)), transforms.CenterCrop((crop, crop)),
                                                 transforms.ToTensor(), norm]),
            'None': None,
        }

    def get_dataloader(self, config):
        from .data import DCLDataset, collate_fn4train, collate_fn4val
        t = config.transformer
        tf = self.get_transformers(t)
        swap = t.swap_num if 'swap_num' in t else [7, 7]
        mc = self.config.model
        return self.rank_loaders(config, {s: DCLDataset(config.root_dir, os.path.join(config.meta_dir, s + '.txt'),
                                                        transforms=tf, swap_size=swap, mode=s, cls_2=mc.cls_2,
                                                        cls_2xmul=mc.cls_2xmul) for s in ('train', 'val')},
                                 {'train': collate_fn4train, 'val': collate_fn4val})

    def get_criterion(self, config):
        from .losses import DCLLoss
        return DCLLoss(config)

    def param_groups(self):
        m = self.get_model_module()
        ratio = self.config.train.optimizer.lr_ratio
        return [(list(m.backbone.parameters()), 1.0), (list(m.classifier.parameters()), ratio),
                (list(m.classifier_swap.parameters()), ratio), (list(m.Convmask.parameters()), ratio)]

    def get_optimizer(self, config):
        from . import engine
        return engine.FusedSGD(self.flat, lr=config.lr, momentum=config.momentum if 'momentum' in config else 0.0,
                               weight_decay=0.0, group_lrs=[config.lr * m for _, m in self.trained_groups()])

    def get_scheduler(self, config):
        return _Step(self.optimizer, config.step_size, config.gamma)

    def batch_tensors(self, data):
        images, labels, labels_swap, swap_law, _ = data
        return images, (labels, labels_swap, swap_law)


class ProtoTreeTrainer(Trainer):
    """Examples/ProtoTreeNet.py with the schedule it actually runs:
    - Parameter groups: the trunk except layer4.2 at 0.01 x lr, layer4.2, the neck and the prototypes at lr, and, with
      model.disable_derivative_free_leaf_optim, the leaves at lr_pi.  Nothing is frozen: the reference's freeze() sets
      ``param.require_grad`` (sic), so its 30-epoch freeze does nothing.
    - Adam or AdamW with eps 1e-7 through engine.FusedAdam.  The groups' ``weight_decay_rate`` is read by no torch optimizer;
      AdamW's global weight_decay (0.0 in the yaml) is the only decay, so a nonzero one, which needs decoupled decay, is
      rejected, and so is SGD, whose prototype group runs without momentum.
    - LinearLR warm-up into cosine annealing (SequentialLR), stepped once per epoch.
    - Loss F.nll_loss(torch.log(pred), labels) (losses.ProtoTreeLoss).
    - After every optimizer step, the derivative-free leaf update against the epoch-start snapshot of the leaves, and then
      ``model.eval()``: only the first batch of an epoch runs the trunk's BatchNorm on batch statistics, every later one on
      the running statistics, with gradients through them, until validate() restores train mode at the end of the epoch.
      With gradient-trained leaves there is no update and no eval().  Under torchrun the ranks all-reduce the update sum
      before applying it, so the update covers the global batch as under the reference's nn.DataParallel.
    The reference's Example calls ``self.model(images, labels)``, which ProtoTreeNet.forward(x) does not accept; the model is
    called with the images alone.  Under ``cuda_graph: true`` the eval-mode steps replay one captured graph and the
    train-mode first batch of each epoch runs eagerly, so a graph never runs in the mode it was not captured in."""

    def __init__(self, config=None, dataloaders=None):
        super().__init__(config, dataloaders)
        self.num_batches = len(self.dataloaders['train']) if 'train' in self.dataloaders else 1
        self._theta0 = None

    def get_criterion(self, config):
        from .losses import ProtoTreeLoss
        return ProtoTreeLoss()

    def _dfo(self):
        mc = self.config.model
        return not (mc.disable_derivative_free_leaf_optim if 'disable_derivative_free_leaf_optim' in mc else False)

    def param_groups(self):
        m = self.get_model_module()
        named = list(m.backbone.named_parameters())
        groups = [([p for n, p in named if '7.2' not in n], 0.01), ([p for n, p in named if '7.2' in n], 1.0),
                  (list(m.neck_conv.parameters()), 1.0), ([m.tree.prototype_layer.prototype_vectors], 1.0)]
        if not self._dfo():
            oc = self.config.train.optimizer
            groups.append(([m.tree.leaf_params], oc.lr_pi / oc.lr))
        return groups

    def get_optimizer(self, config):
        from . import engine
        name = config.name if 'name' in config else 'Adam'
        wd = config.weight_decay if 'weight_decay' in config else 0.0
        if name not in ('Adam', 'AdamW'):
            raise ValueError(f'ProtoTreeTrainer: optimizer {name!r} is not supported (Adam or AdamW)')
        if name == 'AdamW' and wd != 0:
            raise ValueError(f'ProtoTreeTrainer: AdamW with weight_decay={wd} needs decoupled weight decay, which FusedAdam '
                             'does not have; use weight_decay: 0.0')
        return engine.FusedAdam(self.flat, lr=config.lr, eps=1e-7, weight_decay=0.0,
                                group_lrs=[config.lr * m for _, m in self.trained_groups()])

    def get_scheduler(self, config):
        return _warmup_cosine(self.optimizer, config, self.total_epoch)

    def on_start_epoch(self, config):
        self._theta0 = self.get_model_module().tree.leaf_params.detach().clone()

    def _graph_step_on_stream(self, images, labels, gs):
        if self.model.training:
            return self.eager_step(images, labels)
        outputs, loss = super()._graph_step_on_stream(images, labels, gs)
        # the step's own outputs (the graph's static tensors after a replay): on the capturing step the criterion last saw
        # the static tensors of a graph that has not run yet
        self.criterion.last = (outputs[0].detach(), outputs[1]['pa_tensor'].dense, labels)
        return outputs, loss

    def after_optimizer_step(self):
        """The leaf update, enqueued before the step releases its input slot (it reads the step's labels).  With several
        ranks the update sums are all-reduced first: the update then covers the global batch, as under the reference's
        nn.DataParallel, and every rank applies the same one, so the leaves stay identical across ranks."""
        if not self._dfo():
            return
        import torch
        from .ops_prototree import leaf_update
        pred, pa, labels = self.criterion.last
        if self._theta0 is None:
            self.on_start_epoch(None)
        reduce = None
        if self.world > 1:
            import torch.distributed as dist
            reduce = dist.all_reduce
        with torch.no_grad():
            leaf_update(self.get_model_module().tree.leaf_params, self._theta0, pa, pred, labels, self.num_batches, reduce)
        self.model.eval()


class InterpPartsNetTrainer(Trainer):
    """Examples/InterpPartsNet.py: the reference's train / validation transforms; criterion = InterpPartsLoss (cross-entropy
    + coeff x shaping loss on the assignment maps); SGD with momentum 0.9 and weight_decay in two groups, conv1, bn1 and
    layer1-3 at lr and everything else at 20 x lr; CosineAnnealingLR over iterations_per_epoch x epochs, stepped after every
    batch (the per-epoch scheduler step does nothing).  The optimizer and the schedule run outside the captured graph, so
    under ``cuda_graph: true`` the learning rate changes from replay to replay as it does eagerly."""

    FINETUNE = ('conv1', 'bn1', 'layer1', 'layer2', 'layer3')

    def get_transformers(self, config):
        """Examples/InterpPartsNet.py:17-34."""
        from torchvision import transforms
        norm = transforms.Normalize(mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225))
        return {
            'train': transforms.Compose([transforms.Resize(size=config.resize_size), transforms.RandomHorizontalFlip(),
                                         transforms.ColorJitter(0.1), transforms.RandomCrop(size=config.image_size),
                                         transforms.ToTensor(), norm, transforms.RandomErasing(config.p_erasing)]),
            'val': transforms.Compose([transforms.Resize(size=config.resize_size), transforms.CenterCrop(size=config.image_size),
                                       transforms.ToTensor(), norm]),
        }

    def get_criterion(self, config):
        from .losses import InterpPartsLoss
        return InterpPartsLoss(config)

    def param_groups(self):
        named = list(self.get_model_module().named_parameters())
        return [([p for n, p in named if n.split('.')[0] in self.FINETUNE], 1.0),
                ([p for n, p in named if n.split('.')[0] not in self.FINETUNE], 20.0)]

    get_optimizer = _momentum_sgd

    def get_scheduler(self, config):
        iters = len(self.dataloaders['train']) if 'train' in self.dataloaders else 1
        return _Cosine(self.optimizer, iters * self.total_epoch)

    def after_optimizer_step(self):
        self.scheduler.step()

    def do_scheduler_step(self):
        pass


class NTSNetTrainer(Trainer):
    """Examples/NTSNet.py: criterion = NTSLoss on the model's five outputs; Adam over all parameters with lr and
    weight_decay (the base Trainer's); LinearLR(lr_warmup_decay, warmup_epochs) into CosineAnnealingLR(T_max -
    warmup_epochs) through SequentialLR, stepped once per epoch.  Training and validation accuracy are top-1 on
    concat_logits; the training step has no host synchronisation, so ``cuda_graph: true`` captures and replays it."""

    def get_criterion(self, config):
        from .losses import NTSLoss
        return NTSLoss(config)

    def get_scheduler(self, config):
        return _warmup_cosine(self.optimizer, config, self.total_epoch)


class _EpochCosine:
    """Examples/APCNN.py:69-81: lr(epoch) = lr / 2 (cos(pi (epoch % E) / E) + 1) on every group's initial lr, set at the start
    of each epoch; there is no other scheduler."""

    def __init__(self, opt, epochs):
        self.opt, self.E = opt, epochs

    def set_epoch(self, epoch):
        import math
        for g in self.opt.param_groups:
            g['lr'] = float(g['initial_lr'] / 2 * (math.cos(math.pi * (epoch % self.E) / self.E) + 1))

    def state_dict(self):
        return {}

    def load_state_dict(self, sd):
        pass


class APCNNTrainer(Trainer):
    """Examples/APCNN.py: the reference's transforms (TrivialAugmentWide in training); criterion = APCNNLoss (the sum of the
    eight cross-entropies); SGD with momentum 0.9 and weight_decay in two groups, conv1..layer3 at lr / 10 and layer4 with
    everything after it at lr (the reference's children()[:7] / [7:]); the cosine of the epoch set in on_start_epoch.
    Training and validation accuracy are top-1 on out_mean; validation runs both stages in eval mode (no drop block).  The
    step has no host synchronisation, so ``cuda_graph: true`` captures and replays it."""

    EARLY = ('conv1', 'bn1', 'layer1', 'layer2', 'layer3')

    def get_transformers(self, config):
        """Examples/APCNN.py:18-34."""
        from torchvision.transforms import autoaugment, transforms
        from torchvision.transforms.functional import InterpolationMode
        norm = transforms.Normalize([0.485, 0.456, 0.406], [0.229, 0.224, 0.225])
        return {
            'train': transforms.Compose([transforms.Resize((config.resize_size, config.resize_size)),
                                         transforms.RandomCrop(config.image_size), transforms.RandomHorizontalFlip(),
                                         autoaugment.TrivialAugmentWide(interpolation=InterpolationMode.BILINEAR),
                                         transforms.ToTensor(), norm]),
            'val': transforms.Compose([transforms.Resize((config.resize_size, config.resize_size)),
                                       transforms.CenterCrop(config.image_size), transforms.ToTensor(), norm]),
        }

    def get_criterion(self, config):
        from .losses import APCNNLoss
        return APCNNLoss(config)

    def param_groups(self):
        named = list(self.get_model_module().named_parameters())
        return [([p for n, p in named if n.split('.')[0] in self.EARLY], 0.1),
                ([p for n, p in named if n.split('.')[0] not in self.EARLY], 1.0)]

    get_optimizer = _momentum_sgd

    def get_scheduler(self, config):
        return _EpochCosine(self.optimizer, self.total_epoch)

    def on_start_epoch(self, config):
        self.scheduler.set_epoch(self.epoch)

    def do_scheduler_step(self):
        pass

    def forward_model(self, images, labels):
        return self.model(images, labels)


class MGE_CNNTrainer(Trainer):
    """Examples/MGE_CNN.py: criterion = MGECNNLoss (the mean of the ten label-smoothed cross-entropies); Adam with weight_decay
    in two groups, get_params('classifier') at lr and get_params('extractor') (the four trunks) at lr x lr_rate (default
    0.1); LinearLR(lr_warmup_decay, warmup_epochs) into CosineAnnealingLR(T_max - warmup_epochs), stepped once per epoch.
    Training and validation accuracy are top-1 on logits_gate.  The step has no host synchronisation, so
    ``cuda_graph: true`` captures and replays it.

    cls_cat_a, which forward never uses, stays out of the flat buffers: it never has a gradient, so torch's Adam skips it,
    weight decay included, and a zero gradient in the fused Adam would decay it."""

    def get_criterion(self, config):
        from .losses import MGECNNLoss
        return MGECNNLoss(config)

    def param_groups(self):
        m = self.get_model_module()
        oc = self.config.train.optimizer
        unused = {id(p) for p in m.cls_cat_a.parameters()}
        return [([p for p in m.get_params('classifier') if id(p) not in unused], 1.0),
                (list(m.get_params('extractor')), oc.lr_rate if 'lr_rate' in oc else 0.1)]

    def get_scheduler(self, config):
        return _warmup_cosine(self.optimizer, config, self.total_epoch)


class CINTrainer(Trainer):
    """Examples/CIN.py: class-balanced batches (n_classes x n_samples images); criterion = CINLoss (cross-entropy +
    alpha x the contrastive term through the criterion's own projection ``h``), moved to the device; SGD over two groups,
    the model's parameters and the criterion's, both at lr, with the yaml's weight_decay and momentum (the reference passes
    none: 0 unless the yaml sets one); LinearLR warm-up into cosine annealing over T_max - warmup_epochs.  The step has no
    host synchronisation, so ``cuda_graph: true`` captures and replays it.

    save_model writes the model alone, the reference's format; save_checkpoint adds ``criterion``, the state of ``h``
    (51 M weights with the shipped config), which load_checkpoint restores, so that ``h`` and its slice of the optimizer
    resume together.  A checkpoint without it keeps the freshly initialised ``h``, with a warning."""

    def get_dataloader(self, config):
        return _balanced_loaders(self, config)

    def get_criterion(self, config):
        from .losses import CINLoss
        return self.to_device(CINLoss(config))

    def param_groups(self):
        return [(list(self.get_model_module().parameters()), 1.0), (list(self.criterion.parameters()), 1.0)]

    def get_scheduler(self, config):
        return _warmup_cosine(self.optimizer, config, self.total_epoch)

    def checkpoint_state(self):
        ck = super().checkpoint_state()
        ck['criterion'] = {k: v.detach().cpu().clone() for k, v in self.criterion.state_dict().items()}
        return ck

    def restore_checkpoint(self, ck, path):
        super().restore_checkpoint(ck, path)
        if 'criterion' in ck:
            self.criterion.load_state_dict(ck['criterion'])
        else:
            self.logger.warning('checkpoint %s has no criterion state: the projection h of CINLoss keeps its fresh '
                                'initialisation', path)


class BaselineTrainer(Trainer):
    """Examples/Baseline.py: the plain classifier (ResNet50 in configs/Baseline.yaml) with RandomResizedCrop(224) and a flip
    for training, Resize(256) and CenterCrop(224) for validation.  Everything else is the base Trainer's, which is what the
    reference's Example restates: cross-entropy with label smoothing 0.1, Adam over all parameters with the yaml's lr and
    weight_decay, and CosineAnnealingLR(T_max, eta_min) stepped once per epoch.  The step has no host synchronisation, so
    ``cuda_graph: true`` captures and replays it."""

    def get_transformers(self, config):
        """Examples/Baseline.py:13-27 (fixed sizes: the reference does not read the transformer config)."""
        from torchvision import transforms
        norm = transforms.Normalize(mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225))
        return {
            'train': transforms.Compose([transforms.RandomResizedCrop((224, 224)), transforms.RandomHorizontalFlip(),
                                         transforms.ToTensor(), norm]),
            'val': transforms.Compose([transforms.Resize(256), transforms.CenterCrop(224), transforms.ToTensor(), norm]),
        }


class PCResNetTrainer(Trainer):
    """Examples/PairConfusion.py: criterion = PairwiseConfusionLoss (cross-entropy + lambda_a x the Euclidean confusion of
    the pairs (i, B/2 + i)); Adam with weight_decay in two groups, ``fc`` at lr and every other parameter at 0.1 x lr;
    LinearLR(lr_warmup_decay, warmup_epochs) into CosineAnnealingLR(T_max - warmup_epochs), stepped once per epoch.  The
    base Trainer's transforms, as in the reference.  ``fc`` is listed last so that its gradient, the first one backward
    produces, is all-reduced while the trunk's is still being computed.  The step has no host synchronisation, so
    ``cuda_graph: true`` captures and replays it.

    Under torchrun each rank pairs the two halves of its own batch of B / world images.  Its loss is lambda / (B / world)
    times a sum over B / (2 world) pairs, and the gradient all-reduce averages the ranks, so the objective is the
    reference's: lambda / B times a sum over B / 2 random pairs.  Only which random images get paired differs.  A rank's
    batch must therefore be even: batch_size / world must be even (a ValueError otherwise, when the loaders are built), and
    each rank's training loader drops its final partial batch, which could be odd.  On one GPU the loaders are the base
    Trainer's and an odd final batch raises in the criterion, as in the reference."""

    def get_dataloader(self, config):
        loaders = super().get_dataloader(config)
        if self.world > 1:
            if (config.batch_size // self.world) % 2:
                raise ValueError(f'PCResNetTrainer: dataset.batch_size={config.batch_size} over {self.world} ranks gives '
                                 f'{config.batch_size // self.world} images per rank, which must be even (the criterion '
                                 'pairs the two halves of each rank\'s batch)')
            from torch.utils.data import DataLoader
            t = loaders['train']
            loaders['train'] = DataLoader(t.dataset, t.batch_size, num_workers=t.num_workers, pin_memory=t.pin_memory,
                                          sampler=t.sampler, collate_fn=t.collate_fn, drop_last=True)
        return loaders

    def get_criterion(self, config):
        from .losses import PairwiseConfusionLoss
        return PairwiseConfusionLoss(config)

    def param_groups(self):
        m = self.get_model_module()
        fc = {id(p) for p in m.fc.parameters()}
        return [([p for p in m.parameters() if id(p) not in fc], 0.1), (list(m.fc.parameters()), 1.0)]

    def get_scheduler(self, config):
        return _warmup_cosine(self.optimizer, config, self.total_epoch)


TRAINERS = {'BCNN': BCNNTrainer, 'CBCNN': CBCNNTrainer, 'MPN': MPNTrainer, 'PeerLearning': PeerLearningTrainer,
            'OSMENet': OSMENetTrainer}
# TRAINERS keeps the key set it has always had, so code that enumerates it sees no change; the command line dispatches
# over every method, APINet, DCL, ProtoTreeNet, InterpPartsNet, NTSNet, APCNN, MGE_CNN, CIN, Baseline and PairConfusion
# included.
ALL_TRAINERS = dict(TRAINERS, APINet=APINetTrainer, DCL=DCLTrainer, ProtoTreeNet=ProtoTreeTrainer,
                   InterpPartsNet=InterpPartsNetTrainer, NTSNet=NTSNetTrainer, APCNN=APCNNTrainer, MGE_CNN=MGE_CNNTrainer,
                   CIN=CINTrainer, Baseline=BaselineTrainer, PairConfusion=PCResNetTrainer)


def main(argv=None):
    argv = list(sys.argv[1:] if argv is None else argv)
    if not argv or argv[0] not in ALL_TRAINERS:
        raise SystemExit(f'usage: python -m hawkeye_b200.examples {{{",".join(ALL_TRAINERS)}}} --config <yaml>')
    from .config import setup_config
    trainer = ALL_TRAINERS[argv[0]](setup_config(argv[1:]))
    trainer.train()


if __name__ == '__main__':
    main()
