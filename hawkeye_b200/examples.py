"""Trainer subclasses of the hot-path methods with the reference's Examples/ surface:
``python -m hawkeye_b200.examples {BCNN,CBCNN,MPN,PeerLearning,OSMENet,APINet} --config <yaml>`` replaces
``python Examples/<Method>.py --config <yaml>`` (same yaml files; one process per GPU under torchrun instead of nn.DataParallel).

Only what the reference's Examples override is overridden here: which parameters train, with which learning rates, and
which LR schedule — the step itself is ``Trainer.batch_training``.
"""
import sys

from .train import PeerLearningTrainer, Trainer, _Cosine, _Plateau


def _warmup_cosine(opt, config, total_epoch):
    return _Cosine(opt, config['T_max'] if 'T_max' in config else total_epoch, 0.0,
                   config['warmup_epochs'] if 'warmup_epochs' in config else 0,
                   config['lr_warmup_decay'] if 'lr_warmup_decay' in config else 0.01)


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

    def batch_validate(self, data):
        import torch
        from .train import accuracy
        images, labels = self.to_device(data['img']), self.to_device(data['label'])
        with torch.no_grad():
            pred, _ = self.model(images)
        self.average_meters['acc'].update(accuracy(pred, labels, 1), images.size(0))


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
        return _FrozenWarmupCosine(self.optimizer, config['T_max'] if 'T_max' in config else self.total_epoch, 0.0,
                                   config['warmup_epochs'] if 'warmup_epochs' in config else 0,
                                   config['lr_warmup_decay'] if 'lr_warmup_decay' in config else 0.01)

    def forward_model(self, images, labels):
        return self.model(images, labels, flag='train')

    def meter_counts(self, n):
        return 8 * n, 4 * n


TRAINERS = {'BCNN': BCNNTrainer, 'CBCNN': CBCNNTrainer, 'MPN': MPNTrainer, 'PeerLearning': PeerLearningTrainer,
            'OSMENet': OSMENetTrainer}
# TRAINERS keeps the key set it has always had, so code that enumerates it sees no change; the command line dispatches
# over every method, APINet included.
ALL_TRAINERS = dict(TRAINERS, APINet=APINetTrainer)


def main(argv=None):
    argv = list(sys.argv[1:] if argv is None else argv)
    if not argv or argv[0] not in ALL_TRAINERS:
        raise SystemExit(f'usage: python -m hawkeye_b200.examples {{{",".join(ALL_TRAINERS)}}} --config <yaml>')
    from .config import setup_config
    trainer = ALL_TRAINERS[argv[0]](setup_config(argv[1:]))
    trainer.train()


if __name__ == '__main__':
    main()
