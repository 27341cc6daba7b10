"""Plugin registry with the reference's surface (model/registry.py:3-4, utils/repository.py:10-13):
``MODEL`` / ``BACKBONE`` are dict subclasses; ``register(module)`` keys by ``__name__`` and asserts
uniqueness; lookup is ``MODEL.get(config.name)(config)`` (train.py:161-162)."""


class Repository(dict):
    def register(self, module):
        assert module.__name__ not in self
        self[module.__name__] = module
        return module


MODEL = Repository()
BACKBONE = Repository()


def install_into(model_registry, names=('BCNN', 'CBCNN', 'MPN', 'CIN', 'PeerLearningNet'), backbone_registry=None):
    """Drop-in: overwrite the reference's own ``model.registry.MODEL`` entries with the H100-native classes,
    so an unmodified Hawkeye ``Trainer`` (train.py:158-169) builds them via ``MODEL.get(name)(config)``.  Any registered
    name may be listed (``'APINet'``, ``'DCL'``, ``'NTSNet'``, ...)."""
    for n in names:
        if n in MODEL:
            dict.__setitem__(model_registry, n, MODEL[n])
    if backbone_registry is not None:
        for n, f in BACKBONE.items():
            dict.__setitem__(backbone_registry, n, f)
    return model_registry
