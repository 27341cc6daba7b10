"""Import the UNMODIFIED reference tree as the parity oracle (TEST INFRASTRUCTURE ONLY).

Only tests/, tests/golden/make_golden.py and bench.py's cpu_baseline leg may
import this module.  Nothing under hawkeye_b200/ imports it.

Reference root resolution: $HAWKEYE_REF, then baseline/_ref.
The yacs / tensorboardX stand-ins under oracle/_shims are used only when the real
packages fail to import.  ``pretrained=True`` is hard-coded in the reference
(model/methods/BCNN.py:38, CBCNN.py:21, MPNCOV.py:28) and would hit the network
(model/backbone/vgg.py:83-85, resnet.py:264-266); we force it off so the
reference's own random initialisers (model/utils.py:5-16) are what runs.
"""
import os
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
_REPO = os.path.dirname(_HERE)


def find_reference_root():
    for cand in (os.environ.get("HAWKEYE_REF"), os.path.join(_REPO, "baseline", "_ref")):
        if cand and os.path.isfile(os.path.join(cand, "model", "methods", "BCNN.py")):
            return cand
    return None


def available():
    return find_reference_root() is not None


_loaded = None


def load_reference():
    """Returns the reference's top-level ``model`` package (registers all MODEL entries)."""
    global _loaded
    if _loaded is not None:
        return _loaded
    root = find_reference_root()
    if root is None:
        raise RuntimeError("reference tree not found (set $HAWKEYE_REF)")
    sys.dont_write_bytecode = True
    try:
        import yacs.config  # noqa: F401
    except Exception:
        sys.path.insert(0, os.path.join(_HERE, "_shims"))
    try:
        import tensorboardX  # noqa: F401
    except Exception:
        shim = os.path.join(_HERE, "_shims")
        if shim not in sys.path:
            sys.path.insert(0, shim)
    if root not in sys.path:
        sys.path.insert(0, root)
    # neutralise the hub download before `import model` binds vgg16/resnet50
    import importlib
    import torch.hub

    def _no_download(*a, **k):
        raise RuntimeError("offline: pretrained weights are not available")

    torch.hub.load_state_dict_from_url = _no_download
    vgg = importlib.import_module("model.backbone.vgg")
    resnet = importlib.import_module("model.backbone.resnet")
    _ovgg, _ores = vgg._vgg, resnet._resnet

    def _vgg_np(arch, cfg, batch_norm, pretrained, progress, **kw):
        return _ovgg(arch, cfg, batch_norm, False, progress, **kw)

    def _resnet_np(arch, block, layers, pretrained, progress, **kw):
        return _ores(arch, block, layers, False, progress, **kw)

    vgg._vgg = _vgg_np
    resnet._resnet = _resnet_np
    model = importlib.import_module("model")
    _loaded = model
    return model


def cfg(**kw):
    """A CfgNode for ``MODEL.get(name)(cfg)`` built from keyword args."""
    load_reference()
    from yacs.config import CfgNode
    return CfgNode(dict(kw))
