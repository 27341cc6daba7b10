"""Initialisers / helpers mirrored from the reference's model/utils.py:5-28 (same RNG call order so that the
same torch seed gives the same weights), and the loader of torchvision's pretrained checkpoints."""
import logging
import os

import torch
import torch.nn as nn

from ._lib import HawkeyeLibError


def initialize_weights(m):
    if isinstance(m, nn.Conv2d):
        nn.init.kaiming_normal_(m.weight, mode='fan_out', nonlinearity='relu')
        if m.bias is not None:
            nn.init.constant_(m.bias, 0)
    elif isinstance(m, nn.BatchNorm2d):
        nn.init.constant_(m.weight, 1)
        nn.init.constant_(m.bias, 0)
    elif isinstance(m, nn.Linear):
        nn.init.kaiming_normal_(m.weight.data)
        if m.bias is not None:
            nn.init.constant_(m.bias.data, val=0)


def load_state_dict(model, state_dict):
    """Shape-filtered load (model/utils.py:24-28); also strips a DataParallel ``module.`` prefix (train.py:369-376)."""
    state_dict = {(k[7:] if k.startswith('module.') else k): v for k, v in state_dict.items()}
    model_dict = model.state_dict()
    model_dict.update({k: v for k, v in state_dict.items() if k in model_dict and v.shape == model_dict[k].shape})
    model.load_state_dict(model_dict)


def rename_state(state, names):
    """The tensors of ``state`` whose top-level name is a key of ``names``, renamed to its value ('' drops the name:
    ``features.0.weight`` -> ``0.weight``); every other tensor is left out."""
    out = {}
    for k, v in state.items():
        head, _, rest = k.partition('.')
        if head in names:
            out[names[head] + '.' + rest if names[head] else rest] = v
    return out


def load_pretrained(module, env, arch, names, own=()):
    """torchvision's ``arch`` checkpoint at $``env`` into ``module``, its top-level names mapped by ``names`` (see
    ``rename_state``).  Only the mapped tensors load, so torchvision's ``fc.*`` is ignored unless mapped; a file that lacks
    any tensor of the mapped modules raises, and so does a shape mismatch; ``own`` lists substrings of the module's keys
    that torchvision's checkpoint does not have by design (they keep their initial values).  Without the file the module keeps its own
    (random) initialisation, with a warning unless HAWKEYE_ALLOW_RANDOM_INIT=1 (benchmarks and parity tests).  -> module"""
    path = os.environ.get(env)
    if not (path and os.path.exists(path)):
        if os.environ.get('HAWKEYE_ALLOW_RANDOM_INIT', '0') != '1':
            logging.getLogger('hawkeye_b200').warning(
                'no %s checkpoint at $%s (%r): the weights keep the reference\'s RANDOM initialisation.  Point %s at '
                'torchvision\'s %s .pth, or set HAWKEYE_ALLOW_RANDOM_INIT=1 (benchmarks / parity tests) to silence this.',
                arch, env, path, env, arch)
        return module
    missing, _ = module.load_state_dict(rename_state(torch.load(path, map_location='cpu'), names), strict=False)
    missing = [k for k in missing if not any(o in k for o in own)]
    source = {v: k for k, v in names.items()}             # the module's top-level name -> the checkpoint's
    if '' in source:
        lacking = [source[''] + '.' + k for k in missing]
    else:
        lacking = [source[h] + '.' + r for h, _, r in (k.partition('.') for k in missing) if h in source]
    if lacking:
        raise HawkeyeLibError(f'${env} = {path} lacks {len(lacking)} tensors of {arch}, first {lacking[:4]}')
    return module
