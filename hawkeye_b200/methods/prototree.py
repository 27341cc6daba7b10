"""ProtoTree (neural prototype trees, Nauta et al., CVPR 2021) with the reference's surface
(model/methods/ProtoTree/ProtoTreeNet.py, prototree.py).

Same constructor, attributes (``backbone`` = the ResNet-50 trunk, ``neck_conv`` = 1x1 convolution + sigmoid, ``tree``,
``tree.prototype_layer.prototype_vectors``) and 832-entry ``state_dict`` at the shipped height 9, so reference checkpoints
load strictly.  ``forward(x)`` returns ``(pred, info)``; ``info['pa_tensor']`` and ``info['ps']`` map node indices to [N, 1]
views of one dense tensor each, as the reference's dicts do.

Prototype row k belongs to the k-th branch in pre-order (the reference's ``node.index`` order among branches).  The
reference maps rows to branches through ``zip(range(P), self.branches)`` over a set ordered by object hash
(prototree.py:51), so that mapping changes from process to process and a reference checkpoint does not record it; this
package fixes it.  The leaf parameters are one [L, K] tensor, ``tree.leaf_params``, that state-dict hooks save and load under
the reference's nested keys (``tree._root.l.….l._dist_params``); there are no per-node modules.

The neck, distances, routing, loss and leaf update run on hk_prototree_* and the GEMMs.  The reference's host-side NaN check
after every distance (l2conv.py:61-62) is a host synchronisation and is not made here.  Out of scope, and rejected:
``log_probabilities``, ``kontschieder_normalization``, ``kontschieder_train``, and the ``sample_max`` / ``greedy`` strategies.
"""
import collections.abc
import copy

import torch
import torch.nn as nn

from .. import _lib, ops, ops_prototree
from ..backbone.resnet import TRUNK_KEYS, resnet50
from ..registry import MODEL
from ..utils import rename_state


def _opt(cfg, key, default):
    return cfg[key] if key in cfg else default


def tree_layout(height):
    """-> (branch node indices, leaf node indices, leaf key paths), each in pre-order, of a complete tree of the given
    height (prototree.py:275-287: the left child of node i is i + 1, the right one i + 1 + the left subtree's size)."""
    branches, leaves, paths = [], [], []

    def walk(i, d, path):
        if d == height:
            leaves.append(i)
            paths.append(path)
            return 1
        branches.append(i)
        left = walk(i + 1, d + 1, path + ('l',))
        right = walk(i + 1 + left, d + 1, path + ('r',))
        return 1 + left + right

    walk(0, 0, ())
    return branches, leaves, ['_root.' + '.'.join(p) + '._dist_params' for p in paths]


class NodeViews(collections.abc.Mapping):
    """node index -> [N, 1] column of ``dense`` [N, columns] (no per-node work until a node is looked up)."""

    def __init__(self, dense, columns):
        self.dense, self._col = dense, columns

    def __getitem__(self, node):
        c = self._col[node]
        return self.dense[:, c:c + 1]

    def __iter__(self):
        return iter(self._col)

    def __len__(self):
        return len(self._col)


class PrototypeLayer(nn.Module):
    """L2Conv2D's parameter container (l2conv.py:11-22): prototype_vectors [P, D, W1, H1]."""

    def __init__(self, num_prototypes, num_features, w1, h1):
        super().__init__()
        self.prototype_vectors = nn.Parameter(torch.randn(num_prototypes, num_features, w1, h1), requires_grad=True)


class ProtoTree(nn.Module):
    SAMPLING_STRATEGIES = ['distributed', 'sample_max', 'greedy']

    def __init__(self, args):
        super().__init__()
        for k in ('log_probabilities', 'kontschieder_normalization', 'kontschieder_train'):
            if _opt(args, k, False):
                raise _lib.HawkeyeLibError(f'ProtoTree: model.{k} is not supported (the probability-space tree with softmax '
                                           'leaves is); set it to False')
        if int(_opt(args, 'W1', 1)) != 1 or int(_opt(args, 'H1', 1)) != 1:
            raise _lib.HawkeyeLibError(f'ProtoTree: prototypes of W1 x H1 = {_opt(args, "W1", 1)} x {_opt(args, "H1", 1)} '
                                       'are not supported, only 1 x 1 (the reference does not guarantee others either)')
        self.height = int(args.height)
        ops_prototree.check_height(self.height)
        self._num_classes = int(args.num_classes)
        self.num_features = int(args.num_features)
        branches, leaves, paths = tree_layout(self.height)
        self.num_prototypes = len(branches)
        self.prototype_shape = (1, 1, self.num_features)
        self._node_cols = {i: i for i in range(2 * len(leaves) - 1)}
        self._branch_cols = {n: k for k, n in enumerate(branches)}
        self._leaf_keys = paths
        dfo_off = bool(_opt(args, 'disable_derivative_free_leaf_optim', False))
        init = torch.randn if dfo_off else torch.zeros                     # leaf.py:18-23
        self.leaf_params = nn.Parameter(init(len(leaves), self._num_classes), requires_grad=dfo_off)
        self.prototype_layer = PrototypeLayer(self.num_prototypes, self.num_features, 1, 1)
        self.register_state_dict_post_hook(ProtoTree._save_leaves)
        self.register_load_state_dict_pre_hook(ProtoTree._load_leaves)

    @staticmethod
    def _save_leaves(module, state, prefix, local_metadata):
        """leaf_params [L, K] -> the reference's L nested [K] entries, ahead of the prototypes as the reference orders them."""
        theta = state.pop(prefix + 'leaf_params')
        rest = [(k, state.pop(k)) for k in list(state) if k.startswith(prefix)]
        for j, key in enumerate(module._leaf_keys):
            state[prefix + key] = theta[j]
        state.update(rest)

    @staticmethod
    def _load_leaves(module, state, prefix, local_metadata, strict, missing, unexpected, errors):
        keys = [prefix + k for k in module._leaf_keys]
        if all(k in state for k in keys):
            state[prefix + 'leaf_params'] = torch.stack([state.pop(k) for k in keys])

    @property
    def num_leaves(self):
        return self.leaf_params.shape[0]

    @property
    def num_branches(self):
        return self.num_prototypes

    def forward(self, xs, features, sampling_strategy='distributed'):
        """features [N, D, H, W] (the neck's output) -> (pred [N, K], info), prototree.py:97-147."""
        if sampling_strategy != 'distributed':
            raise _lib.HawkeyeLibError(f'ProtoTree: sampling_strategy={sampling_strategy!r} is not supported, only '
                                       "'distributed'")
        N, D, H, W = features.shape
        z = features.permute(0, 2, 3, 1).reshape(N, H * W, D)
        mind, _ = ops_prototree.PrototypeDistanceFn.apply(z, self.prototype_layer.prototype_vectors, False)
        return self.route(mind)

    def route(self, mind):
        pred, ps, pa = ops_prototree.RouteFn.apply(mind, self.leaf_params, self.height)
        return pred, {'pa_tensor': NodeViews(pa, self._node_cols), 'ps': NodeViews(ps, self._branch_cols)}


def inat_resnet50_state(path):
    """ProtoTreeNet.get_inat_resnet50_weight (ProtoTreeNet.py:41-59): ``module.backbone.*`` loses its prefix, ``cb_block``
    becomes ``layer4.2``, ``rb_block.*`` and ``module.classifier.*`` are dropped; other keys pass through unchanged."""
    sd = torch.load(path, map_location='cpu')
    out = copy.copy(sd)
    for k in sd:
        if k.startswith('module.backbone.cb_block'):
            out['layer4.2' + k.split('cb_block')[-1]] = sd[k]
            del out[k]
        elif k.startswith('module.backbone.rb_block'):
            del out[k]
        elif k.startswith('module.backbone.'):
            out[k.split('backbone.')[-1]] = sd[k]
            del out[k]
        elif k.startswith('module.classifier'):
            del out[k]
    return out


@MODEL.register
class ProtoTreeNet(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.config = config
        ops.check_num_classes(config.num_classes)
        self.backbone = resnet50(pretrained=True)              # children()[:-2] of the reference ResNet, same keys
        pretrain = _opt(_opt(config, 'backbone', {}), 'pretrain', '')
        if pretrain:
            import os
            if not os.path.isfile(pretrain):
                raise _lib.HawkeyeLibError(f'ProtoTreeNet: model.backbone.pretrain={pretrain!r} is not a file (the iNat '
                                           'ResNet-50 checkpoint); set model.backbone.pretrain to its path, or to \'\'')
            # resnet.load_state_dict(state_dict, strict=False) on the full ResNet: keys outside the trunk are ignored
            self.backbone.load_state_dict(rename_state(inat_resnet50_state(pretrain), TRUNK_KEYS), strict=False)
        self.neck_conv = nn.Sequential(nn.Conv2d(self.backbone.out_channels, config.num_features, kernel_size=1, bias=False),
                                       nn.Sigmoid())
        self.tree = ProtoTree(config)
        with torch.no_grad():                                  # ProtoTreeNet.py:31-33
            nn.init.normal_(self.tree.prototype_layer.prototype_vectors, mean=0.5, std=0.1)
            nn.init.xavier_normal_(self.neck_conv[0].weight, gain=nn.init.calculate_gain('sigmoid'))

    def forward(self, x):
        feat = self.backbone(x)
        w = self.neck_conv[0].weight
        if feat.dim() != 4 or w.dim() != 4 or w.shape[1] != feat.shape[1] or w.shape[2:] != (1, 1):
            raise _lib.HawkeyeLibError(f'ProtoTree neck: map {tuple(feat.shape)} and weight {tuple(w.shape)} are not a '
                                       '[N, C, H, W] map and a [D, C, 1, 1] convolution')
        N, _, H, W = feat.shape
        # the neck's pre-activation [N, H*W, D], position-major: the layout hk_prototree_dist_fwd reads
        c = ops.Conv1x1Fn.apply(ops.ToNHWCFn.apply(feat), w, None).view(N, H * W, w.shape[0])
        mind, _ = ops_prototree.PrototypeDistanceFn.apply(c, self.tree.prototype_layer.prototype_vectors, True)
        return self.tree.route(mind)

    def prediction(self, outputs):
        return outputs[0]
