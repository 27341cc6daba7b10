"""Training-step plumbing around the kernels: flat parameter/gradient buffers, fused optimizers and the
one-process-per-GPU data-parallel gradient all-reduce that replaces ``nn.DataParallel`` (reference
train.py:220-228).  torch.distributed/NCCL is plumbing here; all arithmetic runs in libhawkeye_b200.so.
"""
import contextlib
import os

import torch
import torch.distributed as dist

from . import _lib


def _align(n, a=4):
    return (n + a - 1) // a * a


class FlatParams:
    """Re-homes the trainable parameters of ``module`` into ONE flat fp32 buffer and their gradients into
    another, keeping every ``nn.Parameter`` (and therefore ``state_dict()`` keys/shapes) intact as views.

    One flat gradient buffer = one NCCL all-reduce per bucket and one fused optimizer launch per step.
    Slices are padded to 16 bytes so TMA / float4 alignment holds for every view.
    ``groups``: optional list of lists of parameters -> contiguous slices (buckets / param groups).
    """

    def __init__(self, module_or_params, groups=None):
        if groups is None:
            params = list(module_or_params.parameters()) if hasattr(module_or_params, 'parameters') \
                else list(module_or_params)
            groups = [[p for p in params if p.requires_grad]]
        groups = [[p for p in g if p.requires_grad] for g in groups]
        self.groups = groups
        self.params = [p for g in groups for p in g]
        if not self.params:
            raise ValueError('no trainable parameters')
        dev = self.params[0].device
        total = sum(_align(p.numel()) for p in self.params)
        self.flat = torch.zeros(total, device=dev, dtype=torch.float32)
        self.grad = torch.zeros(total, device=dev, dtype=torch.float32)
        self.group_slices = []
        off = 0
        for g in groups:
            start = off
            for p in g:
                n = p.numel()
                view = self.flat[off:off + n].view_as(p)
                view.copy_(p.data)
                p.data = view
                p.grad = self.grad[off:off + n].view_as(p)
                off += _align(n)
            self.group_slices.append((start, off))
        self.numel = total

    def zero_grad(self):
        self.grad.zero_()
        for p in self.params:          # keep .grad pointing at the flat views (autograd then accumulates in place)
            if p.grad is None or p.grad.data_ptr() < self.grad.data_ptr() or \
                    p.grad.data_ptr() >= self.grad.data_ptr() + self.numel * 4:
                self.rebind_grads()
                break

    def rebind_grads(self):
        off = 0
        for p in self.params:
            n = p.numel()
            p.grad = self.grad[off:off + n].view_as(p)
            off += _align(n)


class FusedSGD:
    """torch.optim.SGD(momentum, weight_decay) semantics (Examples/BCNN.py:40) as ONE kernel over the flat buffers.
    ``param_groups`` mirrors torch's so LR schedulers (ReduceLROnPlateau etc.) can drive ``lr``."""

    def __init__(self, flat: FlatParams, lr, momentum=0.0, weight_decay=0.0, group_lrs=None):
        self.flat = flat
        self.buf = torch.zeros_like(flat.flat)
        self.defaults = dict(lr=lr, momentum=momentum, weight_decay=weight_decay)
        self.param_groups = []
        for gi, g in enumerate(flat.groups):
            glr = group_lrs[gi] if group_lrs else lr
            self.param_groups.append(dict(params=g, lr=glr, momentum=momentum, weight_decay=weight_decay, initial_lr=glr))
        self.first = True
        self.grad_scale = 1.0
        self.state = {}

    def zero_grad(self, set_to_none=False):
        self.flat.zero_grad()

    def step(self, closure=None):
        s = _lib.stream_ptr()
        for pg, (a, b) in zip(self.param_groups, self.flat.group_slices):
            n = b - a
            _lib.call('hk_sgd_momentum', self.flat.flat[a:b], self.flat.grad[a:b], self.buf[a:b], n, float(pg['lr']),
                      float(pg['momentum']), float(pg['weight_decay']), float(self.grad_scale), int(self.first), s)
        self.first = False

    def state_dict(self):
        return dict(buf=self.buf, first=self.first, param_groups=[{k: v for k, v in g.items() if k != 'params'}
                                                                   for g in self.param_groups])

    def load_state_dict(self, sd):
        self.buf.copy_(sd['buf'])
        self.first = sd['first']
        for g, s in zip(self.param_groups, sd['param_groups']):
            g.update(s)


class FusedAdam:
    """torch.optim.Adam semantics (train.py:214-215, Examples/MPN.py:14-18) over the flat buffers."""

    def __init__(self, flat: FlatParams, lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, group_lrs=None):
        self.flat = flat
        self.m = torch.zeros_like(flat.flat)
        self.v = torch.zeros_like(flat.flat)
        self.betas, self.eps = betas, eps
        self.param_groups = [dict(params=g, lr=(group_lrs[gi] if group_lrs else lr), weight_decay=weight_decay,
                                  initial_lr=(group_lrs[gi] if group_lrs else lr)) for gi, g in enumerate(flat.groups)]
        self.t = 0
        self.grad_scale = 1.0
        self.state = {}

    def zero_grad(self, set_to_none=False):
        self.flat.zero_grad()

    def step(self, closure=None):
        self.t += 1
        s = _lib.stream_ptr()
        for pg, (a, b) in zip(self.param_groups, self.flat.group_slices):
            _lib.call('hk_adam', self.flat.flat[a:b], self.flat.grad[a:b], self.m[a:b], self.v[a:b], b - a,
                      float(pg['lr']), float(self.betas[0]), float(self.betas[1]), float(self.eps),
                      float(pg['weight_decay']), float(self.grad_scale), self.t, s)

    def state_dict(self):
        return dict(m=self.m, v=self.v, t=self.t, param_groups=[{k: v for k, v in g.items() if k != 'params'}
                                                                for g in self.param_groups])

    def load_state_dict(self, sd):
        self.m.copy_(sd['m'])
        self.v.copy_(sd['v'])
        self.t = sd['t']
        for g, s in zip(self.param_groups, sd.get('param_groups', [])):     # lr reduced by a plateau scheduler survives
            g.update(s)


EMA_COLS = 5                    # hk_ema_cols(): model pointer, average pointer, elements, kind, first chunk
_EMA_KINDS = {torch.float32: 0, torch.int64: 1}


class ModelEMA:
    """Exponential moving average of ``model``: what ``torch.optim.swa_utils.AveragedModel(model, avg_fn=lambda a, p, n:
    decay * a + (1 - decay) * p, use_buffers=True)`` computes, torchvision's ``ExponentialMovingAverage``, in one launch
    (``hk_ema_update``) with no host synchronisation.

    The average covers the flat parameter buffer ``flat`` (one float4 segment), every parameter outside it and every buffer
    in ``model.buffers()``.  Only float32 and int64 tensors are supported; another dtype raises ValueError naming the
    tensor.  If the flat buffer holds tensors other than the model's (CIN's criterion), those are averaged and swapped
    along with the rest, but no state dict contains them.  The counter ``n_averaged`` is an int64 on the device: the
    next update copies the model when it is 0.

    ``swapped()`` evaluates the averaged weights by exchanging contents in place (``hk_ema_swap``), so every pointer, and
    therefore every captured CUDA graph and every view into the flat buffer, stays valid."""

    def __init__(self, model, flat: FlatParams, decay):
        decay = float(decay)
        if not 0.0 <= decay <= 1.0:
            raise ValueError(f'ModelEMA: decay {decay} outside [0, 1]')
        self.model, self.decay = model, decay
        lo, hi = flat.flat.data_ptr(), flat.flat.data_ptr() + flat.numel * 4
        self.model_tensors, self.averages = [flat.flat], [flat.flat.detach().clone()]
        for name, t in list(model.named_parameters()) + list(model.named_buffers()):
            if t.dtype not in _EMA_KINDS:
                raise ValueError(f'ModelEMA: {name} is {t.dtype}; only float32 and int64 tensors can be averaged')
            if lo <= t.data_ptr() < hi or t.numel() == 0:
                continue
            if t.device != flat.flat.device or not t.is_contiguous():
                raise ValueError(f'ModelEMA: {name} must be a contiguous tensor on {flat.flat.device}')
            self.model_tensors.append(t.detach())
            self.averages.append(t.detach().clone())
        table = torch.zeros(len(self.model_tensors), EMA_COLS, dtype=torch.int64)
        for row, t, a in zip(table, self.model_tensors, self.averages):
            row[:4] = torch.tensor([t.data_ptr(), a.data_ptr(), t.numel(), _EMA_KINDS[t.dtype]])
        self.nseg = table.shape[0]
        self.chunks = _lib.query('hk_ema_plan', table, self.nseg)
        if self.chunks <= 0:
            raise _lib.HawkeyeLibError(f'hk_ema_plan failed (rc={self.chunks}): {_lib.lib().hk_last_error().decode()}')
        self.table = table.to(flat.flat.device)
        self.n_averaged = torch.zeros((), dtype=torch.int64, device=flat.flat.device)

    def update(self, reset_after=False):
        """One averaging step of the model's current weights; with ``reset_after`` the counter is then set to 0, so the
        next update copies the weights again (torchvision's warm-up reset)."""
        _lib.call('hk_ema_update', self.table, self.nseg, self.chunks, self.n_averaged, self.decay, 1.0 - self.decay,
                  int(bool(reset_after)), _lib.stream_ptr())

    def reset(self):
        """Sets the counter to 0: the next update copies the model."""
        self.n_averaged.zero_()

    def swap(self):
        """Exchanges the contents of the model and the average; a second swap restores both bit for bit."""
        _lib.call('hk_ema_swap', self.table, self.nseg, self.chunks, _lib.stream_ptr())

    @contextlib.contextmanager
    def swapped(self):
        """The averaged weights in the model for the duration of the block, the model's own afterwards."""
        self.swap()
        try:
            yield self.model
        finally:
            self.swap()

    def model_state_dict(self):
        """The average as a plain state_dict of the model, on the host: ``model.state_dict()`` with the average swapped
        in, so the model's state-dict hooks apply (ProtoTree's nested leaf keys)."""
        with self.swapped():
            return {k: v.detach().cpu().clone() for k, v in self.model.state_dict().items()}

    def state_dict(self):
        return averaged_state(self.n_averaged.detach().cpu().clone(), self.model_state_dict())

    def load_state_dict(self, sd):
        """Loads a ``state_dict()`` (``AveragedModel``'s layout) through the model's ``load_state_dict``, strictly."""
        with self.swapped():
            self.model.load_state_dict(averaged_model_state(sd))
        self.n_averaged.copy_(torch.as_tensor(sd['n_averaged']))


def averaged_state(n_averaged, model_state):
    """``AveragedModel.state_dict()``'s layout: ``n_averaged``, then the model's state_dict entries under ``module.``."""
    sd = {'n_averaged': n_averaged}
    sd.update(('module.' + k, v) for k, v in model_state.items())
    return sd


def averaged_model_state(sd):
    """The model's state_dict entries of an ``averaged_state`` dict."""
    return {k[len('module.'):]: v for k, v in sd.items() if k.startswith('module.')}


# ----------------------------------------------------------------------------------------------------------
# data parallelism: one process per GPU, gradient all-reduce (sum) over NCCL, averaged inside the optimizer
# ----------------------------------------------------------------------------------------------------------
def init_distributed(backend=None):
    """Reads RANK / LOCAL_RANK / WORLD_SIZE / MASTER_* from the environment (torchrun contract)."""
    world = int(os.environ.get('WORLD_SIZE', '1'))
    if world <= 1:
        return 0, 0, 1
    rank = int(os.environ['RANK'])
    local = int(os.environ.get('LOCAL_RANK', rank))
    if backend is None:
        backend = 'nccl' if torch.cuda.is_available() else 'gloo'
    if backend == 'nccl':
        torch.cuda.set_device(local)
    if not dist.is_initialized():
        kw = {}
        if backend == 'nccl':
            kw['device_id'] = torch.device('cuda', local)
        dist.init_process_group(backend=backend, **kw)
    return rank, local, world


class GradAllReduce:
    """Bucketed gradient all-reduce over the flat gradient buffer.

    ``early``: parameters whose gradients are complete early in backward (the 210 MB BCNN classifier, produced
    before the whole backbone backward).  Their slice is all-reduced on a side stream as soon as autograd has
    accumulated them, overlapping the backbone backward; the rest goes after backward.  The 1/world average is
    folded into the optimizer kernel (``grad_scale``), so the collective is a pure sum.
    """

    def __init__(self, flat: FlatParams, early_group=None, world=None):
        self.flat = flat
        self.world = world if world is not None else (dist.get_world_size() if dist.is_initialized() else 1)
        self.enabled = self.world > 1
        self.early_group = early_group
        self._pending = []
        self._early_work = None
        self._fired = 0
        self.comm_stream = None
        if not self.enabled:
            return
        if flat.flat.is_cuda:
            self.comm_stream = torch.cuda.Stream()
        if early_group is not None:
            self._early_params = flat.groups[early_group]
            for p in self._early_params:
                p.register_post_accumulate_grad_hook(self._hook)

    def _slice(self, gi):
        a, b = self.flat.group_slices[gi]
        return self.flat.grad[a:b]

    def _hook(self, p):
        self._fired += 1
        if self._fired == len(self._early_params):
            self._fired = 0
            self._launch(self._slice(self.early_group))

    def _launch(self, t):
        if self.comm_stream is not None:
            self.comm_stream.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(self.comm_stream):
                dist.all_reduce(t, op=dist.ReduceOp.SUM)
        else:
            dist.all_reduce(t, op=dist.ReduceOp.SUM)

    def finish(self):
        """Call after backward: reduce the remaining buckets, then make the compute stream wait for comm."""
        if not self.enabled:
            return
        for gi in range(len(self.flat.groups)):
            if gi != self.early_group:
                self._launch(self._slice(gi))
        if self.comm_stream is not None:
            torch.cuda.current_stream().wait_stream(self.comm_stream)
