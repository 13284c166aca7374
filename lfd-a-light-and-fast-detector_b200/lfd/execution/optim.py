# -*- coding: utf-8 -*-
"""FusedSGD -- `clip_grad_norm_` + `torch.optim.SGD.step` of the reference's optimizer hook
(lfd/execution/hooks/optimizer_hook.py:21-36; the shipped configs build torch.optim.SGD(momentum=0.9, weight_decay=1e-4),
e.g. WIDERFACE_train/WIDERFACE_LFD_L.py) as TWO kernel launches over the model's flat parameter / gradient buffers
(lfd_grad_sqnorm + lfd_sgd_step), instead of ~6 small kernels per parameter tensor.

It is a torch.optim.Optimizer: `param_groups` (and the dicts in it) are shared with the torch optimizer it was made from, so
lr schedulers and the warm-up hook that were built on the original optimizer keep driving the learning rate; `state_dict()` /
`load_state_dict()` use torch.optim.SGD's format (per-parameter 'momentum_buffer'), i.e. checkpoints stay interchangeable
with the reference's.

Like torch.optim.SGD, a parameter's momentum buffer starts as its first (weight-decayed) gradient, undamped: the flat runs whose
parameters have no buffer yet step with dampening 0 on their zeroed buffer slots, which gives exactly that.
"""
import ctypes as C

import torch

from .. import _native as nat
from .._train import flat_parameters

__all__ = ['FusedSGD']


class FusedSGD(torch.optim.Optimizer):

    def __init__(self, model, param_groups):
        """param_groups: torch.optim.SGD-style group dicts (shared, not copied)."""
        defaults = dict(lr=param_groups[0]['lr'], momentum=0.0, dampening=0.0, weight_decay=0.0, nesterov=False)
        super(FusedSGD, self).__init__([dict(g) for g in param_groups], defaults)
        self.param_groups = param_groups          # SHARED with the optimizer the schedulers were built on
        self.model = model
        self._flat, self._mom, self._runs = None, None, None
        self._sq = None
        self._pending = None      # momentum buffers loaded before the flat buffer exists
        self._has_buf = set()     # id() of the parameters that have a momentum buffer (stepped, or loaded from a state)
        for g in param_groups:
            if g.get('maximize'):
                raise NotImplementedError('FusedSGD implements minimisation only')

    @classmethod
    def from_torch(cls, optimizer, model):
        if type(optimizer) is not torch.optim.SGD:
            raise TypeError('FusedSGD.from_torch expects a torch.optim.SGD (got %s)' % type(optimizer).__name__)
        new = cls(model, optimizer.param_groups)
        new._torch_optimizer = optimizer
        optimizer._opt_called = True       # lr schedulers built on `optimizer` check that it stepped before they do
        if optimizer.state:
            new._pending = {id(p): st['momentum_buffer'] for p, st in optimizer.state.items() if st.get('momentum_buffer') is not None}
        return new

    # ------------------------------------------------------------------ flat buffers
    def _sync(self):
        flat = flat_parameters(self.model)
        if flat is not self._flat:
            old = self._state_buffers() if self._flat is not None else (self._pending or {})
            self._flat = flat
            self._mom = torch.zeros_like(flat.data)
            self._has_buf = set()
            for p, off in zip(flat.params, flat.offsets):
                buf = old.get(id(p))
                if buf is not None:
                    self._mom[off:off + p.numel()].copy_(buf.reshape(-1))
                    self._has_buf.add(id(p))
            self._pending = None
            self._sq = torch.zeros(1, dtype=torch.float64, device=flat.data.device)
            self._make_runs()
        elif tuple(p.requires_grad for p in flat.params) != self._requires_grad:      # parameters frozen / unfrozen since
            self._make_runs()
        return flat

    def _make_runs(self):
        """Maximal runs of flat slots with the same hyper-parameters and the same momentum-buffer state: (begin, end, group index,
        every parameter of the run has a buffer).  Frozen parameters (requires_grad False) have no gradient, and torch.optim.SGD
        skips them -- no weight decay, no momentum, no buffer: they are in no run."""
        group_of = {}
        for gi, g in enumerate(self.param_groups):
            for p in g['params']:
                group_of[id(p)] = gi
        runs = []
        self._requires_grad = tuple(p.requires_grad for p in self._flat.params)
        for p, off in zip(self._flat.params, self._flat.offsets):
            if id(p) not in group_of:
                raise ValueError('a model parameter is missing from the optimizer param_groups')
            if not p.requires_grad:
                continue
            end = off + (p.numel() + 3) // 4 * 4
            key = (group_of[id(p)], id(p) in self._has_buf)
            if runs and runs[-1][2:] == list(key) and runs[-1][1] == off:
                runs[-1][1] = end
            else:
                runs.append([off, end, key[0], key[1]])
        self._runs = runs

    def _state_buffers(self):
        return {id(p): self._mom[off:off + p.numel()].view(p.shape) for p, off in zip(self._flat.params, self._flat.offsets)
                if id(p) in self._has_buf}

    # ------------------------------------------------------------------ torch.optim.Optimizer interface
    def zero_grad(self, set_to_none=False):
        flat = self._sync()
        flat.attach_grads()
        flat.grad.zero_()

    @torch.no_grad()
    def step(self, closure=None, max_norm=0.0, grad_scale=1.0):
        """One SGD step over the flat buffers.  max_norm > 0: clip_grad_norm_(parameters, max_norm, norm_type=2) first; returns the
        total gradient norm (a 0-dim CUDA tensor, not synchronised) in that case."""
        if closure is not None:
            raise NotImplementedError('FusedSGD does not re-evaluate a closure')
        flat = self._sync()
        L = nat.lib()
        st = nat.stream_ptr()
        with torch.cuda.device(flat.data.device):
            if max_norm and max_norm > 0:
                nat.check(L.lfd_grad_sqnorm(nat.ptr(flat.grad), flat.numel, nat.ptr(self._sq), st))
            started = []
            for b, e, gi, has_buf in self._runs:
                g = self.param_groups[gi]
                mom = float(g.get('momentum', 0.0))
                # first step of a buffer: torch.optim.SGD sets buf = grad, i.e. momentum * 0 + (1 - 0) * grad on the zeroed slots
                damp = float(g.get('dampening', 0.0)) if has_buf else 0.0
                nat.check(L.lfd_sgd_step(C.c_void_p(flat.data.data_ptr() + 4 * b), C.c_void_p(flat.grad.data_ptr() + 4 * b),
                                         C.c_void_p(self._mom.data_ptr() + 4 * b), e - b, float(g['lr']), mom, damp,
                                         float(g.get('weight_decay', 0.0)), int(bool(g.get('nesterov', False))), float(max_norm or 0.0),
                                         float(grad_scale), nat.ptr(self._sq), st))
                if not has_buf and mom != 0.0:
                    started.append((b, e))
            if started:
                self._has_buf |= {id(p) for p, off in zip(flat.params, flat.offsets) if any(b <= off < e for b, e in started)}
                self._make_runs()
        if max_norm and max_norm > 0:
            return self._sq.sqrt() * abs(float(grad_scale))
        return None

    def state_dict(self):
        """torch.optim.SGD format."""
        flat = self._sync()
        index = {id(p): i for i, p in enumerate(p for g in self.param_groups for p in g['params'])}
        bufs = self._state_buffers()          # (torch.optim.SGD has no entry for a parameter that never stepped with momentum)
        state = {index[id(p)]: {'momentum_buffer': bufs[id(p)].clone()} for p in flat.params if id(p) in bufs}
        groups, n = [], 0
        for g in self.param_groups:
            d = {k: v for k, v in g.items() if k != 'params'}
            d['params'] = list(range(n, n + len(g['params'])))
            n += len(g['params'])
            groups.append(d)
        return {'state': state, 'param_groups': groups}

    def load_state_dict(self, state_dict):
        params = [p for g in self.param_groups for p in g['params']]
        for g, sg in zip(self.param_groups, state_dict['param_groups']):
            g.update({k: v for k, v in sg.items() if k != 'params'})
        bufs = {id(params[int(i)]): st['momentum_buffer'] for i, st in state_dict.get('state', {}).items() if st.get('momentum_buffer') is not None}
        if self._flat is None:
            self._pending = bufs
        else:
            for p, off in zip(self._flat.params, self._flat.offsets):     # the loaded state replaces the current one, as in torch
                if id(p) in bufs:
                    self._mom[off:off + p.numel()].copy_(bufs[id(p)].reshape(-1).to(self._mom.device))
                else:
                    self._mom[off:off + p.numel()].zero_()
            self._has_buf = {id(p) for p in self._flat.params if id(p) in bufs}
            self._make_runs()
