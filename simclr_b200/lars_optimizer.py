"""LARS optimizer of the reference (`tf2/lars_optimizer.py`) as a multi-tensor
sm_90a update: two launches per step over device pointer tables, fixed
reduction order (all replicas apply bit-identical updates).
"""
import re

import numpy as np
import torch

from ._lib import lib, stream_ptr
from .engine import get_engine

EETA_DEFAULT = 0.001  # tf2/lars_optimizer.py:22
CHUNK_ELEMS = 16384


class LARSOptimizer:
    """Layer-wise Adaptive Rate Scaling for large batch training
    (tf2/lars_optimizer.py:25-169; same constructor arguments)."""

    def __init__(self, learning_rate, momentum=0.9, use_nesterov=False, weight_decay=0.0,
                 exclude_from_weight_decay=None, exclude_from_layer_adaptation=None, classic_momentum=True,
                 eeta=EETA_DEFAULT, name='LARSOptimizer'):
        self.learning_rate = learning_rate      # float or callable schedule(step)
        self.momentum = momentum
        self.weight_decay = weight_decay
        self.use_nesterov = use_nesterov
        self.classic_momentum = classic_momentum
        self.eeta = eeta
        self.exclude_from_weight_decay = exclude_from_weight_decay
        # exclude_from_layer_adaptation is set to exclude_from_weight_decay if the arg is None.
        if exclude_from_layer_adaptation:
            self.exclude_from_layer_adaptation = exclude_from_layer_adaptation
        else:
            self.exclude_from_layer_adaptation = exclude_from_weight_decay
        self.name = name
        self.iterations = 0
        self._tables = None
        self._slots = {}
        if use_nesterov or not classic_momentum:
            raise NotImplementedError(
                'only classic momentum without Nesterov (the branch build_optimizer reaches, '
                'tf2/lars_optimizer.py:99-115) is implemented on the GPU path')

    # -- name filters (tf2/lars_optimizer.py:139-157) ------------------------
    def _use_weight_decay(self, param_name):
        """Whether to use L2 weight decay for `param_name`."""
        if not self.weight_decay:
            return False
        if self.exclude_from_weight_decay:
            for r in self.exclude_from_weight_decay:
                if re.search(r, param_name) is not None:
                    return False
        return True

    def _do_layer_adaptation(self, param_name):
        """Whether to do layer-wise learning rate adaptation for `param_name`."""
        if self.exclude_from_layer_adaptation:
            for r in self.exclude_from_layer_adaptation:
                if re.search(r, param_name) is not None:
                    return False
        return True

    def get_slot(self, var, slot_name='Momentum'):
        return self._slots[var.name]

    def lr_t(self):
        lr = self.learning_rate
        return float(lr(self.iterations)) if callable(lr) else float(lr)

    def _build(self, variables):
        e = get_engine()
        dev = e.device
        n = len(variables)
        total = sum((v.numel + 63) // 64 * 64 for v in variables)
        self._flat_v = torch.zeros(total, dtype=torch.float32, device=dev)
        off = 0
        w_ptrs, g_ptrs, v_ptrs, numels, flags = [], [], [], [], []
        chunk_tensor, chunk_offset, begin = [], [], [0]
        for i, v in enumerate(variables):
            slot = self._flat_v[off:off + v.numel].view(v.shape)      # slot "Momentum", zeros
            off += (v.numel + 63) // 64 * 64
            self._slots[v.name] = slot
            w_ptrs.append(v.value.data_ptr()); g_ptrs.append(v.grad.data_ptr()); v_ptrs.append(slot.data_ptr())
            numels.append(v.numel)
            flags.append((1 if self._use_weight_decay(v.name) else 0) | (2 if self._do_layer_adaptation(v.name) else 0))
            for o in range(0, v.numel, CHUNK_ELEMS):
                chunk_tensor.append(i); chunk_offset.append(o)
            begin.append(len(chunk_tensor))
        t = lambda a, dt: torch.from_numpy(np.asarray(a, dtype=dt)).to(dev)
        self._tables = dict(
            n=n, n_chunks=len(chunk_tensor), names=[v.name for v in variables],
            w=t(w_ptrs, np.int64), g=t(g_ptrs, np.int64), v=t(v_ptrs, np.int64), numel=t(numels, np.int64),
            flags=t(flags, np.int32), ct=t(chunk_tensor, np.int32), co=t(chunk_offset, np.int64),
            begin=t(begin, np.int64),
            partials=torch.zeros(2 * len(chunk_tensor), dtype=torch.float32, device=dev),
            lr_dev=torch.zeros(1, dtype=torch.float32, device=dev))

    def apply_gradients(self, grads_and_vars, name=None):
        """`optimizer.apply_gradients(zip(grads, vars))` (tf2/run.py:622).  Gradients
        must already be summed across replicas.  `grads` are the variables' `.grad`
        views (the zip is accepted for interface parity)."""
        variables = [v for _, v in grads_and_vars]
        if self._tables is None or self._tables['names'] != [v.name for v in variables]:
            self._build(variables)
        T = self._tables
        capturing = torch.cuda.is_current_stream_capturing()
        if not capturing:
            self.stage_learning_rate()       # inside a graph capture the kernel just reads lr_dev
        lib.lars_apply(T['n'], T['n_chunks'], T['w'], T['g'], T['v'], T['numel'], T['flags'], T['ct'], T['co'],
                       T['begin'], CHUNK_ELEMS, T['lr_dev'], float(self.momentum), float(self.weight_decay),
                       float(self.eeta), T['partials'], stream_ptr())
        if not capturing:                    # a capture records the update, it does not execute one:
            self.iterations += 1             # `prepare_replay` advances the schedule per replay

    def ensure_built(self, variables):
        """Builds the pointer tables / momentum slots (host->device copies) ahead of a graph capture."""
        if self._tables is None or self._tables['names'] != [v.name for v in variables]:
            self._build(variables)

    def stage_learning_rate(self):
        """Writes lr_t -- the schedule at the pre-increment iteration (SURVEY A7) -- into
        the device scalar the update kernel reads (stream-ordered fill)."""
        if self._tables is not None:
            self._tables['lr_dev'].fill_(self.lr_t())

    def prepare_replay(self):
        """Call before replaying a CUDA graph that captured `apply_gradients`."""
        self.stage_learning_rate()
        self.iterations += 1

    def get_config(self):
        return {
            'learning_rate': self.learning_rate if not callable(self.learning_rate) else 'schedule',
            'momentum': self.momentum,
            'classic_momentum': self.classic_momentum,
            'weight_decay': self.weight_decay,
            'eeta': self.eeta,
            'use_nesterov': self.use_nesterov,
        }
