"""`momentum` and `adam` of the reference's `build_optimizer` (tf2/model.py:31-34) on the H100 path:
`tf.keras.optimizers.SGD(learning_rate, FLAGS.momentum, nesterov=True)` and
`tf.keras.optimizers.Adam(learning_rate)` as element-wise kernels over the flat parameter buffer
(`csrc/optim.cu`).  Same host interface as `LARSOptimizer` (`apply_gradients`, `iterations`,
`stage_learning_rate` / `prepare_replay` for CUDA-graph replay).
"""
import math

import torch

from ._lib import lib, stream_ptr
from .engine import get_engine


class _FlatOptimizer:
    def __init__(self, learning_rate, name):
        self.learning_rate = learning_rate          # float or callable schedule(step)
        self.name = name
        self.iterations = 0
        self._span = None
        self._hyper = None

    def lr_t(self):
        lr = self.learning_rate
        return float(lr(self.iterations)) if callable(lr) else float(lr)

    def _flat(self, variables):
        """The variables are views into one flat value buffer and one flat gradient buffer with the same
        layout (engine.VarStore): returns (w, g) covering all of them, padding included (its gradient is 0)."""
        key = tuple(v.name for v in variables)
        if self._span is None or self._span[0] != key:
            lo = min(v.value.data_ptr() for v in variables)
            hi = max(v.value.data_ptr() + v.numel * 4 for v in variables)
            glo = min(v.grad.data_ptr() for v in variables)
            for v in variables:
                if v.value.data_ptr() - lo != v.grad.data_ptr() - glo:
                    raise ValueError('value / gradient buffers of %s are not laid out alike' % v.name)
            first = min(variables, key=lambda v: v.value.data_ptr())
            n = (hi - lo) // 4
            w = torch.as_strided(first.value, (n,), (1,), first.value.storage_offset())
            g = torch.as_strided(first.grad, (n,), (1,), first.grad.storage_offset())
            dev = first.value.device
            self._span = (key, w, g, n)
            self._slots = [torch.zeros(n, dtype=torch.float32, device=dev) for _ in range(self.NUM_SLOTS)]
            self._hyper = torch.zeros(1, dtype=torch.float32, device=dev)
        return self._span[1], self._span[2], self._span[3]

    def ensure_built(self, variables):
        self._flat(variables)

    def _hyper_value(self):
        raise NotImplementedError

    def stage_learning_rate(self):
        if self._hyper is not None:
            self._hyper.fill_(self._hyper_value())

    def prepare_replay(self):
        self.stage_learning_rate()
        self.iterations += 1

    def apply_gradients(self, grads_and_vars, name=None):
        variables = [v for _, v in grads_and_vars]
        w, g, n = self._flat(variables)
        capturing = torch.cuda.is_current_stream_capturing()
        if not capturing:
            self.stage_learning_rate()
        self._launch(w, g, n)
        if not capturing:
            self.iterations += 1


class SGD(_FlatOptimizer):
    """tf.keras.optimizers.SGD(learning_rate, momentum, nesterov)."""
    NUM_SLOTS = 1

    def __init__(self, learning_rate, momentum=0.0, nesterov=False, name='SGD'):
        super().__init__(learning_rate, name)
        self.momentum, self.nesterov = float(momentum), bool(nesterov)

    def _hyper_value(self):
        return self.lr_t()

    def _launch(self, w, g, n):
        lib.sgd_momentum_apply(w, g, self._slots[0], n, self._hyper, self.momentum, int(self.nesterov), stream_ptr())

    def get_config(self):
        return {'learning_rate': self.learning_rate if not callable(self.learning_rate) else 'schedule',
                'momentum': self.momentum, 'nesterov': self.nesterov}


class Adam(_FlatOptimizer):
    """tf.keras.optimizers.Adam(learning_rate): beta_1 0.9, beta_2 0.999, epsilon 1e-7."""
    NUM_SLOTS = 2

    def __init__(self, learning_rate, beta_1=0.9, beta_2=0.999, epsilon=1e-7, name='Adam'):
        super().__init__(learning_rate, name)
        self.beta_1, self.beta_2, self.epsilon = float(beta_1), float(beta_2), float(epsilon)

    def _hyper_value(self):
        t = self.iterations + 1
        return self.lr_t() * math.sqrt(1.0 - self.beta_2 ** t) / (1.0 - self.beta_1 ** t)

    def _launch(self, w, g, n):
        lib.adam_apply(w, g, self._slots[0], self._slots[1], n, self._hyper, self.beta_1, self.beta_2, self.epsilon,
                       stream_ptr())

    def get_config(self):
        return {'learning_rate': self.learning_rate if not callable(self.learning_rate) else 'schedule',
                'beta_1': self.beta_1, 'beta_2': self.beta_2, 'epsilon': self.epsilon}
