"""Optional bf16-STORAGE emulation for the oracle -- TEST INFRASTRUCTURE ONLY.

The reference computes the whole step in fp32.  The throughput mode of the CUDA path
stores activations, activation gradients and the conv / dense operands in bf16
(fp32 accumulation, fp32 BatchNorm / loss / LARS arithmetic, fp32 master weights).
Inside `with emulate_bf16():` the oracle rounds to bf16 at exactly the points where the
CUDA path writes a bf16 tensor to HBM, in the forward AND in the backward pass:

  q(t)   tensor materialised in bf16: forward value rounded, incoming gradient rounded
         (conv outputs y, BN[+add][+ReLU] outputs z, pooled features)
  qb(t)  value untouched, incoming gradient rounded (a conv / dense input: its dgrad
         output is written in bf16 before anything is added to it; an fp32 tensor whose
         gradient the backward pass stores in bf16)
  qw(w)  weight operand: forward value rounded (the packed bf16 copy), gradient in fp32

With it the oracle answers two separate questions the fp32 oracle cannot:
  1. does the bf16 tensor-core step compute the bf16-storage algorithm correctly?
     (CUDA bf16 step vs emulating oracle: only accumulation order and rare rounding
     flips differ)
  2. what does bf16 storage itself cost on a given fixture?
     (emulating oracle vs fp32 / fp64 oracle, measurable on the CPU alone)
Outside the context manager every function is the identity and the oracle is the
plain restatement of the reference.
"""
import contextlib

import torch

_ENABLED = False
_FWD = True      # round forward values (stored activations, packed weights)
_BWD = True      # round stored activation gradients


def enabled():
    return _ENABLED


@contextlib.contextmanager
def emulate_bf16(on=True, forward=True, backward=True):
    """`forward` / `backward` switch the two families of rounding points separately (to attribute
    the cost of bf16 storage: see tests/test_oracle.py::test_bf16_storage_rounding_model)."""
    global _ENABLED, _FWD, _BWD
    prev = (_ENABLED, _FWD, _BWD)
    _ENABLED, _FWD, _BWD = bool(on), bool(forward), bool(backward)
    try:
        yield
    finally:
        _ENABLED, _FWD, _BWD = prev


def _round(t):
    return t.to(torch.bfloat16).to(t.dtype)


class _Round(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, fwd, bwd):
        ctx.bwd = bwd and _BWD
        return _round(x) if (fwd and _FWD) else x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        return (_round(g) if ctx.bwd else g), None, None


def q(t):
    return _Round.apply(t, True, True) if _ENABLED else t


def qb(t):
    return _Round.apply(t, False, True) if _ENABLED else t


def qw(t):
    return _Round.apply(t, True, False) if _ENABLED else t
