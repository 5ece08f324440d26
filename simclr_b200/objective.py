"""Contrastive objective of the reference (`tf2/objective.py`) on the H100 kernels.

`add_contrastive_loss(hidden, hidden_norm, temperature, strategy)` keeps the
reference signature and returns `(loss, logits_ab, labels)`.  The returned loss
is a torch tensor with autograd support (a custom Function over the explicit
kernels), and `contrastive_forward` / `contrastive_backward` expose the explicit
schedule the training step uses.

Multi-replica: `tpu_cross_replica_concat` (scatter + all-reduce SUM,
tf2/objective.py:92-127) becomes an NCCL all-gather of the normalised [2B,D]
embeddings; its backward (an all-reduce in TF) is replaced by an all-gather of
the per-row log-sum-exp [2B] and a local recomputation of the key-side terms
(SURVEY.md 8e) -- no second bulk collective.
"""
import torch

from ._lib import lib, stream_ptr
from .engine import get_engine

LARGE_NUM = 1e9  # tf2/objective.py:24 (masked logits underflow to exactly 0 in the softmax)


def add_supervised_loss(labels, logits, grad_scale=None):
    """tf2/objective.py:27-32: mean softmax CE.  labels one-hot [rows or rows/2, classes].
    With `grad_scale` also returns dlogits = (softmax - labels) * grad_scale."""
    e = get_engine()
    rows, classes = logits.shape
    out = e.empty((1 + rows,), torch.float32)
    dlogits = e.empty(logits.shape, torch.float32) if grad_scale is not None else None
    lib.softmax_xent(logits, labels, rows, labels.shape[0], classes,
                     0.0 if grad_scale is None else float(grad_scale), out, dlogits, stream_ptr())
    if grad_scale is None:
        return out[0]
    return out[0], dlogits


class _Ctx:
    pass


def contrastive_forward(hidden, hidden_norm=True, temperature=1.0, strategy=None, want_labels=True):
    """Forward of `add_contrastive_loss`; returns (loss, logits_ab, labels, ctx)."""
    e = get_engine()
    assert hidden.dtype == torch.float32 and hidden.dim() == 2 and hidden.shape[0] % 2 == 0
    hidden = hidden.contiguous()
    rows, D = hidden.shape
    B = rows // 2
    R = strategy.num_replicas_in_sync if strategy is not None else 1
    rid = strategy.replica_id if strategy is not None else 0
    st = stream_ptr()
    z = e.empty((rows, D), torch.float32)
    inv_norm = e.empty((rows,), torch.float32)
    lib.ntxent_normalize(hidden, rows, D, int(bool(hidden_norm)), z, inv_norm, st)
    z_all = strategy.all_gather(z, channel='z') if R > 1 else z            # [R][2][B][D]
    G = R * B
    ws_bytes = lib.ntxent_workspace_bytes(B, R, D)
    ws = e.empty((ws_bytes,), torch.uint8)
    logits_ab = e.empty((B, G), torch.float32)
    lse = e.empty((rows,), torch.float32)
    row_loss = e.empty((rows,), torch.float32)
    loss = e.empty((1,), torch.float32)
    lib.ntxent_forward(z_all, B, R, D, rid, float(temperature), logits_ab, lse, row_loss, loss, ws, ws_bytes, st)
    labels = None
    if want_labels:
        labels = e.empty((B, 2 * G), torch.float32)
        lib.ntxent_labels(B, R, rid, None, labels, None, st)
    ctx = _Ctx()
    ctx.z_all, ctx.lse, ctx.inv_norm, ctx.ws, ctx.ws_bytes = z_all, lse, inv_norm, ws, ws_bytes
    ctx.B, ctx.R, ctx.D, ctx.rid = B, R, D, rid
    ctx.hidden_norm, ctx.temperature, ctx.strategy = bool(hidden_norm), float(temperature), strategy
    return loss[0], logits_ab, labels, ctx


def contrastive_backward(ctx, grad_scale):
    """d(job loss)/d(hidden) for this replica's rows; grad_scale = dL/d(row loss)
    (the step uses 1/(B*R): local mean over B, then loss / num_replicas, tf2/run.py:617)."""
    e = get_engine()
    lse_all = ctx.strategy.all_gather(ctx.lse, channel='lse') if ctx.R > 1 else ctx.lse     # [R][2][B]
    dhidden = e.empty((2 * ctx.B, ctx.D), torch.float32)
    lib.ntxent_backward(ctx.z_all, lse_all, ctx.inv_norm, int(ctx.hidden_norm), ctx.B, ctx.R, ctx.D, ctx.rid,
                        ctx.temperature, float(grad_scale), dhidden, ctx.ws, ctx.ws_bytes, stream_ptr())
    return dhidden


def labels_and_masks(batch_size, num_replicas=1, replica_id=0):
    """tf2/objective.py:64-69 (integer-exact): returns (labels_idx int64 [B],
    labels [B, 2G], masks [B, G])."""
    e = get_engine()
    G = batch_size * num_replicas
    idx = e.empty((batch_size,), torch.int64)
    labels = e.empty((batch_size, 2 * G), torch.float32)
    masks = e.empty((batch_size, G), torch.float32)
    lib.ntxent_labels(batch_size, num_replicas, replica_id, idx, labels, masks, stream_ptr())
    return idx, labels, masks


class _NTXentFn(torch.autograd.Function):
    @staticmethod
    def forward(fctx, hidden, hidden_norm, temperature, strategy):
        loss, logits_ab, labels, ctx = contrastive_forward(hidden, hidden_norm, temperature, strategy)
        fctx.ctx = ctx
        fctx.mark_non_differentiable(logits_ab, labels)
        return loss, logits_ab, labels

    @staticmethod
    def backward(fctx, g_loss, g_logits, g_labels):
        ctx = fctx.ctx
        # d loss_r / d row_loss = 1/B; cross-replica key-side terms are included, which
        # equals TF's gradient of sum_r loss_r (the all-reduce backward sums them).
        d = contrastive_backward(ctx, 1.0 / ctx.B)
        return d * g_loss, None, None, None


def add_contrastive_loss(hidden, hidden_norm=True, temperature=1.0, strategy=None):
    """tf2/objective.py:35-89.

    Args:
      hidden: hidden vector (`Tensor`) of shape (bsz, dim), view-major ([view1; view2]).
      hidden_norm: whether or not to use normalization on the hidden vector.
      temperature: a `floating` number for temperature scaling.
      strategy: replica context (`engine.ReplicaContext`) or None for one replica.

    Returns:
      A loss scalar, the logits for the contrastive prediction task ([B, G]) and
      the one-hot labels ([B, 2G]).
    """
    return _NTXentFn.apply(hidden, hidden_norm, temperature, strategy)


def tpu_cross_replica_concat(tensor, strategy=None):
    """tf2/objective.py:92-127: concatenation of `tensor` across replicas."""
    if strategy is None or strategy.num_replicas_in_sync <= 1:
        return tensor
    out = strategy.all_gather(tensor)
    return out.reshape((-1,) + tuple(tensor.shape[1:]))


def contrast_metrics(logits_ab, replica_id=0):
    """tf2/metrics.py:23-36: (contrastive accuracy, entropy) as a [2] device tensor."""
    e = get_engine()
    B, G = logits_ab.shape
    out = e.empty((2 + 2 * B,), torch.float32)
    lib.contrast_metrics(logits_ab, B, G, replica_id, out, stream_ptr())
    return out[:2]
