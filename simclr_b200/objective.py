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


def add_distillation_loss(student_logits, teacher_logits, temperature, grad_scale=None):
    """SimCLRv2 distillation (the distillation colab's `add_kd_loss`): T^2 * mean_r CE(softmax(teacher/T),
    softmax(student/T)).  Returns (loss, agreement, dstudent): `agreement` is the fraction of rows whose student
    argmax equals the teacher argmax; with `grad_scale`, dstudent = (softmax(s/T) - softmax(t/T)) * grad_scale
    (the step passes T / (rows * replicas)), else None."""
    e = get_engine()
    assert student_logits.dtype == torch.float32 and teacher_logits.dtype == torch.float32
    assert student_logits.shape == teacher_logits.shape and student_logits.dim() == 2, \
        (tuple(student_logits.shape), tuple(teacher_logits.shape))
    student_logits, teacher_logits = student_logits.contiguous(), teacher_logits.contiguous()
    rows, classes = student_logits.shape
    out = e.empty((2 + rows,), torch.float32)
    dstudent = e.empty((rows, classes), torch.float32) if grad_scale is not None else None
    lib.distill_xent(student_logits, teacher_logits, rows, classes, float(temperature),
                     0.0 if grad_scale is None else float(grad_scale), out, dstudent, stream_ptr())
    return out[0], out[1], dstudent


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


GCL_DISTS = ('logsumexp', 'normal', 'uniform')
GCL_MAX_DIM = 256            # the tiled kernels keep a row of z in registers
GCL_MAX_SORT_ROWS = 16384    # the sliced Wasserstein terms sort 2G keys per column in one CTA's shared memory


def generalized_contrastive_dist():
    """The `--b200_gcl_dist` of this run, or None when the pretraining objective is NT-Xent; raises ValueError
    outside `--train_mode=pretrain`."""
    from .flags_def import FLAGS
    if FLAGS.b200_gcl_dist == 'none':
        return None
    if FLAGS.train_mode != 'pretrain':
        raise ValueError('--b200_gcl_dist=%s needs --train_mode=pretrain (got %r): the generalized contrastive loss '
                         'is a pretraining objective' % (FLAGS.b200_gcl_dist, FLAGS.train_mode))
    return FLAGS.b200_gcl_dist


def check_generalized_contrastive(dist, dim, global_rows):
    """Raises ValueError for a configuration the kernels do not support: an unknown `dist`, D > 256, or, for the
    sliced Wasserstein distributions, more than 16384 rows (2G) in the global batch."""
    if dist not in GCL_DISTS:
        raise ValueError('generalized contrastive loss: dist must be one of %s (got %r)' % (GCL_DISTS, dist))
    if dim > GCL_MAX_DIM:
        raise ValueError('generalized contrastive loss: the hidden dimension %d is above the supported %d'
                         % (dim, GCL_MAX_DIM))
    if dist != 'logsumexp' and global_rows > GCL_MAX_SORT_ROWS:
        raise ValueError('generalized contrastive loss: dist=%r sorts %d rows (two views of the global batch) per '
                         'column, above the supported %d' % (dist, global_rows, GCL_MAX_SORT_ROWS))


def generalized_contrastive_forward(hidden, dist='normal', lambda_weight=1.0, temperature=1.0, hidden_norm=True,
                                    loss_scaling=1.0, strategy=None, step=None, seed=0, draws=None):
    """Forward of the generalized contrastive loss over the global batch; returns (loss, align, dist_loss, ctx).

    hidden [2B, D] fp32, view-major.  `step` (an int, or a device int64 [1] that a captured graph reads on every
    replay) and `seed` key the SWD draws: the prior [2G, D] and the orthogonal W [D, D], the same on every replica
    for the same key.  `step=None` (one replica only) draws with a fresh key on every call, as the colab does; the
    key's seed then comes from torch's default generator.  `draws=(W, prior)` replaces the draws (prior already
    l2-normalised when hidden_norm); ctx.W and ctx.prior hold the draws of the call.  With more than one
    replica the loss is this replica's L_r: the alignment over its rows, the logsumexp of its rows against all 2G
    rows, or the SWD of all 2G rows (the same on every replica); the job's loss is the mean over replicas."""
    e = get_engine()
    assert hidden.dtype == torch.float32 and hidden.dim() == 2 and hidden.shape[0] % 2 == 0
    hidden = hidden.contiguous()
    rows, D = hidden.shape
    B = rows // 2
    R = strategy.num_replicas_in_sync if strategy is not None else 1
    rid = strategy.replica_id if strategy is not None else 0
    G = R * B
    check_generalized_contrastive(dist, D, 2 * G)
    st = stream_ptr()
    z = e.empty((rows, D), torch.float32)
    inv_norm = e.empty((rows,), torch.float32)
    lib.ntxent_normalize(hidden, rows, D, int(bool(hidden_norm)), z, inv_norm, st)
    z_all = strategy.all_gather(z, channel='z') if R > 1 else z            # [R][2][B][D]
    ws_bytes = lib.gcl_workspace_bytes(B, R, D)
    ws = e.empty((ws_bytes,), torch.uint8)
    out = e.empty((3,), torch.float32)                                      # loss, align, dist
    ctx = _Ctx()
    ctx.dist, ctx.lse, ctx.perm, ctx.diff, ctx.W, ctx.prior, ctx.wnormal = dist, None, None, None, None, None, None
    if dist == 'logsumexp':
        ctx.lse = e.empty((rows,), torch.float32)
        lib.gcl_lse_forward(z_all, B, R, D, rid, float(temperature), ctx.lse, out, ws, ws_bytes, st)
    else:
        if draws is None:
            if step is None:
                if R > 1:
                    raise ValueError('generalized contrastive loss: with %d replicas the SWD draws must be the same on '
                                     'every replica; pass the same step and seed on each' % R)
                # a fresh key per call, reproducible through torch.manual_seed
                seed, step = int(torch.randint(0, 2 ** 62, (1,)).item()), 0
            if not torch.is_tensor(step):
                step = torch.full((1,), int(step), dtype=torch.int64, device=e.device)
            ctx.prior = e.empty((2 * G, D), torch.float32)
            ctx.wnormal = e.empty((D, D), torch.float32)
            ctx.W = e.empty((D, D), torch.float32)
            lib.gcl_draw(int(seed), step, 2 * G, D, GCL_DISTS.index(dist) - 1, int(bool(hidden_norm)), ctx.prior,
                         ctx.wnormal, st)
            lib.gcl_orthogonal(ctx.wnormal, D, ctx.W, ws, ws_bytes, st)
        else:
            ctx.W, ctx.prior = (t.contiguous() for t in draws)
            assert ctx.W.shape == (D, D) and ctx.prior.shape == (2 * G, D)
        ctx.perm = e.empty((D, 2 * G), torch.int32)
        ctx.diff = e.empty((D, 2 * G), torch.float32)
        lib.gcl_swd_forward(z_all, ctx.prior, ctx.W, B, R, D, out, ctx.perm, ctx.diff, ws, ws_bytes, st)
    ctx.dz_align = e.empty((rows, D), torch.float32)
    lib.gcl_align(z, B, D, float(lambda_weight), float(loss_scaling), out, ctx.dz_align, st)
    ctx.z, ctx.z_all, ctx.inv_norm, ctx.ws, ctx.ws_bytes = z, z_all, inv_norm, ws, ws_bytes
    ctx.B, ctx.R, ctx.D, ctx.rid = B, R, D, rid
    ctx.hidden_norm, ctx.temperature, ctx.strategy = bool(hidden_norm), float(temperature), strategy
    ctx.lambda_weight, ctx.loss_scaling = float(lambda_weight), float(loss_scaling)
    return out[0], out[1], out[2], ctx


def generalized_contrastive_backward(ctx, grad_scale):
    """d(job loss)/d(hidden) for this replica's rows.  grad_scale = d(job loss)/d(L_r), the same on every replica
    (the step uses 1/R: loss / num_replicas, then the gradient sum).  The logsumexp key-side terms come from the
    all-gathered lse; the SWD is the same on every replica, so each takes R times its weight for its own rows."""
    e = get_engine()
    st = stream_ptr()
    B, R, D = ctx.B, ctx.R, ctx.D
    w = float(grad_scale) * ctx.loss_scaling
    dz_lse = dz_swd = None
    if ctx.dist == 'logsumexp':
        lse_all = ctx.strategy.all_gather(ctx.lse, channel='lse') if R > 1 else ctx.lse      # [R][2][B]
        dz_lse = e.empty((2 * B, D), torch.float32)
        lib.gcl_lse_backward(ctx.z_all, lse_all, B, R, D, ctx.rid, ctx.temperature, dz_lse, ctx.ws, ctx.ws_bytes, st)
    else:
        dz_swd = e.empty((2 * B, D), torch.float32)
        lib.gcl_swd_backward(ctx.perm, ctx.diff, ctx.W, B, R, D, ctx.rid, dz_swd, ctx.ws, ctx.ws_bytes, st)
    dhidden = e.empty((2 * B, D), torch.float32)
    lib.gcl_normalize_backward(ctx.z, ctx.inv_norm, int(ctx.hidden_norm), 2 * B, D, ctx.dz_align, w,
                               dz_lse, w * ctx.lambda_weight / (2 * B), dz_swd, w * ctx.lambda_weight * R, dhidden, st)
    return dhidden


class _GCLFn(torch.autograd.Function):
    @staticmethod
    def forward(fctx, hidden, lambda_weight, temperature, dist, hidden_norm, loss_scaling, strategy, step, seed):
        loss, _, _, ctx = generalized_contrastive_forward(hidden, dist, lambda_weight, temperature, hidden_norm,
                                                          loss_scaling, strategy, step, seed)
        fctx.ctx = ctx
        return loss

    @staticmethod
    def backward(fctx, g_loss):
        # g_loss is this replica's weight; the job's gradient is the sum over replicas of equal weights
        d = generalized_contrastive_backward(fctx.ctx, 1.0)
        return (d * g_loss,) + (None,) * 8


def generalized_contrastive_loss(hidden1, hidden2, lambda_weight=1.0, temperature=1.0, dist='normal',
                                 hidden_norm=True, loss_scaling=1.0, strategy=None, step=None, seed=0):
    """The intriguing-properties colab's `generalized_contrastive_loss` (Chen, Luo, Li 2021) on the H100 kernels.
    Like the colab, every call draws a fresh W and prior unless `step` is given.

    Args:
      hidden1, hidden2: [B, D] fp32 hidden vectors of the two views.
      lambda_weight: weight of the distribution-matching term.
      temperature: temperature of the 'logsumexp' term.
      dist: 'logsumexp' (decoupled NT-Xent), 'normal' or 'uniform' (sliced Wasserstein distance to that prior).
      hidden_norm: whether to l2-normalise the hidden vectors (and the prior rows).
      loss_scaling: scale of the whole loss.
      strategy: replica context (`engine.ReplicaContext`) or None for one replica.
      step, seed: key of the SWD draws (W and the prior): the same key gives the same draws on every replica.
        None (one replica only): a fresh key on every call, its seed taken from torch's default generator.

    Returns:
      The loss scalar (this replica's L_r), differentiable with respect to hidden1 and hidden2.
    """
    return _GCLFn.apply(torch.cat([hidden1, hidden2], 0), lambda_weight, temperature, dist, hidden_norm,
                        loss_scaling, strategy, step, seed)


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
