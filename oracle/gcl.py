"""Oracle of the generalized contrastive loss of *Intriguing Properties of Contrastive Losses* (Chen, Luo, Li,
NeurIPS 2021), the intriguing-properties colab's `generalized_contrastive_loss`.  Test infrastructure only.

With z = l2_normalize(hidden) (or hidden), h1 = z[:B], h2 = z[B:]:

  L_align = sum (h1 - h2)^2 / (2 B D)
  L_dist  = mean_i [logsumexp_j (z_i . z_j / tau) - ln D]       'logsumexp': j over all 2B rows, i itself included
          = mean over 2B x D of (sort(P W) - sort(z W))^2        'normal' / 'uniform': sliced Wasserstein distance
  L       = loss_scaling * (L_align + lambda * L_dist)

W (a D x D orthogonal matrix) and P (the [2B, D] prior draw, l2-normalised here when hidden_norm) are arguments, so
a test can inject the draws of the kernels.  Columns are sorted ascending over the rows with a stable sort.
"""
import math

import torch

from .objective import l2_normalize

DISTS = ('logsumexp', 'normal', 'uniform')


def orthogonal(d, normal_draw):
    """Keras `Orthogonal()` of a d x d standard-normal draw: Q of its QR, Q's columns times sign(diag R)."""
    q, r = torch.linalg.qr(normal_draw.reshape(d, d))
    return q * torch.sign(torch.diagonal(r)).unsqueeze(0)


def align_loss(h1, h2):
    return ((h1 - h2) ** 2).sum() / (2 * h1.shape[0] * h1.shape[1])


def logsumexp_loss(queries, keys, temperature):
    """mean over the query rows of logsumexp over every key row (no mask) of q.k / tau, minus ln D."""
    lse = torch.logsumexp(queries @ keys.t() / temperature, dim=1)
    return (lse - math.log(queries.shape[1])).mean()


def swd_loss(z, prior, W, hidden_norm):
    """Sliced Wasserstein distance between the rows of z and the prior draw along the columns of W."""
    if hidden_norm:
        prior = l2_normalize(prior, -1)
    s = torch.sort(z @ W, dim=0, stable=True).values
    q = torch.sort(prior @ W, dim=0, stable=True).values
    return ((q - s) ** 2).mean()


def generalized_contrastive_loss(hidden1, hidden2, lambda_weight=1.0, temperature=1.0, dist='normal',
                                 hidden_norm=True, loss_scaling=1.0, W=None, P=None):
    """Returns (loss, L_align, L_dist).  `W` [D, D] and `P` [2B, D] are needed for the SWD distributions."""
    if dist not in DISTS:
        raise ValueError('unknown dist %r' % (dist,))
    if hidden_norm:
        hidden1, hidden2 = l2_normalize(hidden1, -1), l2_normalize(hidden2, -1)
    la = align_loss(hidden1, hidden2)
    z = torch.cat([hidden1, hidden2], 0)
    if dist == 'logsumexp':
        ld = logsumexp_loss(z, z, temperature)
    else:
        ld = swd_loss(z, P, W, hidden_norm)
    return loss_scaling * (la + lambda_weight * ld), la, ld


def gcl_loss_replicas(hiddens, lambda_weight=1.0, temperature=1.0, dist='normal', hidden_norm=True,
                      loss_scaling=1.0, W=None, P=None):
    """The loss on R simulated replicas, as `objective.contrastive_loss_replicas` simulates NT-Xent.

    hiddens: list over replicas of [2B, D] (view-major).  The global batch is hidden1 = every replica's view-1 rows,
    hidden2 = every replica's view-2 rows, gathered as a differentiable concatenation of the replicas' live tensors
    (so the backward is TensorFlow's all-reduce backward).  Replica r reports (L_r, align_r, dist_r): the alignment
    over its own rows, the logsumexp over its own 2B rows against all 2G rows, or the SWD of all 2G rows against the
    [2G, D] prior P (the same on every replica).  The job's loss is sum_r L_r / R."""
    R = len(hiddens)
    normed = [l2_normalize(h, -1) if hidden_norm else h for h in hiddens]
    B = hiddens[0].shape[0] // 2
    h1 = [z[:B] for z in normed]
    h2 = [z[B:] for z in normed]
    z_all = torch.cat(h1 + h2, 0)
    swd = swd_loss(z_all, P, W, hidden_norm) if dist != 'logsumexp' else None
    out = []
    for r in range(R):
        la = align_loss(h1[r], h2[r])
        ld = logsumexp_loss(normed[r], z_all, temperature) if dist == 'logsumexp' else swd
        out.append((loss_scaling * (la + lambda_weight * ld), la, ld))
    return out
