"""Oracle restatement of SimCLRv2 distillation (the distillation colab's `add_kd_loss` and its training step).
Test infrastructure only -- never imported by `simclr_b200/`.

The colab defines the loss as

    teacher_probs = tf.nn.softmax(teacher_logits / temperature)
    kd_loss = tf.reduce_mean(temperature**2 * tf.losses.softmax_cross_entropy(
        tf.stop_gradient(teacher_probs), student_logits / temperature))

and `tf.losses.softmax_cross_entropy` with the scalar weight T^2 and SUM_BY_NONZERO_WEIGHTS reduction is T^2 times the
mean row cross-entropy.  The teacher is a second `oracle.model.Model` with its own `cfg` (train_mode 'finetune'),
run in inference mode under `torch.no_grad()`.
"""
from collections import OrderedDict

import torch

from . import model as model_lib
from . import objective as obj_lib


def add_kd_loss(student_logits, teacher_logits, temperature):
    """T^2 * mean_r softmax_cross_entropy(softmax(teacher / T), student / T); no gradient reaches the teacher."""
    teacher_probs = torch.softmax(teacher_logits / temperature, dim=-1).detach()
    kd = obj_lib.softmax_cross_entropy_with_logits(teacher_probs, student_logits / temperature)
    return temperature ** 2 * kd.mean()


def agreement(student_logits, teacher_logits):
    """Fraction of rows whose student argmax equals the teacher argmax (torch.argmax: first index on ties)."""
    return (student_logits.argmax(1) == teacher_logits.argmax(1)).to(student_logits.dtype).mean()


def forward_backward(model, P, S, features, teacher, temperature):
    """Loss and gradients of one distillation step of the student `model` (finetune cfg).

    features: list over replicas of [B,H,W,3]; teacher = (teacher model, its P, its S).  On each replica the teacher
    runs in inference mode under `torch.no_grad()`, then the student in training mode; the loss of a replica is the
    KD loss plus weight decay, divided by R and summed (per-replica BatchNorm: R == 1 or global_bn off).
    Returns dict(loss, kd_loss, agreement, wd, grads, S_new, sup_out, teacher_out)."""
    cfg = model.cfg
    assert cfg.train_mode == 'finetune'
    tmodel, TP, TS = teacher
    R = len(features)
    assert R == 1 or not cfg.global_bn, 'per-replica BatchNorm only'
    Pg = OrderedDict((k, v.detach().clone().requires_grad_(True)) for k, v in P.items())
    Sn = OrderedDict((k, v.clone()) for k, v in S.items())
    wd = model_lib.add_weight_decay(cfg, Pg, adjust_per_optimizer=True)
    total = 0.
    kd_losses, agree, sup, tout = [], [], [], []
    for r in range(R):
        with torch.no_grad():
            _, t_logits = tmodel(TP, TS, features[r], False)
        _, s_logits = model(Pg, Sn, features[r], True)
        kd = add_kd_loss(s_logits, t_logits, temperature)
        kd_losses.append(kd.detach())
        agree.append(agreement(s_logits.detach(), t_logits))
        sup.append(s_logits.detach())
        tout.append(t_logits)
        total = total + (kd + wd) / R
    grads = torch.autograd.grad(total, list(Pg.values()), allow_unused=True)
    G = OrderedDict()
    for (k, v), g in zip(Pg.items(), grads):
        G[k] = torch.zeros_like(v) if g is None else g
    return dict(loss=total.detach(), kd_loss=kd_losses, agreement=agree,
                wd=wd.detach() if torch.is_tensor(wd) else wd, grads=G, S_new=Sn, sup_out=sup, teacher_out=tout)
