"""Oracle of the BatchNorm-folded inference forward (`--b200_fold_bn`) -- TEST INFRASTRUCTURE ONLY.

In inference mode a BatchNorm runs on its moving statistics, so it is the per-channel affine
z = y * scale + shift with scale = gamma * rsqrt(moving_variance + eps) and shift = beta - moving_mean * scale.
Folded into the conv (or dense layer) before it, conv -> BatchNorm [-> + residual] [-> ReLU] becomes

    v = conv(x, w * scale) + shift;  v += residual;  v = max(v, 0)

This module states that algebra (`fold`) and the whole inference forward of an `oracle.model.Model` built on it
(`Model`).  Under `bf16_emul.emulate_bf16()` it rounds where the CUDA path writes bf16: the folded weights
(bf16_rn(w * scale)), the layer output z after bias, residual and ReLU -- and nowhere in between: no conv output y
is stored.  Outside the emulation it is exact algebra: in fp64 it equals the unfolded oracle forward with
`training=False` to rounding.
"""
import torch
import torch.nn.functional as F

from . import resnet as R
from .bf16_emul import q, qw, enabled as _bf16_emulated


def fold(P, S, bn):
    """(scale, shift) of an inference-mode `oracle.resnet.BatchNormRelu` (gamma = 1 with `scale=False`, beta = 0 with
    `center=False`)."""
    scale = torch.rsqrt(S[bn.mv] + R.BATCH_NORM_EPSILON)
    if bn.gamma is not None:
        scale = scale * P[bn.gamma]
    shift = -S[bn.mm] * scale
    if bn.beta is not None:
        shift = P[bn.beta] + shift
    return scale, shift


def folded_weight(P, S, kernel, bn):
    """HWIO (or [Cin, Cout]) weights with the BatchNorm's scale folded into the output channels, and the bias."""
    scale, shift = fold(P, S, bn)
    return P[kernel] * scale, shift


def _epilogue(v, bias, shape, residual, relu, store=True):
    v = v + bias.view(shape)
    if residual is not None:
        v = v + residual
    if relu:
        v = F.relu(v)
    return q(v) if store else v


def conv_bn(P, S, conv, bn, x, residual=None, relu=None):
    """Folded `Conv2dFixedPadding` -> `BatchNormRelu` on NCHW x."""
    w, b = folded_weight(P, S, conv.kernel, bn)
    w = qw(w).permute(3, 2, 0, 1)
    if conv.s > 1:
        y = F.conv2d(R.fixed_padding(x, conv.k), w, stride=conv.s)
    else:
        y = F.conv2d(x, w, padding=(conv.k - 1) // 2)
    return _epilogue(y, b, (1, -1, 1, 1), residual, bn.relu if relu is None else relu)


def dense_bn(P, S, kernel, bn, x, relu, store=True):
    """Folded dense layer ([N, Cin] @ [Cin, Cout], or a 1x1 conv kernel) -> BatchNorm."""
    w, b = folded_weight(P, S, kernel, bn)
    w = qw(w)
    if w.dim() == 4:
        w = w[0, 0]
    return _epilogue(x @ w, b, (1, -1), None, relu, store)


def sk(P, S, layer, x):
    assert not _bf16_emulated(), 'bf16-storage emulation does not cover SK blocks'
    x = conv_bn(P, S, layer.conv, layer.bn, x)
    streams = torch.stack(torch.split(x, layer.filters, dim=1))
    g = streams.sum(0).mean(dim=(2, 3))
    g = dense_bn(P, S, layer.conv0.kernel, layer.bn1, g, relu=True)
    mixing = layer.conv1(P, S, g[:, :, None, None], False)
    mixing = torch.softmax(torch.stack(torch.split(mixing, layer.filters, dim=1)), dim=0)
    return (streams * mixing).sum(0)


def block(P, S, blk, x):
    """Folded `ResidualBlock` / `BottleneckBlock`: the last BatchNorm takes the shortcut and the ReLU in its epilogue
    (with SE, the SE layer and the add + ReLU follow it as in the unfolded block)."""
    shortcut = x
    if blk.shortcut is not None:
        xs = R.avg_pool_2x2(x, blk.shortcut.strides) if blk.cfg.sk_ratio > 0 else x
        shortcut = conv_bn(P, S, blk.shortcut.conv, blk.shortcut.bn, xs)
    h = conv_bn(P, S, blk.c1, blk.b1, x)
    if isinstance(blk, R.BottleneckBlock):
        h = sk(P, S, blk.sk, h) if blk.sk is not None else conv_bn(P, S, blk.c2, blk.b2, h)
        last_conv, last_bn = blk.c3, blk.b3
    else:
        last_conv, last_bn = blk.c2, blk.b2
    if blk.se is not None:
        h = blk.se(P, S, conv_bn(P, S, last_conv, last_bn, h), False)
        return q(F.relu(h + shortcut))
    return conv_bn(P, S, last_conv, last_bn, h, residual=shortcut, relu=True)


def resnet(P, S, net, x_nhwc):
    """Folded inference forward of `oracle.resnet.Resnet`: [N, H, W, 3] -> [N, C] features."""
    x = q(x_nhwc.permute(0, 3, 1, 2))
    for conv, bn in zip(net.stem[0::2], net.stem[1::2]):
        x = conv_bn(P, S, conv, bn, x)
    if not net.cifar_stem:
        x = R.max_pool_3x3_s2_same(x)
    for g in net.groups:
        for blk in g.layers:
            x = block(P, S, blk, x)
    return q(x.mean(dim=(2, 3)))


class Model:
    """Folded inference forward (`training=False`) of an `oracle.model.Model`: same outputs as
    `model(P, S, inputs, False)`, i.e. (projection output, supervised head output or None)."""

    def __init__(self, model):
        self.model = model

    def __call__(self, P, S, inputs):
        m, cfg = self.model, self.model.cfg
        features = torch.cat(torch.split(inputs, 3, dim=-1), 0)      # view-major, no blur in inference
        hiddens = resnet(P, S, m.resnet_model, features)
        head = m._projection_head
        if cfg.proj_head_mode != 'nonlinear':
            raise ValueError("only proj_head_mode='nonlinear' is callable (reference quirk Q1)")
        hiddens_list = [hiddens]
        for j, layer in enumerate(head.linear_layers):
            last = j == len(head.linear_layers) - 1
            # the last projection layer's output stays fp32 on the CUDA path
            hiddens_list.append(dense_bn(P, S, layer.kernel, layer.bn, hiddens_list[-1], relu=not last, store=not last))
        proj_out, sup_in = hiddens_list[-1], hiddens_list[cfg.ft_proj_selector]
        if cfg.train_mode == 'finetune':
            return None, m.supervised_head(P, S, sup_in, False)
        if cfg.lineareval_while_pretraining:
            return proj_out, m.supervised_head(P, S, sup_in, False)
        return proj_out, None
