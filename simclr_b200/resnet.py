"""ResNet of the reference (`tf2/resnet.py`) with an explicit forward/backward
schedule on the sm_90a kernels -- no framework autograd on the GPU path.

Class names, constructor arguments and the `resnet()` factory mirror
`tf2/resnet.py:31-78,160-208,314-526,529-747`.  Every layer object has
`__call__(inputs, training)` (forward, stashes what backward needs) and
`backward(grad)`.  Activations are NHWC torch tensors in the engine's activation
dtype; variables are fp32 HWIO / [C] views into flat buffers.

SK blocks (`sk_ratio > 0`, with the ResNet-D stem and shortcuts, config 5) and SE
blocks (`se_ratio > 0`) are on the GPU path.
"""
import os

import torch

from ._lib import lib, stream_ptr, F32, BF16
from .engine import get_engine, BATCH_NORM_EPSILON
from .flags_def import FLAGS


class BatchNormRelu:  # pylint: disable=missing-docstring
    """tf2/resnet.py:31-78.  (Sync)BatchNormalization + optional ReLU; the
    residual add + ReLU of the block tail (tf2/resnet.py:382,487) can be fused in."""

    def __init__(self, vs, scope, channels, relu=True, init_zero=False, center=True, scale=True):
        self.relu = relu
        self.C = channels
        lname = vs.namer('batch_norm_relu')
        bn = vs.namer('sync_batch_normalization' if FLAGS.global_bn else 'batch_normalization')
        pre = '%s/%s/%s' % (scope, lname, bn)
        self.gamma = vs.add(pre + '/gamma:0', (channels,), 'zeros' if init_zero else 'ones') if scale else None
        self.beta = vs.add(pre + '/beta:0', (channels,), 'zeros') if center else None
        self.moving_mean = vs.add(pre + '/moving_mean:0', (channels,), 'zeros', trainable=False)
        self.moving_variance = vs.add(pre + '/moving_variance:0', (channels,), 'ones', trainable=False)
        self.saved = None

    def _statistics(self, y, training, sums=None):
        """(mean, rstd, scale, shift) of this call: batch statistics (SyncBN: global, exchanged over peer memory or
        NCCL) with the moving-average update when training, the moving statistics otherwise."""
        e = get_engine()
        C = self.C
        rows = y.numel() // C
        st = stream_ptr()
        stats = e.empty((4, C), torch.float32)     # mean, rstd, scale, shift
        mean, rstd, scale, shift = stats[0], stats[1], stats[2], stats[3]
        g = None if self.gamma is None else self.gamma.value
        b = None if self.beta is None else self.beta.value
        if training:
            if sums is None:
                sums = e.sums(2 * C)
                lib.bn_stats(y, e.code(y.dtype), rows, C, sums, st)
            count = float(rows)
            if e.sync_bn and e.ctx.comm is not None and 2 * C * 8 <= e.ctx.comm.slot_bytes:
                # SyncBatchNormalization (C2): one-shot exchange of (sum x, sum x^2) over NVLink peer memory
                # inside the finalize kernel
                e.ctx.comm.bn_finalize(sums, count, g, b, BATCH_NORM_EPSILON, float(FLAGS.batch_norm_decay),
                                       self.moving_mean.value, self.moving_variance.value, mean, rstd, scale, shift, C)
            else:
                if e.sync_bn:        # same collective through NCCL
                    e.ctx.all_reduce_sum(sums)
                    count *= e.ctx.num_replicas_in_sync
                lib.bn_finalize(sums, count, g, b, BATCH_NORM_EPSILON, float(FLAGS.batch_norm_decay),
                                self.moving_mean.value, self.moving_variance.value, mean, rstd, scale, shift, C, st)
        else:
            r = torch.rsqrt(self.moving_variance.value + BATCH_NORM_EPSILON)
            sc = r if g is None else g * r
            mean.copy_(self.moving_mean.value); rstd.copy_(r); scale.copy_(sc)
            shift.copy_(-self.moving_mean.value * sc if b is None else b - self.moving_mean.value * sc)
        return mean, rstd, scale, shift

    def _coefficients(self, sums, rows, mean, rstd):
        """coef [3][C] of dy = k1*dz + k2*y + k3 from the (global) backward sums; fills dgamma / dbeta."""
        e = get_engine()
        C = self.C
        coef = e.empty((3 * C,), torch.float32)
        gam = None if self.gamma is None else self.gamma.value
        dgam = None if self.gamma is None else self.gamma.grad
        dbet = None if self.beta is None else self.beta.grad
        count = float(rows)
        if e.sync_bn and e.ctx.comm is not None and 2 * C * 8 <= e.ctx.comm.slot_bytes:
            e.ctx.comm.bn_bwd_coef(sums, count, mean, rstd, gam, coef, dgam, dbet, C)
        else:
            sums_g = sums
            if e.sync_bn:
                sums_g = sums.clone()
                e.ctx.all_reduce_sum(sums_g)
                count *= e.ctx.num_replicas_in_sync
            lib.bn_bwd_coef(mean, rstd, gam, sums_g, sums, count, coef, dgam, dbet, C, stream_ptr())
        return coef

    # -- projection-block tail: this BatchNorm + the shortcut's BatchNorm + add + ReLU in one pass ------------------
    @staticmethod
    def tail2_enabled():
        return os.environ.get('SIMCLR_BN_TAIL2', '1') != '0'

    def forward_tail2(self, y, sums, ys, bn_s, sums_s):
        """relu(BN(y) + BN_s(ys)) for a block with a projection shortcut (tf2/resnet.py:342-353,382; :415-423,487):
        the shortcut's BatchNorm output is formed (and rounded) inside the kernel instead of being written and
        re-read.  `sums` / `sums_s`: the statistics the two conv epilogues produced."""
        e = get_engine()
        C = self.C
        rows = y.numel() // C
        mean, rstd, scale, shift = self._statistics(y, True, sums)
        mean2, rstd2, scale2, shift2 = bn_s._statistics(ys, True, sums_s)
        z = e.empty(y.shape, y.dtype)
        bits = e.empty((rows * C // 8,), torch.uint8)
        lib.bn_apply2_relu_mask(y, ys, e.code(y.dtype), z, e.code(z.dtype), rows, C, scale, shift, scale2, shift2, bits,
                                stream_ptr())
        self.saved = ('tail2', y, ys, bits, mean, rstd, mean2, rstd2, rows, bn_s)
        return z

    def backward_tail2(self, dz, dz2=None):
        """dz <- (dz + dz2) * relu_mask in place; returns (d conv output, d shortcut conv output)."""
        e = get_engine()
        _, y, ys, bits, mean, rstd, mean2, rstd2, rows, bn_s = self.saved
        self.saved = None
        C = self.C
        st = stream_ptr()
        sums, sums2 = e.sums(2 * C), e.sums(2 * C)
        lib.bn_bwd_reduce2_bits(dz, dz2, bits, e.code(dz.dtype), y, ys, e.code(y.dtype), rows, C, mean, rstd, mean2, rstd2,
                                sums, sums2, st)
        coef = self._coefficients(sums, rows, mean, rstd)
        coef2 = bn_s._coefficients(sums2, rows, mean2, rstd2)
        dy, dys = e.empty(y.shape, e.act_dtype), e.empty(y.shape, e.act_dtype)
        lib.bn_bwd_apply2_coef(dz, e.code(dz.dtype), y, ys, e.code(y.dtype), dy, dys, e.code(dy.dtype), rows, C, coef, coef2, st)
        return dy, dys

    # -- stem: BN + ReLU + MaxPooling2D(3, 2, 'SAME') without materialising the BN output -----------------
    def forward_maxpool(self, y, sums=None):
        """Training forward of `BatchNormRelu` -> `MaxPooling2D` (tf2/resnet.py:593-611) on the conv output y
        [N,H,W,C]: returns the pooled tensor; the BN output only ever exists inside the pooling kernel."""
        e = get_engine()
        assert self.relu
        N, H, W, C = y.shape
        mean, rstd, scale, shift = self._statistics(y, True, sums)
        Ho, Wo = (H + 1) // 2, (W + 1) // 2
        out = e.empty((N, Ho, Wo, C), y.dtype)
        argmax = e.empty((N, Ho, Wo, C), torch.uint8)
        # bf16: y at each window's argmax, so that the backward BatchNorm reduction reads pooled-size tensors only
        ysel = e.empty((N, Ho, Wo, C), y.dtype) if y.dtype == torch.bfloat16 else None
        lib.bn_relu_maxpool_fwd(y, e.code(y.dtype), scale, shift, out, argmax, ysel, N, H, W, C, stream_ptr())
        self.saved = ('pool', y, argmax, ysel, mean, rstd, scale, shift)
        return out

    def backward_maxpool(self, d, d2=None):
        """d (+ d2): gradient(s) w.r.t. the pooled tensor.  Returns d(conv output)."""
        e = get_engine()
        _, y, argmax, ysel, mean, rstd, scale, shift = self.saved
        self.saved = None
        N, H, W, C = y.shape
        st = stream_ptr()
        sums = e.sums(2 * C)
        lib.maxpool_bn_bwd_reduce(d, d2, argmax, y, ysel, e.code(y.dtype), N, H, W, C, mean, rstd, scale, shift, sums, st)
        coef = self._coefficients(sums, N * H * W, mean, rstd)
        dy = e.empty(y.shape, y.dtype)
        lib.maxpool_bn_bwd_apply(d, d2, argmax, y, e.code(y.dtype), dy, N, H, W, C, coef, scale, shift, st)
        return dy

    @staticmethod
    def pool_fusable(C, dtype):
        v = 8 if dtype == torch.bfloat16 else 4
        return C % 8 == 0 and 256 % (C // v) == 0

    def __call__(self, inputs, training, residual=None, relu=None, out_dtype=None, sums=None):
        """`sums`: [2C] fp64 sum / sum of squares already produced by the conv epilogue."""
        e = get_engine()
        relu = self.relu if relu is None else relu
        C = self.C
        y = inputs
        rows = y.numel() // C
        st = stream_ptr()
        mean, rstd, scale, shift = self._statistics(y, training, sums)
        z = e.empty(y.shape, out_dtype or y.dtype)
        tail = relu and residual is not None
        bits = None
        if tail and training:
            # block tail: the ReLU mask is kept as one bit per element for the backward reduction
            bits = e.empty((rows * C // 8,), torch.uint8)
            lib.bn_apply_relu_mask(y, e.code(y.dtype), residual, z, e.code(z.dtype), rows, C, scale, shift, bits, st)
        else:
            lib.bn_apply(y, e.code(y.dtype), residual, z, e.code(z.dtype), rows, C, scale, shift, int(relu), st)
        if training:
            # BN+ReLU without residual: the backward recomputes the mask from y (scale, shift)
            self.saved = (y, bits, mean, rstd, rows, (scale, shift) if (relu and residual is None) else None)
        return z

    def backward(self, dz, dz2=None, dy_dtype=None):
        """dz (and dz2) are gradients w.r.t. the layer output.  For the block tail
        (residual add + ReLU) dz is overwritten with (dz + dz2) * relu_mask, which the
        caller routes on to the shortcut; a plain BN+ReLU leaves dz untouched.
        Returns d(inputs)."""
        e = get_engine()
        y, zmask, mean, rstd, rows, remask = self.saved
        self.saved = None
        C = self.C
        st = stream_ptr()
        sums = e.sums(2 * C)
        if zmask is not None and zmask.dtype == torch.uint8 and remask is None:
            lib.bn_bwd_reduce_bits(dz, dz2, zmask, e.code(dz.dtype), y, e.code(y.dtype), rows, C, mean, rstd, sums, st)
            msc = msh = None
        elif remask is not None and dz2 is None:
            lib.bn_bwd_relu_reduce(dz, e.code(dz.dtype), y, e.code(y.dtype), rows, C, mean, rstd,
                                   remask[0], remask[1], sums, st)
            msc, msh = remask
        else:
            if remask is not None:      # extra gradient into a plain BN+ReLU: mask in place from z
                zmask = e.empty(y.shape, dz.dtype)
                lib.bn_apply(y, e.code(y.dtype), None, zmask, e.code(zmask.dtype), rows, C, remask[0], remask[1], 1, st)
            lib.bn_bwd_reduce(dz, dz2, zmask, e.code(dz.dtype), y, e.code(y.dtype), rows, C, mean, rstd, sums, st)
            msc = msh = None
        dy = e.empty(y.shape, dy_dtype or e.act_dtype)
        coef = self._coefficients(sums, rows, mean, rstd)
        lib.bn_bwd_apply_coef(dz, e.code(dz.dtype), y, e.code(y.dtype), dy, e.code(dy.dtype), rows, C, coef, msc, msh, st)
        return dy


class ConvOp:
    """Implicit-GEMM convolution on the wgmma engine (or the CUDA-core
    verification engine).  `kernel` is the fp32 HWIO master; the wgmma engine
    reads K-major packed copies refreshed from the master on every forward."""

    def __init__(self, kernel, R, S, cin, cout, stride, stored_cin=None, need_dgrad=True):
        self.kernel = kernel
        self.R, self.S, self.cin, self.cout, self.stride = R, S, cin, cout, stride
        self.cs = stored_cin or cin
        self.need_dgrad = need_dgrad
        self.wf = self.wd = None
        self.wf3 = self.wd3 = None           # tc3: the three bf16 terms of the packed weights
        self.packed_token = None             # == engine.pack_token: operands refreshed by the multi-layer launch
        self.saved_x = None

    def _pack(self, e):
        es = 2 if e.act_dtype == torch.bfloat16 else 4
        kbe = 128 // es
        # the bf16 stem (4 stored channels) packs S+1 slots per filter row (simclr_b200.h, pack_conv_weight)
        K = self.R * (self.S + 1 if (self.cs == 4 and es == 2) else self.S) * self.cs
        Kp = (K + kbe - 1) // kbe * kbe
        if self.wf is None or self.wf.dtype != e.act_dtype:
            self.wf = e.empty((self.cout, Kp))
            kd = self.R * self.S * self.cout
            self.wd = e.empty((self.cin, (kd + kbe - 1) // kbe * kbe)) if self.need_dgrad else None
            e.register_packed(self)
        if e.pack_token is not None and self.packed_token is e.pack_token:
            return                           # refreshed by engine.pack_all() at the start of this forward
        lib.pack_conv_weight(self.kernel.value, self.wf, self.wd, e.code(e.act_dtype), self.R, self.S, self.cin,
                             self.cs, self.cout, Kp, stream_ptr())

    def _pack3(self, e):
        """Split-bf16 operands: the three bf16 terms of every weight in the ordinary packed layouts."""
        K = self.R * (self.S + 1 if self.cs == 4 else self.S) * self.cs
        Kp = (K + 63) // 64 * 64
        if self.wf3 is None:
            kd = (self.R * self.S * self.cout + 63) // 64 * 64
            self.wf3 = [e.empty((self.cout, Kp), torch.bfloat16) for _ in range(3)]
            self.wd3 = [e.empty((self.cin, kd), torch.bfloat16) if self.need_dgrad else None for _ in range(3)]
        st = stream_ptr()
        for part in range(3):
            lib.pack_conv_weight_part(self.kernel.value, self.wf3[part], self.wd3[part], part, self.R, self.S, self.cin,
                                      self.cs, self.cout, Kp, st)

    @staticmethod
    def _split(e, t):
        parts = [e.empty(t.shape, torch.bfloat16) for _ in range(3)]
        lib.split_bf16x3(t, parts[0], parts[1], parts[2], t.numel(), stream_ptr())
        return parts

    def _timed(self, e, kind, x_shape, fn):
        """Optional per-launch CUDA-event timing (bench.py roofline pass)."""
        if e.profile is None:
            return fn()
        N, H, W, _ = x_shape
        s = self.stride
        M = N * ((H - 1) // s + 1) * ((W - 1) // s + 1)
        flops = 2.0 * M * self.R * self.S * self.cin * self.cout
        ev0 = torch.cuda.Event(enable_timing=True); ev1 = torch.cuda.Event(enable_timing=True)
        ev0.record()
        r = fn()
        ev1.record()
        e.profile.append((kind, (N, H, W, self.cin, self.cout, self.R, s), flops, ev0, ev1))
        return r

    def forward(self, x, training, out_dtype=None, bn_sums=None):
        e = get_engine()
        N, H, W, Cs = x.shape
        assert Cs == self.cs, (x.shape, self.cs)
        s = self.stride
        Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
        y = e.empty((N, Ho, Wo, self.cout), out_dtype or e.act_dtype)
        st = stream_ptr()
        if e.conv_engine == 'tc':
            self._pack(e)
            self._timed(e, 'fprop', x.shape, lambda: lib.conv2d_fprop_tc(
                x, self.wf, y, e.code(x.dtype), e.code(y.dtype), N, H, W, Cs, self.cout, self.R, self.S, s, bn_sums, st))
        elif e.conv_engine == 'tc3':
            assert x.dtype == torch.float32 and y.dtype == torch.float32, 'tc3 (split bf16) is the fp32-storage mode'
            self._pack3(e)
            xs = self._split(e, x)
            self._timed(e, 'fprop', x.shape, lambda: lib.conv2d_fprop_tc3(
                xs[0], xs[1], xs[2], self.wf3[0], self.wf3[1], self.wf3[2], y, N, H, W, Cs, self.cout, self.R, self.S, s, st))
            if bn_sums is not None:
                lib.bn_stats(y, e.code(y.dtype), y.numel() // self.cout, self.cout, bn_sums, st)
            if training:
                self.saved_x = (x, xs)
            return y
        else:
            lib.conv2d_fprop_simt(x, self.kernel.value, y, e.code(x.dtype), e.code(y.dtype), N, H, W, Cs,
                                  self.cin, self.cout, self.R, self.S, s, st)
            if bn_sums is not None:
                lib.bn_stats(y, e.code(y.dtype), y.numel() // self.cout, self.cout, bn_sums, st)
        if training:
            self.saved_x = x
        return y

    def backward(self, dy, need_dx=True, dx_dtype=None):
        e = get_engine()
        x = self.saved_x
        self.saved_x = None
        if e.conv_engine == 'tc3':
            return self._backward_tc3(e, x, dy, need_dx, dx_dtype)
        N, H, W, Cs = x.shape
        st = stream_ptr()
        assert dy.dtype == x.dtype, (dy.dtype, x.dtype)
        tc = e.conv_engine == 'tc'
        # fp32 storage (verification mode): the wgmma wgrad kernel is bf16-only (MN-major tf32 needs a
        # different swizzle atom), so the fp32 wgrad runs on the CUDA-core engine.
        # The wgmma wgrad also needs 16-byte rows of dY (Cout % 8 == 0 in bf16): an odd-width supervised head
        # (e.g. 10 classes) takes the CUDA-core kernel for that one small GEMM.
        if tc and x.dtype == torch.bfloat16 and self.cout % 8 == 0:
            self._timed(e, 'wgrad', x.shape, lambda: lib.conv2d_wgrad_tc(
                x, dy, self.kernel.grad, e.code(x.dtype), N, H, W, Cs, self.cin, self.cout, self.R, self.S,
                self.stride, st))
        else:
            lib.conv2d_wgrad_simt(x, dy, self.kernel.grad, e.code(x.dtype), N, H, W, Cs, self.cin, self.cout,
                                  self.R, self.S, self.stride, st)
        if not (need_dx and self.need_dgrad):
            return None
        dx = e.empty((N, H, W, self.cin), dx_dtype or e.act_dtype)
        if tc:
            self._timed(e, 'dgrad', x.shape, lambda: lib.conv2d_dgrad_tc(
                dy, self.wd, dx, e.code(dy.dtype), e.code(dx.dtype), N, H, W, self.cin, self.cout, self.R, self.S,
                self.stride, st))
        else:
            lib.conv2d_dgrad_simt(dy, self.kernel.value, dx, e.code(dy.dtype), e.code(dx.dtype), N, H, W,
                                  self.cin, self.cout, self.R, self.S, self.stride, st)
        return dx


def _convop_backward_tc3(self, e, saved, dy, need_dx, dx_dtype):
    x, xs = saved
    N, H, W, Cs = x.shape
    st = stream_ptr()
    assert dy.dtype == torch.float32
    ds = None
    if self.cout % 8 == 0:
        ds = self._split(e, dy)
        self._timed(e, 'wgrad', x.shape, lambda: lib.conv2d_wgrad_tc3(
            xs[0], xs[1], xs[2], ds[0], ds[1], ds[2], self.kernel.grad, N, H, W, Cs, self.cin, self.cout, self.R, self.S,
            self.stride, st))
    else:       # odd-width supervised head: 16-byte rows of dY are a wgmma wgrad requirement
        lib.conv2d_wgrad_simt(x, dy, self.kernel.grad, F32, N, H, W, Cs, self.cin, self.cout, self.R, self.S,
                              self.stride, st)
    if not (need_dx and self.need_dgrad):
        return None
    if ds is None:
        ds = self._split(e, dy)
    dx = e.empty((N, H, W, self.cin), torch.float32)
    self._timed(e, 'dgrad', x.shape, lambda: lib.conv2d_dgrad_tc3(
        ds[0], ds[1], ds[2], self.wd3[0], self.wd3[1], self.wd3[2], dx, N, H, W, self.cin, self.cout, self.R, self.S,
        self.stride, st))
    return dx


ConvOp._backward_tc3 = _convop_backward_tc3


def conv_bn(conv, bn, x, training, **bn_kwargs):
    """conv -> BatchNorm with the batch statistics produced by the conv epilogue
    (one pass over the conv output saved per layer)."""
    e = get_engine()
    op = conv.op if hasattr(conv, 'op') else conv
    if not training:
        return bn(op.forward(x, training), training, **bn_kwargs)
    sums = e.sums(2 * op.cout)
    y = op.forward(x, training, bn_sums=sums)
    return bn(y, training, sums=sums, **bn_kwargs)


class Conv2dFixedPadding:  # pylint: disable=missing-docstring
    """tf2/resnet.py:183-208: stride 1 -> 'SAME'; stride > 1 -> FixedPadding +
    'VALID' (folded into the gather bounds of the kernel), no bias."""

    def __init__(self, vs, scope, cin, filters, kernel_size, strides, stored_cin=None, need_dgrad=True):
        lname = vs.namer('conv2d_fixed_padding')
        cname = vs.namer('conv2d')
        self.kernel = vs.add('%s/%s/%s/kernel:0' % (scope, lname, cname),
                             (kernel_size, kernel_size, cin, filters), 'variance_scaling')
        self.op = ConvOp(self.kernel, kernel_size, kernel_size, cin, filters, strides, stored_cin, need_dgrad)
        self.cout = filters

    def __call__(self, inputs, training):
        return self.op.forward(inputs, training)

    def backward(self, grad, need_dx=True):
        return self.op.backward(grad, need_dx)


class _Shortcut:
    """Projection shortcut: Conv1x1(stride) + BN without ReLU (tf2/resnet.py:342-353,415-423);
    with SK the ResNet-D form: [FixedPadding(2)] AveragePooling2D(2, stride) + Conv1x1(1) + BN
    (tf2/resnet.py:331-341,401-414)."""

    def __init__(self, vs, scope, cin, filters_out, strides):
        self.resnet_d = FLAGS.sk_ratio > 0
        self.strides = strides
        self.conv = Conv2dFixedPadding(vs, scope, cin, filters_out, 1, 1 if self.resnet_d else strides)
        self.bn = BatchNormRelu(vs, scope, filters_out, relu=False)
        self.in_shape = None

    def _pre(self, x):
        if self.resnet_d:
            e = get_engine()
            N, H, W, C = x.shape
            s = self.strides
            Ho, Wo = (H, W) if s == 1 else ((H - 1) // 2 + 1, (W - 1) // 2 + 1)
            y = e.empty((N, Ho, Wo, C), x.dtype)
            lib.avgpool2x2_fwd(x, y, e.code(x.dtype), N, H, W, C, s, stream_ptr())
            self.in_shape = (N, H, W, C)
            x = y
        return x

    def __call__(self, x, training):
        return conv_bn(self.conv, self.bn, self._pre(x), training)

    def forward_raw(self, x):
        """Training only: the conv output and its batch statistics; the BatchNorm is applied by the block tail
        (`BatchNormRelu.forward_tail2`)."""
        e = get_engine()
        sums = e.sums(2 * self.conv.cout)
        return self.conv.op.forward(self._pre(x), True, bn_sums=sums), sums

    def backward(self, d):
        return self.backward_conv(self.bn.backward(d))

    def backward_conv(self, d):
        d = self.conv.backward(d)
        if self.resnet_d:
            e = get_engine()
            N, H, W, C = self.in_shape
            dx = e.empty((N, H, W, C), d.dtype)
            lib.avgpool2x2_bwd(d, dx, e.code(d.dtype), N, H, W, C, self.strides, stream_ptr())
            d = dx
        return d


class SK_Conv2D:  # pylint: disable=invalid-name
    """Selective kernel convolutional layer (tf2/resnet.py:217-277)."""

    def __init__(self, vs, scope, cin, filters, strides, sk_ratio, min_dim=32):
        from . import model as model_lib       # the two mixing "convs" are dense layers on [N, f]
        scope = scope + '/' + vs.namer('sk_conv2d')
        self.filters = filters
        # Two stream convs (using split and both are 3x3).
        self.conv2d_fixed_padding = Conv2dFixedPadding(vs, scope, cin, 2 * filters, 3, strides)
        self.batch_norm_relu = BatchNormRelu(vs, scope, 2 * filters)
        # Mixing weights for two streams.
        mid_dim = max(int(filters * sk_ratio), min_dim)
        self.mid_dim = mid_dim
        c0 = vs.namer('conv2d')
        self.kernel0 = vs.add('%s/%s/kernel:0' % (scope, c0), (1, 1, filters, mid_dim), 'variance_scaling')
        self.conv2d_0 = ConvOp(self.kernel0, 1, 1, filters, mid_dim, 1)
        self.batch_norm_relu_1 = BatchNormRelu(vs, scope, mid_dim)
        c1 = vs.namer('conv2d')
        self.kernel1 = vs.add('%s/%s/kernel:0' % (scope, c1), (1, 1, mid_dim, 2 * filters), 'variance_scaling')
        self.conv2d_1 = ConvOp(self.kernel1, 1, 1, mid_dim, 2 * filters, 1)
        self.saved = None

    def __call__(self, inputs, training):
        e = get_engine()
        st = stream_ptr()
        f = self.filters
        x = conv_bn(self.conv2d_fixed_padding, self.batch_norm_relu, inputs, training)      # [N,H,W,2f]
        N, H, W, _ = x.shape
        HW = H * W
        g32 = e.empty((N, f), torch.float32)
        lib.sk_pool(x, e.code(x.dtype), g32, N, HW, f, st)                                  # mean of the stream sum
        g = g32 if e.act_dtype == torch.float32 else self._cast(g32, e.act_dtype)
        h = self.conv2d_0.forward(g.view(N, 1, 1, f), training).view(N, self.mid_dim)
        h = self.batch_norm_relu_1(h, training)
        logits = self.conv2d_1.forward(h.view(N, 1, 1, self.mid_dim), training, out_dtype=torch.float32).view(N, 2 * f)
        mixing = e.empty((N, 2 * f), torch.float32)
        out = e.empty((N, H, W, f), x.dtype)
        lib.sk_mix_fwd(x, logits, mixing, out, e.code(x.dtype), N, HW, f, st)
        if training:
            self.saved = (x, mixing, (N, H, W))
        return out

    @staticmethod
    def _cast(t, dtype):
        e = get_engine()
        o = e.empty(t.shape, dtype)
        lib.cast(t, e.code(t.dtype), o, e.code(dtype), t.numel(), stream_ptr())
        return o

    def backward(self, dout):
        e = get_engine()
        st = stream_ptr()
        x, mixing, (N, H, W) = self.saved
        self.saved = None
        f, HW = self.filters, H * W
        dlogits = e.empty((N, 2 * f), torch.float32)
        lib.sk_mix_bwd_reduce(dout, x, mixing, dlogits, e.code(dout.dtype), N, HW, f, st)
        dl = dlogits if e.act_dtype == torch.float32 else self._cast(dlogits, e.act_dtype)
        dh = self.conv2d_1.backward(dl.view(N, 1, 1, 2 * f)).view(N, self.mid_dim)
        dh = self.batch_norm_relu_1.backward(dh)
        dg = self.conv2d_0.backward(dh.view(N, 1, 1, self.mid_dim)).view(N, f)
        dg32 = dg if dg.dtype == torch.float32 else self._cast(dg, torch.float32)
        dx = e.empty(x.shape, x.dtype)
        lib.sk_mix_bwd_apply(dout, mixing, dg32, dx, e.code(dout.dtype), N, HW, f, st)
        d = self.batch_norm_relu.backward(dx)
        return self.conv2d_fixed_padding.backward(d)


class SE_Layer:  # pylint: disable=invalid-name
    """Squeeze and Excitation layer (tf2/resnet.py:280-311).  The expand width follows the input
    (SURVEY Q9).  The two gate "convs" act on [N,1,1,C] and are arbitrarily narrow (max(1,
    int(filters*se_ratio))), so they run on the CUDA-core dense path in fp32."""

    def __init__(self, vs, scope, cin, filters, se_ratio):
        scope = scope + '/' + vs.namer('se_layer')
        self.cin = cin
        self.mid = max(1, int(filters * se_ratio))
        c0 = vs.namer('conv2d')
        self.reduce_kernel = vs.add('%s/%s/kernel:0' % (scope, c0), (1, 1, cin, self.mid), 'variance_scaling')
        self.reduce_bias = vs.add('%s/%s/bias:0' % (scope, c0), (self.mid,), 'zeros')
        c1 = vs.namer('conv2d')
        self.expand_kernel = vs.add('%s/%s/kernel:0' % (scope, c1), (1, 1, self.mid, cin), 'variance_scaling')
        self.expand_bias = vs.add('%s/%s/bias:0' % (scope, c1), (cin,), 'zeros')
        self.saved = None

    def __call__(self, inputs, training):
        e = get_engine()
        st = stream_ptr()
        N, H, W, C = inputs.shape
        m = e.empty((N, C), torch.float32)
        lib.global_avgpool_fwd(inputs, e.code(inputs.dtype), m, F32, N, H * W, C, st)
        h = e.empty((N, self.mid), torch.float32)
        lib.conv2d_fprop_simt(m, self.reduce_kernel.value, h, F32, F32, N, 1, 1, C, C, self.mid, 1, 1, 1, st)
        lib.bias_add(h, self.reduce_bias.value, N, self.mid, st)
        lib.relu_inplace(h, None, h.numel(), st)
        l = e.empty((N, C), torch.float32)
        lib.conv2d_fprop_simt(h, self.expand_kernel.value, l, F32, F32, N, 1, 1, self.mid, self.mid, C, 1, 1, 1, st)
        lib.bias_add(l, self.expand_bias.value, N, C, st)
        out = e.empty(inputs.shape, inputs.dtype)
        lib.se_scale_fwd(inputs, l, out, e.code(inputs.dtype), N, H * W, C, st)
        if training:
            self.saved = (inputs, m, h, l)
        return out

    def backward(self, dout):
        e = get_engine()
        st = stream_ptr()
        x, m, h, l = self.saved
        self.saved = None
        N, H, W, C = x.shape
        dl = e.empty((N, C), torch.float32)
        lib.se_scale_bwd_reduce(dout, x, l, dl, e.code(dout.dtype), N, H * W, C, st)
        lib.bias_grad(dl, self.expand_bias.grad, N, C, st)
        lib.conv2d_wgrad_simt(h, dl, self.expand_kernel.grad, F32, N, 1, 1, self.mid, self.mid, C, 1, 1, 1, st)
        dh = e.empty((N, self.mid), torch.float32)
        lib.conv2d_dgrad_simt(dl, self.expand_kernel.value, dh, F32, F32, N, 1, 1, self.mid, C, 1, 1, 1, st)
        lib.relu_inplace(dh, h, dh.numel(), st)
        lib.bias_grad(dh, self.reduce_bias.grad, N, self.mid, st)
        lib.conv2d_wgrad_simt(m, dh, self.reduce_kernel.grad, F32, N, 1, 1, C, C, self.mid, 1, 1, 1, st)
        dm = e.empty((N, C), torch.float32)
        lib.conv2d_dgrad_simt(dh, self.reduce_kernel.value, dm, F32, F32, N, 1, 1, C, self.mid, 1, 1, 1, st)
        dx = e.empty(x.shape, x.dtype)
        lib.se_scale_bwd_apply(dout, l, dm, dx, e.code(dout.dtype), N, H * W, C, st)
        return dx


class _AddRelu:
    """relu(inputs + shortcut) as its own op (needed when an SE layer sits between the last BN
    and the residual add, tf2/resnet.py:379-382,473-487)."""

    def __init__(self):
        self.saved = None

    def __call__(self, x, shortcut, training):
        e = get_engine()
        C = x.shape[-1]
        ones = torch.ones(C, dtype=torch.float32, device=e.device)
        zeros = torch.zeros(C, dtype=torch.float32, device=e.device)
        out = e.empty(x.shape, x.dtype)
        lib.bn_apply(x, e.code(x.dtype), shortcut, out, e.code(out.dtype), x.numel() // C, C, ones, zeros, 1, stream_ptr())
        if training:
            self.saved = (out, ones, zeros)
        return out

    def backward(self, d_out, d_out2=None):
        """d_out <- (d_out + d_out2) * [out > 0] in place; it is the gradient of both addends."""
        e = get_engine()
        out, ones, zeros = self.saved
        self.saved = None
        C = out.shape[-1]
        scratch = e.empty((2 * C,), torch.float64)
        lib.bn_bwd_reduce(d_out, d_out2, out, e.code(d_out.dtype), out, e.code(out.dtype), out.numel() // C, C,
                          zeros, ones, scratch, stream_ptr())
        return d_out


class ResidualBlock:  # pylint: disable=missing-docstring
    """tf2/resnet.py:314-382."""

    def __init__(self, vs, scope, cin, filters, strides, use_projection=False):
        scope = scope + '/' + vs.namer('residual_block')
        self.shortcut = _Shortcut(vs, scope, cin, filters, strides) if use_projection else None
        self.c1 = Conv2dFixedPadding(vs, scope, cin, filters, 3, strides)
        self.b1 = BatchNormRelu(vs, scope, filters)
        self.c2 = Conv2dFixedPadding(vs, scope, filters, filters, 3, 1)
        self.b2 = BatchNormRelu(vs, scope, filters, relu=False, init_zero=True)
        self.se_layer = SE_Layer(vs, scope, filters, filters, FLAGS.se_ratio) if FLAGS.se_ratio > 0 else None
        self.add_relu = _AddRelu() if self.se_layer is not None else None
        self.cout = filters

    def __call__(self, inputs, training):
        self.fused_tail = (training and self.shortcut is not None and self.se_layer is None and
                           BatchNormRelu.tail2_enabled())
        if self.fused_tail:
            ys, sums_s = self.shortcut.forward_raw(inputs)
        else:
            shortcut = inputs if self.shortcut is None else self.shortcut(inputs, training)
        x = conv_bn(self.c1, self.b1, inputs, training)
        if self.se_layer is not None:
            x = self.se_layer(conv_bn(self.c2, self.b2, x, training), training)
            return self.add_relu(x, shortcut, training)
        if self.fused_tail:
            sums = get_engine().sums(2 * self.c2.cout)
            return self.b2.forward_tail2(self.c2.op.forward(x, True, bn_sums=sums), sums, ys, self.shortcut.bn, sums_s)
        return conv_bn(self.c2, self.b2, x, training, residual=shortcut, relu=True)     # relu(inputs + shortcut), :382

    def backward(self, d_out, d_out2=None):
        dys = None
        if self.se_layer is not None:
            d_out = self.add_relu.backward(d_out, d_out2)
            dy = self.b2.backward(self.se_layer.backward(d_out))
        elif self.fused_tail:
            dy, dys = self.b2.backward_tail2(d_out, d_out2)
        else:
            dy = self.b2.backward(d_out, d_out2)      # d_out <- (d_out + d_out2) * [out > 0]
        d = self.c2.backward(dy)
        d = self.b1.backward(d)
        dx_a = self.c1.backward(d)
        if dys is not None:
            dx_b = self.shortcut.backward_conv(dys)
        else:
            dx_b = d_out if self.shortcut is None else self.shortcut.backward(d_out)
        return dx_a, dx_b


class BottleneckBlock:
    """tf2/resnet.py:385-487 (DropBlock is dead code in the reference, SURVEY Q2)."""

    def __init__(self, vs, scope, cin, filters, strides, use_projection=False):
        scope = scope + '/' + vs.namer('bottleneck_block')
        self.shortcut = _Shortcut(vs, scope, cin, 4 * filters, strides) if use_projection else None
        self.c1 = Conv2dFixedPadding(vs, scope, cin, filters, 1, 1)
        self.b1 = BatchNormRelu(vs, scope, filters)
        if FLAGS.sk_ratio > 0:
            self.sk = SK_Conv2D(vs, scope, filters, filters, strides, FLAGS.sk_ratio)
        else:
            self.sk = None
            self.c2 = Conv2dFixedPadding(vs, scope, filters, filters, 3, strides)
            self.b2 = BatchNormRelu(vs, scope, filters)
        self.c3 = Conv2dFixedPadding(vs, scope, filters, 4 * filters, 1, 1)
        self.b3 = BatchNormRelu(vs, scope, 4 * filters, relu=False, init_zero=True)
        # tf2/resnet.py:474-476 builds SE with `filters`; its expand width follows the input (4*filters)
        self.se_layer = SE_Layer(vs, scope, 4 * filters, filters, FLAGS.se_ratio) if FLAGS.se_ratio > 0 else None
        self.add_relu = _AddRelu() if self.se_layer is not None else None
        self.cout = 4 * filters

    def __call__(self, inputs, training):
        self.fused_tail = (training and self.shortcut is not None and self.se_layer is None and
                           BatchNormRelu.tail2_enabled())
        if self.fused_tail:
            ys, sums_s = self.shortcut.forward_raw(inputs)
        else:
            shortcut = inputs if self.shortcut is None else self.shortcut(inputs, training)
        x = conv_bn(self.c1, self.b1, inputs, training)
        x = self.sk(x, training) if self.sk is not None else conv_bn(self.c2, self.b2, x, training)
        if self.se_layer is not None:
            x = self.se_layer(conv_bn(self.c3, self.b3, x, training), training)
            return self.add_relu(x, shortcut, training)
        if self.fused_tail:
            sums = get_engine().sums(2 * self.c3.cout)
            return self.b3.forward_tail2(self.c3.op.forward(x, True, bn_sums=sums), sums, ys, self.shortcut.bn, sums_s)
        return conv_bn(self.c3, self.b3, x, training, residual=shortcut, relu=True)     # relu(inputs + shortcut), :487

    def backward(self, d_out, d_out2=None):
        dys = None
        if self.se_layer is not None:
            d_out = self.add_relu.backward(d_out, d_out2)
            dy = self.b3.backward(self.se_layer.backward(d_out))
        elif self.fused_tail:
            dy, dys = self.b3.backward_tail2(d_out, d_out2)
        else:
            dy = self.b3.backward(d_out, d_out2)
        d = self.c3.backward(dy)
        if self.sk is not None:
            d = self.sk.backward(d)
        else:
            d = self.b2.backward(d)
            d = self.c2.backward(d)
        d = self.b1.backward(d)
        dx_a = self.c1.backward(d)
        if dys is not None:
            dx_b = self.shortcut.backward_conv(dys)
        else:
            dx_b = d_out if self.shortcut is None else self.shortcut.backward(d_out)
        return dx_a, dx_b


class BlockGroup:  # pylint: disable=missing-docstring
    """tf2/resnet.py:490-526: the first block always has a projection shortcut."""

    def __init__(self, vs, scope, cin, filters, block_fn, blocks, strides, name):
        self._name = name
        scope = scope + '/' + name
        self.layers = [block_fn(vs, scope, cin, filters, strides, use_projection=True)]
        for _ in range(1, blocks):
            self.layers.append(block_fn(vs, scope, self.layers[-1].cout, filters, 1))
        self.cout = self.layers[-1].cout

    def __call__(self, inputs, training):
        for layer in self.layers:
            inputs = layer(inputs, training)
        return inputs

    def backward(self, d, d2=None):
        for layer in reversed(self.layers):
            d, d2 = layer.backward(d, d2)
        return d, d2


class Resnet:  # pylint: disable=missing-docstring
    """tf2/resnet.py:529-699.  Input [N,H,W,4]: 3 image channels + one zero
    channel so every pixel is 8/16 bytes for the stem's gather."""

    STEM_CS = 4

    def __init__(self, vs, block_fn, layers, width_multiplier, cifar_stem=False):
        scope = 'resnet'
        wm = width_multiplier
        self.cifar_stem = cifar_stem
        self.stem_extra = []          # ResNet-D: two more conv+BN pairs after the first
        # Finetuning with --fine_tune_after_block=k >= 0: the stem and block groups 1..k are `trainable=False`
        # Keras layers (tf2/resnet.py:548-549,619-692): variables non-trainable, BatchNorm in inference mode,
        # and a stop_gradient in front of group k+1 (:675-681).
        ft = FLAGS.fine_tune_after_block if FLAGS.train_mode == 'finetune' else -1
        self.frozen_groups = max(ft, 0) if ft >= 0 else 0          # number of leading block groups frozen
        self.stem_frozen = ft >= 0
        vs.default_trainable = not self.stem_frozen
        if cifar_stem:                                            # :551-564
            self.stem_conv = Conv2dFixedPadding(vs, scope, 3, 64 * wm, 3, 1, stored_cin=self.STEM_CS, need_dgrad=False)
            self.stem_bn = BatchNormRelu(vs, scope, 64 * wm)
        elif FLAGS.sk_ratio > 0:                                  # ResNet-D stem :566-591
            self.stem_conv = Conv2dFixedPadding(vs, scope, 3, 64 * wm // 2, 3, 2, stored_cin=self.STEM_CS, need_dgrad=False)
            self.stem_bn = BatchNormRelu(vs, scope, 64 * wm // 2)
            c2 = Conv2dFixedPadding(vs, scope, 64 * wm // 2, 64 * wm // 2, 3, 1)
            b2 = BatchNormRelu(vs, scope, 64 * wm // 2)
            c3 = Conv2dFixedPadding(vs, scope, 64 * wm // 2, 64 * wm, 3, 1)
            b3 = BatchNormRelu(vs, scope, 64 * wm)
            self.stem_extra = [(c2, b2), (c3, b3)]
        else:                                                     # :593-604
            self.stem_conv = Conv2dFixedPadding(vs, scope, 3, 64 * wm, 7, 2, stored_cin=self.STEM_CS, need_dgrad=False)
            self.stem_bn = BatchNormRelu(vs, scope, 64 * wm)
        self.block_groups = []
        cin = 64 * wm
        for i, (f, s) in enumerate(zip([64, 128, 256, 512], [1, 2, 2, 2])):
            if self.stem_frozen and ft == i:
                vs.default_trainable = True
            g = BlockGroup(vs, scope, cin, f * wm, block_fn, layers[i], s, 'block_group%d' % (i + 1))
            self.block_groups.append(g)
            cin = g.cout
        vs.default_trainable = True
        self.cout = cin
        self.saved = None

    def __call__(self, inputs, training, endpoints=None):
        e = get_engine()
        st = stream_ptr()
        train_all = training
        training = train_all and not self.stem_frozen          # frozen layers: inference-mode BN, nothing saved
        layers = [(self.stem_conv, self.stem_bn)] + list(self.stem_extra)
        last_bn = layers[-1][1]
        # training: the last stem BatchNorm + ReLU is applied inside the max-pooling kernel (its output is never stored)
        fuse_pool = (training and not self.cifar_stem and endpoints is None and
                     BatchNormRelu.pool_fusable(last_bn.C, e.act_dtype))
        x = inputs
        for i, (conv, bn) in enumerate(layers):
            op = conv.op
            if fuse_pool and i == len(layers) - 1:
                sums = e.sums(2 * op.cout)
                x = bn.forward_maxpool(op.forward(x, training, bn_sums=sums), sums)
            elif endpoints is not None and i == 0:
                x = conv(x, training)
                endpoints['initial_conv'] = x
                x = bn(x, training)
            else:
                x = conv_bn(conv, bn, x, training)
        self._pool_fused = fuse_pool
        pool_saved = None
        if not self.cifar_stem and not fuse_pool:                 # MaxPooling2D(3, 2, 'SAME'), :605-611
            N, H, W, C = x.shape
            Ho, Wo = (H + 1) // 2, (W + 1) // 2
            y = e.empty((N, Ho, Wo, C))
            argmax = e.empty((N, Ho, Wo, C), torch.uint8)
            lib.maxpool3x3s2_fwd(x, y, argmax, e.code(x.dtype), N, H, W, C, st)
            pool_saved = (argmax, (N, H, W, C))
            x = y
        if endpoints is not None:
            endpoints['initial_max_pool'] = x
        for i, g in enumerate(self.block_groups):
            x = g(x, train_all and not (self.stem_frozen and i < self.frozen_groups))
            if endpoints is not None:
                endpoints['block_group%d' % (i + 1)] = x
        training = train_all
        N, H, W, C = x.shape
        out = e.empty((N, C))
        lib.global_avgpool_fwd(x, e.code(x.dtype), out, e.code(out.dtype), N, H * W, C, st)   # :693-696
        if endpoints is not None:
            endpoints['final_avg_pool'] = out
        if training:
            self.saved = (pool_saved, (N, H, W, C))
        return out

    def backward(self, d_hiddens):
        self.backward_bottom(self.backward_top(d_hiddens, 0), 0)

    def backward_top(self, d_hiddens, split):
        """Backward through the mean over H,W and block groups [split, 4) -- the last groups hold almost all of the
        parameters (ResNet-50: groups 3-4 + heads = 96 %) but little of the backward time, so a data-parallel step
        can start reducing their gradients while `backward_bottom` is still running.  Returns the state
        `backward_bottom(state, split)` continues from (None: a frozen boundary was reached)."""
        e = get_engine()
        st = stream_ptr()
        pool_saved, (N, H, W, C) = self.saved
        self.saved = None
        d = e.empty((N, H, W, C))
        lib.global_avgpool_bwd(d_hiddens, e.code(d_hiddens.dtype), d, e.code(d.dtype), N, H * W, C, st)
        d2 = None
        for i in reversed(range(split, len(self.block_groups))):
            if self.stem_frozen and i < self.frozen_groups:
                return None                 # tf.stop_gradient in front of block group `fine_tune_after_block` + 1
            d, d2 = self.block_groups[i].backward(d, d2)
        return (d, d2, pool_saved)

    def backward_bottom(self, state, split):
        if state is None:
            return
        e = get_engine()
        st = stream_ptr()
        d, d2, pool_saved = state
        for i in reversed(range(0, split)):
            if self.stem_frozen and i < self.frozen_groups:
                return
            d, d2 = self.block_groups[i].backward(d, d2)
        if self.stem_frozen:
            return
        layers = [(self.stem_conv, self.stem_bn)] + list(self.stem_extra)
        if self._pool_fused:
            conv, bn = layers.pop()
            dy = bn.backward_maxpool(d, d2)          # pooling backward + BatchNorm backward, no dz tensor
            d, d2 = conv.backward(dy, need_dx=bool(layers)), None
        elif pool_saved is not None:
            argmax, (N, H, W, C) = pool_saved
            lib.add_inplace(d, d2, e.code(d.dtype), d.numel(), st)
            dx = e.empty((N, H, W, C))
            lib.maxpool3x3s2_bwd(d, argmax, dx, e.code(d.dtype), N, H, W, C, st)
            d, d2 = dx, None
        while layers:
            conv, bn = layers.pop()
            d = conv.backward(bn.backward(d, d2), need_dx=bool(layers))
            d2 = None


MODEL_PARAMS = {  # tf2/resnet.py:709-734
    18: (ResidualBlock, [2, 2, 2, 2]), 34: (ResidualBlock, [3, 4, 6, 3]),
    50: (BottleneckBlock, [3, 4, 6, 3]), 101: (BottleneckBlock, [3, 4, 23, 3]),
    152: (BottleneckBlock, [3, 8, 36, 3]), 200: (BottleneckBlock, [3, 24, 36, 3]),
}


def resnet(resnet_depth, width_multiplier, cifar_stem=False, data_format='channels_last',
           dropblock_keep_probs=None, dropblock_size=None, vs=None):
    """Returns the ResNet model for a given size (tf2/resnet.py:702-747, same arguments).

    `vs` (this implementation only): the `engine.VarStore` the variables are registered in; a
    fresh one is created when omitted (exposed as `.vs`, call `.vs.materialize(device)` before
    use).  Only `channels_last` exists on this path."""
    from .engine import VarStore
    if resnet_depth not in MODEL_PARAMS:
        raise ValueError('Not a valid resnet_depth:', resnet_depth)
    if data_format != 'channels_last':
        raise ValueError('only channels_last is supported')
    del dropblock_keep_probs, dropblock_size      # DropBlock is never enabled by the reference
    block_fn, layers = MODEL_PARAMS[resnet_depth]
    if vs is None:
        vs = VarStore()
    net = Resnet(vs, block_fn, layers, width_multiplier, cifar_stem=cifar_stem)
    net.vs = vs
    return net
