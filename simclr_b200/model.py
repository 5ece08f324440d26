"""Model, heads, LR schedule and optimizer factory of the reference
(`tf2/model.py`) on the H100 engine.  Same class / function names, constructor
arguments and error behaviour; variables are laid out in flat buffers and the
backward pass is an explicit schedule (`Model.backward`).
"""
import math

import torch

from ._lib import lib, stream_ptr
from .engine import VarStore, get_engine
from .flags_def import FLAGS
from . import resnet
from . import lars_optimizer
from . import data_util


def build_optimizer(learning_rate):
    """tf2/model.py:29-44."""
    if FLAGS.optimizer == 'lars':
        return lars_optimizer.LARSOptimizer(
            learning_rate,
            momentum=FLAGS.momentum,
            weight_decay=FLAGS.weight_decay,
            exclude_from_weight_decay=['batch_normalization', 'bias', 'head_supervised'])
    elif FLAGS.optimizer == 'momentum':
        from . import optimizers
        return optimizers.SGD(learning_rate, FLAGS.momentum, nesterov=True)
    elif FLAGS.optimizer == 'adam':
        from . import optimizers
        return optimizers.Adam(learning_rate)
    else:
        raise ValueError('Unknown optimizer {}'.format(FLAGS.optimizer))


def add_weight_decay(model, adjust_per_optimizer=True):
    """tf2/model.py:47-69.  Returns the loss term as a device scalar tensor (or 0)."""
    e = get_engine()
    if adjust_per_optimizer and 'lars' in FLAGS.optimizer:
        vs = [v for v in model.trainable_variables if 'head_supervised' in v.name and 'bias' not in v.name]
    else:
        vs = [v for v in model.trainable_weights if 'batch_normalization' not in v.name]
    if not vs:
        return 0
    total = e.zeros((1,), torch.float32)
    for v in vs:
        out = e.empty((257,), torch.float32)
        lib.l2_loss(v.value, v.numel, out, stream_ptr())
        total += out[:1]
    return FLAGS.weight_decay * total[0]


def get_train_steps(num_examples):
    """tf2/model.py:72-75."""
    return FLAGS.train_steps or (num_examples * FLAGS.train_epochs // FLAGS.train_batch_size + 1)


class WarmUpAndCosineDecay:
    """tf2/model.py:78-116 (host scalar; evaluated at the pre-increment iteration)."""

    def __init__(self, base_learning_rate, num_examples, name=None):
        self.base_learning_rate = base_learning_rate
        self.num_examples = num_examples
        self._name = name

    def __call__(self, step):
        step = int(step)
        warmup_steps = int(round(FLAGS.warmup_epochs * self.num_examples // FLAGS.train_batch_size))
        if FLAGS.learning_rate_scaling == 'linear':
            scaled_lr = self.base_learning_rate * FLAGS.train_batch_size / 256.
        elif FLAGS.learning_rate_scaling == 'sqrt':
            scaled_lr = self.base_learning_rate * math.sqrt(FLAGS.train_batch_size)
        else:
            raise ValueError('Unknown learning rate scaling {}'.format(FLAGS.learning_rate_scaling))
        learning_rate = step / float(warmup_steps) * scaled_lr if warmup_steps else scaled_lr
        total_steps = get_train_steps(self.num_examples)
        decay_steps = total_steps - warmup_steps
        if step < warmup_steps:
            return learning_rate
        s = min(step - warmup_steps, decay_steps)
        return scaled_lr * 0.5 * (1.0 + math.cos(math.pi * s / decay_steps))   # CosineDecay, alpha=0

    def get_config(self):
        return {'base_learning_rate': self.base_learning_rate, 'num_examples': self.num_examples}


class LinearLayer:
    """tf2/model.py:119-154: Dense (a 1x1 'conv' on [rows,1,1,Cin]) + optional BN."""

    def __init__(self, vs, scope, cin, num_classes, use_bias=True, use_bn=False, name='linear_layer',
                 need_dgrad=True):
        self.num_classes = num_classes
        self.use_bias = use_bias
        self.use_bn = use_bn
        self._name = name
        scope = scope + '/' + name
        dname = vs.namer('dense')
        self.kernel = vs.add('%s/%s/kernel:0' % (scope, dname), (cin, num_classes), 'normal_0.01')
        self.bias = None
        if use_bias and not use_bn:
            self.bias = vs.add('%s/%s/bias:0' % (scope, dname), (num_classes,), 'zeros')
        self.op = resnet.ConvOp(self.kernel, 1, 1, cin, num_classes, 1, need_dgrad=need_dgrad)
        if use_bn:
            self.bn_relu = resnet.BatchNormRelu(vs, scope, num_classes, relu=False, center=use_bias)
        self.cin = cin

    def __call__(self, inputs, training, relu=False, out_dtype=None):
        assert inputs.dim() == 2, inputs.shape
        e = get_engine()
        rows = inputs.shape[0]
        y_dtype = out_dtype if (out_dtype is not None and not self.use_bn) else (
            torch.float32 if out_dtype == torch.float32 else None)
        sums = e.sums(2 * self.num_classes) if (self.use_bn and training) else None
        y = self.op.forward(inputs.view(rows, 1, 1, self.cin), training, out_dtype=y_dtype,
                            bn_sums=sums).view(rows, self.num_classes)
        if self.bias is not None:
            assert y.dtype == torch.float32
            lib.bias_add(y, self.bias.value, rows, self.num_classes, stream_ptr())
        if self.use_bn:
            y = self.bn_relu(y, training, relu=relu, out_dtype=out_dtype, sums=sums)
        return y

    def backward(self, d, need_dx=True):
        e = get_engine()
        if self.use_bn:
            d = self.bn_relu.backward(d, dy_dtype=e.act_dtype)
        rows = d.shape[0]
        if self.bias is not None:
            lib.bias_grad(d, self.bias.grad, rows, self.num_classes, stream_ptr())
        if d.dtype != e.act_dtype:
            dc = e.empty(d.shape)
            lib.cast(d, e.code(d.dtype), dc, e.code(dc.dtype), d.numel(), stream_ptr())
            d = dc
        dx = self.op.backward(d.view(rows, 1, 1, self.num_classes), need_dx)
        return None if dx is None else dx.view(rows, self.cin)


class ProjectionHead:
    """tf2/model.py:157-213."""

    def __init__(self, vs=None, cin=None, **kwargs):
        self.linear_layers = []
        scope = 'projection_head'
        if FLAGS.proj_head_mode == 'none':
            pass
        elif FLAGS.proj_head_mode == 'linear':
            self.linear_layers = [LinearLayer(vs, scope, cin, FLAGS.proj_out_dim, use_bias=False, use_bn=True,
                                              name='l_0')]
        elif FLAGS.proj_head_mode == 'nonlinear':
            for j in range(FLAGS.num_proj_layers):
                if j != FLAGS.num_proj_layers - 1:
                    # for the middle layers, use bias and relu for the output.
                    self.linear_layers.append(LinearLayer(vs, scope, cin, cin, use_bias=True, use_bn=True,
                                                          name='nl_%d' % j))
                else:
                    # for the final layer, neither bias nor relu is used.
                    self.linear_layers.append(LinearLayer(vs, scope, cin, FLAGS.proj_out_dim, use_bias=False,
                                                          use_bn=True, name='nl_%d' % j))
        else:
            raise ValueError('Unknown head projection mode {}'.format(FLAGS.proj_head_mode))

    def __call__(self, inputs, training):
        if FLAGS.proj_head_mode == 'none':
            return inputs  # the reference's caller then fails to unpack (SURVEY Q1)
        if FLAGS.proj_head_mode == 'linear':
            raise ValueError("proj_head_mode='linear' returns None in the reference (tf2/model.py:196-199)")
        hiddens_list = [inputs]
        n = FLAGS.num_proj_layers
        for j in range(n):
            last = j == n - 1
            # ReLU of the middle layers (tf2/model.py:203-205) is fused into the BN apply;
            # the final layer's output is fp32 for the loss.
            hiddens = self.linear_layers[j](hiddens_list[-1], training, relu=not last,
                                            out_dtype=torch.float32 if last else None)
            hiddens_list.append(hiddens)
        return hiddens_list[-1], hiddens_list[FLAGS.ft_proj_selector]

    def backward(self, d_proj_out, upto=None):
        """Backward through layers [0, upto) (all of them by default): `upto` = `ft_proj_selector` when the
        gradient enters at hiddens_list[ft_proj_selector] (finetuning, tf2/model.py:213,267-270)."""
        d = d_proj_out
        layers = self.linear_layers if upto is None else self.linear_layers[:upto]
        for layer in reversed(layers):
            d = layer.backward(d)
        return d


class SupervisedHead:
    """tf2/model.py:216-225."""

    def __init__(self, num_classes, vs=None, cin=None, name='head_supervised', **kwargs):
        # pretraining: stop_gradient in front of the head (no dgrad); finetuning: the gradient flows on
        self.need_dx = FLAGS.train_mode == 'finetune'
        self.linear_layer = LinearLayer(vs, name, cin, num_classes, need_dgrad=self.need_dx)

    def __call__(self, inputs, training):
        e = get_engine()
        if inputs.dtype != e.act_dtype:       # ft_proj_selector = -1: the fp32 projection output feeds the head
            c = e.empty(inputs.shape)
            lib.cast(inputs, e.code(inputs.dtype), c, e.code(c.dtype), inputs.numel(), stream_ptr())
            inputs = c
        return self.linear_layer(inputs, training, out_dtype=torch.float32)

    def backward(self, d_logits):
        return self.linear_layer.backward(d_logits, need_dx=self.need_dx)


class Model:
    """Resnet model with projection or supervised layer (tf2/model.py:228-280)."""

    def __init__(self, num_classes, seed=0, **kwargs):
        e = get_engine()
        self.vs = VarStore()
        self.resnet_model = resnet.resnet(
            resnet_depth=FLAGS.resnet_depth, width_multiplier=FLAGS.width_multiplier,
            cifar_stem=FLAGS.image_size <= 32, vs=self.vs)
        self._projection_head = ProjectionHead(self.vs, self.resnet_model.cout)
        if FLAGS.train_mode == 'finetune' or FLAGS.lineareval_while_pretraining:
            self.supervised_head = SupervisedHead(num_classes, self.vs, self.resnet_model.cout)
        self.vs.materialize(e.device, seed)
        self._blur_draws = None

    @property
    def trainable_variables(self):
        return self.vs.trainable

    trainable_weights = trainable_variables

    @property
    def variables(self):
        return self.vs.trainable + self.vs.moving

    def set_blur_draws(self, sigma, selector):
        """Injects the `tf.random` draws of `batch_random_blur` (tf2/data_util.py:407,425):
        sigma [T] floats, selector [T][B] in {0,1}.  None -> drawn on device."""
        e = get_engine()       # on the device now: no host-to-device copy inside the step (CUDA-graph capture)
        if sigma is None:
            self._blur_draws = None
            return
        sigma = torch.as_tensor(sigma, dtype=torch.float32).to(e.device)
        selector = torch.as_tensor(selector).to(torch.uint8).to(e.device)
        self._blur_draws = (sigma, selector)

    def __call__(self, inputs, training, endpoints=None):
        e = get_engine()
        if training and FLAGS.train_mode == 'pretrain':
            if FLAGS.fine_tune_after_block > -1:
                raise ValueError('Does not support layer freezing during pretraining,'
                                 'should set fine_tune_after_block<=-1 for safety.')
        if inputs.dim() != 4 or inputs.shape[3] is None:
            raise ValueError('The input channels dimension must be statically known '
                             f'(got input shape {tuple(inputs.shape)})')
        B, H, W, C6 = inputs.shape
        num_transforms = C6 // 3
        use_blur = bool(FLAGS.use_blur and training and FLAGS.train_mode == 'pretrain')
        # split channels into views, batch_random_blur, concat on batch (view-major),
        # cast to the activation dtype and pad 3 -> 4 channels: one fused prep pass.
        features = data_util.prepare_views(inputs, num_transforms, use_blur, FLAGS.image_size,
                                           draws=self._blur_draws)
        e.pack_all()         # bf16 operands of every conv / dense layer from the fp32 masters: one launch
        try:
            hiddens = self.resnet_model(features, training=training, endpoints=endpoints)
            projection_head_outputs, supervised_head_inputs = self._projection_head(hiddens, training)
            supervised_head_outputs = None
            if FLAGS.train_mode == 'finetune':
                supervised_head_outputs = self.supervised_head(supervised_head_inputs, training)
                projection_head_outputs = None                          # tf2/model.py:267-270
            elif FLAGS.train_mode == 'pretrain' and FLAGS.lineareval_while_pretraining:
                # stop_gradient: nothing flows back from the supervised head (tf2/model.py:272-278)
                supervised_head_outputs = self.supervised_head(supervised_head_inputs, training)
        finally:
            e.pack_done()
        return projection_head_outputs, supervised_head_outputs

    def backward(self, d_projection_head_outputs, d_supervised_head_outputs=None):
        """Explicit `tape.gradient` (tf2/run.py:621): fills `.grad` of every trainable variable."""
        self.backward_bottom(self.backward_top(d_projection_head_outputs, d_supervised_head_outputs, 0), 0)

    def backward_top(self, d_projection_head_outputs, d_supervised_head_outputs=None, split=0):
        """Heads + block groups [split, 4): after it the gradients of every variable from the first one of block
        group `split`+1 to the end of the flat buffer are final (see `grad_split_offset`)."""
        d_sup_in = None
        if d_supervised_head_outputs is not None:
            d_sup_in = self.supervised_head.backward(d_supervised_head_outputs)
        if FLAGS.train_mode == 'finetune':
            # the loss sees hiddens_list[ft_proj_selector] only: backward through the projection layers below it
            sel = FLAGS.ft_proj_selector % (FLAGS.num_proj_layers + 1)
            e = get_engine()
            if d_sup_in.dtype != (torch.float32 if sel == FLAGS.num_proj_layers else e.act_dtype):
                c = e.empty(d_sup_in.shape, torch.float32 if sel == FLAGS.num_proj_layers else e.act_dtype)
                lib.cast(d_sup_in, e.code(d_sup_in.dtype), c, e.code(c.dtype), d_sup_in.numel(), stream_ptr())
                d_sup_in = c
            d_hiddens = self._projection_head.backward(d_sup_in, upto=sel)
        else:
            d_hiddens = self._projection_head.backward(d_projection_head_outputs)
        return self.resnet_model.backward_top(d_hiddens, split)

    def backward_bottom(self, state, split=0):
        self.resnet_model.backward_bottom(state, split)

    def grad_split_offset(self, split):
        """Element offset in the flat gradient buffer of the first variable of block group `split`+1: everything
        from there on (later groups, projection head, supervised head) is produced by `backward_top`."""
        tag = '/block_group%d/' % (split + 1)
        for v in self.vs.trainable:
            if tag in v.name:
                return (v.grad.data_ptr() - self.vs.flat_grad.data_ptr()) // 4
        return None
