"""SimCLRv2 distillation: a frozen teacher whose temperature-softened predictions train the student.

The third stage of SimCLRv2 (pretrain, fine-tune on a few labels, distil into a student on unlabelled images),
defined by the distillation colab's `add_kd_loss`.  The loss is `objective.add_distillation_loss`
(`simclr_distill_xent`); this module holds the teacher:

- `flag_scope(**values)`: layers read the process-global FLAGS when they are built and when they are called, so the
  teacher's construction and every teacher call run with the teacher's flag values, restored afterwards.
- `Teacher`: a `model.Model` built with `train_mode='finetune'` and the teacher's architecture, every variable a
  constant (no gradient buffer, no optimizer state), loaded strictly from a checkpoint and called in inference mode
  (BatchNorm on the moving statistics, nothing saved for a backward pass) on the existing forward kernels.
"""
import contextlib
import os

import numpy as np
import torch
from absl import logging

from .flags_def import FLAGS
from . import checkpoint as ckpt_lib
from . import tf_checkpoint

# teacher architecture flag -> the flag that overrides it (None: the student's value)
TEACHER_FLAGS = {
    'resnet_depth': 'b200_teacher_resnet_depth',
    'width_multiplier': 'b200_teacher_width_multiplier',
    'sk_ratio': 'b200_teacher_sk_ratio',
    'se_ratio': 'b200_teacher_se_ratio',
    'ft_proj_selector': 'b200_teacher_ft_proj_selector',
}


def distilling():
    """True when the training loss is distillation; raises for a teacher with `train_mode=pretrain`."""
    if not FLAGS.b200_distill_teacher:
        return False
    if FLAGS.train_mode != 'finetune':
        raise ValueError('--b200_distill_teacher needs --train_mode=finetune (got %r): distillation trains the '
                         'supervised head of the student' % FLAGS.train_mode)
    if not FLAGS.b200_distill_temperature > 0:
        raise ValueError('--b200_distill_temperature must be positive (got %r)' % FLAGS.b200_distill_temperature)
    return True


@contextlib.contextmanager
def flag_scope(**values):
    """Sets FLAGS.<name> = value for the body and restores every previous value afterwards, also on an exception.
    The flag objects' values are assigned directly, so `using_default_value` and `present` stay as they were."""
    saved = {k: FLAGS[k].value for k in values}
    try:
        for k, v in values.items():
            FLAGS[k].value = v
        yield
    finally:
        for k, v in saved.items():
            FLAGS[k].value = v


def teacher_flag_values():
    """The flag values the teacher is built and called with: finetune mode, no frozen block groups, and the
    teacher architecture flags (each defaulting to the student's value)."""
    vals = {'train_mode': 'finetune', 'fine_tune_after_block': -1}
    for name, override in TEACHER_FLAGS.items():
        v = getattr(FLAGS, override)
        vals[name] = getattr(FLAGS, name) if v is None else v
    return vals


def resolve_checkpoint(path):
    """A ckpt-N.npz, a TensorFlow checkpoint prefix, or a directory (its latest checkpoint, the rule of
    `CheckpointManager.latest_checkpoint`)."""
    if path and os.path.isdir(path):
        latest = ckpt_lib.CheckpointManager(None, None, path).latest_checkpoint
        if latest is None:
            raise FileNotFoundError('no checkpoint in teacher directory %s' % path)
        return latest
    if tf_checkpoint.is_tf_checkpoint(path) or (path and os.path.isfile(path)):
        return path
    raise FileNotFoundError('teacher checkpoint %r not found (a ckpt-N.npz, a TensorFlow checkpoint prefix or a '
                            'directory)' % path)


def checkpoint_shapes(path):
    """{variable name: shape} of the model variables stored in a checkpoint (names as `CheckpointManager.restore`
    joins them: own checkpoints under 'model/', TensorFlow ones on the object graph's full_name)."""
    if tf_checkpoint.is_tf_checkpoint(path):
        reader = tf_checkpoint.TensorBundleReader(path)
        graph = reader.object_graph()
        if graph:
            pairs = [(full, ckey) for ckey, full, name in graph if name == 'VARIABLE_VALUE' and ckey in reader.entries and full]
        else:
            pairs = [(k, k) for k, e in reader.entries.items() if e.dtype != tf_checkpoint.DT_STRING]
        out = {}
        for full, ckey in pairs:
            out.setdefault(full, tuple(reader.entries[ckey].shape))
        return out
    with np.load(path) as data:
        return {k[6:]: tuple(data[k].shape) for k in data.files if k.startswith('model/')}


def checkpoint_num_classes(path):
    """Classes of the supervised head stored in a checkpoint (the second dimension of its dense kernel)."""
    for name, shape in checkpoint_shapes(path).items():
        base = name[:-2] if name.endswith(':0') else name
        if base.startswith('head_supervised/') and base.endswith('/kernel') and len(shape) == 2:
            return int(shape[1])
    raise ValueError('checkpoint %s has no supervised head (head_supervised/.../kernel): a distillation teacher '
                     'must be a fine-tuned model' % path)


def missing_variables(variables, shapes):
    """Names of `variables` that `shapes` ({name: shape} of a checkpoint) does not hold with the right shape."""
    missing = []
    for v in variables:
        shape = shapes.get(v.name)
        if shape is None and v.name.endswith(':0'):
            shape = shapes.get(v.name[:-2])
        if shape is None or tuple(shape) != tuple(v.shape):
            missing.append(v.name if shape is None else '%s (shape %s in the checkpoint, %s in the model)'
                           % (v.name, tuple(shape), tuple(v.shape)))
    return missing


class Teacher:
    """The frozen teacher.  `Teacher(path)` builds it with the teacher's flag values, its class count taken from the
    checkpoint, and loads every variable from `path` -- trainable ones, moving means and moving variances; a
    variable the checkpoint lacks (or holds with another shape) is an error."""

    def __init__(self, path=None, num_classes=None, seed=0, fold_bn=None):
        """`fold_bn` (None: --b200_fold_bn): run the teacher's conv + BatchNorm pairs folded, each one launch on
        weights folded once, on the first forward."""
        self.flag_values = teacher_flag_values()
        self.flag_values['b200_fold_bn'] = FLAGS.b200_fold_bn if fold_bn is None else bool(fold_bn)
        if self.flag_values['b200_fold_bn']:
            from .engine import get_engine
            get_engine().check_fold_bn()
        self.path = resolve_checkpoint(path) if path is not None else None
        if num_classes is None:
            if self.path is None:
                raise ValueError('Teacher needs a checkpoint or num_classes')
            num_classes = checkpoint_num_classes(self.path)
        self.num_classes = num_classes
        from . import model as model_lib
        with flag_scope(**self.flag_values):
            self.model = model_lib.Model(num_classes, seed=seed, constant=True)
        self._called = False
        if self.path is not None:
            self.load(self.path)

    @property
    def variables(self):
        return self.model.variables

    def load(self, path):
        """Strict restore: every teacher variable must be in the checkpoint with the right shape."""
        if self._called:
            raise RuntimeError('teacher weights are constants: load them before the first forward')
        path = resolve_checkpoint(path)
        missing = missing_variables(self.model.variables, checkpoint_shapes(path))
        if missing:
            raise ValueError('teacher checkpoint %s does not match the teacher architecture %s: %d of %d variables '
                             'missing or of another shape: %s' % (path, self.flag_values, len(missing),
                                                                  len(self.model.variables), ', '.join(missing[:20]) +
                                                                  (' ...' if len(missing) > 20 else '')))
        ckpt_lib.CheckpointManager(self.model, None, None).restore(path, weights_only=True)
        logging.info('Distillation teacher: %d variables restored from %s (%s)', len(self.model.variables), path,
                     self.flag_values)

    def __call__(self, features):
        """Teacher logits [B, classes] fp32 on the device: inference-mode forward, nothing saved."""
        self._called = True
        with flag_scope(**self.flag_values):
            _, logits = self.model(features, training=False)
        return logits
