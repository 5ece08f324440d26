"""SimCLRv2 distillation without a GPU: the oracle's `add_kd_loss` against an independent fp64 formula and closed
forms, the distillation flags, the teacher's flag scope, and the argument errors of `simclr_distill_xent`."""
import pytest
import torch


@pytest.fixture
def dflags(flags):
    """`flags` plus the distillation flags, restored after the test."""
    F = flags.FLAGS
    names = ['b200_distill_teacher', 'b200_distill_temperature', 'b200_teacher_resnet_depth',
             'b200_teacher_width_multiplier', 'b200_teacher_sk_ratio', 'b200_teacher_se_ratio',
             'b200_teacher_ft_proj_selector', 'mode']
    saved = {k: getattr(F, k) for k in names}
    yield flags
    for k, v in saved.items():
        setattr(F, k, v)


def _fp64_kd(s, t, T):
    s, t = s.double(), t.double()
    p = torch.softmax(t / T, -1)
    return T * T * (-(p * torch.log_softmax(s / T, -1)).sum(1)).mean()


@pytest.mark.parametrize('T', [0.1, 1.0, 4.0])
@pytest.mark.parametrize('B,C', [(1, 10), (7, 100), (33, 1001)])
def test_oracle_kd_loss_against_fp64_and_its_gradient(T, B, C):
    from oracle import distill as OD
    g = torch.Generator().manual_seed(B * 1000 + C)
    s = (torch.randn(B, C, generator=g, dtype=torch.float64) * 3).requires_grad_(True)
    t = torch.randn(B, C, generator=g, dtype=torch.float64) * 3
    loss = OD.add_kd_loss(s, t, T)
    ref = _fp64_kd(s.detach(), t, T)
    assert abs(loss.item() - ref.item()) <= 1e-12 * abs(ref.item())
    (gs,) = torch.autograd.grad(loss, s)
    q, p = torch.softmax(s.detach() / T, -1), torch.softmax(t / T, -1)
    assert torch.allclose(gs, (T / B) * (q - p), rtol=1e-10, atol=1e-14)
    # no gradient reaches the teacher
    assert not OD.add_kd_loss(s.detach(), t.clone().requires_grad_(True), T).requires_grad


@pytest.mark.parametrize('T', [0.5, 1.0, 3.0])
def test_kd_loss_closed_forms(T):
    from oracle import distill as OD
    g = torch.Generator().manual_seed(7)
    s = (torch.randn(5, 50, generator=g, dtype=torch.float64) * 2).requires_grad_(True)
    # identical logits: the loss is T^2 H(p) and the gradient is zero
    loss = OD.add_kd_loss(s, s.detach().clone(), T)
    p = torch.softmax(s.detach() / T, -1)
    H = (-(p * torch.log(p)).sum(1)).mean()
    assert abs(loss.item() - T * T * H.item()) <= 1e-12 * T * T * H.item()
    (gs,) = torch.autograd.grad(loss, s)
    assert float(gs.abs().max()) < 1e-15
    # a uniform teacher: l_r = logsumexp(s/T) - mean(s/T)
    loss_u = OD.add_kd_loss(s.detach(), torch.zeros(5, 50, dtype=torch.float64), T)
    ref = (torch.logsumexp(s.detach() / T, -1) - (s.detach() / T).mean(1)).mean() * T * T
    assert abs(loss_u.item() - ref.item()) <= 1e-12 * abs(ref.item())


def test_distillation_flags(dflags):
    from simclr_b200 import distill
    F = dflags.FLAGS
    assert len(dflags.REFERENCE_FLAG_NAMES) == 48
    assert not any(k.startswith('b200_') for k in dflags.REFERENCE_FLAG_NAMES)
    defaults = {k: F[k].default for k in ('b200_distill_teacher', 'b200_distill_temperature', 'b200_teacher_resnet_depth',
                                          'b200_teacher_width_multiplier', 'b200_teacher_sk_ratio',
                                          'b200_teacher_se_ratio', 'b200_teacher_ft_proj_selector')}
    assert defaults == dict(b200_distill_teacher=None, b200_distill_temperature=1.0, b200_teacher_resnet_depth=None,
                            b200_teacher_width_multiplier=None, b200_teacher_sk_ratio=None,
                            b200_teacher_se_ratio=None, b200_teacher_ft_proj_selector=None)
    dflags.set_flags(b200_distill_teacher=None, train_mode='pretrain')
    assert distill.distilling() is False
    dflags.set_flags(b200_distill_teacher='/nonexistent/teacher', train_mode='pretrain')
    with pytest.raises(ValueError):
        distill.distilling()
    dflags.set_flags(train_mode='finetune')
    assert distill.distilling() is True
    dflags.set_flags(b200_distill_temperature=0.0)
    with pytest.raises(ValueError):
        distill.distilling()
    # teacher architecture: None means the student's value
    dflags.set_flags(resnet_depth=50, width_multiplier=1, sk_ratio=0.0, se_ratio=0.0, ft_proj_selector=0,
                     b200_teacher_resnet_depth=152, b200_teacher_width_multiplier=None, b200_teacher_sk_ratio=0.0625,
                     b200_teacher_se_ratio=None, b200_teacher_ft_proj_selector=1)
    assert distill.teacher_flag_values() == dict(train_mode='finetune', fine_tune_after_block=-1, resnet_depth=152,
                                                 width_multiplier=1, sk_ratio=0.0625, se_ratio=0.0, ft_proj_selector=1)


def test_flag_scope_restores_every_value(dflags):
    from simclr_b200 import distill
    F = dflags.FLAGS
    dflags.set_flags(train_mode='pretrain', resnet_depth=50, ft_proj_selector=0)

    def snapshot():
        return {k: (F[k].value, F[k].present, F[k].using_default_value) for k in F}
    before = snapshot()
    with distill.flag_scope(train_mode='finetune', resnet_depth=18, sk_ratio=0.0625, ft_proj_selector=2):
        assert (F.train_mode, F.resnet_depth, F.sk_ratio, F.ft_proj_selector) == ('finetune', 18, 0.0625, 2)
    assert snapshot() == before
    with pytest.raises(KeyError):
        with distill.flag_scope(train_mode='finetune', width_multiplier=3):
            assert F.width_multiplier == 3
            raise KeyError('inside the scope')
    assert snapshot() == before
    with distill.flag_scope(resnet_depth=34):
        with distill.flag_scope(resnet_depth=101):
            assert F.resnet_depth == 101
        assert F.resnet_depth == 34
    assert snapshot() == before


def test_teacher_checkpoint_inspection(tmp_path):
    """Class count and variable shapes read from an own .npz and from a TensorFlow bundle; a missing or mis-shaped
    variable is named."""
    import numpy as np
    from simclr_b200 import distill, tf_checkpoint as TC
    from simclr_b200.engine import Variable
    arrays = {'model/resnet/conv2d/kernel:0': np.zeros((3, 3, 3, 8), np.float32),
              'model/resnet/bn/moving_variance:0': np.ones((8,), np.float32),
              'model/head_supervised/linear_layer/dense/kernel:0': np.zeros((8, 17), np.float32),
              'model/head_supervised/linear_layer/dense/bias:0': np.zeros((17,), np.float32)}
    npz = str(tmp_path / 'ckpt-3.npz')
    np.savez(npz, global_step=np.asarray(3), **arrays)
    assert distill.resolve_checkpoint(str(tmp_path)) == npz
    assert distill.checkpoint_num_classes(npz) == 17
    tensors = {'v%d%s' % (i, TC.VARIABLE_SUFFIX): a for i, a in enumerate(arrays.values())}
    names = {'v%d%s' % (i, TC.VARIABLE_SUFFIX): k[6:-2] for i, k in enumerate(arrays)}
    prefix = str(tmp_path / 'tf' / 'ckpt-9')
    TC.write_bundle(prefix, tensors, names)
    assert distill.resolve_checkpoint(str(tmp_path / 'tf')) == prefix
    assert distill.checkpoint_num_classes(prefix) == 17
    want = [Variable('resnet/conv2d/kernel:0', (3, 3, 3, 8), 'zeros'),
            Variable('resnet/bn/moving_variance:0', (8,), 'ones'),
            Variable('resnet/bn/moving_mean:0', (8,), 'zeros'),
            Variable('head_supervised/linear_layer/dense/kernel:0', (8, 10), 'zeros')]
    for path in (npz, prefix):
        missing = distill.missing_variables(want, distill.checkpoint_shapes(path))
        assert len(missing) == 2 and missing[0] == 'resnet/bn/moving_mean:0' and 'dense/kernel:0 (shape (8, 17)' in missing[1]
    with pytest.raises(FileNotFoundError):
        distill.resolve_checkpoint(str(tmp_path / 'nothing'))


def test_distill_xent_argument_errors_are_reported_without_a_gpu():
    from simclr_b200._lib import lib, SimclrError
    cases = [((None, 1, 4, 10, 1.0, 0.0, 1, None, None), 'null pointer'),
             ((1, None, 4, 10, 1.0, 0.0, 1, None, None), 'null pointer'),
             ((1, 1, 4, 10, 1.0, 0.0, None, 1, None), 'null pointer'),
             ((1, 1, 0, 10, 1.0, 0.0, 1, None, None), 'bad shape'),
             ((1, 1, 4, 0, 1.0, 0.0, 1, None, None), 'bad shape'),
             ((1, 1, -2, 10, 1.0, 0.0, 1, None, None), 'bad shape'),
             ((1, 1, 4, 10, 0.0, 0.0, 1, None, None), 'temperature'),
             ((1, 1, 4, 10, -1.0, 0.0, 1, None, None), 'temperature'),
             ((1, 1, 4, 10, float('nan'), 0.0, 1, None, None), 'temperature')]
    for args, msg in cases:
        with pytest.raises(SimclrError) as ei:
            lib.distill_xent(*args)
        assert 'status -1' in str(ei.value) and msg in str(ei.value), (args, str(ei.value))
    assert 'simclr_distill_xent' in lib.declarations
