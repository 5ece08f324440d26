"""SimCLRv2 distillation on the H100: `simclr_distill_xent` against fp64, the distillation step against the oracle,
same bits and CUDA-graph replay on the bf16 tensor-core path, strict teacher loading, and the driver."""
import collections
import glob
import os

import numpy as np
import pytest
import torch

from util import rel_err, cfg_from_flags, structured_batch

pytestmark = pytest.mark.gpu

DISTILL_FLAGS = ['b200_distill_teacher', 'b200_distill_temperature', 'b200_teacher_resnet_depth',
                 'b200_teacher_width_multiplier', 'b200_teacher_sk_ratio', 'b200_teacher_se_ratio',
                 'b200_teacher_ft_proj_selector', 'b200_num_classes', 'b200_num_examples', 'b200_num_eval_examples',
                 'data_dir', 'dataset', 'checkpoint']


@pytest.fixture
def dflags(flags):
    """`flags` plus the distillation / driver flags, restored after the test."""
    F = flags.FLAGS
    saved = {k: getattr(F, k) for k in DISTILL_FLAGS}
    yield flags
    for k, v in saved.items():
        setattr(F, k, v)


# ----------------------------------------------------------------------------------------------------------------
# 1. the kernel against fp64
# ----------------------------------------------------------------------------------------------------------------
def _ref64(s, t, T):
    s, t = s.double(), t.double()
    p = torch.softmax(t / T, -1)
    logq = torch.log_softmax(s / T, -1)
    rows = -(p * logq).sum(1)
    agree = (s.argmax(1) == t.argmax(1)).sum().item()
    return T * T * rows.mean().item(), rows, agree, torch.exp(logq) - p


def _logits(rows, classes, scale, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    s = torch.randn(rows, classes, device='cuda', generator=g) * 3
    t = torch.randn(rows, classes, device='cuda', generator=g) * 3
    if scale:                                   # logits of +-1e4
        s = (torch.rand(rows, classes, device='cuda', generator=g) * 2 - 1) * 1e4
        t = (torch.rand(rows, classes, device='cuda', generator=g) * 2 - 1) * 1e4
    # tied maxima: every third row has its maximum twice (the student at a, b; the teacher at b, a or a, b)
    for r in range(0, rows, 3):
        a, b = (r * 7) % classes, (r * 13 + 1) % classes
        if a == b:
            continue
        ms, mt = float(s[r].max()) + 1, float(t[r].max()) + 1
        s[r, a] = s[r, b] = ms
        t[r, a] = mt
        if r % 2 == 0:
            t[r, b] = mt
    return s.contiguous(), t.contiguous()


@pytest.mark.parametrize('rows', [1, 7, 33, 512])
def test_distill_xent_against_fp64(rows):
    from simclr_b200._lib import lib, stream_ptr
    for classes in (10, 100, 1000, 1001, 21843):
        for T in (0.1, 1.0, 4.0):
            for scale in (False, True):
                s, t = _logits(rows, classes, scale, seed=rows * 100003 + classes * 7 + int(T * 10) + scale)
                loss64, rows64, agree64, dq = _ref64(s, t, T)
                gs = T / rows
                out = torch.full((2 + rows,), float('nan'), device='cuda')
                d = torch.full((rows, classes), float('nan'), device='cuda')
                lib.distill_xent(s, t, rows, classes, T, gs, out, d, stream_ptr())
                torch.cuda.synchronize()
                what = (rows, classes, T, scale)
                assert torch.isfinite(out).all() and torch.isfinite(d).all(), what
                assert abs(out[0].item() - loss64) <= 1e-5 * abs(loss64) + 1e-7 * T * T, (what, out[0].item(), loss64)
                assert out[1].item() == np.float32(agree64 / rows), (what, out[1].item(), agree64)
                assert ((out[2:].double() - rows64).abs() <= 1e-5 * rows64.abs() + 1e-7).all(), what
                ref = dq * gs
                bound = 1e-6 * ref.abs().max().item() + 2.0 ** -20 * T / rows
                err = (d.double() - ref).abs().max().item()
                assert err <= bound, (what, err, bound)
                # the same bits again, and without the gradient
                out2 = torch.full_like(out, float('nan')); d2 = torch.full_like(d, float('nan'))
                lib.distill_xent(s, t, rows, classes, T, gs, out2, d2, stream_ptr())
                out3 = torch.full_like(out, float('nan'))
                lib.distill_xent(s, t, rows, classes, T, 0.0, out3, None, stream_ptr())
                torch.cuda.synchronize()
                assert torch.equal(out, out2) and torch.equal(d, d2) and torch.equal(out, out3), what


def test_distill_xent_tie_breaking_and_graph_replay():
    from simclr_b200._lib import lib, stream_ptr
    s = torch.zeros(4, 6, device='cuda')
    t = torch.zeros(4, 6, device='cuda')
    s[0, [1, 4]] = 2.0; t[0, [1, 4]] = 2.0          # the same tie: lowest index 1 on both sides -> agree
    s[1, [1, 4]] = 2.0; t[1, 4] = 2.0               # student 1, teacher 4 -> disagree
    s[2, 5] = 1.0; t[2, 5] = 3.0                    # agree
    #  row 3: all equal -> index 0 on both sides -> agree
    out = torch.full((6,), float('nan'), device='cuda')
    lib.distill_xent(s, t, 4, 6, 1.0, 0.25, out, None, stream_ptr())
    torch.cuda.synchronize()
    assert out[1].item() == 0.75
    # a captured call replays to the eager call's bits
    s, t = _logits(33, 1001, False, seed=5)
    out_e = torch.empty(35, device='cuda'); d_e = torch.empty(33, 1001, device='cuda')
    lib.distill_xent(s, t, 33, 1001, 2.0, 2.0 / 33, out_e, d_e, stream_ptr())
    out_g = torch.full((35,), float('nan'), device='cuda'); d_g = torch.full((33, 1001), float('nan'), device='cuda')
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        with torch.cuda.graph(g):
            lib.distill_xent(s, t, 33, 1001, 2.0, 2.0 / 33, out_g, d_g, stream_ptr())
    torch.cuda.current_stream().wait_stream(side)
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out_g, out_e) and torch.equal(d_g, d_e)


def test_add_distillation_loss_wrapper():
    from simclr_b200 import engine, objective as obj
    engine.set_engine(engine.Engine(precision='bf16', conv_engine='tc'))
    s, t = _logits(16, 100, False, seed=9)
    loss, agree, d = obj.add_distillation_loss(s, t, 2.0, grad_scale=2.0 / 16)
    loss64, _, agree64, dq = _ref64(s, t, 2.0)
    assert abs(loss.item() - loss64) <= 1e-5 * loss64 and agree.item() == np.float32(agree64 / 16)
    assert (d.double() - dq * (2.0 / 16)).abs().max().item() <= 1e-6
    loss2, _, d2 = obj.add_distillation_loss(s, t, 2.0)
    assert d2 is None and torch.equal(loss2, loss)


# ----------------------------------------------------------------------------------------------------------------
# 2. the step against the oracle (fp32 storage)
# ----------------------------------------------------------------------------------------------------------------
def _warm(P, S_, seed):
    g = torch.Generator().manual_seed(seed)
    for k in P:
        if k.endswith('gamma:0'):
            P[k] = 0.5 + torch.rand(P[k].shape, generator=g)
        elif k.endswith('beta:0'):
            P[k] = torch.randn(P[k].shape, generator=g) * 0.1
    for k in S_:
        S_[k] = (0.5 + torch.rand(S_[k].shape, generator=g)) if 'variance' in k else torch.randn(S_[k].shape, generator=g) * 0.1


def _distill_setup(flags_def, optimizer, precision, conv_engine, B=16, S=64, num_classes=100):
    """Teacher R34 1x SK (ft_proj_selector 1) and student R18 1x (ft_proj_selector 0), both with warm states."""
    from simclr_b200 import engine, run, distill
    from oracle import model as OM
    flags_def.set_flags(resnet_depth=18, width_multiplier=1, sk_ratio=0.0, se_ratio=0.0, image_size=S,
                        train_batch_size=B, use_blur=False, weight_decay=1e-4, train_mode='finetune',
                        fine_tune_after_block=-1, ft_proj_selector=0, optimizer=optimizer,
                        lineareval_while_pretraining=False, b200_precision=precision, b200_conv_engine=conv_engine,
                        b200_distill_temperature=2.0, b200_teacher_resnet_depth=34, b200_teacher_sk_ratio=0.0625,
                        b200_teacher_ft_proj_selector=1, b200_teacher_width_multiplier=None,
                        b200_teacher_se_ratio=None)
    engine.set_engine(engine.Engine(precision=precision, conv_engine=conv_engine))
    before = {k: (flags_def.FLAGS[k].value, flags_def.FLAGS[k].using_default_value) for k in flags_def.FLAGS}
    teacher = distill.Teacher(None, num_classes=num_classes, seed=5)
    assert {k: (flags_def.FLAGS[k].value, flags_def.FLAGS[k].using_default_value) for k in flags_def.FLAGS} == before
    with distill.flag_scope(**teacher.flag_values):
        otm = OM.Model(cfg_from_flags(flags_def.FLAGS), num_classes)
    TP, TS = otm.init(5)
    _warm(TP, TS, 21)
    teacher.model.vs.load(TP); teacher.model.vs.load(TS)
    trainer = run.Trainer(num_examples=50000, seed=0, teacher=teacher)
    om = OM.Model(cfg_from_flags(flags_def.FLAGS), num_classes)
    P, S_ = om.init(0)
    _warm(P, S_, 11)
    trainer.model.vs.load(P); trainer.model.vs.load(S_)
    return trainer, teacher, om, otm, P, S_, TP, TS


@pytest.mark.parametrize('optimizer', ['lars', 'momentum'])
def test_distill_step_parity(dflags, optimizer):
    from oracle import distill as ODi, optimizers as OO, lars as OL
    trainer, teacher, om, otm, P, S_, TP, TS = _distill_setup(dflags, optimizer, 'fp32', 'simt')
    cfg, T = om.cfg, 2.0
    assert trainer.num_classes == 100 and not teacher.model.trainable_variables
    assert teacher.model.vs.flat_grad.numel() == 0
    assert set(v.name for v in teacher.variables) == set(TP) | set(TS)
    assert set(v.name for v in trainer.model.trainable_variables) == set(P)
    f6, lab = structured_batch(16, 64, num_classes=100, seed=2)
    f = f6[..., :3].contiguous()
    info = ODi.forward_backward(om, P, S_, [f], (otm, TP, TS), T)
    d64 = lambda D: collections.OrderedDict((k, v.double()) for k, v in D.items())
    i64 = ODi.forward_backward(om, d64(P), d64(S_), [f.double()], (otm, d64(TP), d64(TS)), T)
    intrinsic = {k: rel_err(info['grads'][k], i64['grads'][k]) for k in P if i64['grads'][k].norm() > 0}
    lr = 0.05
    trainer.optimizer.learning_rate = lr
    t_before = teacher.model.vs.flat_moving.clone()
    loss = trainer.single_step(f.cuda(), lab.cuda())
    torch.cuda.synchronize()
    m = trainer.metrics
    assert rel_err(m['teacher_logits'], i64['teacher_out'][0]) < 1e-4
    assert abs(loss.item() - info['loss'].item()) < 1e-4 * abs(info['loss'].item())
    assert abs(m['distill_loss'].item() - info['kd_loss'][0].item()) < 1e-4 * abs(info['kd_loss'][0].item())
    assert m['distill_acc'].item() == info['agreement'][0].item()
    for v in trainer.model.trainable_variables:
        ref = info['grads'][v.name]
        if ref.norm() == 0:
            assert float(v.grad.abs().max()) < 1e-7 * (1 + float(ref.abs().max())), v.name
        else:
            err = rel_err(v.grad, i64['grads'][v.name])
            assert err < max(2e-3, 5 * intrinsic[v.name]), (v.name, err, intrinsic[v.name])
    # the optimizer's rule applied to the gradients the CUDA step produced gives the CUDA step's weights
    Pt = collections.OrderedDict((k, P[k].double()) for k in P)
    Gt = collections.OrderedDict((v.name, v.grad.detach().double().cpu()) for v in trainer.model.trainable_variables)
    Z = collections.OrderedDict((k, torch.zeros_like(v)) for k, v in Pt.items())
    if optimizer == 'momentum':
        Pn, _ = OO.sgd_nesterov_apply(Pt, Gt, Z, lr, cfg.momentum, True)
    else:
        Pn, _ = OL.lars_apply(Pt, Gt, Z, lr, momentum=cfg.momentum, weight_decay=cfg.weight_decay,
                              exclude_from_weight_decay=OL.LARS_EXCLUDE)
    for v in trainer.model.trainable_variables:
        upd_ref = Pn[v.name] - Pt[v.name]
        if upd_ref.norm() > 0:
            err = (v.value.double().cpu() - Pn[v.name]).norm()
            assert err < 1e-4 * upd_ref.norm() + 2.0 ** -24 * Pt[v.name].norm(), (v.name, float(err), float(upd_ref.norm()))
    assert torch.equal(teacher.model.vs.flat_moving, t_before), 'a teacher variable changed'
    for v in trainer.model.vs.moving:
        assert rel_err(v.value, info['S_new'][v.name]) < 1e-4, v.name


# ----------------------------------------------------------------------------------------------------------------
# 3. the bf16 tensor-core path: same bits, graph replay
# ----------------------------------------------------------------------------------------------------------------
def _state(trainer):
    opt = trainer.optimizer
    return [trainer.model.vs.flat_value.clone(), trainer.model.vs.flat_grad.clone(),
            trainer.model.vs.flat_moving.clone(), opt._flat_v.clone()]


def test_distill_step_same_bits_bf16(dflags):
    from simclr_b200 import run
    f6, lab = structured_batch(16, 64, num_classes=96, seed=3)
    f, lab = f6[..., :3].contiguous().cuda(), lab.cuda()
    trainer, teacher, *_ = _distill_setup(dflags, 'lars', 'bf16', 'tc', num_classes=96)
    assert teacher.model.vs.flat_grad.numel() == 0 and not teacher.model.trainable_variables
    t_before = teacher.model.vs.flat_moving.clone()
    # a second trainer from the same state, sharing the constant teacher
    tr2 = run.Trainer(num_examples=50000, seed=0, teacher=teacher)
    tr2.model.vs.flat_value.copy_(trainer.model.vs.flat_value)
    tr2.model.vs.flat_moving.copy_(trainer.model.vs.flat_moving)
    runs = []
    for tr in (trainer, tr2):
        tr.optimizer.learning_rate = 0.05
        per = []
        for _ in range(2):
            loss = tr.single_step(f, lab)
            per.append([loss.clone(), tr.metrics['distill_acc'].clone(), tr.metrics['teacher_logits'].clone()] + _state(tr))
        torch.cuda.synchronize()
        runs.append(per)
    for a, b in zip(*runs):
        for x, y in zip(a, b):
            assert torch.equal(x, y)
    assert torch.isfinite(runs[1][-1][0]).all() and torch.isfinite(runs[1][-1][3]).all()
    assert torch.equal(teacher.model.vs.flat_moving, t_before)


def test_distill_graph_replay_equals_eager(dflags):
    from simclr_b200 import flags_def
    f6, lab = structured_batch(16, 64, num_classes=96, seed=4)
    f, lab = f6[..., :3].contiguous().cuda(), lab.cuda()
    results = []
    for use_graph in (False, True):
        flags_def.set_flags(warmup_epochs=0, train_steps=4, learning_rate=0.8)      # a learning rate that changes every step
        trainer, teacher, *_ = _distill_setup(dflags, 'lars', 'bf16', 'tc', num_classes=96)
        if use_graph:
            trainer.capture(f, lab, warmup=1, restore=True)
            assert trainer.optimizer.iterations == 0
            for _ in range(3):
                loss = trainer.replay()
        else:
            for _ in range(3):
                loss = trainer.single_step(f, lab)
        torch.cuda.synchronize()
        assert trainer.optimizer.iterations == 3
        results.append((trainer.model.vs.flat_value.clone(), trainer.model.vs.flat_moving.clone(), loss.clone(),
                        teacher.model.vs.flat_moving.clone()))
    for a, b in zip(*results):
        assert torch.equal(a, b)


# ----------------------------------------------------------------------------------------------------------------
# 4. teacher loading and the driver
# ----------------------------------------------------------------------------------------------------------------
def _driver_flags(flags_def, md, **kw):
    base = dict(resnet_depth=18, width_multiplier=1, sk_ratio=0.0, se_ratio=0.0, image_size=32, train_batch_size=8,
                eval_batch_size=8, eval_steps=2, checkpoint_steps=2, keep_checkpoint_max=5, model_dir=md,
                train_mode='finetune', fine_tune_after_block=-1, ft_proj_selector=0, lineareval_while_pretraining=False,
                use_blur=False, optimizer='lars', b200_precision='bf16', b200_conv_engine='tc', b200_num_classes=16,
                b200_num_examples=1000, b200_num_eval_examples=16, warmup_epochs=0, learning_rate=0.1,
                b200_distill_teacher=None, b200_distill_temperature=1.0, b200_teacher_resnet_depth=None,
                b200_teacher_width_multiplier=None, b200_teacher_sk_ratio=None, b200_teacher_se_ratio=None,
                b200_teacher_ft_proj_selector=None, data_dir=None, checkpoint=None)
    base.update(kw)
    flags_def.set_flags(**base)


def _tags(md):
    return b''.join(open(p, 'rb').read() for p in glob.glob(os.path.join(md, 'events.out.tfevents.*')))


def test_teacher_loading_is_strict(dflags, tmp_path):
    from simclr_b200 import engine, run, distill, tf_checkpoint as TC
    tdir = str(tmp_path / 'teacher')
    _driver_flags(dflags, tdir, train_steps=2, mode='train', ft_proj_selector=1)
    engine.set_engine(None)
    run.main(['run'])
    ck = os.path.join(tdir, 'ckpt-2.npz')
    assert os.path.exists(ck)
    _driver_flags(dflags, None, b200_teacher_ft_proj_selector=1)
    engine.set_engine(engine.Engine())
    teacher = distill.Teacher(tdir)
    assert teacher.num_classes == 16 and not teacher.model.trainable_variables
    assert teacher.model.vs.flat_grad.numel() == 0
    data = np.load(ck)
    for v in teacher.variables:
        assert np.array_equal(v.value.cpu().numpy(), data['model/' + v.name]), v.name
    # a missing moving variance is named
    bad = {k: data[k] for k in data.files}
    victim = [k for k in bad if k.endswith('moving_variance:0')][3]
    del bad[victim]
    np.savez(str(tmp_path / 'bad.npz'), **bad)
    with pytest.raises(ValueError) as ei:
        distill.Teacher(str(tmp_path / 'bad.npz'))
    assert victim[6:] in str(ei.value)
    # a TensorFlow bundle of the same weights
    tensors = {'v%d%s' % (i, TC.VARIABLE_SUFFIX): data[k] for i, k in enumerate(data.files) if k.startswith('model/')}
    names = {'v%d%s' % (i, TC.VARIABLE_SUFFIX): k[6:-2] for i, k in enumerate(data.files) if k.startswith('model/')}
    TC.write_bundle(str(tmp_path / 'tf' / 'ckpt-2'), tensors, names)
    tt = distill.Teacher(str(tmp_path / 'tf' / 'ckpt-2'))
    for a, b in zip(tt.variables, teacher.variables):
        assert torch.equal(a.value, b.value), a.name
    # architecture flags that do not match the checkpoint
    dflags.set_flags(b200_teacher_resnet_depth=34)
    with pytest.raises(ValueError):
        distill.Teacher(tdir)
    dflags.set_flags(b200_teacher_resnet_depth=None, b200_teacher_width_multiplier=2)
    with pytest.raises(ValueError):
        distill.Teacher(tdir)


def test_distill_driver(dflags, tmp_path):
    """Fine-tune a small teacher, distil it into a student (synthetic data, an ArrayBuilder .npz, a TensorFlow-bundle
    teacher), evaluate the student, resume."""
    from simclr_b200 import engine, run, tf_checkpoint as TC
    tdir = str(tmp_path / 'teacher')
    _driver_flags(dflags, tdir, train_steps=2, mode='train')
    engine.set_engine(None)
    run.main(['run'])
    assert os.path.exists(os.path.join(tdir, 'ckpt-2.npz'))
    teacher_names = set(np.load(os.path.join(tdir, 'ckpt-2.npz')).files)
    # synthetic data
    md = str(tmp_path / 'student')
    _driver_flags(dflags, md, train_steps=3, mode='train_then_eval', b200_distill_teacher=tdir,
                  b200_distill_temperature=2.0, b200_num_classes=1000)         # the class count comes from the teacher
    engine.set_engine(None)
    result = run.main(['run'])
    assert result is not None and result['global_step'] == 3
    blob = _tags(md)
    for tag in (b'train/distill_loss', b'train/distill_acc', b'train/supervised_acc', b'train/weight_decay',
                b'train/total_loss', b'eval/label_top_1_accuracy'):
        assert tag in blob, tag
    assert b'train/supervised_loss' not in blob
    ck = np.load(os.path.join(md, 'ckpt-3.npz'))
    assert {k for k in ck.files if k.startswith('model/')} == {k for k in teacher_names if k.startswith('model/')}
    assert int(ck['global_step']) == 3
    # resume: the student continues from its step, the teacher comes back from the flag
    _driver_flags(dflags, md, train_steps=4, mode='train', b200_distill_teacher=tdir, b200_distill_temperature=2.0)
    engine.set_engine(None)
    run.main(['run'])
    assert int(np.load(os.path.join(md, 'ckpt-4.npz'))['global_step']) == 4
    # an ArrayBuilder .npz dataset and a TensorFlow-bundle teacher
    rs = np.random.RandomState(0)
    npz = str(tmp_path / 'data.npz')
    np.savez(npz, train_images=rs.randint(0, 256, (24, 32, 32, 3), dtype=np.uint8), train_labels=np.arange(24) % 16,
             validation_images=rs.randint(0, 256, (16, 32, 32, 3), dtype=np.uint8), validation_labels=np.arange(16) % 16,
             num_classes=np.asarray(16))
    data = np.load(os.path.join(tdir, 'ckpt-2.npz'))
    keys = [k for k in data.files if k.startswith('model/')]
    TC.write_bundle(str(tmp_path / 'tf' / 'ckpt-2'), {'v%d%s' % (i, TC.VARIABLE_SUFFIX): data[k] for i, k in enumerate(keys)},
                    {'v%d%s' % (i, TC.VARIABLE_SUFFIX): k[6:-2] for i, k in enumerate(keys)})
    md2 = str(tmp_path / 'student2')
    _driver_flags(dflags, md2, train_steps=3, mode='train_then_eval', data_dir=npz,
                  b200_distill_teacher=str(tmp_path / 'tf' / 'ckpt-2'))
    engine.set_engine(None)
    result = run.main(['run'])
    assert result is not None and result['global_step'] == 3
    assert b'train/distill_acc' in _tags(md2)
    # a dataset with another class count than the teacher's head
    np.savez(str(tmp_path / 'data7.npz'), train_images=rs.randint(0, 256, (24, 32, 32, 3), dtype=np.uint8),
             train_labels=np.arange(24) % 7, validation_images=rs.randint(0, 256, (8, 32, 32, 3), dtype=np.uint8),
             validation_labels=np.arange(8) % 7, num_classes=np.asarray(7))
    _driver_flags(dflags, str(tmp_path / 'student3'), train_steps=1, mode='train', data_dir=str(tmp_path / 'data7.npz'),
                  b200_distill_teacher=tdir)
    engine.set_engine(None)
    with pytest.raises(ValueError):
        run.main(['run'])
    # a teacher with pretraining is refused
    _driver_flags(dflags, str(tmp_path / 'student4'), train_steps=1, mode='train', train_mode='pretrain',
                  b200_distill_teacher=tdir)
    engine.set_engine(None)
    with pytest.raises(ValueError):
        run.main(['run'])
