"""BatchNorm-folded inference forward (--b200_fold_bn) on the H100: the fold kernel bit for bit, every folded launch
of the evaluation forward against fp64, the model end to end against the oracles, linear evaluation and partially
frozen fine-tuning, and the folded distillation teacher (eager and captured)."""
import collections

import pytest
import torch
import torch.nn.functional as F

from util import rel_err, cfg_from_flags, structured_batch

pytestmark = pytest.mark.gpu

FOLD_FLAGS = ['b200_fold_bn', 'b200_distill_teacher', 'b200_distill_temperature', 'b200_teacher_resnet_depth',
              'b200_teacher_width_multiplier', 'b200_teacher_sk_ratio', 'b200_teacher_se_ratio',
              'b200_teacher_ft_proj_selector', 'warmup_epochs', 'train_steps', 'learning_rate']


@pytest.fixture
def fflags(flags):
    """`flags` plus the folding and distillation flags, restored after the test."""
    F_ = flags.FLAGS
    saved = {k: getattr(F_, k) for k in FOLD_FLAGS}
    yield flags
    for k, v in saved.items():
        setattr(F_, k, v)


def _setup(flags_def, fold, B=2, S=64, depth=50, num_classes=100, **kw):
    from simclr_b200 import engine, run
    vals = dict(resnet_depth=depth, image_size=S, train_batch_size=B, use_blur=False, width_multiplier=1, sk_ratio=0.0,
                se_ratio=0.0, b200_precision='bf16', b200_conv_engine='tc', b200_fold_bn=fold)
    vals.update(kw)
    flags_def.set_flags(**vals)
    engine.set_engine(engine.Engine(precision='bf16', conv_engine='tc'))
    return run.Trainer(num_classes=num_classes, num_examples=50000, seed=0)


def _random_moving(S_, seed):
    g = torch.Generator().manual_seed(seed)
    for k in S_:
        S_[k] = (0.5 + torch.rand(S_[k].shape, generator=g)) if 'variance' in k else torch.randn(S_[k].shape, generator=g) * 0.1


def _warm_params(P, seed):
    g = torch.Generator().manual_seed(seed)
    for k in P:
        if k.endswith('gamma:0'):
            P[k] = 0.5 + torch.rand(P[k].shape, generator=g)
        elif k.endswith('beta:0'):
            P[k] = torch.randn(P[k].shape, generator=g) * 0.1


# ----------------------------------------------------------------------------------------------------------------
# 1. the fold kernel, bit for bit
# ----------------------------------------------------------------------------------------------------------------
def _layout(w, R, S, Cin, Cs, Cout, Kp):
    """The packed K-major layout of an HWIO master in fp32 (simclr_pack_conv_weight), built with torch."""
    if Cs == 4:                                            # the stem: S+1 slots per filter row, slot 0 zero
        t = torch.zeros(Cout, R, S + 1, 4, dtype=torch.float32, device=w.device)
        t[:, :, 1:, :Cin] = w.permute(3, 0, 1, 2)
    else:
        t = w.permute(3, 0, 1, 2)
    t = t.reshape(Cout, -1)
    return F.pad(t, (0, Kp - t.shape[1]))


@pytest.mark.parametrize('arch', ['r50', 'r34_sk'])
def test_fold_kernel_bit_exact(fflags, arch):
    from simclr_b200 import engine
    kw = dict(depth=50) if arch == 'r50' else dict(depth=34, sk_ratio=0.0625)
    trainer = _setup(fflags, True, **kw)
    from oracle import model as OM
    om = OM.Model(cfg_from_flags(fflags.FLAGS), 100)
    P, S_ = om.init(0)
    _warm_params(P, 1)
    _random_moving(S_, 2)
    trainer.model.vs.load(P); trainer.model.vs.load(S_)
    f, _ = structured_batch(2, 64, seed=1)
    trainer.model(f.cuda(), training=False)
    trainer.model(f.cuda(), training=False)          # the second forward re-folds through the one-launch table
    torch.cuda.synchronize()
    e = engine.get_engine()
    ops = e._fold_ops
    assert e._fold_table is not None and len(ops) == e._fold_table[1]
    stems = 0
    for op in ops:
        scale, shift = op.fold_coef[0], op.fold_coef[1]
        ref = (_layout(op.kernel.value.view(op.R, op.S, op.cin, op.cout), op.R, op.S, op.cin, op.cs, op.cout,
                       op.wfold.shape[1]) * scale[:, None]).to(torch.bfloat16)
        assert torch.equal(op.wfold.view(torch.int16), ref.view(torch.int16)), (op.R, op.S, op.cin, op.cout)
        assert torch.equal(op.bias_f, shift)
        # the coefficients are the BatchNorm's inference coefficients
        bn = op.fold_bn_layer
        r = torch.rsqrt(bn.moving_variance.value + 1e-5)
        sc = r if bn.gamma is None else bn.gamma.value * r
        assert torch.equal(scale, sc)
        stems += op.cs == 4
    assert stems == 1
    n_bn = sum(1 for v in trainer.model.vs.moving if v.name.endswith('moving_mean:0'))
    assert len(ops) == n_bn                          # every BatchNorm of the network is folded


# ----------------------------------------------------------------------------------------------------------------
# 2. every folded launch against fp64
# ----------------------------------------------------------------------------------------------------------------
class _Recorder:
    """Records the arguments of every simclr_conv2d_fprop_tc_bias call made inside the block."""

    def __enter__(self):
        from simclr_b200._lib import lib
        self.lib = lib
        self.orig = lib.conv2d_fprop_tc_bias
        self.calls = []

        def rec(*a):
            self.orig(*a)
            self.calls.append(a)
        lib.conv2d_fprop_tc_bias = rec
        return self

    def __exit__(self, *exc):
        self.lib.conv2d_fprop_tc_bias = self.orig


def _unpack(wf, R, S, Cs, Cout):
    if Cs == 4:
        w = wf[:, :R * (S + 1) * 4].reshape(Cout, R, S + 1, 4)[:, :, 1:, :]
    else:
        w = wf[:, :R * S * Cs].reshape(Cout, R, S, Cs)
    return w.permute(0, 3, 1, 2).double()


# fp32 accumulation allowance in units of A (the same sum on absolute values), as in test_gpu_layers.py: the
# tensor-core fp32 sums of these launches err by up to 0.011 * 2^-16 A (measured on an H100 SXM, 700 W), which on
# an element with heavy cancellation (|v| ~ 1e-5 A) is more than one bf16 ulp of v.
TAU = 2.0 ** -17


def _check_launch(a):
    """One folded launch against fp64 on the same bf16 operands: every element within 1 bf16 ulp of bf16_rn(ref64)
    plus the fp32 accumulation allowance TAU * A, except where the fp64 pre-activation is within 2e-4 RMS of zero
    (the ReLU edge).  Returns the number of exempt elements."""
    x, wf, b, res, z, _, N, H, W, Cs, Cout, R, S, s, relu, _ = a
    xin = x.reshape(N, H, W, Cs).permute(0, 3, 1, 2).double()
    w = _unpack(wf, R, S, Cs, Cout)
    conv = lambda u, v: F.conv2d(u, v, stride=s, padding=(R - 1) // 2).permute(0, 2, 3, 1)
    pre = conv(xin, w) + b.double()
    A = conv(xin.abs(), w.abs()) + b.double().abs()
    if res is not None:
        pre = pre + res.reshape(pre.shape).double()
        A = A + res.reshape(pre.shape).double().abs()
    ref = pre.clamp_min(0) if relu else pre
    refb = ref.to(torch.bfloat16).double()
    got = z.reshape(ref.shape).double()
    ulp = torch.exp2(torch.floor(torch.log2(refb.abs().clamp_min(1e-30))) - 7)
    exempt = pre.abs() < 2e-4 * pre.pow(2).mean().sqrt()
    bad = ((got - refb).abs() > ulp + TAU * A) & ~exempt
    assert int(bad.sum()) == 0, (int(bad.sum()), (N, H, W, Cs, Cout, R, S, s, relu, res is not None),
                                 float((got - refb).abs().max()))
    return int(exempt.sum())


@pytest.mark.parametrize('arch,S,B', [('r50', 224, 2), ('r18', 32, 4), ('r152_sk', 64, 2)])
def test_every_folded_launch_against_fp64(fflags, arch, S, B):
    depth = {'r50': 50, 'r18': 18, 'r152_sk': 152}[arch]
    trainer = _setup(fflags, True, depth=depth, S=S, B=B, sk_ratio=0.0625 if arch == 'r152_sk' else 0.0)
    from oracle import model as OM
    om = OM.Model(cfg_from_flags(fflags.FLAGS), 100)
    P, S_ = om.init(0)
    _warm_params(P, 5)
    _random_moving(S_, 6)
    trainer.model.vs.load(P); trainer.model.vs.load(S_)
    f, _ = structured_batch(B, S, seed=7)
    with _Recorder() as r:
        trainer.model(f.cuda(), training=False)
    torch.cuda.synchronize()
    calls = r.calls
    kinds = collections.Counter()
    exempt = total = 0
    for a in calls:
        x, wf, b, res, z, zdt, N, H, W, Cs, Cout, R, S2, s, relu, _ = a
        exempt += _check_launch(a)
        total += z.numel()
        kinds['residual' if res is not None else 'plain'] += 1
        kinds['relu' if relu else 'linear'] += 1
        if Cs == 4:
            kinds['stem7x7' if R == 7 else 'stem_gather'] += 1
        elif R == 3 and s == 1 and Cs == Cout and Cs in (64, 128):
            kinds['halo'] += 1
        elif Cs % 64:
            kinds['gathered'] += 1
        else:
            kinds['tma'] += 1
    assert exempt < 1e-3 * total, (exempt, total)
    for k in ('residual', 'plain', 'relu', 'linear', 'tma'):
        assert kinds[k] > 0, (k, kinds)
    if arch == 'r50':
        assert kinds['stem7x7'] == 1 and kinds['halo'] > 0
    if arch == 'r18':
        assert kinds['stem_gather'] == 1
    if arch == 'r152_sk':
        assert kinds['stem_gather'] == 1 and kinds['gathered'] > 0


@pytest.mark.parametrize('cout,z_dtype', [(36, torch.bfloat16), (36, torch.float32), (200, torch.bfloat16)])
def test_dense_direct_store_and_fp32_outputs(fflags, cout, z_dtype):
    """Dense layers whose bf16 rows are not 16-byte multiples take the direct-store epilogue; fp32 outputs (the last
    projection layer) the TMA store.  Both against fp64."""
    from simclr_b200 import engine
    from simclr_b200._lib import lib, stream_ptr, DTYPE_CODE
    engine.set_engine(engine.Engine(precision='bf16', conv_engine='tc'))
    g = torch.Generator(device='cuda').manual_seed(3)
    rows, cin = 300, 128
    x = torch.randn(rows, 1, 1, cin, device='cuda', generator=g).to(torch.bfloat16)
    wf = (torch.randn(cout, cin, device='cuda', generator=g) * 0.1).to(torch.bfloat16)
    b = torch.randn(cout, device='cuda', generator=g)
    for relu in (0, 1):
        z = torch.empty(rows, 1, 1, cout, device='cuda', dtype=z_dtype)
        a = (x, wf, b, None, z, DTYPE_CODE[z_dtype], rows, 1, 1, cin, cout, 1, 1, 1, relu, stream_ptr())
        lib.conv2d_fprop_tc_bias(*a)
        torch.cuda.synchronize()
        _check_launch(a)


# ----------------------------------------------------------------------------------------------------------------
# 3. the model end to end (warm state of test_gpu_step.py)
# ----------------------------------------------------------------------------------------------------------------
FLOOR_FACTOR = 2.5      # the flip-floor bar of test_gpu_parity_bf16.py (DESIGN 6.1)


def _d64(D):
    return collections.OrderedDict((k, v.double()) for k, v in D.items())


def _emulation_bar(om, P, S_, f, outputs):
    """Each output against the bf16 emulation of the folded forward (oracle/fold.py) within FLOOR_FACTOR x the flip
    floor: the distance between that emulation evaluated in fp32 and in fp64 arithmetic, i.e. how far two correct
    implementations of the same rounding points differ by summation order alone."""
    from oracle import fold as OF
    from oracle.bf16_emul import emulate_bf16
    with torch.no_grad(), emulate_bf16():
        e32 = OF.Model(om)(P, S_, f)
        e64 = OF.Model(om)(_d64(P), _d64(S_), f.double())
    for got, a, b in zip(outputs, e32, e64):
        if a is None:
            continue
        err, floor = rel_err(got, b), rel_err(a, b)
        assert err <= FLOOR_FACTOR * floor, (err, floor)


@pytest.mark.parametrize('depth', [18, 50])
def test_eval_forward_end_to_end(fflags, depth):
    """R18 (basic blocks) and R50 (bottleneck blocks, projection shortcuts, the 7x7 stem kernel).  The ResNet-D and
    SK forms are outside the bf16 emulation of the oracle; their launches are held to fp64 above."""
    from test_gpu_step import _warm_state
    from oracle import model as OM, fold as OF
    from oracle.bf16_emul import emulate_bf16
    trainer = _setup(fflags, False, depth=depth, S=64, B=8, lineareval_while_pretraining=True, train_mode='pretrain')
    om = OM.Model(cfg_from_flags(fflags.FLAGS), 100)
    P, S_ = _warm_state(om)
    _random_moving(S_, 9)
    trainer.model.vs.load(P); trainer.model.vs.load(S_)
    f, _ = structured_batch(8, 64, seed=8)
    fc = f.cuda()

    def run():
        out = trainer.model(fc, training=False)
        torch.cuda.synchronize()
        return [t.clone() for t in out]

    unfolded = run()
    fflags.FLAGS.b200_fold_bn = True
    folded, again = run(), run()
    for a, b in zip(folded, again):
        assert torch.equal(a, b)                        # two calls: the same bits
    with torch.no_grad():
        ref32 = om(P, S_, f, False)
    _emulation_bar(om, P, S_, f, folded)
    for got, un, r32 in zip(folded, unfolded, ref32):
        d_fold, d_unfold = rel_err(got, r32), rel_err(un, r32)
        assert d_fold <= 1.25 * d_unfold, (d_fold, d_unfold)
    # new moving statistics written into the variables (what a checkpoint restore does): the next forward folds them
    S2 = collections.OrderedDict((k, v.clone()) for k, v in S_.items())
    _random_moving(S2, 10)
    trainer.model.vs.load(S2)
    after = run()
    _emulation_bar(om, P, S2, f, after)
    with torch.no_grad(), emulate_bf16():
        emul2 = OF.Model(om)(P, S2, f)
    for got, old, em in zip(after, folded, emul2):
        assert rel_err(got, old) > 10 * rel_err(got, em)


# ----------------------------------------------------------------------------------------------------------------
# 4. linear evaluation and partially frozen fine-tuning
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('ft_block', [2, 4])
def test_finetune_step_folded(fflags, ft_block):
    from oracle import model as OM, step as OS
    f6, lab = structured_batch(16, 64, num_classes=100, seed=2)
    f = f6[..., :3].contiguous()
    kw = dict(depth=18, S=64, B=16, train_mode='finetune', fine_tune_after_block=ft_block, ft_proj_selector=0,
              optimizer='momentum', lineareval_while_pretraining=False, weight_decay=1e-4)
    results = {}
    for fold in (False, True):
        trainer = _setup(fflags, fold, **kw)
        om = OM.Model(cfg_from_flags(fflags.FLAGS), 100)
        P, S_ = om.init(0)
        _warm_params(P, 11)
        _random_moving(S_, 12)
        trainer.model.vs.load(P); trainer.model.vs.load(S_)
        trainer.optimizer.learning_rate = 0.05
        loss = trainer.single_step(f.cuda(), lab.cuda())
        torch.cuda.synchronize()
        results[fold] = (loss.item(), {v.name: v.grad.clone() for v in trainer.model.trainable_variables})
    info = OS.forward_backward(om, P, S_, [f], [lab])
    ref_loss = info['loss'].item()
    (lu, gu), (lf, gf) = results[False], results[True]
    assert abs(lf - ref_loss) <= 1.25 * abs(lu - ref_loss), (lf, lu, ref_loss)
    for name, g in gf.items():
        ref = info['grads'][name]
        if ref.norm() == 0:
            continue
        d_f, d_u = rel_err(g, ref), rel_err(gu[name], ref)
        assert d_f <= 1.25 * d_u, (name, d_f, d_u)


def test_finetune_graph_replay_equals_eager(fflags):
    f6, lab = structured_batch(16, 64, num_classes=96, seed=4)
    f, lab = f6[..., :3].contiguous().cuda(), lab.cuda()
    results = []
    for use_graph in (False, True):
        fflags.set_flags(warmup_epochs=0, train_steps=4, learning_rate=0.8)
        # 96 classes: the supervised head's weight gradient stays on the deterministic tensor-core kernel (an
        # odd-width head takes the CUDA-core one, whose atomics make even two eager steps differ in the last bit)
        trainer = _setup(fflags, True, depth=18, S=64, B=16, num_classes=96, train_mode='finetune',
                         fine_tune_after_block=2, ft_proj_selector=0, optimizer='lars',
                         lineareval_while_pretraining=False)
        from oracle import model as OM
        om = OM.Model(cfg_from_flags(fflags.FLAGS), 96)
        P, S_ = om.init(0)
        _warm_params(P, 13)
        _random_moving(S_, 14)
        trainer.model.vs.load(P); trainer.model.vs.load(S_)
        if use_graph:
            trainer.capture(f, lab, warmup=1, restore=True)
            for _ in range(3):
                loss = trainer.replay()
        else:
            for _ in range(3):
                loss = trainer.single_step(f, lab)
        torch.cuda.synchronize()
        results.append((trainer.model.vs.flat_value.clone(), trainer.model.vs.flat_moving.clone(), loss.clone()))
    for a, b in zip(*results):
        assert torch.equal(a, b)


def test_invalid_modes_raise_on_build(fflags):
    from simclr_b200 import engine, run, distill
    fflags.set_flags(resnet_depth=18, image_size=32, train_batch_size=2, b200_fold_bn=True)
    for precision, conv_engine in (('fp32', 'tc3'), ('fp32', 'simt'), ('bf16', 'simt')):
        fflags.set_flags(b200_precision=precision, b200_conv_engine=conv_engine)
        engine.set_engine(engine.Engine(precision=precision, conv_engine=conv_engine))
        with pytest.raises(ValueError, match='b200_fold_bn'):
            run.Trainer(num_classes=10, num_examples=100, seed=0)
        with pytest.raises(ValueError, match='b200_fold_bn'):
            distill.Teacher(None, num_classes=10)


# ----------------------------------------------------------------------------------------------------------------
# 5. the distillation teacher
# ----------------------------------------------------------------------------------------------------------------
def test_folded_teacher_logits(fflags):
    from test_gpu_distill import _distill_setup
    from simclr_b200 import distill
    fflags.FLAGS.b200_fold_bn = True
    trainer, teacher, om, otm, P, S_, TP, TS = _distill_setup(fflags, 'lars', 'bf16', 'tc', num_classes=96)
    assert teacher.flag_values['b200_fold_bn']
    plain = distill.Teacher(None, num_classes=96, seed=5, fold_bn=False)
    plain.model.vs.load(TP); plain.model.vs.load(TS)
    f6, _ = structured_batch(16, 64, num_classes=96, seed=3)
    f = f6[..., :3].contiguous()
    got, got2, un = teacher(f.cuda()).clone(), teacher(f.cuda()).clone(), plain(f.cuda()).clone()
    torch.cuda.synchronize()
    assert torch.equal(got, got2)
    with torch.no_grad():
        _, ref = otm(TP, TS, f, False)
    d_fold, d_unfold = rel_err(got, ref), rel_err(un, ref)
    assert d_fold <= 1.25 * d_unfold, (d_fold, d_unfold)


def test_folded_teacher_against_emulation(fflags):
    """A teacher without SK (R50: bottleneck blocks, projection shortcuts), which the bf16 emulation of the oracle
    covers: its folded logits against the emulated folded teacher and, against the fp32 oracle, no farther than the
    unfolded teacher."""
    from simclr_b200 import engine, distill
    from oracle import model as OM
    fflags.set_flags(resnet_depth=18, width_multiplier=1, sk_ratio=0.0, se_ratio=0.0, image_size=64, train_batch_size=8,
                     use_blur=False, train_mode='finetune', fine_tune_after_block=-1, ft_proj_selector=0,
                     lineareval_while_pretraining=False, b200_precision='bf16', b200_conv_engine='tc',
                     b200_teacher_resnet_depth=50, b200_teacher_sk_ratio=0.0, b200_teacher_ft_proj_selector=1,
                     b200_teacher_width_multiplier=None, b200_teacher_se_ratio=None, b200_fold_bn=True)
    engine.set_engine(engine.Engine(precision='bf16', conv_engine='tc'))
    teacher = distill.Teacher(None, num_classes=96, seed=5)
    plain = distill.Teacher(None, num_classes=96, seed=5, fold_bn=False)
    with distill.flag_scope(**teacher.flag_values):
        otm = OM.Model(cfg_from_flags(fflags.FLAGS), 96)
    TP, TS = otm.init(5)
    _warm_params(TP, 21)
    _random_moving(TS, 22)
    for t in (teacher, plain):
        t.model.vs.load(TP); t.model.vs.load(TS)
    f6, _ = structured_batch(8, 64, num_classes=96, seed=3)
    f = f6[..., :3].contiguous()
    got, un = teacher(f.cuda()).clone(), plain(f.cuda()).clone()
    torch.cuda.synchronize()
    with torch.no_grad():
        _, ref = otm(TP, TS, f, False)
    _emulation_bar(otm, TP, TS, f, (None, got))
    d_fold, d_unfold = rel_err(got, ref), rel_err(un, ref)
    assert d_fold <= 1.25 * d_unfold, (d_fold, d_unfold)


def test_first_fold_inside_capture(fflags):
    """A layer's first folded forward may run inside a CUDA-graph capture (no host-to-device copy): the replay
    gives the eager forward's bits."""
    trainer = _setup(fflags, True, depth=18, S=32, B=4, train_mode='finetune', lineareval_while_pretraining=False)
    f = torch.rand(4, 32, 32, 3, generator=torch.Generator().manual_seed(2)).cuda()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _, out = trainer.model(f, training=False)
    graph.replay()
    torch.cuda.synchronize()
    captured = out.clone()
    _, eager = trainer.model(f, training=False)
    torch.cuda.synchronize()
    assert torch.equal(captured, eager)


def test_folded_teacher_graph_replay_equals_eager(fflags):
    from test_gpu_distill import _distill_setup
    f6, lab = structured_batch(16, 64, num_classes=96, seed=4)
    f, lab = f6[..., :3].contiguous().cuda(), lab.cuda()
    results = []
    for use_graph in (False, True):
        fflags.set_flags(warmup_epochs=0, train_steps=4, learning_rate=0.8, b200_fold_bn=True)
        trainer, teacher, *_ = _distill_setup(fflags, 'lars', 'bf16', 'tc', num_classes=96)
        if use_graph:
            trainer.capture(f, lab, warmup=1, restore=True)
            for _ in range(3):
                loss = trainer.replay()
        else:
            for _ in range(3):
                loss = trainer.single_step(f, lab)
        torch.cuda.synchronize()
        results.append((trainer.model.vs.flat_value.clone(), loss.clone(), trainer.metrics['teacher_logits'].clone()))
    for a, b in zip(*results):
        assert torch.equal(a, b)
