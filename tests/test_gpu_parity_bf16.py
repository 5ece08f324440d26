"""Parity of the BENCHMARKED precision: bf16 storage + wgmma conv engine.

The reference computes the step in fp32 (tf2/run.py:557-622).  bf16 activation storage is not
a 1e-3 approximation of that.  On ANY state of this network (ResNet + 3 BN'd head layers +
NT-Xent, whose gradient is a difference of nearly equal embeddings) rounding every stored
activation to bf16 moves the embeddings by ~3 % and every gradient tensor by ~25 % -- measured on
the CPU alone by `test_oracle.py::test_bf16_storage_rounding_model`, independent of weights, images,
batch size and temperature.  Worse for testing, bf16 rounding is a discontinuity met ~1e8 times per
step: two CORRECT implementations of the same bf16-storage algorithm that differ only in summation
order round a fraction of the elements the other way, and that alone separates their gradient
tensors by ~8 % (the bf16-storage oracle evaluated in fp32 vs in fp64 arithmetic: `flip floor`
below).  No per-tensor gradient comparison of a bf16 step can be tighter than that floor, whatever
the fixture.  What can be pinned, and is:

1. the CUDA bf16 step is as close to the bf16-storage oracle (`oracle/bf16_emul.py`: rounding at
   exactly the CUDA path's storage points) as that oracle is to itself under a change of arithmetic
   precision: per gradient tensor <= `FLOOR_FACTOR` x flip floor + `FLOOR_ABS`; loss to 1e-3;
2. its distance to the fp32 reference is the cost of bf16 storage and nothing else: per tensor
   <= `MODEL_SLACK` x the emulated storage cost on the same fixture + `FLOOR_ABS`, medians within 15 %
   (a kernel bug adds error on top of the rounding model; observed ratio of medians 0.98-1.03);
3. a 20-step LARS trajectory tracks the fp32 oracle's loss curve as closely as the bf16-storage
   oracle's own trajectory does.
On ResNet-18 (config 1) and on plain ResNet-50 bottlenecks (the benchmarked network family).
The 1e-3 bar of the north_star is met on the tensor pipe by the split-bf16 mode (tc3) (test_gpu_step.py::
test_step_parity_tc3) and kernel by kernel in test_gpu_tc.py (2e-4 on bf16-representable inputs).
"""
import collections

import pytest
import torch

from util import rel_err, cfg_from_flags, structured_batch
from test_gpu_step import _setup, _data

pytestmark = pytest.mark.gpu

FLOOR_FACTOR = 2.5    # CUDA-vs-emulation error allowed per tensor, in units of the oracle's own flip floor
FLOOR_ABS = 3e-2
MODEL_SLACK = 1.35    # CUDA-vs-fp32 error may exceed the emulated storage cost by this factor (per tensor)


def _median(d):
    v = sorted(d.values())
    return v[len(v) // 2]


@pytest.mark.parametrize('depth,B,kind,warm', [
    (18, 32, 'noise', False), (18, 32, 'noise', 'lars'),        # config 1 of BASELINE.json
    (18, 64, 'struct', 'lars'),                                 # 128 views, structured images
    (50, 32, 'struct', False), (50, 32, 'struct', 'lars'),      # plain ResNet-50 bottlenecks
])
def test_bf16_tc_step_matches_bf16_storage_oracle(flags, depth, B, kind, warm):
    from oracle import step as OS
    from oracle.bf16_emul import emulate_bf16
    S = 64
    trainer, om, P, S_ = _setup(flags, 'bf16', 'tc', warm, B, S, depth=depth, use_blur=(kind == 'noise'))
    if kind == 'noise':
        f, lab, sigma, sel = _data(B, S)
        draws = [[(sigma[0], sel[0]), (sigma[1], sel[1])]]
        trainer.model.set_blur_draws(torch.tensor(sigma), sel)
    else:
        f, lab = structured_batch(B, S, seed=0)
        draws = None
    i32 = OS.forward_backward(om, P, S_, [f], [lab], blur_draws=draws)
    P64 = collections.OrderedDict((k, v.double()) for k, v in P.items())
    S64 = collections.OrderedDict((k, v.double()) for k, v in S_.items())
    with emulate_bf16():
        ib = OS.forward_backward(om, P, S_, [f], [lab], blur_draws=draws)
        ib64 = OS.forward_backward(om, P64, S64, [f.double()], [lab.double()], blur_draws=draws)
    trainer.optimizer.learning_rate = 0.0
    loss = trainer.single_step(f.cuda(), lab.cuda())
    torch.cuda.synchronize()
    names = [v.name for v in trainer.model.trainable_variables if i32['grads'][v.name].norm() > 0]
    grads = {v.name: v.grad for v in trainer.model.trainable_variables}
    match = {k: rel_err(grads[k], ib['grads'][k]) for k in names}
    floor = {k: rel_err(ib['grads'][k], ib64['grads'][k]) for k in names}       # the oracle vs itself
    gpu32 = {k: rel_err(grads[k], i32['grads'][k]) for k in names}
    emu32 = {k: rel_err(ib['grads'][k], i32['grads'][k]) for k in names}
    wm = max(match, key=match.get)
    print('R%d B%d %s warm=%s | loss cuda %.5f emu %.5f fp32 %.5f | cuda-vs-emu grads: median %.2e worst %.2e (%s)'
          ' | flip floor (emu fp32 vs fp64 arithmetic): median %.2e max %.2e'
          ' | vs fp32: cuda median %.2e, emulation median %.2e'
          % (depth, B, kind, warm, loss.item(), ib['loss'].item(), i32['loss'].item(), _median(match), match[wm], wm,
             _median(floor), max(floor.values()), _median(gpu32), _median(emu32)))
    # 1. same algorithm as the bf16-storage oracle, down to the flip floor
    assert abs(loss.item() - ib['loss'].item()) < 1e-3 * abs(ib['loss'].item())
    assert rel_err(trainer.metrics['logits_con'], ib['logits_con'][0]) < \
        FLOOR_FACTOR * rel_err(ib['logits_con'][0], ib64['logits_con'][0]) + 5e-3
    assert _median(match) < 2.0 * _median(floor) + 1e-2, (_median(match), _median(floor))
    for k in names:
        assert match[k] < FLOOR_FACTOR * floor[k] + FLOOR_ABS, (k, match[k], floor[k])
    for v in trainer.model.trainable_variables:          # exactly-zero gradients at the reference init (Q3)
        if i32['grads'][v.name].norm() == 0:
            assert float(v.grad.abs().max()) == 0.0, v.name
    # 2. distance to the fp32 reference == what storage rounding costs, not more
    assert abs(loss.item() - i32['loss'].item()) < 5e-3 * abs(i32['loss'].item())
    assert 0.85 < _median(gpu32) / _median(emu32) < 1.15, (_median(gpu32), _median(emu32))
    for k in names:
        assert gpu32[k] < MODEL_SLACK * emu32[k] + FLOOR_ABS, (k, gpu32[k], emu32[k])


def test_bf16_tc_loss_curve_20_steps(flags):
    """north_star: "loss curve matching reference within tolerance" at the benchmarked precision.
    20 consecutive LARS steps of config 1 (ResNet-18, batch 32, 64x64; a fresh structured batch per
    step, lr 0.2, weight decay 1e-4) on the bf16 wgmma path against the fp32 oracle trajectory
    (which the fp32 verification mode reproduces to 1e-3, test_gpu_step.py).  Training is chaotic:
    the yardstick for "within tolerance" is how far the bf16-STORAGE ORACLE's own trajectory drifts
    from the fp32 one over the same 20 steps."""
    from oracle import step as OS
    from oracle.bf16_emul import emulate_bf16
    B, S, steps = 32, 64, 20
    trainer, om, P, S_ = _setup(flags, 'bf16', 'tc', False, B, S, use_blur=False)
    V = collections.OrderedDict((k, torch.zeros_like(v)) for k, v in P.items())
    Pe, Se, Ve = P, S_, V
    ours, ref, emu = [], [], []
    lr = 0.2
    trainer.optimizer.learning_rate = lr
    for step in range(steps):
        f, lab = structured_batch(B, S, seed=1000 + step)
        P, S_, V, info = OS.single_step(om, P, S_, V, [f], [lab], lr)
        with emulate_bf16():
            Pe, Se, Ve, ie = OS.single_step(om, Pe, Se, Ve, [f], [lab], lr)
        ref.append(float(info['loss'])); emu.append(float(ie['loss']))
        ours.append(float(trainer.single_step(f.cuda(), lab.cuda())))
    dev = [abs(a - b) / abs(b) for a, b in zip(ours, ref)]
    dev_e = [abs(a - b) / abs(b) for a, b in zip(emu, ref)]
    print('bf16/tc loss curve  ', ['%.4f' % a for a in ours])
    print('fp32 oracle curve   ', ['%.4f' % b for b in ref])
    print('bf16-storage oracle ', ['%.4f' % b for b in emu])
    print('relative deviation from fp32: cuda max %.2e mean %.2e | bf16-storage oracle max %.2e mean %.2e'
          % (max(dev), sum(dev) / steps, max(dev_e), sum(dev_e) / steps))
    assert min(ref[-5:]) < ref[0] - 0.5, 'the trajectory must actually train (loss falls)'
    assert max(dev[:3]) < 5e-3, dev             # before the trajectories decorrelate
    assert max(dev) < 1.5 * max(dev_e) + 2e-2, (max(dev), max(dev_e))
    assert sum(dev) / steps < 1.5 * sum(dev_e) / steps + 5e-3, (dev, dev_e)
    assert abs(sum(ours[-5:]) - sum(ref[-5:])) / sum(ref[-5:]) < 2e-2     # same loss level after 20 steps


def test_num_classes_not_multiple_of_8(flags):
    """CIFAR-10-style supervised head (num_classes=10): the wgmma wgrad needs 16-byte output rows,
    so this layer takes the CUDA-core fallback instead of failing the first backward."""
    from simclr_b200 import engine, run, flags_def
    from oracle import model as OM, step as OS
    from oracle.bf16_emul import emulate_bf16
    B, S = 16, 32
    flags_def.set_flags(resnet_depth=18, image_size=S, train_batch_size=B, use_blur=False,
                        b200_precision='bf16', b200_conv_engine='tc', weight_decay=1e-4)
    engine.set_engine(engine.Engine(precision='bf16', conv_engine='tc'))
    trainer = run.Trainer(num_classes=10, num_examples=50000, seed=0)
    om = OM.Model(cfg_from_flags(flags_def.FLAGS), 10)
    P, S_ = om.init(0)
    trainer.model.vs.load(P); trainer.model.vs.load(S_)
    f, lab = structured_batch(B, S, num_classes=10, seed=3)
    with emulate_bf16():
        ib = OS.forward_backward(om, P, S_, [f], [lab])
    trainer.optimizer.learning_rate = 0.0
    loss = trainer.single_step(f.cuda(), lab.cuda())
    torch.cuda.synchronize()
    assert abs(loss.item() - ib['loss'].item()) < 1e-3 * abs(ib['loss'].item())
    for v in trainer.model.trainable_variables:
        if 'head_supervised' in v.name:
            assert rel_err(v.grad, ib['grads'][v.name]) < 0.1, v.name
