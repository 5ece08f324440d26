"""Activation recomputation (resnet.BlockGroup with `recompute`): a step that replays its block groups in the
backward pass computes the same bits as one that stored their activations -- loss, every gradient, every updated
weight and optimizer slot, every moving statistic -- eagerly and as a replayed CUDA graph; the fused replay
epilogue of the implicit-GEMM fprop (`simclr_conv2d_fprop_tc_apply`) equals conv + BatchNorm apply bit for bit;
and recomputing every group cuts the peak memory of a ResNet-50 step as the byte model predicts."""
import gc

import pytest
import torch

from util import structured_batch

pytestmark = pytest.mark.gpu

ALL = {1, 2, 3, 4}


def _trainer(flags_def, recompute, kw):
    from simclr_b200 import engine, run
    precision, conv_engine = kw['b200_precision'], kw['b200_conv_engine']
    flags_def.set_flags(**kw)
    engine.set_engine(engine.Engine(precision=precision, conv_engine=conv_engine))
    # 128 classes: the supervised head's weight gradient takes the tensor-core kernel (an odd width would take the
    # CUDA-core one, whose fp32 atomics over batch splits make its last bits vary from run to run)
    trainer = run.Trainer(num_classes=128, num_examples=50000, seed=0, recompute=recompute)
    g = torch.Generator().manual_seed(3)
    for v in trainer.model.vs.trainable + trainer.model.vs.moving:      # a warm state: every gradient non-zero
        if v.name.endswith('gamma:0'):
            v.value.copy_(0.5 + torch.rand(v.shape, generator=g))
        elif v.name.endswith('beta:0') or v.name.endswith('moving_mean:0'):
            v.value.copy_(torch.randn(v.shape, generator=g) * 0.1)
        elif v.name.endswith('moving_variance:0'):
            v.value.copy_(0.5 + torch.rand(v.shape, generator=g))
    trainer.optimizer.learning_rate = 0.1
    return trainer


def _state(trainer, loss):
    opt = trainer.optimizer
    slots = [opt._flat_v] if hasattr(opt, '_flat_v') else list(opt._slots)
    vs = trainer.model.vs
    return [loss.detach().clone(), vs.flat_grad.clone(), vs.flat_value.clone(), vs.flat_moving.clone()] + \
        [s.clone() for s in slots]


NAMES = ['loss', 'gradients', 'weights', 'moving statistics', 'optimizer slot']


def _compare(got, ref):
    for n, a, b in zip(NAMES, got, ref):
        assert torch.equal(a, b), '%s differs (%d of %d elements)' % (n, int((a != b).sum()), a.numel())


def _run(flags_def, recompute, kw, graph, B, S):
    trainer = _trainer(flags_def, recompute, kw)
    assert trainer.model.resnet_model.recompute == frozenset(recompute) - set(range(1, 1 + max(
        kw.get('fine_tune_after_block', -1), 0)))
    f, lab = structured_batch(B, S, num_classes=128, seed=4)
    if kw.get('train_mode') == 'finetune':
        f = f[..., :3].contiguous()
    f, lab = f.cuda(), lab.cuda()
    if graph:
        trainer.capture(f, lab, warmup=1)
        trainer.replay()
        loss = trainer.replay()
    else:
        loss = trainer.single_step(f, lab)
    torch.cuda.synchronize()
    return _state(trainer, loss)


BF16 = dict(b200_precision='bf16', b200_conv_engine='tc', use_blur=False, weight_decay=1e-4)
CASES = {
    'r50-se': (dict(BF16, resnet_depth=50, image_size=64, train_batch_size=8, se_ratio=0.25), 8, 64),
    'r18-cfg1': (dict(BF16, resnet_depth=18, image_size=64, train_batch_size=16), 16, 64),
    'r50': (dict(BF16, resnet_depth=50, image_size=64, train_batch_size=16), 16, 64),
    'r50-sk': (dict(BF16, resnet_depth=50, image_size=64, train_batch_size=8, sk_ratio=0.0625), 8, 64),
    'r18-finetune-momentum': (dict(BF16, resnet_depth=18, image_size=64, train_batch_size=16, train_mode='finetune',
                                   fine_tune_after_block=1, optimizer='momentum', lineareval_while_pretraining=False),
                              16, 64),
    'r18-fp32-tc3': (dict(resnet_depth=18, image_size=32, train_batch_size=8, use_blur=False, weight_decay=1e-4,
                          b200_precision='fp32', b200_conv_engine='tc3'), 8, 32),
}


@pytest.mark.parametrize('graph', [False, True], ids=['eager', 'graph'])
@pytest.mark.parametrize('case', sorted(set(CASES) - {'r50-se'}))
def test_recomputed_step_is_bit_identical(flags, case, graph):
    kw, B, S = CASES[case]
    ref = _run(flags, set(), kw, graph, B, S)
    got = _run(flags, ALL, kw, graph, B, S)
    _compare(got, ref)


def test_recomputed_se_step(flags):
    """SE blocks: the gates' weight gradients come from the CUDA-core kernel, which adds batch splits with fp32
    atomics, so two runs of the same step differ in the last bits of their gradients, and over several steps
    (a replayed graph) those differences compound.  One eager step: the forward (loss, moving statistics) is
    bit-identical; gradients, weights and slots differ from the stored step by no more than (4x, in norm) two runs
    without recomputation differ from each other."""
    from util import rel_err
    kw, B, S = CASES['r50-se']
    ref = _run(flags, set(), kw, False, B, S)
    ref2 = _run(flags, set(), kw, False, B, S)
    got = _run(flags, ALL, kw, False, B, S)
    for n, a, b, b2 in zip(NAMES, got, ref, ref2):
        if n in ('loss', 'moving statistics'):
            assert torch.equal(a, b), n
        else:
            assert rel_err(a, b) <= 4 * rel_err(b2, b) + 1e-7, (n, rel_err(a, b), rel_err(b2, b))


def test_mixed_plan_is_bit_identical(flags):
    kw, B, S = CASES['r50']
    ref = _run(flags, set(), kw, False, B, S)
    got = _run(flags, {1, 3}, kw, False, B, S)
    _compare(got, ref)


# ResNet-50 implicit-GEMM layers: (N, H, Cin, Cout, k, stride) -- 1x1, strided 1x1, im2col 3x3 (strided and not),
# projection shortcut
APPLY_SHAPES = [(8, 28, 256, 64, 1, 1), (8, 28, 256, 512, 1, 2), (8, 28, 128, 128, 3, 2), (8, 14, 256, 256, 3, 1),
                (8, 56, 64, 256, 1, 1), (8, 56, 256, 128, 1, 1)]


@pytest.mark.parametrize('relu', [1, 0], ids=['relu', 'linear'])
@pytest.mark.parametrize('shape', APPLY_SHAPES, ids=lambda s: 'n%d_h%d_%d-%d_k%d_s%d' % s)
def test_fprop_apply_matches_conv_then_apply(shape, relu):
    from simclr_b200._lib import lib, stream_ptr, BF16 as B
    N, H, Cin, Cout, k, s = shape
    g = torch.Generator(device='cuda').manual_seed(1)
    x = torch.randn(N, H, H, Cin, device='cuda', generator=g).to(torch.bfloat16)
    w = torch.randn(k, k, Cin, Cout, device='cuda', generator=g) / (k * k * Cin) ** 0.5
    Kp = (k * k * Cin + 63) // 64 * 64
    wf = torch.empty(Cout, Kp, dtype=torch.bfloat16, device='cuda')
    st = stream_ptr()
    lib.pack_conv_weight(w, wf, None, B, k, k, Cin, Cin, Cout, Kp, st)
    scale = torch.randn(Cout, device='cuda', generator=g)
    shift = torch.randn(Cout, device='cuda', generator=g)
    Ho = (H - 1) // s + 1
    y_ref = torch.empty(N, Ho, Ho, Cout, dtype=torch.bfloat16, device='cuda')
    z_ref, y, z = torch.empty_like(y_ref), torch.full_like(y_ref, float('nan')), torch.full_like(y_ref, float('nan'))
    lib.conv2d_fprop_tc(x, wf, y_ref, B, B, N, H, H, Cin, Cout, k, k, s, None, st)
    lib.bn_apply(y_ref, B, None, z_ref, B, N * Ho * Ho, Cout, scale, shift, relu, st)
    lib.conv2d_fprop_tc_apply(x, wf, y, z, B, N, H, H, Cin, Cout, k, k, s, scale, shift, relu, st)
    torch.cuda.synchronize()
    assert torch.equal(y.view(torch.int16), y_ref.view(torch.int16))
    assert torch.equal(z.view(torch.int16), z_ref.view(torch.int16))


def test_recompute_peak_memory(flags):
    """ResNet-50 at 128 samples (256 views) of 224x224: recomputing every group keeps at most 55 % of the peak
    bytes of the stored step, and the byte model predicts the recomputed peak to 10 %."""
    from simclr_b200 import memory
    B, S = 128, 224
    kw = dict(BF16, resnet_depth=50, image_size=S, train_batch_size=B)
    peaks = {}
    f, lab = structured_batch(B, S, num_classes=128, seed=4)
    for name, rc in (('off', set()), ('all', ALL)):
        gc.collect()
        torch.cuda.empty_cache()
        pre = torch.cuda.memory_allocated()         # what earlier tests left: not part of this step
        trainer = _trainer(flags, rc, kw)
        fc, lc = f.cuda(), lab.cuda()
        trainer.single_step(fc, lc)                  # first step: lazy buffers and packed operands
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        trainer.single_step(fc, lc)
        torch.cuda.synchronize()
        peaks[name] = torch.cuda.max_memory_allocated() - pre
        del trainer, fc, lc
        torch.cuda.empty_cache()
    m = memory.model_from_flags(flags.FLAGS, B)
    pred = memory.predicted_peak(m, ALL)
    print('peak allocated: off %.3f GiB, all %.3f GiB (predicted off %.3f, all %.3f)' % (
        memory.gib(peaks['off']), memory.gib(peaks['all']), memory.gib(memory.predicted_peak(m, set())),
        memory.gib(pred)))
    assert peaks['all'] <= 0.55 * peaks['off']
    assert abs(peaks['all'] - pred) <= 0.1 * peaks['all']
