"""Every kernel launch of the configurations outside the benchmarked pretraining families against fp64, element by
element: the CIFAR-10 recipe (bf16 / tc, fp32 / tc3 and fp32 / simt), ResNet-18 at 64, ResNet-34 at 224, SE,
fine-tuning with frozen block groups (momentum and Adam), linear evaluation and inference-mode evaluation.

test_gpu_layers.py, test_gpu_ops.py and test_gpu_layers_tc3.py take their inventory from R50 1x, R50 2x and R50 2x SK
pretraining at 224.  These configurations reach code those steps never run: the CIFAR 3x3/1 stem on 4 stored
channels (the S+1-slot small-channel gather: pixel pairs need stride 2), fprops without fused BatchNorm sums (every
eval forward and every frozen group), 4x4 and 2x2 last stages (one 128-row tile spans 8 or 32 images), basic blocks
(a strided 3x3 with Cout = 2 Cin), the SE gate and scale kernels, the momentum and Adam updates and the CUDA-core
fp32 engine.

The inventory runs one eager step per family at 2 samples and records every `tc`, `tc3` and `simt` conv (its key,
the largest N and every pre-zeroed mode it ran in) and every other C-ABI entry (keyed as test_gpu_ops keys it).
Each distinct launch is replayed once, by the first family that records it, at the recorded N and at a large N,
with the helpers of the earlier files: test_gpu_layers.check_launch (bf16 tc), test_gpu_layers_tc3.check_passes and
check_end_to_end (tc3), test_gpu_ops.REPLAY (the other entries), plus the replayers below for the optimizers, the
SE kernels and the CUDA-core convs.  Every bound is |got - ref| <= rho |ref| + tau A as in those files.
"""
import math
import time

import pytest
import torch

from test_gpu_kernels import conv_reference
import test_gpu_layers as L
import test_gpu_layers_tc3 as L3
import test_gpu_ops as O
from test_gpu_ops import DT, RHO, TAU_EW, U, tau_seq

pytestmark = pytest.mark.gpu

BF16, F32 = torch.bfloat16, torch.float32

_CIFAR = dict(resnet_depth=18, image_size=32, use_blur=False, temperature=0.5, optimizer='lars')
# precision, conv engine, what runs ('pretrain' / 'finetune': one training step; 'eval': the inference forward),
# classes, flags
FAMILIES = {
    'cifar10_r18_32': ('bf16', 'tc', 'pretrain', 10, _CIFAR),
    'cifar10_r18_32_tc3': ('fp32', 'tc3', 'pretrain', 10, _CIFAR),
    'cifar10_r18_32_simt': ('fp32', 'simt', 'pretrain', 10, _CIFAR),
    'r18_64': ('bf16', 'tc', 'pretrain', 1000, dict(resnet_depth=18, image_size=64)),
    'r34_224': ('bf16', 'tc', 'pretrain', 1000, dict(resnet_depth=34, image_size=224)),
    'r50_se_224': ('bf16', 'tc', 'pretrain', 1000, dict(resnet_depth=50, image_size=224, se_ratio=0.0625)),
    'r50_finetune_224': ('bf16', 'tc', 'finetune', 1000,
                         dict(resnet_depth=50, image_size=224, fine_tune_after_block=-1, optimizer='momentum')),
    'r50_lineareval_224': ('bf16', 'tc', 'finetune', 1000,
                           dict(resnet_depth=50, image_size=224, fine_tune_after_block=4, optimizer='momentum')),
    'r18_finetune_adam_32': ('bf16', 'tc', 'finetune', 10,
                             dict(resnet_depth=18, image_size=32, fine_tune_after_block=2, optimizer='adam')),
    'r50_eval_224': ('bf16', 'tc', 'eval', 1000, dict(resnet_depth=50, image_size=224)),
}

TC = ('conv2d_fprop_tc', 'conv2d_dgrad_tc', 'conv2d_wgrad_tc')
TC3 = ('conv2d_fprop_tc3', 'conv2d_dgrad_tc3', 'conv2d_wgrad_tc3')
SIMT = ('conv2d_fprop_simt', 'conv2d_dgrad_simt', 'conv2d_wgrad_simt')
MACS_BUDGET = 1e10                   # multiply-adds per CUDA-core conv at the large batch
SIMT_VIEWS = 128                     # the large batch of a CUDA-core conv, before the MACs budget


def _simt_key(name, a):
    """(kind, H, W, Cs, Cin, Cout, R, S, stride, in dtype, out dtype) and N of one CUDA-core conv call."""
    if name == 'conv2d_fprop_simt':
        din, dout, (N, H, W, Cs, Cin, Cout, R, S, s) = a[3], a[4], a[5:14]
        return ('simt fprop', H, W, Cs, Cin, Cout, R, S, s, DT[din], DT[dout]), N
    if name == 'conv2d_dgrad_simt':
        din, dout, (N, H, W, Cin, Cout, R, S, s) = a[3], a[4], a[5:13]
        return ('simt dgrad', H, W, Cin, Cin, Cout, R, S, s, DT[din], DT[dout]), N
    din, (N, H, W, Cs, Cin, Cout, R, S, s) = a[3], a[4:13]
    return ('simt wgrad', H, W, Cs, Cin, Cout, R, S, s, DT[din], F32), N


def _simt_fmt(key):
    kind, H, W, Cs, Cin, Cout, R, S, s, din, dout = key
    dt = {BF16: 'bf16', F32: 'f32'}
    return '%s %3dx%-3d Cs %4d Cin %4d Cout %4d %dx%d/%d %s->%s' % (kind, H, W, Cs, Cin, Cout, R, S, s, dt[din], dt[dout])


def _run_family(fam):
    """One eager step (or the eval forward) of a family with every C-ABI entry recorded."""
    from simclr_b200 import engine, run, flags_def
    from simclr_b200._lib import lib
    prec, eng, mode, classes, cfg = FAMILIES[fam]
    B, S = 2, cfg['image_size']
    flags_def.set_flags(train_batch_size=B, weight_decay=1e-4, b200_precision=prec, b200_conv_engine=eng,
                        train_mode='pretrain' if mode == 'eval' else mode, **cfg)
    engine.set_engine(engine.Engine(precision=prec, conv_engine=eng))
    trainer = run.Trainer(num_classes=classes, num_examples=50000, seed=0)
    g = torch.Generator().manual_seed(3)
    f = torch.rand(B, S, S, 6 if mode == 'pretrain' else 3, generator=g).cuda()
    lab = torch.nn.functional.one_hot(torch.randint(0, classes, (B,), generator=g), classes).float().cuda()
    rec = dict(tc={}, tc_modes={}, tc3={}, tc3_modes={}, simt={}, simt_modes={}, ops=set())
    state = {'pz': 0}

    def note(conv, modes, key, N):
        conv[key] = max(N, conv.get(key, 0))
        modes.setdefault(key, set()).add(state['pz'])

    with pytest.MonkeyPatch.context() as mp:
        setpz = getattr(lib, 'set_accumulate_prezeroed')

        def wrap_pz(on, _fn=setpz):
            state['pz'] = int(on)
            return _fn(on)
        mp.setattr(lib, 'set_accumulate_prezeroed', wrap_pz)
        for full in lib.declarations:
            name = full[len('simclr_'):]
            if name in TC:
                rk = lambda n, a: L._launch_key(n, a) + ('tc',)
            elif name in TC3:
                rk = lambda n, a: L3._conv_key(n, a)[:2] + ('tc3',)
            elif name in SIMT:
                rk = lambda n, a: _simt_key(n, a) + ('simt',)
            elif O.EXCLUDED.match(name):
                continue
            else:
                rk = None
            fn = getattr(lib, name)             # _Lib.__getattr__ caches the bound call on the instance

            def wrap(*a, _fn=fn, _name=name, _rk=rk):
                if _rk is None:
                    rec['ops'].add(O._launch_key(_name, a, state['pz']))
                else:
                    key, N, kind = _rk(_name, a)
                    note(rec[kind], rec[kind + '_modes'], key, N)
                return _fn(*a)
            mp.setattr(lib, name, wrap)
        if mode == 'eval':
            trainer.model(f, training=False)
        else:
            trainer.single_step(f, lab)
        torch.cuda.synchronize()
    del trainer
    torch.cuda.empty_cache()
    return rec


@pytest.fixture(scope='module')
def inventory():
    """{family: dict(tc=, tc3=, simt= {conv key: N}, tc_modes=, tc3_modes=, simt_modes= {conv key: set of
    pre-zeroed modes}, ops= set of test_gpu_ops launch keys)}."""
    from simclr_b200 import flags_def
    from simclr_b200._lib import lib
    F = flags_def.FLAGS
    if not F.is_parsed():
        F(['test'])
    saved = {k: getattr(F, k) for k in flags_def.REFERENCE_FLAG_NAMES + ['b200_precision', 'b200_conv_engine']}
    inv = {}
    try:
        for fam in FAMILIES:
            for k, v in saved.items():          # each family starts from the reference defaults
                setattr(F, k, v)
            inv[fam] = _run_family(fam)
    finally:
        for k, v in saved.items():
            setattr(F, k, v)
        lib.set_accumulate_prezeroed(0)
    for fam, rec in inv.items():
        print('\n%s: %d tc, %d tc3, %d CUDA-core conv launches, %d other launches' % (
            fam, len(rec['tc']), len(rec['tc3']), len(rec['simt']), len(rec['ops'])))
        for key in sorted(rec['tc'], key=L._fmt):
            print('    N %3d  %-70s prezeroed %s' % (rec['tc'][key], L._fmt(key), sorted(rec['tc_modes'][key])))
        for key in sorted(rec['tc3'], key=L3._fmt):
            print('    N %3d  tc3 %-66s prezeroed %s' % (rec['tc3'][key], L3._fmt(key), sorted(rec['tc3_modes'][key])))
        for key in sorted(rec['simt'], key=_simt_fmt):
            print('    N %3d  %-70s prezeroed %s' % (rec['simt'][key], _simt_fmt(key), sorted(rec['simt_modes'][key])))
        for key in sorted(rec['ops'], key=O._fmt):
            print('    ' + O._fmt(key))
    return inv


# ---------------------------------------------------------------------------------------------------
# landmarks
# ---------------------------------------------------------------------------------------------------
def _conv(kind, pred, engine='tc'):
    """A launch of the given kind (fprop / dgrad / wgrad) whose (H, W, Cs, Cin, Cout, R, S, stride[, ...]) satisfies
    pred."""
    field = {'tc': 'tc', 'tc3': 'tc3', 'simt': 'simt'}[engine]
    want = 'simt ' + kind if engine == 'simt' else kind
    return lambda rec: any(k[0] == want and pred(*k[1:9]) for k in rec[field])


def _entry(name, pred=lambda a: True):
    return lambda rec: any(k[0] == name and pred(dict(k[1])) for k in rec['ops'])


def _none(prefix):
    return lambda rec: not any(k[0].startswith(prefix) for k in rec['ops'])


_CIFAR_STEM = lambda H, W, Cs, Cin, Co, R, S, s: (H, W, Cs, Co, R, s) == (32, 32, 4, 64, 3, 1)
_CIFAR_LANDMARKS = [
    ('no max-pool entry (the CIFAR stem has none)', _none('maxpool')),
    ('no fused stem pool', _none('bn_relu_maxpool')),
]
_STRIDED_2X = lambda H, W, Cs, Cin, Co, R, S, s: R == 3 and s == 2 and Co == 2 * Cin
_FROZEN_BACKBONE = [
    # frozen groups run inference-mode BatchNorm: no fused sums, no dgrad, no wgrad below the heads (H = W = 1)
    ('the 224 stem fprop without fused sums', lambda rec: any(
        k[0] == 'fprop' and (k[1], k[3], k[6], k[8]) == (224, 4, 7, 2) and not k[11] for k in rec['tc'])),
    ('no backbone fprop with fused sums', lambda rec: not any(k[0] == 'fprop' and k[1] > 1 and k[11] for k in rec['tc'])),
    ('no backbone dgrad or wgrad', lambda rec: not any(k[0] in ('dgrad', 'wgrad') and k[1] > 1 for k in rec['tc'])),
    ('the unfused max pool', _entry('maxpool3x3s2_fwd')),
]
LANDMARKS = {
    'cifar10_r18_32': _CIFAR_LANDMARKS + [
        ('3x3/1 CIFAR stem on Cs 4 at 32x32 with fused sums', lambda rec: any(
            k[0] == 'fprop' and _CIFAR_STEM(*k[1:9]) and k[11] for k in rec['tc'])),
        ('3x3/1 CIFAR stem wgrad', _conv('wgrad', _CIFAR_STEM)),
        ('64->64 3x3 at 32x32 with fused sums (im2col: the halo kernel refuses 32x32)', lambda rec: any(
            k[0] == 'fprop' and (k[1], k[4], k[5], k[6], k[8]) == (32, 64, 64, 3, 1) and k[11] for k in rec['tc'])),
        ('512-channel 3x3 at 4x4', _conv('fprop', lambda H, W, Cs, Cin, Co, R, S, s: (H, W, Cin, Co, R) == (4, 4, 512, 512, 3))),
        ('strided 3x3 with Cout = 2 Cin', _conv('fprop', _STRIDED_2X)),
        ('strided 3x3 dgrad with Cout = 2 Cin', _conv('dgrad', _STRIDED_2X)),
    ],
    'cifar10_r18_32_tc3': _CIFAR_LANDMARKS + [
        ('3x3/1 CIFAR stem on Cs 4 at 32x32', _conv('fprop', _CIFAR_STEM, 'tc3')),
        ('3x3/1 CIFAR stem wgrad', _conv('wgrad', _CIFAR_STEM, 'tc3')),
        ('512-channel 3x3 at 4x4', _conv('fprop', lambda H, W, Cs, Cin, Co, R, S, s: (H, W, Cin, R) == (4, 4, 512, 3), 'tc3')),
        ('strided 3x3 dgrad with Cout = 2 Cin', _conv('dgrad', _STRIDED_2X, 'tc3')),
    ],
    'cifar10_r18_32_simt': _CIFAR_LANDMARKS + [
        ('3x3/1 CIFAR stem on Cs 4 at 32x32', _conv('fprop', _CIFAR_STEM, 'simt')),
        ('3x3/1 CIFAR stem wgrad', _conv('wgrad', _CIFAR_STEM, 'simt')),
        ('strided 3x3 dgrad with Cout = 2 Cin', _conv('dgrad', _STRIDED_2X, 'simt')),
        ('512-channel 3x3 wgrad at 4x4', _conv('wgrad', lambda H, W, Cs, Cin, Co, R, S, s: (H, Cin, R) == (4, 512, 3), 'simt')),
    ],
    'r18_64': [
        ('7x7/2 stem at 64', _conv('fprop', lambda H, W, Cs, Cin, Co, R, S, s: (H, Cs, Co, R, s) == (64, 4, 64, 7, 2))),
        ('fused stem pool at 32x32', _entry('bn_relu_maxpool_fwd', lambda a: (a['H'], a['W']) == (32, 32))),
        ('3x3 at 2x2', _conv('fprop', lambda H, W, Cs, Cin, Co, R, S, s: (H, W, R) == (2, 2, 3))),
        ('3x3 dgrad at 2x2', _conv('dgrad', lambda H, W, Cs, Cin, Co, R, S, s: (H, W, R) == (2, 2, 3))),
        ('3x3 wgrad at 2x2', _conv('wgrad', lambda H, W, Cs, Cin, Co, R, S, s: (H, W, R) == (2, 2, 3))),
    ],
    'r34_224': [
        ('strided 3x3 with Cout = 2 Cin', _conv('fprop', _STRIDED_2X)),
        ('strided 3x3 dgrad with Cout = 2 Cin', _conv('dgrad', _STRIDED_2X)),
        ('64->64 halo 3x3 at 56x56', _conv('fprop', lambda H, W, Cs, Cin, Co, R, S, s: (H, Cin, Co, R, s) == (56, 64, 64, 3, 1))),
    ],
    'r50_se_224': [
        ('se_scale_fwd', _entry('se_scale_fwd')),
        ('se_scale_bwd_reduce', _entry('se_scale_bwd_reduce')),
        ('se_scale_bwd_apply', _entry('se_scale_bwd_apply')),
        ('SE gate fprop on the CUDA cores at H = W = 1', _conv('fprop', lambda H, W, *r: H == W == 1, 'simt')),
        ('SE gate dgrad on the CUDA cores at H = W = 1', _conv('dgrad', lambda H, W, *r: H == W == 1, 'simt')),
        ('SE gate wgrad on the CUDA cores at H = W = 1', _conv('wgrad', lambda H, W, *r: H == W == 1, 'simt')),
    ],
    'r50_finetune_224': [
        ('sgd_momentum_apply', _entry('sgd_momentum_apply')),
        ('no NT-Xent entry', _none('ntxent')),
        ('softmax_xent at 1000 classes', _entry('softmax_xent', lambda a: a['classes'] == 1000)),
        ('the 224 stem wgrad', _conv('wgrad', lambda H, W, Cs, Cin, Co, R, S, s: (H, Cs, R, s) == (224, 4, 7, 2))),
    ],
    'r50_lineareval_224': _FROZEN_BACKBONE + [
        ('sgd_momentum_apply', _entry('sgd_momentum_apply')),
        ('no NT-Xent entry', _none('ntxent')),
    ],
    'r18_finetune_adam_32': [
        ('adam_apply', _entry('adam_apply')),
        ('no NT-Xent entry', _none('ntxent')),
        ('10-class head wgrad on the CUDA cores', _conv('wgrad', lambda H, W, Cs, Cin, Co, R, S, s: (H, Co) == (1, 10), 'simt')),
        ('10-class head dgrad on the CUDA cores', _conv('dgrad', lambda H, W, Cs, Cin, Co, R, S, s: (H, Co) == (1, 10), 'simt')),
        ('CIFAR stem fprop without fused sums (frozen)', lambda rec: any(
            k[0] == 'fprop' and _CIFAR_STEM(*k[1:9]) and not k[11] for k in rec['tc'])),
    ],
    'r50_eval_224': _FROZEN_BACKBONE + [
        ('no dgrad or wgrad at all', lambda rec: not any(k[0] in ('dgrad', 'wgrad') for k in rec['tc'])),
        ('no fused sums at all', lambda rec: not any(k[0] == 'fprop' and k[11] for k in rec['tc'])),
    ],
}


@pytest.mark.parametrize('family', list(FAMILIES))
def test_inventory_landmarks(inventory, family):
    rec = inventory[family]
    missing = [what for what, check in LANDMARKS[family] if not check(rec)]
    assert not missing, '%s fails its landmarks: %s' % (family, missing)
    prec, eng, mode, classes, cfg = FAMILIES[family]
    if eng == 'tc':
        # the CUDA-core engine runs only the SE gate and an odd-width head (wgmma needs 16-byte rows of dY)
        se = cfg.get('se_ratio', 0) > 0
        stray = [_simt_fmt(k) for k in rec['simt'] if not (k[1] == k[2] == 1 and (se or k[5] == classes == 10))]
        assert not stray, '%s: unexpected CUDA-core convs %s' % (family, stray)
        assert not rec['tc3']
    if mode != 'eval':
        # the step adds every wgrad into the zeroed flat gradient buffer and every fused fprop into the sums pool
        acc = [k for k in rec['tc'] if L.accumulates(k)]
        assert all(rec['tc_modes'][k] == {1} for k in acc), [L._fmt(k) for k in acc if rec['tc_modes'][k] != {1}]
        assert all(rec['tc3_modes'][k] == {1} for k in rec['tc3'] if k[0] == 'wgrad')
    else:
        assert all(m == {0} for m in rec['tc_modes'].values())


def test_every_entry_has_a_replayer(inventory):
    missing = sorted({k[0] for rec in inventory.values() for k in rec['ops'] if k[0] not in ALL_REPLAY})
    assert not missing, 'recorded entries without an fp64 replayer: %s' % missing


# ---------------------------------------------------------------------------------------------------
# replayers for the entries the benchmarked step does not reach
# ---------------------------------------------------------------------------------------------------
# Adam's weight update: m carries 3 roundings (of g - m, the product by 1 - b1 -- exact in fp32 by Sterbenz -- and the
# add: 3u of A_m), v 4 (4u of A_v, and A_v <= 1.003 v for beta2 = 0.999, so v is 4u relative); sqrtf halves that and
# adds one rounding, + eps, the division, the product by lr_t and the final subtraction one each.  Relative to
# A_w = |w| + lr_t A_m / (sqrt(v) + eps): 3u + (2 + 5) u = 10u <= 2^-20 = 16u.
TAU_ADAM = 2.0 ** -20


def _f32(v):
    return float(torch.tensor(v, dtype=F32))


def _slices(n, k, offset):
    """k fp32 tensors of n elements, each with its base `offset` floats past the start of its own buffer."""
    bufs = [torch.empty(n + 4, device='cuda') for _ in range(k)]
    return [b[offset:offset + n] for b in bufs]


def sgd_case(n, momentum, nesterov, chk, seed=0, offset=0, zero_g=False, lr=0.1):
    """One sgd_momentum_apply: v <- m v - lr g; w <- w + (m v - lr g if nesterov else v).  Two or three fp32
    roundings per output (TAU_EW = 8u), relative to the same sums on absolute values."""
    from simclr_b200._lib import lib, stream_ptr
    g_ = O._gen(seed + n + nesterov)
    w, gr, v = _slices(n, 3, offset)
    w.copy_(torch.randn(n, generator=g_, device='cuda') * 0.05)
    gr.copy_(torch.randn(n, generator=g_, device='cuda') * (0.0 if zero_g else 0.01))
    v.copy_(torch.randn(n, generator=g_, device='cuda') * 1e-3)
    w0, g0, v0 = w.double(), gr.double(), v.double()
    hyper = torch.tensor([lr], device='cuda')
    lib.sgd_momentum_apply(w, gr, v, n, hyper, momentum, nesterov, stream_ptr())
    m, lrf = _f32(momentum), _f32(lr)
    v_ref, A_v = m * v0 - lrf * g0, m * v0.abs() + lrf * g0.abs()
    step, A_s = (m * v_ref - lrf * g0, m * A_v + lrf * g0.abs()) if nesterov else (v_ref, A_v)
    chk.close('v', v, v_ref, A_v, 0, TAU_EW)
    chk.close('w', w, w0 + step, w0.abs() + A_s, 0, TAU_EW)
    return n


def adam_case(n, beta1, beta2, eps, chk, seed=0, offset=0, zero_g=False, lr_t=1e-3):
    from simclr_b200._lib import lib, stream_ptr
    g_ = O._gen(seed + n + 1)
    w, gr, m, v = _slices(n, 4, offset)
    w.copy_(torch.randn(n, generator=g_, device='cuda') * 0.05)
    gr.copy_(torch.randn(n, generator=g_, device='cuda') * (0.0 if zero_g else 0.01))
    m.copy_(torch.randn(n, generator=g_, device='cuda') * 1e-3)
    v.copy_(torch.rand(n, generator=g_, device='cuda') * 1e-4)
    w0, g0, m0, v0 = w.double(), gr.double(), m.double(), v.double()
    hyper = torch.tensor([lr_t], device='cuda')
    lib.adam_apply(w, gr, m, v, n, hyper, beta1, beta2, eps, stream_ptr())
    om1, om2, ep, lr = 1.0 - _f32(beta1), 1.0 - _f32(beta2), _f32(eps), _f32(lr_t)
    m_ref, A_m = m0 + (g0 - m0) * om1, m0.abs() + (g0.abs() + m0.abs()) * om1
    v_ref, A_v = v0 + (g0 * g0 - v0) * om2, v0 + (g0 * g0 + v0) * om2
    den = v_ref.sqrt() + ep
    chk.close('m', m, m_ref, A_m, 0, TAU_EW)
    chk.close('v', v, v_ref, A_v, 0, TAU_EW)
    chk.close('w', w, w0 - lr * m_ref / den, w0.abs() + lr * A_m / den, 0, TAU_ADAM)
    return n


def r_sgd_momentum_apply(a, big, pz, chk, seed=0):
    n = O._n_large(a['n']) if big else a['n']
    return sgd_case(n, a['momentum'], a['nesterov'], chk, seed)


def r_adam_apply(a, big, pz, chk, seed=0):
    n = O._n_large(a['n']) if big else a['n']
    return adam_case(n, a['beta1'], a['beta2'], a['eps'], chk, seed)


def se_case(name, N, HW, C, dtype, chk, seed=0):
    """The SE scale kernels against fp64.  g = sigmoid(l) from expf (2 ulp), an add and a division: 4u relative.
      fwd        out = x g: one more rounding; rho of the storage type, TAU_EW of |out|.
      bwd_reduce dl = g (1 - g) sum_hw dout x: the sum is sequential (tau_seq(HW)); 1 - g cancels when g -> 1, so
                 g's 4u error is carried as 4u g |sum| and A = g sum_hw |dout x| (two products: TAU_EW covers it).
      bwd_apply  dx = fma(dout, g, dmean * (1 / HW)): 5 roundings of A = |dout| g + |dmean| / HW.  dmean is the
                 gradient of a mean over HW pixels, so it is drawn at HW times the scale of dout, as in the step."""
    from simclr_b200._lib import lib, stream_ptr
    dt = DT[dtype]
    g_ = O._gen(seed + N + HW + C)
    x = O._randn((N, HW, C), dt, g_)
    l = torch.randn(N, C, generator=g_, device='cuda') * 2.0
    sig = torch.sigmoid(l.double()).view(N, 1, C)
    x64 = x.double()
    if name == 'se_scale_fwd':
        out = O._nan((N, HW, C), dt)
        lib.se_scale_fwd(x, l, out, dtype, N, HW, C, stream_ptr())
        ref = x64 * sig
        chk.close('out', out, ref, ref.abs(), RHO[dt], TAU_EW)
    elif name == 'se_scale_bwd_reduce':
        dout = O._randn((N, HW, C), dt, g_)
        dl = O._nan((N, C), F32)
        lib.se_scale_bwd_reduce(dout, x, l, dl, dtype, N, HW, C, stream_ptr())
        p = dout.double() * x64
        s = sig.view(N, C)
        chk.close('dlogits', dl, p.sum(1) * s * (1 - s), p.abs().sum(1) * s, 0, tau_seq(HW) + TAU_EW)
    else:
        dout = O._randn((N, HW, C), dt, g_)
        dmean = torch.randn(N, C, generator=g_, device='cuda') * HW
        dx = O._nan((N, HW, C), dt)
        lib.se_scale_bwd_apply(dout, l, dmean, dx, dtype, N, HW, C, stream_ptr())
        d64, dm = dout.double(), dmean.double().view(N, 1, C)
        chk.close('dx', dx, d64 * sig + dm / HW, d64.abs() * sig + dm.abs() / HW, RHO[dt], TAU_EW)
    return N


def _r_se(name):
    def replay(a, big, pz, chk, seed=0):
        N = O._large_n(a['N'], a['HW'] * a['C']) if big else a['N']
        return se_case(name, N, a['HW'], a['C'], a['dtype'], chk, seed)
    return replay


NEW_REPLAY = {
    'sgd_momentum_apply': r_sgd_momentum_apply,
    'adam_apply': r_adam_apply,
    'se_scale_fwd': _r_se('se_scale_fwd'),
    'se_scale_bwd_reduce': _r_se('se_scale_bwd_reduce'),
    'se_scale_bwd_apply': _r_se('se_scale_bwd_apply'),
}
ALL_REPLAY = dict(O.REPLAY, **NEW_REPLAY)


# ---------------------------------------------------------------------------------------------------
# the CUDA-core fp32 engine
# ---------------------------------------------------------------------------------------------------
def _simt_wgrad_splits(key, N, sms):
    """(splits, pixels per split) of conv_simt.cu's wgrad launch."""
    kind, H, W, Cs, Cin, Cout, R, S, s = key[:9]
    M = N * ((H - 1) // s + 1) * ((W - 1) // s + 1)
    bx = (R * S * Cin * Cout + 255) // 256
    splits = max(1, min((4 * sms + bx - 1) // bx, M, 1024))
    mps = (M + splits - 1) // splits
    return (M + mps - 1) // mps, mps


def check_simt(key, N, pz=0, seed=0):
    """One CUDA-core conv launch against fp64: [(mode, ratio, where)].  One thread per output, sequential fp32 FMAs
    of bf16 or fp32 operands by the fp32 master weights, so fprop and dgrad err by at most tau_seq(K) A, with K the
    taps times channels of the reduction.  The wgrad splits the M pixels over `splits` blocks of m_per_split each;
    each block's sequential sum errs by tau_seq(m_per_split) of its own A (<= A), and the blocks are added with fp32
    atomics into the zeroed dW: the running sum stays below A, so each of the `splits` adds rounds by at most u A.
    tau = tau_seq(m_per_split) + splits u.  A dropped term (1 / K of A) stays above these up to K = 2^15."""
    from simclr_b200._lib import lib, stream_ptr, DTYPE_CODE
    kind, H, W, Cs, Cin, Cout, R, S, s, din, dout = key
    Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
    g = torch.Generator(device='cuda').manual_seed(seed + sum(v for v in key if type(v) is int))
    x = torch.randn(N, H, W, Cin, generator=g, device='cuda').to(din)
    w = torch.randn(R, S, Cin, Cout, generator=g, device='cuda') * (1.0 / (R * S * Cin) ** 0.5)
    dy = torch.randn(N, Ho, Wo, Cout, generator=g, device='cuda').to(din)
    xs = L3._pad_cs(x, Cs)
    x64, w64, dy64 = x.double(), w.double(), dy.double()
    st = stream_ptr()
    guards = ()
    prev = lib.set_accumulate_prezeroed(pz)
    try:
        if kind == 'simt fprop':
            got = O._nan((N, Ho, Wo, Cout), dout)
            lib.conv2d_fprop_simt(xs, w, got, DTYPE_CODE[din], DTYPE_CODE[dout], N, H, W, Cs, Cin, Cout, R, S, s, st)
            ref, A = conv_reference(x64, w64, R, s), conv_reference(x64.abs(), w64.abs(), R, s)
            tau = tau_seq(R * S * Cin)
        elif kind == 'simt dgrad':
            got = O._nan((N, H, W, Cin), dout)
            lib.conv2d_dgrad_simt(dy, w, got, DTYPE_CODE[din], DTYPE_CODE[dout], N, H, W, Cin, Cout, R, S, s, st)
            ref = L._ref_dx(dy64, w64, R, s, (N, H, W, Cin))
            A = L._ref_dx(dy64.abs(), w64.abs(), R, s, (N, H, W, Cin))
            tau = tau_seq(R * S * Cout)
        else:
            got, guards = L3._out_buf((R, S, Cin, Cout), 'wgrad', pz)
            lib.conv2d_wgrad_simt(xs, dy, got, DTYPE_CODE[din], N, H, W, Cs, Cin, Cout, R, S, s, st)
            ref = L._ref_dw(x64, dy64, R, s, (R, S, Cin, Cout))
            A = L._ref_dw(x64.abs(), dy64.abs(), R, s, (R, S, Cin, Cout))
            splits, mps = _simt_wgrad_splits(key, N, L3._sms())
            tau = tau_seq(mps) + splits * U
    finally:
        lib.set_accumulate_prezeroed(prev)
    torch.cuda.synchronize()
    ratio, where = L._ratio(got, ref, A, RHO[dout], tau)
    if not all(bool(torch.isnan(gd).all()) for gd in guards):
        ratio, where = math.inf, 'NaN guard of the flat buffer overwritten'
    return ratio, where


def _simt_large_n(key, N):
    kind, H, W, Cs, Cin, Cout, R, S, s = key[:9]
    rows = ((H - 1) // s + 1) * ((W - 1) // s + 1)
    n = max(N + 1, min(SIMT_VIEWS, int(MACS_BUDGET // (rows * R * S * Cin * Cout))))
    return n


# ---------------------------------------------------------------------------------------------------
# replay of the inventory: each distinct launch once, by the first family that records it
# ---------------------------------------------------------------------------------------------------
def _owned(inventory, family, field):
    """[(key, largest N over the families, union of modes)] of the launches `family` is the first to record."""
    earlier = set()
    for fam in FAMILIES:
        if fam == family:
            break
        earlier |= set(inventory[fam][field])
    out = []
    for key in inventory[family][field]:
        if key in earlier:
            continue
        N = max(rec[field].get(key, 0) for rec in inventory.values())
        modes = set().union(*(rec[field + '_modes'].get(key, set()) for rec in inventory.values()))
        out.append((key, N, modes))
    return out


def _report_simt(items, what):
    bad, worst = [], 0.0
    t0 = time.time()
    for key, N, pz in items:
        ratio, where = check_simt(key, N, pz)
        worst = max(worst, ratio)
        print('    %-70s N %4d  pz %d  worst |err|/bound %.3f at %s' % (_simt_fmt(key), N, pz, ratio, where))
        if not ratio <= 1.0:
            bad.append((_simt_fmt(key), N, pz, ratio, where))
    print('%s: %d launches, worst |err|/bound = %.3f (tau = tau_seq(K)), %.1f s' % (what, len(items), worst, time.time() - t0))
    assert not bad, bad


@pytest.mark.parametrize('size', ['recorded', 'large'])
@pytest.mark.parametrize('family', list(FAMILIES))
def test_launches_vs_fp64(inventory, family, size):
    """Every distinct launch the family is the first to record, per element against fp64: the bf16 tc convs in each
    pre-zeroed mode the step ran them in (and with the mode off), the tc3 convs pass by pass in both modes and end to
    end, the CUDA-core convs, and every other entry (again in pre-zeroed mode where the step issued it so)."""
    big = size == 'large'
    sms = L3._sms()
    ran = 0
    tc = sorted(_owned(inventory, family, 'tc'), key=lambda t: L._fmt(t[0]))
    if big:
        tc = [(k, L._large_n(k, n, sms), m) for k, n, m in tc]
        tc = [(k, n, m) for k, n, m in tc if n is not None]
    if tc:
        L._run_launches([(k, n, pz) for k, n, m in tc for pz in L.replay_modes(k, m)],
                        '%s tc at the %s batch' % (family, size))
        ran += len(tc)
    tc3 = sorted(_owned(inventory, family, 'tc3'), key=lambda t: L3._fmt(t[0]))
    if big:
        tc3 = [(k, L3._large_n(k, n, sms)) for k, n, _ in tc3]
        tc3 = [(k, n) for k, n in tc3 if n is not None]
    else:
        tc3 = [(k, n) for k, n, _ in tc3]
    if tc3:
        L3._report(tc3, L3.check_passes, '%s tc3 pass structure at the %s batch' % (family, size), L.TAU)
        if not big:
            L3._report(tc3, lambda k, n: L3.check_end_to_end(k, n, False), '%s tc3 end to end' % family, L3.TAU_E2E)
        ran += len(tc3)
    simt = sorted(_owned(inventory, family, 'simt'), key=lambda t: _simt_fmt(t[0]))
    if simt:
        _report_simt([(k, _simt_large_n(k, n) if big else n, pz) for k, n, m in simt for pz in sorted(m | {0})],
                     '%s CUDA-core convs at the %s batch' % (family, size))
        ran += len(simt)
    earlier = set()
    for fam in FAMILIES:
        if fam == family:
            break
        earlier |= inventory[fam]['ops']
    items, seen = [], set()
    for key in sorted(inventory[family]['ops'] - earlier, key=O._fmt):
        name, it, pz = key
        if name not in ALL_REPLAY or (big and name in O.NO_LARGE):
            continue
        a = dict(it)
        if name in ('ntxent_forward', 'ntxent_backward'):      # one replay covers both
            dedup = ('ntxent', a['B'], a['R'], a['D'], a['temperature'])
            if dedup in seen:
                continue
            seen.add(dedup)
        items.append((O._fmt(key), ALL_REPLAY[name], a, big, 0))
        if pz:
            items.append((O._fmt(key) + ' [into a pre-zeroed slice]', ALL_REPLAY[name], a, big, 1))
    if items:
        O._run_replays(items, '%s other entries at the %s size' % (family, size))
        ran += len(items)
    if not ran:
        pytest.skip('every launch of %s is replayed by an earlier family' % family)


# ---------------------------------------------------------------------------------------------------
# hand-picked edges beyond the inventory
# ---------------------------------------------------------------------------------------------------
def _tc(kind, H, W, Cs, Cin, Cout, k, s, fused=False):
    return L._k(kind, H, W, Cs, Cin, Cout, k, s, F32 if kind == 'wgrad' else BF16, fused)


# the CIFAR stem (3x3/1 on 4 stored channels: never pixel pairs) at even and odd extents, 64 and 128 outputs
_STEM_HW = [((32, 32), 2), ((31, 33), 2), ((33, 31), 2), ((7, 9), 4)]
TC_EDGES = [(_tc('fprop', H, W, 4, 3, co, 3, 1, fu), n) for (H, W), n in _STEM_HW for co in (64, 128) for fu in (True, False)]
TC_EDGES += [(_tc('wgrad', H, W, 4, 3, co, 3, 1), n) for (H, W), n in _STEM_HW for co in (64, 128)]
# 3x3 at 1x1, 2x2 and 3x3, stride 1 and 2, 512 channels: one 128-row tile spans many images; at 1x1 only the centre
# tap is real
TC_EDGES += [(_tc(kind, H, H, 512, 512, 512, 3, s, kind == 'fprop'), 40)
             for H in (1, 2, 3) for s in (1, 2) for kind in ('fprop', 'dgrad', 'wgrad')]
# basic-block strided 3x3 with Cout = 2 Cin at 5 -> 3 and 3 -> 2
TC_EDGES += [(_tc(kind, H, H, 256, 256, 512, 3, 2, kind == 'fprop'), 8) for H in (5, 3) for kind in ('fprop', 'dgrad', 'wgrad')]
# the halo and 7x7 stem kernels without fused sums (eval, frozen groups): halo at H = 55, stem at 64 and 224
TC_EDGES += [(_tc('fprop', 55, 56, c, c, c, 3, 1), 2) for c in (64, 128)]
TC_EDGES += [(_tc('fprop', 64, 64, 4, 3, 64, 7, 2), 4), (_tc('fprop', 224, 224, 4, 3, 64, 7, 2), 2),
             (_tc('fprop', 224, 224, 4, 3, 128, 7, 2), 2)]


@pytest.mark.parametrize('key,N', TC_EDGES, ids=[L._fmt(k).replace(' ', '') + '-N%d' % n for k, n in TC_EDGES])
def test_tc_edge_vs_fp64(key, N):
    L._run_launches([(key, N, pz) for pz in L.replay_modes(key, (1,))], 'tc edge')


TC3_EDGES = [(L3._k(kind, H, W, 4, 3, co, 3, 1), n) for (H, W), n in _STEM_HW for co in (64, 128) for kind in ('fprop', 'wgrad')]
TC3_EDGES += [(L3._k(kind, H, H, 512, 512, 512, 3, s), 40) for H in (1, 2, 3) for s in (1, 2) for kind in ('fprop', 'dgrad', 'wgrad')]
TC3_EDGES += [(L3._k(kind, H, H, 256, 256, 512, 3, 2), 8) for H in (5, 3) for kind in ('fprop', 'dgrad', 'wgrad')]


@pytest.mark.parametrize('key,N', TC3_EDGES, ids=[L3._fmt(k).replace(' ', '') + '-N%d' % n for k, n in TC3_EDGES])
def test_tc3_edge_vs_fp64(key, N):
    L3._report([(key, N)], L3.check_passes, 'tc3 edge, pass structure', L.TAU)
    L3._report([(key, N)], lambda k, n: L3.check_end_to_end(k, n, False), 'tc3 edge, end to end', L3.TAU_E2E)


R50_PARAMS = 25_557_032              # ResNet-50 with its 1000-class head: 25.6 M parameters


def _optim_items():
    items = []
    for n in (1, 3, 4097, R50_PARAMS):
        for off in (0, 1):
            for zg in (False, True):
                tag = 'n %d offset %d zero grad %d' % (n, 4 * off, zg)
                for nest in (0, 1):
                    items.append(('sgd_momentum_apply nesterov %d %s' % (nest, tag),
                                  lambda a, big, pz, chk, n=n, nest=nest, off=off, zg=zg:
                                  sgd_case(n, 0.9, nest, chk, offset=off, zero_g=zg), {}, False, 0))
                items.append(('adam_apply %s' % tag, lambda a, big, pz, chk, n=n, off=off, zg=zg:
                              adam_case(n, 0.9, 0.999, 1e-7, chk, offset=off, zero_g=zg), {}, False, 0))
    return items


def test_optimizers_edges_vs_fp64():
    """sgd_momentum_apply (nesterov 0 and 1) and adam_apply at n = 1, 3, 4k+1 and ResNet-50's 25.6 M parameters (the
    grid-stride loop of a capped grid), with zero gradients and with every base one float past a 16-byte boundary."""
    O._run_replays(_optim_items(), 'optimizer edges')


@pytest.mark.parametrize('dtype', [1, 0], ids=['bf16', 'fp32'])
@pytest.mark.parametrize('C', [64, 2048])
def test_se_scale_edges_vs_fp64(C, dtype):
    items = [('%s HW %d C %d dtype %d' % (name, HW, C, dtype),
              lambda a, big, pz, chk, name=name, HW=HW: se_case(name, 2, HW, C, dtype, chk), {}, False, 0)
             for HW in (1, 16, 49, 3136) for name in ('se_scale_fwd', 'se_scale_bwd_reduce', 'se_scale_bwd_apply')]
    O._run_replays(items, 'SE scale at C %d' % C)
