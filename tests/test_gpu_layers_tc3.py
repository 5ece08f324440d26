"""Every split-bf16 (`tc3`) conv launch of the fp32 step against an fp64 reference, element by element and pass by
pass, and bitwise reproducibility of the fp32 / tc3 training step.

The `tc3` engine (`--b200_precision=fp32 --b200_conv_engine=tc3`, bench.py's `fp32_accurate_tensor_core_mode`)
splits every fp32 operand three ways, v = v0 + v1 + v2 (`simclr_split_bf16x3`, `simclr_pack_conv_weight_part`),
and runs six bf16 GEMMs -- the pairs (0,0) (0,1) (1,0) (1,1) (0,2) (2,0) -- summed in fp32 into one output
(TMA reduce-add, or atomics where an fp32 row is not 16 bytes; dW accumulates into the step's pre-zeroed gradient
buffer).  The inventory is taken from the model, as in test_gpu_layers.py: one eager fp32 / tc3 step per
benchmarked family at 2 samples, with the tc3 convs, the CUDA-core convs, the split and the weight packing wrapped
to record every launch and the pre-zeroed mode it ran in.

Pass-structure replay: each launch runs on six INDEPENDENT seeded bf16 tensors of equal scale (x0, x1, x2 and w0,
w1, w2, or dy0, dy1, dy2), not on the parts of a split.  The reference is the sum of the six pair convolutions in
fp64; products of bf16 values are exact in fp32, so fp32 accumulation (and five reduce-add roundings, 5 * 2^-24 A)
is the only error:

    |got - ref| <= rho * |ref| + tau * A,   rho = 0, tau = test_gpu_layers.TAU = 2^-17

with A the same sum on absolute values.  Every part has full size, so a dropped, doubled or swapped pass, or an
excluded pair such as (1,2) taken in, moves an output by O(A / sqrt(K)): orders above tau at every K of the step.
A real split would hide this -- its v1 and v2 parts are 2^-9 and 2^-17 of v0.

End-to-end replay: the same launches on unrounded fp32 operands through the real split and packing, against the
fp64 conv of the fp32 values.  Operand preparation is checked bit for bit against a torch restatement.
"""
import math
import time
import types

import pytest
import torch

from test_gpu_kernels import conv_reference
from test_gpu_layers import _ratio, _ref_dw, _ref_dx, _snapshot, TAU
from test_gpu_ops import tau_seq
from test_gpu_tc import _pack

pytestmark = pytest.mark.gpu

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
U = 2.0 ** -24                       # unit roundoff of fp32
# End to end: the fp32 accumulation allowance of the pass replay (TAU), plus the three products the split drops
# (a1 b2, a2 b1, a2 b2: each part is at most 2^-9 of the one before, so each is at most 2^-26 |a b|; 3 * 2^-24 A
# bounds them with room), plus five fp32 reduce-add roundings of partial sums no larger than A (5 * 2^-24 A).
TAU_E2E = TAU + (3 + 5) * U
MACS_BUDGET = 4e10                  # multiply-adds per fp64 reference conv at the large batch
BENCH_VIEWS = 128                    # bench.py's fp32 / tc3 secondary run: 64 samples, two views
GUARD = 64                           # NaN floats on each side of a dW slice of the flat gradient buffer (256 bytes)

FAMILIES = {
    'r50_1x_224': dict(resnet_depth=50, width_multiplier=1, image_size=224, sk_ratio=0.0),
    'r50_2x_224': dict(resnet_depth=50, width_multiplier=2, image_size=224, sk_ratio=0.0),
    'r50_2x_sk_224': dict(resnet_depth=50, width_multiplier=2, image_size=224, sk_ratio=0.0625),
}

TC3 = ('conv2d_fprop_tc3', 'conv2d_dgrad_tc3', 'conv2d_wgrad_tc3')
SIMT = ('conv2d_fprop_simt', 'conv2d_dgrad_simt', 'conv2d_wgrad_simt')


def tau_spread(K):
    """End-to-end allowance for operands whose magnitudes are spread over 2^+-20.  A few products then carry most of
    A, so the running fp32 sum sits near A from the first large term on, and each of the K accumulation steps rounds
    by up to 2^-24 A with random sign: the error grows like sqrt(K) u A (measured on an H100 up to 1.8 sqrt(K) u A at
    K = 18432, above TAU).  test_gpu_ops.tau_seq(K) = 8 sqrt(K) u takes the place of TAU.  At the step's K this is up
    to ~2^-14 A, far above any term of the v2 parts: this replay checks the range of the split and packing (no
    overflow, underflow or lost exponent across 2^40), not v2 itself.  The v2 parts are checked bit for bit by
    test_split_* and test_pack_parts_bit_exact, and their place in the six passes by the pass-structure replay."""
    return max(TAU, tau_seq(K)) + (3 + 5) * U


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _conv_key(name, a):
    """(kind, H, W, Cs, Cin, Cout, R, S, stride), N and whether the output is 16-byte aligned, of one conv call."""
    if name == 'conv2d_fprop_tc3':
        out, (N, H, W, Cs, Cout, R, S, s) = a[6], a[7:15]
        Cin = 3 if Cs == 4 else Cs               # the stem stores its 3 image channels as 4
        return ('fprop', H, W, Cs, Cin, Cout, R, S, s), N, out
    if name == 'conv2d_dgrad_tc3':
        out, (N, H, W, Cin, Cout, R, S, s) = a[6], a[7:15]
        return ('dgrad', H, W, Cin, Cin, Cout, R, S, s), N, out
    if name == 'conv2d_wgrad_tc3':
        out, (N, H, W, Cs, Cin, Cout, R, S, s) = a[6], a[7:16]
        return ('wgrad', H, W, Cs, Cin, Cout, R, S, s), N, out
    if name == 'conv2d_fprop_simt':
        out, (N, H, W, Cs, Cin, Cout, R, S, s) = a[2], a[5:14]
        return ('simt fprop', H, W, Cs, Cin, Cout, R, S, s), N, out
    if name == 'conv2d_dgrad_simt':
        out, (N, H, W, Cin, Cout, R, S, s) = a[2], a[5:13]
        return ('simt dgrad', H, W, Cin, Cin, Cout, R, S, s), N, out
    out, (N, H, W, Cs, Cin, Cout, R, S, s) = a[2], a[4:13]
    return ('simt wgrad', H, W, Cs, Cin, Cout, R, S, s), N, out


def _fmt(key):
    kind, H, W, Cs, Cin, Cout, R, S, s = key
    return '%s %3dx%-3d Cs %4d Cin %4d Cout %4d %dx%d/%d' % (kind, H, W, Cs, Cin, Cout, R, S, s)


@pytest.fixture(scope='module')
def inventory():
    """{family: dict(convs={key: N}, prezeroed={key: set of modes}, aligned={key: bool}, splits={numel},
    packs={(R, S, Cin, Cs, Cout, Kp, has_wd): set of parts})} of one eager fp32 / tc3 step per family."""
    from simclr_b200 import engine, run, flags_def
    from simclr_b200._lib import lib
    F = flags_def.FLAGS
    if not F.is_parsed():
        F(['test'])
    saved = {k: getattr(F, k) for k in flags_def.REFERENCE_FLAG_NAMES + ['b200_precision', 'b200_conv_engine']}
    inv = {}
    try:
        for fam, cfg in FAMILIES.items():
            B, S = 2, cfg['image_size']
            flags_def.set_flags(train_batch_size=B, use_blur=True, optimizer='lars', weight_decay=1e-4,
                                b200_precision='fp32', b200_conv_engine='tc3', **cfg)
            engine.set_engine(engine.Engine(precision='fp32', conv_engine='tc3'))
            trainer = run.Trainer(num_classes=1000, num_examples=50000, seed=0)
            g = torch.Generator().manual_seed(3)
            f = torch.rand(B, S, S, 6, generator=g).cuda()
            lab = torch.nn.functional.one_hot(torch.randint(0, 1000, (B,), generator=g), 1000).float().cuda()
            rec = dict(convs={}, prezeroed={}, aligned={}, splits=set(), packs={})
            state = {'pz': 0}
            with pytest.MonkeyPatch.context() as mp:
                setpz = getattr(lib, 'set_accumulate_prezeroed')

                def wrap_pz(on, _fn=setpz):
                    state['pz'] = int(on)
                    return _fn(on)
                mp.setattr(lib, 'set_accumulate_prezeroed', wrap_pz)
                for name in TC3 + SIMT:
                    fn = getattr(lib, name)             # _Lib.__getattr__ caches the bound call on the instance

                    def wrap(*a, _fn=fn, _name=name):
                        key, N, out = _conv_key(_name, a)
                        rec['convs'][key] = max(N, rec['convs'].get(key, 0))
                        rec['prezeroed'].setdefault(key, set()).add(state['pz'])
                        rec['aligned'][key] = rec['aligned'].get(key, True) and out.data_ptr() % 16 == 0
                        return _fn(*a)
                    mp.setattr(lib, name, wrap)
                split = getattr(lib, 'split_bf16x3')

                def wrap_split(x, a, b, c, n, st, _fn=split):
                    rec['splits'].add(int(n))
                    return _fn(x, a, b, c, n, st)
                mp.setattr(lib, 'split_bf16x3', wrap_split)
                pack = getattr(lib, 'pack_conv_weight_part')

                def wrap_pack(w, wf, wd, part, R, S, Cin, Cs, Cout, Kp, st, _fn=pack):
                    rec['packs'].setdefault((R, S, Cin, Cs, Cout, Kp, wd is not None), set()).add(part)
                    return _fn(w, wf, wd, part, R, S, Cin, Cs, Cout, Kp, st)
                mp.setattr(lib, 'pack_conv_weight_part', wrap_pack)
                trainer.single_step(f, lab)
                torch.cuda.synchronize()
            inv[fam] = rec
            del trainer
            torch.cuda.empty_cache()
    finally:
        for k, v in saved.items():
            setattr(F, k, v)
        lib.set_accumulate_prezeroed(0)
    for fam, rec in inv.items():
        print('\n%s: %d distinct conv launches, %d split sizes, %d packed layers' % (
            fam, len(rec['convs']), len(rec['splits']), len(rec['packs'])))
        for key in sorted(rec['convs'], key=_fmt):
            print('    N %3d  %-62s prezeroed %s%s' % (rec['convs'][key], _fmt(key), sorted(rec['prezeroed'][key]),
                                                     '' if rec['aligned'][key] else '  unaligned output'))
        print('    split sizes: %s' % sorted(rec['splits']))
    return inv


def _has(convs, kind, pred):
    return any(k[0] == kind and pred(*k[1:]) for k in convs)


# what the networks must keep launching: the shapes that take the stem, halo and strided paths, and the heads
_STEM = lambda cout: (lambda H, W, Cs, Cin, Co, R, S, s: (H, Cs, Co, R, s) == (224, 4, cout, 7, 2))
LANDMARKS = {
    'r50_1x_224': [
        ('7x7/2 stem at 224, 64 outputs', 'fprop', _STEM(64)),
        ('7x7/2 stem wgrad at 224, 64 outputs (stem7x7_wgrad)', 'wgrad', _STEM(64)),
        ('64->64 halo 3x3 wgrad at 56x56', 'wgrad', lambda H, W, Cs, Cin, Co, R, S, s: (H, W, Cin, Co, R, s) == (56, 56, 64, 64, 3, 1)),
        ('strided 3x3 dgrad', 'dgrad', lambda H, W, Cs, Cin, Co, R, S, s: R == 3 and s == 2),
        ('strided 1x1 dgrad', 'dgrad', lambda H, W, Cs, Cin, Co, R, S, s: R == 1 and s == 2),
        ('2048-deep head dense fprop', 'fprop', lambda H, W, Cs, Cin, Co, R, S, s: (H, W, Cin) == (1, 1, 2048) and Co != 1000),
        ('2048-deep head dense wgrad', 'wgrad', lambda H, W, Cs, Cin, Co, R, S, s: (H, W, Cin) == (1, 1, 2048) and Co != 1000),
        ('2048-deep head dense dgrad', 'dgrad', lambda H, W, Cs, Cin, Co, R, S, s: (H, W, Cin) == (1, 1, 2048)),
        ('1000-class supervised head fprop', 'fprop', lambda H, W, Cs, Cin, Co, R, S, s: (H, W, Co) == (1, 1, 1000)),
        ('1000-class supervised head wgrad', 'wgrad', lambda H, W, Cs, Cin, Co, R, S, s: (H, W, Co) == (1, 1, 1000)),
    ],
    'r50_2x_224': [
        ('7x7/2 stem at 224, 128 outputs', 'fprop', _STEM(128)),
        ('7x7/2 stem wgrad at 224, 128 outputs', 'wgrad', _STEM(128)),
        ('strided 3x3 dgrad', 'dgrad', lambda H, W, Cs, Cin, Co, R, S, s: R == 3 and s == 2),
        ('strided 1x1 dgrad', 'dgrad', lambda H, W, Cs, Cin, Co, R, S, s: R == 1 and s == 2),
        ('1000-class supervised head fprop', 'fprop', lambda H, W, Cs, Cin, Co, R, S, s: (H, W, Co) == (1, 1, 1000)),
    ],
    'r50_2x_sk_224': [
        ('ResNet-D 3x3/2 stem on 4 stored channels', 'fprop', lambda H, W, Cs, Cin, Co, R, S, s: (H, Cs, R, s) == (224, 4, 3, 2)),
        ('ResNet-D 3x3/2 stem wgrad', 'wgrad', lambda H, W, Cs, Cin, Co, R, S, s: (H, Cs, R, s) == (224, 4, 3, 2)),
        ('SK 1x1 mixing dense fprop', 'fprop', lambda H, W, Cs, Cin, Co, R, S, s: (H, W, R) == (1, 1, 1) and Co in (32, 64)),
        ('SK 1x1 mixing dense back to 2f streams', 'fprop',
         lambda H, W, Cs, Cin, Co, R, S, s: (H, W, R) == (1, 1, 1) and Cin in (32, 64) and Co >= 256),
        ('SK 1x1 mixing dense wgrad', 'wgrad', lambda H, W, Cs, Cin, Co, R, S, s: (H, W, R) == (1, 1, 1) and Co in (32, 64)),
        ('1000-class supervised head fprop', 'fprop', lambda H, W, Cs, Cin, Co, R, S, s: (H, W, Co) == (1, 1, 1000)),
    ],
}


@pytest.mark.parametrize('family', list(FAMILIES))
def test_inventory_landmarks(inventory, family):
    rec = inventory[family]
    convs = rec['convs']
    missing = [what for what, kind, pred in LANDMARKS[family] if not _has(convs, kind, pred)]
    assert not missing, '%s no longer launches: %s' % (family, missing)
    # at 1000 classes every conv and dense layer of the tc3 step runs on the tensor cores: a silent fall-back to the
    # CUDA-core engine would leave those layers outside everything this file checks
    simt = [_fmt(k) for k in convs if k[0].startswith('simt')]
    assert not simt, '%s: CUDA-core convs in the tc3 step: %s' % (family, simt)
    # every dW is accumulated into the step's pre-zeroed flat gradient buffer, 16-byte aligned
    wg = [k for k in convs if k[0] == 'wgrad']
    assert wg
    assert all(rec['prezeroed'][k] == {1} for k in wg), [(_fmt(k), rec['prezeroed'][k]) for k in wg]
    assert all(rec['aligned'][k] for k in convs), [_fmt(k) for k in convs if not rec['aligned'][k]]
    # every weight is packed as three parts
    assert all(p == {0, 1, 2} for p in rec['packs'].values()), rec['packs']


# ---------------------------------------------------------------------------------------------------
# replay of one launch
# ---------------------------------------------------------------------------------------------------
def _out_buf(shape, kind, pz):
    """NaN-filled output.  A wgrad in pre-zeroed mode gets a zeroed slice of a NaN-filled flat buffer, as the step
    hands out dW; returns (out, guards) where guards are the NaN borders that must survive."""
    if kind == 'wgrad' and pz:
        n = math.prod(shape)
        flat = torch.full((GUARD + n + GUARD,), float('nan'), dtype=F32, device='cuda')
        flat[GUARD:GUARD + n].zero_()
        return flat[GUARD:GUARD + n].view(shape), (flat[:GUARD], flat[GUARD + n:])
    return torch.full(shape, float('nan'), dtype=F32, device='cuda'), ()


def _pad_cs(x, Cs):
    N, H, W, Cin = x.shape
    if Cs == Cin:
        return x.contiguous()
    return torch.cat([x, torch.zeros(N, H, W, Cs - Cin, dtype=x.dtype, device=x.device)], -1).contiguous()


def _pair_ref(kind, a, b, key, N):
    """sum over the pairs (0,0) (0,1) (1,0) (1,1) (0,2) (2,0) of the fp64 op on (a_i, b_j), and the same on
    absolute values.  By bilinearity: op(a0, b0 + b1 + b2) + op(a1, b0 + b1) + op(a2, b0)."""
    _, H, W, Cs, Cin, Cout, R, S, s = key

    def op(u, v):
        if kind == 'fprop':
            return conv_reference(u, v, R, s)                       # x, w
        if kind == 'dgrad':
            return _ref_dx(u, v, R, s, (N, H, W, Cin))               # dy, w
        return _ref_dw(u, v, R, s, (R, S, Cin, Cout))                # x, dy
    a64 = [t.double() for t in a]
    b64 = [t.double() for t in b]
    ref = op(a64[0], b64[0] + b64[1] + b64[2]) + op(a64[1], b64[0] + b64[1]) + op(a64[2], b64[0])
    aa = [t.abs() for t in a64]
    ba = [t.abs() for t in b64]
    A = op(aa[0], ba[0] + ba[1] + ba[2]) + op(aa[1], ba[0] + ba[1]) + op(aa[2], ba[0])
    return ref, A


def _call_tc3(kind, key, N, a, b, out):
    """a, b: three bf16 parts each (x / dy / x and w / w / dy), b already packed for fprop and dgrad."""
    from simclr_b200._lib import lib, stream_ptr
    _, H, W, Cs, Cin, Cout, R, S, s = key
    st = stream_ptr()
    if kind == 'fprop':
        lib.conv2d_fprop_tc3(a[0], a[1], a[2], b[0], b[1], b[2], out, N, H, W, Cs, Cout, R, S, s, st)
    elif kind == 'dgrad':
        lib.conv2d_dgrad_tc3(a[0], a[1], a[2], b[0], b[1], b[2], out, N, H, W, Cin, Cout, R, S, s, st)
    else:
        lib.conv2d_wgrad_tc3(a[0], a[1], a[2], b[0], b[1], b[2], out, N, H, W, Cs, Cin, Cout, R, S, s, st)


def _run_modes(key, N, a, b, ref, A, tau):
    """Runs the launch with set_accumulate_prezeroed(0) and as the step issues it (1).  Returns [(mode, ratio,
    where)]; an overwritten NaN guard is an infinite ratio."""
    from simclr_b200._lib import lib
    kind, H, W, Cs, Cin, Cout, R, S, s = key
    shape = tuple(ref.shape)
    res = []
    for pz in (0, 1):
        out, guards = _out_buf(shape, kind, pz)
        prev = lib.set_accumulate_prezeroed(pz)
        try:
            _call_tc3(kind, key, N, a, b, out)
        finally:
            lib.set_accumulate_prezeroed(prev)
        torch.cuda.synchronize()
        ratio, where = _ratio(out, ref, A, 0.0, tau)
        if not all(bool(torch.isnan(gd).all()) for gd in guards):
            ratio, where = math.inf, 'NaN guard of the flat buffer overwritten'
        res.append((pz, ratio, where))
    return res


def _bf16_operands(key, N, seed):
    """Six independent seeded bf16 tensors of equal scale per operand: a (x, dy or x) and b (w, w or dy)."""
    kind, H, W, Cs, Cin, Cout, R, S, s = key
    Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
    g = torch.Generator(device='cuda').manual_seed(seed + sum(v for v in key if type(v) is int))
    x = lambda: torch.randn(N, H, W, Cin, generator=g, device='cuda').to(BF16)
    w = lambda: (torch.randn(R, S, Cin, Cout, generator=g, device='cuda') * (1.0 / (R * S * Cin) ** 0.5)).to(BF16)
    dy = lambda: torch.randn(N, Ho, Wo, Cout, generator=g, device='cuda').to(BF16)
    if kind == 'fprop':
        return [x() for _ in range(3)], [w() for _ in range(3)]
    if kind == 'dgrad':
        return [dy() for _ in range(3)], [w() for _ in range(3)]
    return [x() for _ in range(3)], [dy() for _ in range(3)]


def check_passes(key, N, seed=0):
    """Pass-structure replay of one launch at batch N: [(prezeroed mode, worst ratio, where)]."""
    kind, H, W, Cs, Cin, Cout, R, S, s = key
    a, b = _bf16_operands(key, N, seed)
    ref, A = _pair_ref(kind, a, b, key, N)
    if kind == 'fprop':
        a_dev = [_pad_cs(t, Cs) for t in a]
        b_dev = [_pack(t, BF16, R, Cin, Cs, Cout, want_wd=False)[0] for t in b]
    elif kind == 'dgrad':
        a_dev = [t.contiguous() for t in a]
        b_dev = [_pack(t, BF16, R, Cin, Cs, Cout)[1] for t in b]
    else:
        a_dev = [_pad_cs(t, Cs) for t in a]
        b_dev = [t.contiguous() for t in b]
    return _run_modes(key, N, a_dev, b_dev, ref, A, TAU)


def _large_n(key, N, sms):
    """bench's 128 views capped by MACS_BUDGET, but never fewer 128 x 128 output tiles than SMs (persistent CTAs
    loop, the wgrad splits K more than once); None if that is not beyond the recorded N."""
    kind, H, W, Cs, Cin, Cout, R, S, s = key
    rows = ((H - 1) // s + 1) * ((W - 1) // s + 1)
    tiles_n = ((Cin if kind == 'dgrad' else Cout) + 127) // 128
    want = (sms // tiles_n + 1) * 128 // rows + 1
    cap = int(MACS_BUDGET // (rows * R * S * Cin * Cout))
    n = max(want, min(BENCH_VIEWS, cap))
    return n if n > N else None


def _report(items, check, what, tau):
    """items: [(key, N)].  Runs check(key, N) -> [(mode, ratio, where)], prints the worst ratio of each launch in both
    modes and fails listing every offender.  tau: a number, or a description of the per-launch tau."""
    bad, worst = [], 0.0
    t0 = time.time()
    for key, N in items:
        res = check(key, N)
        for pz, ratio, where in res:
            worst = max(worst, ratio)
            if not ratio <= 1.0:
                bad.append((_fmt(key), N, 'prezeroed %d' % pz, ratio, where))
        print('    %-62s N %5d  worst |err|/bound %s' % (
            _fmt(key), N, '  '.join('%.3f (pz %d) at %s' % (r, pz, w) for pz, r, w in res)))
    print('%s: %d launches, worst |err|/(tau A) = %.3f (tau = %s), %.1f s' % (
        what, len(items), worst, tau if isinstance(tau, str) else '2^%.2f' % math.log2(tau), time.time() - t0))
    assert not bad, bad


def _tc3_items(rec):
    return sorted(((k, n) for k, n in rec['convs'].items() if not k[0].startswith('simt')), key=lambda kv: _fmt(kv[0]))


@pytest.mark.parametrize('size', ['recorded', 'large'])
@pytest.mark.parametrize('family', list(FAMILIES))
def test_passes_vs_fp64(inventory, family, size):
    """Each distinct tc3 launch of the family's fp32 step on six independent bf16 parts, per element against the
    fp64 sum of the six pair convolutions, with the pre-zeroed mode off and as the step issues it."""
    items = _tc3_items(inventory[family])
    if size == 'large':
        sms = _sms()
        items = [(k, _large_n(k, n, sms)) for k, n in items]
        items = [(k, n) for k, n in items if n is not None]
        assert items, 'the time budget leaves no launch at a larger batch'
    _report(items, check_passes, '%s pass structure at the %s batch' % (family, size), TAU)


# ---------------------------------------------------------------------------------------------------
# end to end: unrounded fp32 operands through the real split and packing
# ---------------------------------------------------------------------------------------------------
def _split(t):
    from simclr_b200._lib import lib, stream_ptr
    t = t.contiguous()
    parts = [torch.full(t.shape, float('nan'), dtype=BF16, device='cuda') for _ in range(3)]
    lib.split_bf16x3(t, parts[0], parts[1], parts[2], t.numel(), stream_ptr())
    return parts


def _kp(R, S, Cs):
    return (R * (S + 1 if Cs == 4 else S) * Cs + 63) // 64 * 64


def _pack3(w, key, want_wd):
    from simclr_b200._lib import lib, stream_ptr
    _, H, W, Cs, Cin, Cout, R, S, s = key
    Kp, Kdp = _kp(R, S, Cs), (R * S * Cout + 63) // 64 * 64
    wf = [torch.full((Cout, Kp), float('nan'), dtype=BF16, device='cuda') for _ in range(3)]
    wd = [torch.full((Cin, Kdp), float('nan'), dtype=BF16, device='cuda') if want_wd else None for _ in range(3)]
    for part in range(3):
        lib.pack_conv_weight_part(w.contiguous(), wf[part], wd[part], part, R, S, Cin, Cs, Cout, Kp, stream_ptr())
    return wf, wd


def _fp32(shape, g, scale, spread):
    """randn * scale; with spread, each element further scaled by 2^k, k uniform in [-20, 20]."""
    t = torch.randn(shape, generator=g, device='cuda') * scale
    if spread:
        t = t * torch.exp2(torch.randint(-20, 21, shape, generator=g, device='cuda').float())
    return t


def check_end_to_end(key, N, spread, seed=0):
    kind, H, W, Cs, Cin, Cout, R, S, s = key
    Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
    g = torch.Generator(device='cuda').manual_seed(seed + 7 + sum(v for v in key if type(v) is int))
    x = _fp32((N, H, W, Cin), g, 1.0, spread)
    w = _fp32((R, S, Cin, Cout), g, 1.0 / (R * S * Cin) ** 0.5, spread)
    dy = _fp32((N, Ho, Wo, Cout), g, 1.0, spread)
    x64, w64, dy64 = x.double(), w.double(), dy.double()
    if kind == 'fprop':
        a, b = _split(_pad_cs(x, Cs)), _pack3(w, key, False)[0]
        ref, A = conv_reference(x64, w64, R, s), conv_reference(x64.abs(), w64.abs(), R, s)
    elif kind == 'dgrad':
        a, b = _split(dy), _pack3(w, key, True)[1]
        ref, A = _ref_dx(dy64, w64, R, s, (N, H, W, Cin)), _ref_dx(dy64.abs(), w64.abs(), R, s, (N, H, W, Cin))
    else:
        a, b = _split(_pad_cs(x, Cs)), _split(dy)
        ref = _ref_dw(x64, dy64, R, s, (R, S, Cin, Cout))
        A = _ref_dw(x64.abs(), dy64.abs(), R, s, (R, S, Cin, Cout))
    K = {'fprop': R * S * Cin, 'dgrad': R * S * Cout, 'wgrad': N * Ho * Wo}[kind]     # reduction length
    return _run_modes(key, N, a, b, ref, A, tau_spread(K) if spread else TAU_E2E)


@pytest.mark.parametrize('spread', [False, True], ids=['randn', 'spread2^20'])
@pytest.mark.parametrize('family', list(FAMILIES))
def test_end_to_end_vs_fp64(inventory, family, spread):
    """Each distinct tc3 launch at its recorded batch on unrounded fp32 operands, split and packed by the library,
    per element against the fp64 conv of the fp32 values."""
    items = _tc3_items(inventory[family])
    _report(items, lambda k, n: check_end_to_end(k, n, spread),
            '%s end to end (%s)' % (family, 'magnitudes spread over 2^+-20' if spread else 'randn'),
            'max(2^-17, 8 sqrt(K) u) + 8 u' if spread else TAU_E2E)


# ---------------------------------------------------------------------------------------------------
# operand preparation, bit for bit
# ---------------------------------------------------------------------------------------------------
def _split_ref(v):
    """torch restatement on the CPU (IEEE fp32, subnormals kept): v0 = bf16(v), v1 = bf16(v - v0),
    v2 = bf16(v - v0 - v1)."""
    v = v.cpu()
    v0 = v.to(BF16)
    r1 = v - v0.float()
    v1 = r1.to(BF16)
    v2 = (r1 - v1.float()).to(BF16)
    return v0, v1, v2


def _bits(t):
    return t.cpu().view(torch.int16)


def _edge_values():
    """±0, bf16 ties, values up to the largest finite bf16 and down to fp32 subnormals."""
    vals = [0.0, -0.0, 1.0, -1.0]
    ties = torch.tensor([0x3F808000, 0x3F818000, 0xBF808000, 0x40490000 | 0x8000, 0x3F80C000], dtype=torch.int64)
    vals += ties.to(torch.int32).view(torch.float32).tolist()              # low 16 bits 0x8000: exactly halfway
    max_bf16 = float(torch.finfo(BF16).max)                                 # 0x7F7F0000 = 3.3895e38
    vals += [max_bf16, -max_bf16, max_bf16 * (1 - 2 ** -10), 2.0 ** 127, 1e38]
    vals += [2.0 ** -100, 2.0 ** -110 * 1.2345678, 2.0 ** -115 * 1.7654321, -(2.0 ** -120) * 1.3333333,
             2.0 ** -126, 2.0 ** -126 * 1.9999999, 2.0 ** -130, 2.0 ** -140, 2.0 ** -149, -(2.0 ** -149)]
    g = torch.Generator().manual_seed(17)
    rnd = torch.randn(4096, generator=g) * torch.exp2(torch.randint(-140, 120, (4096,), generator=g).float())
    return torch.cat([torch.tensor(vals, dtype=F32), rnd.float()])


def test_split_edges_bit_exact():
    """simclr_split_bf16x3 against the torch restatement, bit for bit, on signed zeros, ties, the top of the bf16
    range and subnormal third parts; v0 + v1 + v2 == v wherever the three parts can hold v."""
    v = _edge_values().cuda()
    parts = _split(v)
    want = _split_ref(v)
    for i in range(3):
        bad = (_bits(parts[i]) != _bits(want[i])).nonzero()
        assert len(bad) == 0, 'v%d differs at %s: v = %s' % (i, bad[:5].flatten().tolist(), v[bad[:5].flatten()].tolist())
    vc = v.cpu().double()
    total = sum(p.cpu().double() for p in parts)
    # 24 mantissa bits in 3 x 8: exact while the lowest bit of v (2^(e-23)) is no finer than the bf16 subnormal
    # step 2^-133, i.e. for |v| >= 2^-110
    whole = (vc.abs() >= 2.0 ** -110) | (vc == 0)
    assert torch.equal(total[whole], vc[whole])
    # below 2^-110 the third part is a bf16 subnormal: kept (no flush to zero), and the sum is v to half its step
    tiny = (vc.abs() < 2.0 ** -110) & (vc != 0)
    assert int(((want[2].float() != 0) & tiny).sum()) > 10
    assert float((total[tiny] - vc[tiny]).abs().max()) <= 2.0 ** -134
    # from the midpoint between the largest finite bf16 and 2^128 up, bf16(v) is inf and no three-way split exists:
    # the kernel gives v0 = ±inf, v1 = ∓inf, v2 = NaN
    top = torch.tensor([0x7F7F8000, 0x7F7FFFFF, -0x00808000, -0x00800001], dtype=torch.int64).to(torch.int32)
    top = top.view(F32)            # ±3.3962e38 (the tie, rounded to even: inf) and ±3.4028e38 (the largest fp32)
    assert bool(torch.isinf(top.to(BF16)).all()) and bool(torch.isfinite(top).all())
    p = [t.float().cpu() for t in _split(top.cuda())]
    assert torch.equal(p[0], torch.sign(top) * math.inf) and torch.equal(p[1], -torch.sign(top) * math.inf), p
    assert bool(torch.isnan(p[2]).all()), p


def test_split_sizes_bit_exact(inventory):
    """simclr_split_bf16x3 at every tensor size the step splits (odd tails included), against the restatement."""
    sizes = sorted(set().union(*(rec['splits'] for rec in inventory.values())))
    assert sizes
    g = torch.Generator(device='cuda').manual_seed(5)
    for n in sizes:
        v = torch.randn(n, generator=g, device='cuda') * torch.exp2(
            torch.randint(-30, 30, (n,), generator=g, device='cuda').float())
        parts = _split(v)
        want = _split_ref(v)
        for i in range(3):
            assert torch.equal(_bits(parts[i]), _bits(want[i])), 'split of %d elements, part %d' % (n, i)
        assert torch.equal(sum(p.double() for p in parts), v.double()), n


def _pack_ref(part, R, S, Cin, Cs, Cout, Kp):
    """The layouts of include/simclr_b200.h: wf [Cout][Kp], k = (r*S + s)*Cs + c (the stem, Cs = 4:
    k = (r*(S+1) + s+1)*4 + c with slot 0 zero), and wd [Cin][Kdp], k = (r*S + s)*Cout + co; zero padded."""
    Kdp = (R * S * Cout + 63) // 64 * 64
    if Cs == 4:
        t = torch.zeros(R, S + 1, 4, Cout, dtype=BF16)
        t[:, 1:, :Cin] = part
    else:
        t = torch.zeros(R, S, Cs, Cout, dtype=BF16)
        t[:, :, :Cin] = part
    t = t.reshape(-1, Cout)
    wf = torch.zeros(Cout, Kp, dtype=BF16)
    wf[:, :t.shape[0]] = t.t()
    wd = torch.zeros(Cin, Kdp, dtype=BF16)
    wd[:, :R * S * Cout] = part.permute(2, 0, 1, 3).reshape(Cin, -1)
    return wf, wd


def test_pack_parts_bit_exact(inventory):
    """simclr_pack_conv_weight_part, parts 0, 1 and 2, for every packed layer of the three steps: equal to the torch
    split of the fp32 master laid out by hand, zero slots and padding included, and with wd = NULL."""
    from simclr_b200._lib import lib, stream_ptr
    layers = sorted(set().union(*(rec['packs'].keys() for rec in inventory.values())))
    assert any(L[3] == 4 for L in layers) and any(not L[6] for L in layers)
    g = torch.Generator(device='cuda').manual_seed(9)
    for R, S, Cin, Cs, Cout, Kp, has_wd in layers:
        w = torch.randn(R, S, Cin, Cout, generator=g, device='cuda') * torch.exp2(
            torch.randint(-20, 21, (R, S, Cin, Cout), generator=g, device='cuda').float())
        Kdp = (R * S * Cout + 63) // 64 * 64
        want = _split_ref(w)
        for part in range(3):
            wf = torch.full((Cout, Kp), float('nan'), dtype=BF16, device='cuda')
            wd = torch.full((Cin, Kdp), float('nan'), dtype=BF16, device='cuda') if has_wd else None
            lib.pack_conv_weight_part(w, wf, wd, part, R, S, Cin, Cs, Cout, Kp, stream_ptr())
            torch.cuda.synchronize()
            rf, rd = _pack_ref(want[part], R, S, Cin, Cs, Cout, Kp)
            what = 'part %d of %dx%d Cin %d Cs %d Cout %d Kp %d' % (part, R, S, Cin, Cs, Cout, Kp)
            assert torch.equal(_bits(wf), _bits(rf)), 'wf ' + what
            if has_wd:
                assert torch.equal(_bits(wd), _bits(rd)), 'wd ' + what


# ---------------------------------------------------------------------------------------------------
# edges the inventory does not reach
# ---------------------------------------------------------------------------------------------------
def _k(kind, H, W, Cs, Cin, Cout, k, s):
    return (kind, H, W, Cs, Cin, Cout, k, k, s)


EDGES = [
    # fp32 rows that are not 16 bytes: the epilogue accumulates passes 1-5 with atomics
    (_k('fprop', 1, 1, 2048, 2048, 10, 1, 1), 64),
    (_k('fprop', 1, 1, 2048, 2048, 1001, 1, 1), 64),
    (_k('fprop', 9, 9, 64, 64, 1001, 1, 1), 3),
    # strided dgrad on odd extents: parity classes of unequal size; with 1x1, three of the four classes have no
    # tap and must come out exactly 0 over the NaN fill (ref = A = 0)
    (_k('dgrad', 9, 9, 64, 64, 64, 3, 2), 3),
    (_k('dgrad', 7, 7, 512, 512, 512, 3, 2), 2),
    (_k('dgrad', 9, 7, 64, 64, 128, 1, 2), 3),
    (_k('dgrad', 15, 15, 256, 256, 512, 1, 2), 2),
    # the halo wgrad at H = 55 (not a multiple of the two rows per tile), and with 5 * 28 = 140 tiles: not a multiple
    # of the SM count, some CTAs take two
    (_k('wgrad', 55, 56, 64, 64, 64, 3, 1), 2),
    (_k('wgrad', 56, 56, 64, 64, 64, 3, 1), 5),
    # the 224 stem at 128 outputs: generic fprop, and the generic small-channel wgrad
    (_k('fprop', 224, 224, 4, 3, 128, 7, 2), 2),
    (_k('wgrad', 224, 224, 4, 3, 128, 7, 2), 2),
]


@pytest.mark.parametrize('key,N', EDGES, ids=[_fmt(k).replace(' ', '') + '-N%d' % n for k, n in EDGES])
def test_edge_passes_vs_fp64(key, N):
    _report([(key, N)], check_passes, 'edge', TAU)


@pytest.mark.parametrize('Cout', [10, 100])
@pytest.mark.parametrize('precision,conv_engine', [('fp32', 'tc3'), ('bf16', 'tc')])
def test_odd_width_head_vs_fp64(flags, precision, conv_engine, Cout):
    """An odd-width supervised head (10 or 100 classes: output rows that are not 16 bytes) through ConvOp, forward
    and backward with dX as finetuning asks for it, each output per element against fp64.  The forward takes the
    tensor cores (tc3: atomics into the rows); dW and dX take the CUDA-core kernels on the fp32 master, because the
    wgmma wgrad and dgrad both read 16-byte rows of dY.  Before the CUDA-core dgrad, asking for dX here raised."""
    from simclr_b200 import engine, resnet
    from simclr_b200._lib import lib
    dt = F32 if precision == 'fp32' else BF16
    engine.set_engine(engine.Engine(precision=precision, conv_engine=conv_engine))
    N, Cin = 64, 2048
    g = torch.Generator(device='cuda').manual_seed(21 + Cout)
    kern = types.SimpleNamespace(value=torch.randn(1, 1, Cin, Cout, generator=g, device='cuda') / Cin ** 0.5,
                                 constant=False, name='head')
    kern.grad = torch.full_like(kern.value, float('nan'))
    op = resnet.ConvOp(kern, 1, 1, Cin, Cout, 1, need_dgrad=True)
    x = torch.randn(N, 1, 1, Cin, generator=g, device='cuda').to(dt)
    dy = torch.randn(N, 1, 1, Cout, generator=g, device='cuda').to(dt)
    # the bf16 forward multiplies by the bf16-packed weights, the CUDA-core dgrad by the fp32 master
    x64, w64, dy64 = x.double(), kern.value.double(), dy.double()
    wf64 = kern.value.to(dt).double()
    prev = lib.set_accumulate_prezeroed(0)
    try:
        y = op.forward(x, training=True)
        dx = op.backward(dy, need_dx=True)
        torch.cuda.synchronize()
    finally:
        lib.set_accumulate_prezeroed(prev)
    assert y.dtype == dt and dx.dtype == dt and dx.shape == x.shape
    rho = 0.0 if dt == F32 else 2.0 ** -8           # a bf16 output adds one rounding
    tau_y = TAU_E2E if dt == F32 else TAU
    ry, wy = _ratio(y, conv_reference(x64, wf64, 1, 1), conv_reference(x64.abs(), wf64.abs(), 1, 1), rho, tau_y)
    # one thread per output, sequential fp32 sums: of the N rows for dW, of the Cout classes for dX
    rw, ww = _ratio(kern.grad, _ref_dw(x64, dy64, 1, 1, (1, 1, Cin, Cout)),
                    _ref_dw(x64.abs(), dy64.abs(), 1, 1, (1, 1, Cin, Cout)), 0.0, tau_seq(N))
    rx, wx = _ratio(dx, _ref_dx(dy64, w64, 1, 1, (N, 1, 1, Cin)), _ref_dx(dy64.abs(), w64.abs(), 1, 1, (N, 1, 1, Cin)),
                    rho, tau_seq(Cout))
    print('%s/%s %d-class head: fprop %.3f at %s, CUDA-core wgrad %.3f at %s, CUDA-core dgrad %.3f at %s' % (
        precision, conv_engine, Cout, ry, wy, rw, ww, rx, wx))
    assert ry <= 1.0 and rw <= 1.0 and rx <= 1.0, (ry, rw, rx)


@pytest.mark.parametrize('precision,conv_engine', [('fp32', 'tc3'), ('bf16', 'tc')])
def test_finetune_step_odd_classes(flags, precision, conv_engine):
    """A finetuning step (whole network trained, LARS) at 100 classes on the tensor-core engines: the supervised head's
    dX reaches the backbone.  Loss and every gradient against the fp32 CUDA-core step from the same state: 1e-4 and
    1e-2 for tc3 (fp32-accurate products), 2e-2 on the loss for bf16 storage, whose gradients must be finite and not
    all zero in every tensor that the fp32 step gives a gradient."""
    from test_gpu_modes import _finetune_setup
    from util import rel_err, structured_batch
    runs = {}
    for prec, eng in (('fp32', 'simt'), (precision, conv_engine)):
        trainer, om = _finetune_setup(flags, 'lars', -1, 0, prec, eng)           # ResNet-18, batch 16, 64x64
        P, S_ = om.init(0)
        trainer.model.vs.load(P)
        trainer.model.vs.load(S_)
        f6, lab = structured_batch(16, 64, num_classes=100, seed=2)
        trainer.optimizer.learning_rate = 0.0
        loss = trainer.single_step(f6[..., :3].contiguous().cuda(), lab.cuda())
        torch.cuda.synchronize()
        runs[eng] = (float(loss), {v.name: v.grad.clone() for v in trainer.model.trainable_variables})
        del trainer
    (l0, g0), (l1, g1) = runs['simt'], runs[conv_engine]
    assert g0.keys() == g1.keys()
    moving = [k for k in g0 if float(g0[k].abs().max()) > 0]
    assert any('head_supervised' not in k for k in moving), 'the backbone must receive a gradient'
    assert all(bool(torch.isfinite(g1[k]).all()) for k in g1)
    errs = {k: rel_err(g1[k], g0[k]) for k in moving}
    worst = max(errs, key=errs.get)
    print('%s/%s finetune at 100 classes: loss %.6f vs %.6f, worst gradient rel err %.2e (%s)' % (
        precision, conv_engine, l1, l0, errs[worst], worst))
    if conv_engine == 'tc3':
        assert abs(l1 - l0) <= 1e-4 * abs(l0), (l1, l0)
        assert errs[worst] < 1e-2, (worst, errs[worst])
    else:
        assert abs(l1 - l0) <= 2e-2 * abs(l0), (l1, l0)
        assert all(float(g1[k].abs().max()) > 0 for k in moving), [k for k in moving if float(g1[k].abs().max()) == 0]


# ---------------------------------------------------------------------------------------------------
# the fp32 / tc3 step gives the same bits on every run
# ---------------------------------------------------------------------------------------------------
def test_step_same_bits_tc3(flags):
    """Two trainers built from the same state run two eager fp32 / tc3 steps (ResNet-50, 64x64, batch 16, fixed blur
    draws) on the same inputs: loss, every gradient, every updated weight, every moving statistic and the LARS
    momentum slots agree bit for bit after each step.  Each pass's reduce-add is stream-ordered after the previous
    pass, the atomic epilogues write each element once per launch, and split partials are summed in a fixed order."""
    from test_gpu_step import _setup, _data
    B, S = 16, 64
    runs = []
    for _ in range(2):
        trainer, _, _, _ = _setup(flags, 'fp32', 'tc3', True, B, S, depth=50)
        f, lab, sigma, sel = _data(B, S)
        f, lab = f.cuda(), lab.cuda()
        trainer.model.set_blur_draws(torch.tensor(sigma), sel)
        trainer.optimizer.learning_rate = 0.3
        snaps = []
        for _ in range(2):
            loss = trainer.single_step(f, lab)
            torch.cuda.synchronize()
            snaps.append(_snapshot(trainer, loss))
        runs.append(snaps)
        del trainer
    for step, (a, b) in enumerate(zip(*runs)):
        assert a.keys() == b.keys()
        differ = [k for k in a if not torch.equal(a[k], b[k])]
        assert not differ, 'step %d: %d of %d tensors differ, e.g. %s' % (step + 1, len(differ), len(a), differ[:5])
    assert any(not torch.equal(runs[0][0][k], runs[0][1][k]) for k in runs[0][0] if k.startswith('value ')), \
        'the second step must change the weights'
