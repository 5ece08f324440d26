"""Every non-tensor-core kernel launch of the benchmarked step against an fp64 reference, element by element.

The inventory is taken from the model, as in test_gpu_layers.py: one eager step per benchmarked family (bf16 / `tc`
R50 1x, R50 2x and R50 2x SK at 224, and the fp32 / `tc3` R50 1x step of bench's secondary mode), 2 samples each,
with every `lib.<entry>` except the convolutions, the weight packing and the bookkeeping calls wrapped to record its
launch: the entry, every integer and float argument (dtype codes included), which pointers are NULL, and whether the
call accumulated into pre-zeroed sums.  A recorded entry without a replayer below fails the test by name.

Each launch is replayed on seeded operands into NaN-filled outputs (fp64 sums included) at the recorded size and at
a large one (bench's 256 samples / 512 views, capped at ELEM_BUDGET elements per operand, never less than what
reaches the grid-capped loops: see _large_rows), and compared per element with a float64 reference on the GPU:

    |got - ref| <= rho * |ref| + tau * A

A is the same operation on absolute values; rho is 2^-8 for bf16 outputs and 0 for fp32.  Outputs whose arithmetic
is fully defined (pooling maxima and argmax codes, ReLU mask bits, the rewritten gradients of the BatchNorm
reductions, ysel, casts, in-place adds, labels, the global-pool backward) must match exactly.  Launches the step
issues into the pre-zeroed sums pool are replayed a second time that way, into a zeroed slice of a NaN buffer.
"""
import contextlib
import ctypes
import math
import re
import time

import pytest
import torch

from test_gpu_layers import _ratio

pytestmark = pytest.mark.gpu

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
DT = {0: F32, 1: BF16}
RHO = {BF16: 2.0 ** -8, F32: 0.0}
U = 2.0 ** -24                          # unit roundoff of fp32

# tau, in units of A.  A wrong element, channel, block or tail is off by O(A / sqrt(K)) for a reduction of K terms,
# far above all of these.
TAU_EW = 2.0 ** -21        # element-wise fp32 arithmetic: at most four roundings of 2^-24 A (fma, add, store)
TAU_CAST = 2.0 ** -23      # one fp64 -> fp32 rounding (bn_bwd_coef, the mean of bn_finalize)
# rsqrtf: 2 ulp (CUDA C++ Programming Guide, single-precision maximum ulp error table); with the roundings of
# var + eps, gamma * rstd and beta - mean * scale, at most 5 ulp = 2^-20.7.
TAU_RSQRT = 2.0 ** -20
# per-thread fp32 partial sums before the fp64 block tree: at most ~64 terms per thread at ELEM_BUDGET (2^-18 A
# in the worst case); random rounding errors stay far below.  Same allowance as test_gpu_layers.TAU.
TAU_RED = 2.0 ** -17
# expf (2 ulp), logf (1 ulp) and __expf (2 + floor(|1.173 x + 1.4|) ulp: 26 ulp for |x| <= 20 = 2 / temperature
# at 0.1) plus fp32 sums over the classes / columns of a row: 2^-16 of A.
TAU_EXP = 2.0 ** -16
TAU_LARS = 2.0 ** -17      # fp32 norm partials (64 terms per thread per chunk), sqrtf (correctly rounded), division


def tau_seq(K):
    """Sequential fp32 sum of K terms, one thread per output: rounding errors of random sign grow like sqrt(K);
    8 sqrt(K) u bounds them with a wide margin while a dropped term (1/K of A) is still caught for K <= 2^15."""
    return 8.0 * U * math.sqrt(K)


ELEM_BUDGET = 1 << 25       # elements per operand at the large size (fp64 reference + |.| twin: 0.5 GB)
BENCH_VIEWS = 512           # bench.py: 256 samples, two views

FAMILIES = {
    'r50_1x_224': dict(precision='bf16', engine='tc', resnet_depth=50, width_multiplier=1, sk_ratio=0.0),
    'r50_2x_224': dict(precision='bf16', engine='tc', resnet_depth=50, width_multiplier=2, sk_ratio=0.0),
    'r50_2x_sk_224': dict(precision='bf16', engine='tc', resnet_depth=50, width_multiplier=2, sk_ratio=0.0625),
    'r50_1x_224_fp32': dict(precision='fp32', engine='tc3', resnet_depth=50, width_multiplier=1, sk_ratio=0.0),
}

EXCLUDED = re.compile(r'^(conv2d_\w+_(tc|tc3|simt)|pack_\w+|split_bf16x3|memset_zero|set_accumulate_prezeroed|version|'
                      r'last_error|\w+_workspace_bytes)$')


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---------------------------------------------------------------------------------------------------
# inventory
# ---------------------------------------------------------------------------------------------------
def _launch_key(name, args, prezeroed):
    """(entry, ((arg name, value), ...), prezeroed): pointers reduce to whether they are NULL."""
    from simclr_b200._lib import lib
    _, argl = lib.declarations['simclr_' + name]
    items = []
    for (ct, an), v in zip(argl, args):
        if an == 'stream':
            continue
        items.append((an, v is not None) if ct is ctypes.c_void_p else (an, v))
    if name == 'lars_apply':         # the parameter table: sizes and weight-decay / adaptation flags
        items += [('numels', tuple(args[5].tolist())), ('flags', tuple(args[6].tolist()))]
    return name, tuple(items), int(prezeroed)


def _fmt(key):
    name, items, pz = key
    s = ' '.join('%s=%s' % (k, ('-' if v is False else 'P') if isinstance(v, bool) else
                            ('<%d>' % len(v) if isinstance(v, tuple) else ('%.4g' % v if isinstance(v, float) else v)))
                 for k, v in items)
    return '%s(%s)%s' % (name, s, ' prezeroed' if pz else '')


@pytest.fixture(scope='module')
def inventory():
    """{family: set of launch keys}: every non-conv C-ABI launch of one eager step per family."""
    from simclr_b200 import engine, run, flags_def
    from simclr_b200._lib import lib
    F = flags_def.FLAGS
    if not F.is_parsed():
        F(['test'])
    saved = {k: getattr(F, k) for k in flags_def.REFERENCE_FLAG_NAMES + ['b200_precision', 'b200_conv_engine']}
    inv = {}
    try:
        for fam, cfg in FAMILIES.items():
            cfg = dict(cfg)
            prec, eng = cfg.pop('precision'), cfg.pop('engine')
            B, S = 2, 224
            flags_def.set_flags(train_batch_size=B, use_blur=True, optimizer='lars', weight_decay=1e-4, image_size=S,
                                b200_precision=prec, b200_conv_engine=eng, **cfg)
            engine.set_engine(engine.Engine(precision=prec, conv_engine=eng))
            trainer = run.Trainer(num_classes=1000, num_examples=50000, seed=0)
            g = torch.Generator().manual_seed(3)
            f = torch.rand(B, S, S, 6, generator=g).cuda()
            lab = torch.nn.functional.one_hot(torch.randint(0, 1000, (B,), generator=g), 1000).float().cuda()
            launches = set()
            state = {'pz': 0}
            with pytest.MonkeyPatch.context() as mp:
                setpz = getattr(lib, 'set_accumulate_prezeroed')

                def wrap_pz(on, _fn=setpz):
                    state['pz'] = int(on)
                    return _fn(on)
                mp.setattr(lib, 'set_accumulate_prezeroed', wrap_pz)
                for full in lib.declarations:
                    name = full[len('simclr_'):]
                    if EXCLUDED.match(name):
                        continue
                    fn = getattr(lib, name)

                    def wrap(*a, _fn=fn, _name=name):
                        launches.add(_launch_key(_name, a, state['pz']))
                        return _fn(*a)
                    mp.setattr(lib, name, wrap)
                trainer.single_step(f, lab)
                torch.cuda.synchronize()
            inv[fam] = launches
            del trainer
            torch.cuda.empty_cache()
    finally:
        for k, v in saved.items():
            setattr(F, k, v)
        lib.set_accumulate_prezeroed(0)
    for fam, launches in inv.items():
        print('\n%s: %d distinct non-conv launches' % (fam, len(launches)))
        for key in sorted(launches, key=_fmt):
            print('    ' + _fmt(key))
    return inv


def _has(launches, name, pred=lambda a: True):
    return any(k[0] == name and pred(dict(k[1])) for k in launches)


_BF = lambda a: a.get('dtype') == 1
LANDMARKS = {
    'r50_1x_224': [
        ('fused stem forward at 112x112, C 64', 'bn_relu_maxpool_fwd', lambda a: (a['H'], a['W'], a['C']) == (112, 112, 64)),
        ('fused stem reduce at 112x112, C 64', 'maxpool_bn_bwd_reduce', lambda a: (a['H'], a['C']) == (112, 64)),
        ('fused stem apply at 112x112, C 64', 'maxpool_bn_bwd_apply', lambda a: (a['H'], a['C']) == (112, 64)),
    ],
    'r50_2x_224': [
        ('fused stem forward at 112x112, C 128', 'bn_relu_maxpool_fwd', lambda a: (a['H'], a['W'], a['C']) == (112, 112, 128)),
        ('fused stem apply at 112x112, C 128', 'maxpool_bn_bwd_apply', lambda a: (a['H'], a['C']) == (112, 128)),
    ],
    'r50_2x_sk_224': [
        ('ResNet-D shortcut avgpool2x2 at stride 2', 'avgpool2x2_fwd', lambda a: a['stride'] == 2),
        ('ResNet-D shortcut avgpool2x2 backward at stride 2', 'avgpool2x2_bwd', lambda a: a['stride'] == 2),
        ('sk_pool in bf16', 'sk_pool', _BF),
        ('sk_mix_fwd in bf16', 'sk_mix_fwd', _BF),
        ('sk_mix_bwd_reduce in bf16', 'sk_mix_bwd_reduce', _BF),
        ('sk_mix_bwd_apply in bf16', 'sk_mix_bwd_apply', _BF),
    ],
    'r50_1x_224_fp32': [],
}
COMMON_LANDMARKS = [
    ('projection tail forward', 'bn_apply2_relu_mask', lambda a: True),
    ('projection tail reduce', 'bn_bwd_reduce2_bits', lambda a: True),
    ('block tail forward with mask bits', 'bn_apply_relu_mask', lambda a: True),
    ('block tail reduce from mask bits', 'bn_bwd_reduce_bits', lambda a: True),
    ('BN + ReLU reduce recomputing the mask', 'bn_bwd_relu_reduce', lambda a: True),
    ('NT-Xent forward', 'ntxent_forward', lambda a: True),
    ('NT-Xent backward', 'ntxent_backward', lambda a: True),
    ('softmax_xent at 1000 classes', 'softmax_xent', lambda a: a['classes'] == 1000),
    ('LARS update', 'lars_apply', lambda a: True),
]


@pytest.mark.parametrize('family', list(FAMILIES))
def test_inventory_landmarks(inventory, family):
    from simclr_b200 import run, flags_def, engine
    launches = inventory[family]
    missing = [what for what, name, pred in LANDMARKS[family] + COMMON_LANDMARKS if not _has(launches, name, pred)]
    assert not missing, '%s no longer launches: %s' % (family, missing)
    # LARS updates every trainable tensor in one launch
    lars = [dict(k[1]) for k in launches if k[0] == 'lars_apply']
    assert len(lars) == 1, lars
    cfg = dict(FAMILIES[family])
    prec, eng = cfg.pop('precision'), cfg.pop('engine')
    F = flags_def.FLAGS
    saved = {k: getattr(F, k) for k in flags_def.REFERENCE_FLAG_NAMES + ['b200_precision', 'b200_conv_engine']}
    try:
        flags_def.set_flags(train_batch_size=2, use_blur=True, optimizer='lars', weight_decay=1e-4, image_size=224,
                            b200_precision=prec, b200_conv_engine=eng, **cfg)
        engine.set_engine(engine.Engine(precision=prec, conv_engine=eng))
        trainer = run.Trainer(num_classes=1000, num_examples=50000, seed=0)
        numels = tuple(v.numel for v in trainer.model.trainable_variables)
        del trainer
    finally:
        for k, v in saved.items():
            setattr(F, k, v)
    assert lars[0]['numels'] == numels, 'lars_apply does not cover every trainable tensor'
    # the step issues every accumulating BatchNorm reduction into the pre-zeroed pool
    for k in launches:
        if k[0] in SUMS_ENTRIES:
            assert k[2] == 1, _fmt(k)


def test_every_entry_has_a_replayer(inventory):
    missing = sorted({k[0] for launches in inventory.values() for k in launches if k[0] not in REPLAY})
    assert not missing, 'recorded entries without an fp64 replayer: %s' % missing


# ---------------------------------------------------------------------------------------------------
# replay helpers
# ---------------------------------------------------------------------------------------------------
class Checks:
    """Collects (what, worst ratio, where) of every output of one replay."""

    def __init__(self):
        self.items = []

    def close(self, what, got, ref, A, rho, tau):
        torch.cuda.synchronize()
        r, w = _ratio(got.reshape(ref.shape), ref, A, rho, tau)
        self.items.append((what, r, w))

    def exact(self, what, got, ref):
        torch.cuda.synchronize()
        got, ref = got.reshape(ref.shape), ref.to(got.dtype)
        bad = ~(got == ref)
        if bool(bad.any()):
            i = int(torch.nonzero(bad.reshape(-1))[0])
            w = tuple(int(v) for v in torch.unravel_index(torch.tensor(i), got.shape))
            self.items.append((what + ' (exact)', math.inf, w))
        else:
            self.items.append((what + ' (exact)', 0.0, ()))

    def worst(self):
        return max(self.items, key=lambda t: t[1])


def _gen(seed):
    return torch.Generator(device='cuda').manual_seed(seed)


def _randn(shape, dt, g, scale=1.0, shift=0.0):
    return (torch.randn(shape, generator=g, device='cuda') * scale + shift).to(dt)


def _nan(shape, dt):
    if dt == torch.uint8:
        return torch.full(shape, 0xff, dtype=dt, device='cuda')
    return torch.full(shape, float('nan'), dtype=dt, device='cuda')


def _rounded(x64, dt):
    """fp64 -> the fp32 value an fmaf produces -> storage type, as fp64."""
    return x64.float().to(dt).double()


@contextlib.contextmanager
def _prezeroed(on):
    from simclr_b200._lib import lib
    prev = lib.set_accumulate_prezeroed(int(on))
    try:
        yield
    finally:
        lib.set_accumulate_prezeroed(prev)


def _sums_buf(n, pz):
    """fp64 sums output: NaN-filled (the call must zero it), or with prezeroed = 1 a zeroed slice inside a larger
    NaN buffer, as the step's pool hands them out."""
    if not pz:
        return _nan((n,), F64)
    buf = _nan((n + 64,), F64)
    buf[16:16 + n].zero_()
    return buf[16:16 + n]


def _red_threshold(C):
    """Rows beyond which launch_reduce caps its grid at 2 * SMs blocks and each block loops (bn.cu red_layout)."""
    cvecs, P = C // 8, 1
    while P * 2 <= cvecs and P * 2 <= 256:
        P *= 2
    return 2 * _sms() * (256 // P) * 8


def _ew_threshold_rows(C):
    """Rows beyond which the element-wise BatchNorm kernels run two grid-stride iterations and a tail."""
    return 2 * 16 * _sms() * 256 * 8 // C


def _large_rows(rows, C, reduce):
    """Bench's batch (rows scaled from 4 to 512 views) capped by ELEM_BUDGET, but at least past the grid caps."""
    need = (_red_threshold(C) if reduce else _ew_threshold_rows(C)) + 1
    n = min(max(rows * BENCH_VIEWS // 4, need), ELEM_BUDGET // C)
    assert n >= need, ('the element budget does not reach the large-size loops', rows, C)
    return n


def _large_n(N, per_sample):
    return max(N + 1, min(N * BENCH_VIEWS // 4, ELEM_BUDGET // per_sample))


def _bn_params(C, g):
    mean = torch.randn(C, generator=g, device='cuda') * 2.0
    rstd = torch.rand(C, generator=g, device='cuda') + 0.5
    scale = torch.randn(C, generator=g, device='cuda') * 0.8         # both signs
    shift = torch.randn(C, generator=g, device='cuda') * 0.3
    return mean, rstd, scale, shift


def _act(rows, C, dt, g):
    """BatchNorm input with per-channel offsets: the pivot of bn_stats matters and a miscounted row shows."""
    off = torch.randn(C, generator=g, device='cuda') * 3.0
    return (torch.randn(rows, C, generator=g, device='cuda') * 1.5 + off).to(dt)


def _unpack_bits(bits, rows, C):
    k = torch.arange(8, device='cuda', dtype=torch.uint8)
    return ((bits.view(-1, 1) >> k) & 1).bool().reshape(rows, C)


def _pack_bits(mask):
    k = torch.arange(8, device='cuda', dtype=torch.int32)
    return (mask.reshape(-1, 8).int() << k).sum(1).to(torch.uint8)


def _check_sums(chk, what, got, ref, A):
    chk.close(what, got, ref, A, 0.0, TAU_RED)


# ---------------------------------------------------------------------------------------------------
# BatchNorm family
# ---------------------------------------------------------------------------------------------------
def r_bn_stats(a, big, pz, chk, seed=0):
    from simclr_b200._lib import lib, stream_ptr
    C, dt = a['C'], DT[a['dtype']]
    rows = _large_rows(a['rows'], C, True) if big else a['rows']
    g = _gen(seed + rows + C)
    x = _act(rows, C, dt, g)
    sums = _sums_buf(2 * C, pz)
    with _prezeroed(pz):
        lib.bn_stats(x, a['dtype'], rows, C, sums, stream_ptr())
    xd = x.double()
    p = xd[0]                               # the pivot: row 0 (bn.cu mode 0)
    u = xd - p
    ref = torch.cat([xd.sum(0), (xd * xd).sum(0)])
    A = torch.cat([u.abs().sum(0), (u * u).sum(0) + 2 * p.abs() * u.abs().sum(0)])
    _check_sums(chk, 'sums', sums, ref, A)
    return rows


def r_bn_finalize(a, big, pz, chk, seed=0):
    from simclr_b200._lib import lib, stream_ptr
    C, count = a['C'], a['count']
    g = _gen(seed + C)
    m = torch.randn(C, generator=g, device='cuda', dtype=F64) * 2
    var = torch.rand(C, generator=g, device='cuda', dtype=F64) + 0.05
    var[::7] = 0.0                                                      # constant channels
    sums = torch.cat([count * m, count * (var + m * m)])
    sums[C::5] = count * m[::5] * m[::5] * (1 - 1e-15)                  # E[x^2] - mean^2 slightly negative: clamped
    gamma = (torch.rand(C, generator=g, device='cuda') + 0.5) if a['gamma'] else None
    beta = torch.randn(C, generator=g, device='cuda') if a['beta'] else None
    mm0 = torch.randn(C, generator=g, device='cuda') if a['moving_mean'] else None
    mv0 = (torch.rand(C, generator=g, device='cuda') + 0.5) if a['moving_var'] else None
    mm, mv = (None if t is None else t.clone() for t in (mm0, mv0))
    out = [_nan((C,), F32) for _ in range(4)]
    lib.bn_finalize(sums, count, gamma, beta, a['eps'], a['momentum'], mm, mv, *out, C, stream_ptr())
    mean_r = sums[:C] / count
    var_r = (sums[C:] / count - mean_r * mean_r).clamp_min(0)
    mf = mean_r.float().double()
    rstd_r = 1.0 / torch.sqrt(var_r.float().double() + float(torch.tensor(a['eps'], dtype=F32)))
    gam = gamma.double() if gamma is not None else torch.ones_like(m)
    bet = beta.double() if beta is not None else torch.zeros_like(m)
    sc = gam * rstd_r
    chk.close('mean', out[0], mean_r, mean_r.abs(), 0, TAU_CAST)
    chk.close('rstd', out[1], rstd_r, rstd_r, 0, TAU_RSQRT)
    chk.close('scale', out[2], sc, sc.abs(), 0, TAU_RSQRT)
    chk.close('shift', out[3], bet - mf * sc, bet.abs() + (mf * sc).abs(), 0, TAU_RSQRT)
    om = 1.0 - float(torch.tensor(a['momentum'], dtype=F32))          # exact in fp32 (Sterbenz)
    if mm is not None:
        r = mm0.double() - (mm0.double() - mf) * om
        chk.close('moving_mean', mm, r, mm0.double().abs() + mf.abs(), 0, TAU_EW)
    if mv is not None:
        vf = var_r.float().double()
        r = mv0.double() - (mv0.double() - vf) * om
        chk.close('moving_var', mv, r, mv0.double().abs() + vf, 0, TAU_EW)
    return C


def r_bn_apply(a, big, pz, chk, seed=0, name='bn_apply'):
    from simclr_b200._lib import lib, stream_ptr
    C = a['C']
    rows = _large_rows(a['rows'], C, False) if big else a['rows']
    g = _gen(seed + rows + C)
    ty, tz = DT[a['y_dtype']], DT[a['z_dtype']]
    y = _act(rows, C, ty, g)
    res = _randn((rows, C), tz, g) if a['residual'] else None
    _, _, scale, shift = _bn_params(C, g)
    z = _nan((rows, C), tz)
    st = stream_ptr()
    if name == 'bn_apply':
        relu = a['relu']
        lib.bn_apply(y, a['y_dtype'], res, z, a['z_dtype'], rows, C, scale, shift, relu, st)
    else:
        relu = 1
        bits = _nan((rows * C // 8,), torch.uint8)
        lib.bn_apply_relu_mask(y, a['y_dtype'], res, z, a['z_dtype'], rows, C, scale, shift, bits, st)
    v = y.double() * scale.double() + shift.double()
    A = (y.double() * scale.double()).abs() + shift.double().abs()
    if res is not None:
        v = v + res.double()
        A = A + res.double().abs()
    ref = v.clamp_min(0) if relu else v
    chk.close('z', z, ref, A, RHO[tz], TAU_EW)
    if name != 'bn_apply':
        chk.exact('mask bits', bits, _pack_bits(z.float() > 0))
    return rows


def r_bn_apply2(a, big, pz, chk, seed=0):
    from simclr_b200._lib import lib, stream_ptr
    C = a['C']
    rows = _large_rows(a['rows'], C, False) if big else a['rows']
    g = _gen(seed + rows + C)
    ty, tz = DT[a['y_dtype']], DT[a['z_dtype']]
    y, y2 = _act(rows, C, ty, g), _act(rows, C, ty, g)
    _, _, scale, shift = _bn_params(C, g)
    _, _, scale2, shift2 = _bn_params(C, g)
    z = _nan((rows, C), tz)
    bits = _nan((rows * C // 8,), torch.uint8)
    lib.bn_apply2_relu_mask(y, y2, a['y_dtype'], z, a['z_dtype'], rows, C, scale, shift, scale2, shift2, bits,
                            stream_ptr())
    zs = _rounded(y2.double() * scale2.double() + shift2.double(), tz)      # the shortcut BN output as stored
    v = y.double() * scale.double() + shift.double() + zs
    A = (y.double() * scale.double()).abs() + shift.double().abs() + zs.abs()
    chk.close('z', z, v.clamp_min(0), A, RHO[tz], TAU_EW)
    chk.exact('mask bits', bits, _pack_bits(z.float() > 0))
    return rows


def _reduce_ref(chk, what, v, y, mean, rstd, sums):
    """sums = (sum v, sum v (y - mean) rstd) per channel over the stored gradient v."""
    yd, mu, r = y.double(), mean.double(), rstd.double()
    ref = torch.cat([v.sum(0), (v * (yd - mu)).sum(0) * r])
    A = torch.cat([v.abs().sum(0), (v.abs() * ((yd - mu).abs() + U * (yd.abs() + mu.abs()))).sum(0) * r])
    _check_sums(chk, what, sums, ref, A)


def r_bn_bwd_reduce(a, big, pz, chk, seed=0, name='bn_bwd_reduce'):
    """Modes 1, 3 and 4 of bn_reduce_kernel: dz <- T(mask * (fp32(dz) + fp32(dz2))) in place, then the sums."""
    from simclr_b200._lib import lib, stream_ptr
    C = a['C']
    rows = _large_rows(a['rows'], C, True) if big else a['rows']
    g = _gen(seed + rows + C)
    td, ty = DT[a['dtype']], DT[a['y_dtype']]
    dz = _randn((rows, C), td, g)
    dz2 = _randn((rows, C), td, g) if a['dz2'] else None
    y = _act(rows, C, ty, g)
    mean, rstd, _, _ = _bn_params(C, g)
    st = stream_ptr()
    sums = _sums_buf(2 * C, pz)
    mask = None
    dz_in = dz.clone()
    if name == 'bn_bwd_reduce':
        zm = _randn((rows, C), td, g) if a['relu_mask_z'] else None
        if zm is not None:
            mask = zm.float() > 0
        with _prezeroed(pz):
            lib.bn_bwd_reduce(dz, dz2, zm, a['dtype'], y, a['y_dtype'], rows, C, mean, rstd, sums, st)
    else:
        bits = torch.randint(0, 256, (rows * C // 8,), generator=g, device='cuda', dtype=torch.uint8)
        mask = _unpack_bits(bits, rows, C)
        if name == 'bn_bwd_reduce_bits':
            with _prezeroed(pz):
                lib.bn_bwd_reduce_bits(dz, dz2, bits, a['dtype'], y, a['y_dtype'], rows, C, mean, rstd, sums, st)
        else:
            y2 = _act(rows, C, ty, g)
            mean2, rstd2, _, _ = _bn_params(C, g)
            sums2 = _sums_buf(2 * C, pz)
            with _prezeroed(pz):
                lib.bn_bwd_reduce2_bits(dz, dz2, bits, a['dtype'], y, y2, a['y_dtype'], rows, C, mean, rstd, mean2,
                                        rstd2, sums, sums2, st)
    v = dz_in.float()
    if dz2 is not None:
        v = v + dz2.float()
    if mask is not None:
        v = torch.where(mask, v, torch.zeros((), device='cuda'))
    v = v.to(td)
    chk.exact('dz rewritten', dz, v)
    _reduce_ref(chk, 'sums', v.double(), y, mean, rstd, sums)
    if name == 'bn_bwd_reduce2_bits':
        _reduce_ref(chk, 'sums2', v.double(), y2, mean2, rstd2, sums2)
    return rows


def r_bn_bwd_relu_reduce(a, big, pz, chk, seed=0):
    from simclr_b200._lib import lib, stream_ptr
    C = a['C']
    rows = _large_rows(a['rows'], C, True) if big else a['rows']
    g = _gen(seed + rows + C)
    td, ty = DT[a['dtype']], DT[a['y_dtype']]
    dz = _randn((rows, C), td, g)
    y = _act(rows, C, ty, g)
    mean, rstd, scale, shift = _bn_params(C, g)
    dz_in = dz.clone()
    sums = _sums_buf(2 * C, pz)
    with _prezeroed(pz):
        lib.bn_bwd_relu_reduce(dz, a['dtype'], y, a['y_dtype'], rows, C, mean, rstd, scale, shift, sums, stream_ptr())
    chk.exact('dz untouched', dz, dz_in)
    # fmaf(y, scale, shift) > 0: the fp64 product is exact and the sum keeps its sign
    m = (y.double() * scale.double() + shift.double()) > 0
    v = torch.where(m, dz.double(), torch.zeros((), device='cuda', dtype=F64))
    _reduce_ref(chk, 'sums', v, y, mean, rstd, sums)
    return rows


def r_bn_bwd_coef(a, big, pz, chk, seed=0):
    from simclr_b200._lib import lib, stream_ptr
    C, count = a['C'], a['count']
    g = _gen(seed + C)
    mean, rstd, _, _ = _bn_params(C, g)
    gamma = (torch.rand(C, generator=g, device='cuda') + 0.5) if a['gamma'] else None
    sums = torch.randn(2 * C, generator=g, device='cuda', dtype=F64) * count
    sums_local = torch.randn(2 * C, generator=g, device='cuda', dtype=F64) * count
    coef = _nan((3 * C,), F32)
    dgamma = _nan((C,), F32) if a['dgamma'] else None
    dbeta = _nan((C,), F32) if a['dbeta'] else None
    lib.bn_bwd_coef(mean, rstd, gamma, sums, sums_local, count, coef, dgamma, dbeta, C, stream_ptr())
    r, mu = rstd.double(), mean.double()
    gm = gamma.double() if gamma is not None else torch.ones_like(r)
    A0, A1 = sums[:C] / count, sums[C:] / count
    ref = torch.cat([gm * r, -gm * r * r * A1, gm * r * (mu * r * A1 - A0)])
    chk.close('coef', coef, ref, ref.abs(), 0, TAU_CAST)
    if dbeta is not None:
        chk.exact('dbeta', dbeta, sums_local[:C].float())
    if dgamma is not None:
        chk.exact('dgamma', dgamma, sums_local[C:].float())
    return C


def _coef(C, g):
    return (torch.randn(3 * C, generator=g, device='cuda') * 0.5).contiguous()


def r_bn_bwd_apply_coef(a, big, pz, chk, seed=0):
    from simclr_b200._lib import lib, stream_ptr
    C = a['C']
    rows = _large_rows(a['rows'], C, False) if big else a['rows']
    g = _gen(seed + rows + C)
    td, ty, to = DT[a['dtype']], DT[a['y_dtype']], DT[a['dy_dtype']]
    dz = _randn((rows, C), td, g)
    y = _act(rows, C, ty, g)
    coef = _coef(C, g)
    _, _, ms, mh = _bn_params(C, g)
    masked = a['mask_scale']
    dy = _nan((rows, C), to)
    lib.bn_bwd_apply_coef(dz, a['dtype'], y, a['y_dtype'], dy, a['dy_dtype'], rows, C, coef,
                          ms if masked else None, mh if masked else None, stream_ptr())
    _apply_ref(chk, 'dy', dy, dz, y, coef, C, (ms, mh) if masked else None, to)
    return rows


def _apply_ref(chk, what, dy, dz, y, coef, C, mask, to):
    k = coef.double().view(3, C)
    gd = dz.double()
    if mask is not None:
        gd = torch.where(y.double() * mask[0].double() + mask[1].double() > 0, gd, torch.zeros((), device='cuda', dtype=F64))
    ref = k[0] * gd + k[1] * y.double() + k[2]
    A = (k[0] * gd).abs() + (k[1] * y.double()).abs() + k[2].abs()
    chk.close(what, dy, ref, A, RHO[to], TAU_EW)


def r_bn_bwd_apply(a, big, pz, chk, seed=0):
    """Coefficients and the element-wise pass in one call."""
    from simclr_b200._lib import lib, stream_ptr
    C, count = a['C'], a['count']
    rows = _large_rows(a['rows'], C, False) if big else a['rows']
    g = _gen(seed + rows + C)
    td, ty, to = DT[a['dtype']], DT[a['y_dtype']], DT[a['dy_dtype']]
    dz, y = _randn((rows, C), td, g), _act(rows, C, ty, g)
    mean, rstd, ms, mh = _bn_params(C, g)
    gamma = torch.rand(C, generator=g, device='cuda') + 0.5
    sums = torch.randn(2 * C, generator=g, device='cuda', dtype=F64) * count
    ws = _nan((3 * C,), F32)
    dy = _nan((rows, C), to)
    masked = a['mask_scale']
    lib.bn_bwd_apply(dz, a['dtype'], y, a['y_dtype'], dy, a['dy_dtype'], rows, C, mean, rstd, gamma, sums, sums, count,
                     None, None, ws, ms if masked else None, mh if masked else None, stream_ptr())
    _apply_ref(chk, 'dy', dy, dz, y, ws, C, (ms, mh) if masked else None, to)
    return rows


def r_bn_bwd_apply2_coef(a, big, pz, chk, seed=0):
    from simclr_b200._lib import lib, stream_ptr
    C = a['C']
    rows = _large_rows(a['rows'], C, False) if big else a['rows']
    g = _gen(seed + rows + C)
    td, ty, to = DT[a['dtype']], DT[a['y_dtype']], DT[a['dy_dtype']]
    dz, y, y2 = _randn((rows, C), td, g), _act(rows, C, ty, g), _act(rows, C, ty, g)
    coef, coef2 = _coef(C, g), _coef(C, g)
    dy, dy2 = _nan((rows, C), to), _nan((rows, C), to)
    lib.bn_bwd_apply2_coef(dz, a['dtype'], y, y2, a['y_dtype'], dy, dy2, a['dy_dtype'], rows, C, coef, coef2, stream_ptr())
    _apply_ref(chk, 'dy', dy, dz, y, coef, C, None, to)
    _apply_ref(chk, 'dy2', dy2, dz, y2, coef2, C, None, to)
    return rows


# ---------------------------------------------------------------------------------------------------
# pooling and the fused stem
# ---------------------------------------------------------------------------------------------------
def _pads(H, W):
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    return Ho, Wo, max((Ho - 1) * 2 + 3 - H, 0) // 2, max((Wo - 1) * 2 + 3 - W, 0) // 2


def _pool_ref(z):
    """MaxPooling2D(3, 2, 'SAME') of z [N,H,W,C] (exact values): (max, argmax code dh*3+dw, first maximum wins)."""
    N, H, W, C = z.shape
    Ho, Wo, pbh, pbw = _pads(H, W)
    zp = torch.full((N, 2 * Ho + 1 + 1, 2 * Wo + 1 + 1, C), -math.inf, dtype=F64, device='cuda')
    zp[:, pbh:pbh + H, pbw:pbw + W] = z
    taps = torch.stack([zp[:, dh:dh + 2 * Ho:2, dw:dw + 2 * Wo:2] for dh in range(3) for dw in range(3)], -1)
    best, code = taps.max(-1)
    first = torch.argmax((taps == best.unsqueeze(-1)).to(torch.uint8), -1)     # first maximum in scan order
    return best, first.to(torch.uint8)


def _route(gp, code, H, W):
    """Pooling backward: the window gradients gp [N,Ho,Wo,C] added into their argmax pixels (fp64, exact)."""
    N, Ho, Wo, C = gp.shape
    _, _, pbh, pbw = _pads(H, W)
    out = torch.zeros((N, 2 * Ho + 2, 2 * Wo + 2, C), dtype=F64, device='cuda')
    for t in range(9):
        dh, dw = divmod(t, 3)
        out[:, dh:dh + 2 * Ho:2, dw:dw + 2 * Wo:2] += torch.where(code == t, gp, torch.zeros((), device='cuda', dtype=F64))
    return out[:, pbh:pbh + H, pbw:pbw + W]


def _stem_operands(N, H, W, C, dt, g, zero_windows=False):
    y = (torch.randn(N, H, W, C, generator=g, device='cuda') * 1.5 + 0.2).to(dt)
    mean, rstd, scale, shift = _bn_params(C, g)
    if zero_windows:            # many channels with relu(scale*y + shift) = 0 everywhere: all-tie windows
        shift[::3] = -100.0
    return y, mean, rstd, scale, shift


def _stem_z(y, scale, shift):
    return _rounded((y.double() * scale.double() + shift.double()).clamp_min(0), y.dtype)


def r_bn_relu_maxpool_fwd(a, big, pz, chk, seed=0, zero_windows=False):
    from simclr_b200._lib import lib, stream_ptr
    H, W, C, dt = a['H'], a['W'], a['C'], DT[a['dtype']]
    N = _large_n(a['N'], H * W * C) if big else a['N']
    g = _gen(seed + N * H + W + C)
    y, _, _, scale, shift = _stem_operands(N, H, W, C, dt, g, zero_windows)
    Ho, Wo, pbh, pbw = _pads(H, W)
    out, am = _nan((N, Ho, Wo, C), dt), _nan((N, Ho, Wo, C), torch.uint8)
    ysel = _nan((N, Ho, Wo, C), dt) if a['ysel'] else None
    lib.bn_relu_maxpool_fwd(y, a['dtype'], scale, shift, out, am, ysel, N, H, W, C, stream_ptr())
    best, code = _pool_ref(_stem_z(y, scale, shift))
    chk.exact('pooled', out.double(), best)
    chk.exact('argmax', am, code)
    if ysel is not None:
        chk.exact('ysel', ysel, _gather(y, code, H, W))
    return N


def _gather(y, code, H, W):
    N, Ho, Wo, C = code.shape
    _, _, pbh, pbw = _pads(H, W)
    c = code.long()
    n_i = torch.arange(N, device='cuda').view(N, 1, 1, 1).expand_as(c)
    h_i = torch.arange(Ho, device='cuda').view(1, Ho, 1, 1) * 2 - pbh + c // 3
    w_i = torch.arange(Wo, device='cuda').view(1, 1, Wo, 1) * 2 - pbw + c % 3
    c_i = torch.arange(C, device='cuda').view(1, 1, 1, C).expand_as(c)
    return y[n_i, h_i, w_i, c_i]


def _stem_bwd_inputs(a, big, seed, zero_windows=False):
    H, W, C, dt = a['H'], a['W'], a['C'], DT[a['dtype']]
    N = _large_n(a['N'], H * W * C) if big else a['N']
    g = _gen(seed + N * H + W + C + 1)
    y, mean, rstd, scale, shift = _stem_operands(N, H, W, C, dt, g, zero_windows)
    Ho, Wo, _, _ = _pads(H, W)
    best, code = _pool_ref(_stem_z(y, scale, shift))
    d = _randn((N, Ho, Wo, C), dt, g)
    d2 = _randn((N, Ho, Wo, C), dt, g) if a['d2'] else None
    gp = d.float() if d2 is None else (d.float() + d2.float()).to(dt).float()     # T(d + d2), as the unfused add
    return N, H, W, C, dt, y, mean, rstd, scale, shift, best, code, d, d2, gp.double()


def r_maxpool_bn_bwd_reduce(a, big, pz, chk, seed=0, zero_windows=False):
    from simclr_b200._lib import lib, stream_ptr
    N, H, W, C, dt, y, mean, rstd, scale, shift, best, code, d, d2, gp = _stem_bwd_inputs(a, big, seed, zero_windows)
    ysel = _gather(y, code, H, W) if a['ysel'] else None
    sums = _sums_buf(2 * C, pz)
    with _prezeroed(pz):
        lib.maxpool_bn_bwd_reduce(d, d2, code, y, ysel, a['dtype'], N, H, W, C, mean, rstd, scale, shift, sums,
                                  stream_ptr())
    mu, r = mean.double(), rstd.double()
    if ysel is not None:
        # the bf16 kernel reduces over the pooled tensor: each window's gradient at its argmax pixel
        m = (ysel.double() * scale.double() + shift.double()) > 0
        v = torch.where(m, gp, torch.zeros((), device='cuda', dtype=F64)).reshape(-1, C)
        yy = ysel.double().reshape(-1, C)
    else:
        px = _route(gp, code, H, W)
        if dt == BF16:
            px = _rounded(px, dt)
        m = (y.double() * scale.double() + shift.double()) > 0
        v = torch.where(m, px, torch.zeros((), device='cuda', dtype=F64)).reshape(-1, C)
        yy = y.double().reshape(-1, C)
    ref = torch.cat([v.sum(0), (v * (yy - mu)).sum(0) * r])
    A = torch.cat([v.abs().sum(0), (v.abs() * ((yy - mu).abs() + U * (yy.abs() + mu.abs()))).sum(0) * r])
    if dt == F32:         # fp32 window sums per pixel (up to four terms) round once more
        A = A + torch.cat([v.abs().sum(0), (v.abs() * (yy - mu).abs()).sum(0) * r]) * 4
    _check_sums(chk, 'sums', sums, ref, A)
    return N


def r_maxpool_bn_bwd_apply(a, big, pz, chk, seed=0, zero_windows=False):
    from simclr_b200._lib import lib, stream_ptr
    N, H, W, C, dt, y, mean, rstd, scale, shift, best, code, d, d2, gp = _stem_bwd_inputs(a, big, seed, zero_windows)
    g = _gen(seed + 7)
    coef = _coef(C, g)
    dy = _nan((N, H, W, C), dt)
    lib.maxpool_bn_bwd_apply(d, d2, code, y, a['dtype'], dy, N, H, W, C, coef, scale, shift, stream_ptr())
    px = _route(gp, code, H, W)
    pxa = _route(gp.abs(), code, H, W)
    if dt == BF16:
        px = _rounded(px, dt)       # the pooling backward stores bf16
    m = (y.double() * scale.double() + shift.double()) > 0
    dz = torch.where(m, px, torch.zeros((), device='cuda', dtype=F64))
    k = coef.double().view(3, C)
    yd = y.double()
    ref = k[0] * dz + k[1] * yd + k[2]
    A = (k[0] * dz).abs() + (k[1] * yd).abs() + k[2].abs() + (k[0].abs() * pxa if dt == F32 else 0)
    chk.close('dy', dy, ref, A, RHO[dt], TAU_EW)
    return N


def r_maxpool3x3s2_fwd(a, big, pz, chk, seed=0):
    from simclr_b200._lib import lib, stream_ptr
    H, W, C, dt = a['H'], a['W'], a['C'], DT[a['dtype']]
    N = _large_n(a['N'], H * W * C) if big else a['N']
    g = _gen(seed + N * H + C)
    x = _randn((N, H, W, C), dt, g).clamp_min(0)           # ReLU outputs: ties at zero
    Ho, Wo, _, _ = _pads(H, W)
    y, am = _nan((N, Ho, Wo, C), dt), _nan((N, Ho, Wo, C), torch.uint8)
    lib.maxpool3x3s2_fwd(x, y, am, a['dtype'], N, H, W, C, stream_ptr())
    best, code = _pool_ref(x.double())
    chk.exact('pooled', y.double(), best)
    chk.exact('argmax', am, code)
    return N


def r_maxpool3x3s2_bwd(a, big, pz, chk, seed=0):
    from simclr_b200._lib import lib, stream_ptr
    H, W, C, dt = a['H'], a['W'], a['C'], DT[a['dtype']]
    N = _large_n(a['N'], H * W * C) if big else a['N']
    g = _gen(seed + N * H + C)
    x = _randn((N, H, W, C), dt, g).clamp_min(0)
    _, code = _pool_ref(x.double())
    Ho, Wo, _, _ = _pads(H, W)
    dy = _randn((N, Ho, Wo, C), dt, g)
    dx = _nan((N, H, W, C), dt)
    lib.maxpool3x3s2_bwd(dy, code, dx, a['dtype'], N, H, W, C, stream_ptr())
    chk.close('dx', dx, _route(dy.double(), code, H, W), _route(dy.double().abs(), code, H, W), RHO[dt], TAU_EW)
    return N


def r_global_avgpool_fwd(a, big, pz, chk, seed=0):
    from simclr_b200._lib import lib, stream_ptr
    HW, C = a['HW'], a['C']
    N = _large_n(a['N'], HW * C) if big else a['N']
    g = _gen(seed + N + HW + C)
    x = _randn((N, HW, C), DT[a['dtype']], g)
    y = _nan((N, C), DT[a['y_dtype']])
    lib.global_avgpool_fwd(x, a['dtype'], y, a['y_dtype'], N, HW, C, stream_ptr())
    chk.close('y', y, x.double().mean(1), x.double().abs().mean(1), RHO[DT[a['y_dtype']]], tau_seq(HW) + TAU_EW)
    return N


def r_global_avgpool_bwd(a, big, pz, chk, seed=0):
    from simclr_b200._lib import lib, stream_ptr
    HW, C = a['HW'], a['C']
    N = _large_n(a['N'], HW * C) if big else a['N']
    g = _gen(seed + N + HW + C)
    dy = _randn((N, C), DT[a['dy_dtype']], g)
    dx = _nan((N, HW, C), DT[a['dtype']])
    lib.global_avgpool_bwd(dy, a['dy_dtype'], dx, a['dtype'], N, HW, C, stream_ptr())
    inv = torch.tensor(1.0 / HW, dtype=F32, device='cuda')
    chk.exact('dx', dx, (dy.float() * inv).to(DT[a['dtype']]).view(N, 1, C).expand(N, HW, C))
    return N


def _avg2x2_ref(x64, stride):
    from oracle import resnet as OR
    return OR.avg_pool_2x2(x64.permute(0, 3, 1, 2), stride).permute(0, 2, 3, 1)


def r_avgpool2x2_fwd(a, big, pz, chk, seed=0):
    from simclr_b200._lib import lib, stream_ptr
    H, W, C, s, dt = a['H'], a['W'], a['C'], a['stride'], DT[a['dtype']]
    N = _large_n(a['N'], H * W * C) if big else a['N']
    g = _gen(seed + N + H + W + C)
    x = _randn((N, H, W, C), dt, g)
    ref = _avg2x2_ref(x.double(), s)
    y = _nan(tuple(ref.shape), dt)
    lib.avgpool2x2_fwd(x, y, a['dtype'], N, H, W, C, s, stream_ptr())
    chk.close('y', y, ref, _avg2x2_ref(x.double().abs(), s), RHO[dt], TAU_EW)
    return N


def r_avgpool2x2_bwd(a, big, pz, chk, seed=0):
    from simclr_b200._lib import lib, stream_ptr
    H, W, C, s, dt = a['H'], a['W'], a['C'], a['stride'], DT[a['dtype']]
    N = _large_n(a['N'], H * W * C) if big else a['N']
    g = _gen(seed + N + H + W + C)
    x = torch.zeros((N, H, W, C), dtype=F64, device='cuda', requires_grad=True)
    yo = _avg2x2_ref(x, s)
    dy = _randn(tuple(yo.shape), dt, g)
    ref = torch.autograd.grad(yo, x, dy.double())[0]
    A = torch.autograd.grad(_avg2x2_ref(x, s), x, dy.double().abs())[0]
    dx = _nan((N, H, W, C), dt)
    lib.avgpool2x2_bwd(dy, dx, a['dtype'], N, H, W, C, s, stream_ptr())
    chk.close('dx', dx, ref, A, RHO[dt], TAU_EW)
    return N


# ---------------------------------------------------------------------------------------------------
# selective kernel
# ---------------------------------------------------------------------------------------------------
def _sk_n(a, big):
    return _large_n(a['N'], a['HW'] * 2 * a['f']) if big else a['N']


def r_sk_pool(a, big, pz, chk, seed=0):
    from simclr_b200._lib import lib, stream_ptr
    HW, f, dt = a['HW'], a['f'], DT[a['dtype']]
    N = _sk_n(a, big)
    x = _randn((N, HW, 2 * f), dt, _gen(seed + N + HW + f))
    gq = _nan((N, f), F32)
    lib.sk_pool(x, a['dtype'], gq, N, HW, f, stream_ptr())
    xd = x.double()
    ref = (xd[..., :f] + xd[..., f:]).mean(1)
    A = (xd[..., :f].abs() + xd[..., f:].abs()).mean(1)
    chk.close('g', gq, ref, A, 0, tau_seq(2 * HW) + TAU_EW)
    return N


def _mixing(logits, f):
    l64 = logits.double().view(-1, 2, f)
    return torch.softmax(l64, 1)


def r_sk_mix_fwd(a, big, pz, chk, seed=0):
    from simclr_b200._lib import lib, stream_ptr
    HW, f, dt = a['HW'], a['f'], DT[a['dtype']]
    N = _sk_n(a, big)
    g = _gen(seed + N + HW + f)
    x = _randn((N, HW, 2 * f), dt, g)
    logits = torch.randn(N, 2 * f, generator=g, device='cuda') * 3
    mixing, out = _nan((N, 2 * f), F32), _nan((N, HW, f), dt)
    lib.sk_mix_fwd(x, logits, mixing, out, a['dtype'], N, HW, f, stream_ptr())
    m = _mixing(logits, f)                                   # [N, 2, f]
    chk.close('mixing', mixing, m.reshape(N, 2 * f), m.reshape(N, 2 * f), 0, TAU_EXP)
    xd = x.double()
    ref = xd[..., :f] * m[:, 0:1] + xd[..., f:] * m[:, 1:2]
    A = xd[..., :f].abs() * m[:, 0:1] + xd[..., f:].abs() * m[:, 1:2]
    chk.close('out', out, ref, A, RHO[dt], TAU_EXP)
    return N


def r_sk_mix_bwd_reduce(a, big, pz, chk, seed=0):
    from simclr_b200._lib import lib, stream_ptr
    HW, f, dt = a['HW'], a['f'], DT[a['dtype']]
    N = _sk_n(a, big)
    g = _gen(seed + N + HW + f)
    dout, x = _randn((N, HW, f), dt, g), _randn((N, HW, 2 * f), dt, g)
    mixing = _mixing(torch.randn(N, 2 * f, generator=g, device='cuda'), f).float().reshape(N, 2 * f).contiguous()
    dl = _nan((N, 2 * f), F32)
    lib.sk_mix_bwd_reduce(dout, x, mixing, dl, a['dtype'], N, HW, f, stream_ptr())
    dd, xd, m = dout.double(), x.double(), mixing.double().view(N, 2, f)
    d0, d1 = (dd * xd[..., :f]).sum(1), (dd * xd[..., f:]).sum(1)
    a0, a1 = (dd.abs() * xd[..., :f].abs()).sum(1), (dd.abs() * xd[..., f:].abs()).sum(1)
    dot = m[:, 0] * d0 + m[:, 1] * d1
    adot = m[:, 0] * a0 + m[:, 1] * a1
    ref = torch.cat([m[:, 0] * (d0 - dot), m[:, 1] * (d1 - dot)], 1)
    A = torch.cat([m[:, 0] * (a0 + adot), m[:, 1] * (a1 + adot)], 1)
    chk.close('dlogits', dl, ref, A, 0, tau_seq(HW) + TAU_EW)
    return N


def r_sk_mix_bwd_apply(a, big, pz, chk, seed=0):
    from simclr_b200._lib import lib, stream_ptr
    HW, f, dt = a['HW'], a['f'], DT[a['dtype']]
    N = _sk_n(a, big)
    g = _gen(seed + N + HW + f)
    dout = _randn((N, HW, f), dt, g)
    mixing = _mixing(torch.randn(N, 2 * f, generator=g, device='cuda'), f).float().reshape(N, 2 * f).contiguous()
    dg = torch.randn(N, f, generator=g, device='cuda') * HW ** 0.5
    dx = _nan((N, HW, 2 * f), dt)
    lib.sk_mix_bwd_apply(dout, mixing, dg, dx, a['dtype'], N, HW, f, stream_ptr())
    dd, m, pool = dout.double(), mixing.double().view(N, 1, 2, f), (dg.double() / HW).view(N, 1, 1, f)
    ref = (dd.view(N, HW, 1, f) * m + pool).reshape(N, HW, 2 * f)
    A = (dd.abs().view(N, HW, 1, f) * m + pool.abs()).reshape(N, HW, 2 * f)
    chk.close('dx', dx, ref, A, RHO[dt], TAU_EW)
    return N


# ---------------------------------------------------------------------------------------------------
# small helpers and heads
# ---------------------------------------------------------------------------------------------------
def _n_large(n):
    return max(n + 1, min(n * BENCH_VIEWS // 4, ELEM_BUDGET))


def r_cast(a, big, pz, chk, seed=0):
    from simclr_b200._lib import lib, stream_ptr
    n = _n_large(a['n']) if big else a['n']
    src = _randn((n,), DT[a['src_dtype']], _gen(seed + n), 3.0)
    dst = _nan((n,), DT[a['dst_dtype']])
    lib.cast(src, a['src_dtype'], dst, a['dst_dtype'], n, stream_ptr())
    chk.exact('dst', dst, src.float().to(DT[a['dst_dtype']]))
    return n


def r_add_inplace(a, big, pz, chk, seed=0):
    from simclr_b200._lib import lib, stream_ptr
    dt = DT[a['dtype']]
    n = (_n_large(a['n']) // 8 * 8) if big else a['n']
    g = _gen(seed + n)
    x, y = _randn((n,), dt, g), _randn((n,), dt, g)
    ref = (x.float() + y.float()).to(dt)
    lib.add_inplace(x, y, a['dtype'], n, stream_ptr())
    chk.exact('a', x, ref)
    return n


def r_axpy(a, big, pz, chk, seed=0):
    from simclr_b200._lib import lib, stream_ptr
    n = _n_large(a['n']) if big else a['n']
    g = _gen(seed + n)
    x, y = torch.randn(n, generator=g, device='cuda'), torch.randn(n, generator=g, device='cuda') * 1e-3
    al = float(torch.tensor(a['a'], dtype=F32))
    ref = al * x.double() + y.double()
    A = (al * x.double()).abs() + y.double().abs()
    lib.axpy(a['a'], x, y, n, stream_ptr())
    chk.close('y', y, ref, A, 0, TAU_EW)
    return n


def r_l2_loss(a, big, pz, chk, seed=0):
    from simclr_b200._lib import lib, stream_ptr
    n = a['n']            # the step's own sizes: a weight tensor
    x = torch.randn(n, generator=_gen(seed + n), device='cuda') * 0.05
    out = _nan((257,), F32)
    lib.l2_loss(x, n, out, stream_ptr())
    ref = (x.double() ** 2).sum() / 2
    chk.close('loss', out[:1], ref.view(1), ref.view(1), 0, TAU_RED)
    return n


def r_relu_inplace(a, big, pz, chk, seed=0):
    from simclr_b200._lib import lib, stream_ptr
    n = _n_large(a['n']) if big else a['n']
    g = _gen(seed + n)
    x = torch.randn(n, generator=g, device='cuda')
    m = torch.randn(n, generator=g, device='cuda') if a['mask_src'] else None
    ref = torch.where((m if m is not None else x) > 0, x, torch.zeros((), device='cuda'))
    lib.relu_inplace(x, m, n, stream_ptr())
    chk.exact('x', x, ref)
    return n


def r_bias_add(a, big, pz, chk, seed=0):
    from simclr_b200._lib import lib, stream_ptr
    C = a['C']
    rows = max(a['rows'] + 1, min(a['rows'] * BENCH_VIEWS // 4, ELEM_BUDGET // C)) if big else a['rows']
    g = _gen(seed + rows + C)
    y, b = torch.randn(rows, C, generator=g, device='cuda'), torch.randn(C, generator=g, device='cuda')
    ref = y + b              # one IEEE fp32 add per element
    lib.bias_add(y, b, rows, C, stream_ptr())
    chk.exact('y', y, ref)
    return rows


def r_bias_grad(a, big, pz, chk, seed=0):
    from simclr_b200._lib import lib, stream_ptr
    C = a['C']
    rows = max(a['rows'] + 1, min(a['rows'] * BENCH_VIEWS // 4, ELEM_BUDGET // C)) if big else a['rows']
    dy = torch.randn(rows, C, generator=_gen(seed + rows + C), device='cuda')
    db = _nan((C,), F32)
    lib.bias_grad(dy, db, rows, C, stream_ptr())
    chk.close('dbias', db, dy.double().sum(0), dy.double().abs().sum(0), 0, tau_seq(rows // 8 + 8))
    return rows


def softmax_xent_case(rows, label_rows, classes, gs, chk, seed=0, big_logits=False, want_grad=True):
    from simclr_b200._lib import lib, stream_ptr
    g = _gen(seed + rows + classes)
    x = torch.randn(rows, classes, generator=g, device='cuda') * (1e4 if big_logits else 3.0)
    lab = torch.nn.functional.one_hot(torch.randint(0, classes, (label_rows,), generator=g, device='cuda'),
                                      classes).float()
    loss = _nan((1 + rows,), F32)
    dl = _nan((rows, classes), F32) if want_grad else None
    lib.softmax_xent(x, lab, rows, label_rows, classes, gs, loss, dl, stream_ptr())
    xd = x.double()
    L = lab.double()[torch.arange(rows, device='cuda') % label_rows]
    lse = torch.logsumexp(xd, 1)
    dot = (L * xd).sum(1)
    row = lse - dot
    A = 1.0 + lse.abs() + dot.abs()
    chk.close('row loss', loss[1:], row, A, 0, TAU_EXP)
    chk.close('loss', loss[:1], row.mean().view(1), A.mean().view(1), 0, TAU_EXP)
    if want_grad:
        p = torch.softmax(xd, 1)
        # + 2^-100: expf results below 2^-126 are subnormal in fp32 and keep no relative precision
        chk.close('dlogits', dl, (p - L) * gs, (p + L + 2.0 ** -100) * abs(gs), 0, TAU_EXP)


def r_softmax_xent(a, big, pz, chk, seed=0):
    rows = a['rows'] * BENCH_VIEWS // 4 if big else a['rows']
    lr = a['label_rows'] * BENCH_VIEWS // 4 if big else a['label_rows']
    softmax_xent_case(rows, lr, a['classes'], a['grad_scale'], chk, seed, want_grad=a['dlogits'])
    return rows


# ---------------------------------------------------------------------------------------------------
# NT-Xent
# ---------------------------------------------------------------------------------------------------
def _splits(B, R):
    """pick_splits of ntxent.cu: column splits of the forward / backward."""
    rows, cols = 2 * B, 2 * R * B
    rb, nt = (rows + 31) // 32, (cols + 63) // 64
    want = min(max((2 * _sms() + rb - 1) // rb, 1), 16, nt)
    tps = (nt + want - 1) // want
    return (nt + tps - 1) // tps


def ntxent_case(B, R, D, temp, norm, chk, seed=0, hscale=1.0, metrics=False):
    """Normalize, forward and backward of every replica from a hand-built all-gather (as
    test_gpu_kernels.test_ntxent_replicas_in_one_process) against oracle/objective.py in fp64."""
    from oracle import objective as O
    from simclr_b200._lib import lib, stream_ptr
    g = _gen(seed + B * R + D)
    st = stream_ptr()
    hs = [torch.randn(2 * B, D, generator=g, device='cuda') * hscale for _ in range(R)]
    zs, invs = [], []
    for h in hs:
        z, inv = _nan((2 * B, D), F32), _nan((2 * B,), F32)
        lib.ntxent_normalize(h, 2 * B, D, int(norm), z, inv, st)
        hd = h.double()
        if norm:
            ss = (hd * hd).sum(1, keepdim=True)
            inv_r = torch.rsqrt(ss.clamp_min(1e-12))
            chk.close('inv_norm', inv, inv_r.view(-1), inv_r.view(-1), 0, TAU_RSQRT + D * U)
            chk.close('z', z, hd * inv_r, (hd * inv_r).abs(), 0, TAU_RSQRT + D * U)
        else:
            chk.exact('z', z, h)
        zs.append(z)
        invs.append(inv)
    z_all = torch.stack(zs).contiguous()
    ws_bytes = lib.ntxent_workspace_bytes(B, R, D)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device='cuda')
    zo = [z.double().cpu().requires_grad_(True) for z in zs]          # the oracle builds its labels on the CPU
    outs = O.contrastive_loss_replicas(zo, False, temp)
    lses = []
    for r in range(R):
        logits, lse = _nan((B, R * B), F32), _nan((2 * B,), F32)
        rl, loss = _nan((2 * B,), F32), _nan((1,), F32)
        lib.ntxent_forward(z_all, B, R, D, r, temp, logits, lse, rl, loss, ws, ws_bytes, st)
        lses.append(lse)
        za = z_all.double()
        h1, h2 = za[r, :B], za[r, B:]
        k1, k2 = za[:, :B].reshape(-1, D), za[:, B:].reshape(-1, D)
        eye = torch.zeros(B, R * B, dtype=torch.bool, device='cuda')
        eye[torch.arange(B), torch.arange(B) + r * B] = True
        neg = torch.full((), -math.inf, dtype=F64, device='cuda')
        ab, ba = h1 @ k2.t() / temp, h2 @ k1.t() / temp
        aa, bb = torch.where(eye, neg, h1 @ k1.t() / temp), torch.where(eye, neg, h2 @ k2.t() / temp)
        lse_r = torch.cat([torch.logsumexp(torch.cat([ab, aa], 1), 1), torch.logsumexp(torch.cat([ba, bb], 1), 1)])
        pos = torch.cat([ab[eye], ba[eye]])
        Al = (h1.abs() @ k2.abs().t()) / temp
        span = 2.0 / temp                       # |logit| <= 1 / temperature for unit rows
        chk.close('logits_ab r%d' % r, logits, outs[r][1].detach().cuda(), Al, 0, TAU_RED)
        chk.close('lse r%d' % r, lse, lse_r, span + lse_r.abs(), 0, TAU_EXP)
        chk.close('row_loss r%d' % r, rl, lse_r - pos, span + lse_r.abs() + pos.abs(), 0, TAU_EXP)
        chk.close('loss r%d' % r, loss, outs[r][0].detach().cuda().view(1), (span + lse_r.abs() + pos.abs()).mean().view(1), 0,
                  TAU_EXP)
        if metrics:
            out = _nan((2 + 2 * B,), F32)
            lib.contrast_metrics(logits, B, R * B, r, out, st)
            lab = torch.arange(B, device='cuda') + r * B
            acc = (logits.argmax(1) == lab).double().mean()
            p = torch.softmax(logits.double(), 1)
            ent = -(p * torch.log(p + 1e-8)).sum(1).mean()
            chk.exact('accuracy r%d' % r, out[:1], acc.float().view(1))
            chk.close('entropy r%d' % r, out[1:2], ent.view(1), (ent.abs() + 1).view(1), 0, TAU_EXP)
    total = sum(o[0] for o in outs) / R
    total.backward()
    lse_all = torch.stack(lses).contiguous()
    gs = 1.0 / (B * R)
    for r in range(R):
        dh = _nan((2 * B, D), F32)
        lib.ntxent_backward(z_all, lse_all, invs[r], int(norm), B, R, D, r, temp, gs, dh, ws, ws_bytes, st)
        # d total / d z_r, through the normalisation when it is on: dh = inv (dz - z (z . dz))
        dz = zo[r].grad.cuda() * (gs * B * R)
        zr = z_all[r].double().reshape(2 * B, D)
        if norm:
            ref = invs[r].double().view(-1, 1) * (dz - zr * (zr * dz).sum(1, keepdim=True))
            A = invs[r].double().view(-1, 1) * (2 * span * gs * 4) * torch.ones_like(ref)
        else:
            ref = dz
            A = (2 * span * gs * 4) * zr.abs().amax(1, keepdim=True).expand_as(ref)
        chk.close('dhidden r%d' % r, dh, ref, A, 0, TAU_EXP)
    return _splits(B, R)


def r_ntxent_normalize(a, big, pz, chk, seed=0):
    from simclr_b200._lib import lib, stream_ptr
    rows = a['rows'] * BENCH_VIEWS // 4 if big else a['rows']
    D = a['dim']
    h = torch.randn(rows, D, generator=_gen(seed + rows), device='cuda')
    z, inv = _nan((rows, D), F32), _nan((rows,), F32)
    lib.ntxent_normalize(h, rows, D, a['hidden_norm'], z, inv, stream_ptr())
    hd = h.double()
    inv_r = torch.rsqrt((hd * hd).sum(1, keepdim=True).clamp_min(1e-12))
    if a['hidden_norm']:
        chk.close('inv_norm', inv, inv_r.view(-1), inv_r.view(-1), 0, TAU_RSQRT + D * U)
        chk.close('z', z, hd * inv_r, (hd * inv_r).abs(), 0, TAU_RSQRT + D * U)
    else:
        chk.exact('z', z, h)
    return rows


def r_ntxent_fwd_bwd(a, big, pz, chk, seed=0):
    B = a['B'] * BENCH_VIEWS // 4 if big else a['B']
    splits = ntxent_case(B, a['R'], a['D'], a['temperature'], True, chk, seed, metrics=True)
    if big:
        assert splits > 1, ('the large NT-Xent replay has one column split', B, a['R'])
    return B


def r_ntxent_labels(a, big, pz, chk, seed=0):
    from oracle import objective as O
    from simclr_b200._lib import lib, stream_ptr
    B, R, rid = a['B'], a['R'], a['replica_id']
    if big:
        B = B * BENCH_VIEWS // 4
    G = B * R
    idx = _nan((B,), torch.uint8).long().fill_(-1) if a['labels_idx'] else None
    lab = _nan((B, 2 * G), F32) if a['labels'] else None
    msk = _nan((B, G), F32) if a['masks'] else None
    lib.ntxent_labels(B, R, rid, idx, lab, msk, stream_ptr())
    i_o, l_o, m_o = O.labels_and_masks(B, rid, G, torch.float32)
    for what, got, ref in (('labels_idx', idx, i_o), ('labels', lab, l_o), ('masks', msk, m_o)):
        if got is not None:
            chk.exact(what, got, ref.cuda())
    return B


def r_contrast_metrics(a, big, pz, chk, seed=0):
    from simclr_b200._lib import lib, stream_ptr
    B, G, rid = a['B'], a['G'], a['replica_id']
    if big:
        B, G = B * BENCH_VIEWS // 4, G * BENCH_VIEWS // 4
    logits = torch.randn(B, G, generator=_gen(seed + B + G), device='cuda') * 5
    out = _nan((2 + 2 * B,), F32)
    lib.contrast_metrics(logits, B, G, rid, out, stream_ptr())
    lab = torch.arange(B, device='cuda') + rid * B
    acc = (logits.argmax(1) == lab).double().mean()
    p = torch.softmax(logits.double(), 1)
    ent = -(p * torch.log(p + 1e-8)).sum(1).mean()
    chk.close('accuracy', out[:1], acc.view(1), torch.ones(1, dtype=F64, device='cuda'), 0, 2 * U)
    chk.close('entropy', out[1:2], ent.view(1), (ent.abs() + 1).view(1), 0, TAU_EXP)
    return B


# ---------------------------------------------------------------------------------------------------
# LARS
# ---------------------------------------------------------------------------------------------------
def lars_case(numels, flags, chk, momentum=0.9, weight_decay=1e-4, eeta=0.001, lr=1.2, seed=0, offset=(),
              zero_w=(), zero_g=()):
    """One lars_apply over a parameter table against oracle/lars.py in fp64, per element of w and v.
    offset: tensors whose base is one float past a 16-byte boundary (the scalar path)."""
    from oracle import lars as L
    from simclr_b200._lib import lib, stream_ptr
    CH = 16384
    g = _gen(seed + len(numels))
    W, G, V, keep = [], [], [], []
    for i, n in enumerate(numels):
        o = 1 if i in offset else 0
        buf = [torch.empty(n + 4, device='cuda') for _ in range(3)]
        w, gr, v = (b[o:o + n] for b in buf)
        w.copy_(torch.randn(n, generator=g, device='cuda') * 0.05 * (0 if i in zero_w else 1))
        gr.copy_(torch.randn(n, generator=g, device='cuda') * 0.01 * (0 if i in zero_g else 1))
        v.copy_(torch.randn(n, generator=g, device='cuda') * 1e-3)
        W.append(w); G.append(gr); V.append(v); keep += buf
    names, P, Gd, Vd = [], {}, {}, {}
    for i, fl in enumerate(flags):
        assert fl in (0, 2, 3) and (fl != 2 or weight_decay == 0), fl
        nm = 'layer%d/%s' % (i, 'kernel' if fl else 'batch_normalization/gamma')
        names.append(nm)
        P[nm], Gd[nm], Vd[nm] = W[i].double(), G[i].double(), V[i].double()
    ct, co, begin = [], [], [0]
    for i, n in enumerate(numels):
        for o in range(0, n, CH):
            ct.append(i); co.append(o)
        begin.append(len(ct))
    dev = lambda x, dt: torch.tensor(x, dtype=dt, device='cuda')
    lr_dev = dev([lr], F32)
    partials = _nan((2 * len(ct),), F32)
    lrf = float(lr_dev[0])
    mom, wd = float(torch.tensor(momentum, dtype=F32)), float(torch.tensor(weight_decay, dtype=F32))
    P1, V1 = L.lars_apply(P, Gd, Vd, lrf, mom, weight_decay=wd, exclude_from_weight_decay=L.LARS_EXCLUDE,
                          eeta=float(torch.tensor(eeta, dtype=F32)))
    lib.lars_apply(len(numels), len(ct), dev([w.data_ptr() for w in W], torch.int64),
                   dev([x.data_ptr() for x in G], torch.int64), dev([v.data_ptr() for v in V], torch.int64),
                   dev(list(numels), torch.int64), dev(list(flags), torch.int32), dev(ct, torch.int32),
                   dev(co, torch.int64), dev(begin, torch.int64), CH, lr_dev, momentum, weight_decay, eeta, partials,
                   stream_ptr())
    worst_v = worst_w = (0.0, None)
    for i, nm in enumerate(names):
        step = (P[nm] - P1[nm])               # = next_v
        gabs = (Gd[nm].abs() + (wd * P[nm].abs() if flags[i] & 1 else 0))
        trust_lr = (step - mom * Vd[nm]).abs().sum() / gabs.sum().clamp_min(1e-300) if float(gabs.sum()) > 0 else 0.0
        Av = mom * Vd[nm].abs() + trust_lr * gabs
        sub = Checks()
        sub.close('v', V[i], V1[nm], Av, 0, TAU_LARS)
        sub.close('w', W[i], P1[nm], P[nm].abs() + Av, 0, TAU_LARS)
        rv, rw = sub.items[0][1], sub.items[1][1]
        if rv >= worst_v[0]:
            worst_v = (rv, (i, nm, numels[i]) + sub.items[0][2])
        if rw >= worst_w[0]:
            worst_w = (rw, (i, nm, numels[i]) + sub.items[1][2])
    chk.items.append(('v (momentum)', worst_v[0], worst_v[1]))
    chk.items.append(('w', worst_w[0], worst_w[1]))


def r_lars_apply(a, big, pz, chk, seed=0):
    lars_case(a['numels'], a['flags'], chk, a['momentum'], a['weight_decay'], a['eeta'], seed=seed)
    return sum(a['numels'])


# ---------------------------------------------------------------------------------------------------
# input preparation
# ---------------------------------------------------------------------------------------------------
def r_input_prep(a, big, pz, chk, seed=0):
    from oracle import data_util as OD
    from simclr_b200._lib import lib, stream_ptr
    B, H, W, T, dt = a['B'], a['H'], a['W'], a['T'], DT[a['dtype']]
    g = torch.Generator().manual_seed(seed + B + H)
    f = torch.rand(B, H, W, 3 * T, generator=g, dtype=F64)
    sigma = [0.4 + 1.3 * t for t in range(T)]
    sel = (torch.arange(T * B).view(T, B) + torch.arange(T).view(T, 1)) % 2
    out = _nan((T * B, H, W, 4), dt)
    tmp = _nan((T * B, H, W, 3), F32)
    fd = f.float().cuda()
    lib.input_prep(fd, out, a['dtype'], B, H, W, T, a['use_blur'], a['blur_kernel_size'],
                   torch.tensor(sigma, device='cuda'), sel.to(torch.uint8).cuda().contiguous(), tmp, stream_ptr())
    views = list(torch.split(fd.double().cpu(), 3, dim=-1))
    if a['use_blur']:
        assert a['blur_kernel_size'] == H // 10
        views = OD.batch_random_blur(views, H, W, draws=[(sigma[t], sel[t]) for t in range(T)])
    ref = torch.cat(views, 0).cuda()
    chk.close('out', out[..., :3], ref, ref.abs(), RHO[dt], 2.0 ** -19)    # expf weights (2 ulp) and two 1-D sums
    chk.exact('pad channel', out[..., 3], torch.zeros((T * B, H, W), device='cuda'))
    return B


# ---------------------------------------------------------------------------------------------------
REPLAY = {
    'bn_stats': r_bn_stats,
    'bn_finalize': r_bn_finalize,
    'bn_apply': r_bn_apply,
    'bn_apply_relu_mask': lambda a, big, pz, chk, seed=0: r_bn_apply(a, big, pz, chk, seed, 'bn_apply_relu_mask'),
    'bn_apply2_relu_mask': r_bn_apply2,
    'bn_bwd_reduce': r_bn_bwd_reduce,
    'bn_bwd_reduce_bits': lambda a, big, pz, chk, seed=0: r_bn_bwd_reduce(a, big, pz, chk, seed, 'bn_bwd_reduce_bits'),
    'bn_bwd_reduce2_bits': lambda a, big, pz, chk, seed=0: r_bn_bwd_reduce(a, big, pz, chk, seed, 'bn_bwd_reduce2_bits'),
    'bn_bwd_relu_reduce': r_bn_bwd_relu_reduce,
    'bn_bwd_coef': r_bn_bwd_coef,
    'bn_bwd_apply': r_bn_bwd_apply,
    'bn_bwd_apply_coef': r_bn_bwd_apply_coef,
    'bn_bwd_apply2_coef': r_bn_bwd_apply2_coef,
    'bn_relu_maxpool_fwd': r_bn_relu_maxpool_fwd,
    'maxpool_bn_bwd_reduce': r_maxpool_bn_bwd_reduce,
    'maxpool_bn_bwd_apply': r_maxpool_bn_bwd_apply,
    'maxpool3x3s2_fwd': r_maxpool3x3s2_fwd,
    'maxpool3x3s2_bwd': r_maxpool3x3s2_bwd,
    'global_avgpool_fwd': r_global_avgpool_fwd,
    'global_avgpool_bwd': r_global_avgpool_bwd,
    'avgpool2x2_fwd': r_avgpool2x2_fwd,
    'avgpool2x2_bwd': r_avgpool2x2_bwd,
    'sk_pool': r_sk_pool,
    'sk_mix_fwd': r_sk_mix_fwd,
    'sk_mix_bwd_reduce': r_sk_mix_bwd_reduce,
    'sk_mix_bwd_apply': r_sk_mix_bwd_apply,
    'cast': r_cast,
    'add_inplace': r_add_inplace,
    'axpy': r_axpy,
    'l2_loss': r_l2_loss,
    'relu_inplace': r_relu_inplace,
    'bias_add': r_bias_add,
    'bias_grad': r_bias_grad,
    'softmax_xent': r_softmax_xent,
    'ntxent_normalize': r_ntxent_normalize,
    'ntxent_forward': r_ntxent_fwd_bwd,
    'ntxent_backward': r_ntxent_fwd_bwd,
    'ntxent_labels': r_ntxent_labels,
    'contrast_metrics': r_contrast_metrics,
    'lars_apply': r_lars_apply,
    'input_prep': r_input_prep,
}
SUMS_ENTRIES = ('bn_stats', 'bn_bwd_reduce', 'bn_bwd_reduce_bits', 'bn_bwd_reduce2_bits', 'bn_bwd_relu_reduce',
                'maxpool_bn_bwd_reduce')
NO_LARGE = ('lars_apply', 'l2_loss', 'input_prep', 'bn_finalize', 'bn_bwd_coef')    # per-tensor / per-channel sizes


def _run_replays(items, what):
    """items: [(label, fn, args dict, big, pz)].  Prints the worst ratio per replay; fails listing every offender."""
    bad, worst = [], (0.0, None)
    t0 = time.time()
    for label, fn, a, big, pz in items:
        chk = Checks()
        size = fn(a, big, pz, chk)
        w = chk.worst()
        print('    %-110s size %9d  worst |err|/bound %.3f (%s at %s)' % (label[:110], size, w[1], w[0], w[2]))
        if w[1] > worst[0]:
            worst = (w[1], label)
        offenders = [it for it in chk.items if not it[1] <= 1.0]
        if offenders:
            bad.append((label, size, offenders))
        torch.cuda.empty_cache()
    print('%s: %d replays, worst |err|/bound %.3f (%s), %.1f s' % (what, len(items), worst[0], worst[1], time.time() - t0))
    assert not bad, bad


@pytest.mark.parametrize('size', ['recorded', 'large'])
@pytest.mark.parametrize('family', list(FAMILIES))
def test_launches_vs_fp64(inventory, family, size):
    """Each distinct non-conv launch of the family's step, per element against fp64."""
    big = size == 'large'
    items, seen = [], set()
    for key in sorted(inventory[family], key=_fmt):
        name, it, pz = key
        if name not in REPLAY or (big and name in NO_LARGE):
            continue
        a = dict(it)
        if name in ('ntxent_forward', 'ntxent_backward'):      # one replay covers both
            dedup = ('ntxent', a['B'], a['R'], a['D'], a['temperature'])
            if dedup in seen:
                continue
            seen.add(dedup)
        items.append((_fmt(key), REPLAY[name], a, big, 0))
        if pz:
            items.append((_fmt(key) + ' [into a pre-zeroed slice]', REPLAY[name], a, big, 1))
    assert items
    _run_replays(items, '%s at the %s size' % (family, size))


# ---------------------------------------------------------------------------------------------------
# hand-picked edges beyond the inventory
# ---------------------------------------------------------------------------------------------------
def _rows_per_block(rows, C):
    cvecs, P = C // 8, 1
    while P * 2 <= cvecs and P * 2 <= 256:
        P *= 2
    nb = min(max((rows + (256 // P) * 8 - 1) // ((256 // P) * 8), 1), 2 * _sms())
    return (rows + nb - 1) // nb


def _bn_edge_items():
    items = []
    for C in (8, 24, 72, 520):
        big = _red_threshold(C) + 1
        rpb = _rows_per_block(big, C)
        # the last block holds one row
        short = (big // rpb) * rpb + 1
        for rows in (1, 7, 255, short):
            for dt in (0, 1):
                b = dict(rows=rows, C=C)
                items.append(('bn_stats C %d rows %d dtype %d' % (C, rows, dt), r_bn_stats, dict(b, dtype=dt), False, 0))
                items.append(('bn_bwd_reduce_bits C %d rows %d dtype %d' % (C, rows, dt), REPLAY['bn_bwd_reduce_bits'],
                              dict(b, dtype=dt, y_dtype=dt, dz2=True), False, 1))
                items.append(('bn_bwd_relu_reduce C %d rows %d dtype %d' % (C, rows, dt), r_bn_bwd_relu_reduce,
                              dict(b, dtype=dt, y_dtype=1 - dt), False, 0))
                items.append(('bn_apply_relu_mask C %d rows %d dtype %d' % (C, rows, dt), REPLAY['bn_apply_relu_mask'],
                              dict(b, y_dtype=dt, z_dtype=dt, residual=True), False, 0))
        # element-wise kernels past the 16 * SMs grid cap; C = 520 (65 vectors) never lets ew_grid_c fix the channel
        rows = _ew_threshold_rows(C) * 2 + 3
        for yd in (0, 1):
            for zd in (0, 1):
                items.append(('bn_apply C %d rows %d y %d z %d' % (C, rows, yd, zd), r_bn_apply,
                              dict(rows=rows, C=C, y_dtype=yd, z_dtype=zd, residual=True, relu=1), False, 0))
        items.append(('bn_apply2_relu_mask C %d rows %d' % (C, rows), r_bn_apply2,
                      dict(rows=rows, C=C, y_dtype=1, z_dtype=1), False, 0))
        items.append(('bn_bwd_apply2_coef C %d rows %d' % (C, rows), r_bn_bwd_apply2_coef,
                      dict(rows=rows, C=C, dtype=1, y_dtype=1, dy_dtype=1), False, 0))
    # every (dz, y, dy) dtype combination of the BatchNorm backward apply, with and without the recomputed mask
    for key in range(8):
        d, yd, o = key >> 2, (key >> 1) & 1, key & 1
        for masked in (False, True):
            b = dict(rows=3001, C=72, dtype=d, y_dtype=yd, dy_dtype=o, mask_scale=masked)
            items.append(('bn_bwd_apply_coef dz %d y %d dy %d mask %d' % (d, yd, o, masked), r_bn_bwd_apply_coef, b, False, 0))
            items.append(('bn_bwd_apply dz %d y %d dy %d mask %d' % (d, yd, o, masked), r_bn_bwd_apply,
                          dict(b, count=3001.0), False, 0))
    # reductions over every dtype pair of dz / y, with and without dz2 and the z mask
    for d in (0, 1):
        for yd in (0, 1):
            for two in (False, True):
                for zm in (False, True):
                    items.append(('bn_bwd_reduce dz %d y %d dz2 %d z %d' % (d, yd, two, zm), r_bn_bwd_reduce,
                                  dict(rows=4099, C=64, dtype=d, y_dtype=yd, dz2=two, relu_mask_z=zm), False, 0))
    # bn_finalize with gamma / beta / moving statistics absent
    for gm in (False, True):
        items.append(('bn_finalize gamma/beta %d' % gm, r_bn_finalize,
                      dict(C=72, count=1234.0, gamma=gm, beta=gm, moving_mean=gm, moving_var=gm, eps=1.001e-5,
                           momentum=0.9), False, 0))
        items.append(('bn_bwd_coef gamma %d' % gm, r_bn_bwd_coef,
                      dict(C=72, count=1234.0, gamma=gm, dgamma=gm, dbeta=gm), False, 0))
    return items


def test_batchnorm_edges_vs_fp64():
    _run_replays(_bn_edge_items(), 'BatchNorm edges')


@pytest.mark.parametrize('dtype,sigma', [(F32, 1e-2), (BF16, 10.0)])      # bf16 resolves 4 at 1e3
def test_bn_stats_pivot(dtype, sigma):
    """Nearly constant channels (mean 1e3, sigma << mean) whose row 0 -- the pivot -- is a 50-sigma outlier: the
    variance taken from the fp64 sums keeps its digits.  Without the pivot shift the fp32 squares would lose them."""
    from simclr_b200._lib import lib, stream_ptr
    C = 64
    for rows in (255, _red_threshold(C) + 1):
        g = _gen(rows)
        x = (1e3 + torch.randn(rows, C, generator=g, device='cuda') * sigma)
        x[0] += 50 * sigma
        x = x.to(dtype)
        sums = _nan((2 * C,), F64)
        lib.bn_stats(x, 1 if dtype == BF16 else 0, rows, C, sums, stream_ptr())
        xd = x.double()
        var_ref = xd.var(0, unbiased=False)
        m = sums[:C] / rows
        var = sums[C:] / rows - m * m
        u = xd - xd[0]
        # errors of the shifted fp32 sums (TAU_RED of sum u^2 and of 2 |mean u| sum |u|), carried into the variance
        A = ((u * u).sum(0) + 2 * (u.sum(0) / rows).abs() * u.abs().sum(0)) / rows
        r, w = _ratio(var, var_ref, A, 0.0, TAU_RED)
        print('bn_stats pivot %s rows %d: worst |var err| / bound %.3f at %s; var %.3g, bound/var %.2g' % (
            dtype, rows, r, w, float(var_ref.mean()), float((TAU_RED * A / var_ref).max())))
        assert r <= 1.0
        assert float((TAU_RED * A / var_ref).max()) < 0.1       # the bound is meaningful for these channels


STEM_EDGES = [(N, H, W, C, dt, two) for (H, W) in ((112, 112), (112, 111), (111, 112), (111, 111))
              for C in (64, 128) for two in (False, True) for (N, dt) in ((2, 1),)] + \
             [(3, 28, 27, 24, 1, True), (3, 27, 28, 32, 0, True), (2, 29, 29, 64, 0, False)]


@pytest.mark.parametrize('N,H,W,C,dtype,two', STEM_EDGES)
def test_fused_stem_vs_fp64(N, H, W, C, dtype, two):
    """The fused stem at all four (H, W) parities (each an instance of maxpool_bn_bwd_apply_bf16_kernel), with and
    without the second gradient, the generic bf16 forward (C = 24: 256 % (C / 8) != 0, no ysel), fp32, and windows
    that are all zero (ties) -- forward, both reductions and the apply against fp64."""
    a = dict(N=N, H=H, W=W, C=C, dtype=dtype, d2=two)
    fast = dtype == 1 and 256 % (C // 8) == 0
    bwd = 256 % (C // (8 if dtype == 1 else 4)) == 0          # the backward kernels need C / V dividing 256
    items = [('fwd', lambda *x, **k: r_bn_relu_maxpool_fwd(*x, zero_windows=True), dict(a, ysel=fast), False, 0)]
    if bwd:
        items.append(('reduce per pixel', lambda *x, **k: r_maxpool_bn_bwd_reduce(*x, zero_windows=True),
                      dict(a, ysel=False), False, 1))
    if fast:
        items.append(('reduce pooled', lambda *x, **k: r_maxpool_bn_bwd_reduce(*x, zero_windows=True),
                      dict(a, ysel=True), False, 1))
    if bwd:
        items.append(('apply', lambda *x, **k: r_maxpool_bn_bwd_apply(*x, zero_windows=True), a, False, 0))
    _run_replays([('stem %s %s' % (lbl, (N, H, W, C, dtype, two)), f, x, b, p) for lbl, f, x, b, p in items], 'stem edge')


@pytest.mark.parametrize('f', [128, 256])
def test_sk_bf16_56(f):
    a = dict(N=4, HW=56 * 56, f=f, dtype=1)
    _run_replays([('%s f %d' % (n, f), REPLAY[n], a, False, 0) for n in
                  ('sk_pool', 'sk_mix_fwd', 'sk_mix_bwd_reduce', 'sk_mix_bwd_apply')], 'SK at 56x56')


@pytest.mark.parametrize('H,W', [(7, 9), (9, 7), (13, 13), (56, 55)])
@pytest.mark.parametrize('stride', [1, 2])
@pytest.mark.parametrize('dtype', [0, 1])
def test_avgpool2x2_odd(H, W, stride, dtype):
    a = dict(N=3, H=H, W=W, C=64, stride=stride, dtype=dtype)
    _run_replays([('avgpool2x2_fwd', r_avgpool2x2_fwd, a, False, 0), ('avgpool2x2_bwd', r_avgpool2x2_bwd, a, False, 0)],
                 'avgpool2x2 %dx%d/%d' % (H, W, stride))


NTX_EDGES = [(1, 1, 128, 0.1, True, 1.0), (31, 1, 1, 0.5, True, 1.0), (33, 1, 256, 0.1, True, 1.0),
             (256, 1, 128, 0.1, True, 1.0), (512, 1, 128, 0.1, True, 1.0), (33, 2, 128, 0.2, True, 1.0),
             (256, 8, 128, 0.1, True, 1.0), (64, 1, 128, 0.1, False, 0.05), (16, 2, 128, 0.1, False, 0.05)]


@pytest.mark.parametrize('B,R,D,temp,norm,hscale', NTX_EDGES)
def test_ntxent_vs_fp64(B, R, D, temp, norm, hscale):
    """Every replica's normalize / forward / metrics / backward.  R = 8 at B = 256 is bench --gpus 8 (G = 2048);
    hidden_norm = 0 with |h| up to ~10 / temperature keeps logits large (max-subtraction)."""
    chk = Checks()
    if not norm:
        hscale = 1.0 / math.sqrt(D) * 3.0            # |logit| up to ~10 / temperature: the LSE must subtract its max
    splits = ntxent_case(B, R, D, temp, norm, chk, metrics=True, hscale=hscale)
    w = chk.worst()
    print('ntxent B %d R %d D %d: %d column splits, worst |err|/bound %.3f (%s at %s)' % (B, R, D, splits, w[1], w[0], w[2]))
    if 2 * R * B >= 1024:
        assert splits > 1
    assert all(it[1] <= 1.0 for it in chk.items), [it for it in chk.items if not it[1] <= 1.0]


@pytest.mark.parametrize('classes', [10, 1000, 1001])
@pytest.mark.parametrize('big_logits', [False, True])
def test_softmax_xent_vs_fp64(classes, big_logits):
    chk = Checks()
    softmax_xent_case(66, 33, classes, 1.0 / 66, chk, big_logits=big_logits)
    assert all(it[1] <= 1.0 for it in chk.items), chk.items


def _r50_2x_numels_flags():
    from simclr_b200 import run, flags_def, engine
    from oracle import lars as L
    F = flags_def.FLAGS
    if not F.is_parsed():
        F(['test'])
    saved = {k: getattr(F, k) for k in flags_def.REFERENCE_FLAG_NAMES + ['b200_precision', 'b200_conv_engine']}
    try:
        flags_def.set_flags(train_batch_size=2, optimizer='lars', weight_decay=1e-4, image_size=224, resnet_depth=50,
                            width_multiplier=2, sk_ratio=0.0, b200_precision='bf16', b200_conv_engine='tc')
        engine.set_engine(engine.Engine(precision='bf16', conv_engine='tc'))
        trainer = run.Trainer(num_classes=1000, num_examples=50000, seed=0)
        vs = trainer.model.trainable_variables
        numels = [v.numel for v in vs]
        flags = [3 if L._use_weight_decay(v.name, 1e-4, L.LARS_EXCLUDE) else 0 for v in vs]
        del trainer
    finally:
        for k, v in saved.items():
            setattr(F, k, v)
    torch.cuda.empty_cache()
    return numels, flags


def test_lars_edges_vs_fp64():
    """The full R50 2x parameter table; plus tensors whose base is one float off (float4 path off), numel % 4 != 0,
    all-zero weights (trust 1) and all-zero gradients."""
    numels, flags = _r50_2x_numels_flags()
    chk = Checks()
    lars_case(numels, flags, chk)
    extra_n = [5, 1027, 16384 * 2 + 3, 777, 4096, 4096, 130]
    extra_f = [3, 3, 3, 0, 3, 3, 3]
    lars_case(extra_n, extra_f, chk, offset=(1, 2, 3), zero_w=(4,), zero_g=(5,), seed=1)
    lars_case(extra_n, [2 if f else 0 for f in extra_f], chk, weight_decay=0.0, offset=(0, 2), seed=2)
    for it in chk.items:
        print('    lars %-14s worst |err|/bound %.3f at %s' % it)
    assert all(it[1] <= 1.0 for it in chk.items), chk.items


def test_l2_loss_whole_r50_2x():
    numels, _ = _r50_2x_numels_flags()
    chk = Checks()
    r_l2_loss(dict(n=sum(numels)), False, 0, chk)
    print('l2_loss over %d: %.3f' % (sum(numels), chk.items[0][1]))
    assert chk.items[0][1] <= 1.0
