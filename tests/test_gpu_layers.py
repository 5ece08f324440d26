"""Every tensor-core conv launch of the benchmarked networks against an fp64 reference, element by element,
and bitwise reproducibility of the bf16 training step.

The inventory is taken from the model itself: one eager bf16 / `tc` step per benchmarked family at 2 samples
(4 views), with `conv2d_{fprop,dgrad,wgrad}_tc` wrapped to record every launch.  Each distinct launch is then
replayed as the step issues it (same dtypes, fused BatchNorm sums where the step fuses them, bf16 dX, fp32 dW)
on seeded inputs, at the recorded batch and at a batch with more 128-row tiles than the GPU has SMs, into
NaN-filled outputs, and compared per element with torch's own convolution in float64 on the GPU.  Inside a step
`Engine.begin_step` switches `set_accumulate_prezeroed(1)` on: every fused-sums fprop then adds into a slice of the
zeroed sums pool and every wgrad into a slice of the zeroed flat gradient buffer.  Each launch is replayed in every
mode the step ran it in, and a fused fprop or wgrad also with the mode off (the call zeroes its own output):

    |got - ref| <= rho * |ref| + tau * A

A is the same operation in fp64 on absolute values (|x| with |w|, |dy| with |w|, |x| with |dy|).  bf16 x bf16
products are exact in fp32, so fp32 accumulation is the only error of an fp32 output (rho = 0); a bf16 output
adds one rounding (rho = 2^-8, the unit roundoff of bf16).  A wrong tap, a dropped split partial or a wrong
pixel is off by O(A / sqrt(K)): above 1e-3 A for any reduction length K up to 1e6, far above tau.  A bf16 output
rounded by almost half an ulp sits just below a ratio of 1 by construction; the fp32 outputs measure tau.
"""
import math
import time

import pytest
import torch

from test_gpu_kernels import conv_reference
from test_gpu_tc import _pack

pytestmark = pytest.mark.gpu

BF16, F32 = torch.bfloat16, torch.float32
RHO = {BF16: 2.0 ** -8, F32: 0.0}
# fp32 accumulation allowance, in units of A.  Measured on an H100 SXM (80 GB HBM3, 700 W): the worst fp32-output
# launch of the inventory erred by 0.096 * 2^-16 A (the wgrad of the SK 3x3 512->1024 at 14x14, N 87: a reduction
# over 17052 pixels); the 4096-deep dense layers of the heads by 0.046 * 2^-16 A.  2^-17 keeps a 5x margin.
TAU = 2.0 ** -17
SUMS_TOL = 1e-5                      # fused BatchNorm sums against the fp64 sums of the stored outputs
MACS_BUDGET = 1e11                   # multiply-adds per launch at the larger batch (fp64 reference time and memory)

# the benchmarked families of bench.py (GFLOP_PER_IMAGE).  R152 2x SK has the per-stage block shapes of
# R50 2x SK, only more blocks per stage, so R50 2x SK stands in for it here.
FAMILIES = {
    'r50_1x_224': dict(resnet_depth=50, width_multiplier=1, image_size=224, sk_ratio=0.0),
    'r50_2x_224': dict(resnet_depth=50, width_multiplier=2, image_size=224, sk_ratio=0.0),
    'r50_2x_sk_224': dict(resnet_depth=50, width_multiplier=2, image_size=224, sk_ratio=0.0625),
}

KINDS = ('conv2d_fprop_tc', 'conv2d_dgrad_tc', 'conv2d_wgrad_tc')


def _launch_key(name, a):
    """(kind, H, W, Cs, Cin, Cout, R, S, stride, in dtype, out dtype, fused sums) and N of one recorded call."""
    if name == 'conv2d_fprop_tc':
        x, wf, y, _, _, N, H, W, Cs, Cout, R, S, s, sums, _ = a
        Cin = 3 if Cs == 4 else Cs              # the stem stores its 3 image channels as 4
        return ('fprop', H, W, Cs, Cin, Cout, R, S, s, x.dtype, y.dtype, sums is not None), N
    if name == 'conv2d_dgrad_tc':
        dy, wd, dx, _, _, N, H, W, Cin, Cout, R, S, s, _ = a
        return ('dgrad', H, W, Cin, Cin, Cout, R, S, s, dy.dtype, dx.dtype, False), N
    x, dy, dw, _, N, H, W, Cs, Cin, Cout, R, S, s, _ = a
    return ('wgrad', H, W, Cs, Cin, Cout, R, S, s, x.dtype, dw.dtype, False), N


def _fmt(key):
    kind, H, W, Cs, Cin, Cout, R, S, s, din, dout, fused = key
    dt = {BF16: 'bf16', F32: 'f32'}
    return '%s %3dx%-3d Cs %4d Cin %4d Cout %4d %dx%d/%d %s->%s%s' % (
        kind, H, W, Cs, Cin, Cout, R, S, s, dt[din], dt[dout], ' +sums' if fused else '')


@pytest.fixture(scope='module')
def inventory():
    """{family: ({launch key: N}, {launch key: set of pre-zeroed modes})}: every tensor-core conv launch of one
    eager bf16 / tc step per family."""
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
                                b200_precision='bf16', b200_conv_engine='tc', **cfg)
            engine.set_engine(engine.Engine(precision='bf16', conv_engine='tc'))
            trainer = run.Trainer(num_classes=1000, num_examples=50000, seed=0)
            g = torch.Generator().manual_seed(3)
            f = torch.rand(B, S, S, 6, generator=g).cuda()
            lab = torch.nn.functional.one_hot(torch.randint(0, 1000, (B,), generator=g), 1000).float().cuda()
            launches, modes = {}, {}
            state = {'pz': 0}
            with pytest.MonkeyPatch.context() as mp:
                setpz = getattr(lib, 'set_accumulate_prezeroed')

                def wrap_pz(on, _fn=setpz):
                    state['pz'] = int(on)
                    return _fn(on)
                mp.setattr(lib, 'set_accumulate_prezeroed', wrap_pz)
                for name in KINDS:
                    fn = getattr(lib, name)             # _Lib.__getattr__ caches the bound call on the instance

                    def wrap(*a, _fn=fn, _name=name):
                        key, N = _launch_key(_name, a)
                        launches[key] = max(N, launches.get(key, 0))
                        modes.setdefault(key, set()).add(state['pz'])
                        return _fn(*a)
                    mp.setattr(lib, name, wrap)
                trainer.single_step(f, lab)
                torch.cuda.synchronize()
            inv[fam] = (launches, modes)
            del trainer
            torch.cuda.empty_cache()
    finally:
        for k, v in saved.items():
            setattr(F, k, v)
        lib.set_accumulate_prezeroed(0)
    for fam, (launches, modes) in inv.items():
        print('\n%s: %d distinct tensor-core conv launches' % (fam, len(launches)))
        for key in sorted(launches, key=_fmt):
            print('    N %3d  %-70s prezeroed %s' % (launches[key], _fmt(key), sorted(modes[key])))
    return inv


def _has(launches, kind, pred):
    return any(k[0] == kind and pred(*k[1:]) for k in launches)


# what the networks must keep launching: the shapes that only these configurations reach
LANDMARKS = {
    'r50_1x_224': [
        ('1x1 stride-1 dgrad, bf16 dX', 'dgrad', lambda H, W, Cs, Cin, Co, R, S, s, di, do, f: R == 1 and s == 1 and do == BF16),
        ('generic 3x3 dgrad at 256 channels, bf16 dX', 'dgrad',
         lambda H, W, Cs, Cin, Co, R, S, s, di, do, f: (H, Cin, Co, R, s, do) == (14, 256, 256, 3, 1, BF16)),
        ('generic 3x3 dgrad at 512 channels, bf16 dX', 'dgrad',
         lambda H, W, Cs, Cin, Co, R, S, s, di, do, f: (H, Cin, Co, R, s, do) == (7, 512, 512, 3, 1, BF16)),
        ('strided 3x3 dgrad, bf16 dX', 'dgrad', lambda H, W, Cs, Cin, Co, R, S, s, di, do, f: R == 3 and s == 2 and do == BF16),
        ('strided 1x1 projection dgrad, bf16 dX', 'dgrad',
         lambda H, W, Cs, Cin, Co, R, S, s, di, do, f: R == 1 and s == 2 and do == BF16),
        ('7x7/2 stem at 224, 64 outputs', 'fprop', lambda H, W, Cs, Cin, Co, R, S, s, di, do, f: (H, Cs, Co, R, s) == (224, 4, 64, 7, 2)),
        ('stage-4 conv at 7x7', 'fprop', lambda H, W, Cs, Cin, Co, R, S, s, di, do, f: (H, W, R) == (7, 7, 3)),
    ],
    'r50_2x_224': [
        ('128->128 halo 3x3 at 56x56', 'fprop', lambda H, W, Cs, Cin, Co, R, S, s, di, do, f: (H, W, Cin, Co, R, s) == (56, 56, 128, 128, 3, 1)),
        ('128->128 halo 3x3 dgrad at 56x56, bf16 dX', 'dgrad',
         lambda H, W, Cs, Cin, Co, R, S, s, di, do, f: (H, W, Cin, Co, R, s, do) == (56, 56, 128, 128, 3, 1, BF16)),
        ('128->128 halo 3x3 wgrad at 56x56', 'wgrad', lambda H, W, Cs, Cin, Co, R, S, s, di, do, f: (H, W, Cin, Co, R, s) == (56, 56, 128, 128, 3, 1)),
        ('7x7/2 stem at 224, 128 outputs', 'fprop', lambda H, W, Cs, Cin, Co, R, S, s, di, do, f: (H, Cs, Co, R, s) == (224, 4, 128, 7, 2)),
        ('7x7/2 stem wgrad at 224, 128 outputs', 'wgrad', lambda H, W, Cs, Cin, Co, R, S, s, di, do, f: (H, Cs, Co, R, s) == (224, 4, 128, 7, 2)),
        ('stage-4 conv at 7x7', 'fprop', lambda H, W, Cs, Cin, Co, R, S, s, di, do, f: (H, W, R) == (7, 7, 3)),
    ],
    'r50_2x_sk_224': [
        ('ResNet-D 3x3/2 stem on 4 stored channels', 'fprop', lambda H, W, Cs, Cin, Co, R, S, s, di, do, f: (H, Cs, R, s) == (224, 4, 3, 2)),
        ('ResNet-D 3x3/2 stem wgrad', 'wgrad', lambda H, W, Cs, Cin, Co, R, S, s, di, do, f: (H, Cs, R, s) == (224, 4, 3, 2)),
        ('SK 3x3 with Cout = 2 Cin', 'fprop', lambda H, W, Cs, Cin, Co, R, S, s, di, do, f: R == 3 and Co == 2 * Cin),
        ('SK mixing dense, 32 outputs', 'fprop', lambda H, W, Cs, Cin, Co, R, S, s, di, do, f: (H, W, R, Co) == (1, 1, 1, 32)),
        ('SK mixing dense, 64 outputs', 'fprop', lambda H, W, Cs, Cin, Co, R, S, s, di, do, f: (H, W, R, Co) == (1, 1, 1, 64)),
        ('SK mixing dense back to 2f streams, fp32 logits', 'fprop',
         lambda H, W, Cs, Cin, Co, R, S, s, di, do, f: (H, W, R, do) == (1, 1, 1, F32) and Cin in (32, 64) and Co >= 256),
        ('stage-4 conv at 7x7', 'fprop', lambda H, W, Cs, Cin, Co, R, S, s, di, do, f: (H, W, R) == (7, 7, 3)),
    ],
}


@pytest.mark.parametrize('family', list(FAMILIES))
def test_inventory_landmarks(inventory, family):
    launches, modes = inventory[family]
    missing = [what for what, kind, pred in LANDMARKS[family] if not _has(launches, kind, pred)]
    assert not missing, '%s no longer launches: %s' % (family, missing)
    # the bf16 step writes bf16 dX from every dgrad and fp32 dW from every wgrad
    assert all(k[10] == BF16 for k in launches if k[0] == 'dgrad'), family
    assert all(k[10] == F32 for k in launches if k[0] == 'wgrad'), family
    # every wgrad adds into the step's zeroed flat gradient buffer and every fused fprop into its zeroed sums pool
    acc = [k for k in launches if accumulates(k)]
    assert any(k[0] == 'wgrad' for k in acc) and any(k[0] == 'fprop' for k in acc), family
    assert all(modes[k] == {1} for k in acc), [(_fmt(k), modes[k]) for k in acc if modes[k] != {1}]


# ---------------------------------------------------------------------------------------------------
# replay of one launch against fp64
# ---------------------------------------------------------------------------------------------------
def _ratio(got, ref, A, rho, tau):
    """max |got - ref| / (rho |ref| + tau A) and the index of that element; an element whose bound is 0
    (ref = A = 0) must be exactly 0; a NaN (never written) or Inf is an infinite ratio."""
    g = got.double()
    err = (g - ref).abs()
    bound = rho * ref.abs() + tau * A
    r = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
    r = torch.where(torch.isfinite(g), r, torch.full_like(r, math.inf))
    i = int(torch.argmax(r))
    return float(r.reshape(-1)[i]), tuple(int(v) for v in torch.unravel_index(torch.tensor(i), got.shape))


def _ref_dx(dy, w, k, s, x_shape):
    x = torch.zeros(x_shape, dtype=torch.float64, device='cuda', requires_grad=True)
    return torch.autograd.grad(conv_reference(x, w, k, s), x, dy)[0]


def _ref_dw(x, dy, k, s, w_shape):
    w = torch.zeros(w_shape, dtype=torch.float64, device='cuda', requires_grad=True)
    return torch.autograd.grad(conv_reference(x, w, k, s), w, dy)[0]


def accumulates(key):
    """True for the launches whose output depends on the pre-zeroed mode: wgrads and fprops with fused sums."""
    return key[0] == 'wgrad' or (key[0] == 'fprop' and key[11])


GUARD = 64          # NaN elements on each side of a pre-zeroed output slice


def _zeroed_slice(n, dtype):
    """A zeroed slice of a NaN-filled buffer, as the step's pools hand out sums and dW; returns (slice, guards)."""
    buf = torch.full((GUARD + n + GUARD,), float('nan'), dtype=dtype, device='cuda')
    buf[GUARD:GUARD + n].zero_()
    return buf[GUARD:GUARD + n], (buf[:GUARD], buf[GUARD + n:])


def check_launch(key, N, seed=0, prezeroed=0):
    """Replays one launch at batch N into NaN-filled outputs.  Returns (worst bound ratio, location, sums
    error) -- the sums error is max |S - sum| / allowance over channels, None without fused sums.
    prezeroed = 1 replays it as the step issues it: with set_accumulate_prezeroed(1), fused sums into a zeroed
    slice of a NaN fp64 buffer and dW into a zeroed slice of a NaN flat buffer; an overwritten NaN guard of
    either is an infinite ratio."""
    from simclr_b200._lib import lib, stream_ptr, DTYPE_CODE
    kind, H, W, Cs, Cin, Cout, R, S, s, din, dout, fused = key
    assert R == S and din == BF16, key
    Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
    g = torch.Generator(device='cuda').manual_seed(seed + sum(v for v in key if type(v) is int))
    x = torch.randn(N, H, W, Cin, generator=g, device='cuda').to(BF16)
    w = (torch.randn(R, S, Cin, Cout, generator=g, device='cuda') * (1.0 / (R * S * Cin) ** 0.5)).to(BF16)
    dy = torch.randn(N, Ho, Wo, Cout, generator=g, device='cuda').to(BF16)
    xs = x if Cs == Cin else torch.cat([x, torch.zeros(N, H, W, Cs - Cin, dtype=BF16, device='cuda')], -1).contiguous()
    x64, w64, dy64 = x.double(), w.double(), dy.double()
    st = stream_ptr()
    # mode 0: the calls zero their own accumulation outputs
    prev = lib.set_accumulate_prezeroed(prezeroed)
    guards = ()
    sums_err = None
    if kind == 'fprop':
        wf, _ = _pack(w, BF16, R, Cin, Cs, Cout, want_wd=False)
        got = torch.full((N, Ho, Wo, Cout), float('nan'), dtype=dout, device='cuda')
        sums = None
        if fused and prezeroed:
            sums, guards = _zeroed_slice(2 * Cout, torch.float64)
        elif fused:
            sums = torch.full((2 * Cout,), float('nan'), dtype=torch.float64, device='cuda')
        try:
            lib.conv2d_fprop_tc(xs, wf, got, DTYPE_CODE[din], DTYPE_CODE[dout], N, H, W, Cs, Cout, R, S, s, sums, st)
        finally:
            lib.set_accumulate_prezeroed(prev)
        ref = conv_reference(x64, w64, R, s)
        A = conv_reference(x64.abs(), w64.abs(), R, s)
        if fused:
            torch.cuda.synchronize()
            yf = got.double().reshape(-1, Cout)
            d = sums - torch.cat([yf.sum(0), (yf * yf).sum(0)])
            r = d.abs() / (SUMS_TOL * torch.cat([yf.abs().sum(0), (yf * yf).sum(0)]))
            sums_err = float(torch.where(d == 0, 0.0, r.nan_to_num(nan=math.inf)).max())     # NaN: never written
    elif kind == 'dgrad':
        _, wd = _pack(w, BF16, R, Cin, Cs, Cout)
        got = torch.full((N, H, W, Cin), float('nan'), dtype=dout, device='cuda')
        try:
            lib.conv2d_dgrad_tc(dy, wd, got, DTYPE_CODE[din], DTYPE_CODE[dout], N, H, W, Cin, Cout, R, S, s, st)
        finally:
            lib.set_accumulate_prezeroed(prev)
        ref = _ref_dx(dy64, w64, R, s, (N, H, W, Cin))
        A = _ref_dx(dy64.abs(), w64.abs(), R, s, (N, H, W, Cin))
    else:
        if prezeroed:
            got, guards = _zeroed_slice(R * S * Cin * Cout, dout)
            got = got.view(R, S, Cin, Cout)
        else:
            got = torch.full((R, S, Cin, Cout), float('nan'), dtype=dout, device='cuda')
        try:
            lib.conv2d_wgrad_tc(xs, dy, got, DTYPE_CODE[din], N, H, W, Cs, Cin, Cout, R, S, s, st)
        finally:
            lib.set_accumulate_prezeroed(prev)
        ref = _ref_dw(x64, dy64, R, s, (R, S, Cin, Cout))
        A = _ref_dw(x64.abs(), dy64.abs(), R, s, (R, S, Cin, Cout))
    torch.cuda.synchronize()
    ratio, where = _ratio(got, ref, A, RHO[dout], TAU)
    if not all(bool(torch.isnan(gd).all()) for gd in guards):
        ratio, where = math.inf, 'NaN guard around the pre-zeroed slice overwritten'
    return ratio, where, sums_err


def _large_n(key, N, sms):
    """A batch with more 128-row GEMM tiles than SMs (persistent CTAs loop, wgrad splits more than once),
    capped by MACS_BUDGET; None if the cap leaves nothing beyond the recorded N."""
    kind, H, W, Cs, Cin, Cout, R, S, s = key[:9]
    rows = ((H - 1) // s + 1) * ((W - 1) // s + 1)
    want = sms * 128 // rows + 1
    cap = int(MACS_BUDGET // (rows * R * S * Cin * Cout))
    n = min(want, cap)
    return n if n > N else None


def replay_modes(key, recorded=(0,)):
    """The pre-zeroed modes to replay a launch in: every mode it was recorded in, and mode 0 as well where the
    mode changes what the call does (wgrad, fused fprop)."""
    return sorted(set(recorded) | ({0} if accumulates(key) else set()))


def _run_launches(items, what):
    """items: [(key, N)] or [(key, N, prezeroed)].  Checks each, prints the worst ratio per launch and fails
    listing every offender."""
    bad, worst = [], 0.0
    t0 = time.time()
    for item in items:
        key, N, pz = item if len(item) == 3 else item + (0,)
        ratio, where, sums_err = check_launch(key, N, prezeroed=pz)
        worst = max(worst, ratio)
        print('    %-70s N %4d  pz %d  worst |err|/bound %.3f at %s%s' % (
            _fmt(key), N, pz, ratio, where, '' if sums_err is None else '  sums %.3f' % sums_err))
        if not ratio <= 1.0 or (sums_err is not None and not sums_err <= 1.0):
            bad.append((_fmt(key), N, 'prezeroed %d' % pz, ratio, where, sums_err))
    print('%s: %d launches, worst |err|/(rho|ref| + tau A) = %.3f (tau = 2^%.1f), %.1f s' % (
        what, len(items), worst, math.log2(TAU), time.time() - t0))
    assert not bad, bad


@pytest.mark.parametrize('size', ['recorded', 'large'])
@pytest.mark.parametrize('family', list(FAMILIES))
def test_launches_vs_fp64(inventory, family, size):
    """Each distinct conv launch of the family's bf16 step, per element against fp64, in every pre-zeroed mode
    the step ran it in (and with the mode off)."""
    launches, modes = inventory[family]
    items = sorted(launches.items(), key=lambda kv: _fmt(kv[0]))
    if size == 'large':
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        items = [(k, _large_n(k, n, sms)) for k, n in items]
        items = [(k, n) for k, n in items if n is not None]
        assert items, 'the time budget leaves no launch at a larger batch'
    _run_launches([(k, n, pz) for k, n in items for pz in replay_modes(k, modes[k])],
                  '%s at the %s batch' % (family, size))


# ---------------------------------------------------------------------------------------------------
# hand-picked edges beyond the inventory
# ---------------------------------------------------------------------------------------------------
def _k(kind, H, W, Cs, Cin, Cout, k, s, dout, fused=False):
    return (kind, H, W, Cs, Cin, Cout, k, k, s, BF16, dout, fused)


EDGES = [
    # strided bf16-dX dgrad on odd extents: parity classes of unequal size
    (_k('dgrad', 9, 9, 64, 64, 64, 3, 2, BF16), 3),
    (_k('dgrad', 9, 9, 512, 512, 512, 3, 2, BF16), 2),
    (_k('dgrad', 7, 7, 64, 64, 64, 3, 2, BF16), 3),
    (_k('dgrad', 7, 7, 512, 512, 512, 3, 2, BF16), 2),
    # strided 1x1: three of the four parity classes have no tap and must come out zero
    (_k('dgrad', 8, 8, 256, 256, 512, 1, 2, BF16), 2),
    (_k('dgrad', 9, 7, 64, 64, 128, 1, 2, BF16), 3),
    # bf16 rows stored element by element: a strided dgrad whose Cin ends in a 16-column slice, and outputs whose
    # rows are not 16-byte multiples (Cout % 8 != 0: no TMA store)
    (_k('dgrad', 9, 9, 176, 176, 128, 3, 2, BF16), 2),
    (_k('fprop', 10, 10, 64, 64, 132, 3, 1, BF16), 2),
    (_k('fprop', 9, 9, 64, 64, 132, 1, 2, BF16), 2),
    # ResNet-D stem, 3x3/2 on 4 stored channels: even width (pixel pairs) and odd width (8-byte gather)
    (_k('fprop', 32, 32, 4, 3, 64, 3, 2, BF16, True), 2),
    (_k('wgrad', 32, 32, 4, 3, 64, 3, 2, F32), 2),
    (_k('fprop', 29, 31, 4, 3, 64, 3, 2, BF16, True), 2),
    (_k('wgrad', 29, 31, 4, 3, 64, 3, 2, F32), 2),
    (_k('fprop', 30, 30, 4, 3, 32, 3, 2, BF16, True), 3),
    (_k('wgrad', 30, 30, 4, 3, 32, 3, 2, F32), 3),
    # the 128->128 halo 3x3 at H = 55, not a multiple of the two rows per tile
    (_k('fprop', 55, 56, 128, 128, 128, 3, 1, BF16, True), 2),
    (_k('dgrad', 55, 56, 128, 128, 128, 3, 1, BF16), 2),
    (_k('wgrad', 55, 56, 128, 128, 128, 3, 1, F32), 2),
    # the 224 stem with 128 outputs (its wgrad takes the generic small-channel path)
    (_k('fprop', 224, 224, 4, 3, 128, 7, 2, BF16, True), 1),
    (_k('wgrad', 224, 224, 4, 3, 128, 7, 2, F32), 1),
    # SK mixing dense layers on [N,1,1,f]: narrow outputs, column tiles that are mostly empty
    (_k('fprop', 1, 1, 128, 128, 32, 1, 1, BF16), 4),
    (_k('dgrad', 1, 1, 128, 128, 32, 1, 1, BF16), 4),
    (_k('wgrad', 1, 1, 128, 128, 32, 1, 1, F32), 4),
    (_k('fprop', 1, 1, 1024, 1024, 64, 1, 1, BF16), 50),
    (_k('dgrad', 1, 1, 1024, 1024, 64, 1, 1, BF16), 50),
    (_k('wgrad', 1, 1, 1024, 1024, 64, 1, 1, F32), 50),
    (_k('fprop', 1, 1, 32, 32, 256, 1, 1, F32), 4),
    (_k('dgrad', 1, 1, 32, 32, 256, 1, 1, BF16), 4),
    (_k('fprop', 1, 1, 64, 64, 2048, 1, 1, F32), 50),
    (_k('dgrad', 1, 1, 64, 64, 2048, 1, 1, BF16), 50),
]


@pytest.mark.parametrize('key,N', EDGES, ids=[_fmt(k).replace(' ', '') + '-N%d' % n for k, n in EDGES])
def test_edge_launch_vs_fp64(key, N):
    _run_launches([(key, N, pz) for pz in replay_modes(key, (1,))], 'edge')


def test_strided_1x1_dgrad_zero_classes():
    """dX of a stride-2 1x1 conv is zero at every pixel with an odd row or column -- written as zeros over a
    NaN-filled buffer, not left untouched."""
    from simclr_b200._lib import lib, stream_ptr
    N, H, W, Cin, Cout = 3, 9, 7, 64, 128
    torch.manual_seed(5)
    w = (torch.randn(1, 1, Cin, Cout) * 0.1).to(BF16)
    dy = torch.randn(N, 5, 4, Cout, device='cuda').to(BF16)
    _, wd = _pack(w, BF16, 1, Cin, Cin, Cout)
    lib.set_accumulate_prezeroed(0)
    dx = torch.full((N, H, W, Cin), float('nan'), dtype=BF16, device='cuda')
    lib.conv2d_dgrad_tc(dy, wd, dx, 1, 1, N, H, W, Cin, Cout, 1, 1, 2, stream_ptr())
    torch.cuda.synchronize()
    assert torch.equal(dx[:, 1::2], torch.zeros_like(dx[:, 1::2]))
    assert torch.equal(dx[:, :, 1::2], torch.zeros_like(dx[:, :, 1::2]))
    assert torch.isfinite(dx[:, ::2, ::2].float()).all()


# ---------------------------------------------------------------------------------------------------
# the bf16 / tc step gives the same bits on every run
# ---------------------------------------------------------------------------------------------------
def _snapshot(trainer, loss):
    snap = {'loss': loss.detach().clone(), 'momentum': trainer.optimizer._flat_v.clone()}
    for v in trainer.model.trainable_variables:
        snap['grad ' + v.name] = v.grad.clone()
        snap['value ' + v.name] = v.value.clone()
    for v in trainer.model.vs.moving:
        snap['moving ' + v.name] = v.value.clone()
    return snap


def test_step_same_bits(flags):
    """Two trainers built from the same state run two eager bf16 / tc steps (ResNet-50, 64x64, batch 16, fixed
    blur draws) on the same inputs: loss, every gradient, every updated weight, every moving statistic and the
    LARS momentum slots agree bit for bit after each step.  No atomics remain on this path: weight-gradient
    splits and BatchNorm statistics are added in a fixed order."""
    from test_gpu_step import _setup, _data
    B, S = 16, 64
    runs = []
    for _ in range(2):
        trainer, _, _, _ = _setup(flags, 'bf16', 'tc', True, B, S, depth=50)
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
