"""2-CTA TMA multicast in the implicit-GEMM and weight-gradient kernels changes no bit.  (It is off by default:
it measured slower on ResNet-50, DESIGN.md 4.1.  `simclr_set_tc_multicast` selects it for an A/B run.)

With multicast the two CTAs of a cluster each load half of the operand tile they share and send it to both; every
CTA still receives the same bytes, runs the same MMAs in the same order and keeps the same tiles.  Every recorded
`conv2d_{fprop,dgrad,wgrad}_tc` launch of the benchmarked bf16 steps (the inventory of test_gpu_layers.py) is replayed
with multicast off and on, at the recorded batch and at one with more tiles than SMs, into NaN-filled outputs; the
outputs and fused BatchNorm sums must be the same bits.  Hand-picked edges cover the unpaired tail of the last wave,
the non-cluster fallback, multi-split wgrad, strided dgrad and the split-bf16 (tc3) accumulate passes.  Last, two
trainers, one per setting, must give the same bits through two eager ResNet-50 steps and a CUDA-graph replay.
"""
import pytest
import torch

from test_gpu_layers import inventory, replay_modes, _fmt, _large_n, _k, _zeroed_slice, _snapshot  # noqa: F401
from test_gpu_tc import _pack

pytestmark = pytest.mark.gpu

BF16, F32 = torch.bfloat16, torch.float32
_INT = {BF16: torch.int16, F32: torch.int32, torch.float64: torch.int64}


def _bits(t):
    return t.contiguous().view(_INT[t.dtype])


def _same_bits(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(_bits(a), _bits(b))


@pytest.fixture
def multicast_arm():
    """Sets the multicast switch for one call and restores the process setting afterwards."""
    from simclr_b200._lib import lib
    prev = lib.set_tc_multicast(1)
    lib.set_tc_multicast(prev)

    def set_arm(on):
        lib.set_tc_multicast(on)
    yield set_arm
    lib.set_tc_multicast(prev)


def _run(key, N, mc, prezeroed, seed=0):
    """One launch at batch N on seeded inputs with multicast `mc`; returns its output tensors (guards included)."""
    from simclr_b200._lib import lib, stream_ptr, DTYPE_CODE
    kind, H, W, Cs, Cin, Cout, R, S, s, din, dout, fused = key
    Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
    g = torch.Generator(device='cuda').manual_seed(seed + sum(v for v in key if type(v) is int))
    x = torch.randn(N, H, W, Cin, generator=g, device='cuda').to(BF16)
    w = (torch.randn(R, S, Cin, Cout, generator=g, device='cuda') * (1.0 / (R * S * Cin) ** 0.5)).to(BF16)
    dy = torch.randn(N, Ho, Wo, Cout, generator=g, device='cuda').to(BF16)
    xs = x if Cs == Cin else torch.cat([x, torch.zeros(N, H, W, Cs - Cin, dtype=BF16, device='cuda')], -1).contiguous()
    st = stream_ptr()
    prev_mc = lib.set_tc_multicast(mc)
    prev_pz = lib.set_accumulate_prezeroed(prezeroed)
    try:
        if kind == 'fprop':
            wf, _ = _pack(w, BF16, R, Cin, Cs, Cout, want_wd=False)
            y = torch.full((N, Ho, Wo, Cout), float('nan'), dtype=dout, device='cuda')
            outs = [y]
            sums = None
            if fused and prezeroed:
                sums, guards = _zeroed_slice(2 * Cout, torch.float64)
                outs += [sums, *guards]
            elif fused:
                sums = torch.full((2 * Cout,), float('nan'), dtype=torch.float64, device='cuda')
                outs.append(sums)
            lib.conv2d_fprop_tc(xs, wf, y, DTYPE_CODE[din], DTYPE_CODE[dout], N, H, W, Cs, Cout, R, S, s, sums, st)
        elif kind == 'dgrad':
            _, wd = _pack(w, BF16, R, Cin, Cs, Cout)
            dx = torch.full((N, H, W, Cin), float('nan'), dtype=dout, device='cuda')
            outs = [dx]
            lib.conv2d_dgrad_tc(dy, wd, dx, DTYPE_CODE[din], DTYPE_CODE[dout], N, H, W, Cin, Cout, R, S, s, st)
        else:
            if prezeroed:
                dw, guards = _zeroed_slice(R * S * Cin * Cout, dout)
                outs = [dw, *guards]
            else:
                dw = torch.full((R * S * Cin * Cout,), float('nan'), dtype=dout, device='cuda')
                outs = [dw]
            lib.conv2d_wgrad_tc(xs, dy, dw, DTYPE_CODE[din], N, H, W, Cs, Cin, Cout, R, S, s, st)
        torch.cuda.synchronize()
    finally:
        lib.set_accumulate_prezeroed(prev_pz)
        lib.set_tc_multicast(prev_mc)
    return outs


def _check_arms(items, what):
    """items: [(key, N, prezeroed)].  Every output of each launch must be the same bits with multicast off and on."""
    bad = []
    for key, N, pz in items:
        off, on = _run(key, N, 0, pz), _run(key, N, 1, pz)
        differ = [i for i, (a, b) in enumerate(zip(off, on)) if not _same_bits(a, b)]
        nan = bool(torch.isnan(off[0].float()).any())            # the main output is written everywhere
        print('    %-70s N %4d  pz %d  %s' % (_fmt(key), N, pz, 'differ in outputs %s' % differ if differ else 'same bits'))
        if differ or nan:
            bad.append((_fmt(key), N, pz, differ, 'unwritten elements' if nan else ''))
    print('%s: %d launches' % (what, len(items)))
    assert not bad, bad


def test_cluster_pairs_fit():
    """The persistent grids take at most one CTA per SM; a multicast launch keeps its grid only if that many CTAs
    fit as clusters of 2 (otherwise it runs without clusters)."""
    from simclr_b200._lib import lib
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    pairs, quads = lib.tc_max_active_clusters(2), lib.tc_max_active_clusters(4)
    print('SMs %d, co-resident clusters of 2: %d, of 4: %d' % (sms, pairs, quads))
    assert 0 < pairs <= sms // 2 and 0 <= quads <= sms // 4


@pytest.mark.parametrize('size', ['recorded', 'large'])
@pytest.mark.parametrize('family', ['r50_1x_224', 'r50_2x_224', 'r50_2x_sk_224'])
def test_launches_multicast_same_bits(inventory, family, size):   # noqa: F811
    launches, modes = inventory[family]
    items = sorted(launches.items(), key=lambda kv: _fmt(kv[0]))
    if size == 'large':
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        items = [(k, _large_n(k, n, sms)) for k, n in items]
        items = [(k, n) for k, n in items if n is not None]
        assert items
    _check_arms([(k, n, pz) for k, n in items for pz in replay_modes(k, modes[k])], '%s at the %s batch' % (family, size))


EDGES = [
    # one column block (the pair shares B), 265 row tiles: the last wave's last CTA has no partner
    (_k('fprop', 8, 8, 256, 256, 128, 1, 1, BF16, True), 529),
    (_k('dgrad', 8, 8, 128, 128, 256, 1, 1, BF16), 529),
    # one column block of 64 (B halves of 32 rows), and an odd grid of 5 CTAs: no clusters
    (_k('fprop', 8, 8, 256, 256, 64, 1, 1, BF16, True), 10),
    (_k('fprop', 8, 8, 256, 256, 64, 1, 1, BF16, True), 529),
    # im2col A halves: 3x3 stride 1 and 2 at 256 channels, a partial last row tile
    (_k('fprop', 14, 14, 256, 256, 256, 3, 1, BF16, True), 37),
    (_k('fprop', 28, 28, 256, 256, 256, 3, 2, BF16, True), 37),
    # multi-split wgrad sharing X (two column blocks) and sharing dY (one column block of 128, even row blocks)
    (_k('wgrad', 14, 14, 256, 256, 256, 1, 1, F32), 64),
    (_k('wgrad', 14, 14, 512, 512, 128, 1, 1, F32), 64),
    (_k('wgrad', 28, 28, 256, 256, 256, 3, 2, F32), 16),
    (_k('wgrad', 7, 7, 512, 512, 512, 3, 1, F32), 40),
    # strided dgrad parity classes: 1x1 (three empty classes) and 3x3, odd extents
    (_k('dgrad', 28, 28, 512, 512, 1024, 1, 2, BF16), 16),
    (_k('dgrad', 27, 27, 256, 256, 256, 3, 2, BF16), 16),
    (_k('dgrad', 14, 14, 512, 512, 512, 3, 2, BF16), 16),
    # fp32 outputs
    (_k('fprop', 7, 7, 512, 512, 2048, 1, 1, F32), 64),
    (_k('dgrad', 7, 7, 2048, 2048, 512, 1, 1, F32), 64),
]


@pytest.mark.parametrize('key,N', EDGES, ids=[_fmt(k).replace(' ', '') + '-N%d' % n for k, n in EDGES])
def test_edge_multicast_same_bits(key, N):
    _check_arms([(key, N, pz) for pz in replay_modes(key, (1,))], 'edge')


@pytest.mark.parametrize('kind', ['fprop', 'dgrad', 'dgrad_strided', 'wgrad'])
def test_tc3_multicast_same_bits(kind):
    """The six split-bf16 passes of the fp32 step (the last five add into the output) give the same bits."""
    from simclr_b200._lib import lib, stream_ptr
    N, H, Cin, Cout, k = 32, 14, 256, 256, 3
    s = 2 if kind == 'dgrad_strided' else 1
    Ho = (H - 1) // s + 1
    g = torch.Generator(device='cuda').manual_seed(11)
    xs = [torch.randn(N, H, H, Cin, generator=g, device='cuda').to(BF16) for _ in range(3)]
    ds = [torch.randn(N, Ho, Ho, Cout, generator=g, device='cuda').to(BF16) for _ in range(3)]
    ws = [(torch.randn(k, k, Cin, Cout, generator=g, device='cuda') * 0.02).to(BF16) for _ in range(3)]
    packed = [_pack(w, BF16, k, Cin, Cin, Cout) for w in ws]
    st = stream_ptr()
    outs = []
    for mc in (0, 1):
        prev = lib.set_tc_multicast(mc)
        try:
            if kind == 'fprop':
                y = torch.full((N, Ho, Ho, Cout), float('nan'), dtype=F32, device='cuda')
                lib.conv2d_fprop_tc3(*xs, *[p[0] for p in packed], y, N, H, H, Cin, Cout, k, k, s, st)
            elif kind.startswith('dgrad'):
                y = torch.full((N, H, H, Cin), float('nan'), dtype=F32, device='cuda')
                lib.conv2d_dgrad_tc3(*ds, *[p[1] for p in packed], y, N, H, H, Cin, Cout, k, k, s, st)
            else:
                y = torch.full((k, k, Cin, Cout), float('nan'), dtype=F32, device='cuda')
                lib.conv2d_wgrad_tc3(*xs, *ds, y, N, H, H, Cin, Cin, Cout, k, k, s, st)
            torch.cuda.synchronize()
        finally:
            lib.set_tc_multicast(prev)
        outs.append(y)
    assert not torch.isnan(outs[0]).any()
    assert _same_bits(outs[0], outs[1])


def test_step_multicast_same_bits(flags, multicast_arm):
    """Two trainers built from the same state, one with multicast off and one with it on, run two eager bf16 / tc
    ResNet-50 steps and one CUDA-graph replay on the same inputs: loss, every gradient, every weight, every moving
    statistic and the LARS momentum slots agree bit for bit after each."""
    from test_gpu_step import _setup, _data
    B, S = 32, 96
    runs = []
    for mc in (0, 1):
        multicast_arm(mc)
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
        trainer.capture(f, lab, warmup=0)
        loss = trainer.replay()
        torch.cuda.synchronize()
        snaps.append(_snapshot(trainer, loss))
        runs.append(snaps)
        del trainer
        torch.cuda.empty_cache()
    for step, (a, b) in enumerate(zip(*runs)):
        assert a.keys() == b.keys()
        differ = [k for k in a if not _same_bits(a[k], b[k])]
        assert not differ, 'step %d: %d of %d tensors differ, e.g. %s' % (step + 1, len(differ), len(a), differ[:5])
    assert any(not torch.equal(runs[0][1][k], runs[0][2][k]) for k in runs[0][1] if k.startswith('value ')), \
        'the graph replay must change the weights'
