"""Parity of the wgmma / TMA implicit-GEMM engine (fprop, dgrad, wgrad, dense)
against the oracle's convolution on the same (bf16-rounded) inputs.

bf16 x bf16 products are exact in fp32, so with fp32 outputs the only
difference from the fp64 reference is fp32 accumulation order: tolerance 2e-4.
bf16 outputs add one rounding (2^-9 relative): tolerance 8e-3.  tf32 operands
(fp32 storage, kind::tf32) carry 10 mantissa bits: tolerance 3e-3.
"""
import pytest
import torch

from util import rel_err
from test_gpu_kernels import conv_reference

pytestmark = pytest.mark.gpu

# N, H, W, Cin, Cs, Cout, k, stride
CASES = [
    (2, 16, 16, 64, 64, 256, 1, 1),      # plain GEMM: activations through TMA, two 128-column tiles
    (3, 10, 10, 256, 256, 64, 1, 1),     # M=300 (ragged last tile), BN=64
    (2, 12, 12, 64, 64, 64, 3, 1),       # gathered 3x3
    (2, 8, 8, 128, 128, 128, 3, 1),      # BN=128, two K blocks per tap
    (2, 12, 12, 128, 128, 128, 3, 2),    # strided 3x3 (FixedPadding + VALID)
    (2, 8, 8, 256, 256, 512, 1, 2),      # strided 1x1 projection shortcut
    (2, 32, 32, 3, 4, 64, 7, 2),         # stem: 3 channels stored as 4
    (100, 1, 1, 2048, 2048, 128, 1, 1),  # projection-head dense
    (64, 1, 1, 512, 512, 1000, 1, 1),    # supervised head: n_out not a tile multiple
    (1, 5, 7, 64, 64, 64, 3, 1),         # tiny M (35 rows)
    (4, 28, 28, 128, 128, 512, 1, 1),    # several tiles per CTA? (M=3136 -> 25 tiles x 2)
    (2, 14, 14, 1024, 1024, 256, 1, 1),  # long K (16 K blocks) through the smem ring
    (2, 14, 14, 256, 256, 256, 3, 1),    # TMA im2col: four channel blocks per tap, tiles crossing images
    (3, 9, 9, 64, 64, 64, 3, 2),         # odd extent, strided: im2col fprop/wgrad, dgrad classes of unequal size
    (2, 12, 12, 64, 64, 128, 3, 2),      # 64-channel strided 3x3 (two taps per 128 k-rows in wgrad)
    (1, 9, 11, 64, 64, 64, 5, 1),        # 5x5, rectangular image
    (2, 31, 31, 3, 4, 64, 7, 2),         # stem on an odd width: 8-byte gather (no pixel pairs)
    (2, 16, 16, 3, 4, 64, 3, 1),         # CIFAR stem: 3x3 stride 1 on 4 stored channels
    (3, 20, 28, 3, 4, 64, 7, 2),         # stem, rectangular, pixel-pair path, ragged last tile
    # halo-reuse 3x3 kernel (tc_halo.cu): bf16 in/out, 64->64 (resident filter) and 128->128 (streamed filter)
    (2, 56, 56, 64, 64, 64, 3, 1),       # the ResNet-50 stage-1 3x3: Wp 58, 2 rows per tile
    (3, 28, 28, 128, 128, 128, 3, 1),    # stage-2 3x3: Wp 30, 4 rows per tile, two channel blocks
    (2, 27, 28, 128, 128, 128, 3, 1),    # H not a multiple of the rows per tile: last tile clipped by the TMA store
    (5, 18, 30, 64, 64, 64, 3, 1),       # Wp 32, more tiles than one wave of a small grid
    (1, 10, 62, 64, 64, 64, 3, 1),       # widest supported row (Wp 64)
    # stem kernel (tc_stem.cu): slab of pixel pairs, overlapping no-swizzle descriptors, one output row per tile
    (2, 224, 224, 3, 4, 64, 7, 2),       # the benchmark shape: Q = 112 of 128 GEMM rows real
    (40, 16, 16, 3, 4, 64, 7, 2),        # 320 tiles: several per CTA, slab ring and both accumulators wrap
    (2, 64, 64, 3, 4, 128, 7, 2),        # width multiplier 2: two 64-column boxes per tile
    (1, 48, 40, 3, 4, 256, 7, 2),        # width multiplier 4, rectangular: beyond the stem kernel's 128 columns, generic path
]


def _mk(case, dtype, seed_off=0):
    N, H, W, Cin, Cs, Cout, k, s = case
    torch.manual_seed(sum(case) + seed_off)
    x = torch.randn(N, H, W, Cin).to(dtype)
    w = (torch.randn(k, k, Cin, Cout) * (1.0 / (k * k * Cin) ** 0.5)).to(dtype)   # weights rounded like the packed copy
    xs = torch.zeros(N, H, W, Cs, dtype=dtype); xs[..., :Cin] = x
    return x, w, xs


def _pack(w, dtype, k, Cin, Cs, Cout, want_wd=True):
    from simclr_b200._lib import lib, stream_ptr, DTYPE_CODE
    es = 2 if dtype == torch.bfloat16 else 4
    kbe = 128 // es
    K = k * (k + 1 if (Cs == 4 and es == 2) else k) * Cs     # bf16 stem: S+1 slots per filter row
    Kp = (K + kbe - 1) // kbe * kbe
    wf = torch.empty(Cout, Kp, dtype=dtype, device='cuda')
    kd = k * k * Cout
    wd = torch.empty(Cin, (kd + kbe - 1) // kbe * kbe, dtype=dtype, device='cuda') if (want_wd and Cs == Cin) else None
    lib.pack_conv_weight(w.float().cuda().contiguous(), wf, wd, DTYPE_CODE[dtype], k, k, Cin, Cs, Cout, Kp, stream_ptr())
    return wf, wd


@pytest.mark.parametrize('out_dtype', [torch.float32, torch.bfloat16])
@pytest.mark.parametrize('case', CASES)
def test_tc_fprop_bf16(case, out_dtype):
    from simclr_b200._lib import lib, stream_ptr, DTYPE_CODE
    N, H, W, Cin, Cs, Cout, k, s = case
    x, w, xs = _mk(case, torch.bfloat16)
    yo = conv_reference(x.double(), w.double(), k, s)
    wf, _ = _pack(w, torch.bfloat16, k, Cin, Cs, Cout, want_wd=False)
    y = torch.full(yo.shape, float('nan'), dtype=out_dtype, device='cuda')
    sums = torch.full((2 * Cout,), float('nan'), dtype=torch.float64, device='cuda') if (Cout * y.element_size()) % 16 == 0 else None
    lib.conv2d_fprop_tc(xs.cuda(), wf, y, 1, DTYPE_CODE[out_dtype], N, H, W, Cs, Cout, k, k, s, sums, stream_ptr())
    torch.cuda.synchronize()
    # BatchNorm statistics fused into the epilogue: sums of the *stored* outputs
    yf = y.double().reshape(-1, Cout)
    if sums is not None:
        assert rel_err(sums[:Cout], yf.sum(0)) < 1e-5
        assert rel_err(sums[Cout:], (yf * yf).sum(0)) < 1e-5
    assert rel_err(y, yo) < (2e-4 if out_dtype == torch.float32 else 8e-3)


@pytest.mark.parametrize('case', [c for c in CASES if c[3] == c[4]])
def test_tc_dgrad_bf16(case):
    from simclr_b200._lib import lib, stream_ptr
    N, H, W, Cin, Cs, Cout, k, s = case
    x, w, xs = _mk(case, torch.bfloat16)
    xo = x.double().requires_grad_(True)
    yo = conv_reference(xo, w.double(), k, s)
    dy = torch.randn(yo.shape).to(torch.bfloat16)
    yo.backward(dy.double())
    _, wd = _pack(w, torch.bfloat16, k, Cin, Cs, Cout)
    dx = torch.full((N, H, W, Cin), float('nan'), dtype=torch.float32, device='cuda')
    lib.conv2d_dgrad_tc(dy.cuda(), wd, dx, 1, 0, N, H, W, Cin, Cout, k, k, s, stream_ptr())
    torch.cuda.synchronize()
    assert rel_err(dx, xo.grad) < 2e-4


@pytest.mark.parametrize('case', CASES)
def test_tc_wgrad_bf16(case):
    from simclr_b200._lib import lib, stream_ptr
    N, H, W, Cin, Cs, Cout, k, s = case
    x, w, xs = _mk(case, torch.bfloat16)
    wo = w.double().requires_grad_(True)
    yo = conv_reference(x.double(), wo, k, s)
    dy = torch.randn(yo.shape).to(torch.bfloat16)
    yo.backward(dy.double())
    dw = torch.full((k, k, Cin, Cout), float('nan'), dtype=torch.float32, device='cuda')
    lib.conv2d_wgrad_tc(xs.cuda(), dy.cuda(), dw, 1, N, H, W, Cs, Cin, Cout, k, k, s, stream_ptr())
    torch.cuda.synchronize()
    assert rel_err(dw, wo.grad) < 2e-4
    # split / per-CTA partials are added in a fixed order: the same inputs give the same bits
    dw2 = torch.full_like(dw, float('nan'))
    lib.conv2d_wgrad_tc(xs.cuda(), dy.cuda(), dw2, 1, N, H, W, Cs, Cin, Cout, k, k, s, stream_ptr())
    torch.cuda.synchronize()
    assert torch.equal(dw, dw2)


@pytest.mark.parametrize('case', [CASES[0], CASES[2], CASES[4], CASES[7], CASES[9]])
def test_tc_tf32(case):
    """fp32 storage, kind::tf32 operands."""
    from simclr_b200._lib import lib, stream_ptr
    N, H, W, Cin, Cs, Cout, k, s = case
    x, w, xs = _mk(case, torch.float32, 7)
    xo = x.double().requires_grad_(True); wo = w.double().requires_grad_(True)
    yo = conv_reference(xo, wo, k, s)
    dy = torch.randn(yo.shape)
    yo.backward(dy.double())
    wf, wd = _pack(w, torch.float32, k, Cin, Cs, Cout)
    st = stream_ptr()
    y = torch.full(yo.shape, float('nan'), device='cuda')
    lib.conv2d_fprop_tc(xs.cuda(), wf, y, 0, 0, N, H, W, Cs, Cout, k, k, s, None, st)
    dx = torch.full((N, H, W, Cin), float('nan'), device='cuda')
    lib.conv2d_dgrad_tc(dy.cuda(), wd, dx, 0, 0, N, H, W, Cin, Cout, k, k, s, st)
    torch.cuda.synchronize()
    assert rel_err(y, yo) < 3e-3
    assert rel_err(dx, xo.grad) < 3e-3
    # wgrad on tf32 operands is not implemented on the wgmma engine: must fail loudly, not silently
    from simclr_b200._lib import SimclrError
    dw = torch.empty((k, k, Cin, Cout), device='cuda')
    with pytest.raises(SimclrError):
        lib.conv2d_wgrad_tc(xs.cuda(), dy.cuda(), dw, 0, N, H, W, Cs, Cin, Cout, k, k, s, st)


@pytest.mark.parametrize('shape', [(64, 28, 28, 128, 128, 3, 1), (16, 56, 56, 64, 64, 3, 1), (16, 56, 56, 128, 128, 3, 2),
                                   (16, 28, 28, 256, 512, 1, 2), (8, 56, 56, 64, 256, 1, 1)])
def test_tc_matches_simt_large(shape):
    """Size-independent check at BASELINE-sized layers (many tiles per CTA, tiles crossing image
    rows and images): wgmma vs the CUDA-core engine on the same bf16 inputs."""
    from simclr_b200._lib import lib, stream_ptr
    N, H, W, C, Co, k, s = shape
    Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
    torch.manual_seed(11)
    x = torch.randn(N, H, W, C, device='cuda').to(torch.bfloat16)
    w = (torch.randn(k, k, C, Co, device='cuda') * 0.03).to(torch.bfloat16)
    dy = torch.randn(N, Ho, Wo, Co, device='cuda').to(torch.bfloat16)
    wf, wd = _pack(w.cpu(), torch.bfloat16, k, C, C, Co)
    st = stream_ptr()
    wf32 = w.float().contiguous()
    y_tc = torch.empty(N, Ho, Wo, Co, device='cuda'); y_ref = torch.empty_like(y_tc)
    lib.conv2d_fprop_tc(x, wf, y_tc, 1, 0, N, H, W, C, Co, k, k, s, None, st)
    lib.conv2d_fprop_simt(x, wf32, y_ref, 1, 0, N, H, W, C, C, Co, k, k, s, st)
    dx_tc = torch.empty(N, H, W, C, device='cuda'); dx_ref = torch.empty_like(dx_tc)
    lib.conv2d_dgrad_tc(dy, wd, dx_tc, 1, 0, N, H, W, C, Co, k, k, s, st)
    lib.conv2d_dgrad_simt(dy, wf32, dx_ref, 1, 0, N, H, W, C, Co, k, k, s, st)
    dw_tc = torch.empty(k, k, C, Co, device='cuda'); dw_ref = torch.empty_like(dw_tc)
    lib.conv2d_wgrad_tc(x, dy, dw_tc, 1, N, H, W, C, C, Co, k, k, s, st)
    lib.conv2d_wgrad_simt(x, dy, dw_ref, 1, N, H, W, C, C, Co, k, k, s, st)
    torch.cuda.synchronize()
    assert rel_err(y_tc, y_ref) < 2e-4
    assert rel_err(dx_tc, dx_ref) < 2e-4
    assert rel_err(dw_tc, dw_ref) < 5e-4


def _split(t):
    from simclr_b200._lib import lib, stream_ptr
    t = t.float().cuda().contiguous()
    parts = [torch.empty(t.shape, dtype=torch.bfloat16, device='cuda') for _ in range(3)]
    lib.split_bf16x3(t, parts[0], parts[1], parts[2], t.numel(), stream_ptr())
    return parts


@pytest.mark.parametrize('case', [CASES[i] for i in (0, 1, 2, 4, 5, 6, 8, 12, 13, 16)])
def test_tc3_split_bf16_fp32_accuracy(case):
    """tc3 (fp32 operands split into three bf16 terms, six wgmma GEMMs summed in fp32): fprop, dgrad and
    wgrad against the fp64 oracle conv on UNROUNDED fp32 inputs at 5e-6 -- three orders below a single
    bf16 pass (4e-3), at the level of an fp32 CUDA-core conv."""
    from simclr_b200._lib import lib, stream_ptr
    N, H, W, Cin, Cs, Cout, k, s = case
    x, w, xs = _mk(case, torch.float32, 11)
    xo = x.double().requires_grad_(True); wo = w.double().requires_grad_(True)
    yo = conv_reference(xo, wo, k, s)
    dy = torch.randn(yo.shape)
    yo.backward(dy.double())
    xp = _split(xs)
    assert torch.equal((xp[0].double() + xp[1].double() + xp[2].double()).float().cpu(), xs)     # 24 mantissa bits recovered
    K = k * (k + 1 if Cs == 4 else k) * Cs
    Kp = (K + 63) // 64 * 64
    kd = (k * k * Cout + 63) // 64 * 64
    has_wd = Cs == Cin
    wf = [torch.empty(Cout, Kp, dtype=torch.bfloat16, device='cuda') for _ in range(3)]
    wd = [torch.empty(Cin, kd, dtype=torch.bfloat16, device='cuda') if has_wd else None for _ in range(3)]
    wc = w.float().cuda().contiguous()
    for part in range(3):
        lib.pack_conv_weight_part(wc, wf[part], wd[part], part, k, k, Cin, Cs, Cout, Kp, stream_ptr())
    y = torch.full(yo.shape, float('nan'), dtype=torch.float32, device='cuda')
    lib.conv2d_fprop_tc3(xp[0], xp[1], xp[2], wf[0], wf[1], wf[2], y, N, H, W, Cs, Cout, k, k, s, stream_ptr())
    torch.cuda.synchronize()
    assert rel_err(y, yo) < 5e-6
    dp = _split(dy)
    if Cout % 8 == 0:
        dw = torch.full((k, k, Cin, Cout), float('nan'), dtype=torch.float32, device='cuda')
        lib.conv2d_wgrad_tc3(xp[0], xp[1], xp[2], dp[0], dp[1], dp[2], dw, N, H, W, Cs, Cin, Cout, k, k, s, stream_ptr())
        torch.cuda.synchronize()
        assert rel_err(dw, wo.grad) < 5e-6
    if has_wd:
        dx = torch.full((N, H, W, Cin), float('nan'), dtype=torch.float32, device='cuda')
        lib.conv2d_dgrad_tc3(dp[0], dp[1], dp[2], wd[0], wd[1], wd[2], dx, N, H, W, Cin, Cout, k, k, s, stream_ptr())
        torch.cuda.synchronize()
        assert rel_err(dx, xo.grad) < 5e-6


@pytest.mark.parametrize('case', [c for c in CASES if c[6] == 3 and c[7] == 1 and c[3] == c[5] and c[3] in (64, 128)])
def test_tc_dgrad_bf16_out(case):
    """Stride-1 3x3 dgrad with bf16 output -- the dtype of the training step, and the only one the
    halo-reuse kernel serves (flipped taps over a dY slab)."""
    from simclr_b200._lib import lib, stream_ptr
    N, H, W, Cin, Cs, Cout, k, s = case
    x, w, xs = _mk(case, torch.bfloat16)
    xo = x.double().requires_grad_(True)
    yo = conv_reference(xo, w.double(), k, s)
    dy = torch.randn(yo.shape).to(torch.bfloat16)
    yo.backward(dy.double())
    _, wd = _pack(w, torch.bfloat16, k, Cin, Cs, Cout)
    dx = torch.full((N, H, W, Cin), float('nan'), dtype=torch.bfloat16, device='cuda')
    lib.conv2d_dgrad_tc(dy.cuda(), wd, dx, 1, 1, N, H, W, Cin, Cout, k, k, s, stream_ptr())
    torch.cuda.synchronize()
    assert rel_err(dx, xo.grad) < 8e-3


def test_pack_weights_multi_matches_single():
    """One-launch packing of many layers (balanced 32x32 transposition tiles) == per-layer `simclr_pack_conv_weight`,
    including the stem layout (Cs = 4), Kp padding, Cout not a multiple of 32 and layers without a dgrad operand."""
    from simclr_b200._lib import lib, stream_ptr
    torch.manual_seed(0)
    st = stream_ptr()
    layers = [(7, 3, 4, 64, False), (1, 64, 64, 256, True), (3, 64, 64, 64, True), (3, 128, 128, 128, True),
              (1, 2048, 2048, 16, True), (1, 512, 512, 1000, False), (3, 8, 8, 24, True), (1, 256, 256, 40, True)]
    rows, keep = [], []
    for k, Cin, Cs, Cout, has_wd in layers:
        w = torch.randn(k, k, Cin, Cout, device='cuda')
        Kp = ((k * (k + 1) if Cs == 4 else k * k) * Cs + 63) // 64 * 64
        Kdp = (k * k * Cout + 63) // 64 * 64
        wf = torch.full((Cout, Kp), 7.0, dtype=torch.bfloat16, device='cuda'); wf_ref = torch.empty_like(wf)
        wd = torch.full((Cin, Kdp), 7.0, dtype=torch.bfloat16, device='cuda') if has_wd else None
        wd_ref = torch.empty_like(wd) if has_wd else None
        lib.pack_conv_weight(w, wf_ref, wd_ref, 1, k, k, Cin, Cs, Cout, Kp, st)
        rows.append([w.data_ptr(), wf.data_ptr(), wd.data_ptr() if has_wd else 0, k, k, Cin, Cs, Cout, Kp, Kdp if has_wd else 0])
        keep.append((w, wf, wf_ref, wd, wd_ref))
    table = torch.tensor(rows, dtype=torch.int64).cuda()
    lib.pack_conv_weights_multi(table, len(rows), st)
    torch.cuda.synchronize()
    for i, (w, wf, wf_ref, wd, wd_ref) in enumerate(keep):
        assert torch.equal(wf, wf_ref), 'wf of layer %d' % i
        if wd is not None:
            assert torch.equal(wd, wd_ref), 'wd of layer %d' % i
