"""The augmentation kernel (`simclr_augment`, csrc/augment.cu) against the fp64 oracle (oracle/data_util.py), per pixel,
at the shapes and draws of the input pipeline.

A  every bicubic tap position of crop sides 1..4096 at output sides 32..256, on each axis;
B  replays of `draw_train_augmentation` at colour strengths 0.5, 1 and 1.5 over ImageNet-like, huge and tiny images,
   at 224 (two views into [B,224,224,6]), 32, 64, 48x80 and 80x48, and the eval centre crop;
C  the colour ops at edge factors in all 24 orders, on near-gray, tied and hue-wrapping pixels;
D  output layouts, batch sizes, a source image past 2^31 bytes, repeatability and argument checks;
E  `build_input_fn` over a TFRecord directory, host and device JPEG decode, against the oracle on recorded draws.

Each output element must satisfy |got - ref| <= tau, with tau derived below.  The CPU tests (unmarked) check the
tap-position patterns and validate the colour-op bounds in float32 torch against float64."""
import io
import json
import math
import os
import random

import numpy as np
import pytest
import torch

U = 2.0 ** -24            # fp32 unit roundoff
S_W = 1.25                # max over taps of sum_t |w_t| for one axis (Keys a = -0.5 at frac 1/2; checked below)
SIDES = (32, 64, 96, 128, 160, 192, 224, 256)
MAX_CROP = 4096
AT = 512                  # threads per image in augment_kernel

gpu = pytest.mark.gpu


# --------------------------------------------------------------------------
# Bounds
# --------------------------------------------------------------------------
# Resize.  The kernel forms v = fl(px * fl(1/255)) (2 roundings), casts each fp64 weight to fp32 (1 per axis) and
# accumulates 4 x taps then 4 y taps with fmaf (<= 4 roundings per axis, each bounded by u times the sum of
# |w| |v| over the taps).  To first order, |got - ref| <= (2 + 1 + 4 + 1 + 4) u sum_ab |wy_a| |wx_b| <= 12 S_W^2 u;
# one more u S_W^2 covers the second-order terms.
TAU_RESIZE = 13 * S_W ** 2 * U
# Section A: in == out on y gives the taps (0, 1, 0, 0), so the y pass is exact and only the x pass rounds:
# (2 + 1 + 4) u S_W, plus one u S_W for second-order terms.  8 S_W u = 10 u ~ 2^-20.7.
TAU_A = 8 * S_W * U
# Section C: at in == out on both axes only v = fl(px * fl(1/255)) rounds: 2u.
TAU_IDENTITY = 2 * U

# Colour ops.  The error after op k+1 is err_{k+1} <= L_k err_k + eps_k, with L_k the op's Lipschitz constant in
# the max norm over the three channels (and, for contrast, over the pixels through the mean); the clip after each op
# is 1-Lipschitz and exact.  Inputs lie in [0, 1].
#  brightness  y = f x: L = |f|, eps = |f| u (one product).
#  contrast    y = (x - m) f + m = f x + (1 - f) m: L = |f| + |1 - f|.  The kernel's mean sums k = ceil(npix / 512)
#              values per thread, 5 warp-shuffle levels, 16 warp partials and a division: (k + 20) u relative to a
#              mean <= 1, entering with weight |1 - f|.  The update rounds x - m (<= u), the product (<= |f| u) and the
#              sum (<= (1 + |f|) u): eps = |1 - f| (k + 20) u + (2 + 2|f|) u.
#  hue         c = v - rng (1 - d_c(6 h)) with rng = max - min, h the hue and d_c piecewise linear of slope 1 in 6h.
#              In the sector where r is the max, h = (g - b) / (6 rng) + const and |g - b| <= rng, so a perturbation
#              of size D moves h by <= 4 D / (6 rng) and rng d_c by <= 4 D; rng moves by <= 2 D and v by <= D:
#              L = 7.  This holds for near-gray pixels too: h is ill-conditioned there, but it enters multiplied by
#              rng.  Rounding: h has relative error <= 4u (rng, 6 rng, the reciprocal, g - b and the product) and
#              absolute error <= 5u after the sector offset, the wrap and the fp32 hue delta; 6h and the three
#              clamped distances add 6u + 6u; the products with s rng / v <= 1 and the final sum and scale add 4u;
#              s = rng / v adds 2u.  About 48u; eps = 64 u.
#  saturation  s' = clip(s f, 0, 1).  If f <= 0, c = v: L = 1.  If f s <= 1, c = (1 - f) v + f c_in:
#              L = |1 - f| + |f|.  Otherwise (f > 1, rng > v / f) c = v d_c(h): L <= 1 + 4 v / rng < 1 + 4 f.
#              eps = 64 u as for hue (plus the s f product and the fp32 factor, inside the margin).
#  grayscale   y = 0.2989 r + 0.587 g + 0.114 b with fp32 weights: L = 0.9999 <= 1; the weights' representation
#              (<= u each) and three roundings: eps = 5 u.
EPS_HSV = 64 * U


def l_saturation(f):
    if f <= 0:
        return 1.0
    if f <= 1:
        return abs(1 - f) + abs(f)
    return max(abs(1 - f) + abs(f), 1 + 4 * f)


def op_bound(op, f, err, npix):
    """(error after the op, given `err` before it) for op 0 brightness, 1 contrast, 2 saturation, 3 hue."""
    if op == 0:
        return abs(f) * err + abs(f) * U
    if op == 1:
        k = -(-npix // AT)
        return (abs(f) + abs(1 - f)) * err + abs(1 - f) * (k + 20) * U + (2 + 2 * abs(f)) * U
    if op == 2:
        return l_saturation(f) * err + EPS_HSV
    return 7 * err + EPS_HSV


def colour_bound(err, colour, npix):
    """Bound after `random_color_jitter` (tf2/data_util.py:382-390) and the final clip, from an input bound `err`."""
    if colour['apply_jitter']:
        fs = (colour['brightness'], colour['contrast'], colour['saturation'], colour['hue'])
        for op in colour['perm']:
            err = op_bound(op, fs[op], err, npix)
    if colour['apply_gray']:
        err = err + 5 * U
    return err


# --------------------------------------------------------------------------
# Helpers
# --------------------------------------------------------------------------
NO_COLOUR = dict(apply_jitter=False, perm=(0, 1, 2, 3), brightness=1., contrast=1., saturation=1., hue=0.,
                 apply_gray=False)


def _eng():
    from simclr_b200 import engine, flags_def
    if not flags_def.FLAGS.is_parsed():
        flags_def.FLAGS(['test'])
    return engine.set_engine(engine.Engine(precision='fp32', conv_engine='simt'))


def _pack(images):
    """uint8 [H,W,3] tensors -> (packed uint8 on the GPU, offsets int64, sizes int32 [n][2])."""
    offs, hw, total = [], [], 0
    for im in images:
        offs.append(total)
        hw.append([im.shape[0], im.shape[1]])
        total += im.numel()
    src = torch.cat([im.reshape(-1).cuda() for im in images])
    return src, np.asarray(offs, dtype=np.int64), np.asarray(hw, dtype=np.int32)


def _launch(src, offs, hw, draws, H, W, stride=3, ch_off=0, fill=float('nan')):
    """One `simclr_augment` launch into an output of `stride` channels filled with `fill`."""
    from simclr_b200 import data_util as D
    out = torch.full((len(draws), H, W, stride), fill, dtype=torch.float32, device='cuda')
    D.preprocess_for_train_packed(src, offs, hw, draws, H, W, out=out, channel_offset=ch_off)
    return out


def _oracle(im_u8, draw, H, W):
    """oracle.preprocess_for_train in float64 on the GPU."""
    from oracle import data_util as OD
    x = im_u8.cuda().double() / 255.0
    return OD.preprocess_for_train(x, H, W, draw)


def _check(got, ref, tau, what):
    """Per element |got - ref| <= tau (tau broadcasts); returns the worst ratio."""
    assert not torch.isnan(got).any(), what + ': NaN in the output (an element was not written)'
    err = (got.double() - ref.double()).abs()
    rel = torch.where(err == 0, 0.0, err / tau)           # tau = 0 (brightness 0 last): the output must be exact
    ratio = rel.max().item()
    if ratio > 1:
        i = int(torch.argmax(rel.flatten()))
        raise AssertionError('%s: |got - ref| / tau = %.3g at flat index %d (got %r, ref %r)'
                             % (what, ratio, i, got.flatten()[i].item(), ref.flatten()[i].item()))
    return ratio


WORST = {}


def _note(section, ratio):
    WORST[section] = max(WORST.get(section, 0.0), ratio)
    print('worst ratio to the bound, section %s: %.4f' % (section, WORST[section]))


# --------------------------------------------------------------------------
# A. Tap positions, exhaustive
# --------------------------------------------------------------------------
def _pattern():
    """[4, MAX_CROP, 3] uint8: per row, channel 0 random, channel 1 an impulse every 4 px, channel 2 a squared ramp."""
    rs = np.random.RandomState(1)
    x = np.arange(MAX_CROP)
    p = np.empty((4, MAX_CROP, 3), dtype=np.uint8)
    for r in range(4):
        p[r, :, 0] = rs.randint(0, 256, MAX_CROP)
        p[r, :, 1] = np.where((x + r) % 4 == 0, 255, 0)
        p[r, :, 2] = ((x + 5 * r) ** 2) % 256
    return p


def _fp64_positions(in_size, out_size):
    """The table positions fl + off / 1024 the pre-fp32 kernel took: scale, position and offset in fp64."""
    n = np.asarray(in_size, dtype=np.float64)[..., None]
    src = (np.arange(out_size) + 0.5) * (n / out_size) - 0.5
    fl = np.floor(src)
    return fl + np.rint((src - fl) * 1024) / 1024


def _fp32_positions(in_size, out_size):
    f32 = np.float32
    n = np.asarray(in_size, dtype=np.int64)[..., None]
    src = (np.arange(out_size, dtype=f32) + f32(0.5)) * (n.astype(f32) / f32(out_size)) - f32(0.5)
    fl = np.floor(src)
    return fl.astype(np.float64) + np.rint((src - fl) * f32(1024)).astype(np.float64) / 1024


def _taps_at(pos, in_size):
    """Oracle weights (fp64 table entry, edge taps dropped, renormalised) at table positions `pos` (fl + off/1024)."""
    from oracle import data_util as OD
    fl = np.floor(pos)
    off = np.rint((pos - fl) * 1024).astype(np.int64)
    w = OD._keys_cubic_table(dtype=torch.float64).numpy()[off]
    idx = fl.astype(np.int64)[..., None] - 1 + np.arange(4)
    n = np.asarray(in_size)[..., None]
    w = np.where((idx >= 0) & (idx < n), w, 0.0)
    return np.clip(idx, 0, n - 1), w / w.sum(-1, keepdims=True)


def test_tap_weight_sum_and_oracle_positions():
    """S_W bounds sum |w| over every tap set of section A, and the oracle takes TF's fp32 positions."""
    from oracle import data_util as OD
    crops = np.arange(1, MAX_CROP + 1)
    for side in SIDES:
        idx, w = OD._bicubic_axis_taps(crops, side)
        assert np.abs(w).sum(-1).max() <= S_W
        assert np.allclose(w.sum(-1), 1.0, atol=1e-12)
        assert ((0 <= idx) & (idx < crops[:, None, None])).all()
        # the oracle samples at the fp32 position: the same functional on a random row (the entries (fl, 1024) and
        # (fl + 1, 0) are one position with shifted taps)
        i2, w2 = _taps_at(_fp32_positions(crops, side), crops[:, None])
        z = np.random.RandomState(side).rand(MAX_CROP)
        assert np.abs((w * z[idx]).sum(-1) - (w2 * z[i2]).sum(-1)).max() < 1e-12
    # Counts of (crop side, output index) pairs whose fp64 and fp32 positions differ, crop sides 1..4096.
    diff = {s: int((_fp64_positions(crops, s) != _fp32_positions(crops, s)).sum()) for s in SIDES}
    assert diff == {32: 0, 64: 0, 96: 13417, 128: 0, 160: 0, 192: 26827, 224: 52831, 256: 0}


def test_tap_pattern_is_sensitive():
    """Wherever the fp64 and fp32 positions differ, the oracle outputs for the two tap sets differ by >= 16 TAU_A in
    some channel of some row, so section A sees every such position."""
    pat = _pattern().astype(np.float64) / 255.0
    crops = np.arange(1, MAX_CROP + 1)
    for side in SIDES:
        p32, p64 = _fp32_positions(crops, side), _fp64_positions(crops, side)
        ci, oi = np.nonzero(p32 != p64)
        if len(ci) == 0:
            continue
        n = crops[ci]
        ia, wa = _taps_at(p32[ci, oi], n)
        ib, wb = _taps_at(p64[ci, oi], n)
        ya = np.clip(np.einsum('kt,rktc->krc', wa, pat[:, ia]), 0, 1)          # the kernel clips its output
        yb = np.clip(np.einsum('kt,rktc->krc', wb, pat[:, ib]), 0, 1)
        sep = np.abs(ya - yb).max(axis=(1, 2))
        assert sep.min() >= 16 * TAU_A, (side, int(n[np.argmin(sep)]), sep.min() / TAU_A)


def _section_a_images(transpose):
    pat = _pattern()
    ims = [np.ascontiguousarray(pat[:, :I].transpose(1, 0, 2) if transpose else pat[:, :I])
           for I in range(1, MAX_CROP + 1)]
    flat = torch.from_numpy(np.concatenate([im.reshape(-1) for im in ims])).cuda()
    sizes = np.arange(1, MAX_CROP + 1, dtype=np.int64)
    offs = np.concatenate([[0], np.cumsum(12 * sizes)[:-1]]).astype(np.int64)
    hw = np.stack([np.full(MAX_CROP, 4), sizes], 1) if not transpose else np.stack([sizes, np.full(MAX_CROP, 4)], 1)
    return flat, offs, hw.astype(np.int32)


@gpu
@pytest.mark.parametrize('axis', ['x', 'y'])
def test_a_tap_positions_exhaustive(axis):
    """One launch per output side of 4096 images, 4 rows by I columns (I = 1..4096; transposed for y), the crop the
    whole image.  The other axis is in == out, an exact identity, so only this axis' taps are tested."""
    from oracle import data_util as OD
    _eng()
    tr = axis == 'y'
    src, offs, hw = _section_a_images(tr)
    srcf = src.double() / 255.0
    crops = np.arange(1, MAX_CROP + 1)
    offs_t = torch.from_numpy(offs).cuda()
    sizes_t = torch.from_numpy(crops).cuda()
    bad, worst = [], 0.0
    for side in SIDES:
        draws = [dict(box=(0, 0, int(h), int(w)), flip=False, color=NO_COLOUR) for h, w in hw]
        H, W = (side, 4) if tr else (4, side)
        got = _launch(src, offs, hw, draws, H, W).double()
        if tr:
            got = got.transpose(1, 2)                                   # -> [n, 4, side, 3]
        idx, w = OD._bicubic_axis_taps(crops, side)
        idx, w = torch.from_numpy(idx).cuda(), torch.from_numpy(w).cuda()
        r = torch.arange(4, device='cuda').view(1, 4, 1)
        ref = torch.zeros(MAX_CROP, 4, side, 3, dtype=torch.float64, device='cuda')
        for t in range(4):
            it = idx[:, None, :, t]                                     # [n, 1, side]
            pix = (it * 4 + r) if tr else (r * sizes_t.view(-1, 1, 1) + it)
            base = offs_t.view(-1, 1, 1) + 3 * pix
            for c in range(3):
                ref[..., c] += w[:, None, :, t] * srcf[base + c]
        assert not torch.isnan(got).any()
        ref.clamp_(0., 1.)                                              # the final clip (tf2/data_util.py:474)
        err = ((got - ref).abs() / TAU_A).amax(dim=(1, 3))              # [n, side]
        worst = max(worst, err.max().item())
        wrong = (err > 1).nonzero().cpu().numpy()
        if len(wrong):
            bad.append((side, len(wrong), sorted(set(int(k) + 1 for k in wrong[:, 0]))))
    _note('A', worst)
    assert not bad, '%s axis: %d (crop side, output index) positions wrong; per output side (side, positions, ' \
        'first crop sides): %s' % (axis, sum(b[1] for b in bad), [(s, k, c[:8]) for s, k, c in bad])


# --------------------------------------------------------------------------
# B. Replay of the pipeline's draws
# --------------------------------------------------------------------------
SIZES_B = [(375, 500), (500, 375), (333, 500), (480, 640), (768, 1024), (1200, 1600), (1536, 2048), (32, 32),
           (1, 1), (1, 7), (7, 1), (2, 2), (3, 5)]


def _images_b(n, seed, huge=True):
    """n uint8 images cycling over SIZES_B (one 3000x4000 first when `huge`), random content on the GPU."""
    g = torch.Generator(device='cuda').manual_seed(seed)
    sizes = ([(3000, 4000)] if huge else []) + [SIZES_B[k % len(SIZES_B)] for k in range(n - int(huge))]
    return [torch.randint(0, 256, (h, w, 3), dtype=torch.uint8, device='cuda', generator=g) for h, w in sizes]


def _replay(images, draws_per_view, H, W, strength):
    """Launch every view into one [n,H,W,3*views] tensor and compare each view with the oracle."""
    src, offs, hw = _pack(images)
    V = len(draws_per_view)
    out = torch.full((len(images), H, W, 3 * V), float('nan'), device='cuda')
    from simclr_b200 import data_util as D
    for v, draws in enumerate(draws_per_view):
        D.preprocess_for_train_packed(src, offs, hw, draws, H, W, out=out, channel_offset=3 * v)
    worst = 0.0
    for v, draws in enumerate(draws_per_view):
        for i, (im, d) in enumerate(zip(images, draws)):
            ref = _oracle(im, d, H, W)
            tau = colour_bound(TAU_RESIZE, d['color'], H * W)
            worst = max(worst, _check(out[i, ..., 3 * v:3 * v + 3], ref, tau,
                                      'strength %g, %dx%d, view %d, image %d (%dx%d), draw %r'
                                      % (strength, H, W, v, i, im.shape[0], im.shape[1], d)))
    return worst


@gpu
@pytest.mark.parametrize('strength', [1.0, 0.5, 1.5])
def test_b_replay_train_224_two_views(strength):
    _eng()
    rng = random.Random(int(strength * 100))
    images = _images_b(256, seed=int(strength * 10))
    draws = [[_draw(im, strength, rng) for im in images] for _ in range(2)]
    _note('B', _replay(images, draws, 224, 224, strength))


def _draw(im, strength, rng):
    from simclr_b200 import data_util as D
    return D.draw_train_augmentation(im.shape[0], im.shape[1], strength, rng)


@gpu
@pytest.mark.parametrize('H,W', [(32, 32), (64, 64), (48, 80), (80, 48)])
def test_b_replay_train_small_and_non_square(H, W):
    _eng()
    worst = 0.0
    for strength in (1.0, 0.5, 1.5):
        rng = random.Random(H * 1000 + W + int(strength * 7))
        images = _images_b(40, seed=H + W, huge=(H == 48))
        worst = max(worst, _replay(images, [[_draw(im, strength, rng) for im in images]], H, W, strength))
    _note('B', worst)


@gpu
def test_b_replay_eval_centre_crop():
    from oracle import data_util as OD
    from simclr_b200 import data_util as D
    _eng()
    images = _images_b(len(SIZES_B) + 1, seed=5)
    src, offs, hw = _pack(images)
    out = D.preprocess_for_eval_packed(src, offs, hw, 224, 224)
    worst = 0.0
    for i, im in enumerate(images):
        ref = OD.preprocess_for_eval(im.double() / 255.0, 224, 224)
        worst = max(worst, _check(out[i], ref, TAU_RESIZE, 'eval 224, image %dx%d' % tuple(im.shape[:2])))
    _note('B', worst)
    # crop=False at 32 (CIFAR sizes): the identity resize, exactly uint8 * float32(1/255)
    small = [im for im in _images_b(20, seed=6, huge=False) if im.shape[:2] == (32, 32)]
    src, offs, hw = _pack(small)
    out = D.preprocess_for_eval_packed(src, offs, hw, 32, 32, crop=False)
    assert torch.equal(out, torch.stack(small).float() * np.float32(1 / 255))


# --------------------------------------------------------------------------
# C. Colour-op edges
# --------------------------------------------------------------------------
def _colour_image():
    """256x256 uint8: an RGB grid, gray ramps with black and white, pure and near-pure hues, near-gray pixels
    (r = g = b +- 1), ties r = g > b and their permutations, and hues just either side of 0 and 1."""
    px = []
    lv = [0, 1, 2, 31, 64, 127, 128, 191, 254, 255]
    px += [(r, g, b) for r in lv for g in lv for b in lv]                                   # 1000
    px += [(k, k, k) for k in range(256)]                                                   # gray ramp
    for k in range(0, 256, 3):                                                              # pure / near-pure hues
        for c in range(3):
            for p in ((255, k, 0), (255, 0, k), (k, 255, 0), (254, k, 1), (255, k, k // 2)):
                px.append(tuple(p[(j + c) % 3] for j in range(3)))
    for k in range(1, 255):                                                                 # near-gray
        for d in ((1, 0, 0), (0, 1, 0), (0, 0, 1), (-1, 0, 0), (0, -1, 0), (0, 0, -1), (1, 1, 0), (1, -1, 0),
                  (0, 1, -1), (-1, 0, 1)):
            px.append(tuple(k + e for e in d))
    for k in range(1, 256, 2):                                                              # ties
        for m in (0, k // 2, k - 1):
            px += [(k, k, m), (k, m, k), (m, k, k)]
    for k in range(1, 256, 2):                                                              # hue near 0 and 1
        px += [(255, 0, k // 16), (255, k // 16, 0), (255, 1, 0), (255, 0, 1), (k, 0, 1), (k, 1, 0)]
    px = np.asarray(px, dtype=np.int64)
    assert len(px) <= 256 * 256 and px.min() >= 0 and px.max() <= 255
    rs = np.random.RandomState(4)
    fill = rs.randint(0, 256, (256 * 256 - len(px), 3))
    return torch.from_numpy(np.concatenate([px, fill]).astype(np.uint8).reshape(256, 256, 3))


BRIGHT = (0.0, 0.2, 1.8, 2.2)
CONTRAST = (-0.2, 0.0, 0.2, 1.8)
SAT = (0.0, 0.2, 1.8, 3.0)
HUE = (0.5, -0.5, 0.2, -0.2, 1e-3, -1e-3, 0.0)


def _colour_draws():
    """Every op order with every hue delta; the other factors cycle so that each value meets each order."""
    import itertools
    out = []
    for p, perm in enumerate(itertools.permutations(range(4))):
        for h, hue in enumerate(HUE):
            out.append(dict(apply_jitter=True, perm=perm, brightness=BRIGHT[(p + h) % 4],
                            contrast=CONTRAST[(p // 4 + h) % 4], saturation=SAT[(p // 2 + 3 * h) % 4], hue=hue,
                            apply_gray=(h == 2)))
    out.append(dict(NO_COLOUR, apply_gray=True))
    out.append(dict(NO_COLOUR))
    return out


@gpu
def test_c_colour_op_edges():
    from oracle import data_util as OD
    _eng()
    im = _colour_image()
    colours = _colour_draws()
    draws = [dict(box=(0, 0, 256, 256), flip=False, color=c) for c in colours]
    src, offs, hw = _pack([im] * len(draws))
    got = _launch(src, offs, hw, draws, 256, 256)
    x = im.cuda().double() / 255.0
    worst = 0.0
    for i, c in enumerate(colours):
        ref = torch.clamp(OD.random_color_jitter(x, c), 0., 1.)
        tau = colour_bound(TAU_IDENTITY, c, 256 * 256)
        worst = max(worst, _check(got[i], ref, tau, 'colour %r' % (c,)))
    _note('C', worst)


def test_colour_bounds_hold_in_float32():
    """The bounds above, for the oracle's colour ops in float32 torch against float64 on the section C image: every
    single op at every factor, and every chain of section C, within half its bound."""
    from oracle import data_util as OD
    im = _colour_image()
    x64 = im.double() / 255.0
    x32 = im.float() / 255.0
    npix = 256 * 256
    e0 = 2 * U
    worst = 0.0
    ops = [(0, f) for f in BRIGHT] + [(1, f) for f in CONTRAST] + [(2, f) for f in SAT] + [(3, f) for f in HUE]
    for op, f in ops:
        c = dict(NO_COLOUR, apply_jitter=True, perm=(op,), brightness=f, contrast=f, saturation=f, hue=f)
        err = (OD.random_color_jitter(x32, c).double() - OD.random_color_jitter(x64, c)).abs().max().item()
        r = err / op_bound(op, f, e0, npix) if err else 0.0
        assert r <= 0.5, (op, f, r)
        worst = max(worst, r)
    for c in _colour_draws():
        err = (OD.random_color_jitter(x32, c).double() - OD.random_color_jitter(x64, c)).abs().max().item()
        r = err / colour_bound(e0, c, npix) if err else 0.0
        assert r <= 0.5, (c, r)
        worst = max(worst, r)
    print('worst float32 / float64 ratio to the colour bounds: %.4f' % worst)
    assert worst > 0


# --------------------------------------------------------------------------
# D. Layout and edges
# --------------------------------------------------------------------------
def _small_batch(n, seed, strength=1.5):
    g = torch.Generator(device='cuda').manual_seed(seed)
    rng = random.Random(seed)
    images = []
    for k in range(n):
        h, w = SIZES_B[k % len(SIZES_B)] if k % 3 else (40 + k % 29, 50 + k % 31)
        h, w = min(h, 600), min(w, 600)
        images.append(torch.randint(0, 256, (h, w, 3), dtype=torch.uint8, device='cuda', generator=g))
    return images, [_draw(im, strength, rng) for im in images]


@gpu
def test_d_layouts_keep_other_channels():
    """Strides 6 (offsets 0 and 3) and 4 (offset 1): the view's channels hold the stride-3 result bit for bit, and
    every other channel keeps its NaN."""
    _eng()
    images, draws = _small_batch(12, seed=21)
    src, offs, hw = _pack(images)
    plain = _launch(src, offs, hw, draws, 48, 80)
    assert not torch.isnan(plain).any()
    for stride, off in ((6, 0), (6, 3), (4, 1)):
        out = _launch(src, offs, hw, draws, 48, 80, stride=stride, ch_off=off)
        assert torch.equal(out[..., off:off + 3], plain), (stride, off)
        rest = [c for c in range(stride) if not off <= c < off + 3]
        assert torch.isnan(out[..., rest]).all(), (stride, off)


@gpu
@pytest.mark.parametrize('n', [1, 1024])
def test_d_batch_sizes(n):
    """n = 1, and n = 1024 against launches of 100 images: each image's result does not depend on its batch; every
    37th is checked against the oracle."""
    _eng()
    images, draws = _small_batch(n, seed=n)
    src, offs, hw = _pack(images)
    out = _launch(src, offs, hw, draws, 64, 64)
    for a in range(0, n, 100):
        b = min(n, a + 100)
        part = _launch(*_pack(images[a:b]), draws[a:b], 64, 64)
        assert torch.equal(out[a:b], part)
    worst = 0.0
    for i in range(0, n, 37):
        worst = max(worst, _check(out[i], _oracle(images[i], draws[i], 64, 64),
                                  colour_bound(TAU_RESIZE, draws[i]['color'], 64 * 64), 'n=%d image %d' % (n, i)))
    _note('D', worst)


@gpu
def test_d_source_past_2_31_bytes():
    """An image stored at a byte offset >= 2^31 of the packed source gives the same bits as at offset 0."""
    _eng()
    images, draws = _small_batch(2, seed=31)
    im = images[1]
    big_off = 2 ** 31 + 5
    src = torch.zeros(big_off + im.numel(), dtype=torch.uint8, device='cuda')
    try:
        src[:images[0].numel()] = images[0].reshape(-1)
        src[big_off:] = im.reshape(-1)
        offs = np.asarray([0, big_off], dtype=np.int64)
        hw = np.asarray([im.shape[:2] for im in images], dtype=np.int32)
        far = _launch(src, offs, hw, draws, 64, 64)
    finally:
        del src
        torch.cuda.empty_cache()
    near = _launch(*_pack(images), draws, 64, 64)
    assert torch.equal(far, near)
    _check(far[1], _oracle(im, draws[1], 64, 64), colour_bound(TAU_RESIZE, draws[1]['color'], 64 * 64), 'far image')


@gpu
def test_d_repeatable_and_bad_arguments():
    from simclr_b200._lib import lib, stream_ptr, SimclrError
    _eng()
    images, draws = _small_batch(16, seed=41)
    src, offs, hw = _pack(images)
    a = _launch(src, offs, hw, draws, 224, 224)
    b = _launch(src, offs, hw, draws, 224, 224)
    assert torch.equal(a, b)
    # out_channel_offset + 3 > stride, and n = 0: SIMCLR_ERR_INVALID_ARG (-1), nothing written
    t = lambda x, dt: torch.as_tensor(x).to('cuda', dt)
    box = t([d['box'] for d in draws], torch.int32)
    flip = t([0] * 16, torch.uint8)
    col = torch.zeros(16, 8, device='cuda')
    out = torch.full((16, 8, 8, 4), float('nan'), device='cuda')
    for n, stride, off in ((16, 4, 2), (16, 3, 1), (0, 3, 0), (-1, 3, 0)):
        with pytest.raises(SimclrError, match='status -1'):
            lib.augment(src, t(offs, torch.int64), t(hw, torch.int32), box, flip, col, out, n, 8, 8, stride, off,
                        stream_ptr())
    torch.cuda.synchronize()
    assert torch.isnan(out).all()


# --------------------------------------------------------------------------
# E. End to end through build_input_fn
# --------------------------------------------------------------------------
def _toy_tfds(root, n_train=16, n_val=16):
    """<root>/toy/1.0.0 as test_gpu_jpeg.py makes it, with ImageNet-like and small sizes and one PNG."""
    import jpeg_corpus as JC
    from simclr_b200 import tfrecord as T
    d = os.path.join(root, 'toy', '1.0.0')
    os.makedirs(d)
    sizes = [(375, 500), (500, 333), (61, 90), (240, 180), (33, 47), (300, 300)]

    def enc(k):
        h, w = sizes[k % len(sizes)]
        a = JC.picture(h, w, 200 + k)
        if k % 7 == 3:
            return JC.png(a)
        return JC.jpeg(a, quality=90, subsampling=2 if k % 2 else 0)
    ex = [T.encode_example({'image': enc(k), 'label': k % 5}) for k in range(n_train + n_val)]
    T.write_records(os.path.join(d, 'toy-train.tfrecord-00000-of-00001'), ex[:n_train])
    T.write_records(os.path.join(d, 'toy-validation.tfrecord-00000-of-00001'), ex[n_train:])
    with open(os.path.join(d, 'features.json'), 'w') as f:
        json.dump({'featuresDict': {'features': {'label': {'classLabel': {'numClasses': '5'}}}}}, f)
    return root


@gpu
@pytest.mark.parametrize('decode', ['host', 'device'])
def test_e_input_fn_against_oracle(flags, tmp_path, monkeypatch, decode):
    """Pretraining at 224 and eval with the centre crop: every view of every feature row equals the oracle applied
    to the Pillow-decoded image with the draws the pipeline made."""
    from PIL import Image
    from simclr_b200 import data as DA, data_util as DU, engine
    from oracle import data_util as OD
    root = _toy_tfds(str(tmp_path))
    engine.set_engine(engine.Engine(precision='fp32', conv_engine='simt'))
    drawn = []
    orig_draw = DU.draw_train_augmentation

    def record(*a, **k):
        d = orig_draw(*a, **k)
        drawn.append(d)
        return d
    monkeypatch.setattr(DU, 'draw_train_augmentation', record)
    worst = 0.0
    for mode in ('pretrain', 'eval'):
        flags.set_flags(image_size=224, train_mode='pretrain', train_split='train', eval_split='validation',
                        color_jitter_strength=1.0)
        b = DA.TFRecordBuilder(root, 'toy', decode=decode)
        tokens = []
        for name in ('fetch_many', 'fetch_device'):
            fn = getattr(b, name)
            setattr(b, name, (lambda fn: lambda split, toks, *rest: (tokens.extend(toks), fn(split, toks, *rest))[1])(fn))
        del drawn[:]
        it = DA.build_input_fn(b, 8, None, mode == 'pretrain')(DA.InputContext(1, 0, 1), seed=3)
        for step in range(2):
            feats, _ = next(it)
            toks = tokens[8 * step:8 * step + 8]
            assert len(toks) == 8
            for i, (data, _) in enumerate(toks):
                with Image.open(io.BytesIO(data)) as pim:
                    im = torch.from_numpy(np.array(pim.convert('RGB')))
                if mode == 'pretrain':
                    for v in range(2):
                        d = drawn[16 * step + 8 * v + i]
                        ref = _oracle(im, d, 224, 224)
                        tau = colour_bound(TAU_RESIZE, d['color'], 224 * 224)
                        worst = max(worst, _check(feats[i, ..., 3 * v:3 * v + 3], ref, tau,
                                                  '%s decode, step %d, image %d, view %d' % (decode, step, i, v)))
                else:
                    ref = OD.preprocess_for_eval(im.cuda().double() / 255.0, 224, 224)
                    worst = max(worst, _check(feats[i], ref, TAU_RESIZE,
                                              '%s decode, eval, image %d (%dx%d)' % (decode, i, *im.shape[:2])))
        if mode == 'pretrain':
            assert len(drawn) == 32
        else:
            assert not drawn
    _note('E', worst)


def test_section_c_image_covers_the_edges():
    """The section C image holds near-gray pixels, ties and hues within 1e-3 of the wrap."""
    from oracle import data_util as OD
    im = _colour_image()
    x = im.double() / 255.0
    hsv = OD.rgb_to_hsv(x)
    rng = (x.amax(-1) - x.amin(-1))
    assert ((rng > 0) & (rng <= 1 / 255 + 1e-12)).sum() > 1000
    r, g, b = x.unbind(-1)
    assert ((r == g) & (g > b)).sum() > 100
    h = hsv[..., 0][rng > 0]
    assert ((h > 0) & (h < 1e-3)).any() and ((h > 1 - 1e-3) & (h < 1)).any()
    assert math.isclose(float(x.max()), 1.0) and float(x.min()) == 0.0
