"""CPU oracle of the baseline JPEG decode that Pillow runs through libjpeg-turbo -- TEST INFRASTRUCTURE ONLY.

It restates, in plain Python / numpy integer arithmetic, what libjpeg-turbo does for the subset the device decoder
(`simclr_b200/csrc/jpeg.cu`) accepts: baseline / extended sequential Huffman (SOF0 / SOF1), 8-bit, one interleaved
scan, 1 or 3 components, luma sampling h, v in {1, 2} with 1x1 chroma.  Stage by stage:

  * marker parsing (DQT, DHT, SOF, DRI, SOS; APPn / COM skipped);
  * Huffman decoding with DC prediction, restart markers (DC predictors reset, bit buffer realigned) and
    0xFF 0x00 byte stuffing;
  * dequantisation and de-zigzag;
  * `jpeg_idct_islow` (jidctint.c): CONST_BITS 13, PASS1_BITS 2, the zero-AC column / row shortcuts, and the
    post-IDCT range limit (10-bit wrap-around table, then clamp to [0, 255]);
  * fancy upsampling (jdsample.c): h2v1 and h2v2 "triangle" filters with the alternating +1/+2 and +8/+7 biases,
    first / last column special cases and edge-replicated context rows; h1v2 with biases +1/+2; box replication when
    the downsampled width is <= 2 (libjpeg-turbo picks the plain upsampler there);
  * YCbCr -> RGB with the 16-bit fixed-point tables of jdcolor.c; grayscale replicated to RGB as `convert('RGB')`.

Nothing here is fast: it is the specification the CUDA kernels are tested against, and it must equal
`np.array(Image.open(f).convert('RGB'))` exactly (tests/test_jpeg.py).
"""
import numpy as np

ZIGZAG = np.array([                       # jpeg_natural_order: zigzag index -> natural (row-major) index
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21,
    28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61,
    54, 47, 55, 62, 63], dtype=np.int64)


class Unsupported(ValueError):
    pass


def _u16(b, i):
    return (b[i] << 8) | b[i + 1]


def parse(data):
    """Markers up to the first SOS -> dict(frame, tables, scan, restart interval, entropy-data start)."""
    b = data
    if len(b) < 4 or b[0] != 0xFF or b[1] != 0xD8:
        raise Unsupported('not a JPEG')
    i, q, huff, dri, frame, jfif, adobe = 2, {}, {}, 0, None, False, None
    while True:
        while i < len(b) and b[i] == 0xFF and i + 1 < len(b) and b[i + 1] == 0xFF:
            i += 1                                            # fill bytes
        if i + 4 > len(b) or b[i] != 0xFF:
            raise Unsupported('truncated header')
        m, L = b[i + 1], _u16(b, i + 2)
        seg = b[i + 4:i + 2 + L]
        if L < 2 or i + 2 + L > len(b):
            raise Unsupported('bad segment length')
        i += 2 + L
        if m == 0xDB:                                         # DQT
            j = 0
            while j < len(seg):
                pq, tq = seg[j] >> 4, seg[j] & 15
                n = 64 * (pq + 1)
                vals = np.frombuffer(bytes(seg[j + 1:j + 1 + n]), dtype='>u2' if pq else np.uint8).astype(np.int64)
                if pq > 1 or tq > 3 or len(vals) != 64:
                    raise Unsupported('bad DQT')
                nat = np.zeros(64, np.int64)
                nat[ZIGZAG] = vals
                q[tq] = nat
                j += 1 + n
        elif m == 0xC4:                                       # DHT
            j = 0
            while j < len(seg):
                tc, th = seg[j] >> 4, seg[j] & 15
                counts = list(seg[j + 1:j + 17])
                n = sum(counts)
                if tc > 1 or th > 3 or len(counts) != 16 or n > 256 or j + 17 + n > len(seg):
                    raise Unsupported('bad DHT')
                huff[(tc, th)] = _huff_table(counts, list(seg[j + 17:j + 17 + n]))
                j += 17 + n
        elif m in (0xC0, 0xC1):                               # SOF0 / SOF1
            if frame is not None or len(seg) < 6:
                raise Unsupported('bad SOF')
            P, H, W, nf = seg[0], _u16(seg, 1), _u16(seg, 3), seg[5]
            comps = [(seg[6 + 3 * k], seg[7 + 3 * k] >> 4, seg[7 + 3 * k] & 15, seg[8 + 3 * k]) for k in range(nf)]
            if P != 8 or H == 0 or W == 0 or nf not in (1, 3) or len(seg) != 6 + 3 * nf:
                raise Unsupported('frame outside the subset')
            frame = (H, W, comps)
        elif 0xC2 <= m <= 0xCF and m not in (0xC4, 0xC8, 0xCC):
            raise Unsupported('SOF%d' % (m - 0xC0))
        elif m == 0xDD:
            dri = _u16(seg, 0)
        elif m == 0xE0 and bytes(seg[:5]) == b'JFIF\0':
            jfif = True
        elif m == 0xEE and bytes(seg[:5]) == b'Adobe' and len(seg) >= 12:
            adobe = seg[11]
        elif m == 0xDA:                                       # SOS
            ns = seg[0]
            scomps = [(seg[1 + 2 * k], seg[2 + 2 * k] >> 4, seg[2 + 2 * k] & 15) for k in range(ns)]
            if frame is None or ns != len(frame[2]) or [c[0] for c in scomps] != [c[0] for c in frame[2]]:
                raise Unsupported('scan outside the subset')
            H, W, comps = frame
            if len(comps) == 3 and (not jfif and (adobe == 0 or (adobe is None and [c[0] for c in comps] == [82, 71, 66]))):
                raise Unsupported('RGB JPEG')
            return dict(H=H, W=W, comps=comps, q=[q[c[3]] for c in comps],
                        dc=[huff[(0, s[1])] for s in scomps], ac=[huff[(1, s[2])] for s in scomps], dri=dri, start=i)
        elif m in (0xD8, 0xD9) or 0xD0 <= m <= 0xD7:
            raise Unsupported('unexpected marker')


def _huff_table(counts, vals):
    """(maxcode, valptr - mincode, vals) of jdhuff.c's derived table; lengths 1..16."""
    maxcode, valoff, code, k = [-1] * 18, [0] * 18, 0, 0
    for l in range(1, 17):
        if counts[l - 1]:
            valoff[l] = k - code
            code += counts[l - 1]
            k += counts[l - 1]
            maxcode[l] = code - 1
            if code >= (1 << l):
                raise Unsupported('over-subscribed Huffman table')
        code <<= 1
    maxcode[17] = 1 << 30
    return maxcode, valoff, vals


class _Bits:
    """MSB-first bit reader over the entropy-coded bytes: 0xFF 0x00 -> 0xFF; at any other marker the data ends and
    zeros are supplied (jdhuff.c's fill_bit_buffer)."""

    def __init__(self, b, pos):
        self.b, self.pos, self.acc, self.n = b, pos, 0, 0

    def bit(self):
        if self.n == 0:
            c = 0
            if self.pos < len(self.b):
                c = self.b[self.pos]
                if c == 0xFF:
                    if self.pos + 1 < len(self.b) and self.b[self.pos + 1] == 0:
                        self.pos += 2
                    else:
                        c = 0                                # a marker: stay on it, supply zeros
                else:
                    self.pos += 1
            self.acc, self.n = c, 8
        self.n -= 1
        return (self.acc >> self.n) & 1

    def bits(self, s):
        v = 0
        for _ in range(s):
            v = (v << 1) | self.bit()
        return v

    def restart(self, k):
        """Discard the rest of the current byte, then read RSTk."""
        self.n = 0
        if self.b[self.pos:self.pos + 2] != bytes([0xFF, 0xD0 + (k & 7)]):
            raise Unsupported('missing restart marker')
        self.pos += 2

    def decode(self, tab):
        maxcode, valoff, vals = tab
        code, l = self.bit(), 1
        while code > maxcode[l]:
            code, l = (code << 1) | self.bit(), l + 1
        if l > 16:
            raise Unsupported('bad Huffman code')
        return vals[code + valoff[l]]


def _extend(v, s):
    return v - (1 << s) + 1 if s and v < (1 << (s - 1)) else v


def entropy_decode(data, hdr):
    """-> per component int64 coefficient blocks [bh, bw, 64] in natural order (padded to whole MCUs)."""
    H, W, comps = hdr['H'], hdr['W'], hdr['comps']
    if len(comps) == 1:
        hs, vs = [1], [1]
        mx, my = -(-W // 8), -(-H // 8)
    else:
        hs, vs = [c[1] for c in comps], [c[2] for c in comps]
        mx, my = -(-W // (8 * max(hs))), -(-H // (8 * max(vs)))
    blocks = [np.zeros((my * v, mx * h, 64), np.int64) for h, v in zip(hs, vs)]
    rd = _Bits(data, hdr['start'])
    pred = [0] * len(comps)
    dri, nrst = hdr['dri'], 0
    for m in range(mx * my):
        if dri and m and m % dri == 0:
            rd.restart(nrst)
            nrst += 1
            pred = [0] * len(comps)
        y0, x0 = divmod(m, mx)
        for c in range(len(comps)):
            for v in range(vs[c]):
                for h in range(hs[c]):
                    blk = blocks[c][y0 * vs[c] + v, x0 * hs[c] + h]
                    s = rd.decode(hdr['dc'][c])
                    pred[c] += _extend(rd.bits(s), s)
                    blk[0] = np.int16(np.int64(pred[c]).astype(np.int16))    # JCOEF is 16-bit
                    k = 1
                    while k < 64:
                        rs = rd.decode(hdr['ac'][c])
                        r, s = rs >> 4, rs & 15
                        if s:
                            k += r
                            if k > 63:
                                raise Unsupported('coefficient index past 63')
                            blk[ZIGZAG[k]] = _extend(rd.bits(s), s)
                        elif r != 15:
                            break
                        else:
                            k += 15
                        k += 1
    return blocks


CONST_BITS, PASS1_BITS = 13, 2
FIX = dict(c0_298631336=2446, c0_390180644=3196, c0_541196100=4433, c0_765366865=6270, c0_899976223=7373,
           c1_175875602=9633, c1_501321110=12299, c1_847759065=15137, c1_961570560=16069, c2_053119869=16819,
           c2_562915447=20995, c3_072711026=25172)


def _idct_1d(x, shift):
    """One jidctint.c pass over 8 int64 arrays (the 8 inputs of a column / row); DESCALE by `shift`."""
    f = FIX
    z2, z3 = x[2], x[6]
    z1 = (z2 + z3) * f['c0_541196100']
    tmp2 = z1 + z3 * -f['c1_847759065']
    tmp3 = z1 + z2 * f['c0_765366865']
    tmp0 = (x[0] + x[4]) << CONST_BITS
    tmp1 = (x[0] - x[4]) << CONST_BITS
    tmp10, tmp13, tmp11, tmp12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    t0, t1, t2, t3 = x[7], x[5], x[3], x[1]
    z1, z2, z3, z4 = t0 + t3, t1 + t2, t0 + t2, t1 + t3
    z5 = (z3 + z4) * f['c1_175875602']
    t0, t1, t2, t3 = t0 * f['c0_298631336'], t1 * f['c2_053119869'], t2 * f['c3_072711026'], t3 * f['c1_501321110']
    z1, z2 = z1 * -f['c0_899976223'], z2 * -f['c2_562915447']
    z3, z4 = z3 * -f['c1_961570560'] + z5, z4 * -f['c0_390180644'] + z5
    t0, t1, t2, t3 = t0 + z1 + z3, t1 + z2 + z4, t2 + z2 + z3, t3 + z1 + z4
    r = 1 << (shift - 1)
    return [(tmp10 + t3 + r) >> shift, (tmp11 + t2 + r) >> shift, (tmp12 + t1 + r) >> shift, (tmp13 + t0 + r) >> shift,
            (tmp13 - t0 + r) >> shift, (tmp12 - t1 + r) >> shift, (tmp11 - t2 + r) >> shift, (tmp10 - t3 + r) >> shift]


def _range_limit(v):
    """libjpeg's IDCT range-limit table: index (v & 1023) -> clamp(v + 128) with 10-bit wrap-around."""
    s = ((v + 512) & 1023) - 512
    return np.clip(s + 128, 0, 255)


def idct_islow(coef, qtab):
    """coef [..., 64] natural order, qtab [64] -> uint8 [..., 8, 8]."""
    d = (coef * qtab).reshape(coef.shape[:-1] + (8, 8))
    # pass 1: columns (input rows are frequencies v); an all-zero AC column is the DC << PASS1_BITS (same value)
    cols = _idct_1d([d[..., k, :] for k in range(8)], CONST_BITS - PASS1_BITS)
    zero = np.all(d[..., 1:, :] == 0, axis=-2)
    ws = np.stack([np.where(zero, d[..., 0, :] << PASS1_BITS, c) for c in cols], axis=-2)
    # pass 2: rows, final descale by 3 more bits (the 8-point normalisation), then the range limit
    rows = _idct_1d([ws[..., :, k] for k in range(8)], CONST_BITS + PASS1_BITS + 3)
    zero = np.all(ws[..., :, 1:] == 0, axis=-1)
    out = np.stack([np.where(zero, (ws[..., :, 0] + (1 << (PASS1_BITS + 2))) >> (PASS1_BITS + 3), r) for r in rows], -1)
    return _range_limit(out).astype(np.uint8)


def planes(blocks, q):
    """Component planes, padded to whole MCUs: [bh*8, bw*8] uint8 each."""
    out = []
    for blk, qt in zip(blocks, q):
        bh, bw = blk.shape[:2]
        px = idct_islow(blk, qt)                               # [bh, bw, 8, 8]
        out.append(px.transpose(0, 2, 1, 3).reshape(bh * 8, bw * 8))
    return out


def _h2v1(c):
    """jdsample.c h2v1_fancy_upsample on one row set [rows, cw] -> [rows, 2cw]."""
    c = c.astype(np.int64)
    cw = c.shape[1]
    if cw <= 2:
        return np.repeat(c, 2, axis=1)
    left = np.concatenate([c[:, :1], c[:, :-1]], 1)
    right = np.concatenate([c[:, 1:], c[:, -1:]], 1)
    even = (3 * c + left + 1) >> 2
    odd = (3 * c + right + 2) >> 2
    even[:, 0], odd[:, -1] = c[:, 0], c[:, -1]
    return np.stack([even, odd], -1).reshape(c.shape[0], 2 * cw)


def _context_rows(c):
    """(row above, row below) of every row, edge rows replicated (jdmainct.c context pointers)."""
    return np.concatenate([c[:1], c[:-1]], 0), np.concatenate([c[1:], c[-1:]], 0)


def _h1v2(c):
    c = c.astype(np.int64)
    above, below = _context_rows(c)
    top = (3 * c + above + 1) >> 2
    bot = (3 * c + below + 2) >> 2
    return np.stack([top, bot], 1).reshape(2 * c.shape[0], c.shape[1])


def _h2v2(c):
    c = c.astype(np.int64)
    cw = c.shape[1]
    if cw <= 2:
        return np.repeat(np.repeat(c, 2, axis=0), 2, axis=1)
    above, below = _context_rows(c)
    out = []
    for far in (above, below):
        s = 3 * c + far                                        # column sums
        left = np.concatenate([s[:, :1], s[:, :-1]], 1)
        right = np.concatenate([s[:, 1:], s[:, -1:]], 1)
        even = (3 * s + left + 8) >> 4
        odd = (3 * s + right + 7) >> 4
        even[:, 0] = (4 * s[:, 0] + 8) >> 4
        odd[:, -1] = (4 * s[:, -1] + 7) >> 4
        out.append(np.stack([even, odd], -1).reshape(c.shape[0], 2 * cw))
    return np.stack(out, 1).reshape(2 * c.shape[0], 2 * cw)


def ycc_to_rgb(y, cb, cr):
    """jdcolor.c ycc_rgb_convert: SCALEBITS 16, FIX(x) = round(x * 65536), ONE_HALF rounding in the tables."""
    y, xb, xr = y.astype(np.int64), cb.astype(np.int64) - 128, cr.astype(np.int64) - 128
    half = 1 << 15
    r = y + ((91881 * xr + half) >> 16)
    g = y + ((-46802 * xr - 22554 * xb + half) >> 16)
    b = y + ((116130 * xb + half) >> 16)
    return np.clip(np.stack([r, g, b], -1), 0, 255).astype(np.uint8)


def decode(data):
    """JPEG bytes -> uint8 [H, W, 3], as `np.array(Image.open(...).convert('RGB'))`.  Raises `Unsupported`
    outside the subset."""
    data = bytes(data)
    hdr = parse(data)
    H, W, comps = hdr['H'], hdr['W'], hdr['comps']
    if len(comps) == 3:
        hmax, vmax = comps[0][1], comps[0][2]
        if hmax not in (1, 2) or vmax not in (1, 2) or any(c[1:3] != (1, 1) for c in comps[1:]):
            raise Unsupported('sampling outside the subset')
    elif comps[0][1] not in (1, 2) or comps[0][2] not in (1, 2):
        raise Unsupported('sampling outside the subset')
    p = planes(entropy_decode(data, hdr), hdr['q'])
    if len(comps) == 1:
        return np.repeat(p[0][:H, :W, None], 3, axis=2)
    cw, ch = -(-W // hmax), -(-H // vmax)
    up = {(1, 1): lambda c: c, (2, 1): _h2v1, (1, 2): _h1v2, (2, 2): _h2v2}[(hmax, vmax)]
    cb, cr = (up(x[:ch, :cw])[:H, :W] for x in p[1:])
    return ycc_to_rgb(p[0][:H, :W], cb, cr)
