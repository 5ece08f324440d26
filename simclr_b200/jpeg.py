"""Host half of the device JPEG decoder: header parsing, batch packing, and the Pillow fall-back.

`parse(data)` reads the markers up to the first SOS (never the entropy-coded bytes) and returns a `Header`, or None
for anything the device kernels do not decode:

  * supported: SOF0 / SOF1, 8-bit samples, 1 or 3 components in one interleaved scan, luma sampling h, v in {1, 2}
    with 1x1 chroma (4:4:4, 4:2:2, 4:2:0, 4:4:0, grayscale), restart intervals, any APPn / COM segment (EXIF is
    ignored, as Pillow ignores it);
  * unsupported: progressive, arithmetic-coded, lossless and 12-bit frames, CMYK / YCCK, RGB JPEGs (Adobe
    transform 0), non-interleaved scans, other sampling factors, malformed headers, and bytes that are not a JPEG
    (the PNGs of many TFDS datasets).  These keep the host path: Pillow decodes them, or raises, as before.

`decode_batch(datas, device)` returns the packed layout `simclr_augment` reads -- uint8 HWC images back to back on the
device, `src_offset [n] int64`, `src_hw [n][2] int32` -- decoding the supported images with one
`simclr_jpeg_decode` call on a side stream and the others with Pillow.  `start_decode` splits it in two so that the
image sizes, known from the headers, are available before the decode finishes.  The output equals
`np.array(Image.open(b).convert('RGB'))` bit for bit (libjpeg-turbo's JDCT_ISLOW IDCT and fancy upsampling are
integer arithmetic, restated in oracle/jpeg.py).
"""
import collections
import io

import numpy as np
import torch

from ._lib import lib

Header = collections.namedtuple('Header', 'width height mode comps q dc ac restart_interval scan_start scan_end')
Header.__doc__ = """mode 'L' or 'RGB' (Pillow's); comps [(id, h, v)]; q per component: 64 uint16 in natural order
(bytes); dc / ac per component: (16 code-length counts, symbols) as bytes; restart_interval in MCUs (0: none);
[scan_start, scan_end): the entropy-coded bytes."""

_ZIGZAG = np.array([
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21,
    28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61,
    54, 47, 55, 62, 63])
_HUFF_BYTES = 1424          # uint16 look[512], int32 maxcode[18], int32 valoff[18], uint8 vals[256]
_D_FIELDS, _S_FIELDS = 40, 8


class _Bad(Exception):
    pass


def _valid_huffman(counts, vals, is_dc):
    """The checks of libjpeg's jpeg_make_d_derived_tbl: no over-subscribed code length, DC symbols <= 15."""
    code = 0
    for l in range(1, 17):
        code += counts[l - 1]
        if code >= (1 << l) and counts[l - 1]:
            return False
        code <<= 1
    return not (is_dc and any(v > 15 for v in vals))


def parse(data):
    """-> Header, or None when the device decoder does not take these bytes (see the module docstring).  Never
    raises on malformed input."""
    try:
        return _parse(memoryview(data).cast('B'))
    except (_Bad, IndexError, KeyError, ValueError, TypeError):
        return None


def _parse(b):
    n = len(b)
    if n < 4 or b[0] != 0xFF or b[1] != 0xD8:
        raise _Bad
    i, q, huff, dri, frame, jfif, adobe = 2, {}, {}, 0, None, False, None
    while True:
        while i + 1 < n and b[i] == 0xFF and b[i + 1] == 0xFF:
            i += 1
        if i + 4 > n or b[i] != 0xFF:
            raise _Bad
        m, L = b[i + 1], (b[i + 2] << 8) | b[i + 3]
        if L < 2 or i + 2 + L > n:
            raise _Bad
        seg = b[i + 4:i + 2 + L]
        i += 2 + L
        if m == 0xDB:                                          # DQT
            j = 0
            while j < len(seg):
                pq, tq = seg[j] >> 4, seg[j] & 15
                size = 64 * (pq + 1)
                if pq > 1 or tq > 3 or j + 1 + size > len(seg):
                    raise _Bad
                zz = np.frombuffer(seg[j + 1:j + 1 + size], dtype='>u2' if pq else np.uint8)
                nat = np.empty(64, np.uint16)
                nat[_ZIGZAG] = zz
                q[tq] = nat.tobytes()
                j += 1 + size
        elif m == 0xC4:                                        # DHT
            j = 0
            while j < len(seg):
                tc, th = seg[j] >> 4, seg[j] & 15
                if tc > 1 or th > 3 or j + 17 > len(seg):
                    raise _Bad
                counts = bytes(seg[j + 1:j + 17])
                k = sum(counts)
                vals = bytes(seg[j + 17:j + 17 + k])
                if k > 256 or len(vals) != k or not _valid_huffman(counts, vals, tc == 0):
                    raise _Bad
                huff[(tc, th)] = (counts, vals)
                j += 17 + k
        elif m in (0xC0, 0xC1):                                # SOF0 / SOF1 (Huffman, sequential)
            if frame is not None or len(seg) < 6:
                raise _Bad
            P, H, W, nf = seg[0], (seg[1] << 8) | seg[2], (seg[3] << 8) | seg[4], seg[5]
            if P != 8 or H == 0 or W == 0 or nf not in (1, 3) or len(seg) != 6 + 3 * nf:
                raise _Bad
            comps = [(seg[6 + 3 * k], seg[7 + 3 * k] >> 4, seg[7 + 3 * k] & 15, seg[8 + 3 * k]) for k in range(nf)]
            if len({c[0] for c in comps}) != nf or any(c[3] > 3 for c in comps):
                raise _Bad
            if comps[0][1] not in (1, 2) or comps[0][2] not in (1, 2) or any(c[1:3] != (1, 1) for c in comps[1:]):
                raise _Bad
            frame = (H, W, comps)
        elif 0xC2 <= m <= 0xCF or m in (0xDC, 0xDE, 0xDF):     # other SOFn, DAC, DNL, DHP, EXP
            raise _Bad
        elif m == 0xDD:                                        # DRI
            if len(seg) != 2:
                raise _Bad
            dri = (seg[0] << 8) | seg[1]
        elif m == 0xE0 and bytes(seg[:5]) == b'JFIF\0':
            jfif = True
        elif m == 0xEE and len(seg) >= 12 and bytes(seg[:5]) == b'Adobe':
            adobe = seg[11]
        elif m == 0xDA:                                        # SOS: the one scan must hold every component
            if frame is None or len(seg) < 1:
                raise _Bad
            H, W, comps = frame
            ns = seg[0]
            if ns != len(comps) or len(seg) != 4 + 2 * ns:
                raise _Bad
            sc = [(seg[1 + 2 * k], seg[2 + 2 * k] >> 4, seg[2 + 2 * k] & 15) for k in range(ns)]
            if [c[0] for c in sc] != [c[0] for c in comps] or tuple(seg[1 + 2 * ns:4 + 2 * ns]) != (0, 63, 0):
                raise _Bad
            if len(comps) == 3 and not jfif and (adobe == 0 or (adobe is None and [c[0] for c in comps] == [82, 71, 66])):
                raise _Bad                                     # libjpeg would read these as RGB
            end = n - 2 if b[n - 2] == 0xFF and b[n - 1] == 0xD9 else n
            return Header(W, H, 'L' if len(comps) == 1 else 'RGB', [c[:3] for c in comps],
                          [q[c[3]] for c in comps], [huff[(0, s[1])] for s in sc], [huff[(1, s[2])] for s in sc],
                          dri, i, max(end, i))
        elif m in (0xD8, 0xD9) or 0xD0 <= m <= 0xD7 or m == 0x01:
            raise _Bad


# ---- device tables ------------------------------------------------------------------------------------------------
_huff_cache = {}


def _huffman_table(counts, vals):
    """The 1424-byte table simclr_jpeg_decode reads (include/simclr_b200.h)."""
    key = counts + vals
    t = _huff_cache.get(key)
    if t is not None:
        return t
    look = np.zeros(512, np.uint16)
    maxcode = np.full(18, -1, np.int32)
    valoff = np.zeros(18, np.int32)
    code = k = 0
    for l in range(1, 17):
        c = counts[l - 1]
        if c:
            valoff[l] = k - code
            if l <= 9:
                for j in range(c):
                    look[(code + j) << (9 - l):(code + j + 1) << (9 - l)] = (l << 8) | vals[k + j]
            code += c
            k += c
            maxcode[l] = code - 1
        code <<= 1
    v = np.zeros(256, np.uint8)
    v[:len(vals)] = np.frombuffer(vals, np.uint8)
    t = look.tobytes() + maxcode.tobytes() + valoff.tobytes() + v.tobytes()
    assert len(t) == _HUFF_BYTES
    if len(_huff_cache) > 4096:
        _huff_cache.clear()
    _huff_cache[key] = t
    return t


def _geometry(h):
    """(mcux, mcuy, hmax, vmax, [(bw, bh, hs, vs)] per component)."""
    if len(h.comps) == 1:
        bw, bh = -(-h.width // 8), -(-h.height // 8)
        return bw, bh, 1, 1, [(bw, bh, 1, 1)]
    hmax, vmax = h.comps[0][1], h.comps[0][2]
    mx, my = -(-h.width // (8 * hmax)), -(-h.height // (8 * vmax))
    return mx, my, hmax, vmax, [(mx * c[1], my * c[2], c[1], c[2]) for c in h.comps]


def _segments(data, h, nmcu):
    """[(start, end, first MCU, MCU count)]: the whole scan, or one entry per restart interval.  Restart markers are
    located with a vectorised search (0xFF is always followed by 0x00 or a marker in entropy-coded data); a marker
    out of sequence or missing sends the image to the host path."""
    ri = h.restart_interval
    nint = -(-nmcu // ri) if ri else 1
    if nint == 1:
        return [(h.scan_start, h.scan_end, 0, nmcu)]
    a = np.frombuffer(data, np.uint8, count=h.scan_end - h.scan_start, offset=h.scan_start)
    idx = np.flatnonzero((a[:-1] == 0xFF) & ((a[1:] & 0xF8) == 0xD0))[:nint - 1]
    if len(idx) != nint - 1 or np.any(a[idx + 1] != 0xD0 + (np.arange(nint - 1) & 7)):
        return None
    starts = np.concatenate([[0], idx + 2]) + h.scan_start
    ends = np.concatenate([idx, [h.scan_end - h.scan_start]]) + h.scan_start
    return [(int(s), int(e), k * ri, min(ri, nmcu - k * ri)) for k, (s, e) in enumerate(zip(starts, ends))]


def _pillow(data):
    from PIL import Image
    with Image.open(io.BytesIO(data)) as im:
        return np.array(im.convert('RGB'), dtype=np.uint8)


def _align(x, a=16):
    return (x + a - 1) // a * a


_streams = {}


def _side_stream(device):
    s = _streams.get(device)
    if s is None:
        s = _streams[device] = torch.cuda.Stream(device)
    return s


class DecodeJob:
    """One batch in flight.  `hw` (int64 [n, 2] numpy) is known on return from `start_decode`; `finish()` waits for
    the device error flags, decodes the fall-back images with Pillow and returns `(src, src_offset, src_hw)` on the
    device, with the current stream ordered after every write to `src`.  `bytes_to_device` counts the
    host-to-device traffic of the batch."""

    def __init__(self, datas, device, pool=None, fill=None):
        device = torch.device(device)
        if device.type == 'cuda' and device.index is None:
            device = torch.device('cuda', torch.cuda.current_device())
        self.device, self._pool = device, pool
        n = len(datas)
        hdrs = [parse(d) for d in datas]
        dev_idx = [i for i, h in enumerate(hdrs) if h is not None]
        self._datas = datas
        self._host = {}                                         # image -> Pillow decode (future or array)
        hw = np.zeros((n, 2), np.int64)
        for i in dev_idx:
            hw[i] = hdrs[i].height, hdrs[i].width
        for i, h in enumerate(hdrs):
            if h is None:                                      # Pillow reads the size without decoding
                from PIL import Image
                with Image.open(io.BytesIO(datas[i])) as im:
                    hw[i] = im.size[1], im.size[0]
                self._host[i] = self._submit(i)
        self.hw = hw
        nbytes = hw[:, 0] * hw[:, 1] * 3
        self.offsets = np.concatenate([[0], np.cumsum(nbytes)[:-1]]).astype(np.int64)
        cur = torch.cuda.current_stream(device)
        self._stream = _side_stream(device)
        self.src = torch.empty(int(nbytes.sum()), dtype=torch.uint8, device=device)
        if fill is not None:
            self.src.fill_(fill)
        self.bytes_to_device = 0
        self._dev_idx, self._err_host, self._err_event, self._keep = [], None, None, []
        self.on_device = []                                     # images the kernels decoded ...
        self.device_failed = []                                 # ... and those whose error flag came back set
        plan = self._pack([(i, hdrs[i]) for i in dev_idx]) if dev_idx else None
        self._stream.wait_stream(cur)                           # the allocations above are cur-stream ordered
        if plan is not None:
            self._launch(*plan)

    def _pack(self, items):
        """Descriptors, segments, tables and entropy-coded bytes of the device images in one pinned buffer."""
        descs, segs, tabs, tab_off, chunks = [], [], [], {}, []
        tab_bytes = data_bytes = blk = max_blocks = max_pixels = 0
        dev_idx = []

        def table(t):
            nonlocal tab_bytes
            o = tab_off.get(t)
            if o is None:
                o = tab_off[t] = tab_bytes
                tabs.append(t)
                tab_bytes += _align(len(t))
            return o
        for i, h in items:
            mx, my, hmax, vmax, geo = _geometry(h)
            sg = _segments(self._datas[i], h, mx * my)
            if sg is None:
                self._host[i] = self._submit(i)
                continue
            d = np.zeros(_D_FIELDS, np.int64)
            nb = [bw * bh for bw, bh, _, _ in geo]
            d[:10] = [self.offsets[i], h.height, h.width, len(geo), hmax, vmax, mx, my, blk, sum(nb)]
            for c, (bw, bh, hs, vs) in enumerate(geo):
                d[10 + c], d[13 + c], d[16 + c], d[19 + c], d[22 + c] = sum(nb[:c]), bw, bh, hs, vs
                d[25 + c] = table(h.q[c])
                d[28 + c] = table(_huffman_table(*h.dc[c]))
                d[31 + c] = table(_huffman_table(*h.ac[c]))
            base = data_bytes - h.scan_start
            k = len(descs)
            segs += [(k, s + base, e + base, m0, nm, 0, 0, 0) for s, e, m0, nm in sg]
            chunks.append(memoryview(self._datas[i])[h.scan_start:h.scan_end])
            data_bytes += h.scan_end - h.scan_start
            descs.append(d)
            dev_idx.append(i)
            blk += int(d[9])
            max_blocks, max_pixels = max(max_blocks, int(d[9])), max(max_pixels, h.height * h.width)
        if not descs:
            return None
        self._dev_idx = dev_idx
        o_seg = _align(len(descs) * _D_FIELDS * 8)
        o_tab = o_seg + _align(len(segs) * _S_FIELDS * 8)
        o_dat = o_tab + tab_bytes
        total = _align(o_dat + data_bytes + 8)
        buf = torch.empty(total, dtype=torch.uint8, pin_memory=True)
        a = buf.numpy()
        a[:o_seg].view(np.int64)[:len(descs) * _D_FIELDS] = np.concatenate(descs)
        a[o_seg:o_tab].view(np.int64)[:len(segs) * _S_FIELDS] = np.asarray(segs, np.int64).reshape(-1)
        o = o_tab
        for t in tabs:
            a[o:o + len(t)] = np.frombuffer(t, np.uint8)
            o += _align(len(t))
        o = o_dat
        for c in chunks:
            a[o:o + len(c)] = np.frombuffer(c, np.uint8)
            o += len(c)
        return buf, (o_seg, o_tab, o_dat), len(descs), len(segs), blk, max_blocks, max_pixels

    def _launch(self, buf, offs, n, nseg, blk, max_blocks, max_pixels):
        o_seg, o_tab, o_dat = offs
        dev = torch.empty(buf.numel(), dtype=torch.uint8, device=self.device)
        ws = torch.empty(blk * 192, dtype=torch.uint8, device=self.device)
        err = torch.empty(n, dtype=torch.uint8, device=self.device)
        self._err_host = torch.empty(n, dtype=torch.uint8, pin_memory=True)
        with torch.cuda.stream(self._stream):
            dev.copy_(buf, non_blocking=True)
            p = dev.data_ptr()
            lib.jpeg_decode(p, n, p + o_seg, nseg, p + o_tab, p + o_dat, blk, max_blocks, max_pixels, ws, ws.numel(),
                            self.src, err, self._stream.cuda_stream)
            self._err_host.copy_(err, non_blocking=True)
            self._err_event = torch.cuda.Event()
            self._err_event.record(self._stream)
        self.bytes_to_device += buf.numel()
        self._keep = [buf, dev, ws, err]

    def _submit(self, i):
        return self._pool.submit(_pillow, self._datas[i]) if self._pool is not None else _pillow(self._datas[i])

    def finish(self):
        if self._err_event is not None:
            self._err_event.synchronize()                      # n bytes: the only host wait on the decode
            self.device_failed = [self._dev_idx[k] for k in np.flatnonzero(self._err_host.numpy())]
            self.on_device = [i for i in self._dev_idx if i not in set(self.device_failed)]
            for i in self.device_failed:
                self._host[i] = self._submit(i)                 # truncated / corrupt data: the host path's result
        host = {i: (f.result() if hasattr(f, 'result') else f) for i, f in sorted(self._host.items())}
        if host:
            stage = torch.empty(int(sum(a.size for a in host.values())), dtype=torch.uint8, pin_memory=True)
            s = stage.numpy()
            o = 0
            with torch.cuda.stream(self._stream):              # after the kernels that wrote the failed slots
                for i, arr in host.items():
                    if arr.shape[:2] != tuple(self.hw[i]):
                        raise ValueError('image %d: decoded size %s differs from its header' % (i, arr.shape[:2]))
                    s[o:o + arr.size] = arr.reshape(-1)
                    self.src[self.offsets[i]:self.offsets[i] + arr.size].copy_(stage[o:o + arr.size], non_blocking=True)
                    o += arr.size
            self.bytes_to_device += stage.numel()
        ev = torch.cuda.Event()
        ev.record(self._stream)
        torch.cuda.current_stream(self.device).wait_event(ev)
        self._keep = []
        offset = torch.from_numpy(self.offsets).to(self.device)
        hw = torch.from_numpy(self.hw.astype(np.int32)).to(self.device)
        return self.src, offset, hw


def start_decode(datas, device, pool=None, fill=None):
    """Parse, pack and enqueue the device decode of a batch of encoded images; returns a `DecodeJob`.  `pool`
    (a concurrent.futures executor) decodes the unsupported images with Pillow in parallel; `fill` pre-fills the
    output with a byte value (tests: unwritten pixels show)."""
    return DecodeJob(datas, device, pool, fill)


def decode_batch(datas, device, stream=None, pool=None):
    """-> (src uint8 [sum H*W*3], src_offset int64 [n], src_hw int32 [n, 2]) on `device`: the packed HWC layout of
    `simclr_augment`, equal to Pillow's RGB decode of every image.  Work that reads the result is ordered after it
    on `stream` (default: the current stream)."""
    if stream is None:
        return start_decode(datas, device, pool).finish()
    with torch.cuda.stream(stream):
        return start_decode(datas, device, pool).finish()
