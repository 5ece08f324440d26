"""Seeded JPEG corpus for the decoder tests (tests/test_jpeg.py, tests/test_gpu_jpeg.py), encoded with Pillow."""
import io

import numpy as np
from PIL import Image


def picture(h, w, seed):
    """Gradients, hard edges and noise: every AC band and long Huffman codes get exercised."""
    rs = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    a = np.stack([(3 * yy + 5 * xx) % 256, (200 - 2 * yy + xx) % 256, (7 * xx * yy // (w + 1)) % 256], -1).astype(np.int64)
    a += rs.randint(-40, 40, a.shape)
    a[(yy // 5 + xx // 7) % 3 == 0] = 255
    return np.clip(a, 0, 255).astype(np.uint8)


def jpeg(a, **kw):
    b = io.BytesIO()
    Image.fromarray(a).save(b, format='JPEG', **kw)
    return b.getvalue()


def png(a):
    b = io.BytesIO()
    Image.fromarray(a).save(b, format='PNG')
    return b.getvalue()


def sof_offset(data):
    """Byte offset of the SOF0 marker."""
    i = 2
    while data[i + 1] != 0xC0:
        i += 2 + ((data[i + 2] << 8) | data[i + 3])
    return i


def as_440(h, w, seed):
    """4:4:0 (luma 1x2): Pillow cannot write it, so a 4:2:2 file of W x H is relabelled as (W/2) x (2H) with luma
    sampling 1x2.  Both have the same MCU count and four blocks per MCU, so the entropy data decodes completely."""
    assert w % 16 == 0 and h % 8 == 0
    d = bytearray(jpeg(picture(h, w, seed), quality=90, subsampling=1))
    s = sof_offset(d)
    d[s + 5:s + 7] = (2 * h).to_bytes(2, 'big')
    d[s + 7:s + 9] = (w // 2).to_bytes(2, 'big')
    assert d[s + 11] == 0x21
    d[s + 11] = 0x12
    return bytes(d)


def corpus():
    """[(name, bytes)]: every case the device decoder supports."""
    out = []
    k = 0
    for h, w in [(1, 1), (7, 9), (8, 8), (15, 17), (16, 16), (33, 47), (150, 200)]:
        for ss, tag in [(0, '444'), (1, '422'), (2, '420')]:
            out.append(('%s_%dx%d' % (tag, h, w), jpeg(picture(h, w, k), quality=90, subsampling=ss)))
            k += 1
        out.append(('gray_%dx%d' % (h, w), jpeg(picture(h, w, k)[..., 0], quality=90)))
        k += 1
    for q in (50, 75, 95, 100):
        out.append(('q%d' % q, jpeg(picture(40, 52, k), quality=q, subsampling=2)))
        k += 1
    out.append(('optimize', jpeg(picture(40, 52, k), quality=85, optimize=True)))
    out.append(('restart_blocks', jpeg(picture(41, 53, k + 1), quality=85, restart_marker_blocks=3)))
    out.append(('restart_rows', jpeg(picture(41, 53, k + 2), quality=85, subsampling=0, restart_marker_rows=1)))
    out.append(('restart_gray', jpeg(picture(30, 30, k + 3)[..., 1], quality=85, restart_marker_blocks=2)))
    exif = Image.Exif()
    exif[0x0112] = 6                      # orientation: Pillow does not apply it on open
    exif[0x010F] = 'maker ' * 200
    out.append(('app_heavy', jpeg(picture(37, 29, k + 4), quality=88, exif=exif.tobytes(), icc_profile=b'\0' * 3000,
                                  comment=b'c' * 500)))
    out.append(('440_32x96', as_440(48, 64, k + 5)))
    out.append(('440_8x16', as_440(8, 16, k + 6)))
    return out


def unsupported():
    """[(name, bytes)] the parser must send to the host path (Pillow decodes them)."""
    a = picture(24, 40, 99)
    out = [('progressive', jpeg(a, quality=80, progressive=True)),
           ('cmyk', _cmyk(a)),
           ('png', png(a))]
    d = bytearray(jpeg(a, quality=80))
    d[sof_offset(d) + 1] = 0xC9                                    # SOF9: arithmetic coding
    out.append(('sof9', bytes(d)))
    return out


def _cmyk(a):
    b = io.BytesIO()
    Image.frombytes('CMYK', (a.shape[1], a.shape[0]), np.concatenate([a, a[..., :1]], -1).tobytes()).save(b, format='JPEG')
    return b.getvalue()


def marker_offsets(data):
    """Offsets of every marker up to and including SOS."""
    offs, i = [0], 2
    while True:
        offs.append(i)
        m = data[i + 1]
        i += 2 + ((data[i + 2] << 8) | data[i + 3])
        if m == 0xDA:
            return offs, i
