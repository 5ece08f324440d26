"""CPU tests of the JPEG decoder's specification and host half: the oracle (oracle/jpeg.py) equals Pillow bit for bit
on a corpus covering every supported case, and the header parser (simclr_b200/jpeg.py) agrees with Pillow on
geometry, sends everything outside the device subset to the host path, and never raises."""
import io

import numpy as np
import pytest
from PIL import Image

import jpeg_corpus as JC

CORPUS = JC.corpus()


def _pillow(d):
    with Image.open(io.BytesIO(d)) as im:
        return np.array(im.convert('RGB'))


@pytest.mark.parametrize('name,data', CORPUS, ids=[c[0] for c in CORPUS])
def test_oracle_equals_pillow(name, data):
    from oracle import jpeg as OJ
    ref = _pillow(data)
    got = OJ.decode(data)
    assert got.shape == ref.shape and got.dtype == np.uint8
    assert np.array_equal(got, ref), (name, int(np.abs(got.astype(int) - ref).max()))


def test_corpus_covers_the_subset():
    from simclr_b200 import jpeg as J
    hs = {n: J.parse(d) for n, d in CORPUS}
    assert all(h is not None for h in hs.values()), [n for n, h in hs.items() if h is None]
    sampling = {(h.mode, h.comps[0][1], h.comps[0][2]) for h in hs.values()}
    assert {('RGB', 1, 1), ('RGB', 2, 1), ('RGB', 2, 2), ('RGB', 1, 2), ('L', 1, 1)} <= sampling
    assert hs['restart_blocks'].restart_interval == 3 and hs['restart_rows'].restart_interval > 0
    assert hs['q100'].q[0] == np.ones(64, np.uint16).tobytes()
    assert hs['optimize'].ac[0] != hs['q50'].ac[0]                     # image-specific tables


@pytest.mark.parametrize('name,data', CORPUS, ids=[c[0] for c in CORPUS])
def test_parser_geometry_equals_pillow(name, data):
    from simclr_b200 import jpeg as J
    h = J.parse(data)
    with Image.open(io.BytesIO(data)) as im:
        assert (h.width, h.height) == im.size and h.mode == im.mode
    assert 0 < h.scan_start < h.scan_end <= len(data)


@pytest.mark.parametrize('name,data', JC.unsupported(), ids=[c[0] for c in JC.unsupported()])
def test_parser_rejects_outside_the_subset(name, data):
    from simclr_b200 import jpeg as J
    assert J.parse(data) is None
    if name != 'sof9':
        _pillow(data)                                   # the host path still decodes these


def test_parser_rejects_truncated_and_malformed_headers():
    from simclr_b200 import jpeg as J
    for name, data in CORPUS[:6] + [c for c in CORPUS if c[0] in ('app_heavy', 'restart_rows', 'gray_33x47')]:
        offs, sos_end = JC.marker_offsets(data)
        assert J.parse(data).scan_start == sos_end
        for o in offs:
            for cut in (o, o + 1, o + 2, o + 3, o + 5):
                if cut < sos_end:
                    assert J.parse(data[:cut]) is None, (name, cut)
    d = CORPUS[0][1]
    assert J.parse(b'') is None and J.parse(b'\xff\xd8') is None and J.parse(b'\x00' * 100) is None
    s = JC.sof_offset(d)
    for patch in ({s + 4: 12}, {s + 5: 0, s + 6: 0}, {s + 9: 4}, {s + 11: 0x31}, {s + 14: 0x22}, {s + 12: 7}):
        bad = bytearray(d)
        for k, v in patch.items():
            bad[k] = v
        assert J.parse(bytes(bad)) is None, patch             # 12-bit, zero height, 4 components, bad sampling, ...
    i = d.index(b'\xff\xc4')                                   # an over-subscribed DHT: 3 codes of length 1
    bad = bytearray(d)
    bad[i + 5] = 3
    assert J.parse(bytes(bad)) is None


def test_restart_segments():
    """One segment per restart interval, each ending on its RSTn marker; MCU ranges cover the scan once."""
    from simclr_b200 import jpeg as J
    for name in ('restart_blocks', 'restart_rows', 'restart_gray'):
        data = dict(CORPUS)[name]
        h = J.parse(data)
        mx, my, _, _, _ = J._geometry(h)
        segs = J._segments(data, h, mx * my)
        assert len(segs) == -(-mx * my // h.restart_interval) > 1
        assert sum(s[3] for s in segs) == mx * my and [s[2] for s in segs] == [k * h.restart_interval for k in range(len(segs))]
        for k, (s, e, _, _) in enumerate(segs[:-1]):
            assert data[e] == 0xFF and data[e + 1] == 0xD0 + (k & 7) and segs[k + 1][0] == e + 2


def test_huffman_tables_decode_like_the_oracle():
    """The lookahead / maxcode tables the kernel reads give the oracle's symbol for every code of every table."""
    from simclr_b200 import jpeg as J
    from oracle import jpeg as OJ
    h = J.parse(dict(CORPUS)['optimize'])
    for counts, vals in h.dc + h.ac:
        t = np.frombuffer(J._huffman_table(counts, vals), np.uint8)
        look, maxcode, valoff = t[:1024].view(np.uint16), t[1024:1096].view(np.int32), t[1096:1168].view(np.int32)
        tv = t[1168:]
        maxc, voff, _ = OJ._huff_table(list(counts), list(vals))
        code = 0
        k = 0
        for l in range(1, 17):
            for _ in range(counts[l - 1]):
                want = vals[k]
                pk = code << (16 - l)
                e = look[pk >> 7]
                if l <= 9:
                    assert e == (l << 8) | want
                else:
                    assert e == 0 and maxcode[l] == maxc[l] and tv[code + valoff[l]] == want
                code += 1
                k += 1
            code <<= 1


def test_jpeg_decode_flag(flags):
    F = flags.FLAGS
    assert F['b200_jpeg_decode'].default == 'host' and F.b200_jpeg_decode == 'host'
    with pytest.raises(Exception):
        F['b200_jpeg_decode'].parse('nvjpeg')
    from simclr_b200 import data as D
    with pytest.raises(FileNotFoundError):
        D.TFRecordBuilder('/nonexistent-dir-for-test', 'toy')
