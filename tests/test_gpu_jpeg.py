"""GPU tests of the device JPEG decoder (simclr_b200/jpeg.py + csrc/jpeg.cu): bit-exact with Pillow on the corpus,
over more images than SMs, in mixed batches, back to back, with truncated entropy data, and through
`build_input_fn` / `run.main` against the host-decode pipeline."""
import io
import json
import os

import numpy as np
import pytest
import torch
from PIL import Image

import jpeg_corpus as JC

pytestmark = pytest.mark.gpu


def _host(d):
    """The host path's result for these bytes: the decoded array, or the exception it raises."""
    try:
        with Image.open(io.BytesIO(d)) as im:
            return np.array(im.convert('RGB'))
    except Exception as ex:            # noqa: BLE001  (compared by type)
        return ex


def _check(datas, fill, **kw):
    from simclr_b200 import jpeg as J
    job = J.start_decode(datas, 'cuda', fill=fill, **kw)
    src, off, hw = job.finish()
    torch.cuda.synchronize()
    src, off, hw = src.cpu().numpy(), off.cpu().numpy(), hw.cpu().numpy()
    assert len(off) == len(hw) == len(datas)
    for i, d in enumerate(datas):
        ref = _host(d)
        h, w = hw[i]
        got = src[off[i]:off[i] + h * w * 3].reshape(h, w, 3)
        assert got.shape == ref.shape and np.array_equal(got, ref), (i, fill)
    assert off[-1] + hw[-1, 0] * hw[-1, 1] * 3 == len(src)
    return job


def test_decode_batch_corpus_bit_exact():
    corpus = JC.corpus()
    datas = [d for _, d in corpus]
    for fill in (0x00, 0xFF):          # two sentinels: a pixel the kernels do not write fails one of them
        job = _check(datas, fill)
        assert sorted(job.on_device) == list(range(len(datas))) and job.device_failed == []


def test_decode_batch_more_images_than_sms_and_back_to_back():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rs = np.random.RandomState(3)
    datas = []
    for k in range(sms + 37):
        h, w = int(rs.randint(20, 140)), int(rs.randint(20, 140))
        kw = dict(quality=int(rs.choice([60, 85, 95])), subsampling=int(rs.choice([0, 1, 2])))
        if k % 7 == 3:
            kw['restart_marker_blocks'] = int(rs.randint(1, 5))
        a = JC.picture(h, w, k)
        datas.append(JC.jpeg(a[..., 0] if k % 11 == 5 else a, **kw))
    from simclr_b200 import jpeg as J
    a = J.decode_batch(datas, 'cuda')
    b = J.decode_batch(datas, 'cuda')
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    job = _check(datas, 0x5A)
    assert len(job.on_device) == len(datas)


def test_decode_batch_mixed_supported_unsupported_png():
    """Supported JPEGs interleaved with a progressive JPEG, a CMYK JPEG and PNGs (Pillow on a thread pool)."""
    import concurrent.futures
    from simclr_b200 import jpeg as J
    corpus = JC.corpus()
    others = [d for name, d in JC.unsupported() if name != 'sof9']           # (Pillow cannot decode SOF9 either)
    datas = []
    for k, d in enumerate(others):
        datas += [corpus[3 * k + 1][1], d]
    datas += [JC.png(JC.picture(13, 19, 1)), corpus[-1][1]]
    with concurrent.futures.ThreadPoolExecutor(4) as pool:
        job = _check(datas, 0xA5, pool=pool)
    assert job.on_device == [i for i, d in enumerate(datas) if J.parse(d) is not None] == [0, 2, 4, 7]


@pytest.mark.parametrize('with_eoi', [False, True])
def test_truncated_entropy_sets_error_flag(with_eoi):
    """The header is intact, the entropy-coded data stops early: the image's error flag comes back set and the
    batch holds the host path's result for it (or raises the host path's exception); its neighbours decode on the
    device as usual."""
    from simclr_b200 import jpeg as J
    good = JC.corpus()
    d = JC.jpeg(JC.picture(96, 120, 5), quality=92, subsampling=2)
    h = J.parse(d)
    cut = d[:h.scan_start + (h.scan_end - h.scan_start) // 3] + (b'\xff\xd9' if with_eoi else b'')
    datas = [good[2][1], cut, good[5][1]]
    ref = _host(cut)
    if isinstance(ref, Exception):
        job = J.start_decode(datas, 'cuda')
        with pytest.raises(type(ref)):
            job.finish()
    else:
        job = _check(datas, 0x00)
    assert job.device_failed == [1]


def _toy_tfds(root, n_train=40, n_val=20):
    """<root>/toy/1.0.0: JPEG shards (two of them hold a few PNGs and one progressive JPEG), ImageNet-like aspect."""
    from simclr_b200 import tfrecord as T
    d = os.path.join(root, 'toy', '1.0.0')
    os.makedirs(d)
    rs = np.random.RandomState(7)

    def enc(k):
        h, w = int(rs.randint(48, 120)), int(rs.randint(48, 120))
        a = JC.picture(h, w, 100 + k)
        if k % 13 == 4:
            return JC.png(a)
        if k % 17 == 9:
            return JC.jpeg(a, quality=80, progressive=True)
        return JC.jpeg(a, quality=int(rs.choice([80, 90, 95])), subsampling=int(rs.choice([0, 2, 2])))
    ex = [T.encode_example({'image': enc(k), 'label': k % 5}) for k in range(n_train + n_val)]
    T.write_records(os.path.join(d, 'toy-train.tfrecord-00000-of-00002'), ex[:n_train // 2])
    T.write_records(os.path.join(d, 'toy-train.tfrecord-00001-of-00002'), ex[n_train // 2:n_train])
    T.write_records(os.path.join(d, 'toy-validation.tfrecord-00000-of-00001'), ex[n_train:])
    json.dump({'featuresDict': {'features': {'label': {'classLabel': {'numClasses': '5'}}}}}, open(os.path.join(d, 'features.json'), 'w'))
    return root


def test_input_fn_device_decode_equals_host(flags, tmp_path):
    from simclr_b200 import data as D, engine
    root = _toy_tfds(str(tmp_path))
    engine.set_engine(engine.Engine(precision='bf16', conv_engine='tc'))
    for mode in ('pretrain', 'finetune', 'eval'):
        flags.set_flags(image_size=64, train_mode='pretrain' if mode == 'eval' else mode, train_split='train',
                        eval_split='validation', color_jitter_strength=1.0)
        out = {}
        for dec in ('host', 'device'):
            b = D.TFRecordBuilder(root, 'toy', decode=dec)
            it = D.build_input_fn(b, 16, None, mode != 'eval')(D.InputContext(1, 0, 1), seed=11)
            out[dec] = [next(it) for _ in range(2)]
        for (fh, lh), (fd, ld) in zip(out['host'], out['device']):
            assert fd.is_cuda and fh.shape == fd.shape and torch.equal(fh, fd), mode
            assert torch.equal(lh, ld), mode
        assert out['host'][0][0].shape[-1] == (6 if mode == 'pretrain' else 3)


def test_run_main_with_device_decode(flags, tmp_path):
    from simclr_b200 import run, engine
    root = _toy_tfds(str(tmp_path))
    saved = flags.FLAGS.b200_jpeg_decode
    try:
        flags.set_flags(resnet_depth=18, image_size=32, train_batch_size=8, eval_batch_size=8, train_steps=2,
                        mode='train', train_mode='pretrain', data_dir=root, dataset='toy', model_dir=str(tmp_path / 'm'),
                        b200_precision='bf16', b200_conv_engine='tc', b200_jpeg_decode='device', warmup_epochs=0,
                        checkpoint_steps=2)
        engine.set_engine(None)
        run.main(['run'])
        assert os.path.exists(os.path.join(str(tmp_path / 'm'), 'ckpt-2.npz'))
    finally:
        flags.set_flags(b200_jpeg_decode=saved)
