"""Host (Pillow) vs device (simclr_jpeg_decode) JPEG decode, and the TFRecord input pipeline with each.

No ImageNet here: a seeded corpus is encoded with Pillow at ImageNet-like sizes (each side drawn around 500 x 375,
clipped to [200, 800]), quality 85-95, 80 % 4:2:0 (the rest 4:2:2 / 4:4:4), content mixing smooth gradients, hard
edges and textured noise (about 100 KB per file).  Reports, with the GPU and CPU model:
  * Pillow decode img/s on 1, 8 and 32 threads;
  * device decode img/s at the batch size, host-to-device bytes per batch in each mode, and the device time of
    one batch (events around the decode stream's copy + kernels);
  * `build_input_fn` batches/s for pretraining at 224 with decode='host' and decode='device';
and prints one JSON line.  Writes only to a temporary directory.

    python scripts/jpeg_bench.py [--images 768] [--batch 256] [--steps 6]
"""
import argparse
import concurrent.futures
import io
import json
import os
import platform
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def natural(h, w, seed):
    rs = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    a = np.zeros((h, w, 3), np.float32)
    for c in range(3):
        fx, fy, ph = rs.uniform(0.005, 0.05), rs.uniform(0.005, 0.05), rs.uniform(0, 6)
        a[..., c] = 128 + 90 * np.sin(fx * xx + fy * yy + ph) * np.cos(0.3 * fy * xx - 0.7 * fx * yy)
    for _ in range(12):
        y0, x0, r = rs.randint(0, h), rs.randint(0, w), rs.randint(10, 80)
        a[(yy - y0) ** 2 + (xx - x0) ** 2 < r * r] = rs.uniform(0, 255, 3)
    a += rs.normal(0, 25, (h // 4 + 1, w // 4 + 1, 3)).repeat(4, 0).repeat(4, 1)[:h, :w] + rs.normal(0, 9, a.shape)
    return np.clip(a, 0, 255).astype(np.uint8)


def corpus(n, seed=0):
    from PIL import Image
    rs = np.random.RandomState(seed)
    out = []
    for k in range(n):
        h = int(np.clip(rs.normal(375, 60), 200, 800))
        w = int(np.clip(rs.normal(500, 80), 200, 800))
        ss = 2 if rs.rand() < 0.8 else int(rs.choice([0, 1]))
        b = io.BytesIO()
        Image.fromarray(natural(h, w, seed * 100003 + k)).save(b, format='JPEG', quality=int(rs.randint(85, 96)), subsampling=ss)
        out.append(b.getvalue())
    return out


def machine():
    import torch
    cpu = platform.processor() or platform.machine()
    try:
        out = subprocess.run(['lscpu'], capture_output=True, text=True, timeout=30).stdout
        cpu = next(l.split(':', 1)[1].strip() for l in out.splitlines() if l.startswith('Model name')) + ' (%s)' % platform.machine()
    except (OSError, subprocess.SubprocessError, StopIteration):
        pass
    gpu = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = 'unknown'
    return dict(gpu=gpu, gpu_power_limit=power, cpu=cpu, cpu_count=os.cpu_count())


def pillow_rate(datas, threads, passes=2):
    from simclr_b200.jpeg import _pillow
    with concurrent.futures.ThreadPoolExecutor(threads) as pool:
        list(pool.map(_pillow, datas[:threads * 2]))
        t = time.perf_counter()
        for _ in range(passes):
            list(pool.map(_pillow, datas))
        return passes * len(datas) / (time.perf_counter() - t)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--images', type=int, default=768)
    ap.add_argument('--batch', type=int, default=256)
    ap.add_argument('--steps', type=int, default=6, help='timed build_input_fn batches per mode')
    args = ap.parse_args()
    import torch
    from simclr_b200 import jpeg as J, data as D, engine, flags_def, tfrecord as T
    assert torch.cuda.is_available(), 'jpeg_bench measures the device decoder: it needs a GPU'
    torch.cuda.set_device(0)
    info = machine()
    t0 = time.perf_counter()
    datas = corpus(args.images)
    res = dict(info, images=len(datas), mean_bytes=float(np.mean([len(d) for d in datas])),
               corpus_seconds=round(time.perf_counter() - t0, 1))
    B = args.batch
    batches = [datas[i:i + B] for i in range(0, len(datas) - B + 1, B)]
    assert batches, '--images must be at least --batch'

    # Pillow on 1 / 8 / 32 threads
    for th in (1, 8, 32):
        res['pillow_img_s_%dthreads' % th] = round(pillow_rate(datas if th > 1 else datas[:64], th, 1 if th == 1 else 2), 1)

    # device decode: whole decode_batch (parse + pack + copy + kernels + wait) and the device span of one batch
    dev = torch.device('cuda', 0)
    for bt in batches:                                          # warm-up (module load, allocator, table cache)
        J.decode_batch(bt, dev)
    torch.cuda.synchronize()
    reps = max(1, 8 // len(batches))
    t = time.perf_counter()
    for _ in range(reps):
        for bt in batches:
            J.decode_batch(bt, dev)
    torch.cuda.synchronize()
    res['device_decode_img_s'] = round(reps * len(batches) * B / (time.perf_counter() - t), 1)
    side = J._side_stream(dev)
    spans = []
    for bt in batches:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record(side)
        job = J.start_decode(bt, dev)
        job.finish()
        e1.record(side)
        torch.cuda.synchronize()
        spans.append(e0.elapsed_time(e1))
        assert not job.device_failed and len(job.on_device) == len(bt)
    res['device_batch_ms'] = round(float(np.median(spans)), 3)
    res['h2d_bytes_per_batch_device'] = int(job.bytes_to_device)
    res['h2d_bytes_per_batch_host'] = int(sum(h * w * 3 for h, w in job.hw))
    # spot check: the device output equals Pillow on the first batch
    src, off, hw = J.decode_batch(batches[0], dev)
    src, off, hw = src.cpu().numpy(), off.cpu().numpy(), hw.cpu().numpy()
    res['bit_exact_first_batch'] = all(
        np.array_equal(src[off[i]:off[i] + hw[i, 0] * hw[i, 1] * 3].reshape(hw[i, 0], hw[i, 1], 3), J._pillow(d))
        for i, d in enumerate(batches[0]))

    # build_input_fn, pretraining at 224, one input pipeline, batch B
    flags_def.set_flags(image_size=224, train_mode='pretrain', train_split='train', color_jitter_strength=1.0)
    engine.set_engine(engine.Engine(precision='bf16', conv_engine='tc'))
    with tempfile.TemporaryDirectory() as tmp:
        d = os.path.join(tmp, 'bench', '1.0.0')
        os.makedirs(d)
        T.write_records(os.path.join(d, 'bench-train.tfrecord-00000-of-00001'),
                        [T.encode_example({'image': x, 'label': k % 1000}) for k, x in enumerate(datas)])
        for mode in ('host', 'device', 'host', 'device'):        # alternated: the second pair is reported
            b = D.TFRecordBuilder(tmp, 'bench', num_classes=1000, decode=mode)
            it = D.build_input_fn(b, B, None, True)(D.InputContext(1, 0, 1), seed=1)
            for _ in range(2):
                next(it)
            torch.cuda.synchronize()
            t = time.perf_counter()
            for _ in range(args.steps):
                f, _ = next(it)
            torch.cuda.synchronize()
            res['input_fn_batches_s_%s' % mode] = round(args.steps / (time.perf_counter() - t), 3)
            b._pool.shutdown()
    res['input_fn_img_s_host'] = round(res['input_fn_batches_s_host'] * B, 1)
    res['input_fn_img_s_device'] = round(res['input_fn_batches_s_device'] * B, 1)
    for k, v in res.items():
        print('%-32s %s' % (k, v))
    print(json.dumps(res))


if __name__ == '__main__':
    main()
