"""Input pipeline of the reference (`tf2/data.py:29-115`) over decoded images held in host memory.

`build_input_fn(builder, global_batch_size, topology, is_training)` keeps the reference's signature and
returns `_input_fn(input_context)`, an iterator factory yielding `(features, labels)` batches of the model's
input contract (`tf2/data.py:52-62`): pretraining -> two augmented views concatenated on channels
`[B,H,W,6]`, otherwise one view `[B,H,W,3]`, fp32 in [0,1] on the device, labels one-hot.  The per-image
map (`get_preprocess_fn` -> `data_util.preprocess_image`) runs as ONE augmentation kernel launch per view
over the whole batch (`simclr_augment`: crop + bicubic resize [+ flip + colour ops], draws on the host).

What stands in for `tfds.builder(...)` (`tf2/run.py:469-475`):
  * `TFRecordBuilder`: a prepared TFDS dataset directory -- `<name>-<split>.tfrecord-XXXXX-of-NNNNN` shards of
    `tf.train.Example{image: encoded bytes, label: int64}` plus `dataset_info.json` / `features.json` -- read with
    `tfrecord.py` (no TensorFlow); images are decoded on host threads with Pillow, everything after the decode
    (crop, resize, flip, colour) is the GPU kernel.  Input pipelines take whole shard files (`files[p::P]`), files
    are reshuffled every epoch when training;
  * `ArrayBuilder`: uint8 images + integer labels per split in host memory (e.g. an `.npz` under `--data_dir`).
Shuffling follows the reference's recipe -- a buffer of `batch_size * (50 if image_size <= 32 else 10)` elements
drawn uniformly, `repeat(-1)`, `drop_remainder` when training.
"""
import collections
import concurrent.futures
import functools
import io
import json
import os
import random
import re

import numpy as np
import torch
from absl import logging

from .flags_def import FLAGS
from . import data_util
from .engine import get_engine

InputContext = collections.namedtuple('InputContext', 'num_input_pipelines input_pipeline_id num_replicas_in_sync')


def _per_replica_batch_size(ctx, global_batch_size):
    if global_batch_size % ctx.num_replicas_in_sync:
        raise ValueError('global batch %d is not divisible by %d replicas' % (global_batch_size, ctx.num_replicas_in_sync))
    return global_batch_size // ctx.num_replicas_in_sync


class _Split:
    def __init__(self, images, labels):
        assert len(images) == len(labels)
        self.images, self.labels = images, np.asarray(labels, dtype=np.int64)
        self.num_examples = len(labels)


class _Info:
    def __init__(self, splits, num_classes):
        self.splits = splits
        self.features = {'label': collections.namedtuple('L', 'num_classes')(num_classes)}


class ArrayBuilder:
    """Stand-in for the `tfds.builder(...)` object `tf2/run.py:469-475` uses: `.info.splits[name].num_examples`,
    `.info.features['label'].num_classes`, and the decoded examples of a split."""

    def __init__(self, splits, num_classes):
        """splits: {name: (images, labels)}; images: list / object array of uint8 [Hs,Ws,3] arrays (any sizes)
        or one uint8 array [N,Hs,Ws,3]."""
        self.info = _Info({k: _Split(*v) for k, v in splits.items()}, num_classes)

    @classmethod
    def from_npz(cls, path):
        """`<split>_images`, `<split>_labels` arrays (+ optional scalar `num_classes`)."""
        z = np.load(path, allow_pickle=True)
        names = sorted(k[:-7] for k in z.files if k.endswith('_images'))
        splits = {n: (z[n + '_images'], z[n + '_labels']) for n in names}
        nc = int(z['num_classes']) if 'num_classes' in z.files else int(max(int(np.max(v[1])) for v in splits.values()) + 1)
        return cls(splits, nc)

    def download_and_prepare(self):
        pass

    def examples(self, split):
        return self.info.splits[split]

    # -- token stream (what the shuffle buffer holds) / fetch (what `map_fn` decodes) ---------------------------
    def tokens(self, split, input_context, shuffle_files, rng):
        """One pass over this pipeline's contiguous shard of the split: example indices."""
        del shuffle_files, rng
        n = self.info.splits[split].num_examples
        P, p = input_context.num_input_pipelines, input_context.input_pipeline_id
        return iter(range(n * p // P, n * (p + 1) // P))

    def fetch(self, split, token):
        sp = self.info.splits[split]
        return np.ascontiguousarray(sp.images[token]), int(sp.labels[token])


_SHARD_RE = re.compile(r'^(?P<ds>.+)-(?P<split>[A-Za-z0-9_]+)\.tfrecord(-(?P<i>\d+)-of-(?P<n>\d+))?$')


class TFRecordBuilder:
    """A prepared TFDS dataset on disk, read without TensorFlow (module docstring).  `data_dir` may be the TFDS root
    (`<data_dir>/<name>/[<config>/]<version>/`), or the version directory itself."""

    IMAGE_KEY, LABEL_KEY = 'image', 'label'

    def __init__(self, data_dir, name=None, num_classes=None, decode_threads=None, decode=None):
        """decode: 'host' (Pillow on `decode_threads` threads) or 'device' (`jpeg.decode_batch`: JPEGs the sm_90a
        decoder supports on the GPU, bit-exact with 'host', the rest with Pillow); default --b200_jpeg_decode."""
        from . import tfrecord
        self._tf = tfrecord
        self.decode = decode or FLAGS['b200_jpeg_decode'].value
        if self.decode not in ('host', 'device'):
            raise ValueError("decode must be 'host' or 'device', got %r" % (self.decode,))
        root = os.path.join(data_dir, name) if name and os.path.isdir(os.path.join(data_dir, name)) else data_dir
        files = collections.defaultdict(list)
        self.dir = None
        for d, _, fs in sorted(os.walk(root)):
            for f in sorted(fs):
                m = _SHARD_RE.match(f)
                if m and (name is None or m.group('ds') == name):
                    if self.dir is None:
                        self.dir = d
                    if d == self.dir:               # one version directory only (the first in sorted order)
                        files[m.group('split')].append(os.path.join(d, f))
        if not files:
            raise FileNotFoundError('no <name>-<split>.tfrecord* files under %s' % root)
        self.files = dict(files)
        counts = self._counts_from_info()
        splits = {}
        for sp, fl in self.files.items():
            n = counts.get(sp)
            if n is None:
                n = sum(tfrecord.count_records(f) for f in fl)
            splits[sp] = collections.namedtuple('S', 'num_examples')(n)
        nc = num_classes if num_classes is not None else self._num_classes_from_info()
        if nc is None:
            raise ValueError('number of classes not found in %s (features.json / label.labels.txt): pass num_classes' % self.dir)
        self.info = _Info(splits, nc)
        self._pool = concurrent.futures.ThreadPoolExecutor(decode_threads or min(32, (os.cpu_count() or 4)))

    def _counts_from_info(self):
        path = os.path.join(self.dir, 'dataset_info.json')
        out = {}
        if os.path.exists(path):
            try:
                for sp in json.load(open(path)).get('splits', []):
                    if 'shardLengths' in sp:
                        out[sp['name']] = sum(int(x) for x in sp['shardLengths'])
                    elif 'numExamples' in sp:
                        out[sp['name']] = int(sp['numExamples'])
            except (ValueError, KeyError, TypeError):
                pass
        return out

    def _num_classes_from_info(self):
        fj = os.path.join(self.dir, 'features.json')
        if os.path.exists(fj):
            try:
                feats = json.load(open(fj))
                lab = (feats.get('featuresDict', {}).get('features', {}) or feats.get('features', {})).get(self.LABEL_KEY, {})
                cl = lab.get('classLabel', lab)
                if 'numClasses' in cl:
                    return int(cl['numClasses'])
            except (ValueError, AttributeError):
                pass
        for cand in (self.LABEL_KEY + '.labels.txt', 'labels.txt'):
            lt = os.path.join(self.dir, cand)
            if os.path.exists(lt):
                return sum(1 for line in open(lt) if line.strip())
        return None

    def download_and_prepare(self):
        pass            # the directory IS the prepared dataset

    def tokens(self, split, input_context, shuffle_files, rng):
        """One pass over this pipeline's files: (encoded image bytes, label).  With fewer files than pipelines every
        pipeline reads all files and keeps records i % P == p."""
        files = list(self.files[split])
        P, p = input_context.num_input_pipelines, input_context.input_pipeline_id
        by_file = len(files) >= P
        if by_file:
            files = files[p::P]
        if shuffle_files:
            rng.shuffle(files)
        i = 0
        for f in files:
            for rec in self._tf.read_records(f):
                if by_file or i % P == p:
                    ex = self._tf.parse_example(rec)
                    yield ex[self.IMAGE_KEY][0], int(ex[self.LABEL_KEY][0])
                i += 1

    def fetch(self, split, token):
        from PIL import Image
        del split
        data, label = token
        with Image.open(io.BytesIO(data)) as im:
            return np.array(im.convert('RGB'), dtype=np.uint8), label

    def fetch_many(self, split, tokens):
        """Parallel decode (Pillow releases the GIL): the `num_parallel_calls=AUTOTUNE` of the reference's map."""
        return list(self._pool.map(lambda t: self.fetch(split, t), tokens))

    def fetch_device(self, split, tokens, device):
        """-> (jpeg.DecodeJob, labels): the batch's decode enqueued on the device (image sizes in `job.hw` at once,
        pixels from `job.finish()`); images the device decoder does not take go to Pillow on this builder's pool."""
        from . import jpeg
        del split
        return jpeg.start_decode([t[0] for t in tokens], device, self._pool), [t[1] for t in tokens]


def get_preprocess_fn(is_training, is_pretrain):
    """Get function that accepts an image and returns a preprocessed image (tf2/data.py:101-115)."""
    # Disable test cropping for small images (e.g. CIFAR)
    test_crop = not (FLAGS.image_size <= 32)
    color_jitter_strength = FLAGS.color_jitter_strength if is_pretrain else 0.
    return functools.partial(data_util.preprocess_image, height=FLAGS.image_size, width=FLAGS.image_size,
                             is_training=is_training, color_jitter_strength=color_jitter_strength, test_crop=test_crop)


def build_input_fn(builder, global_batch_size, topology, is_training):
    """tf2/data.py:29-92.  `topology` is accepted for signature parity (TPU only)."""
    del topology

    def _input_fn(input_context, seed=0, make_batch=None):
        batch_size = _per_replica_batch_size(input_context, global_batch_size)
        logging.info('Global batch size: %d', global_batch_size)
        logging.info('Per-replica batch size: %d', batch_size)
        num_classes = builder.info.features['label'].num_classes
        split_name = FLAGS.train_split if is_training else FLAGS.eval_split
        P, p = input_context.num_input_pipelines, input_context.input_pipeline_id
        logging.info('num_input_pipelines: %d', P)
        pretrain = is_training and FLAGS.train_mode == 'pretrain'
        H = FLAGS.image_size
        jitter = FLAGS.color_jitter_strength if pretrain else 0.
        test_crop = not (FLAGS.image_size <= 32)
        rng = random.Random(seed * 1000003 + p)

        def order():
            """dataset.shuffle(batch * buffer_multiplier).repeat(-1) when training; one ordered pass otherwise."""
            if not is_training:
                yield from builder.tokens(split_name, input_context, False, rng)
                return
            buffer_size = batch_size * (50 if FLAGS.image_size <= 32 else 10)
            buf = []
            while True:
                n_seen = 0
                for tok in builder.tokens(split_name, input_context, True, rng):
                    n_seen += 1
                    buf.append(tok)
                    if len(buf) >= buffer_size:
                        yield buf.pop(rng.randrange(len(buf)))
                if n_seen == 0:
                    raise ValueError('split %r has no examples for input pipeline %d of %d' % (split_name, p, P))
                # (repeat: the buffer keeps its remainder across epochs, as tf.data does)

        def batches():
            e = get_engine() if make_batch is None else None
            idx = []
            for i in order():
                idx.append(i)
                if len(idx) == batch_size:
                    yield (make_batch or make)(e, idx)
                    idx = []
            if idx and not is_training:            # drop_remainder=is_training
                yield (make_batch or make)(e, idx)

        def make(e, idx):
            if getattr(builder, 'decode', 'host') == 'device':
                return make_packed(e, idx)
            fetched = (builder.fetch_many(split_name, idx) if hasattr(builder, 'fetch_many')
                       else [builder.fetch(split_name, t) for t in idx])
            images = [torch.from_numpy(im) for im, _ in fetched]
            labels = torch.tensor([l for _, l in fetched], dtype=torch.int64)
            n = len(idx)
            if pretrain:
                feats = torch.empty((n, H, H, 6), dtype=torch.float32, device=e.device)
                for v in range(2):                       # two transformations (tf2/data.py:55-58)
                    draws = [data_util.draw_train_augmentation(im.shape[0], im.shape[1], jitter, rng) for im in images]
                    if jitter <= 0:
                        draws = [dict(d, color=dict(d['color'], apply_jitter=False, apply_gray=False)) for d in draws]
                    data_util.preprocess_for_train_batch(images, draws, H, H, out=feats, channel_offset=3 * v)
            elif is_training:
                draws = [data_util.draw_train_augmentation(im.shape[0], im.shape[1], 0., rng) for im in images]
                draws = [dict(d, color=dict(d['color'], apply_jitter=False, apply_gray=False)) for d in draws]
                feats = data_util.preprocess_for_train_batch(images, draws, H, H)
            else:
                feats = data_util.preprocess_for_eval_batch(images, H, H, crop=test_crop)
            lab = torch.nn.functional.one_hot(labels, num_classes).float().to(e.device)
            return feats, lab

        def make_packed(e, idx):
            """`make` with the decode on the device: the same draws, in the same order, from the header sizes while
            the decode runs; the augmentation reads the decoder's packed output."""
            job, labels = builder.fetch_device(split_name, idx, e.device)
            hw = [(int(h), int(w)) for h, w in job.hw]
            n = len(idx)
            if is_training:
                view_draws = []
                for _ in range(2 if pretrain else 1):
                    draws = [data_util.draw_train_augmentation(h, w, jitter, rng) for h, w in hw]
                    if jitter <= 0:
                        draws = [dict(d, color=dict(d['color'], apply_jitter=False, apply_gray=False)) for d in draws]
                    view_draws.append(draws)
            src, offs, src_hw = job.finish()
            if pretrain:
                feats = torch.empty((n, H, H, 6), dtype=torch.float32, device=e.device)
                for v, draws in enumerate(view_draws):
                    data_util.preprocess_for_train_packed(src, offs, job.hw, draws, H, H, out=feats, channel_offset=3 * v)
            elif is_training:
                feats = data_util.preprocess_for_train_packed(src, offs, job.hw, view_draws[0], H, H)
            else:
                feats = data_util.preprocess_for_eval_packed(src, offs, job.hw, H, H, crop=test_crop)
            lab = torch.nn.functional.one_hot(torch.tensor(labels, dtype=torch.int64), num_classes).float().to(e.device)
            return feats, lab

        return batches()

    return _input_fn


def build_distributed_dataset(builder, batch_size, is_training, strategy, topology):
    """tf2/data.py:95-98: one input pipeline per replica (process)."""
    input_fn = build_input_fn(builder, batch_size, topology, is_training)
    R = strategy.num_replicas_in_sync
    return input_fn(InputContext(R, strategy.replica_id, R))
