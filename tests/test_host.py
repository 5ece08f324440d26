"""CPU tests of the host side: the C-ABI library loads and exports every symbol
the header declares, the flag surface equals the reference's, the variable
inventory equals the oracle's, and the multi-replica plumbing (gloo, 2 ranks)."""
import math
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    from simclr_b200 import _lib
    decls = _lib.parse_header()
    assert len(decls) >= 30
    _lib.lib.load()                 # getattr on every declared symbol: raises if one is missing
    assert _lib.lib.version() >= 100
    import ctypes
    dll = ctypes.CDLL(_lib.LIB_PATH)
    for name in decls:
        assert hasattr(dll, name), name


def test_argument_errors_are_reported_without_a_gpu():
    from simclr_b200._lib import lib, SimclrError
    with pytest.raises(SimclrError) as ei:
        lib.ntxent_normalize(None, 4, 8, 1, None, None, None)
    assert 'null pointer' in str(ei.value)
    with pytest.raises(SimclrError):
        lib.conv2d_fprop_tc(1, 1, 1, 1, 1, 1, 8, 8, 8, 8, 2, 2, 1, None, None)     # even kernel size


def test_flag_surface(flags):
    F = flags.FLAGS
    assert len(flags.REFERENCE_FLAG_NAMES) == 48
    expected = dict(learning_rate=0.3, learning_rate_scaling='linear', warmup_epochs=10, weight_decay=1e-6,
                    batch_norm_decay=0.9, train_batch_size=512, train_epochs=100, train_steps=0,
                    optimizer='lars', momentum=0.9, temperature=0.1, hidden_norm=True, proj_head_mode='nonlinear',
                    proj_out_dim=128, num_proj_layers=3, ft_proj_selector=0, global_bn=True, width_multiplier=1,
                    resnet_depth=50, sk_ratio=0., se_ratio=0., image_size=224, color_jitter_strength=1.0,
                    use_blur=True, use_tpu=True, lineareval_while_pretraining=True, fine_tune_after_block=-1,
                    mode='train', train_mode='pretrain', dataset='imagenet2012', eval_batch_size=256)
    for k in flags.REFERENCE_FLAG_NAMES:
        assert k in F, k
    fresh = {k: F[k].default for k in expected}
    assert fresh == expected
    with pytest.raises(Exception):
        F['learning_rate_scaling'].parse('cubic')        # enum is enforced like in the reference


def test_flag_names_match_reference_source():
    """The flag names, in order, equal those the reference's tf2/run.py defines (tests/golden/reference_flag_names.json:
    its `flags.DEFINE_*('<name>'` calls)."""
    import json
    from simclr_b200 import flags_def
    names = json.load(open(os.path.join(os.path.dirname(__file__), 'golden', 'reference_flag_names.json')))
    assert names == flags_def.REFERENCE_FLAG_NAMES


@pytest.mark.parametrize('kw', [dict(resnet_depth=18, image_size=64), dict(resnet_depth=50), dict(resnet_depth=50, width_multiplier=2),
                                dict(resnet_depth=34, image_size=32, global_bn=False),
                                dict(resnet_depth=50, sk_ratio=0.0625, image_size=64), dict(resnet_depth=152, width_multiplier=2, sk_ratio=0.0625),
                                dict(resnet_depth=18, se_ratio=0.0625, image_size=64), dict(resnet_depth=50, se_ratio=0.25, sk_ratio=0.0625)])
def test_variable_inventory_matches_oracle(flags, kw):
    from simclr_b200 import resnet, model, engine
    from oracle import model as OM
    from util import cfg_from_flags
    flags.set_flags(**kw)
    vs = engine.VarStore()
    net = resnet.resnet(flags.FLAGS.resnet_depth, flags.FLAGS.width_multiplier, cifar_stem=flags.FLAGS.image_size <= 32, vs=vs)
    model.ProjectionHead(vs, net.cout)
    model.SupervisedHead(1000, vs, net.cout)
    om = OM.Model(cfg_from_flags(flags.FLAGS), 1000)
    assert [(v.name, v.shape, v.init) for v in vs.trainable] == [(k, s, i) for k, (s, i) in om.vs.trainable.items()]
    assert [(v.name, v.shape) for v in vs.moving] == [(k, s) for k, (s, i) in om.vs.moving.items()]


def test_lr_schedule_matches_oracle(flags):
    from simclr_b200 import model
    from oracle import model as OM
    from util import cfg_from_flags
    flags.set_flags(train_batch_size=4096, warmup_epochs=10, train_epochs=100)
    sched = model.WarmUpAndCosineDecay(0.3, 1281167)
    cfg = cfg_from_flags(flags.FLAGS)
    for step in [0, 1, 100, 3127, 3128, 20000, 31279, 40000]:
        assert sched(step) == OM.warmup_and_cosine_decay(cfg, 0.3, 1281167, step)
    assert model.get_train_steps(1281167) == 1281167 * 100 // 4096 + 1


def test_lars_name_filters(flags):
    from simclr_b200 import lars_optimizer
    opt = lars_optimizer.LARSOptimizer(0.1, weight_decay=1e-4,
                                       exclude_from_weight_decay=['batch_normalization', 'bias', 'head_supervised'])
    assert opt._use_weight_decay('resnet/conv2d/kernel:0') and opt._do_layer_adaptation('resnet/conv2d/kernel:0')
    for n in ['resnet/batch_norm_relu/sync_batch_normalization/gamma:0', 'head_supervised/linear_layer/dense_3/kernel:0',
              'head_supervised/linear_layer/dense_3/bias:0']:
        assert not opt._use_weight_decay(n) and not opt._do_layer_adaptation(n)
    with pytest.raises(NotImplementedError):
        lars_optimizer.LARSOptimizer(0.1, use_nesterov=True)


def test_model_errors(flags):
    from simclr_b200 import resnet, engine
    with pytest.raises(ValueError):
        resnet.resnet(51, 1)


# ---- multi-replica plumbing over gloo (2 ranks on CPU) ------------------------
def _worker(rank, world, port, out):
    import torch.distributed as dist
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    sys.path.insert(0, ROOT)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    from simclr_b200.engine import ReplicaContext
    from oracle import objective as O
    ctx = ReplicaContext()
    assert ctx.num_replicas_in_sync == world and ctx.replica_id == rank
    B, D = 6, 16
    g = torch.Generator().manual_seed(100)
    hs = [torch.randn(2 * B, D, generator=g, dtype=torch.float64) for _ in range(world)]
    z = O.l2_normalize(hs[rank])
    z_all = ctx.all_gather(z)                                   # [R][2B][D] rank-major
    assert z_all.shape == (world, 2 * B, D)
    for r in range(world):
        assert torch.equal(z_all[r], O.l2_normalize(hs[r]))
    # sharded loss from the gathered tensor == the oracle's replica simulation
    h1 = z_all[:, :B].reshape(world * B, D); h2 = z_all[:, B:].reshape(world * B, D)
    st = O.SimStrategy(world, rank, list(z_all[:, :B]), list(z_all[:, B:]))
    loss, _, labels = O.add_contrastive_loss(z, False, 0.1, st)
    ref = O.contrastive_loss_replicas(hs, True, 0.1)[rank]
    assert abs(loss.item() - ref[0].item()) < 1e-12
    assert torch.equal(labels, ref[2])
    t = torch.full((4,), float(rank + 1), dtype=torch.float64)
    ctx.all_reduce_sum(t)
    assert torch.equal(t, torch.full((4,), float(sum(range(1, world + 1))), dtype=torch.float64))
    dist.barrier()
    dist.destroy_process_group()
    out.put((rank, 'ok'))


def test_peer_comm_layout():
    """comm.layout at W = 2..64: the bn slots, gather regions and flag words are disjoint and inside `total`; data
    regions start on 16-byte boundaries (the kernels copy 16-byte vectors) and flag words on 8-byte ones."""
    from simclr_b200 import comm
    for W in range(2, 65):
        L = comm.layout(W)
        regions = [('bn %d/%d' % (k, q), L.bn_off + (k * W + q) * comm.SLOT_BYTES, comm.SLOT_BYTES, 16)
                   for k in range(comm.NSLOT) for q in range(W)]
        regions += [('flag bn %d/%d' % (k, q), L.bn_flag_off + (k * W + q) * 8, 8, 8)
                    for k in range(comm.NSLOT) for q in range(W)]
        for ch, cap in comm.GATHER_CHANNELS.items():
            regions += [('%s %d' % (ch, q), L.gather_off[ch] + q * cap, cap, 16) for q in range(W)]
            regions += [('flag %s %d' % (ch, q), L.gather_flag_off[ch] + q * 8, 8, 8) for q in range(W)]
        regions.sort(key=lambda t: t[1])
        assert regions[0][1] >= 0 and regions[-1][1] + regions[-1][2] <= L.total, W
        assert L.total % 4096 == 0, W
        for (n0, o0, s0, _), (n1, o1, _, _) in zip(regions, regions[1:]):
            assert o0 + s0 <= o1, (W, n0, n1)
        for name, off, _, align in regions:
            assert off % align == 0, (W, name)


def test_gather_fit_rule():
    """The peer channels carry 16-byte multiples up to their capacity; the rest goes through NCCL (an odd
    per-replica batch makes the [2B] fp32 lse 8B bytes)."""
    from simclr_b200 import comm
    assert comm.gather_fits('lse', 2 * 16 * 4) and not comm.gather_fits('lse', 2 * 3 * 4)
    assert not comm.gather_fits('lse', 2 * 25 * 4) and comm.gather_fits('lse', 256 << 10)
    assert comm.gather_fits('z', 2 * 4096 * 128 * 4) and not comm.gather_fits('z', 2 * 4097 * 128 * 4)
    assert not comm.gather_fits('z', 0) and not comm.gather_fits('z', 8)


def test_replica_context_gloo_world2():
    import torch.multiprocessing as mp
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = 29500 + os.getpid() % 2000
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(120)
        assert p.exitcode == 0
    got = sorted(q.get(timeout=5) for _ in range(2))
    assert got == [(0, 'ok'), (1, 'ok')]


def test_augmentation_draws_follow_the_reference_ranges():
    """`draw_train_augmentation` reproduces the distributions of tf2/data_util.py:53-75,246-320,382-390."""
    import random
    from simclr_b200 import data_util
    rng = random.Random(1)
    n_flip = n_jit = n_gray = 0
    for _ in range(400):
        d = data_util.draw_train_augmentation(240, 320, 1.0, rng)
        y, x, h, w = d['box']
        assert 0 <= y and 0 <= x and y + h <= 240 and x + w <= 320
        assert h * w >= 0.1 * 240 * 320 - 1e-9                      # min_object_covered (A9)
        assert 0.70 <= w / h <= 1.40                                  # aspect in [3/4, 4/3] up to rounding
        c = d['color']
        assert sorted(c['perm']) == [0, 1, 2, 3]
        assert 0.2 <= c['brightness'] <= 1.8 and 0.2 <= c['contrast'] <= 1.8 and 0.2 <= c['saturation'] <= 1.8
        assert -0.2 <= c['hue'] <= 0.2
        n_flip += d['flip']; n_jit += c['apply_jitter']; n_gray += c['apply_gray']
    assert 150 < n_flip < 250 and 280 < n_jit < 360 and 40 < n_gray < 120


def test_bench_reference_arm_prints_one_json_line():
    """bench.py contract (CPU arm): exactly one JSON line on stdout, with the reference-arm keys, even when a
    library writes to fd 1 behind Python's back."""
    import json, subprocess, sys, os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, os.path.join(root, 'bench.py'), '--impl', 'reference', '--steps', '1', '--warmup', '1',
                        '--cpu_batch', '2', '--image_size', '32', '--resnet_depth', '18'],
                       capture_output=True, text=True, timeout=600, env=dict(os.environ, OMP_NUM_THREADS='4'))
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, r.stdout
    d = json.loads(lines[0])
    assert d['impl'] == 'reference' and d['metric'] == 'images/sec pretrain step' and d['unit'] == 'images/s'
    assert d['higher_is_better'] is True and d['value'] > 0
    assert d['e2e']['h2d_bytes_per_step'] == 0 and d['e2e']['d2h_bytes_per_step'] == 0
    assert d['cpu_baseline']['kind'] == 'port' and d['cpu_baseline']['cores'] >= 1
    assert 'workload' in d['config'] and 'model' not in d['config']


def test_metrics_and_event_file(tmp_path):
    """tf2/metrics.py stand-ins and the hand-encoded TensorBoard event records."""
    import struct
    import torch
    from simclr_b200 import metrics as M
    assert M.crc32c(b'123456789') == 0xE3069283                     # CRC-32C check value
    m = M.Mean('train/x'); m.update_state(1.0); m.update_state(torch.tensor(3.0)); assert m.result() == 2.0
    m.reset_states(); assert m.result() == 0.0
    logits = torch.tensor([[0.1, 0.9, 0.0], [0.8, 0.1, 0.1], [0.2, 0.3, 0.5]])
    labels = torch.nn.functional.one_hot(torch.tensor([1, 2, 2]), 3).float()
    a1 = M.Accuracy('a1'); a5 = M.TopKCategoricalAccuracy(2, 'a2')
    M.update_finetune_metrics_eval(a1, a5, logits, labels)
    assert abs(a1.result() - 2 / 3) < 1e-6 and abs(a5.result() - 2 / 3) < 1e-6
    sl, sa = M.Mean('l'), M.Mean('a')
    M.update_finetune_metrics_train(sl, sa, 0.5, labels[:1], torch.cat([logits[:1], logits[:1]]))   # labels doubled
    assert sa.result() == 1.0
    w = M.SummaryWriter(str(tmp_path))
    w.scalar('train/total_loss', 1.5, step=7); w.flush(); w.close()
    data = open(w.path, 'rb').read()
    recs, off = [], 0
    while off < len(data):
        (n,) = struct.unpack('<Q', data[off:off + 8])
        assert struct.unpack('<I', data[off + 8:off + 12])[0] == M._masked_crc(data[off:off + 8])
        body = data[off + 12:off + 12 + n]
        assert struct.unpack('<I', data[off + 12 + n:off + 16 + n])[0] == M._masked_crc(body)
        recs.append(body); off += 16 + n
    assert len(recs) == 2 and b'brain.Event:2' in recs[0]
    assert b'train/total_loss' in recs[1] and struct.pack('<f', 1.5) in recs[1] and recs[1][9:11] == bytes([0x10, 0x07])   # step = 7


def test_checkpoint_manager_roundtrip(tmp_path):
    """CheckpointManager: reference variable names, pruning to max_to_keep, latest, partial restore."""
    import torch
    from simclr_b200 import checkpoint as C

    class V:
        def __init__(self, name, t): self.name, self.value, self.shape = name, t, tuple(t.shape)

    class FakeModel:
        def __init__(self):
            self.variables = [V('resnet/conv2d/kernel:0', torch.arange(6.).view(1, 1, 2, 3)), V('head/bias:0', torch.ones(4))]
            self.trainable_variables = self.variables

    class FakeOpt:
        def __init__(self): self._flat_v = torch.full((8,), 2.0); self.iterations = 0
        def ensure_built(self, vs): pass

    m, o = FakeModel(), FakeOpt()
    mgr = C.CheckpointManager(m, o, str(tmp_path), max_to_keep=2)
    assert mgr.latest_checkpoint is None
    for step in (10, 20, 30):
        m.variables[1].value.fill_(float(step)); mgr.save(step)
    assert [os.path.basename(p) for p in mgr._paths()] == ['ckpt-20.npz', 'ckpt-30.npz']
    m2, o2 = FakeModel(), FakeOpt(); o2._flat_v.zero_()
    m2.variables.append(V('new/extra:0', torch.zeros(2)))               # not in the file: skipped (expect_partial)
    step = C.CheckpointManager(m2, o2, str(tmp_path)).restore(mgr.latest_checkpoint)
    assert step == 30 and o2.iterations == 30 and float(m2.variables[1].value[0]) == 30.0 and float(o2._flat_v[0]) == 2.0
    m3 = FakeModel(); m3.variables[1].value.zero_()
    assert C.CheckpointManager(m3, None, str(tmp_path)).restore(mgr.latest_checkpoint, weights_only=True) == 0
    assert float(m3.variables[1].value[0]) == 30.0


def test_input_pipeline_host_logic(tmp_path):
    """tf2/data.py:29-98 over an ArrayBuilder: per-replica batch size, per-pipeline shards, shuffle buffer + repeat +
    drop_remainder when training, one ordered pass with a ragged last batch otherwise, npz round trip."""
    import numpy as np
    from simclr_b200 import data as D, flags_def
    F = flags_def.FLAGS
    if not F.is_parsed():
        F(['test'])
    saved = {k: getattr(F, k) for k in ('image_size', 'train_mode', 'train_split', 'eval_split')}
    try:
        flags_def.set_flags(image_size=64, train_mode='pretrain', train_split='train', eval_split='validation')
        imgs = np.zeros((50, 8, 8, 3), dtype=np.uint8)
        path = str(tmp_path / 'toy.npz')
        np.savez(path, train_images=imgs, train_labels=np.arange(50) % 5, validation_images=imgs[:11],
                 validation_labels=np.arange(11) % 5, num_classes=5)
        b = D.ArrayBuilder.from_npz(path)
        assert b.info.splits['train'].num_examples == 50 and b.info.features['label'].num_classes == 5
        fake = lambda e, idx: list(idx)
        ctx0, ctx1 = D.InputContext(2, 0, 2), D.InputContext(2, 1, 2)
        it0 = D.build_input_fn(b, 8, None, True)(ctx0, seed=1, make_batch=fake)
        it1 = D.build_input_fn(b, 8, None, True)(ctx1, seed=1, make_batch=fake)
        a = [next(it0) for _ in range(20)]; c = [next(it1) for _ in range(20)]
        assert all(len(x) == 4 for x in a + c)                                  # 8 global / 2 replicas
        assert set(sum(a, [])) <= set(range(0, 25)) and set(sum(c, [])) <= set(range(25, 50))   # disjoint shards
        assert set(sum(a, [])) == set(range(0, 25))                             # repeat(-1): every example comes around
        assert sum(a, [])[:25] != list(range(25))                               # shuffled (buffer of 40 > shard)
        ev = list(D.build_input_fn(b, 8, None, False)(D.InputContext(1, 0, 1), make_batch=fake))
        assert [len(x) for x in ev] == [8, 3] and sum(ev, []) == list(range(11))   # ordered, ragged last batch kept
        with pytest.raises(ValueError):
            D.build_input_fn(b, 9, None, True)(ctx0, make_batch=fake)
    finally:
        flags_def.set_flags(**saved)


def _example_message_classes():
    """tf.train.Example / Features / Feature built with the protobuf runtime from the published schema
    (tensorflow/core/example/{example,feature}.proto) -- an independent encoder / decoder for the wire format."""
    from google.protobuf import descriptor_pb2, descriptor_pool, message_factory
    fd = descriptor_pb2.FileDescriptorProto(name='simclr_test_example.proto', package='tftest', syntax='proto3')
    F = descriptor_pb2.FieldDescriptorProto

    def msg(name, fields):
        m = fd.message_type.add(name=name)
        for fname, num, typ, label, tname in fields:
            f = m.field.add(name=fname, number=num, type=typ, label=label)
            if tname:
                f.type_name = tname
        return m
    msg('BytesList', [('value', 1, F.TYPE_BYTES, F.LABEL_REPEATED, None)])
    msg('FloatList', [('value', 1, F.TYPE_FLOAT, F.LABEL_REPEATED, None)])
    msg('Int64List', [('value', 1, F.TYPE_INT64, F.LABEL_REPEATED, None)])
    feat = msg('Feature', [('bytes_list', 1, F.TYPE_MESSAGE, F.LABEL_OPTIONAL, '.tftest.BytesList'),
                           ('float_list', 2, F.TYPE_MESSAGE, F.LABEL_OPTIONAL, '.tftest.FloatList'),
                           ('int64_list', 3, F.TYPE_MESSAGE, F.LABEL_OPTIONAL, '.tftest.Int64List')])
    feat.oneof_decl.add(name='kind')
    for f in feat.field:
        f.oneof_index = 0
    feats = msg('Features', [('feature', 1, F.TYPE_MESSAGE, F.LABEL_REPEATED, '.tftest.Features.FeatureEntry')])
    entry = feats.nested_type.add(name='FeatureEntry')
    entry.options.map_entry = True
    entry.field.add(name='key', number=1, type=F.TYPE_STRING, label=F.LABEL_OPTIONAL)
    entry.field.add(name='value', number=2, type=F.TYPE_MESSAGE, label=F.LABEL_OPTIONAL, type_name='.tftest.Feature')
    msg('Example', [('features', 1, F.TYPE_MESSAGE, F.LABEL_OPTIONAL, '.tftest.Features')])
    pool = descriptor_pool.DescriptorPool()
    pool.Add(fd)
    return message_factory.GetMessageClass(pool.FindMessageTypeByName('tftest.Example'))


def test_tf_example_wire_format_against_protobuf():
    """`tfrecord.parse_example` reads what the protobuf runtime serialises for the Example schema, and the protobuf
    runtime parses what `tfrecord.encode_example` writes (negative labels, multi-element lists, empty features)."""
    from simclr_b200 import tfrecord as T
    Example = _example_message_classes()
    ex = Example()
    ex.features.feature['image'].bytes_list.value.append(b'\x00\xff\x10JPEGDATA' * 50)
    ex.features.feature['label'].int64_list.value.extend([7])
    ex.features.feature['neg'].int64_list.value.extend([-3, 1 << 40, 0])
    ex.features.feature['scores'].float_list.value.extend([0.5, -2.25, 1e-3])
    ex.features.feature['file_name'].bytes_list.value.extend([b'n01440764_10026.JPEG', b'second'])
    ex.features.feature['empty'].bytes_list.SetInParent()
    got = T.parse_example(ex.SerializeToString())
    assert got['image'] == [b'\x00\xff\x10JPEGDATA' * 50] and got['label'] == [7] and got['neg'] == [-3, 1 << 40, 0]
    assert got['file_name'] == [b'n01440764_10026.JPEG', b'second'] and got['empty'] == []
    assert [round(x, 6) for x in got['scores']] == [0.5, -2.25, 0.001]
    mine = T.encode_example({'image': b'abc' * 100, 'label': 999, 'neg': [-1, 5], 'scores': [1.5, 2.5]})
    back = Example()
    back.ParseFromString(mine)
    assert back.features.feature['image'].bytes_list.value[0] == b'abc' * 100
    assert list(back.features.feature['label'].int64_list.value) == [999]
    assert list(back.features.feature['neg'].int64_list.value) == [-1, 5]
    assert list(back.features.feature['scores'].float_list.value) == [1.5, 2.5]
    assert T.parse_example(mine) == {'image': [b'abc' * 100], 'label': [999], 'neg': [-1, 5], 'scores': [1.5, 2.5]}


def test_tfrecord_framing_and_tfds_directory(tmp_path):
    """TFRecord framing (the CRC-32C check value and a corrupted header), and `data.TFRecordBuilder` over a directory in
    the TFDS layout: split discovery, example counts from dataset_info.json, classes from features.json, PNG / JPEG
    decode, whole files per input pipeline, shuffled repeat for training, one ordered pass for eval."""
    import io, json
    import numpy as np
    from PIL import Image
    from simclr_b200 import tfrecord as T, data as D, flags_def
    p = str(tmp_path / 'x.tfrecord')
    T.write_records(p, [b'', b'hello', b'x' * 1000])
    assert list(T.read_records(p, verify_data_crc=True)) == [b'', b'hello', b'x' * 1000] and T.count_records(p) == 3
    raw = bytearray(open(p, 'rb').read()); raw[2] ^= 1
    open(p, 'wb').write(bytes(raw))
    with pytest.raises(T.TFRecordError):
        list(T.read_records(p))
    # a TFDS-style directory: toy/1.0.0/toy-train.tfrecord-0000i-of-00004, toy-validation.tfrecord-00000-of-00001
    d = tmp_path / 'tfds' / 'toy' / '1.0.0'
    d.mkdir(parents=True)
    rs = np.random.RandomState(0)
    imgs = [rs.randint(0, 256, (20 + i % 5, 24 + i % 3, 3), dtype=np.uint8) for i in range(22)]
    yy, xx = np.mgrid[0:20, 0:26]
    imgs[20] = np.stack([4 * yy + 3 * xx, 200 - 5 * yy, 9 * xx], -1).astype(np.uint8)       # smooth: JPEG stays close
    imgs[21] = imgs[20][::-1].copy()

    def enc(a, fmt):
        b = io.BytesIO(); Image.fromarray(a).save(b, format=fmt, **({'quality': 95} if fmt == 'JPEG' else {})); return b.getvalue()
    shard_len = [5, 5, 5, 5]
    k = 0
    for s_i, n in enumerate(shard_len):
        T.write_records(str(d / ('toy-train.tfrecord-%05d-of-00004' % s_i)),
                        [T.encode_example({'image': enc(imgs[k + j], 'PNG'), 'label': (k + j) % 7, 'file_name': b'f%d' % (k + j)}) for j in range(n)])
        k += n
    T.write_records(str(d / 'toy-validation.tfrecord-00000-of-00001'),
                    [T.encode_example({'image': enc(imgs[20 + j], 'JPEG'), 'label': j}) for j in range(2)])
    json.dump({'name': 'toy', 'splits': [{'name': 'train', 'shardLengths': [str(x) for x in shard_len]}]}, open(d / 'dataset_info.json', 'w'))
    json.dump({'featuresDict': {'features': {'label': {'classLabel': {'numClasses': '7'}}, 'image': {'image': {}}}}}, open(d / 'features.json', 'w'))
    b = D.TFRecordBuilder(str(tmp_path / 'tfds'), 'toy')
    assert b.info.splits['train'].num_examples == 20 and b.info.splits['validation'].num_examples == 2     # json / counted
    assert b.info.features['label'].num_classes == 7
    ctx = D.InputContext(2, 1, 2)
    toks = list(b.tokens('train', ctx, False, None))
    assert [l for _, l in toks] == [(i % 7) for i in list(range(5, 10)) + list(range(15, 20))]             # files 1 and 3
    im, lab = b.fetch('train', toks[0])
    assert lab == 5 and np.array_equal(im, imgs[5])                                                       # PNG: exact
    jm, _ = b.fetch('validation', next(iter(b.tokens('validation', D.InputContext(1, 0, 1), False, None))))
    assert jm.shape == imgs[20].shape and np.abs(jm.astype(int) - imgs[20].astype(int)).mean() < 3        # JPEG: lossy
    # fewer files than pipelines: records are dealt round-robin
    t3 = [list(b.tokens('validation', D.InputContext(3, q, 3), False, None)) for q in range(3)]
    assert [len(x) for x in t3] == [1, 1, 0]
    F = flags_def.FLAGS
    if not F.is_parsed():
        F(['test'])
    saved = {k2: getattr(F, k2) for k2 in ('image_size', 'train_mode', 'train_split', 'eval_split')}
    try:
        flags_def.set_flags(image_size=64, train_mode='pretrain', train_split='train', eval_split='validation')
        fake = lambda e, toks_: [l for _, l in toks_]
        it = D.build_input_fn(b, 4, None, True)(D.InputContext(2, 0, 2), seed=5, make_batch=fake)
        seen = sum([next(it) for _ in range(10)], [])
        assert len(seen) == 20 and set(seen) <= {i % 7 for i in list(range(0, 5)) + list(range(10, 15))}  # pipeline 0: files 0, 2
        ev = list(D.build_input_fn(b, 4, None, False)(D.InputContext(1, 0, 1), make_batch=fake))
        assert ev == [[0, 1]]
    finally:
        flags_def.set_flags(**saved)


def test_input_pipeline_batch_assembly_on_cpu(tmp_path, monkeypatch):
    """The per-batch map of `build_input_fn` (fetch / decode -> augmentation draws -> kernel launches -> one-hot labels)
    with the two GPU entry points replaced by CPU stand-ins: checks the host plumbing for both builders and all three
    modes (two pretraining views, one finetune-training view, centre-crop eval)."""
    import io
    import numpy as np
    import torch
    from PIL import Image
    from simclr_b200 import data as D, data_util as DU, tfrecord as T, flags_def
    calls = []

    def fake_train(images, draws, h, w, out=None, channel_offset=0):
        assert len(images) == len(draws) and all(im.dtype == torch.uint8 and im.dim() == 3 for im in images)
        calls.append(('train', len(images), channel_offset))
        if out is None:
            out = torch.zeros(len(images), h, w, 3)
        out[..., channel_offset:channel_offset + 3] = torch.stack([im.float().mean() / 255.0 for im in images]).view(-1, 1, 1, 1)
        return out

    def fake_eval(images, h, w, crop=True):
        calls.append(('eval', len(images), crop))
        return torch.stack([im.float().mean() / 255.0 for im in images]).view(-1, 1, 1, 1).expand(len(images), h, w, 3).contiguous()
    monkeypatch.setattr(DU, 'preprocess_for_train_batch', fake_train)
    monkeypatch.setattr(DU, 'preprocess_for_eval_batch', fake_eval)
    monkeypatch.setattr(D, 'get_engine', lambda: type('E', (), {'device': torch.device('cpu')})())
    F = flags_def.FLAGS
    if not F.is_parsed():
        F(['test'])
    saved = {k: getattr(F, k) for k in ('image_size', 'train_mode', 'train_split', 'eval_split', 'color_jitter_strength')}
    rs = np.random.RandomState(1)
    arr = rs.randint(0, 256, (12, 30, 34, 3), dtype=np.uint8)
    labels = np.arange(12) % 4
    d = tmp_path / 'toy' / '1.0.0'
    d.mkdir(parents=True)

    def png(a):
        b = io.BytesIO(); Image.fromarray(a).save(b, format='PNG'); return b.getvalue()
    T.write_records(str(d / 'toy-train.tfrecord-00000-of-00001'), [T.encode_example({'image': png(arr[i]), 'label': int(labels[i])}) for i in range(12)])
    T.write_records(str(d / 'toy-validation.tfrecord-00000-of-00001'), [T.encode_example({'image': png(arr[i]), 'label': int(labels[i])}) for i in range(5)])
    builders = [D.ArrayBuilder({'train': (arr, labels), 'validation': (arr[:5], labels[:5])}, 4),
                D.TFRecordBuilder(str(tmp_path), 'toy', num_classes=4)]
    try:
        for b in builders:
            flags_def.set_flags(image_size=48, train_mode='pretrain', train_split='train', eval_split='validation')
            calls.clear()
            f, lab = next(D.build_input_fn(b, 4, None, True)(D.InputContext(1, 0, 1), seed=2))
            assert f.shape == (4, 48, 48, 6) and lab.shape == (4, 4) and torch.equal(lab.sum(1), torch.ones(4))
            assert calls == [('train', 4, 0), ('train', 4, 3)] and torch.equal(f[..., 0], f[..., 3])      # both views of the same images
            flags_def.set_flags(train_mode='finetune')
            calls.clear()
            f, lab = next(D.build_input_fn(b, 4, None, True)(D.InputContext(1, 0, 1), seed=2))
            assert f.shape == (4, 48, 48, 3) and calls == [('train', 4, 0)]
            calls.clear()
            ev = list(D.build_input_fn(b, 4, None, False)(D.InputContext(1, 0, 1)))
            assert [x[0].shape[0] for x in ev] == [4, 1] and calls == [('eval', 4, True), ('eval', 1, True)]
            assert torch.equal(torch.cat([x[1] for x in ev]).argmax(1), torch.from_numpy(labels[:5]))
            want = torch.from_numpy(arr[:5]).float().mean(dim=(1, 2, 3)) / 255.0                           # ordered pass, exact decode
            assert torch.allclose(torch.cat([x[0][:, 0, 0, 0] for x in ev]), want)
    finally:
        flags_def.set_flags(**saved)


def test_tensorflow_checkpoint_bundle_reader(tmp_path):
    """tf_checkpoint: LevelDB-format table (prefix compression across restart points, several data blocks, block
    checksums, footer magic), BundleEntryProto, the object graph's full_name join, bf16 / int64 tensors, and
    CheckpointManager restoring from a TensorFlow-format prefix (`--checkpoint`) or from a model_dir of them."""
    import struct
    import numpy as np
    import torch
    from simclr_b200 import tf_checkpoint as TC, checkpoint as C
    from simclr_b200.tfrecord import _varint, _ld
    from simclr_b200.metrics import _masked_crc
    rs = np.random.RandomState(0)
    # many keys with long shared prefixes: exercises shared-prefix decoding, restart points and the index block
    tensors, names = {}, {}
    for i in range(150):
        key = 'model/resnet_model/block_group%d/layer_with_a_long_name_%03d/kernel%s' % (i % 4, i, TC.VARIABLE_SUFFIX)
        tensors[key] = rs.randn(1 + i % 3, 2, 3).astype(np.float32)
        names[key] = 'resnet/block_group%d/conv2d_%d/kernel' % (i % 4, i)
    tensors['global_step' + TC.VARIABLE_SUFFIX] = np.asarray(4321, dtype=np.int64)
    tensors['flag'] = np.asarray([True, False])
    prefix = str(tmp_path / 'tf' / 'ckpt-4321')
    TC.write_bundle(prefix, tensors, names)
    raw = open(prefix + '.index', 'rb').read()
    assert struct.unpack('<Q', raw[-8:])[0] == 0xdb4775248b80fb57
    r = TC.TensorBundleReader(prefix)
    assert set(r.keys()) == set(tensors) | {TC.OBJECT_GRAPH_KEY} and r.keys() == sorted(r.keys(), key=lambda k: k.encode())
    for k, v in tensors.items():
        got = r.get_tensor(k)
        assert got.dtype == v.dtype and got.shape == v.shape and np.array_equal(got, v)
    assert int(r.get_tensor('global_step' + TC.VARIABLE_SUFFIX)) == 4321
    byname = r.variables_by_name()
    assert len(byname) == 150 and np.array_equal(byname['resnet/block_group3/conv2d_7/kernel'], tensors[[k for k in names if names[k].endswith('conv2d_7/kernel')][0]])
    # the stored entry checksum is the masked CRC-32C of the tensor bytes
    k0 = sorted(names)[0]
    assert r.entries[k0].crc32c == _masked_crc(tensors[k0].tobytes())
    # corruption inside a data block is detected
    bad = bytearray(raw); bad[10] ^= 0xFF
    open(prefix + '.index', 'wb').write(bytes(bad))
    with pytest.raises(TC.CheckpointFormatError):
        TC.TensorBundleReader(prefix)
    open(prefix + '.index', 'wb').write(raw)
    # a hand-assembled bf16 entry (DT_BFLOAT16 = 14): 1.0, -2.0 as 0x3F80, 0xC000
    p2 = str(tmp_path / 'tf' / 'bf')
    entry = _varint(1 << 3) + _varint(14) + _ld(2, _ld(2, _varint(1 << 3) + _varint(2))) + _varint(4 << 3) + _varint(0) + _varint(5 << 3) + _varint(4)
    TC.write_table(p2 + '.index', [(b'', _varint(1 << 3) + _varint(1)), (b'w', entry)])
    open(p2 + '.data-00000-of-00001', 'wb').write(struct.pack('<HH', 0x3F80, 0xC000))
    assert TC.TensorBundleReader(p2).get_tensor('w').tolist() == [1.0, -2.0]

    class V:
        def __init__(self, name, t): self.name, self.value, self.shape = name, t, tuple(t.shape)

    class FakeModel:
        def __init__(self):
            self.variables = [V('resnet/block_group3/conv2d_7/kernel:0', torch.zeros(2, 2, 3)), V('resnet/block_group0/conv2d_0/kernel:0', torch.zeros(1, 2, 3)),
                              V('not/in/file:0', torch.ones(3)), V('resnet/block_group1/conv2d_1/kernel:0', torch.zeros(9, 9))]   # last: shape mismatch
            self.trainable_variables = self.variables

    class FakeOpt:
        iterations = 0
    m = FakeModel()
    assert C.CheckpointManager(m, None, None).restore(prefix, weights_only=True) == 0
    assert np.array_equal(m.variables[0].value.numpy(), byname['resnet/block_group3/conv2d_7/kernel'])
    assert np.array_equal(m.variables[1].value.numpy(), byname['resnet/block_group0/conv2d_0/kernel'])
    assert float(m.variables[2].value.sum()) == 3.0 and float(m.variables[3].value.abs().sum()) == 0.0
    # a model_dir written by the reference: latest ckpt-N.index is picked up, the step comes from global_step
    m2, o2 = FakeModel(), FakeOpt()
    mgr = C.CheckpointManager(m2, o2, str(tmp_path / 'tf'))
    assert mgr.latest_checkpoint == prefix
    assert mgr.restore(mgr.latest_checkpoint) == 4321 and o2.iterations == 4321


def test_formats_pinned_against_tensorboard_protos_and_reader(tmp_path):
    """Independent implementations available offline (TensorBoard vendors TensorFlow's protos and ships a pure-Python
    TFRecord reader that checks both CRCs): the object graph / shape / dtype numbering `tf_checkpoint` assumes, the
    TFRecord framing `tfrecord.write_records` and `metrics.SummaryWriter` emit, and the scalar events they carry."""
    tb = pytest.importorskip('tensorboard')
    import numpy as np
    from tensorboard.compat.proto import trackable_object_graph_pb2 as TG, types_pb2, tensor_shape_pb2, event_pb2
    from tensorboard.compat.tensorflow_stub.pywrap_tensorflow import PyRecordReader_New
    from simclr_b200 import tf_checkpoint as TC, tfrecord as T, metrics as M
    # dtype numbering
    for code, dt in TC._DTYPES.items():
        name = {'bfloat16': 'DT_BFLOAT16'}.get(dt) if isinstance(dt, str) else None
        name = name or {'float32': 'DT_FLOAT', 'float64': 'DT_DOUBLE', 'int32': 'DT_INT32', 'uint8': 'DT_UINT8', 'int16': 'DT_INT16',
                        'int8': 'DT_INT8', 'int64': 'DT_INT64', 'bool': 'DT_BOOL', 'uint16': 'DT_UINT16', 'float16': 'DT_HALF',
                        'uint32': 'DT_UINT32', 'uint64': 'DT_UINT64'}[np.dtype(dt).name]
        assert getattr(types_pb2, name) == code, name
    assert types_pb2.DT_STRING == TC.DT_STRING
    # an object graph serialised by the real proto classes, stored as the bundle's string tensor, read back by our parser
    g = TG.TrackableObjectGraph()
    root = g.nodes.add()
    for i, (key, full) in enumerate([('model/a/kernel' + TC.VARIABLE_SUFFIX, 'resnet/conv2d/kernel'), ('model/a/bias' + TC.VARIABLE_SUFFIX, 'head/bias')]):
        c = root.children.add(); c.node_id = i + 1; c.local_name = 'child%d' % i
        n = g.nodes.add()
        a = n.attributes.add(); a.name = 'VARIABLE_VALUE'; a.full_name = full; a.checkpoint_key = key
        n.slot_variables.add().slot_name = 'Momentum'
    prefix = str(tmp_path / 'ck')
    tensors = {'model/a/kernel' + TC.VARIABLE_SUFFIX: np.arange(6, dtype=np.float32).reshape(1, 1, 2, 3),
               'model/a/bias' + TC.VARIABLE_SUFFIX: np.ones(3, dtype=np.float32), TC.OBJECT_GRAPH_KEY: g.SerializeToString()}
    TC.write_bundle(prefix, tensors)
    r = TC.TensorBundleReader(prefix)
    assert sorted(r.object_graph()) == sorted([(a.checkpoint_key, a.full_name, a.name) for n in g.nodes for a in n.attributes])
    assert set(r.variables_by_name()) == {'resnet/conv2d/kernel', 'head/bias'}
    # ... and our writer's object graph parses with the real proto classes
    TC.write_bundle(prefix + '2', {k: v for k, v in tensors.items() if k != TC.OBJECT_GRAPH_KEY}, {k: 'n/' + k[:9] for k in tensors if k != TC.OBJECT_GRAPH_KEY})
    g2 = TG.TrackableObjectGraph(); g2.ParseFromString(TC.TensorBundleReader(prefix + '2').get_string(TC.OBJECT_GRAPH_KEY))
    assert len(g2.nodes) == 3 and len(g2.nodes[0].children) == 2 and g2.nodes[1].attributes[0].name == 'VARIABLE_VALUE'
    # TensorShapeProto as written into BundleEntryProto.shape
    sh = tensor_shape_pb2.TensorShapeProto(); sh.ParseFromString(TC._shape_proto((7, 1, 3)))
    assert [d.size for d in sh.dim] == [7, 1, 3]
    assert TC._parse_shape(memoryview(tensor_shape_pb2.TensorShapeProto(dim=[tensor_shape_pb2.TensorShapeProto.Dim(size=5), tensor_shape_pb2.TensorShapeProto.Dim(size=0)]).SerializeToString())) == (5, 0)
    # TFRecord framing: TensorBoard's reader (verifies length and data CRCs) reads what we write
    p = str(tmp_path / 'r.tfrecord')
    payloads = [b'', b'abc', bytes(range(256)) * 9]
    T.write_records(p, payloads)
    rd = PyRecordReader_New(p); got = []
    while True:
        try:
            rd.GetNext()
        except Exception:
            break
        got.append(rd.record())
    assert got == payloads
    # event file written by metrics.SummaryWriter -> real Event protos
    w = M.SummaryWriter(str(tmp_path)); w.scalar('train/total_loss', 1.5, step=7); w.scalar('lr', 0.25, step=8); w.flush(); w.close()
    evs = []
    for rec in T.read_records(w.path, verify_data_crc=True):
        e = event_pb2.Event(); e.ParseFromString(rec); evs.append(e)
    vals = [(e.step, v.tag, v.simple_value) for e in evs for v in e.summary.value]
    assert vals == [(7, 'train/total_loss', 1.5), (8, 'lr', 0.25)] and evs[0].file_version.startswith('brain.Event')
