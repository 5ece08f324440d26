#!/usr/bin/env python
"""bench.py -- images/sec of the SimCLR pretrain step (BASELINE.json metric).

    python bench.py --gpus N --steps K --warmup W            # this implementation
    python bench.py --impl reference --steps K --warmup W    # CPU restatement of the reference step

N=1 workload: ResNet-50 1x, batch 256 per GPU (what one 80 GB H100 holds next
to the profiling pass), 224x224 synthetic, proj_dim 128, temperature 0.1, LARS,
blur + linear-eval head on, SyncBN flag on.  Under torchrun (N>1) every rank
keeps 256 samples (weak scaling).  A "step" is one complete
`single_step` (tf2/run.py:557-622): forward, NT-Xent, backward, gradient
all-reduce, LARS.  One JSON line is printed by rank 0.

--dump-outputs DIR writes, after the timed steps, what the last timed step
computed: its loss and a fixed, seeded sample of every updated trainable
variable, as DIR/<name>.npy (float64 / float32), so that two builds can be
compared output for output on identical seeded inputs.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

# SURVEY.md 8d: algorithmic conv GFLOP per image (2 views, fwd + dgrad + wgrad); key (depth, width, size, SK)
GFLOP_PER_IMAGE = {(50, 1, 224, False): 48.574, (18, 1, 64, False): 1.751, (50, 2, 224, False): 192.406,
                   (152, 2, 224, True): 841.196}


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument('--gpus', type=int, default=1)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--impl', default='b200', choices=['b200', 'reference'])
    ap.add_argument('--batch', type=int, default=256, help='samples per GPU')
    ap.add_argument('--resnet_depth', type=int, default=50)
    ap.add_argument('--width_multiplier', type=int, default=1)
    ap.add_argument('--image_size', type=int, default=224)
    ap.add_argument('--precision', default='bf16', choices=['bf16', 'fp32'])
    ap.add_argument('--engine', default='tc', choices=['tc', 'tc3', 'simt'],
                    help='tc: bf16 wgmma (the benchmarked mode); tc3: fp32-accurate split-bf16 wgmma (needs --precision fp32)')
    ap.add_argument('--sk_ratio', type=float, default=0.0, help='config 5: 0.0625')
    ap.add_argument('--num_proj_layers', type=int, default=3)
    ap.add_argument('--learning_rate', type=float, default=0.3)
    ap.add_argument('--learning_rate_scaling', default='linear', choices=['linear', 'sqrt'])
    ap.add_argument('--no_secondary', action='store_true', help='skip the fp32-accurate tensor-core mode measurement')
    ap.add_argument('--no_graph', action='store_true')
    ap.add_argument('--no_cpu_baseline', action='store_true')
    ap.add_argument('--cpu_batch', type=int, default=16)
    ap.add_argument('--cpu_steps', type=int, default=2)
    ap.add_argument('--dump-outputs', dest='dump_outputs', default=None, metavar='DIR',
                    help='write the last timed step\'s outputs as DIR/<name>.npy')
    return ap.parse_args()


def workload_string(args, world):
    return ('ResNet-%d %dx%s, batch %d per GPU (global %d), %dx%d synthetic, proj_dim 128, %d-layer head, temperature 0.1, '
            'LARS, blur on, lineareval head on, global_bn on'
            % (args.resnet_depth, args.width_multiplier, ' SK' if args.sk_ratio > 0 else '', args.batch,
               args.batch * world, args.image_size, args.image_size, args.num_proj_layers))


def measured_peaks():
    p = os.path.join(ROOT, 'MEASURED_PEAKS.json')
    if os.path.exists(p):
        d = json.load(open(p))
        return dict(tflops=d['bf16_tflops_sustained'], hbm=d['hbm_gbs'], which='measured (sustained bf16, MEASURED_PEAKS.json)')
    return dict(tflops=989.0, hbm=3350.0, which='H100 SXM data sheet (dense bf16, HBM3; 700 W), not a measured peak')


class ClockSampler(threading.Thread):
    """Samples nvidia-smi clocks / throttle reasons during the timed region."""
    Q = ('clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,'
         'clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,'
         'clocks_event_reasons.sw_power_cap')

    def __init__(self, index=0):
        super().__init__(daemon=True)
        self.index, self.samples, self.stop_flag = index, [], False

    def run(self):
        while not self.stop_flag:
            try:
                out = subprocess.run(['nvidia-smi', '-i', str(self.index), '--query-gpu=' + self.Q,
                                      '--format=csv,noheader,nounits'], capture_output=True, text=True, timeout=5).stdout
                parts = [x.strip() for x in out.strip().split(',')]
                if len(parts) >= 7:
                    self.samples.append(parts)
            except Exception:
                pass
            time.sleep(0.1)

    def summary(self):
        if not self.samples:
            return {'sm_mhz': None, 'sm_max_mhz': None, 'reasons': ['no samples']}
        sm = [float(s[0]) for s in self.samples if s[0].replace('.', '').isdigit()]
        names = ['hw_slowdown', 'hw_thermal_slowdown', 'sw_thermal_slowdown', 'sw_power_cap']
        reasons = [n for i, n in enumerate(names) if any(s[3 + i].lower().startswith('active') for s in self.samples)]
        return {'sm_mhz': statistics.median(sm) if sm else None, 'sm_max_mhz': float(self.samples[0][1]),
                'power_w_max': max(float(s[2]) for s in self.samples), 'samples': len(self.samples), 'reasons': reasons}


def oracle_step_time(args, batch, steps, warmup=1):
    """Times the CPU restatement of the reference step (oracle/) on the host cores."""
    import torch
    from oracle.config import default_cfg
    from oracle import model as OM, step as OS
    import collections
    torch.set_num_threads(cpu_threads())
    cfg = default_cfg(resnet_depth=args.resnet_depth, width_multiplier=args.width_multiplier,
                      image_size=args.image_size, train_batch_size=batch, sk_ratio=args.sk_ratio,
                      num_proj_layers=args.num_proj_layers)
    m = OM.Model(cfg, 1000)
    P, S = m.init(0)
    V = collections.OrderedDict((k, torch.zeros_like(v)) for k, v in P.items())
    g = torch.Generator().manual_seed(1234)
    f = torch.rand(batch, args.image_size, args.image_size, 6, generator=g)
    lab = torch.nn.functional.one_hot(torch.randint(0, 1000, (batch,), generator=g), 1000).float()
    times = []
    for i in range(warmup + steps):
        t0 = time.perf_counter()
        P, S, V, info = OS.single_step(m, P, S, V, [f], [lab], 0.1)
        dt = time.perf_counter() - t0
        if i >= warmup:
            times.append(dt)
    return sum(times) / len(times), float(info['loss'])


def cpu_threads():
    """Threads for the CPU arm: all cores up to 32 (PyTorch-CPU scales negatively beyond that on the
    128-core GPU hosts: 0.28 img/s at 128 threads vs ~3 img/s at 8-32)."""
    return int(os.environ.get('SIMCLR_CPU_THREADS', min(os.cpu_count() or 1, 32)))


def cpu_model_name():
    try:
        for line in open('/proc/cpuinfo'):
            if line.startswith('model name'):
                return line.split(':', 1)[1].strip()
    except Exception:
        pass
    return 'unknown'


def run_reference(args):
    rank = int(os.environ.get('RANK', '0'))
    if rank != 0:
        return
    workload = workload_string(args, max(1, args.gpus))
    sec, loss = oracle_step_time(args, args.cpu_batch, max(1, args.steps), max(1, min(args.warmup, 1)))
    ips = args.cpu_batch / sec
    line = {
        'impl': 'reference', 'metric': 'images/sec pretrain step', 'value': ips, 'unit': 'images/s', 'n_gpus': max(1, args.gpus),
        'steps': args.steps, 'warmup': args.warmup, 'ms_per_step': sec * 1e3, 'higher_is_better': True,
        'scaling': 'weak', 'vs_baseline': None, 'dtype': 'f32', 'data': 'synthetic',
        'config': {'workload': workload, 'sample': 'batch %d per step (CPU throughput is ~batch independent)' % args.cpu_batch},
        'cpu_baseline': {'value': ips, 'unit': 'images/s', 'cores': cpu_threads(), 'kind': 'port',
                         'sample': '%d steps of batch %d on %s; oracle restatement of tf2/run.py single_step '
                                   '(TensorFlow is not installable here)' % (args.steps, args.cpu_batch, cpu_model_name())},
        'e2e': {'value': ips, 'unit': 'images/s', 'h2d_bytes_per_step': 0, 'd2h_bytes_per_step': 0},
        'loss': loss,
    }
    emit(line)


def run_b200(args):
    import torch
    import torch.distributed as dist
    from simclr_b200 import engine, run, flags_def
    from simclr_b200._lib import lib

    t_start = time.time()

    def log(msg):
        sys.stderr.write('[bench rank %s +%.1fs] %s\n' % (os.environ.get('RANK', '0'), time.time() - t_start, msg))
        sys.stderr.flush()

    rank = run.init_distributed()
    log('process group ready')
    # the per-step random draws of the step (blur sigma / selector) come from torch's default generators: seed them,
    # so that the same arguments give the same inputs, and the same outputs, on every run
    torch.manual_seed(1234 + rank)
    world = dist.get_world_size() if dist.is_initialized() else 1
    local = int(os.environ.get('LOCAL_RANK', '0'))
    torch.cuda.set_device(local)
    B, S = args.batch, args.image_size
    flags_def.set_flags(resnet_depth=args.resnet_depth, width_multiplier=args.width_multiplier, image_size=S,
                        train_batch_size=B * world, temperature=0.1, proj_out_dim=128, optimizer='lars',
                        sk_ratio=args.sk_ratio, num_proj_layers=args.num_proj_layers, learning_rate=args.learning_rate,
                        learning_rate_scaling=args.learning_rate_scaling,
                        use_tpu=False, b200_precision=args.precision, b200_conv_engine=args.engine)
    eng = engine.set_engine(engine.Engine(precision=args.precision, conv_engine=args.engine))
    trainer = run.Trainer(num_classes=1000, num_examples=1281167, seed=0)
    features, labels = run.synthetic_batch(B, S, 1000, eng.device, 1234 + rank)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    log('model built')
    # ---- capture -------------------------------------------------------------
    # One CUDA graph per step on a single GPU.  With more than one rank the in-step collectives (SyncBN
    # statistics, embedding / lse all-gathers) are our own NVLink peer-memory kernels, so forward + backward
    # is one graph, the NCCL gradient all-reduce sits between it and a second graph with the LARS update.
    # Without peer memory (SIMCLR_COMM=nccl) the step is launched eagerly.
    peer = trainer.strategy.comm is not None
    use_graph = (not args.no_graph) and (world == 1 or peer)
    launches0 = lib.launch_count
    graph_note = None
    if use_graph:
        ok = 1
        try:
            trainer.capture(features, labels, warmup=1)
            trainer.replay()
            torch.cuda.synchronize()
        except Exception as ex:           # every rank must agree before anyone changes path
            ok = 0
            graph_note = 'graph / peer-memory path failed on rank %d: %r' % (rank, ex)
            log(graph_note)
        if world > 1:
            t_ok = torch.tensor([ok], device=eng.device)
            dist.all_reduce(t_ok, op=dist.ReduceOp.MIN)
            ok = int(t_ok.item())
        if not ok:
            # fall back for the whole job: eager launches, every collective through NCCL
            use_graph = False
            peer = False
            trainer.strategy.comm = None
            trainer._graph = trainer._graph_bottom = trainer._graph_apply = None
            eng.end_step()
            graph_note = graph_note or 'graph / peer-memory path failed on another rank'
    step_fn = trainer.replay if use_graph else (lambda: trainer.single_step(features, labels))
    if use_graph:
        # launches recorded during the capture pass == launches per replay
        c0 = lib.launch_count
        trainer2_count = (c0 - launches0) // 2      # warm-up step + capture pass
        launches_per_step = trainer2_count
    else:
        c0 = lib.launch_count
        step_fn()
        launches_per_step = lib.launch_count - c0

    log('first step / capture done')
    for _ in range(max(args.warmup, 3)):
        step_fn()
    barrier()
    log('warm-up done')

    # ---- timed region: K steps, inputs resident in HBM -----------------------
    sampler = ClockSampler(local) if rank == 0 else None
    if sampler:
        sampler.start()
        time.sleep(0.3)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    barrier()
    comm = trainer.strategy.comm if world > 1 else None
    wait0 = comm.wait_ns() if comm is not None else 0
    ev0.record()
    for _ in range(args.steps):
        loss = step_fn()
    ev1.record()
    barrier()
    ms = ev0.elapsed_time(ev1)
    # per-rank slack: time spent inside the SyncBN / all-gather kernels waiting for the peers' contributions.  The
    # slowest GPU of the step waits ~0 ms, the others wait for it: min over ranks = cost of the exchanges themselves,
    # max - min = GPU-to-GPU speed spread (power capping) that lock-step data parallelism cannot hide.
    sync_wait = None
    if comm is not None:
        w = torch.tensor([(comm.wait_ns() - wait0) / 1e6 / args.steps], device=eng.device)
        allw = [torch.zeros_like(w) for _ in range(world)]
        dist.all_gather(allw, w)
        sync_wait = [round(float(x.item()), 3) for x in allw]
    if sampler:
        sampler.stop_flag = True
        sampler.join(2)
    t = torch.tensor([ms], device=eng.device)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms = float(t.item())
    ms_per_step = ms / args.steps
    ips = B * world * args.steps / (ms / 1e3)
    loss_val = float(loss)

    log('timed region done: %.2f ms/step' % ms_per_step + ('' if sync_wait is None else ' peer-wait ms/step per rank %s' % sync_wait))
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, loss, trainer.model.trainable_variables)
        log('outputs written to %s' % args.dump_outputs)
    # ---- e2e: host buffers, H2D inside the timed region, D2H of the loss ------
    host_f = [torch.rand(B, S, S, 6).pin_memory() for _ in range(2)]
    host_l = [labels.cpu().pin_memory() for _ in range(2)]
    loss_host = torch.zeros(1).pin_memory()
    copy_stream = torch.cuda.Stream()
    dev_f = [torch.empty_like(features), torch.empty_like(features)]
    dev_l = [torch.empty_like(labels), torch.empty_like(labels)]
    ready = [torch.cuda.Event(), torch.cuda.Event()]
    consumed = [torch.cuda.Event(), torch.cuda.Event()]

    def h2d(i):
        with torch.cuda.stream(copy_stream):
            copy_stream.wait_event(consumed[i % 2])
            dev_f[i % 2].copy_(host_f[i % 2], non_blocking=True)
            dev_l[i % 2].copy_(host_l[i % 2], non_blocking=True)
            ready[i % 2].record(copy_stream)

    def e2e_step(i):
        cur = torch.cuda.current_stream()
        cur.wait_event(ready[i % 2])
        features.copy_(dev_f[i % 2]); labels.copy_(dev_l[i % 2])      # into the graph's static inputs
        consumed[i % 2].record(cur)
        l = step_fn()
        loss_host.copy_(l.reshape(1), non_blocking=True)
        return l

    for i in range(2):
        consumed[i].record(torch.cuda.current_stream())
    e2e_steps = args.steps
    h2d(0)
    for i in range(2):              # warm the copy path
        h2d(i + 1); e2e_step(i)
    barrier()
    ev0.record()
    base = 2
    for i in range(e2e_steps):
        h2d(base + i + 1)           # prefetch next step's inputs while this step computes
        e2e_step(base + i)
    ev1.record()
    barrier()
    e2e_ms = ev0.elapsed_time(ev1)
    t = torch.tensor([e2e_ms], device=eng.device)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    e2e_ips = B * world * e2e_steps / (float(t.item()) / 1e3)
    h2d_bytes = features.numel() * 4 + labels.numel() * 4

    log('e2e done')
    # ---- roofline pass: per-launch CUDA-event timing of the tensor-core kernels ----
    roof = None
    # every rank runs the profiled step (it contains collectives); rank 0 reports its own timings
    eng.profile = []
    trainer.single_step(features, labels)
    torch.cuda.synchronize()
    if rank == 0:
        peaks = measured_peaks()
        by = {}
        for kind, shape, flops, a, b in eng.profile:
            d = by.setdefault(kind, [0.0, 0.0, 0])
            d[0] += flops; d[1] += a.elapsed_time(b) * 1e-3; d[2] += 1
        tot_f = sum(v[0] for v in by.values()); tot_t = sum(v[1] for v in by.values())
        achieved = tot_f / tot_t / 1e12 if tot_t > 0 else 0.0
        # algorithmic bytes of the conv kernels (activations in + out once, packed weights once)
        alg = 0.0
        for kind, shape, flops, a, b in eng.profile:
            n_, h_, w_, ci, co, r_, s_ = shape
            ho, wo = (h_ - 1) // s_ + 1, (w_ - 1) // s_ + 1
            alg += 2.0 * (n_ * h_ * w_ * ci + n_ * ho * wo * co + r_ * r_ * ci * co)
        n_launch = max(len(eng.profile), 1)
        key = (args.resnet_depth, args.width_multiplier, S, args.sk_ratio > 0)
        step_tflops = (ips / world) * GFLOP_PER_IMAGE[key] / 1e3 if key in GFLOP_PER_IMAGE else None
        roof = {'bound': 'tensor', 'kernel': 'igemm / wgrad / halo3x3 / stem7x7 kernels (wgmma implicit GEMM, %d conv calls per step)' % sum(v[2] for v in by.values()),
                'achieved': achieved, 'peak': peaks['tflops'], 'unit': 'TFLOP/s', 'frac': achieved / peaks['tflops'],
                'algorithmic_bytes': alg / n_launch,
                'peak_source': peaks['which'],
                'conv_share_of_step': tot_t * 1e3 / ms_per_step,
                'conv_kernel_ms': tot_t * 1e3,
                'by_kind': {k: {'tflops': v[0] / v[1] / 1e12, 'ms': v[1] * 1e3, 'launches': v[2]} for k, v in by.items()},
                'whole_step_tflops': step_tflops,
                'whole_step_frac': None if step_tflops is None else step_tflops / peaks['tflops']}

    eng.profile = None
    log('profile pass done')
    # ---- the fp32-accurate tensor-core mode (tc3: split-bf16 products, fp32 storage) beside the headline ----
    # same network and image size on a smaller batch (its activations are fp32 and the headline graph keeps its
    # own memory pool); eager launches, inputs resident, device-timed like `value`.
    secondary = None
    if world == 1 and args.engine == 'tc' and args.precision == 'bf16' and not args.no_secondary:
        try:
            free, _ = torch.cuda.mem_get_info()
            b2 = min(64, B)
            if free > 48 << 30:
                flags_def.set_flags(train_batch_size=b2, b200_precision='fp32', b200_conv_engine='tc3')
                eng2 = engine.set_engine(engine.Engine(precision='fp32', conv_engine='tc3'))
                tr2 = run.Trainer(num_classes=1000, num_examples=1281167, seed=0)
                f2, l2 = run.synthetic_batch(b2, S, 1000, eng2.device, 4321)
                for _ in range(2):
                    tr2.single_step(f2, l2)
                torch.cuda.synchronize()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                n2 = 3
                for _ in range(n2):
                    l2v = tr2.single_step(f2, l2)
                b.record(); torch.cuda.synchronize()
                ms2 = a.elapsed_time(b) / n2
                secondary = {'engine': 'tc3 (three-way split-bf16 products on wgmma, fp32 storage; 1e-3 step parity: '
                                       'tests/test_gpu_step.py::test_step_parity_tc3)',
                             'value': b2 / (ms2 / 1e3), 'unit': 'images/s', 'batch': b2, 'ms_per_step': ms2, 'steps': n2,
                             'cuda_graph': False, 'loss': float(l2v)}
                del tr2, f2, l2
                engine.set_engine(eng)
                flags_def.set_flags(train_batch_size=B * world, b200_precision=args.precision, b200_conv_engine=args.engine)
            else:
                secondary = {'skipped': 'only %.0f GiB free next to the headline graph' % (free / 2 ** 30)}
        except Exception as ex:
            secondary = {'failed': repr(ex)[:300]}
        log('fp32-accurate tensor-core mode done')
    cpu = None
    if rank == 0 and world == 1 and not args.no_cpu_baseline:
        try:
            sec, _ = oracle_step_time(args, args.cpu_batch, args.cpu_steps, 1)
            cpu = {'value': args.cpu_batch / sec, 'unit': 'images/s', 'cores': cpu_threads(), 'kind': 'port',
                   'sample': '%d steps of batch %d (same network, %dx%d) on %s; oracle restatement, not TensorFlow'
                             % (args.cpu_steps, args.cpu_batch, S, S, cpu_model_name())}
        except Exception as ex:      # the CPU leg must never take the GPU number down
            cpu = {'value': None, 'unit': 'images/s', 'cores': cpu_threads(), 'kind': 'port', 'sample': 'failed: %r' % (ex,)}

    if rank == 0:
        line = {
            'metric': 'images/sec pretrain step', 'value': ips, 'unit': 'images/s', 'n_gpus': world,
            'steps': args.steps, 'warmup': max(args.warmup, 3), 'ms_per_step': ms_per_step, 'higher_is_better': True,
            'scaling': 'weak', 'vs_baseline': None,
            'dtype': 'bf16' if args.precision == 'bf16' else ('f32 (split-bf16 tensor-core products)' if args.engine == 'tc3' else 'f32'),
            'data': 'synthetic',
            'config': {'workload': workload_string(args, world),
                       'l2': 'inputs larger than L2 (activations are GBs per step)',
                       'cuda_graph': use_graph, 'graph_fallback': graph_note, 'parallelism': 'dp%d' % world,
                       'collectives': ('none' if world == 1 else ('nvlink peer-memory kernels (SyncBN, all-gathers) + NCCL gradient all-reduce' if peer else 'NCCL'))},
            'e2e': {'value': e2e_ips, 'unit': 'images/s', 'h2d_bytes_per_step': h2d_bytes, 'd2h_bytes_per_step': 4},
            'gpu_launches': launches_per_step * args.steps,
            'peer_wait_ms_per_step_by_rank': sync_wait,
            'clocks': sampler.summary() if sampler else None,
            'roofline': roof, 'cpu_baseline': cpu, 'loss': loss_val,
            'fp32_accurate_tensor_core_mode': secondary,
        }
        emit(line)
    if dist.is_initialized():
        dist.destroy_process_group()


DUMP_SAMPLE = 4096          # elements kept per variable (a fixed, seeded sample of the larger ones)


def dump_outputs(out_dir, loss, variables):
    """The loss of the last timed step and the variables it updated, as .npy files (at most a few MB)."""
    import numpy as np
    import torch
    os.makedirs(out_dir, exist_ok=True)
    np.save(os.path.join(out_dir, 'loss.npy'), np.array([float(loss)], dtype=np.float64))
    g = torch.Generator().manual_seed(0)
    for v in variables:
        flat = v.value.detach().reshape(-1).float().cpu()
        if flat.numel() > DUMP_SAMPLE:
            flat = flat[torch.randperm(flat.numel(), generator=g)[:DUMP_SAMPLE].sort().values]
        name = v.name.replace('/', '.').replace(':', '_')
        np.save(os.path.join(out_dir, name + '.npy'), flat.numpy().astype(np.float32))


def _watchdog(seconds):
    """Abort (instead of hanging a whole GPU box) if the run does not finish in time."""
    import signal

    def handler(signum, frame):
        sys.stderr.write('bench.py: watchdog expired after %d s\n' % seconds)
        os._exit(3)
    signal.signal(signal.SIGALRM, handler)
    signal.alarm(seconds)


_REAL_STDOUT = None


def _quiet_stdout():
    """The contract is ONE JSON line on stdout.  Libraries (NCCL prints its version banner there when
    NCCL_DEBUG is set) write to fd 1 directly, so fd 1 is pointed at stderr for the whole run and the
    saved descriptor is used for the result line only."""
    global _REAL_STDOUT
    sys.stdout.flush()
    _REAL_STDOUT = os.fdopen(os.dup(1), 'w')
    os.dup2(2, 1)


def emit(line):
    out = _REAL_STDOUT or sys.stdout
    out.write(json.dumps(line) + '\n')
    out.flush()


def main():
    args = parse_args()
    _quiet_stdout()
    _watchdog(int(os.environ.get('SIMCLR_BENCH_TIMEOUT', '900')))
    if args.impl == 'reference':
        run_reference(args)
    else:
        run_b200(args)


if __name__ == '__main__':
    main()
