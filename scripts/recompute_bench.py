#!/usr/bin/env python
"""Activation recomputation: predicted and measured memory, step time, and the replay epilogue.

    python scripts/recompute_bench.py                 # no GPU needed: the byte model's predictions
    python scripts/recompute_bench.py --measure       # on an H100: measured peak bytes and step times too

For the target configurations at their per-GPU batches it prints the byte model's predicted peak with
recomputation off, with the plan `Trainer` would choose on an 80 GB card, and with every block group recomputed.
With --measure it runs, for each configuration and each of off / auto / all whose predicted peak fits the card,
one eager step for `torch.cuda.max_memory_allocated` and the captured step's time over --steps replays; a
configuration predicted not to fit is reported as not run rather than run out of memory.  It then times the replay
of the ResNet-50 blocks (every block group, --replay_views views of 224x224) with the fused conv + BatchNorm
epilogue (`simclr_conv2d_fprop_tc_apply`) and with conv followed by the BatchNorm apply kernel.  The card's name and
power limit are printed with the numbers.
"""
import argparse
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# (name, resnet_depth, width_multiplier, sk_ratio, samples per GPU): SURVEY 8d at their global batches on 8 GPUs
CONFIGS = [('cfg2 R50 1x', 50, 1, 0.0, 256), ('cfg3 R50 1x', 50, 1, 0.0, 512), ('cfg4 R50 2x', 50, 2, 0.0, 512),
           ('cfg5 R152 2x SK', 152, 2, 0.0625, 256)]
CARD = 80e9


def predictions():
    from simclr_b200 import memory
    rows = []
    for name, depth, wm, sk, b in CONFIGS:
        m = memory.step_model(depth, wm, b, 224, sk_ratio=sk)
        p = memory.plan(m, CARD)
        rows.append((name, depth, wm, sk, b, p, memory.predicted_peak(m, set()), memory.predicted_peak(m, p),
                     memory.predicted_peak(m, {1, 2, 3, 4})))
        print('%-16s batch %3d/GPU  predicted peak: off %6.1f GiB | plan %-12s %6.1f GiB | all %6.1f GiB' % (
            name, b, memory.gib(rows[-1][6]), memory.describe(p), memory.gib(rows[-1][7]), memory.gib(rows[-1][8])))
    return rows


def card():
    import torch
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        q = torch.cuda.get_device_name(0) + ', power limit unknown'
    return q


def measure(rows, steps, only):
    import torch
    from simclr_b200 import engine, flags_def, memory, run
    total = torch.cuda.get_device_properties(0).total_memory
    for name, depth, wm, sk, b, p, off, auto, allp in rows:
        if only and name.split()[0] not in only:
            continue
        for mode, groups, pred in (('off', set(), off), ('auto', p, auto), ('all', {1, 2, 3, 4}, allp)):
            if mode == 'auto' and groups in (set(), {1, 2, 3, 4}):
                continue
            if pred > memory.USABLE_FRACTION * total:
                print('%-16s %-4s not run: predicted %.1f GiB does not fit the card' % (name, mode, memory.gib(pred)))
                continue
            flags_def.set_flags(resnet_depth=depth, width_multiplier=wm, sk_ratio=sk, image_size=224,
                                train_batch_size=b, temperature=0.1, proj_out_dim=128, optimizer='lars',
                                b200_precision='bf16', b200_conv_engine='tc')
            engine.set_engine(engine.Engine(precision='bf16', conv_engine='tc'))
            trainer = run.Trainer(num_classes=1000, num_examples=1281167, seed=0, recompute=groups)
            f, lab = run.synthetic_batch(b, 224, 1000, 'cuda', 0)
            trainer.single_step(f, lab)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            trainer.single_step(f, lab)
            torch.cuda.synchronize()
            peak = torch.cuda.max_memory_allocated()
            torch.cuda.empty_cache()          # the captured graph gets its own pool
            trainer.capture(f, lab, warmup=1)
            trainer.replay()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                trainer.replay()
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / steps
            print('%-16s %-4s %-12s peak allocated %6.2f GiB (predicted %6.2f)  step %7.1f ms  %6.0f img/s' % (
                name, mode, memory.describe(groups), memory.gib(peak), memory.gib(pred), ms, b / ms * 1e3))
            del trainer, f, lab
            torch.cuda.empty_cache()


def replay_time(views, reps):
    """Time of replaying every ResNet-50 block (all four groups) with the fused epilogue and without it."""
    import torch
    from simclr_b200 import engine, flags_def, resnet
    from simclr_b200.model import Model
    flags_def.set_flags(resnet_depth=50, width_multiplier=1, sk_ratio=0.0, image_size=224, train_batch_size=views // 2,
                        b200_precision='bf16', b200_conv_engine='tc')
    e = engine.set_engine(engine.Engine(precision='bf16', conv_engine='tc'))
    model = Model(1000)
    net = model.resnet_model
    net.recompute = {1, 2, 3, 4}
    f = torch.rand(views // 2, 224, 224, 6, device='cuda')
    e.begin_step(model.vs.flat_grad)
    model(f, training=True)
    e.end_step()
    blocks = [b for g in net.block_groups for b in g.layers]
    inputs = [b.replay_input for b in blocks]
    fused = resnet.BatchNormRelu.replay_apply

    def unfused(bn, op, x):                      # conv, then the BatchNorm apply kernel with the kept coefficients
        return bn(op.forward(x, True), True)

    def run_all():
        for b, x in zip(blocks, inputs):
            b.replay_input = x
            b.replay()
    res = {}
    for _ in range(2):                           # alternate the two arms
        for arm, fn in (('fused', fused), ('conv+apply', unfused)):
            resnet.BatchNormRelu.replay_apply = fn
            run_all()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                run_all()
            e1.record()
            torch.cuda.synchronize()
            res.setdefault(arm, []).append(e0.elapsed_time(e1) / reps)
    resnet.BatchNormRelu.replay_apply = fused
    for arm, t in res.items():
        print('replay of the 16 ResNet-50 blocks, %d views: %-10s %.2f ms (runs: %s)' % (
            views, arm, min(t), ', '.join('%.2f' % x for x in t)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--measure', action='store_true', help='measure on the GPU (an H100)')
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--only', default='', help='comma-separated configuration names (cfg2,cfg3,...) to measure')
    ap.add_argument('--replay_views', type=int, default=512)
    ap.add_argument('--replay_reps', type=int, default=10)
    args = ap.parse_args()
    rows = predictions()
    if not args.measure:
        return
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('--measure needs a GPU')
    from simclr_b200 import flags_def
    flags_def.set_flags(use_blur=True)
    print('card: %s' % card())
    t0 = time.time()
    measure(rows, args.steps, [s for s in args.only.split(',') if s])
    replay_time(args.replay_views, args.replay_reps)
    print('wall %.0f s' % (time.time() - t0))


if __name__ == '__main__':
    main()
