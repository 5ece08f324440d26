"""Speed of the BatchNorm-folded inference forward (--b200_fold_bn) on one GPU: the same workload with and without
folding, bf16 tensor-core engine, CUDA-graph replay timed with CUDA events, seeded random weights (speed does not
depend on them).  One JSON line per case with both times; the card name and power limit are read in the same run.

Cases:
  eval_r50_b<B>   evaluation forward model(features, training=False), R50 1x at 224x224, B images
  lineval_r50     linear-evaluation step: train_mode=finetune, fine_tune_after_block=4 (frozen backbone), R50 1x
  distill_r152x2sk  distillation step: R152 2x SK teacher, R50 1x student

The folded and unfolded graphs of a case are replayed alternately, `--rounds` times each, and the medians are
reported.

    python scripts/fold_bench.py [--cases eval_r50_b256,eval_r50_b1024,lineval_r50,distill_r152x2sk] [--steps 10]
"""
import argparse
import gc
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_info():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else 'unknown (nvidia-smi failed)'


def _time(fn, steps):
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    ev0.record()
    for _ in range(steps):
        fn()
    ev1.record()
    torch.cuda.synchronize()
    return ev0.elapsed_time(ev1) / steps


def _free():
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _flags(**kw):
    from simclr_b200 import flags_def
    vals = dict(resnet_depth=50, width_multiplier=1, sk_ratio=0.0, se_ratio=0.0, image_size=224, use_blur=False,
                train_mode='finetune', fine_tune_after_block=-1, ft_proj_selector=0, lineareval_while_pretraining=False,
                optimizer='lars', warmup_epochs=0, train_steps=10 ** 6, b200_precision='bf16', b200_conv_engine='tc',
                b200_fold_bn=False)
    vals.update(kw)
    flags_def.set_flags(**vals)


def _graph(fn, warmup):
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(warmup):
            fn()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        fn()
    return graph


def _ab(replays, steps, rounds):
    """Alternating timed windows of the unfolded and folded replays; medians in ms."""
    times = {k: [] for k in replays}
    for _ in range(rounds):
        for k, fn in replays.items():
            times[k].append(_time(fn, steps))
    return {k + '_ms': statistics.median(v) for k, v in times.items()}


def eval_case(batch, steps, warmup, rounds):
    from simclr_b200 import engine, flags_def, run
    _flags(train_batch_size=batch)
    engine.set_engine(engine.Engine(precision='bf16', conv_engine='tc'))
    trainer = run.Trainer(num_classes=1000, num_examples=1281167, seed=0)
    g = torch.Generator(device='cuda').manual_seed(0)
    features = torch.rand(batch, 224, 224, 3, device='cuda', generator=g)
    graphs = {}
    for fold in (False, True):
        flags_def.FLAGS.b200_fold_bn = fold
        graphs['folded' if fold else 'unfolded'] = _graph(lambda: trainer.model(features, training=False), warmup)
    flags_def.FLAGS.b200_fold_bn = False
    out = {'case': 'eval_r50_b%d' % batch, 'model': 'R50 1x', 'batch': batch, 'image_size': 224, 'steps': steps}
    out.update(_ab({k: v.replay for k, v in graphs.items()}, steps, rounds))
    del trainer, graphs
    _free()
    return out


def step_case(name, batch, steps, warmup, rounds):
    """A training step whose inference-mode part is folded or not: linear evaluation (frozen backbone) or
    distillation (the teacher)."""
    from simclr_b200 import engine, run, distill
    g = torch.Generator(device='cuda').manual_seed(0)
    features = torch.rand(batch, 224, 224, 3, device='cuda', generator=g)
    labels = torch.nn.functional.one_hot(torch.randint(0, 1000, (batch,), device='cuda', generator=g), 1000).float()
    replays, keep = {}, []
    for fold in (False, True):
        if name == 'lineval_r50':
            _flags(train_batch_size=batch, fine_tune_after_block=4, b200_fold_bn=fold)
        else:
            _flags(train_batch_size=batch, b200_fold_bn=fold, b200_distill_temperature=1.0,
                   b200_teacher_resnet_depth=152, b200_teacher_width_multiplier=2, b200_teacher_sk_ratio=0.0625)
        engine.set_engine(engine.Engine(precision='bf16', conv_engine='tc'))
        teacher = distill.Teacher(None, num_classes=1000, seed=1) if name != 'lineval_r50' else None
        trainer = run.Trainer(num_classes=1000, num_examples=1281167, seed=0, teacher=teacher, recompute=set())
        trainer.capture(features, labels, warmup=warmup)
        replays['folded' if fold else 'unfolded'] = trainer.replay
        keep.append((trainer, teacher))
    out = {'case': name, 'batch': batch, 'image_size': 224, 'steps': steps,
           'model': 'R50 1x, fine_tune_after_block=4' if name == 'lineval_r50' else 'teacher R152 2x SK, student R50 1x'}
    out.update(_ab(replays, steps, rounds))
    del keep, replays
    _free()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--cases', default='eval_r50_b256,eval_r50_b1024,lineval_r50,distill_r152x2sk')
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--lineval_batch', type=int, default=512)
    ap.add_argument('--distill_batch', type=int, default=128)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('fold_bench needs a CUDA device (H100)')
    from simclr_b200 import flags_def
    flags_def.set_flags()
    gpu = gpu_info()
    print(json.dumps({'gpu': gpu}), flush=True)
    for case in args.cases.split(','):
        if case.startswith('eval_r50_b'):
            r = eval_case(int(case[len('eval_r50_b'):]), args.steps, args.warmup, args.rounds)
        elif case == 'lineval_r50':
            r = step_case(case, args.lineval_batch, args.steps, args.warmup, args.rounds)
        elif case == 'distill_r152x2sk':
            r = step_case(case, args.distill_batch, args.steps, args.warmup, args.rounds)
        else:
            raise SystemExit('unknown case %r' % case)
        r['speedup'] = r['unfolded_ms'] / r['folded_ms']
        r['gpu'] = gpu
        print(json.dumps(r), flush=True)


if __name__ == '__main__':
    main()
