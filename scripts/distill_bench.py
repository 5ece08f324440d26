"""Speed of SimCLRv2 distillation on one GPU: bf16 tensor-core engine, CUDA-graph replay, seeded random weights
(speed does not depend on them).

For each teacher -> student pair it reports, at the same batch and image size:
  - the distillation step (teacher forward + student forward/backward + LARS) in images/s,
  - the teacher forward alone in ms per step,
  - a plain fine-tuning step of the student (no teacher) in images/s,
  - peak device memory of the distillation run.
The card name and power limit are read in the same run and printed with the numbers.

    python scripts/distill_bench.py [--batch 256] [--image_size 224] [--steps 20] [--pairs r50,r152x2sk]
"""
import argparse
import gc
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PAIRS = {
    # name: (teacher depth, width, sk_ratio), student R50 1x
    'r50': (50, 1, 0.0),
    'r152x2sk': (152, 2, 0.0625),
}


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


def run_pair(name, batch, image_size, steps, warmup):
    from simclr_b200 import engine, flags_def, run, distill
    depth, width, sk = PAIRS[name]
    flags_def.set_flags(resnet_depth=50, width_multiplier=1, sk_ratio=0.0, se_ratio=0.0, image_size=image_size,
                        train_batch_size=batch, train_mode='finetune', fine_tune_after_block=-1, ft_proj_selector=0,
                        lineareval_while_pretraining=False, optimizer='lars', use_blur=False, warmup_epochs=0,
                        train_steps=10 ** 6, b200_precision='bf16', b200_conv_engine='tc',
                        b200_distill_temperature=1.0, b200_teacher_resnet_depth=depth,
                        b200_teacher_width_multiplier=width, b200_teacher_sk_ratio=sk)
    engine.set_engine(engine.Engine(precision='bf16', conv_engine='tc'))
    g = torch.Generator(device='cuda').manual_seed(0)
    features = torch.rand(batch, image_size, image_size, 3, device='cuda', generator=g)
    labels = torch.nn.functional.one_hot(torch.randint(0, 1000, (batch,), device='cuda', generator=g), 1000).float()
    out = {'pair': name, 'teacher': 'R%d %dx%s' % (depth, width, ' SK' if sk else ''), 'student': 'R50 1x',
           'batch': batch, 'image_size': image_size, 'steps': steps}

    # plain fine-tuning step of the student
    trainer = run.Trainer(num_classes=1000, num_examples=1281167, seed=0)
    trainer.capture(features, labels, warmup=warmup)
    out['finetune_ms'] = _time(trainer.replay, steps)
    out['finetune_img_s'] = batch / out['finetune_ms'] * 1e3
    del trainer
    engine.set_engine(engine.Engine(precision='bf16', conv_engine='tc'))
    _free()

    # distillation step
    torch.cuda.reset_peak_memory_stats()
    teacher = distill.Teacher(None, num_classes=1000, seed=1)
    trainer = run.Trainer(num_examples=1281167, seed=0, teacher=teacher)
    trainer.capture(features, labels, warmup=warmup)
    out['distill_ms'] = _time(trainer.replay, steps)
    out['distill_img_s'] = batch / out['distill_ms'] * 1e3
    out['distill_peak_mem_gb'] = torch.cuda.max_memory_allocated() / 2 ** 30
    out['distill_loss'] = float(trainer._graph_loss)
    out['teacher_params_m'] = sum(v.numel for v in teacher.variables if 'moving_' not in v.name) / 1e6

    # the teacher forward alone, captured the same way
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        teacher(features)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        teacher(features)
    out['teacher_forward_ms'] = _time(graph.replay, steps)
    out['teacher_share_of_step'] = out['teacher_forward_ms'] / out['distill_ms']
    del trainer, teacher, graph
    _free()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=256)
    ap.add_argument('--image_size', type=int, default=224)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--pairs', default='r50,r152x2sk')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('distill_bench needs a CUDA device (H100)')
    from simclr_b200 import flags_def
    flags_def.set_flags()
    gpu = gpu_info()
    print(json.dumps({'gpu': gpu}), flush=True)
    for name in args.pairs.split(','):
        r = run_pair(name, args.batch, args.image_size, args.steps, args.warmup)
        r['gpu'] = gpu
        print(json.dumps(r), flush=True)


if __name__ == '__main__':
    main()
