"""Cost of the generalized contrastive loss on one GPU.

Reports, with the card name and power limit read in the same run:
  - the loss forward + backward (objective.*_forward / *_backward, CUDA events) of NT-Xent and of each
    --b200_gcl_dist, at 2B = 1024 local rows and D = 128, for one replica and for 8 replicas simulated by a
    pre-filled gathered z (and lse): the kernels then see a global batch of 2G = 8192 rows;
  - the captured ResNet-50 pretraining step (bf16 tc, LARS, batch 256 at 224x224, seeded random weights) in
    images/s with NT-Xent and with each dist.

    python scripts/gcl_bench.py [--iters 50] [--steps 20] [--batch 256] [--image_size 224] [--no_step]
"""
import argparse
import gc
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from distill_bench import gpu_info, _time  # noqa: E402

DISTS = ('ntxent', 'logsumexp', 'normal', 'uniform')


class PrefilledGather:
    """Replica 0 of R: all_gather places this replica's tensor in front of fixed contents of the other replicas."""

    def __init__(self, R, fill):
        self.num_replicas_in_sync, self.replica_id, self.fill = R, 0, fill

    def all_gather(self, t, channel=None):
        out = self.fill[channel]
        out[0].copy_(t)
        return out


def loss_time(dist, R, B, D, iters):
    from simclr_b200 import objective as obj
    g = torch.Generator(device='cuda').manual_seed(0)
    hidden = torch.randn(2 * B, D, device='cuda', generator=g)
    fill = {'z': torch.nn.functional.normalize(torch.randn(R, 2 * B, D, device='cuda', generator=g), dim=-1),
            'lse': torch.full((R, 2 * B), 5.0, device='cuda')}
    st = PrefilledGather(R, fill) if R > 1 else None
    if dist == 'ntxent':
        def fn():
            *_, ctx = obj.contrastive_forward(hidden, True, 0.1, st, want_labels=False)
            obj.contrastive_backward(ctx, 1.0 / (B * R))
    else:
        step = torch.zeros(1, dtype=torch.int64, device='cuda')

        def fn():
            *_, ctx = obj.generalized_contrastive_forward(hidden, dist, 1.0, 0.1, True, 1.0, st, step=step)
            obj.generalized_contrastive_backward(ctx, 1.0 / R)
    for _ in range(3):
        fn()
    return _time(fn, iters)


def step_rate(dist, batch, image_size, steps, warmup):
    from simclr_b200 import engine, flags_def, run
    flags_def.set_flags(resnet_depth=50, width_multiplier=1, sk_ratio=0.0, se_ratio=0.0, image_size=image_size,
                        train_batch_size=batch, train_mode='pretrain', optimizer='lars', use_blur=False,
                        warmup_epochs=0, train_steps=10 ** 6, b200_precision='bf16', b200_conv_engine='tc',
                        b200_gcl_dist='none' if dist == 'ntxent' else dist)
    engine.set_engine(engine.Engine(precision='bf16', conv_engine='tc'))
    features, labels = run.synthetic_batch(batch, image_size, 1000, 'cuda', 0)
    trainer = run.Trainer(num_classes=1000, num_examples=1281167, seed=0)
    trainer.capture(features, labels, warmup=warmup)
    ms = _time(trainer.replay, steps)
    loss = float(trainer._graph_loss)
    del trainer
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return ms, loss


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--batch', type=int, default=256)
    ap.add_argument('--image_size', type=int, default=224)
    ap.add_argument('--no_step', action='store_true')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('gcl_bench needs a CUDA device (H100)')
    from simclr_b200 import engine, flags_def
    flags_def.set_flags()
    gpu = gpu_info()
    print(json.dumps({'gpu': gpu}), flush=True)
    engine.set_engine(engine.Engine(precision='fp32', conv_engine='simt'))
    B, D = 512, 128
    for R in (1, 8):
        for dist in DISTS:
            ms = loss_time(dist, R, B, D, args.iters)
            print(json.dumps({'what': 'loss fwd+bwd', 'dist': dist, 'local_rows': 2 * B, 'global_rows': 2 * B * R,
                              'D': D, 'ms': round(ms, 4), 'gpu': gpu}), flush=True)
    if args.no_step:
        return
    base = None
    for dist in DISTS:
        ms, loss = step_rate(dist, args.batch, args.image_size, args.steps, args.warmup)
        base = base or ms
        print(json.dumps({'what': 'R50 pretraining step (graph replay)', 'dist': dist, 'batch': args.batch,
                          'image_size': args.image_size, 'ms': round(ms, 3), 'img_s': round(args.batch / ms * 1e3, 1),
                          'vs_ntxent': round(ms / base, 4), 'loss': loss, 'gpu': gpu}), flush=True)
    flags_def.set_flags(b200_gcl_dist='none')


if __name__ == '__main__':
    main()
