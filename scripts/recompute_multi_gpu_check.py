"""Run under torchrun with N ranks: the sharded pretrain step with every block group recomputed equals the same
step storing its activations, bit for bit on every rank, through the peer-memory SyncBN -- eagerly and as the
segmented CUDA-graph replay (groups 3-4 replay inside the first graph, groups 1-2 inside the second).  ResNet-50
exercises the bottleneck blocks and the fused projection tails.  Prints RECOMPUTE_MULTI_GPU_CHECK {json} on rank 0."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import torch.distributed as dist
from simclr_b200 import engine, run, flags_def

flags_def.FLAGS(['recompute_multi'])
rank = run.init_distributed()
R = dist.get_world_size()
B, S = 8, 64
flags_def.set_flags(resnet_depth=50, image_size=S, train_batch_size=B * R, use_blur=False, weight_decay=1e-4,
                    global_bn=True, b200_precision='bf16', b200_conv_engine='tc')
g = torch.Generator().manual_seed(1)
feats = [torch.rand(B, S, S, 6, generator=g) for _ in range(R)]
labs = [torch.nn.functional.one_hot(torch.randint(0, 1000, (B,), generator=g), 1000).float() for _ in range(R)]


def state(recompute, graph):
    engine.set_engine(engine.Engine(precision='bf16', conv_engine='tc'))
    trainer = run.Trainer(num_classes=1000, num_examples=50000, seed=0, recompute=recompute)
    gen = torch.Generator().manual_seed(3)
    for v in trainer.model.vs.trainable:
        if v.name.endswith('gamma:0'):
            v.value.copy_(0.5 + torch.rand(v.shape, generator=gen))
    trainer.optimizer.learning_rate = 0.3
    f, lab = feats[rank].cuda(), labs[rank].cuda()
    if graph:
        trainer.capture(f, lab, warmup=1)
        trainer.replay()
        loss = trainer.replay()
    else:
        loss = trainer.single_step(f, lab)
    torch.cuda.synchronize()
    vs = trainer.model.vs
    out = [loss.detach().reshape(1).clone(), vs.flat_grad.clone(), vs.flat_value.clone(), vs.flat_moving.clone(),
           trainer.optimizer._flat_v.clone()]
    del trainer
    return out


res = {}
for graph in (False, True):
    ref, got = state(set(), graph), state({1, 2, 3, 4}, graph)
    same = all(torch.equal(a, b) for a, b in zip(ref, got))
    t = torch.tensor([1.0 if same else 0.0], device='cuda')
    dist.all_reduce(t, op=dist.ReduceOp.MIN)
    res['graph' if graph else 'eager'] = bool(t.item() == 1.0)
res['ok'] = all(res.values())
if rank == 0:
    print('RECOMPUTE_MULTI_GPU_CHECK ' + json.dumps(res), flush=True)
dist.barrier()
dist.destroy_process_group()
sys.exit(0 if res['ok'] else 1)
