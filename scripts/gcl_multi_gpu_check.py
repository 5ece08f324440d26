"""Run under torchrun with N ranks: one sharded fp32 / simt pretraining step with the generalized contrastive loss
(`python -m torch.distributed.run --nproc-per-node 2 scripts/gcl_multi_gpu_check.py <logsumexp|normal|uniform>`),
checked on rank 0 against the oracle's N-replica simulation (`oracle.gcl.gcl_loss_replicas`) of the same global batch
with the draws of the step, at the tolerances of scripts/multi_gpu_check.py; every rank must end with the same
weights.  The collectives are the peer-memory kernels, or NCCL with SIMCLR_COMM=nccl."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402
from util import rel_err, cfg_from_flags, structured_batch  # noqa: E402
from simclr_b200 import engine, run, flags_def  # noqa: E402
from oracle import model as OM, step as OS, gcl as OG  # noqa: E402

gcl_dist = sys.argv[1] if len(sys.argv) > 1 else 'normal'
flags_def.FLAGS(['gcl_multi'])
rank = run.init_distributed()
R = dist.get_world_size()
B, S, lam, ls = 16, 64, 0.5, 2.0
flags_def.set_flags(resnet_depth=18, image_size=S, train_batch_size=B * R, use_blur=False, weight_decay=1e-4,
                    temperature=0.5, b200_precision='fp32', b200_conv_engine='simt', b200_gcl_dist=gcl_dist,
                    b200_gcl_lambda=lam, b200_gcl_loss_scaling=ls)
engine.set_engine(engine.Engine(precision='fp32', conv_engine='simt'))
trainer = run.Trainer(num_classes=1000, num_examples=50000, seed=0)
f, lab = structured_batch(B * R, S, seed=1)
feats = [f[r * B:(r + 1) * B] for r in range(R)]
labs = [lab[r * B:(r + 1) * B] for r in range(R)]
trainer.optimizer.learning_rate = 0.3
loss = trainer.single_step(feats[rank].cuda(), labs[rank].cuda())
torch.cuda.synchronize()
lt = loss.detach().clone().reshape(1)
dist.all_reduce(lt)
W_dev, P_dev = trainer.metrics['gcl_draws']
W = None if W_dev is None else W_dev.double().cpu()
P = None if P_dev is None else P_dev.double().cpu()
ok = True
if rank == 0:
    def loss_replicas(proj, hidden_norm, temperature):
        dt = proj[0].dtype
        outs = OG.gcl_loss_replicas(proj, lam, temperature, gcl_dist, hidden_norm, ls,
                                    None if W is None else W.to(dt), None if P is None else P.to(dt))
        return [(o[0], o[1], o[2]) for o in outs]

    OS.obj_lib.contrastive_loss_replicas = loss_replicas
    om = OM.Model(cfg_from_flags(flags_def.FLAGS), 1000)
    Pm, S_ = om.init(0)
    info = OS.forward_backward(om, Pm, S_, feats, labs)
    job_loss = float(lt.item()) / R
    res = {'world': R, 'dist': gcl_dist, 'collectives': 'peer' if trainer.strategy.comm is not None else 'nccl',
           'loss': job_loss, 'oracle_loss': float(info['loss'])}
    worst, wname = 0.0, ''
    for v in trainer.model.trainable_variables:
        ref = info['grads'][v.name]
        err = rel_err(v.grad, ref)
        if ref.norm() == 0:
            ok = ok and err < 1e-6
        elif err > worst:
            worst, wname = err, v.name
    res['worst_grad_rel_err'] = worst
    res['worst_name'] = wname
    ok = ok and worst < 1e-3 and abs(job_loss - res['oracle_loss']) < 1e-4 * abs(res['oracle_loss'])
    res['ok'] = bool(ok)
    print('GCL_MULTI_GPU_CHECK ' + json.dumps(res), flush=True)
# the draws and, after the LARS step, the weights are the same on every rank
same = True
for t in [trainer.model.vs.flat_value] + ([W_dev, P_dev] if W_dev is not None else []):
    t0 = t.clone()
    dist.broadcast(t0, 0)
    same = same and bool(torch.equal(t, t0))
flag = torch.tensor([1.0 if same else 0.0], device='cuda')
dist.all_reduce(flag, op=dist.ReduceOp.MIN)
if rank == 0:
    print('GCL_MULTI_GPU_IDENTICAL %d' % int(flag.item()), flush=True)
    ok = ok and flag.item() == 1.0
dist.barrier()
dist.destroy_process_group()
sys.exit(0 if ok else 1)
