"""Per-kernel device time of ONE eager pretrain step, from CUPTI activity records (torch.profiler).

Unlike the ncu launch list this runs at full clocks with warm caches and back-to-back launches,
so the absolute times add up to the eager step time.  Output: kernel_times.txt (or --out)
"""
import argparse, collections, os, re, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from torch.profiler import profile, ProfilerActivity
from simclr_b200 import engine, run, flags_def

ap = argparse.ArgumentParser()
ap.add_argument('--batch', type=int, default=512)
ap.add_argument('--resnet_depth', type=int, default=50)
ap.add_argument('--image_size', type=int, default=224)
ap.add_argument('--out', default='kernel_times.txt')
args = ap.parse_args()
flags_def.FLAGS(['kernel_times'])
rank = run.init_distributed()                     # under torchrun: the N>1 step (peer-memory SyncBN, overlapped NCCL)
world = int(os.environ.get('WORLD_SIZE', '1'))
if world > 1:
    args.out = args.out.replace('.txt', '_n%d.txt' % world)
flags_def.set_flags(resnet_depth=args.resnet_depth, image_size=args.image_size, train_batch_size=args.batch,
                    b200_precision='bf16', b200_conv_engine='tc')
eng = engine.set_engine(engine.Engine(precision='bf16', conv_engine='tc'))
trainer = run.Trainer(num_classes=1000, num_examples=1281167, seed=0)
f, l = run.synthetic_batch(args.batch, args.image_size, 1000, eng.device, 1234)
for _ in range(3):
    trainer.single_step(f, l)
torch.cuda.synchronize()
if world > 1:
    torch.distributed.barrier()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    trainer.single_step(f, l)
    torch.cuda.synchronize()
if rank != 0:
    sys.exit(0)

t_first, t_last = None, None
tot = collections.defaultdict(float)
cnt = collections.Counter()
tot_full = collections.defaultdict(float)
cnt_full = collections.Counter()
for ev in prof.events():
    if ev.device_type is not None and 'cuda' in str(ev.device_type).lower() and ev.device_time_total > 0:
        name = ev.name.replace('(anonymous namespace)::', '').replace('simclr::', '')
        name = re.sub(r'^void\s+', '', name)
        full = re.sub(r'\(.*$', '', name)             # keep template arguments, drop the parameter list
        short = re.sub(r'<.*$', '', full)
        tot[short] += ev.device_time_total
        cnt[short] += 1
        try:
            t_first = ev.time_range.start if t_first is None else min(t_first, ev.time_range.start)
            t_last = ev.time_range.end if t_last is None else max(t_last, ev.time_range.end)
        except Exception:
            pass
        tot_full[full] += ev.device_time_total
        cnt_full[full] += 1
total = sum(tot.values())
os.makedirs(os.path.dirname(args.out), exist_ok=True)
with open(args.out, 'w') as fh:
    fh.write('CUPTI kernel times of one eager step on %d GPU(s), rank 0 (ResNet-%d, batch %d per GPU, %d px): total %.2f ms over %d launches\n'
             % (world, args.resnet_depth, args.batch, args.image_size, total / 1e3, sum(cnt.values())))
    if t_first is not None:
        fh.write('device span first kernel start -> last kernel end: %.2f ms\n' % ((t_last - t_first) / 1e3))
    for k, v in sorted(tot.items(), key=lambda kv: -kv[1]):
        fh.write('%-110s n=%4d %9.3f ms %5.1f%%\n' % (k[:110], cnt[k], v / 1e3, 100 * v / total))
    fh.write('\nby template instance:\n')
    for k, v in sorted(tot_full.items(), key=lambda kv: -kv[1])[:40]:
        fh.write('%-150s n=%4d %9.3f ms %5.1f%%\n' % (k[:150], cnt_full[k], v / 1e3, 100 * v / total))
print(open(args.out).read())
