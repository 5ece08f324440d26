"""Per-layer timing of the wgmma engine on the ResNet-50 conv shapes (SURVEY 10.1).
Usage: python scripts/layer_bench.py [--views 256] [--only fprop,dgrad,wgrad] [--out file]"""
import argparse, os, sys, json
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from simclr_b200._lib import lib, stream_ptr

# (Hin, Cin, Cout, k, stride, count)
R50 = [(224, 3, 64, 7, 2, 1), (56, 64, 256, 1, 1, 4), (56, 64, 64, 1, 1, 1), (56, 64, 64, 3, 1, 3), (56, 256, 64, 1, 1, 2),
       (56, 256, 512, 1, 2, 1), (56, 256, 128, 1, 1, 1), (56, 128, 128, 3, 2, 1), (28, 128, 512, 1, 1, 4),
       (28, 512, 128, 1, 1, 3), (28, 128, 128, 3, 1, 3), (28, 512, 1024, 1, 2, 1), (28, 512, 256, 1, 1, 1),
       (28, 256, 256, 3, 2, 1), (14, 256, 1024, 1, 1, 6), (14, 1024, 256, 1, 1, 5), (14, 256, 256, 3, 1, 5),
       (14, 1024, 2048, 1, 2, 1), (14, 1024, 512, 1, 1, 1), (14, 512, 512, 3, 2, 1), (7, 512, 2048, 1, 1, 3),
       (7, 2048, 512, 1, 1, 2), (7, 512, 512, 3, 1, 2)]

ap = argparse.ArgumentParser()
ap.add_argument('--views', type=int, default=256)
ap.add_argument('--only', default='fprop,dgrad,wgrad')
ap.add_argument('--reps', type=int, default=3)
ap.add_argument('--out', default=None)
ap.add_argument('--layers', default=None, help='comma separated indices into the shape list')
ap.add_argument('--fused_stats', action='store_true', help='fprop with BN statistics fused into the epilogue')
args = ap.parse_args()
kinds = args.only.split(',')
sel = range(len(R50)) if args.layers is None else [int(i) for i in args.layers.split(',')]
N = args.views
st = stream_ptr()
rows = []
tot = {k: [0.0, 0.0] for k in kinds}
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device='cuda')
for idx in sel:
    H, Cin, Cout, k, s, cnt = R50[idx]
    Cs = 4 if Cin == 3 else Cin
    Ho = (H - 1) // s + 1
    x = torch.randn(N, H, H, Cs, device='cuda').to(torch.bfloat16)
    dy = torch.randn(N, Ho, Ho, Cout, device='cuda').to(torch.bfloat16)
    w = torch.randn(k, k, Cin, Cout, device='cuda') * 0.05
    K = k * (k + 1 if Cs == 4 else k) * Cs; Kp = (K + 63) // 64 * 64; Kd = (k * k * Cout + 63) // 64 * 64
    wf = torch.empty(Cout, Kp, dtype=torch.bfloat16, device='cuda')
    wd = torch.empty(Cin, Kd, dtype=torch.bfloat16, device='cuda') if Cs == Cin else None
    lib.pack_conv_weight(w, wf, wd, 1, k, k, Cin, Cs, Cout, Kp, st)
    y = torch.empty(N, Ho, Ho, Cout, dtype=torch.bfloat16, device='cuda')
    dx = torch.empty(N, H, H, Cin, dtype=torch.bfloat16, device='cuda')
    dw = torch.empty(k, k, Cin, Cout, device='cuda')
    sums = torch.empty(2 * Cout, dtype=torch.float64, device='cuda')
    M = N * Ho * Ho
    flops = 2.0 * M * k * k * Cin * Cout
    ops = {'fprop': lambda: lib.conv2d_fprop_tc(x, wf, y, 1, 1, N, H, H, Cs, Cout, k, k, s, sums if args.fused_stats else None, st),
           'dgrad': (lambda: lib.conv2d_dgrad_tc(dy, wd, dx, 1, 1, N, H, H, Cin, Cout, k, k, s, st)) if wd is not None else None,
           'wgrad': lambda: lib.conv2d_wgrad_tc(x, dy, dw, 1, N, H, H, Cs, Cin, Cout, k, k, s, st)}
    minbytes = {'fprop': (x.numel() + y.numel()) * 2, 'dgrad': (dy.numel() + dx.numel()) * 2, 'wgrad': (x.numel() + dy.numel()) * 2}
    for kind in kinds:
        fn = ops[kind]
        if fn is None:
            continue
        fn(); torch.cuda.synchronize()
        best = 1e9
        for _ in range(args.reps):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); fn(); e1.record(); torch.cuda.synchronize()
            best = min(best, e0.elapsed_time(e1))
        tf = flops / best / 1e9
        gbs = minbytes[kind] / best / 1e6
        rows.append(dict(idx=idx, kind=kind, H=H, Cin=Cin, Cout=Cout, k=k, s=s, count=cnt, M=M, ms=best, tflops=tf, gbs=gbs))
        tot[kind][0] += flops * cnt; tot[kind][1] += best * cnt
        print('%2d %-5s H%3d %4d->%4d k%d s%d x%d  M=%8d  %8.3f ms  %7.1f TF/s  %7.0f GB/s(min traffic)' % (idx, kind, H, Cin, Cout, k, s, cnt, M, best, tf, gbs), flush=True)
    del x, dy, y, dx
for kind in kinds:
    if tot[kind][1] > 0:
        print('TOTAL %-5s (x count, %d views): %8.2f ms  %7.1f TF/s' % (kind, N, tot[kind][1], tot[kind][0] / tot[kind][1] / 1e9))
if args.out:
    json.dump(rows, open(args.out, 'w'), indent=0)
