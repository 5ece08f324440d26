"""Per-layer operand feed of the wgmma conv kernels on the ResNet-50 shapes, with and without 2-CTA TMA multicast.

For every conv shape of scripts/layer_bench.py (fprop / dgrad / wgrad at --views images) it times the call with the
L2 flushed and prints TF/s and the operand bytes the kernels stream into shared memory per SM clock:
(A + B stage bytes) x stages / time / SMs / max SM clock.  That is the L2 -> SM feed the tensor pipe needs without
multicast; with multicast each CTA of a pair reads half of the shared tile from L2.  Halo and stem layers run other
kernels and show no byte figure.  The card's name, power limit and maximum SM clock are read in the same run.

Usage: python scripts/multicast_bench.py [--views 512] [--arms 0,1] [--reps 5] [--out file.json]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from simclr_b200._lib import lib, stream_ptr

# (Hin, Cin, Cout, k, stride, count): the ResNet-50 conv shapes of layer_bench.py
R50 = [(224, 3, 64, 7, 2, 1), (56, 64, 256, 1, 1, 4), (56, 64, 64, 1, 1, 1), (56, 64, 64, 3, 1, 3), (56, 256, 64, 1, 1, 2),
       (56, 256, 512, 1, 2, 1), (56, 256, 128, 1, 1, 1), (56, 128, 128, 3, 2, 1), (28, 128, 512, 1, 1, 4),
       (28, 512, 128, 1, 1, 3), (28, 128, 128, 3, 1, 3), (28, 512, 1024, 1, 2, 1), (28, 512, 256, 1, 1, 1),
       (28, 256, 256, 3, 2, 1), (14, 256, 1024, 1, 1, 6), (14, 1024, 256, 1, 1, 5), (14, 256, 256, 3, 1, 5),
       (14, 1024, 2048, 1, 2, 1), (14, 1024, 512, 1, 1, 1), (14, 512, 512, 3, 2, 1), (7, 512, 2048, 1, 1, 3),
       (7, 2048, 512, 1, 1, 2), (7, 512, 512, 3, 1, 2)]

A_STAGE = 128 * 128


def cdiv(a, b):
    return (a + b - 1) // b


def bn_of(n):
    return 128 if n > 64 else 64


def gemm_bytes(M, n_out, num_kb):
    bn = bn_of(n_out)
    return cdiv(M, 128) * cdiv(n_out, bn) * num_kb * (A_STAGE + bn * 128)


def operand_bytes(kind, N, H, Cin, Cout, k, s):
    """Bytes the implicit-GEMM / weight-gradient kernel streams into shared memory, or (None, path) for the
    layers that other kernels take (stem, halo 3x3)."""
    Ho = (H - 1) // s + 1
    if Cin == 3:
        return None, 'stem'
    halo = k == 3 and s == 1 and H + 2 <= 64
    if kind == 'fprop':
        if halo and Cin == Cout and Cin in (64, 128):
            return None, 'halo'
        return gemm_bytes(N * Ho * Ho, Cout, cdiv(k * k * Cin, 64)), 'igemm'
    if kind == 'dgrad':
        if s == 1:
            if halo and Cin == Cout and Cin in (64, 128):
                return None, 'halo'
            return gemm_bytes(N * H * H, Cin, cdiv(k * k * Cout, 64)), 'igemm'
        pad, tot = (k - 1) // 2, 0
        for ph in range(s):
            taps_h = sum(1 for r in range(k) if (ph + pad - r) % s == 0)
            for pw in range(s):
                nt = taps_h * sum(1 for r in range(k) if (pw + pad - r) % s == 0)
                P2, Q2 = cdiv(H - ph, s), cdiv(H - pw, s)
                if nt and P2 > 0 and Q2 > 0:
                    tot += gemm_bytes(N * P2 * Q2, Cin, nt * (Cout // 64))
        return tot, 'igemm parity classes'
    if halo and Cin == Cout == 64:
        return None, 'halo'
    bn = bn_of(Cout)
    return cdiv(k * k * Cin, 128) * cdiv(Cout, bn) * cdiv(N * Ho * Ho, 64) * (A_STAGE + bn * 128), 'wgrad'


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader,nounits'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    name, plim, clk = [v.strip() for v in q[0].split(',')]
    return dict(name=name, power_limit_w=float(plim), max_sm_clock_mhz=float(clk),
                sms=torch.cuda.get_device_properties(0).multi_processor_count)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--views', type=int, default=512)
    ap.add_argument('--only', default='fprop,dgrad,wgrad')
    ap.add_argument('--arms', default=None, help='multicast settings to time, e.g. 0,1 (default: 0,1 when the library has the switch)')
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    has_switch = 'simclr_set_tc_multicast' in lib.declarations
    arms = [int(a) for a in (args.arms or ('0,1' if has_switch else '0')).split(',')]
    if arms != [0] and not has_switch:
        sys.exit('this library has no multicast switch')
    kinds = args.only.split(',')
    info = card()
    if has_switch:
        info['max_active_clusters'] = {c: lib.tc_max_active_clusters(c) for c in (2, 4)}
    print(json.dumps(info), flush=True)
    clk_hz = info['max_sm_clock_mhz'] * 1e6
    N, st = args.views, stream_ptr()
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device='cuda')
    rows, tot = [], {(k, a): [0.0, 0.0] for k in kinds for a in arms}
    prev = lib.set_tc_multicast(1) if has_switch else None
    try:
        for idx, (H, Cin, Cout, k, s, cnt) in enumerate(R50):
            Cs = 4 if Cin == 3 else Cin
            Ho = (H - 1) // s + 1
            x = torch.randn(N, H, H, Cs, device='cuda').to(torch.bfloat16)
            dy = torch.randn(N, Ho, Ho, Cout, device='cuda').to(torch.bfloat16)
            w = torch.randn(k, k, Cin, Cout, device='cuda') * 0.05
            K = k * (k + 1 if Cs == 4 else k) * Cs
            Kp, Kd = cdiv(K, 64) * 64, cdiv(k * k * Cout, 64) * 64
            wf = torch.empty(Cout, Kp, dtype=torch.bfloat16, device='cuda')
            wd = torch.empty(Cin, Kd, dtype=torch.bfloat16, device='cuda') if Cs == Cin else None
            lib.pack_conv_weight(w, wf, wd, 1, k, k, Cin, Cs, Cout, Kp, st)
            y = torch.empty(N, Ho, Ho, Cout, dtype=torch.bfloat16, device='cuda')
            dx = torch.empty(N, H, H, Cin, dtype=torch.bfloat16, device='cuda')
            dw = torch.empty(k, k, Cin, Cout, device='cuda')
            sums = torch.empty(2 * Cout, dtype=torch.float64, device='cuda')
            flops = 2.0 * N * Ho * Ho * k * k * Cin * Cout
            ops = {'fprop': lambda: lib.conv2d_fprop_tc(x, wf, y, 1, 1, N, H, H, Cs, Cout, k, k, s, sums, st),
                   'dgrad': (lambda: lib.conv2d_dgrad_tc(dy, wd, dx, 1, 1, N, H, H, Cin, Cout, k, k, s, st)) if wd is not None else None,
                   'wgrad': lambda: lib.conv2d_wgrad_tc(x, dy, dw, 1, N, H, H, Cs, Cin, Cout, k, k, s, st)}
            for kind in kinds:
                fn = ops[kind]
                if fn is None:
                    continue
                nbytes, path = operand_bytes(kind, N, H, Cin, Cout, k, s)
                best = {}
                for arm in arms:                      # the arms alternate inside each repetition
                    if has_switch:
                        lib.set_tc_multicast(arm)
                    fn(); fn(); torch.cuda.synchronize()
                    best[arm] = 1e9
                for _ in range(args.reps):
                    for arm in arms:
                        if has_switch:
                            lib.set_tc_multicast(arm)
                        flush.zero_()
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
                        best[arm] = min(best[arm], e0.elapsed_time(e1))
                line = '%2d %-5s H%3d %4d->%4d k%d s%d x%d %-20s' % (idx, kind, H, Cin, Cout, k, s, cnt, path)
                for arm in arms:
                    ms = best[arm]
                    bpc = None if nbytes is None else nbytes / (ms * 1e-3) / info['sms'] / clk_hz
                    rows.append(dict(idx=idx, kind=kind, H=H, Cin=Cin, Cout=Cout, k=k, s=s, count=cnt, path=path,
                                     multicast=arm, ms=ms, tflops=flops / ms / 1e9, operand_bytes=nbytes,
                                     bytes_per_sm_clk=bpc))
                    tot[(kind, arm)][0] += flops * cnt
                    tot[(kind, arm)][1] += ms * cnt
                    line += ' | mc%d %8.3f ms %6.1f TF/s %s' % (arm, ms, flops / ms / 1e9,
                                                                '   -   B/clk' if bpc is None else '%5.1f B/clk' % bpc)
                if len(arms) == 2:
                    line += ' | %+5.1f%%' % (100.0 * (best[arms[0]] / best[arms[1]] - 1.0))
                print(line, flush=True)
            del x, dy, y, dx
    finally:
        if has_switch:
            lib.set_tc_multicast(prev)
    for (kind, arm), (fl, ms) in tot.items():
        if ms > 0:
            print('TOTAL %-5s mc%d (x count, %d views): %8.2f ms  %7.1f TF/s' % (kind, arm, N, ms, fl / ms / 1e9))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        json.dump(dict(card=info, rows=rows), open(args.out, 'w'), indent=0)


if __name__ == '__main__':
    main()
