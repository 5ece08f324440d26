"""Per-layer roofline reading of a scripts/layer_bench.py log: measured time against
max(tensor time at the measured bf16 peak, HBM time of the minimum traffic).

  python scripts/layer_roofline.py layers.txt [MEASURED_PEAKS.json] > layer_roofline.txt
Layer timings are kernels run alone (L2 flushed), so the burst bf16 figure is the tensor denominator."""
import json, os, re, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
log = sys.argv[1]
pk = sys.argv[2] if len(sys.argv) > 2 else os.path.join(ROOT, 'MEASURED_PEAKS.json')
if os.path.exists(pk):
    d = json.load(open(pk)); TF, HBM, src = d['bf16_tflops'], d['hbm_gbs'], 'MEASURED_PEAKS.json (burst bf16 %.1f TFLOP/s, copy %.1f GB/s)' % (d['bf16_tflops'], d['hbm_gbs'])
else:
    TF, HBM, src = 989.0, 3350.0, 'H100 SXM data-sheet peaks (dense bf16, HBM3)'
pat = re.compile(r'^\s*(\d+)\s+(fprop|dgrad|wgrad)\s+H\s*(\d+)\s+(\d+)->\s*(\d+)\s+k(\d)\s+s(\d)\s+x(\d+)\s+M=\s*(\d+)\s+([\d.]+) ms\s+([\d.]+) TF/s\s+([\d.]+) GB/s')
rows = []
for line in open(log):
    m = pat.match(line)
    if not m:
        continue
    idx, kind, H, cin, cout, k, s, cnt, M, ms, tfs, gbs = m.groups()
    idx, H, cin, cout, k, s, cnt, M = map(int, (idx, H, cin, cout, k, s, cnt, M))
    ms, tfs, gbs = float(ms), float(tfs), float(gbs)
    flops = tfs * 1e12 * ms * 1e-3
    nbytes = gbs * 1e9 * ms * 1e-3
    t_tensor, t_hbm = flops / (TF * 1e12) * 1e3, nbytes / (HBM * 1e9) * 1e3
    roof = max(t_tensor, t_hbm)
    rows.append(dict(idx=idx, kind=kind, H=H, cin=cin, cout=cout, k=k, s=s, cnt=cnt, ms=ms, roof=roof,
                     bound='tensor' if t_tensor >= t_hbm else 'hbm', frac=roof / ms))
print('per-layer roofline, denominators: %s' % src)
print('source log: %s (256 views; x = occurrences in ResNet-50)' % os.path.basename(log))
print('%3s %-5s %-22s %3s %9s %9s %-6s %5s %9s' % ('#', 'kind', 'layer', 'x', 'ms', 'roof ms', 'bound', 'frac', 'lost ms*x'))
tot = {}
for r in rows:
    lost = (r['ms'] - r['roof']) * r['cnt']
    t = tot.setdefault(r['kind'], [0.0, 0.0]); t[0] += r['ms'] * r['cnt']; t[1] += r['roof'] * r['cnt']
    print('%3d %-5s H%-3d %4d->%4d k%d s%d %3d %9.3f %9.3f %-6s %5.2f %9.3f'
          % (r['idx'], r['kind'], r['H'], r['cin'], r['cout'], r['k'], r['s'], r['cnt'], r['ms'], r['roof'], r['bound'], r['frac'], lost))
print()
for k, (a, b) in tot.items():
    print('TOTAL %-5s measured %.2f ms, roofline %.2f ms, fraction %.2f' % (k, a, b, b / a))
worst = sorted(rows, key=lambda r: -(r['ms'] - r['roof']) * r['cnt'])[:8]
print('\nlargest gaps (ms lost x occurrences): ' + ', '.join('%d/%s %.2f' % (r['idx'], r['kind'], (r['ms'] - r['roof']) * r['cnt']) for r in worst))
