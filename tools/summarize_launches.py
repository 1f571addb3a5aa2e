"""Summarise an ncu launch list (csv of gpu__time_duration.sum): per-kernel count / total / share for the LAST step.

usage: python tools/summarize_launches.py launches.csv [n_last_launches]
"""
import csv, sys, re, collections
path = sys.argv[1]
rows = []
with open(path) as f:
    lines = [l for l in f if l.startswith('"')]
for r in csv.DictReader(lines):
    if r.get('Metric Name') != 'gpu__time_duration.sum':
        continue
    v = float(r['Metric Value'].replace(',', ''))
    unit = r['Metric Unit']
    us = v / 1000.0 if unit in ('ns', 'nsecond') else v if unit in ('us', 'usecond') else v * 1000.0
    rows.append((r['Kernel Name'], us))
n_last = int(sys.argv[2]) if len(sys.argv) > 2 else None
if n_last:
    rows = rows[-n_last:]
agg = collections.OrderedDict()
for k, us in rows:
    k = re.sub(r'\(.*', '', k)
    k = re.sub(r'<.*', '', k)
    a = agg.setdefault(k, [0, 0.0])
    a[0] += 1; a[1] += us
tot = sum(a[1] for a in agg.values())
print(f"{len(rows)} launches, {tot/1000:.3f} ms summed kernel time")
for k, (n, us) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
    print(f"{us/1000:9.3f} ms {100*us/tot:5.1f}%  x{n:<4d} {k[:90]}")
