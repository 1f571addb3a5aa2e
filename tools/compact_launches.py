"""Compact an ncu launch list (csv of gpu__time_duration.sum) to one short row per launch:
id, kernel (template and argument lists stripped), grid, block, duration in us.

usage: python tools/compact_launches.py launches.csv [n_last_launches] > launches_compact.csv
"""
import csv
import re
import sys

with open(sys.argv[1]) as f:
    lines = [l for l in f if l.startswith('"')]
rows = []
for r in csv.DictReader(lines):
    if r.get('Metric Name') != 'gpu__time_duration.sum':
        continue
    v = float(r['Metric Value'].replace(',', ''))
    unit = r['Metric Unit']
    us = v / 1000.0 if unit in ('ns', 'nsecond') else v if unit in ('us', 'usecond') else v * 1000.0
    name = re.sub(r'\(.*', '', r['Kernel Name'])
    m = re.match(r'(?:void )?([\w:]+)(<.*)?', name)
    short = m.group(1) if m else name
    tmpl = m.group(2) if m and m.group(2) and short.startswith('p3d::') else ''
    rows.append((r['ID'], short + (tmpl or ''), r['Grid Size'], r['Block Size'], us))
if len(sys.argv) > 2:
    rows = rows[-int(sys.argv[2]):]
w = csv.writer(sys.stdout)
w.writerow(['id', 'kernel', 'grid', 'block', 'us'])
for r in rows:
    w.writerow([r[0], r[1], r[2], r[3], f'{r[4]:.3f}'])
