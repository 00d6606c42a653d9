#!/usr/bin/env python
"""Summarise an `ncu --metrics gpu__time_duration.sum --csv` launch list: kernel | launches | total us | share.

    python tools/launch_summary.py launches.csv [skip_first_n] > launches.txt
Per-launch times under ncu are cold-cache and serialised: compare SHARES, not absolutes.
"""
import collections
import csv
import re
import sys


def main():
    path = sys.argv[1]
    skip = int(sys.argv[2]) if len(sys.argv) > 2 else 0
    lines = [l for l in open(path, errors='replace') if l.startswith('"')]
    rows = list(csv.reader(lines))
    hdr = rows[0]
    ik, iv, iu = hdr.index('Kernel Name'), hdr.index('Metric Value'), hdr.index('Metric Unit')
    agg = collections.OrderedDict()
    n = 0
    for r in rows[1:]:
        n += 1
        if n <= skip:
            continue
        name = re.sub(r'\(.*', '', r[ik])
        name = re.sub(r'^(void )?(cdx::)?(\(anonymous namespace\)::)?', '', name)
        v = float(r[iv].replace(',', ''))
        v = {'ns': v / 1e3, 'us': v, 'ms': v * 1e3, 'ms ': v * 1e3}.get(r[iu], v)
        a = agg.setdefault(name, [0, 0.0])
        a[0] += 1
        a[1] += v
    tot = sum(a[1] for a in agg.values())
    print('# kernel | launches | total us | share')
    for k, a in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print(f'  {k:<52s} {a[0]:6d} {a[1]:10.1f} {100 * a[1] / tot:6.1f}%')
    print(f'TOTAL {sum(a[0] for a in agg.values())} launches {tot:.1f} us')


if __name__ == '__main__':
    main()
