"""Aggregates an `ncu --metrics gpu__time_duration.sum --csv` launch list into per-kernel totals (markdown on stdout).

    python profiles/summarize_launches.py launches.csv [steps_in_window]
Durations are cold-cache, serialised replays: compare SHARES, not absolutes."""
import csv
import re
import sys
from collections import OrderedDict


def main():
    path = sys.argv[1]
    steps = float(sys.argv[2]) if len(sys.argv) > 2 else 1.0
    rows = [r for r in csv.reader(l for l in open(path, errors='replace') if not l.startswith('=='))]
    hdr = next(r for r in rows if 'Kernel Name' in r)
    i_name, i_val, i_unit = hdr.index('Kernel Name'), hdr.index('Metric Value'), hdr.index('Metric Unit')
    agg = OrderedDict()
    for r in rows[rows.index(hdr) + 1:]:
        if len(r) <= i_val:
            continue
        name = re.sub(r'\(.*', '', r[i_name]).replace('void ', '').replace('aph::', '').replace('(int)', '')
        v = float(r[i_val].replace(',', ''))
        u = r[i_unit]
        v = v / 1e3 if u in ('ns', 'nsecond') else (v * 1e3 if u in ('ms', 'msecond') else v)      # -> us
        a = agg.setdefault(name, [0, 0.])
        a[0] += 1; a[1] += v
    tot = sum(a[1] for a in agg.values())
    print('| kernel | launches/step | us/step | share |\n|---|---|---|---|')
    for k, (n, t) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print('| `%s` | %.1f | %.1f | %.1f %% |' % (k, n / steps, t / steps, 100 * t / tot))
    print('| total | %.1f | %.1f | |' % (sum(a[0] for a in agg.values()) / steps, tot / steps))


if __name__ == '__main__':
    main()
