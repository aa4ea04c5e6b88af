"""Summarise repeated `bench.py --quick --dump-ops OPS --dump-outputs DIR` runs and compare their outputs.

    python tools/compare_runs.py LABEL=RESULT.json,OPS.json,DIR [LABEL=...] [--ops 3,17,...]

RESULT.json holds bench.py's stdout (its last JSON line is used).  Prints, per run: the headline value, forward_ms
and by_kind_ms; per label: the mean and the spread (max - min) over its runs; the per-op ms and GB/s of the chosen
ops for every run; and whether every .npy under each DIR (fields and annotations) equals the first run's bit for bit.
Exits non-zero if any output differs."""
import argparse
import glob
import json
import os
import sys

import numpy as np


def find(d, key):
    if isinstance(d, dict):
        if key in d:
            return d[key]
        for v in d.values():
            r = find(v, key)
            if r is not None:
                return r
    return None


def load_result(path):
    lines = [ln for ln in open(path) if ln.lstrip().startswith('{')]
    return json.loads(lines[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('runs', nargs='+', help='LABEL=RESULT.json,OPS.json,DIR')
    ap.add_argument('--ops', default='3,17', help='op indices of the per-op table')
    args = ap.parse_args()
    runs = []
    for spec in args.runs:
        label, files = spec.split('=', 1)
        res, ops, out = files.split(',')
        runs.append((label, load_result(res), json.load(open(ops)), out))

    print('%-10s %10s %10s %9s %8s' % ('run', 'value', 'forward', 'gemm_tc', 'dwconv'))
    per_label = {}
    for label, r, _, _ in runs:
        bk = find(r, 'by_kind_ms')
        fwd = find(r, 'forward_ms')
        print('%-10s %10.1f %10.3f %9.3f %8.3f' % (label, r['value'], fwd, bk['gemm_tc'], bk['dwconv']))
        per_label.setdefault(label.rstrip('0123456789'), []).append((r['value'], fwd, bk['gemm_tc']))
    print('\nper label (trailing run numbers dropped): mean (spread = max - min) of value, forward_ms, gemm_tc')
    for label, v in per_label.items():
        a = np.array(v)
        print('%-10s n=%d  ' % (label, len(a)) + '  '.join('%.3f (%.3f)' % (a[:, i].mean(), np.ptp(a[:, i]))
                                                         for i in range(3)))

    sel = [int(s) for s in args.ops.split(',')]
    print('\nper op: ms / GB/s')
    print('%-10s ' % 'run' + ' '.join('%16s' % ('op %d' % i) for i in sel))
    for label, _, ops, _ in runs:
        table = {o['op']: o for o in ops['ops']}
        print('%-10s ' % label + ' '.join('%7.4f /%7.0f' % (table[i]['ms'], table[i]['gbs']) for i in sel))

    ok = True
    first = runs[0]
    names = sorted(os.path.basename(p) for p in glob.glob(os.path.join(first[3], '*.npy')))
    print('\noutputs against %s (%d arrays):' % (first[0], len(names)))
    for label, _, _, out in runs[1:]:
        other = sorted(os.path.basename(p) for p in glob.glob(os.path.join(out, '*.npy')))
        same = other == names and all(
            np.array_equal(np.load(os.path.join(first[3], n)), np.load(os.path.join(out, n)), equal_nan=True)
            for n in names)
        ok &= same
        print('  %-10s %s' % (label, 'bitwise identical' if same else 'DIFFERENT'))
    sys.exit(0 if ok else 1)


if __name__ == '__main__':
    main()
