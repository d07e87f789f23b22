#!/usr/bin/env python
"""A/B of library builds on one GPU: runs a benchmark once per build in turn, `--runs` rounds, each run in its own process with
GPTQ_B200_LIB pointing at that build, so every build sees the same card, clocks and neighbours.

    python tools/ab_bench.py old=path/to/old.so new=path/to/new.so [--runs 3] [--script bench.py] [--dump DIR] -- [benchmark args]

Prints every run's JSON lines reduced to value, ms_per_step, gpu and clocks, then per build (and batch size) the median and the spread of
the runs, and each build's median against the first build's.  The host reference leg of bench.py (cpu_baseline) is skipped: it runs on
the CPU after the GPU timing and takes minutes.  --dump DIR passes --dump-outputs DIR/<build>_<run> to every run and then compares the
dumped outputs: the largest absolute difference between two runs of the first build, and between the first build and each other one.
"""
import argparse
import glob
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHILD = '''import runpy, sys
sys.argv = sys.argv[1:]
sys.path.insert(0, '.')
import bench
bench.cpu_baseline_subprocess = lambda *a, **k: None
bench.main() if sys.argv[0] == 'bench.py' else runpy.run_path(sys.argv[0], run_name='__main__')
'''


def run_once(lib, script, args):
    env = dict(os.environ, GPTQ_B200_LIB=os.path.abspath(lib))
    out = subprocess.run([sys.executable, '-c', CHILD, script] + args, cwd=ROOT, env=env, capture_output=True, text=True)
    if out.returncode != 0:
        sys.exit(f'{script} with {lib} failed ({out.returncode}):\n{out.stdout[-2000:]}\n{out.stderr[-4000:]}')
    return [json.loads(l) for l in out.stdout.splitlines() if l.startswith('{')]


def compare_dumps(a, b):
    """largest absolute difference per output name of two --dump-outputs directories"""
    res = {}
    for f in sorted(glob.glob(os.path.join(a, '*.npy'))):
        name = os.path.basename(f)[:-4]
        x, y = np.load(f).astype(np.float64), np.load(os.path.join(b, name + '.npy')).astype(np.float64)
        res[name] = float(np.abs(x - y).max()) if x.shape == y.shape else f'shape {x.shape} vs {y.shape}'
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('builds', nargs='+', help='name=path of a libgptq_b200.so; the first one is the baseline')
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--script', default='bench.py', help='bench.py or a tools/ benchmark that prints JSON lines')
    ap.add_argument('--dump', metavar='DIR', default=None)
    argv = sys.argv[1:]
    rest = argv[argv.index('--') + 1:] if '--' in argv else []
    args = ap.parse_args(argv[:argv.index('--')] if '--' in argv else argv)
    builds = [b.split('=', 1) for b in args.builds]
    results = {name: {} for name, _ in builds}  # name -> batch -> values
    for r in range(args.runs):
        for name, lib in builds:
            extra = ['--dump-outputs', os.path.join(args.dump, f'{name}_{r}')] if args.dump else []
            for line in run_once(lib, args.script, rest + extra):
                key = line.get('batch', 1)
                if line.get('value') is not None:
                    results[name].setdefault(key, []).append(line['value'])
                print(json.dumps({'build': name, 'run': r, 'batch': key, 'value': line.get('value'), 'ms_per_step': line.get('ms_per_step'),
                                  'gpu': line.get('gpu'), 'clocks': line.get('clocks')}), flush=True)
    base = builds[0][0]
    for name, _ in builds:
        for key, vals in sorted(results[name].items()):
            med = statistics.median(vals)
            ref = results[base].get(key)
            print(json.dumps({'build': name, 'batch': key, 'values': vals, 'median': med, 'spread': (max(vals) - min(vals)) / med,
                              'vs_' + base: med / statistics.median(ref) if ref else None}))
    if args.dump:
        d = lambda name, r: os.path.join(args.dump, f'{name}_{r}')
        if args.runs > 1:
            print(json.dumps({'max_abs_diff': f'{base} run 0 vs run 1', **compare_dumps(d(base, 0), d(base, 1))}))
        for name, _ in builds[1:]:
            print(json.dumps({'max_abs_diff': f'{base} vs {name} (run 0)', **compare_dumps(d(base, 0), d(name, 0))}))
            if args.runs > 1:
                print(json.dumps({'max_abs_diff': f'{name} run 0 vs run 1', **compare_dumps(d(name, 0), d(name, 1))}))


if __name__ == '__main__':
    main()
