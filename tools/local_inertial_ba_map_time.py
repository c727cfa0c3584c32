"""Time Optimizer::LocalInertialBA as a whole for a batch of maps of the benchmark's inertial size
(synth.local_inertial_ba_problem(n_opt=10, n_cov_fixed=6, n_pts=2500), a predecessor and six older keyframes), at 1 / 24 / 132 maps:
- device: one local_inertial_ba_map_batch call (window walk, solve, erase cascade and write-back on the GPU);
- today: the host walk and finish of every map (the CPU oracle finishing given solver results, which walks the map, runs the erase cascade
  and writes back without solving) plus one local_inertial_ba_batch call for all the walked problems.
Every map of the device call is checked against the oracle's lists first.  Host clocks around calls that end in a stream synchronise;
median of --reps after one warm-up.  Prints the GPU's name, power limit and max SM clock, and one JSON line.
Usage: python tools/local_inertial_ba_map_time.py [--reps 5] [--sizes 1,24,132]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]

import orb_slam3_modified_b200 as orb  # noqa: E402
import local_inertial_ba_map_lib as LM  # noqa: E402
import oracle_lib as O  # noqa: E402
from orb_slam3_modified_b200 import synth  # noqa: E402


def gpu_info():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
    except FileNotFoundError:
        return None
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else None


def med(f, reps):
    f()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        f()
        ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts)


def bench_map(seed):
    pr = synth.local_inertial_ba_problem(n_opt=10, n_cov_fixed=6, n_pts=2500, seed=seed)
    pr['preint'] = O.liba_preints(pr)
    M, ids = LM.from_graph(pr, seed)
    return LM.flatten(M, ids[0], 12)          # KeyFramesInMap 12: Nd = 10, the window and its predecessor


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--sizes', default='1,24,132')
    a = ap.parse_args()
    sizes = [int(s) for s in a.sizes.split(',')]
    base = [bench_map(s) for s in range(4)]
    info = gpu_info()
    print('device:', info)
    rows = []
    for n in sizes:
        maps = [base[i % len(base)] for i in range(n)]
        res = orb.Optimizer.local_inertial_ba_map_batch(maps, debug=True)
        walked = [LM.oracle(m, given=LM.padded(r, m)) for m, r in zip(maps, res)]
        for r, (o, _) in zip(res, walked):
            for k in ('status', 'nLists', 'optKF', 'fixedKF', 'localPoint', 'ieLinked', 'obsFlag'):
                assert np.array_equal(r[k], o[k]), k
        probs = [pr for _, pr in walked]
        dev = med(lambda: orb.Optimizer.local_inertial_ba_map_batch(maps), a.reps)
        host = med(lambda: [LM.oracle(m, given=LM.padded(r, m)) for m, r in zip(maps, res)], a.reps)
        solve = med(lambda: orb.LocalInertialBA(probs), a.reps)
        row = dict(maps=n, device_ms=round(dev, 3), today_ms=round(host + solve, 3), host_walk_finish_ms=round(host, 3),
                   local_inertial_ba_batch_ms=round(solve, 3), points=int(res[0]['num_MPs']), edges=int(res[0]['num_edges']),
                   fixed=int(res[0]['num_fixedKF']))
        rows.append(row)
        print('%4d maps: device %.3f ms, today %.3f ms (host walk + finish %.3f, local_inertial_ba_batch %.3f)' % (n, dev, host + solve, host, solve))
    print(json.dumps(dict(device=info, rows=rows)))


if __name__ == '__main__':
    main()
