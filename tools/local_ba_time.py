"""Time Optimizer::LocalBundleAdjustment as a whole for a batch of maps of config-4 size (20 keyframes, about 5000 points, 40k
observations), at 1 / 8 / 24 / 48 maps:
- device: one lba_local_bundle_adjustment_batch call (walk, solve, erase cascade and write-back on the GPU);
- today: the oracle's host walk of every map, one lba_solve_batch for all, then the oracle's host erase loop and write-back of every map
  (the walk is timed as the oracle returning at the stop flag; the erase and write-back as the oracle finishing given LM results, minus
  that walk);
- host: the oracle's whole function (its CPU Levenberg-Marquardt included) on one host thread, summed over the maps.
Every map of the device call is checked against the oracle (lists, counts, erase flags) first.  Host clocks around calls that end in a
stream synchronise; median of --reps after one warm-up.  Prints the GPU's name, power limit and max SM clock, and one JSON line.
Usage: python tools/local_ba_time.py [--reps 5] [--sizes 1,8,24,48]
"""
import argparse
import ctypes as C
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
import local_ba_lib as LB  # noqa: E402
import oracle_lib as O  # noqa: E402


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
        t = time.perf_counter()
        f()
        ts.append(time.perf_counter() - t)
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--sizes', default='1,8,24,48')
    a = ap.parse_args()
    sizes = [int(s) for s in a.sizes.split(',')]
    n_max = max(sizes)
    flat = []
    for s in range(n_max):
        M, k = LB.scene(500 + s, n_kf=20, n_pts=5000, obs_per_pt=8, n_cov=10, outlier_frac=0.03, inertial=s % 2 == 1)
        flat.append(LB.flatten(M, k))
    print('maps: %d keyframes, %d points, %d observations (map 0)' % (len(flat[0]['kfFlags']), len(flat[0]['pointFlags']), int(flat[0]['obsStart'][-1])))
    refs = [LB.oracle(m) for m in flat]
    info = gpu_info()
    print('GPU:', info)
    opt = orb.Optimizer(max_poses=64, max_points=8192, max_edges=65536, max_batch=n_max)
    L, Lo = orb.lib(), O.lib()
    Lo.orbo_local_ba.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    got = opt.local_bundle_adjustment_batch(flat)
    for j, (g, (r, _)) in enumerate(zip(got, refs)):
        for k in ('status', 'num_fixedKF', 'num_OptKF', 'num_MPs', 'num_edges'):
            assert g[k] == r[k], (j, k)
        for k in ('localKF', 'fixedKF', 'localPoint', 'obsFlag', 'pointBad'):
            assert np.array_equal(g[k], r[k]), (j, k)
    print('device results equal the oracle for all %d maps' % n_max)
    rows = []
    for n in sizes:
        packs = [orb.local_ba_struct(m) for m in flat[:n]]
        arr = (orb.LbaLocalMap * n)(*[p[0] for p in packs])
        t_dev = med(lambda: L.lba_local_bundle_adjustment_batch(opt._h, n, arr), a.reps)
        # today's path
        stops = [dict(m, stop=np.ones(1, np.uint8)) for m in flat[:n]]
        sp = [orb.local_ba_struct(m) for m in stops]
        t_walk = med(lambda: [Lo.orbo_local_ba(C.byref(p[0]), 0, None) for p in sp], a.reps)
        probs = [refs[j][1] for j in range(n)]
        lpk = [orb.Optimizer._pack(p, 10, 100.0 if flat[j]['inertial'] else 0.0, None) for j, p in enumerate(probs)]
        P = (orb._LbaProblem * n)(*[k[1] for k in lpk])
        R = (orb._LbaResult * n)(*[k[3] for k in lpk])
        t_solve = med(lambda: L.lba_solve_batch(opt._h, n, P, R), a.reps)
        given = [orb.local_ba_struct(m, given=dict(optPose=np.pad(refs[j][0]['optPose'], ((0, len(m['kfFlags']) - len(refs[j][0]['optPose'])), (0, 0))),
                                                   optPoint=np.pad(refs[j][0]['optPoint'], ((0, len(m['pointFlags']) - len(refs[j][0]['optPoint'])), (0, 0))),
                                                   edgeChi2=refs[j][0]['edgeChi2'], edgeDepthPositive=refs[j][0]['edgeDepthPositive']))
                 for j, m in enumerate(flat[:n])]
        t_given = med(lambda: [Lo.orbo_local_ba(C.byref(p[0]), 1, None) for p in given], a.reps)
        t_today = t_walk + t_solve + max(0.0, t_given - t_walk)
        full = [orb.local_ba_struct(m) for m in flat[:n]]
        t_host = med(lambda: [Lo.orbo_local_ba(C.byref(p[0]), 0, None) for p in full], max(1, a.reps // 2))
        row = dict(maps=n, device_ms=1e3 * t_dev, today_ms=1e3 * t_today, today_walk_ms=1e3 * t_walk, today_solve_ms=1e3 * t_solve,
                   today_finish_ms=1e3 * max(0.0, t_given - t_walk), host_ms=1e3 * t_host, launches=opt.local_last_launches())
        rows.append(row)
        print('%2d maps: device %.2f ms | today %.2f ms (walk %.2f, lba_solve_batch %.2f, erase+write-back %.2f) | host oracle %.1f ms | %d launches'
              % (n, row['device_ms'], row['today_ms'], row['today_walk_ms'], row['today_solve_ms'], row['today_finish_ms'], row['host_ms'], row['launches']))
    print(json.dumps(dict(tool='local_ba_time', gpu=info, rows=rows)))


if __name__ == '__main__':
    main()
