"""Time LocalMapping::KeyFrameCulling for a batch of maps: the synchronous orbm_keyframe_culling_batch call (one upload through the
matcher's staging, one launch, one download) for 1, 8 and 48 maps, against the CPU oracle (oracle/keyframe_culling_oracle.cpp, a literal
transcription of the reference's loop over a pointer map) on one host thread, in the same run.

Maps are user-scale corridors from tests/keyframe_culling_lib.py: 100 keyframes, the 99 before the current one local (the walk stops at
count 101 anyway), about 370 points per keyframe, 5-20 observations per point, monocular and mono-inertial alternating.  GPU: host clock
around the C call with the ctypes arguments built beforehand, median of --reps calls after warm-up; every map's result is checked against
the oracle first.  Oracle: host clock around orbo_keyframe_culling per map, summed over the batch, median of --reps; it includes building
its pointer map from the flattened arrays.  Prints the GPU's name, power limit and max SM clock with the numbers, and one JSON line.
Without a GPU it runs the scene set-up and the oracle, then fails at the GPU call.
Usage: python tools/keyframe_culling_time.py [--reps 20] [--sizes 1,8,48]
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
import keyframe_culling_lib as K  # noqa: E402
import oracle_lib as O  # noqa: E402


def gpu_info():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
    except FileNotFoundError:
        return None
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else None


def scene(s):
    return K.corridor(1000 + s, n_kf=100, n_kp=800, new_per_kf=30, window=(5, 20), inertial=s % 2 == 1, order='shuffle', kf_extra=20)


def oracle_ms(flat, reps):
    L = O.lib()
    L.orbo_keyframe_culling.argtypes = [C.c_void_p] * 7
    prepared = []
    for m in flat:
        s, out, keep = orb.culling_struct(m)
        nK, nP = len(m['kfFlags']), len(m['pointBad'])
        bufs = [np.zeros(nK, np.uint8), np.zeros(nK, np.int32), np.zeros(nK, np.int32), np.zeros(nP, np.uint8), np.zeros(nP, np.int32), C.c_int(0)]
        prepared.append((s, out, keep, bufs))
    times = []
    for _ in range(reps):
        t = 0.0
        for s, _, _, b in prepared:
            t0 = time.perf_counter()
            L.orbo_keyframe_culling(C.byref(s), *[x.ctypes.data for x in b[:5]], C.byref(b[5]))
            t += time.perf_counter() - t0
        times.append(t * 1e3)
    return statistics.median(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--sizes', default='1,8,48')
    a = ap.parse_args()
    info = gpu_info()
    sizes = [int(x) for x in a.sizes.split(',')]
    flat_all = [K.flatten(scene(s)) for s in range(max(sizes))]
    stats = dict(local=[len(m['local']) for m in flat_all], slots_per_kf=float(np.mean([m['slotStart'][-1] / len(m['local']) for m in flat_all])),
                 obs_per_point=float(np.mean([np.diff(m['obsStart']).mean() for m in flat_all])))
    print('maps: %d-%d local keyframes, %.0f points per local keyframe, %.1f observations per point' %
          (min(stats['local']), max(stats['local']), stats['slots_per_kf'], stats['obs_per_point']))
    refs = [K.oracle(m)[0] for m in flat_all]
    culled = [int(np.isin(r['status'], K.ERASING).sum()) for r in refs]
    print('oracle: %d of %d evaluated keyframes culled' % (sum(culled), sum(r['visited'] for r in refs)))
    rows = []
    for n in sizes:
        rows.append(dict(maps=n, oracle_ms=oracle_ms(flat_all[:n], max(3, a.reps // 4))))
    mt = orb.ORBmatcher(0.6, True, max_batch=1, max_keypoints=64, max_mappoints=64)   # raises without a GPU: no CPU path
    L = orb.lib()
    for row in rows:
        n = row['maps']
        got = mt.keyframe_culling_batch(flat_all[:n])
        for g, r in zip(got, refs):
            assert all(np.array_equal(g[k], r[k]) for k in ('status', 'nMPs', 'nRedundant')) and g['visited'] == r['visited'], 'GPU != oracle'
        built = [orb.culling_struct(m) for m in flat_all[:n]]
        arr = (orb.OrbmCullingMap * n)(*[b[0] for b in built])
        for _ in range(5):
            assert L.orbm_keyframe_culling_batch(mt._h, n, arr) == orb.ORB_OK
        times = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            rc = L.orbm_keyframe_culling_batch(mt._h, n, arr)
            times.append((time.perf_counter() - t0) * 1e3)
            assert rc == orb.ORB_OK
        row.update(gpu_ms=statistics.median(times), gpu_min_ms=min(times), gpu_max_ms=max(times), launches=mt.last_launch_count(),
                   upload_bytes=int(sum(sum(np.asarray(m[k]).nbytes for k, _ in orb.CULLING_ARRAYS if m.get(k) is not None) for m in flat_all[:n])))
        print('%3d maps: GPU call %.3f ms (median of %d; min %.3f, max %.3f; %d launch, %.2f MB uploaded)   oracle, one thread %.3f ms' %
              (n, row['gpu_ms'], a.reps, row['gpu_min_ms'], row['gpu_max_ms'], row['launches'], row['upload_bytes'] / 1e6, row['oracle_ms']))
    print('GPU: %s (name, power limit, max SM clock)' % info)
    print(json.dumps(dict(gpu=info, maps=stats, rows=rows)))


if __name__ == '__main__':
    main()
