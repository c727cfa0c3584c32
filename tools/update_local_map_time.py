"""Time Tracking::UpdateLocalMap for a batch of streams: the synchronous orbm_update_local_map_batch call (one upload through the
matcher's staging, one launch, one download) for 1, 24 and 240 streams, against the CPU oracle (oracle/local_map_oracle.cpp, a literal
transcription of UpdateLocalKeyFrames / UpdateLocalPoints over a pointer model) on one host thread, in the same run.

Streams are corridors from tests/local_map_lib.py: 120 keyframes, 4000 points each seen by a window of 3-10 consecutive keyframes, a
frame whose 700 match-space entries hold points of the 40 newest keyframes; monocular and mono-inertial alternating, both vote branches.
48 distinct streams are cycled to fill the larger batches; the output slabs are as wide as the largest local map, rounded up to 256.
GPU: host clock around the C call with the ctypes arguments built beforehand, median of --reps calls after warm-up; the outputs are
checked against the oracle first.  Oracle: host clock around orbo_update_local_map per stream, summed over the batch; it includes building its pointer model from the flattened arrays.
Also the bytes staged per stream: the keyframe table this call uploads (each array at its C type) against what a host-side UpdateLocalMap uploads to
orbm_track_local_map_batch (70 bytes per local point and 4 per lastToLocal entry).  Prints the GPU's name, power limit and max SM clock with
the numbers, and one JSON line.  Without a GPU it runs the scene set-up and the oracle, then fails at the GPU call.
Usage: python tools/update_local_map_time.py [--reps 20] [--sizes 1,24,240]
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
import local_map_lib as L  # noqa: E402
import oracle_lib as O  # noqa: E402

DISTINCT = 48
LOCAL_MAP_ROW_BYTES = 12 + 12 + 4 + 4 + 4 + 32 + 1 + 1     # worldPos, normal, minDistInv, maxDistInv, maxDistance, mpDesc, hasObs, bad


def gpu_info():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
    except FileNotFoundError:
        return None
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else None


def scene(s):
    return L.scene(2000 + s, n_kf=120, n_pts=4000, window=(3, 10), n_src=700, inertial=s % 2 == 1, vote_last=s % 4 == 3, recent=40)


def oracle_ms(d, reps):
    lib = O.lib()
    lib.orbo_update_local_map.argtypes = [C.c_void_p, C.c_void_p]
    lib.orbo_update_local_map.restype = None
    singles = []
    for b in range(d['batch']):
        one = stream_batch(d, b)
        out = orb.local_map_outputs(one)
        keep = {n: np.ascontiguousarray(one[n], dt) for n, dt in orb.LOCAL_MAP_ARRAYS}
        singles.append(orb.local_map_structs(one, out, lambda n: keep[n].ctypes.data) + (keep, out))
    times = []
    for _ in range(reps):
        t = 0.0
        for s, r, _, _ in singles:
            t0 = time.perf_counter()
            lib.orbo_update_local_map(C.byref(s), C.byref(r))
            t += time.perf_counter() - t0
        times.append(t * 1e3)
    return statistics.median(times)


def stream_batch(d, b):
    """Stream b of batch dict d as a batch of one."""
    k0, k1, p0, p1 = int(d['kfStart'][b]), int(d['kfStart'][b + 1]), int(d['pointStart'][b]), int(d['pointStart'][b + 1])
    one = dict(batch=1, kcap=d['kcap'], mcap=d['mcap'], mcapLast=d['mcapLast'], nKF=k1 - k0, nPoints=p1 - p0)
    one['kfStart'], one['pointStart'] = np.array([0, k1 - k0], np.int32), np.array([0, p1 - p0], np.int32)
    for n in ('kfFlags', 'parent', 'prevKF'):
        one[n] = d[n][k0:k1]
    for start, vals in (('covStart', 'covKF'), ('childStart', 'childKF'), ('slotStart', 'slotPoint')):
        s = d[start][k0:k1 + 1]
        one[start], one[vals] = (s - s[0]).astype(np.int32), d[vals][s[0]:s[-1]]
    s = d['obsStart'][p0:p1 + 1]
    one['obsStart'], one['obsKF'] = (s - s[0]).astype(np.int32), d['obsKF'][s[0]:s[-1]]
    for n in ('pointBad', 'worldPos', 'normal', 'minDistInv', 'maxDistInv', 'maxDistance', 'mpDesc', 'hasObs'):
        one[n] = d[n][p0:p1]
    for n in ('nSrc', 'srcPoint', 'voteLastFrame', 'match', 'nK', 'inertial', 'lastKF'):
        one[n] = d[n][b:b + 1]
    return one


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--sizes', default='1,24,240')
    a = ap.parse_args()
    info = gpu_info()
    sizes = [int(x) for x in a.sizes.split(',')]
    items = [L.flatten(scene(s))[0] for s in range(DISTINCT)]
    d_all = orb.local_map_batch(items, 1 << 14)
    ref_all = L.oracle(d_all)
    mcap = (int(ref_all['nM'].max()) + 255) // 256 * 256
    nM = ref_all['nM'][:DISTINCT]
    table_bytes = [sum(np.asarray(it[n], dt).nbytes for n, dt in orb.LOCAL_MAP_ARRAYS if n in it) for it in items]
    flat_bytes = [LOCAL_MAP_ROW_BYTES * int(m) + 4 * len(it['srcPoint']) for m, it in zip(nM, items)]
    stats = dict(table_kf=float(np.mean(np.diff(d_all['kfStart'][:DISTINCT + 1]))), points=float(np.mean(np.diff(d_all['pointStart'][:DISTINCT + 1]))),
                 local_kf=float(ref_all['nLocalKF'][:DISTINCT].mean()), local_points=float(nM.mean()), mcap=mcap,
                 table_bytes=float(np.mean(table_bytes)), local_map_flatten_bytes=float(np.mean(flat_bytes)))
    print('streams: %.0f table keyframes, %.0f points, %.1f local keyframes, %.0f local points (means); slabs %d wide' %
          (stats['table_kf'], stats['points'], stats['local_kf'], stats['local_points'], mcap))
    print('staged per stream: keyframe table %.0f bytes, current local-map flatten %.0f bytes (ratio %.2f)' %
          (stats['table_bytes'], stats['local_map_flatten_bytes'], stats['table_bytes'] / stats['local_map_flatten_bytes']))
    rows = []
    for n in sizes:
        d = orb.local_map_batch([items[b % DISTINCT] for b in range(n)], mcap)
        rows.append(dict(streams=n, oracle_ms=oracle_ms(d, max(3, a.reps // 4)), d=d))
    mt = orb.ORBmatcher(0.8, False, max_batch=1, max_keypoints=64, max_mappoints=64)   # raises without a GPU: no CPU path
    lib = orb.lib()
    for row in rows:
        d = row.pop('d')
        n = row['streams']
        got = mt.update_local_map_batch(d)
        ref = L.oracle(d)
        assert all(np.array_equal(got[k], ref[k]) for k in got), 'GPU != oracle'
        out = orb.local_map_outputs(d)
        keep = {k: np.ascontiguousarray(d[k], dt) for k, dt in orb.LOCAL_MAP_ARRAYS}
        s, r = orb.local_map_structs(d, out, lambda k: keep[k].ctypes.data)
        for _ in range(5):
            assert lib.orbm_update_local_map_batch(mt._h, C.byref(s), C.byref(r)) == orb.ORB_OK
        times = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            rc = lib.orbm_update_local_map_batch(mt._h, C.byref(s), C.byref(r))
            times.append((time.perf_counter() - t0) * 1e3)
            assert rc == orb.ORB_OK
        row.update(gpu_ms=statistics.median(times), gpu_min_ms=min(times), gpu_max_ms=max(times), launches=mt.last_launch_count())
        print('%3d streams: GPU call %.3f ms (median of %d; min %.3f, max %.3f; %d launch)   oracle, one thread %.3f ms' %
              (n, row['gpu_ms'], a.reps, row['gpu_min_ms'], row['gpu_max_ms'], row['launches'], row['oracle_ms']))
    print('GPU: %s (name, power limit, max SM clock)' % info)
    print(json.dumps(dict(gpu=info, streams=stats, rows=rows)))


if __name__ == '__main__':
    main()
