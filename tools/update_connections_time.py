"""Time ProcessNewKeyFrame's map-point loop / the SearchInNeighbors tail with KeyFrame::UpdateConnections for a batch of keyframes: the
synchronous orbm_update_connections_batch call (one upload through the matcher's staging, one launch, one download) for 1, 8 and 48
keyframes, against the CPU oracle (oracle/update_connections_oracle.cpp, a literal transcription over a pointer map) on one host thread,
in the same run.

Keyframes are seeded scenes from tests/update_connections_lib.py: about 1000 slots (70% holding a point), about 10 observations per point,
a table of 150 keyframes, the two modes alternating.  GPU: host clock around the C call with the ctypes arguments built beforehand, median
of --reps calls after warm-up; every item's outputs are checked against the oracle first.  Oracle: host clock around orbo_update_connections
per item, summed over the batch, median of --reps; it includes building its pointer map from the flattened arrays.  Neither is the
reference's own code: its per-point std::map copies under mutexes are not modelled.  Prints the GPU's name, power limit and max SM clock with
the numbers, and one JSON line.  Without a GPU it runs the scene set-up and the oracle, then fails at the GPU call.
Usage: python tools/update_connections_time.py [--reps 30] [--sizes 1,8,48]
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
import update_connections_lib as U  # noqa: E402
import oracle_lib as O  # noqa: E402


def gpu_info():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
    except FileNotFoundError:
        return None
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else None


def oracle_ms(flat, reps):
    L = O.lib()
    L.orbo_update_connections.argtypes = [C.c_void_p, C.c_void_p]
    prepared = []
    for m in flat:
        s, out, keep = orb.connections_struct(m)
        nK, nP, nS = s.nKF, s.nPoints, s.nSlots
        nO, nC = int(keep['obsStart'][-1]), int(keep['connStart'][-1])
        bufs = [np.zeros(n, np.int32) for n in (nP + 1, nO + nP, nO + nP, nK + 1, nC + 2 * nK, nC + 2 * nK, max(nS, 1), 1, 1)]
        prepared.append((s, out, keep, bufs, U._Final(*[b.ctypes.data for b in bufs])))
    times = []
    for _ in range(reps):
        t = 0.0
        for s, _, _, _, f in prepared:
            t0 = time.perf_counter()
            L.orbo_update_connections(C.byref(s), C.byref(f))
            t += time.perf_counter() - t0
        times.append(t * 1e3)
    return statistics.median(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=30)
    ap.add_argument('--sizes', default='1,8,48')
    a = ap.parse_args()
    info = gpu_info()
    sizes = [int(x) for x in a.sizes.split(',')]
    flat_all = [U.flatten(U.scene(2000 + s, U.PNK if s % 2 == 0 else U.SIN)) for s in range(max(sizes))]
    stats = dict(table=float(np.mean([len(m['order']) for m in flat_all])), slots=float(np.mean([len(m['slotPoint']) for m in flat_all])),
                 filled=float(np.mean([(m['slotPoint'] >= 0).sum() for m in flat_all])),
                 obs_per_point=float(np.mean([np.diff(m['obsStart']).mean() for m in flat_all])))
    print('items: %.0f table keyframes, %.0f slots (%.0f holding a point), %.1f observations per point' %
          (stats['table'], stats['slots'], stats['filled'], stats['obs_per_point']))
    refs = [U.oracle(m)[0] for m in flat_all]
    rows = []
    for n in sizes:
        rows.append(dict(items=n, oracle_ms=oracle_ms(flat_all[:n], a.reps)))
    mt = orb.ORBmatcher(0.6, True, max_batch=1, max_keypoints=64, max_mappoints=64)   # raises without a GPU: no CPU path
    L = orb.lib()
    for row in rows:
        n = row['items']
        got = mt.update_connections_batch(flat_all[:n])
        for g, r in zip(got, refs):
            assert U.same_outputs(g, r), 'GPU != oracle'
        built = [orb.connections_struct(m) for m in flat_all[:n]]
        arr = (orb.OrbmConnectionsItem * n)(*[b[0] for b in built])
        for _ in range(5):
            assert L.orbm_update_connections_batch(mt._h, n, arr) == orb.ORB_OK
        times = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            rc = L.orbm_update_connections_batch(mt._h, n, arr)
            times.append((time.perf_counter() - t0) * 1e3)
            assert rc == orb.ORB_OK
        row.update(gpu_ms=statistics.median(times), gpu_min_ms=min(times), gpu_max_ms=max(times), launches=mt.last_launch_count(),
                   upload_bytes=int(sum(sum(np.asarray(m[k]).nbytes for k, _ in orb.CONNECTIONS_ARRAYS) for m in flat_all[:n])))
        print('%3d keyframes: GPU call %.3f ms (median of %d; min %.3f, max %.3f; %d launch, %.2f MB uploaded)   oracle, one thread %.3f ms' %
              (n, row['gpu_ms'], a.reps, row['gpu_min_ms'], row['gpu_max_ms'], row['launches'], row['upload_bytes'] / 1e6, row['oracle_ms']))
    print('GPU: %s (name, power limit, max SM clock)' % info)
    print(json.dumps(dict(gpu=info, items=stats, rows=rows)))


if __name__ == '__main__':
    main()
