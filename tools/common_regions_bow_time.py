"""Time LoopClosing::DetectCommonRegionsFromBoW's BoW sweep for a batch of place-recognition queries: one synchronous
orbm_common_regions_bow_batch call (one upload through the matcher's staging, the sweep and the merge launches, one download) against the
same (current keyframe, entry) pairs issued one by one as orbm_search_by_bow_kf calls, and against the CPU oracle
(oracle/common_regions_oracle.cpp: the candidate loop over a pointer model, each SearchByBoW the pinned oracle body) on one host thread, in
the same run.

Queries come from tests/common_regions_lib.py: 6 candidates with 10 covisibles each (11 entries), about 1000 features per keyframe plus
10% clutter, 3% bad points, and each keyframe bad / connected to the current keyframe with probability --p-bad / --p-conn, so some
candidates are skipped or aborted by a near keyframe.  The pair count after those is printed.  GPU: host clock around the C call with the
ctypes arguments built beforehand, median of --reps calls after warm-up; every record is checked against the oracle first.  Per-pair
path: host clock around the loop of orbm_search_by_bow_kf calls (arguments prebuilt), median of --reps; it gives the counts, not the merge.
Oracle: host clock around orbo_common_regions_bow per query, summed over the batch, median of max(3, --reps / 4).  Prints the GPU's name,
power limit and max SM clock with the numbers, and one JSON line.  Without a GPU it runs the set-up and the oracle, then fails at the
GPU call.
Usage: python tools/common_regions_bow_time.py [--reps 20] [--sizes 1,7,24]
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
import common_regions_lib as CR  # noqa: E402
import oracle_lib as O  # noqa: E402


def gpu_info():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
    except FileNotFoundError:
        return None
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else None


def pairs(q, rec):
    """The (current keyframe, entry) pairs the sweep runs: every non-bad entry of every RAN candidate."""
    return [e for c in np.flatnonzero(rec['status'] == CR.RAN) for e in rec['covList'][c] if e >= 0 and not q['kfs'][e]['bad']]


def oracle_ms(qs, reps):
    L = O.lib()
    L.orbo_common_regions_bow.restype = None
    L.orbo_common_regions_bow.argtypes = [C.c_void_p]
    built = [orb.common_regions_struct(q) for q in qs]
    times = []
    for _ in range(reps):
        t = 0.0
        for s, _, _ in built:
            t0 = time.perf_counter()
            L.orbo_common_regions_bow(C.byref(s))
            t += time.perf_counter() - t0
        times.append(t * 1e3)
    return statistics.median(times)


def single_calls(qs, refs):
    """Prebuilt orbm_search_by_bow_kf arguments of every pair of the batch."""
    keep, calls = [], []

    def frame(kf, e, q):
        a = [np.ascontiguousarray(kf['kps'], orb.KP_DTYPE), np.ascontiguousarray(kf['desc'], np.uint8), np.ascontiguousarray(kf['fv'][0], np.int32),
             np.ascontiguousarray(kf['fv'][1], np.int32), CR.flags(q, e)]
        keep.append(a)
        return orb._OrbmBowFrame(len(a[0]), a[0].ctypes.data, a[1].ctypes.data, len(a[2]), a[2].ctypes.data, a[3].ctypes.data), a[4]

    for q, r in zip(qs, refs):
        f0, p0 = frame(q['kfs'][0], 0, q)
        m12 = np.zeros(max(len(q['kfs'][0]['kps']), 1), np.int32)
        keep += [f0, m12]
        for e in pairs(q, r):
            f, p = frame(q['kfs'][e], e, q)
            keep.append(f)
            calls.append((C.byref(f0), p0.ctypes.data, C.byref(f), p.ctypes.data, m12.ctypes.data))
    return calls, keep


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--sizes', default='1,7,24')
    ap.add_argument('--p-bad', type=float, default=0.02)
    ap.add_argument('--p-conn', type=float, default=0.02)
    a = ap.parse_args()
    info = gpu_info()
    sizes = [int(x) for x in a.sizes.split(',')]
    qs_all = [CR.random_query(5000 + s, n_cand=6, n_feat=1000, n_cov=(10, 10), share=0.2, p_bad_cand=a.p_bad, p_bad_cov=a.p_bad, p_conn=a.p_conn)
              for s in range(max(sizes))]
    refs = [CR.oracle(q) for q in qs_all]
    st = np.concatenate([r['status'] for r in refs])
    print('queries: 6 candidates x 11 entries, %.0f features per keyframe; candidates skipped %d, aborted %d, ran %d of %d' %
          (np.mean([len(kf['kps']) for q in qs_all for kf in q['kfs']]), (st == CR.SKIPPED).sum(), (st == CR.ABORTED_NEAR).sum(), (st == CR.RAN).sum(), len(st)))
    rows = []
    for n in sizes:
        rows.append(dict(queries=n, pairs=sum(len(pairs(q, r)) for q, r in zip(qs_all[:n], refs)), oracle_ms=oracle_ms(qs_all[:n], max(3, a.reps // 4))))
    mt = orb.ORBmatcher(0.9, True, max_batch=1, max_keypoints=2048, max_mappoints=2048)   # raises without a GPU: no CPU path
    L = orb.lib()
    for row in rows:
        n = row['queries']
        got = mt.common_regions_bow_batch(qs_all[:n])
        for g, r in zip(got, refs):
            assert CR.same(g, r), 'GPU != oracle'
        built = [orb.common_regions_struct(q) for q in qs_all[:n]]
        arr = (orb.OrbmCommonRegionsQuery * n)(*[b[0] for b in built])
        for _ in range(5):
            assert L.orbm_common_regions_bow_batch(mt._h, n, arr) == orb.ORB_OK
        times = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            rc = L.orbm_common_regions_bow_batch(mt._h, n, arr)
            times.append((time.perf_counter() - t0) * 1e3)
            assert rc == orb.ORB_OK
        row.update(gpu_ms=statistics.median(times), gpu_min_ms=min(times), gpu_max_ms=max(times), launches=mt.last_launch_count())
        calls, keep = single_calls(qs_all[:n], refs)
        nm = C.c_int(0)
        for c in calls[:5]:
            assert L.orbm_search_by_bow_kf(mt._h, c[0], c[1], c[2], c[3], 0.9, 1, c[4], C.byref(nm)) == orb.ORB_OK
        times = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            for c in calls:
                L.orbm_search_by_bow_kf(mt._h, c[0], c[1], c[2], c[3], 0.9, 1, c[4], C.byref(nm))
            times.append((time.perf_counter() - t0) * 1e3)
        row.update(single_ms=statistics.median(times))
        print('%3d queries, %4d pairs: batch call %.3f ms (median of %d; min %.3f, max %.3f; %d launches)   %d orbm_search_by_bow_kf calls %.3f ms'
              '   oracle, one thread %.3f ms' % (n, row['pairs'], row['gpu_ms'], a.reps, row['gpu_min_ms'], row['gpu_max_ms'], row['launches'],
                                                 row['pairs'], row['single_ms'], row['oracle_ms']))
    print('GPU: %s (name, power limit, max SM clock)' % info)
    print(json.dumps(dict(gpu=info, rows=rows)))


if __name__ == '__main__':
    main()
