"""Time KeyFrameDatabase's BoW query: the synchronous orbv_db_query_batch call (one upload through the handle's staging, three launches,
one download) for 1, 8 and 48 queries against databases of 100, 1000 and 5000 keyframes, against the CPU oracle
(oracle/keyframe_database_oracle.cpp, the reference's DetectRelocalizationCandidates / DetectNBestCandidates transcribed over a pointer
model, both phases) on one host thread, in the same run.

Databases from tests/keyframe_database_lib.py: large_scene, a 10^6-word vocabulary (ORBvoc's order), 500 +- 50 words per keyframe,
consecutive keyframes sharing a third of their words.  Queries: query_from's mix (perturbed copies of keyframes, random BowVectors, a
few with no shared word), RELOC and NBEST alternating.  GPU: host clock around the C call with the ctypes arguments built beforehand,
median of --reps calls after warm-up; every record is checked against the oracle's phase-1 record first.  Oracle: host clock around each
detection (phase 1 and phase 2), summed over the queries, median of --reps.  Prints the GPU's name, power limit and max SM clock with the
numbers, and one JSON line.  Without a GPU it runs the scene set-up and the oracle, then fails at the GPU call.
Usage: python tools/keyframe_database_time.py [--reps 20] [--sizes 1,8,48] [--keyframes 100,1000,5000]
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
import keyframe_database_lib as K  # noqa: E402


def gpu_info():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
    except FileNotFoundError:
        return None
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else None


def queries(sc, n, first_id):
    rng = np.random.default_rng(first_id)
    return [K.query_from(rng, sc, first_id + i, K.RELOC if i % 2 == 0 else K.NBEST) for i in range(n)]


def oracle_ms(sc, o, qs, reps, next_id):
    times = []
    for r in range(reps):
        t = 0.0
        for q in qs:
            q = dict(q, id=next_id[0])                          # a fresh mark per detection, as the reference's mnId
            next_id[0] += 1
            t0 = time.perf_counter()
            o.query(q)
            t += time.perf_counter() - t0
        times.append(t * 1e3)
    return statistics.median(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--sizes', default='1,8,48')
    ap.add_argument('--keyframes', default='100,1000,5000')
    a = ap.parse_args()
    info = gpu_info()
    sizes = [int(x) for x in a.sizes.split(',')]
    rows, dbs = [], []
    next_id = [10 ** 6]
    for nkf in [int(x) for x in a.keyframes.split(',')]:
        sc = K.large_scene(17 + nkf, n_kf=nkf)
        o = K.Oracle(sc)
        o.apply(('add', list(range(sc.n))))
        qs_all = queries(sc, max(sizes), 1)
        recs = [o.query(q)[0] for q in qs_all]
        print('database: %d keyframes, %.0f words per keyframe; the %d queries list %.0f keyframes on average (max %d), score %.1f' %
              (nkf, np.mean([len(b[0]) for b in sc.bows]), len(qs_all), np.mean([r['nSharing'] for r in recs]), max(r['nSharing'] for r in recs),
               np.mean([r['scored'].sum() for r in recs])))
        dbs.append((nkf, sc, o, qs_all, recs))
        for n in sizes:
            rows.append(dict(keyframes=nkf, queries=n, oracle_ms=oracle_ms(sc, o, qs_all[:n], max(3, a.reps // 4), next_id)))
    L = orb.lib()
    for nkf, sc, o, qs_all, recs in dbs:
        db = orb.KeyFrameDatabase(sc.voc_words, max_keyframes=nkf, max_words=max(len(b[0]) for b in sc.bows))   # raises without a GPU
        db.add(0, [sc.key(k) for k in range(sc.n)], sc.bows)
        back = {int(sc.key(k)): k for k in range(sc.n)}
        gq = [dict(db=0, kind=q['kind'], word_id=q['word_id'], word_value=q['word_value'], connected=[sc.key(k) for k in q['connected']])
              for q in qs_all]
        for g, r in zip(db.query_batch(gq), recs):
            mine = dict(kf=np.array([back[int(x)] for x in g['key']], np.int32), words=g['words'], scored=g['scored'], score=g['score'],
                        nSharing=g['nSharing'], maxCommonWords=g['maxCommonWords'])
            assert K.same_record(mine, r), 'GPU != oracle'
        for row in rows:
            if row['keyframes'] != nkf:
                continue
            n = row['queries']
            built = [orb.db_query_struct(q, nkf) for q in gq[:n]]
            arr = (orb.OrbvDbQuery * n)(*[b[0] for b in built])
            for _ in range(5):
                assert L.orbv_db_query_batch(db._h, n, arr) == orb.ORB_OK
            times = []
            for _ in range(a.reps):
                t0 = time.perf_counter()
                rc = L.orbv_db_query_batch(db._h, n, arr)
                times.append((time.perf_counter() - t0) * 1e3)
                assert rc == orb.ORB_OK
            row.update(gpu_ms=statistics.median(times), gpu_min_ms=min(times), gpu_max_ms=max(times), launches=db.last_launch_count())
            print('%5d keyframes, %2d queries: GPU call %.3f ms (median of %d; min %.3f, max %.3f; %d launches)   oracle, one thread %.3f ms' %
                  (nkf, n, row['gpu_ms'], a.reps, row['gpu_min_ms'], row['gpu_max_ms'], row['launches'], row['oracle_ms']))
        db.close()
    print('GPU: %s (name, power limit, max SM clock)' % info)
    print(json.dumps(dict(gpu=info, rows=rows)))


if __name__ == '__main__':
    main()
