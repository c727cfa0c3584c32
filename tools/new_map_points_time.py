"""Time orbm_create_new_map_points (LocalMapping::CreateNewMapPoints for one new keyframe) against the CPU oracle on one host thread.

For 1, 10 and 30 neighbours of a synthetic keyframe: the median wall time of one synchronous call after warm-up (host clock around the
call, which ends in a stream synchronise), and the same for orbo_create_new_map_points.  Prints the GPU's name and power limit with the
numbers, and one JSON line.  Usage: python tools/new_map_points_time.py [--reps 50]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]

import numpy as np  # noqa: E402

import orb_slam3_modified_b200 as orb  # noqa: E402
import new_points_lib as NP  # noqa: E402
import oracle_lib as O  # noqa: E402


def gpu_info():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
    if q.returncode != 0 or not q.stdout.strip():
        raise SystemExit('no GPU visible to nvidia-smi: this script measures the GPU and has no CPU mode')
    return q.stdout.strip().splitlines()[0]


def median_time(fn, reps, warm=5):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=50)
    a = ap.parse_args()
    info = gpu_info()
    m = orb.ORBmatcher(0.6, False, max_batch=1, max_keypoints=2048, max_mappoints=2048)
    L = O.lib()
    L.orbo_create_new_map_points.argtypes = [C.c_void_p] * 6
    rows = []
    for n in (1, 10, 30):
        dts = tuple(d for k in range(3, 18) for d in (k, -k))[:n]          # frames 1 and 2 apart are mostly below the parallax limit
        sc = NP.scene(18, dts)
        args = (sc['kf1'], sc['kf2'], sc['sf'], sc['sigma2'], sc['ep'], sc['F12'], sc['Tcw'], sc['Ow'], sc['cam'], sc['scale_factor'])
        rec, nm, nc = m.CreateNewMapPoints(*args)
        orec, onm, onc, _ = NP.create(sc)
        assert rec.tobytes() == orec.tobytes() and np.array_equal(nm, onm) and np.array_equal(nc, onc), 'GPU differs from the oracle'
        inp = NP._In(sc)                              # both sides timed as one C call on prepared inputs
        out = np.zeros(len(sc['kf1']['kps']), orb.NEW_POINT_DTYPE)
        cnt, a1, a2 = C.c_int(0), np.zeros(n, np.int32), np.zeros(n, np.int32)
        G = orb.lib()
        tg = median_time(lambda: G.orbm_create_new_map_points(m._h, C.byref(inp.s), out.ctypes.data, C.byref(cnt), a1.ctypes.data, a2.ctypes.data), a.reps)
        tc = median_time(lambda: L.orbo_create_new_map_points(C.byref(inp.s), out.ctypes.data, C.byref(cnt), a1.ctypes.data, a2.ctypes.data, None),
                         max(5, a.reps // 5), warm=1)
        rows.append(dict(neighbours=n, kf1_features=len(sc['kf1']['kps']), matches=int(nm.sum()), created=len(rec), gpu_ms=tg * 1e3, oracle_ms=tc * 1e3))
        print('%2d neighbours: %4d matches, %4d points | GPU call %.3f ms | oracle (1 host thread) %.2f ms | %.1fx'
              % (n, nm.sum(), len(rec), tg * 1e3, tc * 1e3, tc / tg))
    print('GPU: %s (name, power limit, max SM clock)' % info)
    print(json.dumps(dict(gpu=info, rows=rows)))


if __name__ == '__main__':
    main()
