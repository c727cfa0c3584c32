"""Time orbm_create_new_map_points (LocalMapping::CreateNewMapPoints for one new keyframe) against the CPU oracle on one host thread, and
orbm_create_new_map_points_batch (new keyframes of several maps in one call) against one single call per keyframe.

Single rows: for 1, 10 and 30 neighbours of a synthetic keyframe, the median wall time of one synchronous call after warm-up (host clock
around the call, which ends in a stream synchronise), and the same for orbo_create_new_map_points.  Batch rows: B = 1 / 8 / 48 keyframes
(different frames and seeds stand in for different maps) with 30 neighbours each, one batched call against B single calls back to back,
both timed the same way; the input bytes the batch uploads are printed with them.  Every row first asserts that the GPU equals the oracle
and that the batch equals the single calls byte for byte.  Prints the GPU's name, power limit and maximum SM clock with the numbers, and
one JSON line.  Usage: python tools/new_map_points_time.py [--reps 50] [--mode all|single|batch]
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

DTS30 = tuple(d for k in range(3, 18) for d in (k, -k))          # frames 1 and 2 apart are mostly below the parallax limit


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


def args_of(sc):
    return (sc['kf1'], sc['kf2'], sc['sf'], sc['sigma2'], sc['ep'], sc['F12'], sc['Tcw'], sc['Ow'], sc['cam'], sc['scale_factor'])


def upload_bytes(sc):
    """Input bytes one item puts on the staging: level tables, KF1, every neighbour, Tcw / Ow / cam (without the 256-byte piece alignment
    and the item / pair tables)."""
    def kf(k):
        return len(k['kps']) * (orb.KP_DTYPE.itemsize + 32 + 1) + 8 * len(k['fv'][0])
    n = len(sc['kf2'])
    return 8 * len(sc['sf']) + kf(sc['kf1']) + sum(kf(k) for k in sc['kf2']) + (48 + 12 + 16) * (n + 1)


def single_rows(m, reps, L, G):
    rows = []
    for n in (1, 10, 30):
        sc = NP.scene(18, DTS30[:n])
        rec, nm, nc = m.CreateNewMapPoints(*args_of(sc))
        orec, onm, onc, _ = NP.create(sc)
        assert rec.tobytes() == orec.tobytes() and np.array_equal(nm, onm) and np.array_equal(nc, onc), 'GPU differs from the oracle'
        inp = NP._In(sc)                              # both sides timed as one C call on prepared inputs
        out = np.zeros(len(sc['kf1']['kps']), orb.NEW_POINT_DTYPE)
        cnt, a1, a2 = C.c_int(0), np.zeros(n, np.int32), np.zeros(n, np.int32)
        tg = median_time(lambda: G.orbm_create_new_map_points(m._h, C.byref(inp.s), out.ctypes.data, C.byref(cnt), a1.ctypes.data, a2.ctypes.data), reps)
        tc = median_time(lambda: L.orbo_create_new_map_points(C.byref(inp.s), out.ctypes.data, C.byref(cnt), a1.ctypes.data, a2.ctypes.data, None),
                         max(5, reps // 5), warm=1)
        rows.append(dict(neighbours=n, kf1_features=len(sc['kf1']['kps']), matches=int(nm.sum()), created=len(rec), gpu_ms=tg * 1e3, oracle_ms=tc * 1e3))
        print('%2d neighbours: %4d matches, %4d points | GPU call %.3f ms | oracle (1 host thread) %.2f ms | %.1fx'
              % (n, nm.sum(), len(rec), tg * 1e3, tc * 1e3, tc / tg))
    return rows


def batch_rows(m, reps, G):
    rows = []
    scenes = [NP.scene(18 + b % 8, DTS30, seed=b // 8) for b in range(48)]
    for B in (1, 8, 48):
        scs = scenes[:B]
        res = m.create_new_map_points_batch([dict(zip(('kf1', 'kf2_list', 'scale_factors', 'level_sigma2', 'ep', 'F12', 'Tcw', 'Ow', 'cam', 'scale_factor'),
                                                      args_of(sc))) for sc in scs])
        for sc, (rec, nm, nc) in zip(scs, res):
            srec, snm, snc = m.CreateNewMapPoints(*args_of(sc))
            orec, onm, onc, _ = NP.create(sc)
            assert rec.tobytes() == srec.tobytes() == orec.tobytes() and nm.tobytes() == snm.tobytes() == onm.tobytes() and \
                nc.tobytes() == snc.tobytes() == onc.tobytes(), 'batch differs from the single calls or the oracle'
        ins = [NP._In(sc) for sc in scs]
        arr = (orb.OrbmNewPointsItem * B)()
        bufs = []
        for j, i in enumerate(ins):
            b = (np.zeros(i.N1, orb.NEW_POINT_DTYPE), np.zeros(1, np.int32), np.zeros(i.n, np.int32), np.zeros(i.n, np.int32))
            bufs.append(b)
            arr[j] = orb.OrbmNewPointsItem(i.s, *[a.ctypes.data for a in b])

        def singles():
            for i, b in zip(ins, bufs):
                G.orbm_create_new_map_points(m._h, C.byref(i.s), *[a.ctypes.data for a in b])
        tb = median_time(lambda: G.orbm_create_new_map_points_batch(m._h, B, arr), reps)
        assert m.last_launch_count() == 3
        ts = median_time(singles, reps)
        up = sum(upload_bytes(sc) for sc in scs)
        slots = sum(len(sc['kf2']) * len(sc['kf1']['kps']) for sc in scs)
        rows.append(dict(keyframes=B, neighbours=30, created=sum(len(r[0]) for r in res), upload_bytes=up, scratch_bytes=50 * slots,
                         batch_ms=tb * 1e3, singles_ms=ts * 1e3))
        print('B = %2d keyframes x 30 neighbours: %5d points | uploaded %.2f MB, scratch %.1f MB | one batched call %.3f ms | %2d single calls %.3f ms | %.2fx'
              % (B, rows[-1]['created'], up / 1e6, 50 * slots / 1e6, tb * 1e3, B, ts * 1e3, ts / tb))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=50)
    ap.add_argument('--mode', choices=('all', 'single', 'batch'), default='all')
    a = ap.parse_args()
    info = gpu_info()
    m = orb.ORBmatcher(0.6, False, max_batch=1, max_keypoints=2048, max_mappoints=2048)
    L = O.lib()
    L.orbo_create_new_map_points.argtypes = [C.c_void_p] * 6
    G = orb.lib()
    out = dict(gpu=info)
    if a.mode in ('all', 'single'):
        out['rows'] = single_rows(m, a.reps, L, G)
    if a.mode in ('all', 'batch'):
        out['batch_rows'] = batch_rows(m, a.reps, G)
    print('GPU: %s (name, power limit, max SM clock)' % info)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
