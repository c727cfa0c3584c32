"""Time orbm_track_local_map_inertial_batch (PredictStateIMU, SearchLocalPoints, the inertial pose optimiser and its write-back) against the
per-frame chain of the library's existing entry points (orbm_frustum_project, orbm_search_local_map,
pose_inertial_optimization_last_{kf,frame}_batch, with the host doing PredictStateIMU and the rest of the glue, as
tests/track_inertial_lib.py writes it) for batches of 1, 24 and 240 streams, half of them in each mode.

Sizes: 1280x720 scenes, about 1650 keypoints and 2000 local map points per stream.  Both sides are timed with the host clock around
complete synchronous calls (uploads, kernels, downloads, glue), median of --reps runs after warm-up; the batched call's matches and
written-back states are first checked against the chain fed with the call's own prediction.  Prints the GPU's name and power limit with
the numbers, and one JSON line.
Usage: python tools/track_local_map_inertial_time.py [--reps 15]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]

import numpy as np  # noqa: E402

import oracle_lib as O  # noqa: E402
import orb_slam3_modified_b200 as orb  # noqa: E402
import track_inertial_lib as TI  # noqa: E402
import track_lib as T  # noqa: E402


def gpu_info():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
    if q.returncode != 0 or not q.stdout.strip():
        raise SystemExit('no GPU visible to nvidia-smi: this script measures the GPU and has no CPU mode')
    return q.stdout.strip().splitlines()[0]


def median_time(fn, reps, warm=3):
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
    ap.add_argument('--reps', type=int, default=15)
    a = ap.parse_args()
    info = gpu_info()
    g, rg = T.globals_(1280, 720), TI.rig()
    rows = []
    for B in (1, 24, 240):
        streams = [TI.stream(100 + b, g, rg, 1 + b % 2, M=2000, K_extra=250) for b in range(B)]
        th = np.full(B, 2.0, np.float32)
        d, imu = TI.batch(streams, g, rg, th)
        m = orb.ORBmatcher(0.8, False, max_batch=B, max_keypoints=max(2048, d['kcap']), max_mappoints=max(2048, d['mcap']))
        one = orb.ORBmatcher(0.8, False, max_batch=1, max_keypoints=max(2048, d['kcap']), max_mappoints=max(2048, d['mcap']))
        be = TI.GpuChainBackend(orb, one)

        def batched():
            return m.track_local_map_inertial_batch(d, imu)

        def chain(pred=None):
            out = []
            for b, s in enumerate(streams):
                if pred is None:
                    S, P = (s['kfState21'], s['preintKF']) if s['mode'] == 1 else (s['lastState21'], s['preintFrame'])
                    ps, pt = TI.predict_state(O, rg['Tcb7'], S, P)
                else:
                    ps, pt = pred['predState21'][b], pred['predTcw7'][b]
                out.append(TI.local_map_step(be, s, g, rg, s['mode'], ps, pt, th[b]))
            return out

        R = batched()
        for b, lm in enumerate(chain(R)):
            K = len(streams[b]['kps'])
            assert R['match'][b, :K].tobytes() == lm['match'].tobytes() and R['state21'][b].tobytes() == lm['state21'].tobytes(), \
                'batched call differs from the chain'
        tb = median_time(batched, a.reps)
        tc = median_time(chain, max(3, a.reps // 4), warm=1)
        rows.append(dict(streams=B, keypoints=int(d['nK'].mean()), local_points=int(d['nM'].mean()), batched_ms=tb * 1e3, chain_ms=tc * 1e3))
        print('%3d streams (%d keypoints, %d local points each): batched %.2f ms | per-frame chain %.2f ms | %.1fx'
              % (B, d['nK'].mean(), d['nM'].mean(), tb * 1e3, tc * 1e3, tc / tb))
    print('GPU: %s (name, power limit, max SM clock)' % info)
    print(json.dumps(dict(gpu=info, rows=rows)))


if __name__ == '__main__':
    main()
