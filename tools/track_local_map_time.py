"""Time the batched tracking calls (orbm_motion_model_pose_batch + orbm_track_local_map_batch) against the per-frame chain of the
library's existing entry points (pose_optimization_batch, orbm_frustum_project, orbm_search_local_map, with the host doing the glue, as
tests/track_lib.py writes it) for batches of 1, 24 and 240 streams.

Sizes follow configs[2] of tools/extra_configs.py (1280x720, ~1000 keypoints, ~2000 local map points per stream).  Both sides are timed
with the host clock around complete synchronous calls (uploads, kernels, downloads, glue), median of --reps runs after warm-up; the two
sides' results are checked to be byte-identical first.  Prints the GPU's name and power limit with the numbers, and one JSON line.
Usage: python tools/track_local_map_time.py [--reps 20]
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

import orb_slam3_modified_b200 as orb  # noqa: E402
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
    ap.add_argument('--reps', type=int, default=20)
    a = ap.parse_args()
    info = gpu_info()
    g = T.globals_(1280, 720)
    rows = []
    for B in (1, 24, 240):
        streams = [T.stream(100 + b, g, M=2000, K_extra=300) for b in range(B)]
        th = np.ones(B, np.float32)
        mo, lo, st = T.batch(streams, g, th)
        m = orb.ORBmatcher(0.8, False, max_batch=B, max_keypoints=max(2048, mo['kcap']), max_mappoints=max(2048, lo['mcap']))
        one = orb.ORBmatcher(0.8, False, max_batch=1, max_keypoints=max(2048, mo['kcap']), max_mappoints=max(2048, lo['mcap']))
        be = T.GpuChainBackend(orb, one)

        def batched():
            match, claimed, nm = st['match'].copy(), st['claimed'].copy(), st['nmatches'].copy()
            r1 = m.motion_model_pose_batch(mo, g['invLevelSigma2'], match, claimed, nm)
            lo['Tcw7'] = r1['Tcw7']; lo['discarded'] = r1['discarded']
            r2 = m.track_local_map_batch(lo, match)
            return match, r2

        def chain():
            out = []
            for b, s in enumerate(streams):
                match, claimed = s['match'].copy(), s['claimed'].copy()
                mm = T.motion_model_step(be, s, g, match, claimed, s['nmatches'])
                out.append(T.local_map_step(be, s, g, match, mm['discarded'], mm['Tcw7'], th[b]))
            return out

        match, r2 = batched()
        for b, lm in enumerate(chain()):
            K = len(streams[b]['kps'])
            assert match[b, :K].tobytes() == lm['match'].tobytes() and r2['Tcw7'][b].tobytes() == lm['Tcw7'].tobytes(), 'batched call differs from the chain'
        tb = median_time(batched, a.reps)
        tc = median_time(chain, max(3, a.reps // 4), warm=1)
        rows.append(dict(streams=B, keypoints=int(mo['kcap']), local_points=int(lo['mcap']), batched_ms=tb * 1e3, chain_ms=tc * 1e3))
        print('%3d streams: batched %.2f ms | per-frame chain %.2f ms | %.1fx' % (B, tb * 1e3, tc * 1e3, tc / tb))
    print('GPU: %s (name, power limit, max SM clock)' % info)
    print(json.dumps(dict(gpu=info, rows=rows)))


if __name__ == '__main__':
    main()
