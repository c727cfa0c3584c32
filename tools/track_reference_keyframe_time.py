"""Time the batched TrackReferenceKeyFrame (orbm_track_reference_keyframe_batch) against the per-frame chain of the library's existing
entry points (orbv_transform_batch for the frame's BoW is left out of both sides; orbm_search_by_bow, pose_optimization_batch and the host
glue, as tests/track_ref_lib.py writes it) for batches of 1, 24 and 240 streams.

Scenes are 1280x720-sized (about 1650 keypoints per frame, a reference keyframe of similar size, FeatureVectors at level 2 of an L = 6
vocabulary).  Both sides are timed with the host clock around complete synchronous calls (uploads, kernels, downloads, glue), median of
--reps runs after warm-up; the two sides' results are checked to be byte-identical first.  Prints the GPU's name and power limit with the
numbers, and one JSON line.
Usage: python tools/track_reference_keyframe_time.py [--reps 20]
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

import orb_slam3_modified_b200 as orb  # noqa: E402
import track_lib as T  # noqa: E402
import track_ref_lib as TR  # noqa: E402


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


class _FixedBoW:
    """The per-frame chain with the FeatureVectors given (both sides take the frame's BoW as input)."""
    def __init__(self, be, st):
        self.be, self.st = be, st

    def __getattr__(self, k):
        return getattr(self.be, k)

    def feature_vector(self, desc):
        return self.st['fv'] if desc is self.st['desc'] else self.st['kf_fv']


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    a = ap.parse_args()
    info = gpu_info()
    g = T.globals_(1280, 720)
    voc = TR.ref_vocabulary()
    base = [TR.ref_kf_stream(200 + s, g, voc, M=2200, K_extra=220, kf_clutter=150) for s in range(8)]
    rows = []
    for B in (1, 24, 240):
        streams = [base[b % len(base)] for b in range(B)]
        d = TR.ref_batch(streams, g)
        m = orb.ORBmatcher(0.8, False, max_batch=B, max_keypoints=max(2048, d['kcap']), max_mappoints=max(2048, d['mcap']))
        one = orb.ORBmatcher(0.7, True, max_batch=1, max_keypoints=max(2048, d['kcap']), max_mappoints=max(2048, d['mcap']))
        be = TR.GpuChainBackend(orb, one)

        def batched():
            return m.track_reference_keyframe_batch(d)

        def chain():
            return [TR.reference_keyframe_step(_FixedBoW(be, s), s, g) for s in streams]

        R = batched()
        for b, r in enumerate(chain()):
            K = len(streams[b]['kps'])
            assert R['match'][b, :K].tobytes() == r['match'].tobytes() and R['nmatches'][b] == r['nmatches'], 'batched call differs from the chain'
            assert not r['gated'] or R['pose7'][b].tobytes() == r['pose7'].tobytes(), 'batched pose differs from the chain'
        tb = median_time(batched, a.reps)
        tc = median_time(chain, max(3, a.reps // 4), warm=1)
        kp = sum(len(s['kps']) for s in streams) / B
        kf = sum(len(s['kf_kps']) for s in streams) / B
        rows.append(dict(streams=B, keypoints=round(kp), keyframe_features=round(kf), batched_ms=tb * 1e3, chain_ms=tc * 1e3))
        print('%3d streams (%d keypoints, %d keyframe features): batched %.2f ms | per-frame chain %.2f ms | %.1fx'
              % (B, kp, kf, tb * 1e3, tc * 1e3, tc / tb))
    print('GPU: %s (name, power limit, max SM clock)' % info)
    print(json.dumps(dict(gpu=info, rows=rows)))


if __name__ == '__main__':
    main()
