"""Time LocalMapping::SearchInNeighbors for a batch of keyframes of different maps: the lockstep driver on orbm_fuse_search_batch (one
launch per round, max |targets| + 1 in all) against the per-call chain on orbm_fuse_search (one call per target keyframe and one for pass 2,
sum(|targets| + 1) in all), both as tests/search_in_neighbors_lib.py writes them, for 1, 8, 24 and 96 keyframes.

Every keyframe has 8 targets; keyframes come from synthetic 640x480 frames (about 1000 keypoints, about 500 map points each).  Both sides
are timed with the host clock around the complete driver (searches with their uploads and downloads, the host's bookkeeping walk, the
final ComputeDistinctiveDescriptors), median of --reps runs on fresh copies of the same maps after warm-up, the two sides alternating; the two sides' final map states
are checked to be equal first.  The time spent inside the searches (host clock around each synchronous call) is reported apart: the
walk and the map model are Python here, so they dominate the whole.  Also reports the searches' calls and the operand bytes they upload
per batch.  Prints the GPU's name and
power limit with the numbers, and one JSON line.
Usage: python tools/search_in_neighbors_time.py [--reps 3]
"""
import argparse
import copy
import gc
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]

import orb_slam3_modified_b200 as orb  # noqa: E402
import search_in_neighbors_lib as SN  # noqa: E402

OPERANDS = ('kps', 'desc', 'sf', 'isg', 'state', 'xyz', 'normal', 'min_d', 'max_d', 'mp_desc')


def gpu_info():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
    if q.returncode != 0 or not q.stdout.strip():
        raise SystemExit('no GPU visible to nvidia-smi: this script measures the GPU and has no CPU mode')
    return q.stdout.strip().splitlines()[0]


def fresh(jobs):
    """Deep copies of the jobs' maps sharing the (read-only) keyframe arrays."""
    memo = {}
    for j in jobs:
        for kf in j['map'].kfs:
            memo[id(kf.kps)], memo[id(kf.desc)] = kf.kps, kf.desc
    return copy.deepcopy(jobs, memo)


def counted(be):
    """Counts the calls and operand bytes of a backend's searches."""
    stats = dict(calls=0, bytes=0, search_s=0.0)
    inner = be.fuse

    def fuse(items):
        stats['calls'] += bool(items) if isinstance(be, SN.GpuBatchBackend) else len(items)   # launches of the searches
        stats['bytes'] += sum(it[k].nbytes for it in items for k in OPERANDS)
        t0 = time.perf_counter()
        out = inner(items)
        stats['search_s'] += time.perf_counter() - t0
        return out
    be.fuse = fuse
    return be, stats


def median_times(runs, jobs, reps, stats):
    """Median wall time of each run over fresh copies of the jobs, the runs alternating, the garbage collector off inside the timed region;
    and each run's mean time inside its searches."""
    for run in runs:
        run(fresh(jobs))
    for s in stats:
        s['search_s'] = 0.0
    ts = [[] for _ in runs]
    for _ in range(reps):
        for run, t in zip(runs, ts):
            js = fresh(jobs)
            gc.collect()
            gc.disable()
            t0 = time.perf_counter()
            run(js)
            t.append(time.perf_counter() - t0)
            gc.enable()
    return [statistics.median(t) for t in ts], [s['search_s'] / reps for s in stats]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--sizes', default='1,8,24,96')
    a = ap.parse_args()
    info = gpu_info()
    g = SN.globals_()
    base = SN.make_jobs(g, 8, 7, [8] * 8)
    m = orb.ORBmatcher(0.6, True, max_batch=1, max_keypoints=2048, max_mappoints=64)
    rows = []
    for B in [int(v) for v in a.sizes.split(',')]:
        jobs = [fresh([base[b % len(base)]])[0] for b in range(B)]     # one map per keyframe
        batch, sb = counted(SN.GpuBatchBackend(m))
        chain, sc = counted(SN.GpuChainBackend(m))
        x, y = fresh(jobs), fresh(jobs)
        SN.lockstep(batch, x)
        SN.sequential(chain, y)
        assert [j['map'].state() for j in x] == [j['map'].state() for j in y], 'lockstep differs from the per-call chain'
        calls = (sb['calls'], sc['calls'])
        mbytes = (sb['bytes'] / 1e6, sc['bytes'] / 1e6)
        (tb, tc), (sb_s, sc_s) = median_times([lambda js: SN.lockstep(batch, js), lambda js: SN.sequential(chain, js)], jobs, a.reps, [sb, sc])
        pts = sum(int((j['map'].kfs[j['cur']].mp >= 0).sum()) for j in jobs) / B
        rows.append(dict(keyframes=B, targets=8, points_per_keyframe=round(pts), lockstep_ms=tb * 1e3, chain_ms=tc * 1e3,
                         lockstep_search_ms=sb_s * 1e3, chain_search_ms=sc_s * 1e3, lockstep_calls=calls[0],
                         chain_calls=calls[1], lockstep_upload_mb=mbytes[0], chain_upload_mb=mbytes[1]))
        print('%3d keyframes x 8 targets (%d points each): lockstep %.1f ms (searches %.1f ms in %d launches) | per-call chain %.1f ms (searches %.1f ms '
              'in %d calls) | %.2fx whole, %.2fx searches | operands uploaded %.1f / %.1f MB'
              % (B, pts, tb * 1e3, sb_s * 1e3, calls[0], tc * 1e3, sc_s * 1e3, calls[1], tc / tb, sc_s / sb_s, mbytes[0], mbytes[1]))
    print('GPU: %s (name, power limit, max SM clock)' % info)
    print(json.dumps(dict(gpu=info, rows=rows)))


if __name__ == '__main__':
    main()
