"""SearchByProjection(current, last frame) at bench.py's shapes: kernel time of orbm_search_last_frame_batch_device, the phase split of
match_frame_kernel, and a byte-identity check of two builds of the library.

  python tools/match_phases.py                   kernel ms per 240 frames at 240 x 1 and 2 x 120 (two handles, one stream); with a
                                                 library built with -DMF_PHASES also each phase's share of the CTAs' clock64 time
  python tools/match_phases.py save OUT.npz      first saves match / claimed / nmatches of both of bench's 240-frame input sets at
                                                 batch 240, 2 x 120 and 240 x 1, then times as above
  python tools/match_phases.py diff A.npz B.npz  compares two saved files array by array

Select the library with ORB_B200_LIB, e.g. a build of tools/build_variants.sh "ph:matcher:-DMF_PHASES"."""
import ctypes as C
import os
import subprocess
import sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np

if len(sys.argv) > 1 and sys.argv[1] == 'diff':
    a, b = np.load(sys.argv[2]), np.load(sys.argv[3])
    assert sorted(a.files) == sorted(b.files), 'the files hold different arrays'
    bad = [k for k in sorted(a.files) if a[k].shape != b[k].shape or a[k].tobytes() != b[k].tobytes()]
    print('%d arrays compared, %d differ %s' % (len(a.files), len(bad), bad))
    sys.exit(1 if bad else 0)

import torch
import bench
import orb_slam3_modified_b200 as orb
from orb_slam3_modified_b200 import synth

B = 240
dev = torch.device('cuda')
st = torch.cuda.current_stream()
ex = orb.ORBextractor(bench.NFEAT, 1.2, 8, 20, 7, bench.W, bench.H, B)
cap = ex.max_keypoints
sf = ex.GetScaleFactors()
d_sf = torch.from_numpy(sf).to(dev)
cam = [float(c) for c in synth.camera(bench.W, bench.H)]
bounds = (0.0, 0.0, float(bench.W), float(bench.H))
cur, last = [], []          # per input set: the extracted frame (device slabs) and its map points as the next round's last frame
for k in range(2):
    frames = bench.make_frames(B, k)
    _, kl, dl = ex.extract_batch(frames, (0, 1000))
    last.append({n: torch.from_numpy(v).to(dev) for n, v in bench.last_frame_slabs(kl, dl, k, cap).items()})
    S = dict(kps=torch.zeros((B, cap, 7), dtype=torch.float32, device=dev), desc=torch.zeros((B, cap, 32), dtype=torch.uint8, device=dev),
             n=torch.zeros(B, dtype=torch.int32, device=dev), mono=torch.zeros(B, dtype=torch.int32, device=dev))
    ex.extract_batch_device(torch.from_numpy(frames).to(dev), S['kps'], S['desc'], S['n'], S['mono'], (0, 1000), st.cuda_stream)
    cur.append(S)
Tcw = [torch.from_numpy(np.stack([bench.stream_pose(s, k) for s in range(B)])).to(dev) for k in range(2)]
torch.cuda.synchronize()


def args(k, b0, b1):
    """bench.py's round with current set k: the frames of set k against the map points of set k ^ 1, streams b0..b1."""
    S, L = cur[k], last[k ^ 1]
    return dict(batch=b1 - b0, kcap=cap, mcap=cap, nlevels=8, kps=S['kps'][b0:b1], desc=S['desc'][b0:b1], nK=S['n'][b0:b1], scaleFactors=d_sf,
                nM=L['nM'][b0:b1], valid=L['valid'][b0:b1], xyz=L['xyz'][b0:b1], octave=L['octave'][b0:b1], angle=L['angle'][b0:b1],
                hasObs=L['hasObs'][b0:b1], mpDesc=L['mpDesc'][b0:b1], Tcw7=Tcw[k][b0:b1], bounds=bounds, cam=cam, reset=1)


SHAPES = {'240x1': [(0, B)], '2x120': [(0, B // 2), (B // 2, B)], '1x240': [(b, b + 1) for b in range(B)]}
out = {n: (torch.full((B, cap), -1, dtype=torch.int32, device=dev), torch.zeros((B, cap), dtype=torch.uint8, device=dev),
           torch.zeros(B, dtype=torch.int32, device=dev)) for n in SHAPES}
handles = {n: [orb.ORBmatcher(0.9, True, max_batch=b1 - b0, max_keypoints=cap, max_mappoints=cap) for b0, b1 in g[:2]] for n, g in SHAPES.items()}


def round_(name, k):
    m, c, nm = out[name]
    for g, (b0, b1) in enumerate(SHAPES[name]):
        handles[name][min(g, len(handles[name]) - 1)].search_last_frame_batch_device(args(k, b0, b1), bench.TH_PROJ, m[b0:b1], c[b0:b1], nm[b0:b1],
                                                                                     st.cuda_stream)


if len(sys.argv) > 1 and sys.argv[1] == 'save':
    res = {}
    for name in SHAPES:
        for k in range(2):
            round_(name, k)
            for a, t in zip(('match', 'claimed', 'nmatches'), out[name]):
                res['%s_set%d_%s' % (name, k, a)] = t.cpu().numpy()
    np.savez(sys.argv[2], **res)
    print('saved %d arrays to %s (mean matches per frame %.1f)' % (len(res), sys.argv[2], res['240x1_set0_nmatches'].mean()))

L = orb.lib()
phases = L.orbm_match_phases if hasattr(L, 'orbm_match_phases') else None
if phases is not None:
    phases.restype = C.c_int
    phases.argtypes = [C.c_void_p, C.c_void_p]
print(subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                     capture_output=True, text=True).stdout.strip(), '|', os.environ.get('ORB_B200_LIB', 'default library'))
reps = 20
for name in ('240x1', '2x120'):
    for i in range(4):
        round_(name, i & 1)
    ph = np.zeros(8, np.uint64)
    if phases:
        phases(handles[name][0]._h, ph.ctypes.data)       # zeroes the counters
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(st)
    for i in range(reps):
        round_(name, i & 1)
    e1.record(st)
    torch.cuda.synchronize()
    line = '%-6s kernel %.3f ms per 240 frames' % (name, e0.elapsed_time(e1) / reps)
    if phases:
        clus = phases(handles[name][0]._h, ph.ctypes.data)
        ph = ph.astype(np.float64)
        tot = ph[:4].sum()
        line += ' | cluster %d, %d CTAs per round | CTA time: build %.1f %%, pass 1 %.1f %%, pass 2 %.1f %%, outcome %.1f %%' % (
            clus, ph[6] / reps, 100 * ph[0] / tot, 100 * ph[1] / tot, 100 * ph[2] / tot, 100 * ph[3] / tot)
        line += ' | per CTA: build %.1fk, pass 1 %.1fk cycles; per frame: pass 2 %.1fk, outcome %.1fk cycles, %.2f sweeps, %.2f rescans' % (
            ph[0] / ph[6] / 1e3, ph[1] / ph[6] / 1e3, ph[2] / ph[7] / 1e3, ph[3] / ph[7] / 1e3, ph[4] / ph[7], ph[5] / ph[7])
    print(line)
