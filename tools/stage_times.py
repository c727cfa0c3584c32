"""Per-kernel device times of one 240-frame round (CUDA events inside the library, 5 repetitions) + a bit-exactness spot check of two
frames against the CPU oracle.  Use with ORB_B200_LIB=build/liborb_<variant>.so to compare kernel variants.  With a library built with
-DQT_PHASES (tools/build_variants.sh "ph:extractor:-DQT_PHASES") it also prints quadtree_kernel's phase stamps per level: clock64 cycles
per (level, frame) problem of the gather, the roots, the split passes, the careful-phase sorts and passes and the selection, and the
passes per problem."""
import ctypes as C
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
import numpy as np, torch
import bench
import orb_slam3_modified_b200 as orb
import oracle_lib as O
B = int(os.environ.get('B', '240'))
dev = torch.device('cuda')
ex = orb.ORBextractor(1000, 1.2, 8, 20, 7, 640, 480, B)
cap = ex.max_keypoints
sets = [bench.make_frames(B, k) for k in range(2)]
d_sets = [torch.from_numpy(s).to(dev) for s in sets]
d_kps = torch.zeros((B, cap, 7), dtype=torch.float32, device=dev); d_desc = torch.zeros((B, cap, 32), dtype=torch.uint8, device=dev)
d_n = torch.zeros(B, dtype=torch.int32, device=dev); d_mono = torch.zeros(B, dtype=torch.int32, device=dev)
st = torch.cuda.current_stream()
ex.set_profiling(True)
L = orb.lib()
phases = L.orbx_qt_phases if hasattr(L, 'orbx_qt_phases') else None
ph = (C.c_ulonglong * (16 * 9))()
if phases:
    phases(ph)
acc = {}
reps = 5
for i in range(reps + 1):
    ex.extract_batch_device(d_sets[i & 1], d_kps, d_desc, d_n, d_mono, (0, 1000), st.cuda_stream)
    if i:
        for k, v in ex.stage_ms().items():
            acc[k] = acc.get(k, 0.0) + v / reps
torch.cuda.synchronize()
if phases:
    phases(ph)
    a = np.array(ph[:], dtype=np.float64).reshape(16, 9)
    print('quadtree phases, cycles per problem: level gather roots split sort careful select | passes careful_passes problems')
    for lv in range(ex.nlevels):
        k = max(a[lv, 8], 1)
        print('  %d %s | %.2f %.2f %d' % (lv, ' '.join('%7.0f' % (a[lv, j] / k) for j in range(6)), a[lv, 6] / k, a[lv, 7] / k, a[lv, 8]))
last = (reps) & 1
oe = O.OracleExtractor(1000, 1.2, 8, 20, 7)
kps = d_kps.cpu().numpy().view(np.uint8).reshape(B, cap, 28); desc = d_desc.cpu().numpy(); n = d_n.cpu().numpy()
for b in (0, B - 1):
    _, ok, od = oe(sets[last][b], (0, 1000))
    assert n[b] == len(ok) and kps[b, :n[b]].tobytes() == ok.tobytes() and np.array_equal(desc[b, :n[b]], od), 'PARITY FAILURE frame %d' % b
print(os.environ.get('ORB_B200_LIB', 'default'), ' '.join('%s %.3f' % (k, v) for k, v in acc.items()), 'total %.3f' % sum(acc.values()), 'parity ok')
