"""The C++ host mirror (include/orb_b200/orb_slam3.hpp) compiles with plain g++ against the C-ABI (CPU test) and, run on the GPU,
gives the oracle's results on every surface: ORBextractor::operator(), ORBmatcher::SearchByProjection (two stack temporaries),
Optimizer::PoseOptimization, Optimizer::LocalBundleAdjustment (three calls on the per-thread arena, the last with the caller's
bool abort flag set) and Optimizer::LocalInertialBA (plain and with bRecInit)."""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build(out_dir):
    """Compile tests/cpp_example.cpp into `out_dir` (never into the repository tree, which may not be writable) and return its path."""
    exe = os.path.join(str(out_dir), 'cpp_example')
    lib = os.path.join(ROOT, 'orb_slam3_modified_b200')
    subprocess.check_call(['g++', '-std=c++14', '-O2', '-Wall', '-I', os.path.join(ROOT, 'include'), os.path.join(ROOT, 'tests', 'cpp_example.cpp'),
                           '-o', exe, '-L', lib, '-l:liborb_b200.so', '-Wl,-rpath,' + lib, '-lpthread'])
    return exe


def _checksum(b):
    s = 0
    for v in bytes(b):
        s = (s * 1315423911 + v) % (1 << 64)
    return s


def test_cpp_shim_compiles_and_links(tmp_path):
    assert os.path.exists(_build(tmp_path))


@pytest.mark.gpu
def test_cpp_shim_runs_like_the_oracle(tmp_path):
    import oracle_lib as O
    import matcher_scenes as S
    from orb_slam3_modified_b200 import synth
    exe = _build(tmp_path)
    t = 12
    sc = S.last_frame_scene(t)
    img = synth.frame(t)
    (tmp_path / 'img.raw').write_bytes(img.tobytes())
    L = sc['last']
    for name, arr, dt in (('last_valid', L['valid'], np.uint8), ('last_hasobs', L['hasObs'], np.uint8), ('last_desc', L['descriptors'], np.uint8),
                          ('last_xyz', L['xyz'], np.float32), ('last_angle', L['angle'], np.float32), ('last_octave', L['octave'], np.int32),
                          ('tcw', sc['Tcw'], np.float32), ('cam', sc['cam'], np.float32)):
        (tmp_path / (name + '.raw')).write_bytes(np.ascontiguousarray(arr, dt).tobytes())
    p = synth.lba_problem(n_kf=7, n_pts=400, obs_per_pt=5, seed=61, n_fixed=2)
    for name, arr, dt in (('lba_poses', p['poses'], np.float64), ('lba_points', p['points'], np.float64), ('lba_obs', p['obs'], np.float64),
                          ('lba_fixed', p['fixed'], np.uint8), ('lba_cam', p['cam'], np.float32), ('lba_is2', p['inv_sigma2'], np.float32),
                          ('lba_ep', p['edge_point'], np.int32), ('lba_ek', p['edge_pose'], np.int32)):
        (tmp_path / (name + '.raw')).write_bytes(np.ascontiguousarray(arr, dt).tobytes())
    lp = synth.local_inertial_ba_problem(n_opt=5, n_cov_fixed=2, n_pts=200, seed=31)
    lP = O.liba_preints(lp)
    for name, arr, dt in (('liba_state', lp['state'], np.float64), ('liba_tcw', lp['tcw'], np.float64), ('liba_extr', lp['extr'], np.float64), ('liba_points', lp['points'], np.float64),
                          ('liba_obs', lp['obs'], np.float64), ('liba_cam', lp['cam'], np.float32), ('liba_preint', lP, np.float32), ('liba_td', lp['track_depth'], np.float32),
                          ('liba_is2', lp['inv_sigma2'], np.float32), ('liba_k1', lp['ie_kf1'], np.int32), ('liba_k2', lp['ie_kf2'], np.int32), ('liba_ep', lp['e_pt'], np.int32),
                          ('liba_ek', lp['e_kf'], np.int32)):
        (tmp_path / (name + '.raw')).write_bytes(np.ascontiguousarray(arr, dt).tobytes())
    out = dict(l.split(' ', 1) for l in subprocess.check_output([exe, str(tmp_path), '480', '640']).decode().strip().splitlines())
    # extract
    mono, kps, desc = O.OracleExtractor()(img, (0, 1000))
    assert [int(v) for v in out['extract'].split()] == [mono, len(kps), _checksum(desc.tobytes())]
    # SearchByProjection, th = 15 then 30, both from a cleared frame
    sf = O.OracleExtractor().tables()
    matches = None
    for attempt, th in enumerate((15.0, 30.0)):
        om = np.full(len(kps), -1, np.int32); oc = np.zeros(len(kps), np.uint8)
        on = O.search_last_frame(kps, desc, sc['bounds'], sf['scale'], sc['Tcw'], sc['cam'], L, th, True, om, oc)
        assert [int(v) for v in out['match%d' % attempt].split()] == [on, _checksum(om.tobytes())]
        matches = om
    # PoseOptimization on the matches of the second attempt
    sel = np.flatnonzero(matches >= 0)
    fr = dict(pose=sc['Tcw'].astype(np.float64), cam=np.asarray(sc['cam'], np.float32), Xw=L['xyz'][matches[sel]].astype(np.float64),
              obs=np.stack([kps['x'][sel], kps['y'][sel]], 1).astype(np.float64), inv_sigma2=sf['inv_sigma2'][kps['octave'][sel]])
    ref = O.pose_optimization(fr)
    got = out['poseopt'].split()
    assert int(got[0]) == len(sel) and int(got[1]) == ref['inliers']
    assert np.allclose([float(v) for v in got[2:]], ref['pose'], atol=1e-8)
    # LocalBundleAdjustment: two identical solves, then one with the abort flag set (returns before optimising, src/Optimizer.cc:1406-1408)
    refl = O.lba_solve(p)
    for rep in (0, 1):
        g = out['lba%d' % rep].split()
        assert int(g[0]) == refl['iters'] and int(g[1]) == int(refl['stats'][3])
        assert abs(float(g[3]) - refl['poses'].sum()) < 1e-6 and abs(float(g[4]) - refl['points'].sum()) < 1e-5
    assert out['lba0'] == out['lba1']
    assert int(out['lba2'].split()[0]) == -1          # untouched result: the call returned at the stop-flag test
    # LocalInertialBA: the mirror derives iterations / lambda / Huber flags from (bLarge, bRecInit) like src/Optimizer.cc:2387-2394,2497-2509,2633-2643
    for rec in (0, 1):
        q = dict(lp)
        q['ie_robust'] = np.array([1 if (i == lp['n_opt'] - 1 or rec) else 0 for i in range(lp['n_opt'])], np.uint8)
        w = O.local_inertial_ba(q, lP)
        g = out['liba%d' % rec].split()
        assert [int(v) for v in g[:4]] == [0 if w['failed'] else 1, w['iters'], w['trials'], int(w['erase'].sum())]
        assert abs(float(g[4]) - w['state'][:lp['n_opt']].sum()) < 1e-6 and abs(float(g[5]) - w['err_end']) <= 1e-5 * w['err_end']
