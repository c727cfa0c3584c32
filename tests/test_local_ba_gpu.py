"""GPU tests of lba_local_bundle_adjustment_batch (Optimizer::LocalBundleAdjustment as a whole) against the CPU oracle
(oracle/local_ba_oracle.cpp) and against lba_solve_batch, at 1 / 7 / 24 maps, mono and inertial, with NO_FIXED, STOPPED and empty maps
mixed in."""
import os
import subprocess

import numpy as np
import pytest

import local_ba_lib as LB
import oracle_lib as O
import orb_slam3_modified_b200 as orb

pytestmark = pytest.mark.gpu

KEYS = ('status', 'num_fixedKF', 'num_OptKF', 'num_MPs', 'num_edges')
LISTS = ('localKF', 'fixedKF', 'localPoint', 'obsFlag')
FINISH = ('obsFlag', 'kfPose7', 'kfCenter', 'pointPos', 'pointBad', 'pointRefKF', 'normal', 'minDistance', 'maxDistance')


def _empty(init):
    M = LB.Map()
    M.kfs[0] = LB.KeyFrame(0, 3, np.array([1, 0, 0, 0, 0, 0, 0], np.float32), np.array([500, 480, 320, 240], np.float32), np.zeros((0, 2)), [])
    M.kfs[0].init = init
    M.cov[0] = []
    return M, 0


def _maps(n, seed=0):
    P = LB.planted()
    extra = [P['no_fixed'], P['stopped'], _empty(False), _empty(True), P['mixed'], P['init_only'], P['hub_fixed']]
    out = []
    for i in range(n):
        if i % 4 == 3 and extra:
            out.append(extra.pop(0))
        else:
            s = seed + 100 + i
            while True:                             # a scene whose oracle chi2 all clear 5.991 by the margin
                M, k = LB.scene(s, n_kf=10 + i % 5, n_pts=300 + 40 * (i % 3), obs_per_pt=4 + i % 3, n_cov=4 + i % 3, outlier_frac=0.06,
                                inertial=i % 2 == 1)
                try:
                    LB.check_margin(LB.oracle(LB.flatten(M, k))[0])
                    break
                except AssertionError:
                    s += 1000
            out.append((M, k))
    return out


def _opt(n):
    return orb.Optimizer(max_poses=32, max_points=1024, max_edges=8192, max_batch=max(n, 1))


@pytest.mark.parametrize('n', [1, 7, 24])
def test_batch_against_oracle_and_solver(n):
    maps = _maps(n)
    flat = [LB.flatten(M, k) for M, k in maps]
    opt = _opt(n)
    got = opt.local_bundle_adjustment_batch(flat, debug=True)
    assert opt.local_last_launches() in (2, 5)
    probs, where = [], []
    for j, (m, g) in enumerate(zip(flat, got)):
        ref, built = LB.oracle(m)
        for k in KEYS:
            assert g[k] == ref[k], (j, k)
        for k in ('localKF', 'fixedKF', 'localPoint'):
            assert np.array_equal(g[k], ref[k]), (j, k)
        if g['status'] != orb.LBA_LOCAL_RAN:
            assert not g['obsFlag'].any() and g['lmStats'][0] == -1
            continue
        # the GPU's own double results finished by the oracle: bit for bit
        fin, _ = LB.oracle(m, given=dict(optPose=np.pad(g['optPose'], ((0, len(m['kfFlags']) - len(g['optPose'])), (0, 0))),
                                         optPoint=np.pad(g['optPoint'], ((0, len(m['pointFlags']) - len(g['optPoint'])), (0, 0))),
                                         edgeChi2=g['edgeChi2'], edgeDepthPositive=g['edgeDepthPositive']))
        for k in FINISH:
            assert g[k].tobytes() == fin[k].tobytes(), (j, k)
        LB.check_margin(ref)
        # the whole chain against the CPU oracle chain
        if g['lmStats'][0] >= 0:
            assert np.array_equal(g['obsFlag'], ref['obsFlag']) and np.array_equal(g['pointBad'], ref['pointBad'])
            pb = dict(built, poses=built['poses'], points=built['points'])
            vk = {kk: v for v, kk in enumerate(built['vert_kf'])}
            vp = {pp: v for v, pp in enumerate(built['vert_point'])}
            poses = built['poses'].copy(); pts = built['points'].copy()
            for i, kk in enumerate(g['localKF']):
                poses[vk[kk]] = g['optPose'][i]
            for i, pp in enumerate(g['localPoint']):
                pts[vp[pp]] = g['optPoint'][i]
            rposes = built['poses'].copy(); rpts = built['points'].copy()
            for i, kk in enumerate(ref['localKF']):
                rposes[vk[kk]] = ref['optPose'][i]
            for i, pp in enumerate(ref['localPoint']):
                rpts[vp[pp]] = ref['optPoint'][i]
            d = np.abs(O.lba_residuals(pb, poses, pts) - O.lba_residuals(pb, rposes, rpts)).max()
            assert d <= 1e-4, (j, d)
            probs.append(dict(built, fixed=built['fixed'])); where.append((j, vk, vp))
    # the LM outputs equal lba_solve_batch fed the oracle walk's problems, byte for byte
    # (the same batch in the same slot order, so that the solver picks the same cluster size)
    if probs:
        solver = _opt(len(probs))
        packs = [orb.Optimizer._pack(p, 10, 100.0 if flat[j]['inertial'] else 0.0, None) for p, (j, _, _) in zip(probs, where)]
        P = (orb._LbaProblem * len(packs))(*[k[1] for k in packs])
        R = (orb._LbaResult * len(packs))(*[k[3] for k in packs])
        assert orb.lib().lba_solve_batch(solver._h, len(packs), P, R) == orb.ORB_OK
        outs = [orb.Optimizer._finish(k[2], R[i]) for i, k in enumerate(packs)]
        for (j, vk, vp), o in zip(where, outs):
            g = got[j]
            assert o['iters'] == int(g['lmStats'][0]) and o['trials'] == int(g['lmStats'][1])
            for i, kk in enumerate(g['localKF']):
                assert o['poses'][vk[kk]].tobytes() == g['optPose'][i].tobytes()
            for i, pp in enumerate(g['localPoint']):
                assert o['points'][vp[pp]].tobytes() == g['optPoint'][i].tobytes()


def test_batch_equals_single_calls_and_solver_still_works():
    maps = _maps(7, seed=50)
    flat = [LB.flatten(M, k) for M, k in maps]
    opt = _opt(7)
    opt.set_cluster_size(4)                         # the cluster size orders the solver's reductions: the same for both
    batch = opt.local_bundle_adjustment_batch(flat, debug=True)
    for m, b in zip(flat, batch):
        one = opt.local_bundle_adjustment_batch([m], debug=True)[0]
        for k in set(one) & set(b):
            assert np.asarray(one[k]).tobytes() == np.asarray(b[k]).tobytes(), k
    # a later upload / run on the same handle gives its usual results
    _, built = LB.oracle(flat[0])
    prob = dict(built)
    opt.upload([prob])
    opt.run_device()
    after = opt.download()[0]
    fresh = _opt(1).LocalBundleAdjustmentBatch([prob])[0]
    assert after['poses'].tobytes() == fresh['poses'].tobytes() and after['points'].tobytes() == fresh['points'].tobytes()


def test_argument_and_capacity_errors():
    M, k = LB.scene(7, n_kf=10, n_pts=300, obs_per_pt=4, n_cov=4)
    m = LB.flatten(M, k)
    opt = orb.Optimizer(max_poses=32, max_points=1024, max_edges=8192, max_batch=2)
    for key, bad in (('obsKF', lambda a: np.where(np.arange(len(a)) == 3, len(m['kfFlags']), a)),
                     ('obsOctave', lambda a: np.where(np.arange(len(a)) == 0, 8, a)),
                     ('slotStart', lambda a: np.r_[1, a[1:]]),
                     ('obsStart', lambda a: np.r_[a[:2], a[1] - 1, a[3:]]),
                     ('cov', lambda a: np.r_[a, a[:1]]),
                     ('slotPoint', lambda a: np.where(np.arange(len(a)) == 0, len(m['pointFlags']), a))):
        mm = dict(m)
        mm[key] = bad(np.asarray(m[key]))
        with pytest.raises(orb.OrbError) as e:
            opt.local_bundle_adjustment_batch([m, mm])
        assert e.value.code == orb.ORB_ERR_ARG and 'map 1' in str(e.value), key
    # a keyframe listed twice among one point's observations, not next to each other
    p = next(q for q in range(len(m['pointFlags'])) if m['obsStart'][q + 1] - m['obsStart'][q] >= 3)
    mm = dict(m)
    mm['obsKF'] = np.array(m['obsKF'])
    mm['obsKF'][m['obsStart'][p] + 2] = mm['obsKF'][m['obsStart'][p]]
    with pytest.raises(orb.OrbError) as e:
        opt.local_bundle_adjustment_batch([m, mm])
    assert e.value.code == orb.ORB_ERR_ARG and 'map 1' in str(e.value) and 'twice' in str(e.value)
    with pytest.raises(orb.OrbError) as e:
        opt.local_bundle_adjustment_batch([m, m, m])
    assert e.value.code == orb.ORB_ERR_CAPACITY
    small = orb.Optimizer(max_poses=32, max_points=100, max_edges=8192, max_batch=2)
    with pytest.raises(orb.OrbError) as e:
        small.local_bundle_adjustment_batch([m])
    assert e.value.code == orb.ORB_ERR_CAPACITY and 'map 0' in str(e.value)


def test_config4_size_map():
    """A map of the benchmark's LBA size (18 keyframes, 11 free, ~4200 points, ~34k edges), whose solver launch needs about 47 KB of
    dynamic shared memory beside the kernel's static shared memory, through the whole function and through lba_solve_batch."""
    M, k = LB.scene(500, n_kf=20, n_pts=5000, obs_per_pt=8, n_cov=10, outlier_frac=0.03)
    m = LB.flatten(M, k)
    ref, built = LB.oracle(m)
    opt = orb.Optimizer(max_poses=64, max_points=8192, max_edges=65536, max_batch=1)
    g = opt.local_bundle_adjustment_batch([m], debug=True)[0]
    assert g['status'] == orb.LBA_LOCAL_RAN and g['num_edges'] == ref['num_edges'] > 30000
    assert np.array_equal(g['localPoint'], ref['localPoint']) and np.array_equal(g['fixedKF'], ref['fixedKF'])
    o = opt.LocalBundleAdjustmentBatch([built])[0]
    assert o['iters'] == int(g['lmStats'][0])


def _digest(res):
    """FNV-1a over what tests/local_ba_example.cpp hashes, in its order."""
    h = 14695981039346656037
    for r in res:
        parts = [np.int32(r['status']), np.asarray(r['counts'], np.int32), np.asarray(r['nLists'], np.int32), r['localKF'], r['fixedKF'], r['localPoint'],
                 r['obsFlag'], r['kfPose7'], r['kfCenter'], r['pointPos'], r['pointBad'], r['pointRefKF'], r['normal'], r['minDistance'],
                 r['maxDistance'], np.asarray(r['lmStats'], np.float64)]
        for b in b''.join(np.ascontiguousarray(x).tobytes() for x in parts):
            h = ((h ^ b) * 1099511628211) & 0xFFFFFFFFFFFFFFFF
    return h


def test_cpp_local_bundle_adjustment_batch_equals_python(tmp_path):
    """Optimizer::LocalBundleAdjustmentBatch (include/orb_b200/orb_slam3.hpp) from a g++-built caller gives the Python binding's digest."""
    flat = [LB.flatten(M, k) for M, k in _maps(7, seed=70)]
    caps = (32, 1024, 8192)
    lines = ['%d %d %d %d' % ((len(flat),) + caps)]
    for j, m in enumerate(flat):
        lines.append('%d %d %d %d %d' % (len(m['kfFlags']), len(m['cov']), len(m['pointFlags']), len(m['scaleFactors']), m['inertial']))
        for name, dt in orb.LOCAL_BA_ARRAYS + (('stop', np.uint8),):
            data = np.ascontiguousarray(m[name], dt).tobytes() if m.get(name) is not None else b''
            (tmp_path / ('map%d_%s.raw' % (j, name))).write_bytes(data)
    (tmp_path / 'dims.txt').write_text('\n'.join(lines) + '\n')
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib = os.path.join(root, 'orb_slam3_modified_b200')
    exe = tmp_path / 'local_ba_example'
    subprocess.check_call(['g++', '-std=c++14', '-O2', '-Wall', '-I', os.path.join(root, 'include'), os.path.join(root, 'tests', 'local_ba_example.cpp'),
                           '-o', str(exe), '-L', lib, '-l:liborb_b200.so', '-Wl,-rpath,' + lib, '-lpthread'])
    out = dict(l.split() for l in subprocess.check_output([str(exe), str(tmp_path)]).decode().splitlines())
    res = orb.Optimizer(*caps, max_batch=len(flat)).local_bundle_adjustment_batch(flat)
    assert out['digest'] == '%016x' % _digest(res)
    assert int(out['erased']) == sum(int((r['obsFlag'] == orb.LBA_OBS_ERASED).sum()) for r in res) > 10
    assert out['launches'] == '5'
