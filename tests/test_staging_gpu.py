"""The host entry points stage their operands through one growing device buffer + pinned mirror per owner (csrc/staging.h): a matcher
handle's is shared by all its host calls, and the stateless batch entry points share one per host thread.  Calls of growing, then
shrinking, size through one owner must each equal the CPU oracle."""
import numpy as np
import pytest

import frustum_scenes
import matcher_scenes as S
import new_points_lib as NP
import oracle_lib as O
from orb_slam3_modified_b200 import synth
import test_inertial_gpu as TI
from test_local_inertial_ba_cpu import _same_solve

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def orb():
    import orb_slam3_modified_b200 as m
    m.lib()
    return m


def _bow(orb, m, t):
    voc = O.synthetic_vocabulary(10, 4, seed=14)
    rng = np.random.default_rng(t)
    kk, dk = S.extract(t); kf, df = S.extract(t + 1)
    fvk = O.bow_transform(voc, dk, 2)[2:]; fvf = O.bow_transform(voc, df, 2)[2:]
    kf_point = rng.choice([0, 1, 1, 1, 1, 2], len(kk)).astype(np.uint8)
    n, match = m.SearchByBoW(kk, dk, kf_point, fvk, kf, df, fvf)
    on, om = O.search_by_bow(kk, dk, kf_point, fvk, kf, df, fvf, nnratio=m.mfNNratio, check_ori=m.mbCheckOrientation)
    assert n == on and np.array_equal(match, om), (n, on)


def _fuse(m, t, M):
    sc = O.fuse_scene(t, M=M)
    bi, bd = m.FuseSearch(sc['kps'], sc['desc'], sc['bounds'], sc['sf'], sc['isg'], sc['log_sf'], sc['Tcw'], sc['Ow'], sc['cam'], sc['state'], sc['xyz'],
                          sc['normal'], sc['min_d'], sc['max_d'], sc['mp_desc'], 3.0)
    obi, obd = O.fuse_search(sc, 3.0)
    assert np.array_equal(bi, obi) and np.array_equal(bd, obd)


def _triangulation(m, t, dts):
    scs = [O.triangulation_scene(t, dt) for dt in dts]
    kf1 = dict(kps=scs[0]['k1'], desc=scs[0]['d1'], has_mp=scs[0]['mp1'], fv=scs[0]['fv1'])
    for sc in scs:
        sc['mp1'] = scs[0]['mp1']
    geo = [O.triangulation_geometry(sc) for sc in scs]
    kf2 = [dict(kps=sc['k2'], desc=sc['d2'], has_mp=sc['mp2'], fv=sc['fv2']) for sc in scs]
    nm, m12 = m.SearchForTriangulation(kf1, kf2, scs[0]['sf'], scs[0]['sigma2'], np.array([g[0] for g in geo], np.float32).reshape(-1, 2),
                                       np.array([g[1] for g in geo], np.float32).reshape(-1, 9), False)
    for k, sc in enumerate(scs):
        on, om = O.search_for_triangulation(sc, geo[k][0], geo[k][1], False, m.mbCheckOrientation)
        assert nm[k] == on and np.array_equal(m12[k], om), (k, nm[k], on)


def _new_points(m, dts):
    sc = NP.scene(18, dts)
    rec, nm, nc = m.CreateNewMapPoints(sc['kf1'], sc['kf2'], sc['sf'], sc['sigma2'], sc['ep'], sc['F12'], sc['Tcw'], sc['Ow'], sc['cam'], sc['scale_factor'])
    orec, onm, onc, _ = NP.create(sc, False, False, 0.0)
    assert len(rec) > 0 and rec.tobytes() == orec.tobytes() and np.array_equal(nm, onm) and np.array_equal(nc, onc)


def _frustum(m, M, seed):
    sc = frustum_scenes.scene(M, seed)
    ref = O.is_in_frustum(**sc)
    out = m.isInFrustum(sc['pts'], sc['Rcw'], sc['tcw'], sc['Ow'], sc['cam'], sc['bounds'], sc['log_scale_factor'], sc['n_levels'], 0.5, sc['mbf'])
    for k in ('inView', 'projX', 'projY', 'projXR', 'depth', 'level', 'viewCos'):
        assert out[k].tobytes() == ref[k].tobytes(), k


def _knn(m, Q, T, seed):
    rng = np.random.default_rng(seed)
    q = rng.integers(0, 256, (Q, 32)).astype(np.uint8)
    t = rng.integers(0, 256, (T, 32)).astype(np.uint8)
    q[:min(Q, T) // 2] = t[:min(Q, T) // 2]
    idx, dist = m.knnMatch2(q, t)
    oi, od = O.bf_knn2(q, t)
    assert np.array_equal(idx, oi) and np.array_equal(dist, od), (Q, T)
    b = q[rng.permutation(Q)]
    assert np.array_equal(m.DescriptorDistance(q, b), np.unpackbits(q ^ b, axis=1).sum(1))


def _batch_search_last(orb, m):
    """The host batch search (its own fixed device staging) after the handle's staging has grown and shrunk."""
    scenes = [S.last_frame_scene(5 + 7 * b, seed=b % 2) for b in range(2)]
    B, kcap, mcap = 2, 1100, 1100
    kps = np.zeros((B, kcap), orb.KP_DTYPE); desc = np.zeros((B, kcap, 32), np.uint8); nK = np.zeros(B, np.int32)
    nM = np.zeros(B, np.int32); valid = np.zeros((B, mcap), np.uint8); xyz = np.zeros((B, mcap, 3), np.float32)
    octv = np.zeros((B, mcap), np.int32); ang = np.zeros((B, mcap), np.float32); obs = np.zeros((B, mcap), np.uint8)
    mpd = np.zeros((B, mcap, 32), np.uint8); Tcw = np.zeros((B, 7), np.float32)
    for b, s in enumerate(scenes):
        k, n = len(s['kps']), len(s['last']['valid'])
        nK[b], nM[b] = k, n
        kps[b, :k], desc[b, :k] = s['kps'], s['desc']
        L = s['last']
        valid[b, :n], xyz[b, :n], octv[b, :n], ang[b, :n], obs[b, :n], mpd[b, :n] = L['valid'], L['xyz'], L['octave'], L['angle'], L['hasObs'], L['descriptors']
        Tcw[b] = s['Tcw']
    d = dict(batch=B, kcap=kcap, mcap=mcap, nlevels=8, kps=kps, desc=desc, nK=nK, scaleFactors=scenes[0]['sf'], nM=nM, valid=valid, xyz=xyz,
             octave=octv, angle=ang, hasObs=obs, mpDesc=mpd, Tcw7=Tcw, bounds=(0.0, 0.0, 640.0, 480.0), cam=[float(c) for c in scenes[0]['cam']])
    match = np.full((B, kcap), -1, np.int32); claimed = np.zeros((B, kcap), np.uint8); nm = np.zeros(B, np.int32)
    m.mbCheckOrientation = True
    m.search_last_frame_batch(d, 15.0, match, claimed, nm)
    for b, s in enumerate(scenes):
        k = len(s['kps'])
        om = np.full(k, -1, np.int32); oc = np.zeros(k, np.uint8)
        on = O.search_last_frame(s['kps'], s['desc'], s['bounds'], s['sf'], s['Tcw'], s['cam'], s['last'], 15.0, True, om, oc)
        assert nm[b] == on and np.array_equal(match[b, :k], om) and np.array_equal(claimed[b, :k], oc), b


def test_one_matcher_grows_and_shrinks(orb):
    m = orb.ORBmatcher(0.6, False, max_batch=2, max_keypoints=2048, max_mappoints=4096)
    _knn(m, 40, 50, 0)                                                           # the first host call allocates the staging
    _bow(orb, m, 3)
    _fuse(m, 6, 300)
    _triangulation(m, 4, (3, -2))
    _new_points(m, (2, -2, 4, -4, 6))
    _fuse(m, 14, 9000)                                                           # grows
    _new_points(m, tuple(d for a in range(1, 16) for d in (a, -a)))
    _frustum(m, 4096, 2)                                                         # M == max_mappoints
    _knn(m, 3000, 3000, 1)
    _knn(m, 7, 2, 2)                                                             # shrinks
    _frustum(m, 257, 1)
    _fuse(m, 23, 300)
    _triangulation(m, 11, (2,))
    _new_points(m, (3,))
    _bow(orb, m, 8)
    _batch_search_last(orb, m)
    with pytest.raises(orb.OrbError) as e:
        _frustum(m, 4097, 3)                                                     # the frustum test is bounded by max_mappoints
    assert e.value.code == orb.ORB_ERR_CAPACITY
    _frustum(m, 1, 0)


def test_knn_beyond_handle_capacities(orb):
    """knnMatch2 / DescriptorDistance are not bounded by max_keypoints / max_mappoints."""
    m = orb.ORBmatcher(0.6, True, max_batch=1, max_keypoints=1024, max_mappoints=1024)
    _knn(m, 8192, 8192, 4)
    _knn(m, 100, 20000, 5)


def _pose_opt(orb, frames, refs):
    for out, ref in zip(orb.PoseOptimization(frames), refs):
        assert out['inliers'] == ref['inliers'] and np.array_equal(out['outlier'], ref['outlier']) and np.allclose(out['pose'], ref['pose'], atol=1e-9)


def _preint(orb, n):
    acc = np.zeros((n, 48, 3), np.float32); gyr = np.zeros((n, 48, 3), np.float32); dt = np.zeros((n, 48), np.float32); nm = np.zeros(n, np.int32)
    bias = np.tile(np.array((0.02, -0.01, 0.03, 0.002, -0.001, 0.0015), np.float32), (n, 1))
    for e in range(n):
        a, g, d = synth.imu_interval(0.3 + 0.37 * e, 0.3 + 0.37 * e + 1 / 30, seed=e)
        k = len(d)
        acc[e, :k], gyr[e, :k], dt[e, :k], nm[e] = a, g, d, k
    P = orb.imu_preintegrate(acc, gyr, dt, nm, bias, synth.IMU_NOISE)
    info = orb.imu_information(P)[0]
    for e in range(n):
        Po = O.imu_preintegrate(acc[e, :nm[e]], gyr[e, :nm[e]], dt[e, :nm[e]], bias[e], synth.IMU_NOISE)
        assert P[e, 0] == Po[0] and np.abs(P[e, 1:61] - Po[1:61]).max() < 2e-6
        gi = O.imu_information(P[e])[0]
        assert np.abs(info[e] - gi).max() < 1e-9 * np.abs(gi).max()


def _inertial_last_kf(orb, prs, frames, refs):
    for g, want in zip(orb.PoseInertialOptimizationLastKeyFrame(frames, prs[0]['extr']), refs):
        assert np.array_equal(g['outlier'], want['outlier']) and g['ret'] == want['ret'] and np.abs(g['state'] - want['state']).max() < 1e-6
        assert np.abs(g['H'] - want['H']).max() <= 1e-6 * np.abs(want['H']).max()


def _inertial_last_frame(orb, prs, frames, refs):
    for g, want in zip(orb.PoseInertialOptimizationLastFrame(frames, prs[0]['extr']), refs):
        assert np.array_equal(g['outlier'], want['outlier']) and g['ret'] == want['ret'] and np.abs(g['state'] - want['state']).max() < 1e-6
        assert np.abs(g['prev_state'] - want['prev_state']).max() < 1e-6 and np.abs(g['H'] - want['H']).max() <= 1e-5 * np.abs(want['H']).max()


def test_thread_staging_shared_by_the_batch_entry_points(orb):
    """One host thread alternates preintegration + information, the inertial and mono-IMU edges, PoseOptimization, both inertial pose
    optimisers and LocalInertialBA; the batch sizes grow and shrink, and every call goes through the thread's one staging buffer.  The edge
    calls (test_inertial_gpu's checks) run with and without information / Jacobians, i.e. with chi2 / rho / J downloaded or not."""
    po = [synth.pose_opt_problem(n=n, seed=s, outlier_frac=0.2) for s, n in enumerate((400, 900, 60, 300, 700, 9))]
    po_ref = [O.pose_optimization(f) for f in po]
    kf = [synth.pose_inertial_problem(seed=s, n=n, outlier_frac=0.1) for s, n in enumerate((300, 700, 40, 200, 500, 5))]
    kf_fr = [dict(pr, preint=O.imu_preintegrate(pr['acc'], pr['gyr'], pr['dt'], pr['bias6'], synth.IMU_NOISE)) for pr in kf]
    kf_ref = [O.pose_inertial_opt_last_kf(pr, fr['preint']) for pr, fr in zip(kf, kf_fr)]
    lf = [synth.pose_inertial_problem_last_frame(seed=s, n=n, outlier_frac=0.1) for s, n in enumerate((300, 700, 40, 250, 500, 4))]
    lf_fr = [dict(pr, preint_frame=O.imu_preintegrate(pr['acc'], pr['gyr'], pr['dt'], pr['bias6'], synth.IMU_NOISE),
                  preint_kf=O.imu_preintegrate(pr['acc_kf'], pr['gyr_kf'], pr['dt_kf'], pr['bias6'], synth.IMU_NOISE)) for pr in lf]
    lf_ref = [O.pose_inertial_opt_last_frame(pr, fr['preint_frame'], fr['preint_kf']) for pr, fr in zip(lf, lf_fr)]
    liba = []
    for kw in (dict(n_opt=6, n_cov_fixed=2, n_pts=250, seed=21), dict(n_opt=10, n_cov_fixed=3, n_pts=400, seed=1), dict(n_opt=4, n_cov_fixed=0, n_pts=120, seed=6)):
        pr = synth.local_inertial_ba_problem(**kw)
        pr['preint'] = O.liba_preints(pr)
        liba.append(pr)
    liba_ref = [O.local_inertial_ba(pr, pr['preint']) for pr in liba]
    for n, nl in ((1, 1), (6, 3), (2, 1), (6, 2), (1, 1)):
        _preint(orb, 4 * n)
        _pose_opt(orb, po[:n], po_ref[:n])
        _inertial_last_kf(orb, kf, kf_fr[:n], kf_ref[:n])
        for g, pr, want in zip(orb.LocalInertialBA(liba[:nl]), liba, liba_ref):
            _same_solve(g, want, pr)
        TI.test_edge_inertial_residuals_jacobians_chi2(orb)
        _inertial_last_frame(orb, lf, lf_fr[:n], lf_ref[:n])
        TI.test_edge_mono_imu(orb)
