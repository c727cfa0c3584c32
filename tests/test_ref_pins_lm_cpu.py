"""CPU: the control flow of the oracle's Levenberg-Marquardt loops equals g2o's own.  oracle/_ref/libref_g2o_lm.so holds the bodies of
OptimizationAlgorithmLevenberg::solve / computeLambdaInit / computeScale (Thirdparty/g2o/g2o/core/optimization_algorithm_levenberg.cpp:61-194) and
SparseOptimizer::optimize (sparse_optimizer.cpp:354-419), cut out of the reference checkout at build time and compiled verbatim against class shells whose
Solver / SparseOptimizer operations forward to a solver state of the oracle opened step by step (OrboLmBackend).  Running the reference's text over the
oracle's linear algebra must give, bit for bit, what the oracle's own loops give: iterations, Levenberg trials, lambda, poses / keyframe states, points --
for LocalBundleAdjustment (a20) and LocalInertialBA (f1), with the default and the user-given initial lambda, with rejected steps and with the stop flag."""
import ctypes as C
import os

import numpy as np
import pytest

import oracle_lib as O
from orb_slam3_modified_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, 'oracle', '_ref', 'libref_g2o_lm.so')
pytestmark = pytest.mark.skipif(not os.path.exists(SO), reason='oracle/_ref is not built here')


class Backend(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ('self', 'compute_errors', 'robust_chi2', 'build_system', 'solve', 'update', 'push', 'pop', 'vector_size', 'x', 'b', 'n_diag', 'diag')]


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _ref_optimize(be, iterations, lam0, stop=None):
    L = C.CDLL(SO)
    L.ref_g2o_optimize.argtypes = [C.c_void_p, C.c_int, C.c_double, C.c_void_p, C.c_void_p]
    stats = np.zeros(4)
    sf = np.array([1 if stop else 0], np.uint8)
    it = L.ref_g2o_optimize(C.byref(be), iterations, float(lam0), _p(sf) if stop is not None else None, _p(stats))
    return it, stats


def _lba_with_reference_lm(prob, iterations=10, lam0=0.0, stop=None):
    Lo = O.lib()
    c = lambda a, dt: np.ascontiguousarray(a, dt)
    a = [c(prob['poses'], np.float64), c(prob['fixed'], np.uint8), c(prob['cam'], np.float32), c(prob['points'], np.float64), c(prob['edge_point'], np.int32),
         c(prob['edge_pose'], np.int32), c(prob['obs'], np.float64), c(prob['inv_sigma2'], np.float32)]
    be = Backend()
    Lo.orbo_lba_backend_open.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_void_p]
    Lo.orbo_lba_backend_open(len(a[0]), _p(a[0]), _p(a[1]), _p(a[2]), len(a[3]), _p(a[3]), len(a[4]), _p(a[4]), _p(a[5]), _p(a[6]), _p(a[7]),
                             float(np.float32(np.sqrt(5.991))), C.byref(be))
    it, stats = _ref_optimize(be, iterations, lam0, stop)
    poses = np.zeros_like(a[0]); pts = np.zeros_like(a[3])
    Lo.orbo_lba_backend_close.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    Lo.orbo_lba_backend_close(C.byref(be), _p(poses), _p(pts))
    return it, stats, poses, pts


def test_local_bundle_adjustment_loop():
    cases = [dict(n_kf=6, n_pts=300, obs_per_pt=5, seed=3), dict(n_kf=12, n_pts=800, obs_per_pt=6, seed=5, n_fixed=3), dict(n_kf=8, n_pts=400, obs_per_pt=4, seed=8, outlier_frac=0.2)]
    for kw in cases:
        prob = synth.lba_problem(**kw)
        for lam0 in (0.0, 1e-12, 1e3):
            want = O.lba_solve(prob, iterations=10, user_lambda_init=lam0)
            it, stats, poses, pts = _lba_with_reference_lm(prob, 10, lam0)
            assert it == want['iters'] and int(stats[1]) == int(want['stats'][3]) and stats[0] == want['stats'][0], (kw, lam0, it, want['iters'], stats, want['stats'][:4])
            assert poses.tobytes() == want['poses'].tobytes() and pts.tobytes() == want['points'].tobytes()
    # rejected trials happened somewhere in the sweep above? make sure of one case explicitly
    prob = synth.lba_problem(n_kf=6, n_pts=300, obs_per_pt=5, seed=3)
    want = O.lba_solve(prob, iterations=10, user_lambda_init=1e-12)
    assert int(want['stats'][3]) >= want['iters']
    # the stop flag set before the first iteration: optimize() returns 0 iterations and leaves the state alone
    it, stats, poses, pts = _lba_with_reference_lm(prob, 10, 0.0, stop=True)
    assert it == 0 and np.array_equal(pts, prob['points'])


def test_local_inertial_ba_loop():
    Lo = O.lib()
    for kw in (dict(n_opt=6, n_cov_fixed=2, n_pts=250, seed=21), dict(n_opt=10, n_cov_fixed=3, n_pts=400, seed=1), dict(n_opt=8, n_cov_fixed=1, n_pts=300, seed=3, large=True),
               dict(n_opt=5, n_cov_fixed=1, n_pts=150, seed=9, perturb=12.0, lambda_init=1e-12)):
        lam = kw.pop('lambda_init', None)
        pr = synth.local_inertial_ba_problem(**kw)
        if lam is not None:
            pr['lambda_init'] = lam
        P = O.liba_preints(pr)
        want = O.local_inertial_ba(pr, P)
        c = lambda a, dt: np.ascontiguousarray(a, dt)
        a = dict(st=c(pr['state'], np.float64), tc=c(pr['tcw'], np.float64), cam=c(pr['cam'], np.float32), ex=c(pr['extr'], np.float64), k1=c(pr['ie_kf1'], np.int32),
                 k2=c(pr['ie_kf2'], np.int32), P=c(P, np.float32), rob=c(pr['ie_robust'], np.uint8), sc=c(pr['ie_info_scale'], np.float64), pts=c(pr['points'], np.float64),
                 ep=c(pr['e_pt'], np.int32), ek=c(pr['e_kf'], np.int32), obs=c(pr['obs'], np.float64), isg=c(pr['inv_sigma2'], np.float32))
        be = Backend()
        Lo.orbo_liba_backend_open.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 4 + [C.c_int] + [C.c_void_p] * 5 + [C.c_int, C.c_void_p, C.c_int] + [C.c_void_p] * 4 + [C.c_void_p]
        Lo.orbo_liba_backend_open(pr['n_kf'], pr['n_opt'], _p(a['st']), _p(a['tc']), _p(a['cam']), _p(a['ex']), len(a['k1']), _p(a['k1']), _p(a['k2']), _p(a['P']), _p(a['rob']),
                                  _p(a['sc']), len(a['pts']), _p(a['pts']), len(a['ep']), _p(a['ep']), _p(a['ek']), _p(a['obs']), _p(a['isg']), C.byref(be))
        Lo.orbo_imu_information  # (the information matrices are built inside open)
        # LocalInertialBA calls computeActiveErrors() once before optimize() (:2836); harmless for the state, kept for the order of calls
        it, stats = _ref_optimize(be, pr['iterations'], pr['lambda_init'])
        st = np.zeros_like(a['st']); pts = np.zeros_like(a['pts'])
        Lo.orbo_liba_backend_close.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        Lo.orbo_liba_backend_close(C.byref(be), _p(st), _p(pts))
        assert not want['failed']
        assert it == want['iters'] and int(stats[1]) == want['trials'] and stats[0] == want['lam'], (kw, it, want['iters'], stats, want['trials'], want['lam'])
        assert st.tobytes() == want['state'].tobytes() and pts.tobytes() == want['points'].tobytes()


def test_pose_optimization_four_rounds():
    """Optimizer::PoseOptimization: the reference's own four-round loop (src/Optimizer.cc:996-1104) + g2o's optimize() / Levenberg text over the oracle's
    pose-only state == the oracle's orbo_pose_optimization: same return value, outlier flags and pose bit for bit (many outliers, few points, < 10 edges, < 3 edges)."""
    L = C.CDLL(SO)
    O.lib()
    L.ref_pose_optimization.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_void_p]
    cases = [dict(n=300, seed=4), dict(n=700, seed=1, outlier_frac=0.35), dict(n=40, seed=2, outlier_frac=0.3), dict(n=9, seed=3, outlier_frac=0.0), dict(n=2, seed=5, outlier_frac=0.0),
             dict(n=200, seed=6, pose_noise=(0.3, 10.0)), dict(n=12, seed=7, outlier_frac=0.6)]
    for kw in cases:
        fr = synth.pose_opt_problem(**kw)
        want = O.pose_optimization(fr)
        pose = np.ascontiguousarray(fr['pose'], np.float64).copy()
        cam = np.ascontiguousarray(fr['cam'], np.float32); X = np.ascontiguousarray(fr['Xw'], np.float64); ob = np.ascontiguousarray(fr['obs'], np.float64)
        isg = np.ascontiguousarray(fr['inv_sigma2'], np.float32)
        out = np.zeros(len(X), np.uint8)
        ret = L.ref_pose_optimization(_p(pose), _p(cam), len(X), _p(X), _p(ob), _p(isg), float(np.float32(np.sqrt(5.991))), _p(out))
        assert ret == want['inliers'] and np.array_equal(out, want['outlier']), (kw, ret, want['inliers'])
        assert pose.tobytes() == np.ascontiguousarray(want['pose'], np.float64).tobytes(), (kw, np.abs(pose - want['pose']).max())


def test_local_inertial_ba_from_initialize_to_the_fail_test():
    """Optimizer::LocalInertialBA's own text from optimizer.initializeOptimization() to the FAIL test (src/Optimizer.cc:2840-2895: err, optimize(opt_it), err_end, the chi2 /
    depth test that fills vToErase, 2*err < err_end) over the oracle's state == orbo_local_inertial_ba: err, err_end, failed, erase flags, lambda."""
    Lo = O.lib(); L = C.CDLL(SO)
    L.ref_local_inertial_ba_tail.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_int, C.c_void_p, C.c_void_p]
    cases = [dict(n_opt=6, n_cov_fixed=2, n_pts=250, seed=21), dict(n_opt=10, n_cov_fixed=3, n_pts=400, seed=1), dict(n_opt=8, n_cov_fixed=1, n_pts=300, seed=3, large=True),
             dict(n_opt=4, n_cov_fixed=1, n_pts=120, seed=33, nan_obs=True)]
    seen_fail = False
    for kw in cases:
        nan_obs = kw.pop('nan_obs', False)
        pr = synth.local_inertial_ba_problem(**kw)
        if nan_obs:
            pr['obs'][5, 0] = np.nan                     # isnan(err): the FAIL branch (:2891) -- an LM run itself never ends above twice its start
        P = O.liba_preints(pr)
        want = O.local_inertial_ba(pr, P)
        c = lambda a, dt: np.ascontiguousarray(a, dt)
        a = dict(st=c(pr['state'], np.float64), tc=c(pr['tcw'], np.float64), cam=c(pr['cam'], np.float32), ex=c(pr['extr'], np.float64), k1=c(pr['ie_kf1'], np.int32),
                 k2=c(pr['ie_kf2'], np.int32), P=c(P, np.float32), rob=c(pr['ie_robust'], np.uint8), sc=c(pr['ie_info_scale'], np.float64), pts=c(pr['points'], np.float64),
                 ep=c(pr['e_pt'], np.int32), ek=c(pr['e_kf'], np.int32), obs=c(pr['obs'], np.float64), isg=c(pr['inv_sigma2'], np.float32), td=c(pr['track_depth'], np.float32))
        be = Backend()
        Lo.orbo_liba_backend_open.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 4 + [C.c_int] + [C.c_void_p] * 5 + [C.c_int, C.c_void_p, C.c_int] + [C.c_void_p] * 4 + [C.c_void_p]
        Lo.orbo_liba_backend_open(pr['n_kf'], pr['n_opt'], _p(a['st']), _p(a['tc']), _p(a['cam']), _p(a['ex']), len(a['k1']), _p(a['k1']), _p(a['k2']), _p(a['P']), _p(a['rob']),
                                  _p(a['sc']), len(a['pts']), _p(a['pts']), len(a['ep']), _p(a['ep']), _p(a['ek']), _p(a['obs']), _p(a['isg']), C.byref(be))
        erase = np.zeros(len(a['ep']), np.uint8); stats = np.zeros(4)
        L.ref_local_inertial_ba_tail(C.byref(be), len(a['ep']), _p(a['ep']), _p(a['td']), len(a['pts']), pr['iterations'], float(pr['lambda_init']), int(pr['large']), _p(erase), _p(stats))
        st = np.zeros_like(a['st']); pts = np.zeros_like(a['pts'])
        Lo.orbo_liba_backend_close.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        Lo.orbo_liba_backend_close(C.byref(be), _p(st), _p(pts))
        same = lambda x, y: (x == y) or (np.isnan(x) and np.isnan(y))
        assert same(stats[0], want['err']) and same(stats[1], want['err_end']) and bool(stats[2]) == want['failed'] and same(stats[3], want['lam']), (kw, stats, want['err'], want['err_end'], want['failed'])
        seen_fail |= want['failed']
        if not want['failed']:
            assert np.array_equal(erase, want['erase']) and st.tobytes() == want['state'].tobytes()
        else:                                                # on FAIL the text returns before it erases (:2884-2888): the oracle hands the inputs back and sets no flag
            assert np.array_equal(want['state'], pr['state']) and want['erase'].sum() == 0
    assert seen_fail


def test_pose_inertial_optimization_last_keyframe_rounds():
    """Optimizer::PoseInertialOptimizationLastKeyFrame: the reference's own four rounds + recovery of not-too-bad points (src/Optimizer.cc:4698-4823) with g2o's
    Gauss-Newton / optimize() text over the oracle's state == orbo_pose_inertial_opt_last_kf: return value, outlier flags and the frame's state bit for bit
    (outliers, few points incl. fewer than 10 edges and the < 30 inliers recovery, bRecInit)."""
    L = C.CDLL(SO)
    L.ref_pose_inertial_opt_last_kf.argtypes = [C.c_int] + [C.c_void_p] * 9 + [C.c_int, C.c_void_p]
    cases = [dict(seed=0, n=300, outlier_frac=0.1), dict(seed=1, n=700, outlier_frac=0.2), dict(seed=2, n=40, outlier_frac=0.3), dict(seed=3, n=5, outlier_frac=0.0),
             dict(seed=5, n=1000, outlier_frac=0.05, perturb=2.0), dict(seed=6, n=25, outlier_frac=0.4)]
    for kw in cases:
        pr = synth.pose_inertial_problem(**kw)
        P = O.imu_preintegrate(pr['acc'], pr['gyr'], pr['dt'], pr['bias6'], synth.IMU_NOISE)
        for rec in (False, True):
            want = O.pose_inertial_opt_last_kf(pr, P, rec_init=rec)
            c = lambda a, dt: np.ascontiguousarray(a, dt)
            a = [c(pr['Xw'], np.float32), c(pr['obs'], np.float32), c(pr['inv_sigma2'], np.float32), c(pr['track_depth'], np.float32), c(pr['cam'], np.float32), c(pr['extr'], np.float64),
                 c(P, np.float32), c(pr['kf_state'], np.float64)]
            st = c(pr['state'], np.float64).copy(); out = np.zeros(len(a[0]), np.uint8)
            ret = L.ref_pose_inertial_opt_last_kf(len(a[0]), *[_p(x) for x in a], _p(st), int(rec), _p(out))
            assert ret == want['ret'] and np.array_equal(out, want['outlier']), (kw, rec, ret, want['ret'])
            assert st.tobytes() == want['state'].tobytes(), (kw, rec, np.abs(st - want['state']).max())


def test_pose_inertial_optimization_last_frame_rounds():
    """Optimizer::PoseInertialOptimizationLastFrame: the reference's own four rounds + recovery (src/Optimizer.cc:5098-5221) with g2o's Gauss-Newton text over the oracle's
    30-unknown state (prior edge included) == orbo_pose_inertial_opt_last_frame: return value, outlier flags, both frames' states bit for bit.  (The marginalisation that
    follows needs Eigen's JacobiSVD and stays with the oracle's own derivation.)"""
    L = C.CDLL(SO)
    L.ref_pose_inertial_opt_last_frame.argtypes = [C.c_int] + [C.c_void_p] * 12 + [C.c_int, C.c_void_p]
    cases = [dict(seed=0, n=300, outlier_frac=0.1), dict(seed=1, n=700, outlier_frac=0.2), dict(seed=2, n=40, outlier_frac=0.3), dict(seed=3, n=4, outlier_frac=0.0),
             dict(seed=5, n=1000, outlier_frac=0.05, perturb=2.0), dict(seed=7, n=250, outlier_frac=0.1, prior_sigma=(2e-2, 5e-2, 1e-1, 1e-3, 1e-2))]
    for kw in cases:
        pr = synth.pose_inertial_problem_last_frame(**kw)
        Pf = O.imu_preintegrate(pr['acc'], pr['gyr'], pr['dt'], pr['bias6'], synth.IMU_NOISE)
        Pk = O.imu_preintegrate(pr['acc_kf'], pr['gyr_kf'], pr['dt_kf'], pr['bias6'], synth.IMU_NOISE)
        for rec in (False, True):
            want = O.pose_inertial_opt_last_frame(pr, Pf, Pk, rec_init=rec)
            c = lambda a, dt: np.ascontiguousarray(a, dt)
            a = [c(pr['Xw'], np.float32), c(pr['obs'], np.float32), c(pr['inv_sigma2'], np.float32), c(pr['track_depth'], np.float32), c(pr['cam'], np.float32), c(pr['extr'], np.float64),
                 c(Pf, np.float32), c(Pk, np.float32), c(pr['prior_state'], np.float64), c(pr['prior_H'], np.float64)]
            pv = c(pr['prev_state'], np.float64).copy(); st = c(pr['state'], np.float64).copy(); out = np.zeros(len(a[0]), np.uint8)
            ret = L.ref_pose_inertial_opt_last_frame(len(a[0]), *[_p(x) for x in a], _p(pv), _p(st), int(rec), _p(out))
            assert ret == want['ret'] and np.array_equal(out, want['outlier']), (kw, rec, ret, want['ret'])
            assert st.tobytes() == want['state'].tobytes() and pv.tobytes() == want['prev_state'].tobytes(), (kw, rec)
