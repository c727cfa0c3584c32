"""CPU: the tracking pose optimisers' oracles on the frames of tests/pose_scenes.py.  Each frame reaches the branch it is named for, shown
from the oracle: the early return, the `edges().size() < 10` break (rounds run, or the same result with one round as with four), the
Levenberg-Marquardt stops after 10 rejected trials and on rho == 0 (iteration counters of orbo_pose_optimization), every edge excluded
from round two on, the `nInliers < 30` recovery (bRecInit off and on), the trackDepth == 10 close rule, the depth test, and the prior's
Huber kernel.  The oracle against independent evidence on these frames: PoseOptimization's second transcription
(test_poseopt_transcription_cpu.py takes the layouts as parameters), and the first Gauss-Newton step of both inertial optimisers = the
dense step from numerical derivatives (test_inertial_cpu.py's checks) on the frames where no Huber weight is active at the start."""
import numpy as np
import pytest

import oracle_lib as O
import pose_scenes as S
from test_inertial_cpu import _preints, check_first_step_last_frame, check_first_step_last_kf


def _same(a, b):
    return a['state'].tobytes() == b['state'].tobytes() and np.array_equal(a['outlier'], b['outlier']) and a['ret'] == b['ret']


# ---- PoseOptimization ----
def test_pose_optimization_layouts_reach_their_branches():
    r = {name: O.pose_optimization(f()) for name, f in S.PO_LAYOUTS.items()}
    for n in (0, 1, 2):                                     # nInitialCorrespondences < 3: nothing runs
        f = S.PO_LAYOUTS['n_%d' % n]()
        x = r['n_%d' % n]
        assert x['inliers'] == 0 and x['trials'] == 0 and x['rounds'] == 0 and len(x['outlier']) == n
        assert x['pose'].tobytes() == f['pose'].tobytes()
    assert r['n_3']['rounds'] == r['n_9']['rounds'] == 1 and r['n_10']['rounds'] == 4     # edges().size() < 10 ends after round one
    for n in (31, 32, 33, 255, 256, 257, 511, 512, 513, 4000):
        x = r['n_%d' % n]
        assert len(x['outlier']) == n and 0 < x['outlier'].sum() < n and x['rounds'] == 4
    # every edge a gross outlier: excluded after round one, so rounds two to four optimise nothing and the pose is the start pose
    f = S.PO_LAYOUTS['all_gross']()
    x = r['all_gross']
    q = f['pose'][:4] / np.linalg.norm(f['pose'][:4])
    assert x['inliers'] == 0 and x['outlier'].all() and np.abs(x['pose'] - np.concatenate([q, f['pose'][4:]])).max() < 1e-15
    assert r['noise_free']['rho_zero'] == 4 and r['noise_free']['outlier'].sum() == 0          # each round stops on rho == 0
    assert r['bad_start']['exhausted'] > 0                                                     # qmax == 10
    # points behind the camera project where they are observed (inliers), far points too; both kinds are present
    f = S.PO_LAYOUTS['behind_and_far']()
    z = S.depth(f)
    assert (z < 0).sum() == 12 and (z > 400).sum() == 12 and not r['behind_and_far']['outlier'][z < 0].any()
    f = S.PO_LAYOUTS['border']()
    on = (f['obs'][:, 0] == 0) | (f['obs'][:, 0] == S.W - 1) | (f['obs'][:, 1] == 0) | (f['obs'][:, 1] == S.H - 1)
    assert on.sum() == 40 and r['border']['outlier'][on].sum() < 10
    # a non-unit quaternion gives the result of its normalised copy (the SE3Quat constructor)
    f = S.PO_LAYOUTS['non_unit_quaternion']()
    assert abs(np.linalg.norm(f['pose'][:4]) - 1.37) < 1e-6
    g = dict(f, pose=np.concatenate([f['pose'][:4] / np.linalg.norm(f['pose'][:4]), f['pose'][4:]]))
    y = O.pose_optimization(g)
    assert y['inliers'] == r['non_unit_quaternion']['inliers'] and np.abs(y['pose'] - r['non_unit_quaternion']['pose']).max() < 1e-12
    f = S.PO_LAYOUTS['octaves']()
    assert sorted(set(np.round(-np.log(f['inv_sigma2']) / np.log(1.44)).astype(int))) == list(range(8))
    c = S.PO_LAYOUTS['non_square_camera']()['cam']
    assert abs(c[0] - c[1]) > 20 and abs(c[2] - S.W / 2) > 10 and abs(c[3] - S.H / 2) > 10


# ---- PoseInertialOptimizationLastKeyFrame / LastFrame ----
LAYOUTS = {'kf': S.KF_LAYOUTS, 'lf': S.LF_LAYOUTS}


@pytest.mark.parametrize('variant', ['kf', 'lf'])
def test_inertial_layouts_reach_their_branches(variant):
    L = LAYOUTS[variant]
    # edges().size() < 10 (N + 3 edges / N + 4 edges): one round gives the four-round result below the break, not at it
    short, full = (('n_6', 'n_7') if variant == 'kf' else ('n_5', 'n_6'))
    for name, same in ((short, True), (full, False)):
        pr = L[name]()
        assert _same(S.run_oracle(variant, pr), S.run_oracle(variant, pr, rounds=1)) == same, name
    if variant == 'kf':
        pr = L['n_0']()
        r = S.run_oracle(variant, pr)
        assert r['ret'] == 0 and len(r['outlier']) == 0 and np.abs(r['state'] - pr['state']).max() > 0
    for n in (127, 128, 129, 256, 257, 2000):
        pr = L['n_%d' % n]()
        assert len(pr['Xw']) == n
    # the recovery: 29 final inliers < 30 bring the moderate outliers (chi2 < 18) back when bRecInit is off; 30 do not
    for n_in in (29, 30):
        pr = L['inliers_%d' % n_in]()
        off, on = S.run_oracle(variant, pr), S.run_oracle(variant, pr, rec_init=True)
        N = len(pr['Xw'])
        assert on['ret'] == n_in and on['outlier'][n_in:].all() and not on['outlier'][:n_in].any()
        c2, _ = S.chi2(pr, on['state'], range(n_in, N))
        assert (c2 > 5.991).all() and (c2 < 18).all(), c2
        if n_in == 29:
            assert off['ret'] == N and not off['outlier'].any()
        else:
            assert _same(off, on)
    # the close rule: planted chi2 between 5.991 and 1.5 x 5.991 in the last round; trackDepth 10.0f is not close, the float below it is
    for name, flagged in (('depth_10', True), ('depth_below_10', False)):
        pr = L[name]()
        r = S.run_oracle(variant, pr)
        planted = np.flatnonzero(pr['inv_sigma2'] == 1.0)[-8:]
        assert len(planted) == 8 and (pr['track_depth'][planted] == (np.float32(10) if flagged else np.nextafter(np.float32(10), np.float32(0)))).all()
        c2, _ = S.chi2(pr, r['state'], planted)
        assert ((c2 > 5.991) & (c2 < 1.5 * 5.991)).all(), c2
        assert (r['outlier'][planted] == flagged).all() and r['outlier'].sum() == (8 if flagged else 0)
    # points behind the camera with a small chi2: outliers by the depth test alone
    pr = L['behind']()
    r = S.run_oracle(variant, pr)
    c2, dp = S.chi2(pr, r['state'])
    assert (~dp).sum() == 8 and r['outlier'][~dp].all() and (c2[~dp] < 5.991).all() and not r['outlier'][dp].any()
    # every mono edge a gross outlier: the inertial edges alone move the state
    pr = L['all_gross']()
    r = S.run_oracle(variant, pr)
    assert r['ret'] == 0 and r['outlier'].all() and np.abs(r['state'] - pr['state']).max() > 1e-4
    if variant == 'lf':
        pr = L['prior_huber']()
        r = S.run_oracle(variant, pr)
        assert S.prior_chi2(pr, pr['prev_state']) > 25 and S.prior_chi2(pr, r['prev_state']) > 25


@pytest.mark.parametrize('name', S.KF_CLEAN)
def test_last_keyframe_first_step_on_the_layouts(name):
    pr = S.KF_LAYOUTS[name]()
    check_first_step_last_kf(pr, pr['preint'])


@pytest.mark.parametrize('name', S.LF_CLEAN)
def test_last_frame_first_step_on_the_layouts(name):
    pr = S.LF_LAYOUTS[name]()
    Pf, Pk = _preints(pr)
    assert Pf.tobytes() == pr['preint_frame'].tobytes() and Pk.tobytes() == pr['preint_kf'].tobytes()
    check_first_step_last_frame(pr, Pf, Pk)
