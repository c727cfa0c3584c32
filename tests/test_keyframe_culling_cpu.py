"""CPU tests of LocalMapping::KeyFrameCulling's oracle (oracle/keyframe_culling_oracle.cpp) against the Python restatement and the host
replay of tests/keyframe_culling_lib.py: seeded corridors, every status, the sequential rule, the float boundaries of the decision, the
inertial guards and the break test.  No GPU needed."""

import numpy as np
import pytest

import keyframe_culling_lib as K

F32 = np.float32


def check(cm):
    """Oracle == restatement (result and final map) == the replay of the oracle's statuses; returns the oracle's result."""
    res, state = K.oracle(K.flatten(cm))
    r2, s2, merges = K.restate(cm)
    assert K.same_result(res, r2), (res, r2)
    assert K.same_state(state, s2)
    s3, m3 = K.replay(cm, res)
    assert K.same_state(state, s3) and m3 == merges
    return res


@pytest.mark.parametrize('inertial', [False, True])
@pytest.mark.parametrize('seed', range(6))
def test_oracle_equals_restatement_on_corridors(seed, inertial):
    cm = K.corridor(seed, inertial=inertial, order='newest' if seed % 2 else 'shuffle', kf_extra=5)
    res = check(cm)
    culled = np.isin(res['status'], K.ERASING).sum()
    assert 0 < culled < len(cm.local)


def _status_scenes():
    yield K.corridor(1)
    yield K.corridor(2, inertial=True, kf_extra=5)
    yield K.corridor(3, inertial=True, kf_extra=-12)                      # KeyFramesInMap() reaches Nd
    yield K.corridor(4, n_kf=30, abort=True)                              # the break after count 20
    recent = K.dense(30, inertial=True)
    recent.kfs[-2].mnId = recent.current_id - 1
    yield recent
    cm = K.dense(30, inertial=True)
    cm.kfs[27].prev = None; cm.kfs[26].next = None                        # no mPrevKF
    yield cm


def test_every_status_reached():
    seen = set()
    for cm in _status_scenes():
        seen |= set(check(cm)['status'].tolist())
    assert seen == set(range(11)), sorted(set(range(11)) - seen)



def test_cascade_flips_a_later_decision():
    cm = K.cascade()
    res = check(cm)
    assert res['status'].tolist() == [K.CULLED, K.CULLED]
    assert res['nMPs'].tolist() == [20, 9] and res['nRedundant'].tolist() == [19, 9]
    static, _, _ = K.restate(cm, static=True)
    assert static['status'].tolist() == [K.CULLED, K.KEPT] and static['nMPs'].tolist() == [20, 10]



def test_redundancy_threshold_is_a_float_product():
    for n in range(10, 260, 10):
        for nr in (n * 9 // 10 - 1, n * 9 // 10, n * 9 // 10 + 1):
            if not 0 <= nr <= n:
                continue
            res = check(K.boundary(n, nr))
            want = F32(nr) > F32(0.9) * F32(n)
            assert (res['status'][0] == K.CULLED) == want, (n, nr)
            if nr * 10 == n * 9:
                assert F32(0.9) * F32(n) == F32(nr) and not want            # 0.9f * nMPs rounds to nr: equality keeps the keyframe



def test_t_is_rounded_to_float():
    for limit, init in ((3.0, True), (0.5, False)):
        below = limit - 1e-9                                              # below the limit in double, rounds to it in float
        assert below < limit and F32(below) == F32(limit)
        assert check(K.one_inertial(below, imu_init=init))['status'][0] == K.KEPT_IMU
        assert check(K.one_inertial(limit - 1e-6, imu_init=init))['status'][0] == K.CULLED_TIME
    assert check(K.one_inertial(2.0, imu_init=True, mnid_below_last=False))['status'][0] == K.KEPT_IMU    # mnId >= last_ID


def test_imu_position_gap_around_002():
    for d, want in ((0.02 - 1e-5, K.CULLED_STILL), (0.02 + 1e-5, K.KEPT_IMU), (0.019, K.CULLED_STILL)):
        cm = K.one_inertial(1.0, gap=d)
        assert abs(float(np.linalg.norm(cm.kfs[5].pos.astype(np.float64) - cm.kfs[4].pos)) - 0.02) >= 1e-5 - 1e-7
        assert check(cm)['status'][0] == want, d
        assert check(K.one_inertial(1.0, gap=d, ba2=True))['status'][0] == K.KEPT_IMU
        assert check(K.one_inertial(3.5, gap=d))['status'][0] == K.KEPT_IMU


def test_unsigned_id_guard():
    cm = K.dense(30, inertial=True)
    cm.local = [28, 27]
    res = check(cm)
    assert res['status'].tolist() == [K.KEPT_RECENT, K.CULLED_TIME]       # 28 > 29 - 2
    cm.current_id = 1                                                     # 1 - 2 wraps: no keyframe is recent
    assert check(cm)['status'].tolist() == [K.CULLED_TIME, K.KEPT_IMU]    # 27 is relinked to 29: t = 0.6


def test_keyframes_in_map_falls_to_nd():
    cm = K.dense(30, inertial=True, kf_in_map=24)
    res = check(cm)
    st = res['status'].tolist()
    # every cull relinks its neighbours, so the next keyframe's t is 0.6: culls alternate until three of them bring 24 down to Nd
    assert st[:6] == [K.KEPT_RECENT, K.CULLED_TIME, K.KEPT_IMU, K.CULLED_TIME, K.KEPT_IMU, K.CULLED_TIME]
    assert set(st[6:]) == {K.KEPT_FEW_KFS} and res['visited'] == len(cm.local)


def test_continue_paths_skip_the_break_test():
    # abortBA: a monocular walk stops after the 21st keyframe; an inertial one whose keyframes all take the KeyFramesInMap() continue does not
    cm = K.dense(40)
    cm.abort = True
    res = check(cm)
    assert res['visited'] == 21 and (res['status'][21:] == K.NOT_VISITED).all()
    cm = K.dense(40, inertial=True, kf_in_map=21)
    cm.abort = True
    res = check(cm)
    assert res['visited'] == len(cm.local) and set(res['status'].tolist()) == {K.KEPT_FEW_KFS}
    # bad keyframes (a continue) from the 21st on: the walk goes on to the first keyframe that falls through
    cm = K.dense(40)
    cm.abort = True
    for k in cm.local[20:25]:
        cm.kfs[k].bad = True
    res = check(cm)
    assert res['visited'] == 26 and res['status'][25] != K.NOT_VISITED and (res['status'][26:] == K.NOT_VISITED).all()


def test_count_over_100():
    cm = K.corridor(7, n_kf=130, new_per_kf=6)
    res = check(cm)
    assert len(cm.local) > 101 and res['visited'] == 101
    assert (res['status'][101:] == K.NOT_VISITED).all() and (res['status'][:101] != K.NOT_VISITED).all()
    assert (res['nMPs'][101:] == -1).all()


def test_new_entry_point_without_gpu():
    import torch
    import orb_slam3_modified_b200 as orb
    L = orb.lib()
    assert hasattr(L, 'orbm_keyframe_culling_batch')
    assert L.orbm_keyframe_culling_batch(None, 0, None) == orb.ORB_ERR_ARG
    if torch.cuda.is_available():
        pytest.skip('GPU present')
    with pytest.raises(orb.OrbError) as ei:
        orb.ORBmatcher(0.6, True).keyframe_culling_batch([K.flatten(K.corridor(0))])
    assert ei.value.code == orb.ORB_ERR_CUDA
