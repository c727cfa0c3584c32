"""CPU tests of the ProcessNewKeyFrame / SearchInNeighbors-tail oracle (oracle/update_connections_oracle.cpp): it equals the independent
Python restatement on seeded scenes in both modes, every planted rule is reached, and the host replay of its outputs gives its final map."""
import numpy as np
import pytest

import update_connections_lib as U


def _check(sc):
    m = U.flatten(sc)
    got, fin = U.oracle(m)
    assert U.same_outputs(got, U.restate(sc))
    assert U.final_state(U.replay(sc, got)) == fin
    return got


@pytest.mark.parametrize('mode', [U.PNK, U.SIN])
@pytest.mark.parametrize('seed', [1, 2, 3])
def test_oracle_equals_restatement_and_replay(mode, seed):
    sc = U.scene(seed, mode, n_kf=60, n_slots=300, first=seed == 2, init=seed == 3)
    got = _check(sc)
    st = got['slotStatus']
    if mode == U.PNK:
        assert (st == U.ADDED).sum() > 50 and (st == U.IN_KF).sum() > 20
    else:
        assert (st == U.UPDATED).sum() > 100
    assert got['nConnected'] > 3 and (got['nbrCount'] >= 0).sum() > 2
    assert ((got['counter'] > 0) & (got['counter'] < U.TH)).any()          # counts below the threshold stay in the weight map


def test_user_scale_scene():
    """About 1000 slots, 10 observations per point, 150 keyframes: the timing tool's size."""
    got = _check(U.scene(5, U.PNK))
    assert got['pointUpdated'].sum() > 400


def test_empty_item():
    sc = U.scene(4, U.SIN, n_kf=8, n_slots=0)
    got = _check(sc)
    assert got['nConnected'] == -1 and got['parent'] == -1


@pytest.fixture(scope='module')
def planted():
    return {name: (sc, _check(sc)) for name, sc in U.planted().items()}


def test_tie_decided_by_key(planted):
    sc, g = planted['tie_by_key']
    assert g['nConnected'] == 2 and g['orderedKF'][:2].tolist() == [1, 2] and g['orderedWeight'][:2].tolist() == [20, 20]
    assert sc.kfs[1].order > sc.kfs[2].order and sc.kfs[1].mnId < sc.kfs[2].mnId


def test_fallback_takes_first_strict_maximum_by_key(planted):
    sc, g = planted['fallback_tie']
    assert g['counter'][1:].tolist() == [5, 5] and g['nConnected'] == 1 and g['orderedKF'][0] == 2
    assert g['nbrCount'][2] >= 0 and g['nbrCount'][1] == -1


def test_empty_counter_changes_nothing(planted):
    sc, g = planted['empty_counter']
    assert g['nConnected'] == -1 and g['parent'] == -1 and not g['counter'].any() and (g['nbrCount'] == -1).all()
    assert (g['slotStatus'][:12] == U.ADDED).all()
    assert U.final_state(U.replay(sc, g))['firstConnection'] == 1


def test_bad_and_other_map_observers(planted):
    sc, g = planted['bad_other_observers']
    assert g['counter'].tolist() == [0, 18, 18, 0, 0]
    upd = g['pointUpdated'].astype(bool)
    assert upd.sum() == 18 and not np.isin(g['descKF'][upd], [3]).any()
    # the bad observer is in the normal: leaving it out changes it
    p = sc.pts[0]
    n_wo = U._update_point(sc, p, {t: i for t, i in {**p.obs, 0: 0}.items() if t != 3}, 0, 'order', 'key')[0]
    assert n_wo.tobytes() != g['normal'][0].tobytes()


def test_point_in_two_slots(planted):
    sc, g = planted['two_slots']
    assert g['slotStatus'][0] == U.ADDED and g['slotStatus'][5] == U.IN_KF
    assert g['counter'][1] == 2
    assert U.replay(sc, g).recent == [0]


def test_equal_weight_leaves_stale_list_and_resort_drops_bad(planted):
    sc, g = planted['equal_weight_and_resort']
    assert g['counter'][1] == 20 == sc.kfs[1].conn[0] and g['nbrCount'][1] == -1      # equal weight: keyframe 1 keeps its list (with bad 3)
    off = sum(len(k.conn) + 1 for k in sc.kfs[:2])          # keyframe 2's list: connStart[2] + 2
    n = g['nbrCount'][2]
    assert n == 3 and g['nbrKF'][off:off + n].tolist() == [1, 0, 4] and g['nbrWeight'][off:off + n].tolist() == [16, 16, 7]


def test_parent_only_outside_the_init_keyframe(planted):
    g_init, g_plain = planted['init_no_parent'][1], planted['first_connection_parent'][1]
    assert g_init['nConnected'] == g_plain['nConnected'] == 1 and g_init['orderedKF'][0] == 1
    assert g_init['parent'] == -1 and g_plain['parent'] == 1


def test_median_tie_decided_by_insert_position(planted):
    sc, g = planted['median_tie_insert']
    p = sc.kfs[0].mp[3]
    assert (g['descKF'][p], g['descIdx'][p]) == (0, 3)
    assert U.restate(sc, new_row='end')['descKF'][p] == 1


def test_normal_sum_order_is_exercised(planted):
    sc, g = planted['normal_order']
    alt = U.restate(sc, sum_order='mnId')
    upd = np.nonzero(g['pointUpdated'])[0]
    obs = np.array([len(sc.pts[p].obs) + 1 for p in upd])
    differ = [p for p in upd if alt['normal'][p].tobytes() != g['normal'][p].tobytes()]
    assert differ and min(len(sc.pts[p].obs) + 1 for p in differ) >= 3 and obs.max() >= 3
