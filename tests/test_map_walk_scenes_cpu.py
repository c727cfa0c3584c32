"""CPU tests of the map_walk_scenes.py cases: each reaches the shape it is built for (lba_shape / liba_shape on the oracle's record), its
solve keeps the outlier tests' margins, and the oracle (oracle/local_ba_oracle.cpp, oracle/local_inertial_ba_map_oracle.cpp) equals the
independent restatements of local_ba_lib / local_inertial_ba_map_lib on it."""
import copy

import numpy as np
import pytest

import local_ba_lib as LB
import local_inertial_ba_map_lib as LM
import map_walk_scenes as S
import orb_slam3_modified_b200 as orb

LBA = S.lba_cases()
LIBA = S.liba_cases()


def _cascade(m, r, flag, erased):
    """The three cascade cases among the local points: nObs 3 turned bad with a later erase; mpRefKF's observation (the first in key order)
    erased first, the point still good; every observation of a point erased."""
    os_ = m['obsStart']
    three = refmoved = every = False
    for i, p in enumerate(r['localPoint']):
        f = r['obsFlag'][os_[p]:os_[p + 1]]
        n = len(f)
        e = int((f == erased).sum())
        three |= n == 3 and e >= 2 and bool(r['pointBad'][i])
        refmoved |= n >= 4 and f[0] == erased and m['refKF'][p] == m['obsKF'][os_[p]] and not r['pointBad'][i] and \
            r['pointRefKF'][i] == m['obsKF'][os_[p] + int(np.argmax(f != erased))]
        every |= n >= 3 and e == n
    assert three and refmoved and every, (three, refmoved, every)


@pytest.mark.parametrize('name', sorted(LBA))
def test_lba_case_reaches_its_shape_and_oracle_equals_restatement(name):
    build, want = LBA[name]
    M, pkf = build()
    m = LB.flatten(M, pkf)
    r, built = LB.oracle(m)
    shape = S.lba_shape(m, r)
    assert S.meets(shape, want), (want, shape)
    if name == 'cov_600':
        assert r['status'] == orb.LBA_LOCAL_STOPPED
    else:
        assert r['status'] == orb.LBA_LOCAL_RAN
        if name not in S.NO_MARGIN:
            LB.check_margin(r)
    if name.startswith('qs_10') or name == 'fixed_500':
        assert shape['split'] and shape['late_first']   # a point seen in two tiles; a first appearance after a repeat in a later tile
    if name == 'fixed_500':
        assert shape['fix_late'] and shape['fix_skipped']
    if name in ('nl_4095', 'nl_4096'):
        assert shape['n2L'] == 4096 and shape['sortCap'] == 8192    # nPoints > 4096: sortCap past n2
    if name == 'np_17':
        assert (m['mnId'] > np.uint64(2 ** 64 - 4096)).all() and (m['pointId'] > np.uint64(2 ** 64 - 2 ** 20)).all()
    if want.get('cascade'):
        _cascade(m, r, r['obsFlag'], orb.LBA_OBS_ERASED)
    # the oracle against the restatement: lists, counts, erasures, the graph's vertex order and edges
    mine = LB.copy_map(M)
    rec = LB.restate(mine, pkf, LB.lm_of(m, r))
    got = LB.record_in_ids(m, r)
    for k in ('status', 'local', 'fixed', 'points', 'counts', 'erase'):
        assert got[k] == rec[k], k
    kid, pid = m['kf_ids'], m['pt_ids']
    assert [kid[k] for k in built['vert_kf']] == rec['built']['vert_kf'] and [pid[p] for p in built['vert_point']] == rec['built']['vert_point']
    assert [(pid[built['vert_point'][p]], kid[built['vert_kf'][k]]) for p, k in zip(built['edge_point'], built['edge_pose'])] == rec['built']['edges']
    if r['status'] == orb.LBA_LOCAL_RAN:
        for i, k in enumerate(r['localKF']):
            assert r['kfPose7'][i].tobytes() == mine.kfs[kid[k]].Tcw.tobytes()
        for i, p in enumerate(r['localPoint']):
            q = mine.pts[pid[p]]
            assert bool(r['pointBad'][i]) == q.bad and r['pointPos'][i].tobytes() == q.pos.tobytes()
            assert r['pointRefKF'][i] == (kid.index(q.ref) if q.ref >= 0 else -1)
            if not q.bad:
                assert r['normal'][i].tobytes() == q.normal.tobytes() and r['maxDistance'][i] == q.max_d and r['minDistance'][i] == q.min_d


@pytest.mark.parametrize('name', sorted(LIBA))
def test_liba_case_reaches_its_shape_and_oracle_equals_restatement(name):
    build, want = LIBA[name]
    M, pkf, kim, large, rec_init = build()
    m = LM.flatten(M, pkf, kim, large, rec_init)
    r, pr = LM.oracle(m)
    shape = S.liba_shape(m, r)
    assert S.meets(shape, want), (want, shape)
    assert r['status'] == orb.LIBA_LOCAL_RAN
    c2 = r['edgeChi2'][r['obsFlag'] != orb.LBA_OBS_NO_EDGE]
    assert not (np.abs(c2 - 5.991) < 1e-3).any() and not (np.abs(c2 - 1.5 * 5.991) < 1e-3).any()
    if want.get('cascade'):
        _cascade(m, r, r['obsFlag'], orb.LBA_OBS_ERASED)
    if name == 'ne_5000':
        # the window keyframes' edges spread over several 512-edge tiles (pKF's, listed first, fill the first one)
        e_kf = np.asarray(pr['e_kf'])
        assert sum(len(set(np.flatnonzero(e_kf == k) // S.WT)) > 1 for k in range(25)) == 24
    # the mirror's probe = the oracle's lFixedKeyFrames
    assert shape['fixed'] == [int(k) for k in r['fixedKF']]
    # the oracle against the restatement
    mine = copy.deepcopy(M)
    rec = LM.restate(mine, pkf, kim, large, rec_init, LM.lm_of(m, r))
    got = LM.record_in_ids(m, r)
    for k in ('status', 'window', 'fixed', 'points', 'linked', 'edges', 'erase'):
        assert got[k] == rec[k], k
    LM.check_model(mine, m, r)
