"""CPU tests of Optimizer::LocalBundleAdjustment as a whole: the oracle (oracle/local_ba_oracle.cpp) against the independent restatement of
tests/local_ba_lib.py on planted and seeded maps, the replay of the oracle's record, and the new entry point without a device."""
import ctypes as C

import numpy as np
import pytest

import local_ba_lib as LB
import orb_slam3_modified_b200 as orb

PLANTED = LB.planted()


def _check(M, pkf):
    m = LB.flatten(M, pkf)
    r, built = LB.oracle(m)
    mine = LB.copy_map(M)
    rec = LB.restate(mine, pkf, LB.lm_of(m, r))
    got = LB.record_in_ids(m, r)
    for k in ('status', 'local', 'fixed', 'points', 'counts', 'erase'):
        assert got[k] == rec[k], k
    replayed = LB.copy_map(M)
    LB.replay(replayed, m, r)
    if r['status'] == orb.LBA_LOCAL_RAN:
        assert replayed.state() == mine.state()
        # the float write-back bit for bit, and the bad flags / mpRefKF, from the restatement's model
        kid, pid = m['kf_ids'], m['pt_ids']
        for i, k in enumerate(r['localKF']):
            assert r['kfPose7'][i].tobytes() == mine.kfs[kid[k]].Tcw.tobytes() and r['kfCenter'][i].tobytes() == mine.kfs[kid[k]].Ow.tobytes()
        for i, p in enumerate(r['localPoint']):
            q = mine.pts[pid[p]]
            assert bool(r['pointBad'][i]) == q.bad and r['pointPos'][i].tobytes() == q.pos.tobytes()
            if not q.bad:
                assert r['normal'][i].tobytes() == q.normal.tobytes() and r['maxDistance'][i] == q.max_d and r['minDistance'][i] == q.min_d
    else:
        assert replayed.state() == M.state()        # NO_FIXED / STOPPED: nothing to replay
    if r['status'] != orb.LBA_LOCAL_NO_FIXED:
        # the oracle's graph == the restatement's: vertex order, fixed flags, edges in insertion order, their observations and weights
        kid, pid = m['kf_ids'], m['pt_ids']
        want = rec['built']
        vk, vp = [kid[k] for k in built['vert_kf']], [pid[p] for p in built['vert_point']]
        assert vk == want['vert_kf'] and vp == want['vert_point']
        assert [bool(f) for f in built['fixed']] == [bool(f) for f in want['fixed']]
        assert [(vp[p], vk[k]) for p, k in zip(built['edge_point'], built['edge_pose'])] == want['edges']
        assert np.array_equal(built['poses'], np.array(want['poses']).reshape(-1, 7)) and np.array_equal(built['cam'], np.array(want['cam']).reshape(-1, 4))
        assert np.array_equal(built['points'], np.array(want['points']).reshape(-1, 3))
        assert np.array_equal(built['obs'], np.array(want['obs']).reshape(-1, 2))
        assert np.array_equal(built['inv_sigma2'], np.array(want['inv_sigma2'], np.float32))
    return r, rec


@pytest.mark.parametrize('name', sorted(PLANTED))
def test_oracle_equals_restatement_planted(name):
    M, pkf = PLANTED[name]
    r, rec = _check(M, pkf)
    want = dict(no_fixed=orb.LBA_LOCAL_NO_FIXED, stopped=orb.LBA_LOCAL_STOPPED).get(name, orb.LBA_LOCAL_RAN)
    assert r['status'] == want
    if name == 'mixed':
        m = LB.flatten(M, pkf)
        assert len(r['localKF']) == 1 + len(M.cov[pkf]) - 2        # the bad and the other-map covisible are left out
        # the bad and the other-map observers are reached, marked, and neither kept as fixed cameras nor given an edge
        for k in (1, 2):
            t = m['kf_ids'].index(k)
            assert t not in list(r['fixedKF']) and not r['obsFlag'][m['obsKF'] == t].any()
        assert len(r['fixedKF']) > 0
        assert m['pointFlags'][m['slotPoint'][m['slotPoint'] >= 0]].any()
        assert r['pointBad'].any() and len(rec['erase']) > 0
        moved = [i for i, p in enumerate(r['localPoint']) if not r['pointBad'][i] and r['pointRefKF'][i] != m['refKF'][p]]
        assert moved, 'no erase moved mpRefKF'
        # an erase that dropped nObs to 2 and a later erase of the same (then bad) point
        by_pt = {}
        for p, k in rec['erase']:
            by_pt[p] = by_pt.get(p, 0) + 1
        assert any(n > M.pts[p].nObs - 2 for p, n in by_pt.items())
    if name == 'init_only':
        assert r['num_fixedKF'] == 1 and len(r['fixedKF']) == 0
    if name == 'hub_fixed':
        m = LB.flatten(M, pkf)
        assert m['kf_ids'].index(0) in list(r['fixedKF'])
    if name == 'inertial':
        assert r['status'] == orb.LBA_LOCAL_RAN


@pytest.mark.parametrize('seed', [11, 12, 13])
def test_oracle_equals_restatement_seeded(seed):
    M, pkf = LB.scene(seed, n_kf=12, n_pts=400, obs_per_pt=5, n_cov=6, outlier_frac=0.08, inertial=seed % 2 == 0)
    r, rec = _check(M, pkf)
    assert r['status'] == orb.LBA_LOCAL_RAN and len(rec['erase']) > 0


def test_entry_point_handle_and_null_handle():
    """The call needs an lba handle, and a handle needs a device: without one lba_create_batch returns ORB_ERR_CUDA, so the new symbol
    cannot run; on any machine it refuses a null handle or a negative map count with ORB_ERR_ARG before touching a device."""
    M, pkf = PLANTED['mixed']
    s, out, keep = orb.local_ba_struct(LB.flatten(M, pkf))
    arr = (orb.LbaLocalMap * 1)(s)
    try:
        L = orb.lib()
    except (RuntimeError, OSError):
        pytest.skip('library not built')
    assert L.lba_local_bundle_adjustment_batch(None, 1, arr) == orb.ORB_ERR_ARG
    h = C.c_void_p()
    rc = L.lba_create_batch(C.byref(h), 64, 1024, 8192, 4, 0)
    if rc == orb.ORB_OK:
        try:
            assert L.lba_local_bundle_adjustment_batch(h, -1, arr) == orb.ORB_ERR_ARG
            assert L.lba_local_bundle_adjustment_batch(h, 1, arr) == orb.ORB_OK
        finally:
            L.lba_destroy(h)
    else:
        assert rc == orb.ORB_ERR_CUDA
