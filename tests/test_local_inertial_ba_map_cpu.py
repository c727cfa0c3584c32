"""CPU tests of Optimizer::LocalInertialBA as a whole: the oracle (oracle/local_inertial_ba_map_oracle.cpp) against the independent
restatement of tests/local_inertial_ba_map_lib.py on planted and seeded maps, the oracle's built problem against the LocalInertialBA oracle,
the oracle's finish from given solver results, and the entry point's refusals, which come before any device is touched."""
import copy

import numpy as np
import pytest

import local_inertial_ba_map_lib as LM
import oracle_lib as O
import orb_slam3_modified_b200 as orb

PLANTED = LM.planted()


def _check(M, pkf, kim, large, rec_init):
    m = LM.flatten(M, pkf, kim, large, rec_init)
    r, pr = LM.oracle(m)
    mine = copy.deepcopy(M)
    rec = LM.restate(mine, pkf, kim, large, rec_init, LM.lm_of(m, r))
    got = LM.record_in_ids(m, r)
    for k in ('status', 'window', 'fixed', 'points', 'linked', 'edges', 'erase'):
        assert got[k] == rec[k], k
    assert r['num_edges'] == len(rec['edges'])
    if r['status'] == orb.LIBA_LOCAL_RAN:
        LM.check_model(mine, m, r)
    else:
        for n in ('kfPose7', 'kfCenter', 'kfVelocity', 'kfBias6', 'pointPos', 'normal', 'optState21', 'optPoint'):
            assert not r[n].any(), n
        assert not (r['obsFlag'] == orb.LBA_OBS_ERASED).any()
    # the built problem: keyframes window then fixed, the inertial edges keyed on the window index, the edges in insertion order
    vk = rec['window'] + rec['fixed']
    assert pr['n_kf'] == len(vk) and pr['n_opt'] == len(rec['window'])
    assert [(vk[a], vk[b], bool(rb), s) for a, b, rb, s in zip(pr['ie_kf1'], pr['ie_kf2'], pr['ie_robust'], pr['ie_info_scale'])] == rec['ie']
    assert [(rec['points'][p], vk[k]) for p, k in zip(pr['e_pt'], pr['e_kf'])] == rec['edges']
    assert np.array_equal(pr['state'], np.stack([M.kfs[k].state21 for k in vk]).astype(np.float64))
    assert np.array_equal(pr['points'], np.stack([M.pts[p].pos for p in rec['points']]).astype(np.float64).reshape(-1, 3))
    assert pr['iterations'] == (4 if large else 10) and pr['lambda_init'] == (1e-2 if large else 1.0)
    return m, r, pr, rec


@pytest.mark.parametrize('name', sorted(PLANTED))
def test_oracle_equals_restatement_planted(name):
    M, pkf, kim, large, rec_init = PLANTED[name]
    m, r, pr, rec = _check(M, pkf, kim, large, rec_init)
    assert r['status'] == (orb.LIBA_LOCAL_FAILED if name == 'fail' else orb.LIBA_LOCAL_RAN)
    kid = m['kf_ids']
    if name == 'popped_predecessor':
        assert len(rec['window']) == 4 and M.kfs[rec['fixed'][0]].prev < 0 and M.kfs[rec['window'][-1]].prev == rec['fixed'][0]
    if name == 'kf_in_map_limits_nd':
        assert len(rec['window']) == 4 and M.kfs[rec['window'][-1]].prev == rec['fixed'][0]
    if name == 'no_preint':
        assert rec['linked'].count(False) == 2 and not rec['linked'][3] and not rec['linked'][-1] and all(pr['ie_robust'])
    if name == 'bad_other':
        bad = [k for k in kid if M.kfs[k].bad]
        other = [k for k in kid if M.kfs[k].other]
        assert bad and other and not set(bad) & set(rec['fixed']) and set(other) <= set(rec['fixed'])
        assert not {k for _, k in rec['edges']} & (set(bad) | set(other))
    if name == 'large':
        assert len(rec['window']) == 12 and pr['iterations'] == 4
    if name == 'cap_200':
        assert len(rec['fixed']) == 200
        unreached = {k for p in rec['points'] for k in M.pts[p].obs} - set(rec['window']) - set(rec['fixed'])
        assert unreached and not {k for _, k in rec['edges']} & unreached      # the break and the cap leave observers without edges
    if name == 'observers':
        c2 = LM.lm_of(m, r)['chi2']
        near = [e for e in rec['edges'] if M.pts[e[0]].track_depth <= np.float32(10) and LM.TH < c2[e] < 1.5 * LM.TH]
        assert near, 'no edge between 5.991 and 1.5 x 5.991 on a point at the 10 m boundary'
    if name == 'cascade':
        assert r['pointBad'].any()
        moved = [i for i, p in enumerate(r['localPoint']) if not r['pointBad'][i] and r['pointRefKF'][i] != m['refKF'][p]]
        assert moved, 'no erase moved mpRefKF'


@pytest.mark.parametrize('seed', range(6))
def test_oracle_equals_restatement_seeded(seed):
    M, pkf, kim, large, rec_init = LM.seeded(seed)
    _check(M, pkf, kim, large, rec_init)


@pytest.mark.parametrize('name', ['normal', 'no_preint', 'cascade', 'fail', 'popped_predecessor'])
def test_built_problem_gives_the_oracle_results(name):
    """The oracle's problem, solved by the LocalInertialBA oracle on its own, gives the map oracle's doubles; finishing from those doubles
    gives the map oracle's record."""
    M, pkf, kim, large, rec_init = PLANTED[name]
    m = LM.flatten(M, pkf, kim, large, rec_init)
    r, pr = LM.oracle(m)
    w = O.local_inertial_ba(pr, pr['preint'])
    assert w['failed'] == bool(r['stats8'][2]) and np.array_equal([w['err'], w['err_end']], r['stats8'][:2], equal_nan=True)
    order = [o for p in r['localPoint'] for o in range(m['obsStart'][p], m['obsStart'][p + 1]) if r['obsFlag'][o] != orb.LBA_OBS_NO_EDGE]
    assert np.array_equal(r['edgeChi2'][order], w['chi2'], equal_nan=True)
    if not w['failed']:
        assert np.array_equal(r['optState21'], w['state']) and np.array_equal(r['optTcw12'], w['tcw']) and np.array_equal(r['optPoint'], w['points'])
        assert np.array_equal(r['obsFlag'][order] == orb.LBA_OBS_ERASED, w['erase'].astype(bool))
    g, _ = LM.oracle(m, given=LM.padded(r, m))
    for k in orb.LIBA_MAP_OUTPUTS:
        assert np.array_equal(g[k[0]], r[k[0]], equal_nan=k[0] == 'stats8'), k[0]


def _refused(m, what):
    s, out, keep = orb.liba_map_struct(m)
    arr = (orb.LocalInertialBAMap * 1)(s)
    try:
        L = orb.lib()
    except (RuntimeError, OSError):
        pytest.skip('library not built')
    assert L.local_inertial_ba_map_batch(1, arr, 0) == orb.ORB_ERR_ARG
    msg = L.orb_last_error().decode()
    assert 'map 0' in msg and what in msg, msg


def _base():
    M, pkf, kim, large, rec_init = PLANTED['normal']
    return LM.flatten(M, pkf, kim, large, rec_init)


def test_refusals():
    m = _base()
    bad = copy.deepcopy(m); bad['obsKF'] = bad['obsKF'].copy(); bad['obsKF'][3] = len(m['kfFlags'])
    _refused(bad, 'obsKF out of range')
    bad = copy.deepcopy(m); bad['obsOctave'] = bad['obsOctave'].copy(); bad['obsOctave'][0] = 8
    _refused(bad, 'obsOctave')
    bad = copy.deepcopy(m); bad['slotPoint'] = bad['slotPoint'].copy(); bad['slotPoint'][0] = len(m['pointFlags'])
    _refused(bad, 'slotPoint out of range')
    bad = copy.deepcopy(m); bad['prevKF'] = bad['prevKF'].copy(); bad['prevKF'][2] = len(m['kfFlags'])
    _refused(bad, 'prevKF out of range')
    bad = copy.deepcopy(m); bad['obsStart'] = bad['obsStart'].copy(); bad['obsStart'][1] = bad['obsStart'][2] + 1
    _refused(bad, 'obsStart')
    bad = copy.deepcopy(m); bad['slotStart'] = bad['slotStart'].copy(); bad['slotStart'][0] = 1
    _refused(bad, 'slotStart')
    p = next(p for p in range(len(m['pointFlags'])) if m['obsStart'][p + 1] - m['obsStart'][p] >= 2)
    bad = copy.deepcopy(m); bad['obsKF'] = bad['obsKF'].copy(); bad['obsKF'][m['obsStart'][p] + 1] = bad['obsKF'][m['obsStart'][p]]
    _refused(bad, 'observes a point twice')
    bad = copy.deepcopy(m); bad['refKF'] = bad['refKF'].copy()
    bad['refKF'][p] = next(k for k in range(len(m['kfFlags'])) if k not in set(m['obsKF'][m['obsStart'][p]:m['obsStart'][p + 1]]))
    _refused(bad, 'mpRefKF is not among its observers')
    bad = copy.deepcopy(m); bad['kfFlags'] = bad['kfFlags'].copy(); bad['kfFlags'][0] |= orb.KF_OTHER_MAP
    _refused(bad, 'pKF (entry 0) cannot be of another map')
    bad = copy.deepcopy(m); bad['prevKF'] = bad['prevKF'].copy(); bad['prevKF'][0] = -1
    _refused(bad, 'has no mPrevKF')
    bad = copy.deepcopy(m); bad['kfFlags'] = bad['kfFlags'].copy(); bad['kfFlags'][2] &= np.uint8(~orb.KF_IMU & 0xFF)
    _refused(bad, 'no ORBM_KF_IMU')
    bad = copy.deepcopy(m); bad['prevKF'] = bad['prevKF'].copy(); bad['prevKF'][3] = 1
    _refused(bad, 'revisits a keyframe')
    for field, what, debug in (('preint', 'preint is null', False), ('prevKF', 'a keyframe or map array is null', False),
                               ('kfVelocity', 'a keyframe output is null', False), ('trackDepth', 'a point array is null', False),
                               ('obsPt', 'an observation array is null', False), ('optPoint', 'go together', True)):
        s, out, keep = orb.liba_map_struct(m, debug=debug)
        setattr(s, field, None)
        arr = (orb.LocalInertialBAMap * 1)(s)
        assert orb.lib().local_inertial_ba_map_batch(1, arr, 0) == orb.ORB_ERR_ARG
        msg = orb.lib().orb_last_error().decode()
        assert 'map 0' in msg and what in msg, (field, msg)
    assert orb.lib().local_inertial_ba_map_batch(-1, arr, 0) == orb.ORB_ERR_ARG


def test_valid_call_needs_a_device():
    """A well-formed batch passes every check and then needs the device: ORB_ERR_CUDA without one (on a GPU machine it runs)."""
    s, out, keep = orb.liba_map_struct(_base())
    arr = (orb.LocalInertialBAMap * 1)(s)
    try:
        L = orb.lib()
    except (RuntimeError, OSError):
        pytest.skip('library not built')
    rc = L.local_inertial_ba_map_batch(1, arr, 0)
    if rc == orb.ORB_OK:
        assert L.local_inertial_ba_map_last_launches() == 3
    else:
        assert rc == orb.ORB_ERR_CUDA and L.local_inertial_ba_map_last_launches() == 0, rc
