"""GPU: local_inertial_ba_batch on the layouts of tests/liba_scenes.py against the CPU oracle (_same_solve), in every launch shape: each
layout alone, all of them in one launch in two orders (byte-identical to the single runs), 64-keyframe windows next to 1-keyframe maps,
more maps than one wave of SMs, a call after a larger call whose scratch was left full of NaN, the FAIL contract, and the argument checks
(including a packing error found by one of the packer's threads)."""
import numpy as np
import pytest

import liba_scenes as S
import oracle_lib as O
from test_local_inertial_ba_cpu import _same_solve

pytestmark = pytest.mark.gpu
KEYS = ('state', 'tcw', 'points', 'erase', 'chi2')


@pytest.fixture(scope='module')
def orb():
    import orb_slam3_modified_b200 as m
    m.lib()
    return m


@pytest.fixture(scope='module')
def layouts():
    return {name: f() for name, f in S.LAYOUTS.items()}


@pytest.fixture(scope='module')
def oracle(layouts):
    return {name: O.local_inertial_ba(pr, pr['preint']) for name, pr in layouts.items()}


def _same_bytes(a, b):
    assert a['iters'] == b['iters'] and a['trials'] == b['trials'] and a['failed'] == b['failed']
    for k in KEYS:
        assert a[k].tobytes() == b[k].tobytes(), k


@pytest.mark.parametrize('name', list(S.LAYOUTS))
def test_each_layout_alone_equals_the_oracle(orb, layouts, oracle, name):
    _same_solve(orb.LocalInertialBA([layouts[name]])[0], oracle[name], layouts[name])


def test_all_layouts_in_one_launch_in_two_orders(orb, layouts):
    names = list(S.LAYOUTS)
    single = {n: orb.LocalInertialBA([layouts[n]])[0] for n in names}
    for order in (names, names[::-1]):
        got = orb.LocalInertialBA([layouts[n] for n in order])
        for n, g in zip(order, got):
            _same_bytes(g, single[n])


def test_64_keyframe_windows_next_to_single_keyframe_maps(orb, layouts, oracle):
    big, one = layouts['window_64'], layouts['window_1']
    got = orb.LocalInertialBA([big, one, big, one, one])
    _same_solve(got[0], oracle['window_64'], big)
    _same_solve(got[1], oracle['window_1'], one)
    _same_bytes(got[2], got[0])
    _same_bytes(got[3], got[1]); _same_bytes(got[4], got[1])


def test_more_maps_than_one_wave(orb, layouts, oracle):
    names = ['window_10', 'edge_list_lengths', 'observers', 'mixed_orientation', 'n_edges_513', 'indefinite_covariance']
    got = orb.LocalInertialBA([layouts[n] for n in names] * 30)       # 180 CTAs on 132 SMs
    for i, n in enumerate(names):
        _same_solve(got[i], oracle[n], layouts[n])
        for rep in range(1, 30):
            _same_bytes(got[i + len(names) * rep], got[i])


def test_stale_scratch_from_a_larger_call(orb, layouts):
    """Scratch is uninitialised by design and comes from the per-thread staging buffer every call reuses: a large map whose states are NaN
    fills it with NaN, and the small maps that follow on the same host thread must read none of it."""
    small = [layouts[n] for n in ('window_2', 'n_edges_1', 'edge_list_lengths', 'no_inertial')]
    before = orb.LocalInertialBA(small)
    big = dict(layouts['window_64'])
    big['state'] = np.full_like(big['state'], np.nan); big['points'] = np.full_like(big['points'], np.nan)
    r = orb.LocalInertialBA([big])[0]
    assert r['failed'] and np.isnan(r['err'])
    after = orb.LocalInertialBA(small)
    for a, b in zip(after, before):
        _same_bytes(a, b)


@pytest.mark.parametrize('which', ['nan_observation', 'finite_fail', 'single_imu_sample'])
def test_fail_hands_back_the_inputs_and_erases_nothing(orb, which):
    pr = getattr(S, which)()
    want = O.local_inertial_ba(pr, pr['preint'])
    got = orb.LocalInertialBA([pr])[0]
    assert want['failed'] and got['failed'] and got['iters'] == want['iters'] and got['trials'] == want['trials']
    for k in ('state', 'tcw', 'points'):
        assert got[k].tobytes() == pr[k].tobytes() == want[k].tobytes(), k
    assert got['erase'].sum() == 0 and want['erase'].sum() == 0
    if which == 'finite_fail':
        assert np.isfinite(got['err_end']) and got['err_end'] > 2 * got['err'] and (got['chi2'] > 5.991).any()
    if which == 'nan_observation':
        big = dict(pr, large=True)                          # bLarge skips the FAIL test
        assert not orb.LocalInertialBA([big])[0]['failed']


def test_argument_errors(orb, layouts):
    def refused(probs):
        with pytest.raises(orb.OrbError) as e:
            orb.LocalInertialBA(probs)
        assert e.value.code == orb.ORB_ERR_ARG
    refused([S.graph(65, n_cov=1, n_pts=80, seed=1)])
    empty = dict(layouts['window_2'], n_opt=0)
    refused([empty])
    for key, bad in (('ie_kf1', -1), ('ie_kf2', None)):
        pr = dict(layouts['window_10'])
        pr[key] = pr[key].copy(); pr[key][3] = pr['n_kf'] if bad is None else bad
        refused([layouts['window_2'], pr])
    # a batch above the packer's 4 MB threshold, so it packs on several threads; a late map observes one point twice from one keyframe
    maps = [layouts[n] for n in ('window_64', 'fixed_200', 'window_35', 'window_34')] * 12
    packed = sum(m['n_kf'] * 280 + len(m['ie_kf1']) * 1185 + len(m['points']) * 32 + len(m['e_pt']) * 40 for m in maps)     # bytes, a lower bound
    assert packed > 4.5e6, packed
    dup = dict(layouts['n_edges_513'])
    for k in ('e_pt', 'e_kf', 'obs', 'inv_sigma2'):
        dup[k] = np.concatenate([dup[k], dup[k][-1:]])
    refused(maps + [dup])
    # the refused calls left nothing behind: the next call on this thread gives the bytes of the first one
    first = orb.LocalInertialBA([layouts['window_2']])[0]
    refused(maps + [dup])
    _same_bytes(orb.LocalInertialBA([layouts['window_2']])[0], first)
