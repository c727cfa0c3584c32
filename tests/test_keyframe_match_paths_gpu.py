"""SearchByBoW (both overloads), SearchForTriangulation, the Fuse searches, SearchBySim3 and the batched CreateNewMapPoints on the cases of
tests/keyframe_match_scenes.py, byte for byte against the oracle in every output: matches, match12, counts, bestIdx / bestDist and the
new-point records.  tests/test_keyframe_match_scenes_cpu.py shows that each case reaches the shape it names.

The cases reach bow_match_kernel's warp loop over node groups (1 to 300 groups, one node of 2,048 features) and its lane loop over frame
nodes of 1 to 1,000 features; tri_match_kernel's warp loop over E1 and lane loop over KF2 nodes; fuse_search_kernel with the keyframe's
descriptors in shared memory (K = 4,496) and in global memory (4,497 and 14,008 keypoints), 1 to 16 CTAs per item, items of both layouts
in one launch; and new_points_kernel's grid at its 65,535 pairs."""
import numpy as np
import pytest

import keyframe_match_scenes as S
import new_points_lib as NP
import oracle_lib as O

pytestmark = pytest.mark.gpu
BOW, TRI, FUSE, SIM3 = S.bow_cases(), S.tri_cases(), S.fuse_cases(), S.sim3_cases()
KCAP = S.K_MAX + 1                       # handles that can take the refused keyframe to the layout check
_ORACLE = {}


@pytest.fixture(scope='module')
def orb():
    import orb_slam3_modified_b200 as m
    m.lib()
    return m


def fuse_oracle(c, sim3=False):
    key = (c['name'], sim3)
    if key not in _ORACLE:
        _ORACLE[key] = O.fuse_search_sim3(c, c['Tcw'], c['Ow'], c['th']) if sim3 else O.fuse_search(c, c['th'])
    return _ORACLE[key]


def same(a, b):
    return a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()


@pytest.mark.parametrize('ori', (False, True))
@pytest.mark.parametrize('c', BOW, ids=[c['name'] for c in BOW])
def test_search_by_bow(orb, c, ori):
    """Both overloads: the KeyFrame-Frame form (match, nmatches) and the KeyFrame-KeyFrame form (match12, nmatches), each twice."""
    m = orb.ORBmatcher(float(c['nnratio']), ori, max_batch=1, max_keypoints=S.N, max_mappoints=S.N)
    a = (c['kk'], c['dk'], c['kp'], c['fvk'], c['kf'], c['df'], c['fvf'])
    on, om = O.search_by_bow(*a, nnratio=c['nnratio'], check_ori=ori)
    for _ in range(2):
        n, match = m.SearchByBoW(*a)
        assert n == on and match.tobytes() == om.tobytes(), (c['name'], n, on, np.flatnonzero(match != om)[:10])
    b = (c['kk'], c['dk'], c['kp'], c['fvk'], c['kf'], c['df'], c['fp'], c['fvf'])
    on, om = O.search_by_bow_kf(*b, nnratio=c['nnratio'], check_ori=ori)
    for _ in range(2):
        n, m12 = m.SearchByBoWKF(*b)
        assert n == on and m12.tobytes() == om.tobytes(), (c['name'], n, on, np.flatnonzero(m12 != om)[:10])


def tri_oracle(c, ori):
    out = []
    for k, kf2 in enumerate(c['kf2']):
        sc = dict(k1=c['kf1']['kps'], d1=c['kf1']['desc'], mp1=c['kf1']['has_mp'], fv1=c['kf1']['fv'], k2=kf2['kps'], d2=kf2['desc'], mp2=kf2['has_mp'],
                  fv2=kf2['fv'], sf=c['sf'], sigma2=c['sigma2'])
        out.append(O.search_for_triangulation(sc, c['ep'][k], c['F12'][k], c['coarse'], ori))
    return out


@pytest.mark.parametrize('ori', (False, True))
@pytest.mark.parametrize('c', TRI, ids=[c['name'] for c in TRI])
def test_search_for_triangulation(orb, c, ori):
    m = orb.ORBmatcher(0.6, ori, max_batch=1, max_keypoints=S.N, max_mappoints=S.N)
    want = tri_oracle(c, ori)
    for _ in range(2):
        nm, m12 = m.SearchForTriangulation(c['kf1'], c['kf2'], c['sf'], c['sigma2'], c['ep'], c['F12'], c['coarse'])
        for k, (on, om) in enumerate(want):
            assert nm[k] == on and m12[k].tobytes() == om.tobytes(), (c['name'], k, nm[k], on, np.flatnonzero(m12[k] != om)[:10])


FUSE_ARGS = ('kps', 'desc', 'bounds', 'sf', 'isg', 'log_sf', 'Tcw', 'Ow', 'cam', 'state', 'xyz', 'normal', 'min_d', 'max_d', 'mp_desc')


@pytest.mark.parametrize('c', FUSE, ids=[c['name'] for c in FUSE])
def test_fuse_search(orb, c):
    """Fuse(KeyFrame*, vpMapPoints) alone and as a batch of one, and Fuse(KeyFrame*, Scw, ...) (no chi-square gate)."""
    m = orb.ORBmatcher(0.6, True, max_batch=1, max_keypoints=KCAP, max_mappoints=64)
    want = fuse_oracle(c)
    got = m.FuseSearch(*[c[k] for k in FUSE_ARGS], th=c['th'])
    assert same(got, want), (c['name'], np.flatnonzero(got[0] != want[0])[:10])
    assert m.last_launch_count() == 1
    assert same(m.fuse_search_batch([c])[0], want)
    a = [c[k] for k in FUSE_ARGS if k != 'isg']
    got = m.FuseSearchSim3(*a, th=c['th'])
    assert same(got, fuse_oracle(c, True)), c['name']


def _empty(c, what):
    """Item c with no keypoints (K == 0) or no map points (M == 0)."""
    if what == 'K':
        return dict(c, kps=c['kps'][:0], desc=c['desc'][:0])
    return dict(c, **{k: c[k][:0] for k in ('state', 'xyz', 'normal', 'min_d', 'max_d', 'mp_desc')})


def test_fuse_batch_all_cases_two_orders(orb):
    """Every Fuse case in one fuse_search_batch, forwards and backwards, with K == 0 and M == 0 items between them: a small item after a
    global-layout one and the reverse; the shared memory of the launch comes from the largest keyframe.  Repeated: byte-identical."""
    m = orb.ORBmatcher(0.6, True, max_batch=1, max_keypoints=KCAP, max_mappoints=64)
    items = []
    for i, c in enumerate(FUSE):
        items.append(c)
        if i % 3 == 1:
            items.append(_empty(c, 'K' if i % 2 else 'M'))
    for order in (items, items[::-1]):
        res = m.fuse_search_batch(order)
        assert m.last_launch_count() == 1
        for it, got in zip(order, res):
            if len(it['kps']) == 0 or len(it['state']) == 0:
                assert (got[0] == -1).all() and (got[1] == 256).all()
            else:
                assert same(got, fuse_oracle(it)), it['name']
        again = m.fuse_search_batch(order)
        assert all(same(a, b) for a, b in zip(res, again))


def test_fuse_one_handle_alternates_layouts(orb):
    """The 14,008-keypoint keyframe (descriptors in global memory, the largest accepted) and small keyframes in turn on one handle."""
    m = orb.ORBmatcher(0.6, True, max_batch=1, max_keypoints=KCAP, max_mappoints=64)
    big = next(c for c in FUSE if c['shape'].get('K') == S.K_MAX)
    small = [c for c in FUSE if c['name'] in ('real_M_129', 'edges', 'real_M_1')]
    for c in [big, small[0], big, small[1], small[2], big]:
        got = m.FuseSearch(*[c[k] for k in FUSE_ARGS], th=c['th'])
        assert same(got, fuse_oracle(c)), c['name']


def test_fuse_refuses_keyframe_past_the_layout(orb):
    """K = 14,009 fits no shared-memory layout: ORB_ERR_CAPACITY before anything is staged, 0 launches on a fresh handle, the previous call's
    count after an earlier call; an exact call right after the refusal succeeds."""
    big = S.refused_keyframe()
    ok = next(c for c in FUSE if c['shape'].get('K') == S.K_MAX)
    fresh = orb.ORBmatcher(0.6, True, max_batch=1, max_keypoints=KCAP, max_mappoints=64)
    with pytest.raises(orb.OrbError) as e:
        fresh.fuse_search_batch([big])
    assert e.value.code == orb.ORB_ERR_CAPACITY and fresh.last_launch_count() == 0
    m = orb.ORBmatcher(0.6, True, max_batch=1, max_keypoints=KCAP, max_mappoints=64)
    m.fuse_search_batch([ok])
    for items in ([big], [ok, big], [big, ok]):
        with pytest.raises(orb.OrbError) as e:
            m.fuse_search_batch(items)
        assert e.value.code == orb.ORB_ERR_CAPACITY and m.last_launch_count() == 1
    assert same(m.fuse_search_batch([ok])[0], fuse_oracle(ok))
    with pytest.raises(orb.OrbError) as e:
        m.FuseSearch(*[big[k] for k in FUSE_ARGS], th=big['th'])
    assert e.value.code == orb.ORB_ERR_CAPACITY
    assert same(m.FuseSearch(*[ok[k] for k in FUSE_ARGS], th=ok['th']), fuse_oracle(ok))


@pytest.mark.parametrize('c', SIM3, ids=[c['name'] for c in SIM3])
def test_search_by_sim3(orb, c):
    m = orb.ORBmatcher(0.75, True, max_batch=1, max_keypoints=KCAP, max_mappoints=64)
    n, m12 = m.SearchBySim3(c['kf1'], c['kf2'], S.BOUNDS, c['sf'], c['log_sf'], c['cam'], c['pre12'], c['th'])
    sc = dict(sf=c['sf'], log_sf=c['log_sf'], bounds=S.BOUNDS, cam=c['cam'], pre12=c['pre12'])
    for k, kf in ((1, c['kf1']), (2, c['kf2'])):
        sc.update({'k%d' % k: kf['kps'], 'd%d' % k: kf['desc'], 'state%d' % k: kf['state'], 'min%d' % k: kf['min_d'], 'max%d' % k: kf['max_d'],
                   'mpd%d' % k: kf['mp_desc']})
    on, om = O.search_by_sim3(sc, c['kf1']['pcam'], c['kf2']['pcam'], c['th'])
    assert n == on and m12.tobytes() == om.tobytes(), (c['name'], n, on)


def _np_item(sc):
    return dict(kf1=sc['kf1'], kf2_list=sc['kf2'], scale_factors=sc['sf'], level_sigma2=sc['sigma2'], ep=sc['ep'], F12=sc['F12'], Tcw=sc['Tcw'],
                Ow=sc['Ow'], cam=sc['cam'], scale_factor=sc['scale_factor'])


def test_create_new_map_points_at_the_pair_limit(orb):
    """Exactly 65,535 (keyframe, neighbour) pairs in one call (new_points_kernel's gridDim.y): every item equals the oracle, and the item
    holding the last pair equals its single-item call.  The item with the largest KF1 (maxN1) is not the one with the most pairs."""
    items = S.wide_new_points()
    assert sum(len(sc['kf2']) for sc in items) == S.MAX_PAIRS
    m = orb.ORBmatcher(0.6, False, max_batch=1, max_keypoints=S.N, max_mappoints=S.N)
    res = m.create_new_map_points_batch([_np_item(sc) for sc in items])
    assert m.last_launch_count() == 3
    for sc, (rec, nm, nc) in zip(items, res):
        orec, onm, onc, _ = NP.create(sc)
        assert rec.tobytes() == orec.tobytes() and nm.tobytes() == onm.tobytes() and nc.tobytes() == onc.tobytes()
    assert len(res[2][0]) > 0 and res[1][1].sum() > 0
    single = m.CreateNewMapPoints(*_np_item(items[2]).values())
    assert all(a.tobytes() == b.tobytes() for a, b in zip(single, res[2]))
