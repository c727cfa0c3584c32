"""LocalMapping::CreateNewMapPoints on the GPU (orbm_create_new_map_points) against the CPU oracle, bit for bit."""
import ctypes as C

import numpy as np
import pytest

import new_points_lib as NP

pytestmark = pytest.mark.gpu

DTS = {0: (), 1: (3,), 5: (2, -2, 4, -4, 6), 30: tuple(d for a in range(1, 16) for d in (a, -a))}


@pytest.fixture(scope='module')
def orb():
    import orb_slam3_modified_b200 as m
    m.lib()
    return m


@pytest.fixture(scope='module')
def matcher(orb):
    return orb.ORBmatcher(0.6, False, max_batch=1, max_keypoints=2048, max_mappoints=2048)


@pytest.fixture(scope='module')
def scenes():
    return {n: NP.scene(18, dts) for n, dts in DTS.items()}


def gpu(m, sc, coarse=False, inertial=False, th_far=0.0):
    return m.CreateNewMapPoints(sc['kf1'], sc['kf2'], sc['sf'], sc['sigma2'], sc['ep'], sc['F12'], sc['Tcw'], sc['Ow'], sc['cam'], sc['scale_factor'],
                                coarse=coarse, inertial=inertial, th_far_points=th_far)


@pytest.mark.parametrize('n', [0, 1, 5, 30])
@pytest.mark.parametrize('coarse,inertial,th_far', [(False, False, 0.0), (False, True, 0.0), (True, False, 3.3), (True, True, 0.0), (False, False, 3.3)])
def test_equals_oracle(matcher, scenes, n, coarse, inertial, th_far):
    """Records (order, kf2 / idx1 / idx2, float x3D, normal, distances), nmatches and ncreated == the oracle; a second call is byte-identical."""
    sc = scenes[n]
    rec, nm, nc = gpu(matcher, sc, coarse, inertial, th_far)
    orec, onm, onc, why = NP.create(sc, coarse, inertial, th_far)
    assert len(rec) == len(orec) and rec.tobytes() == orec.tobytes(), (len(rec), len(orec))
    assert np.array_equal(nm, onm) and np.array_equal(nc, onc)
    if n:
        assert len(rec) > 0 and matcher.last_launch_count() == 3
        if th_far:
            assert (why == NP.FAR).any()
    rec2, nm2, nc2 = gpu(matcher, sc, coarse, inertial, th_far)
    assert rec2.tobytes() == rec.tobytes() and np.array_equal(nm2, nm) and np.array_equal(nc2, nc)


@pytest.mark.parametrize('n,coarse,inertial', [(1, False, False), (5, False, True), (30, False, False), (30, True, True)])
def test_equals_sequential_loop_of_gpu_searches(matcher, scenes, n, coarse, inertial):
    """One call == the reference's loop built from orbm_search_for_triangulation, one neighbour at a time with KF1's hasMapPoint updated
    after each, followed by the oracle's checks of every match."""
    sc = scenes[n]

    def search(k, has):
        kf1 = dict(sc['kf1'], has_mp=has)
        return matcher.SearchForTriangulation(kf1, [sc['kf2'][k]], sc['sf'], sc['sigma2'], sc['ep'][k:k + 1], sc['F12'][k:k + 1], coarse)[1][0]
    srec, snm, snc = NP.sequential(sc, search, coarse, inertial)
    rec, nm, nc = gpu(matcher, sc, coarse, inertial)
    assert rec.tobytes() == srec.tobytes() and np.array_equal(nm, snm) and np.array_equal(nc, snc)
    if n > 1:
        static = matcher.SearchForTriangulation(sc['kf1'], sc['kf2'], sc['sf'], sc['sigma2'], sc['ep'], sc['F12'], coarse)[0]
        assert (static >= nm).all() and (static > nm).any()          # the one-launch search alone over-counts


def test_bad_arguments(orb, matcher, scenes):
    """ORB_ERR_ARG before any launch: octave out of range, unsorted feature vector, null outputs, missing poses."""
    sc = scenes[5]
    gpu(matcher, sc)
    assert matcher.last_launch_count() == 3
    L = orb.lib()

    def raw(s, out=True, n=True, nm=True, nc=True):
        o = np.zeros(2048, orb.NEW_POINT_DTYPE); a, b = np.zeros(8, np.int32), np.zeros(8, np.int32); k = C.c_int(0)
        return L.orbm_create_new_map_points(matcher._h, C.byref(s.s), o.ctypes.data if out else None, C.byref(k) if n else None,
                                            a.ctypes.data if nm else None, b.ctypes.data if nc else None)
    bad_oct = dict(sc, kf1=dict(sc['kf1'], kps=sc['kf1']['kps'].copy()))
    bad_oct['kf1']['kps']['octave'][7] = 8
    bad_oct2 = dict(sc, kf2=list(sc['kf2']))
    bad_oct2['kf2'][3] = dict(sc['kf2'][3], kps=sc['kf2'][3]['kps'].copy())
    bad_oct2['kf2'][3]['kps']['octave'][0] = -1
    fvn = sc['kf2'][1]['fv'][0].copy(); fvn[[0, -1]] = fvn[[-1, 0]]
    bad_fv = dict(sc, kf2=list(sc['kf2']))
    bad_fv['kf2'][1] = dict(sc['kf2'][1], fv=(fvn, sc['kf2'][1]['fv'][1]))
    for s in (bad_oct, bad_oct2, bad_fv):
        assert raw(NP._In(s)) == orb.ORB_ERR_ARG
    good = NP._In(sc)
    for kw in (dict(out=False), dict(n=False), dict(nm=False), dict(nc=False)):
        assert raw(good, **kw) == orb.ORB_ERR_ARG
    nopose = NP._In(sc)
    nopose.s.Tcw = None
    assert raw(nopose) == orb.ORB_ERR_ARG
    assert matcher.last_launch_count() == 3
    assert raw(good) == orb.ORB_OK
