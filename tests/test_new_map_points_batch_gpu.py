"""GPU tests of orbm_create_new_map_points_batch (LocalMapping::CreateNewMapPoints for new keyframes of several maps in one call): every item
equals orbm_create_new_map_points of that item and the oracle byte for byte, whatever its position in the batch and whatever ran on the
handle before; 3 launches (0 when every item is empty); the argument and capacity errors before any launch; the C++ mirror's digest equals
the Python binding's.  Scenes of tests/new_points_lib.py at different frames / seeds stand in for the new keyframes of different maps."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import new_points_lib as NP
from orb_slam3_modified_b200 import synth

pytestmark = pytest.mark.gpu

DTS = {0: (), 1: (3,), 5: (2, -2, 4, -4, 6), 30: tuple(d for a in range(1, 16) for d in (a, -a))}
SETTINGS = [(False, False, 0.0), (False, True, 0.0), (True, False, 3.3), (True, True, 0.0), (False, False, 3.3)]


@pytest.fixture(scope='module')
def orb():
    import orb_slam3_modified_b200 as m
    m.lib()
    return m


@pytest.fixture(scope='module')
def matcher(orb):
    return orb.ORBmatcher(0.6, False, max_batch=1, max_keypoints=2048, max_mappoints=2048)


def _no_features(sc):
    """The scene with a KF1 of no features (KF1.N == 0)."""
    kf1 = sc['kf1']
    return dict(sc, kf1=dict(kps=kf1['kps'][:0], desc=kf1['desc'][:0], has_mp=kf1['has_mp'][:0], fv=(kf1['fv'][0][:0], kf1['fv'][1][:0])))


_SPECS = {}


def specs(B):
    """B items (scene, coarse, inertial, thFar): neighbour counts 0 / 1 / 5 / 30 in turn, frames 16..22, two seeds, the settings in turn; item 2
    of a batch of 7 or more has KF1.N == 0."""
    if B not in _SPECS:
        out = []
        for j in range(B):
            n = (30, 5, 1, 0)[j % 4] if j else 30
            sc = NP.scene(16 + j % 7, DTS[n], seed=j // 7)
            if j == 2 and B >= 7:
                sc = _no_features(NP.scene(16, DTS[5]))
            out.append((sc,) + SETTINGS[j % len(SETTINGS)])
        _SPECS[B] = out
    return _SPECS[B]


def item(sc, coarse=False, inertial=False, th_far=0.0):
    return dict(kf1=sc['kf1'], kf2_list=sc['kf2'], scale_factors=sc['sf'], level_sigma2=sc['sigma2'], ep=sc['ep'], F12=sc['F12'], Tcw=sc['Tcw'],
                Ow=sc['Ow'], cam=sc['cam'], scale_factor=sc['scale_factor'], coarse=coarse, inertial=inertial, th_far_points=th_far)


def same(a, b):
    return len(a) == len(b) and all(x[0].tobytes() == y[0].tobytes() and x[1].tobytes() == y[1].tobytes() and x[2].tobytes() == y[2].tobytes()
                                    for x, y in zip(a, b))


@pytest.mark.parametrize('B', [1, 7, 24])
def test_batch_equals_single_calls(matcher, B):
    """Records, nNew, nmatches and ncreated of every item == orbm_create_new_map_points of that item, byte for byte; 3 launches."""
    its = [item(*s) for s in specs(B)]
    res = matcher.create_new_map_points_batch(its)
    assert matcher.last_launch_count() == 3
    single = [matcher.CreateNewMapPoints(**it) for it in its]
    assert same(res, single)
    assert sum(len(r[0]) for r in res) > 0
    if B >= 7:
        assert len(res[2][0]) == 0 and not res[2][1].any() and not res[2][2].any() and len(res[2][1]) == 5
        assert len(res[3][1]) == 0


def test_batch_equals_oracle(matcher):
    """Every item of a 24-item batch == the oracle's orbo_create_new_map_points (records in order, per-neighbour counts)."""
    sp = specs(24)
    res = matcher.create_new_map_points_batch([item(*s) for s in sp])
    for j, ((sc, coarse, inertial, th_far), (rec, nm, nc)) in enumerate(zip(sp, res)):
        if len(sc['kf1']['kps']) == 0:
            continue
        orec, onm, onc, _ = NP.create(sc, coarse, inertial, th_far)
        assert rec.tobytes() == orec.tobytes() and np.array_equal(nm, onm) and np.array_equal(nc, onc), j


def test_all_empty_batch_launches_nothing(matcher):
    sp = specs(7)
    matcher.create_new_map_points_batch([item(*sp[0])])
    assert matcher.last_launch_count() == 3
    res = matcher.create_new_map_points_batch([item(*sp[3]), item(*sp[2]), item(*sp[3])])         # no neighbours; KF1 without features
    assert matcher.last_launch_count() == 0
    assert all(len(r[0]) == 0 and not r[1].any() and not r[2].any() for r in res)
    assert matcher.create_new_map_points_batch([]) == [] and matcher.last_launch_count() == 0


def test_position_independence(matcher):
    """A permuted batch gives every item the same bytes (catches offset mistakes in the item and pair tables)."""
    its = [item(*s) for s in specs(24)]
    ref = matcher.create_new_map_points_batch(its)
    perm = np.random.default_rng(5).permutation(len(its))
    res = matcher.create_new_map_points_batch([its[p] for p in perm])
    assert same([res[int(np.nonzero(perm == j)[0][0])] for j in range(len(its))], ref)
    rev = matcher.create_new_map_points_batch(its[::-1])
    assert same(rev[::-1], ref)


def _fuse_item(sc):
    """One Fuse search on KF1 of the scene: the points of its first neighbour's keypoints, back-projected."""
    kps, desc = sc['kf1']['kps'], sc['kf1']['desc']
    k2, d2 = sc['kf2'][0]['kps'], sc['kf2'][0]['desc']
    P = synth.backproject(np.stack([k2['x'], k2['y']], 1), 19).astype(np.float32)
    M = len(P)
    Ow = sc['Ow'][0]
    d = np.linalg.norm(P - Ow, axis=1).astype(np.float32)
    return dict(kps=kps, desc=desc, bounds=(0.0, 0.0, 640.0, 480.0), sf=sc['sf'], isg=(1.0 / sc['sigma2']).astype(np.float32),
                log_sf=np.float32(np.log(np.float32(1.2))), Tcw=synth.pose(17).astype(np.float32), Ow=Ow, cam=synth.camera(),
                state=np.ones(M, np.uint8), xyz=P, normal=((P - Ow) / d[:, None]).astype(np.float32), min_d=d * np.float32(0.5), max_d=d * np.float32(2.0),
                mp_desc=d2)


def test_staging_reuse(matcher):
    """The same batch before and after a Fuse batch and a larger batch on the same handle gives identical bytes."""
    small = [item(*s) for s in specs(7)]
    first = matcher.create_new_map_points_batch(small)
    matcher.fuse_search_batch([_fuse_item(specs(7)[1][0])])
    assert matcher.last_launch_count() == 1
    big = matcher.create_new_map_points_batch([item(*s) for s in specs(24)])
    assert matcher.last_launch_count() == 3 and sum(len(r[0]) for r in big) > sum(len(r[0]) for r in first)
    again = matcher.create_new_map_points_batch(small)
    assert same(again, first)


class _Raw:
    """An OrbmNewPointsItem array over NP._In inputs, with outputs pre-filled with sentinels."""

    def __init__(self, orb, ins):
        self.ins = ins
        self.arr = (orb.OrbmNewPointsItem * max(len(ins), 1))()
        self.outs = []
        for j, i in enumerate(ins):
            o = np.full(max(i.N1, 1) * orb.NEW_POINT_DTYPE.itemsize, 0x5A, np.uint8)
            n, nm, nc = np.full(1, -9, np.int32), np.full(max(i.n, 1), -9, np.int32), np.full(max(i.n, 1), -9, np.int32)
            self.outs.append((o, n, nm, nc))
            self.arr[j] = orb.OrbmNewPointsItem(i.s, o.ctypes.data, n.ctypes.data, nm.ctypes.data, nc.ctypes.data)

    def untouched(self):
        return all((o == 0x5A).all() and (n == -9).all() and (nm == -9).all() and (nc == -9).all() for o, n, nm, nc in self.outs)


def test_bad_arguments(orb, matcher):
    """ORB_ERR_ARG before any launch for a defect in any item: octave out of range in KF1 or a neighbour, an unsorted feature vector, null
    outputs, missing poses, nItems < 0; the launch count and every item's outputs stay as they were."""
    L = orb.lib()
    sc = specs(7)[1][0]                                  # 5 neighbours
    good = [NP._In(s[0]) for s in specs(7)[:2]]
    matcher.create_new_map_points_batch([item(*specs(7)[0])])
    assert matcher.last_launch_count() == 3

    def call(bad_in, n=None, **null):
        r = _Raw(orb, good + [bad_in])
        for f in null:
            setattr(r.arr[len(good)], f, None)
        rc = L.orbm_create_new_map_points_batch(matcher._h, len(good) + 1 if n is None else n, r.arr)
        assert r.untouched() and matcher.last_launch_count() == 3
        return rc
    bad_oct = dict(sc, kf1=dict(sc['kf1'], kps=sc['kf1']['kps'].copy()))
    bad_oct['kf1']['kps']['octave'][7] = 8
    bad_oct2 = dict(sc, kf2=list(sc['kf2']))
    bad_oct2['kf2'][3] = dict(sc['kf2'][3], kps=sc['kf2'][3]['kps'].copy())
    bad_oct2['kf2'][3]['kps']['octave'][0] = -1
    fvn = sc['kf2'][1]['fv'][0].copy(); fvn[[0, -1]] = fvn[[-1, 0]]
    bad_fv = dict(sc, kf2=list(sc['kf2']))
    bad_fv['kf2'][1] = dict(sc['kf2'][1], fv=(fvn, sc['kf2'][1]['fv'][1]))
    for s in (bad_oct, bad_oct2, bad_fv):
        assert call(NP._In(s)) == orb.ORB_ERR_ARG
        assert 'item 2' in L.orb_last_error().decode()
    for f in ('out', 'nNew', 'nmatches', 'ncreated'):
        assert call(NP._In(sc), **{f: None}) == orb.ORB_ERR_ARG
    nopose = NP._In(sc)
    nopose.s.Tcw = None
    assert call(nopose) == orb.ORB_ERR_ARG
    assert call(NP._In(sc), n=-1) == orb.ORB_ERR_ARG
    assert L.orbm_create_new_map_points_batch(matcher._h, 2, None) == orb.ORB_ERR_ARG
    r = _Raw(orb, good + [NP._In(sc)])
    assert L.orbm_create_new_map_points_batch(matcher._h, 3, r.arr) == orb.ORB_OK and not r.untouched()


def test_too_many_pairs(orb, matcher):
    """More than 65535 (keyframe, neighbour) pairs: ORB_ERR_CAPACITY naming the item where the count passes the limit, before any launch.
    Neighbours without features keep the check cheap: a pair counts whenever KF1 has features."""
    L = orb.lib()
    sc = specs(7)[1][0]
    empty = NP.scene(16, ())['kf1']
    empty = dict(kps=empty['kps'][:0], desc=empty['desc'][:0], has_mp=empty['has_mp'][:0], fv=(empty['fv'][0][:0], empty['fv'][1][:0]))

    def wide(n):
        return dict(sc, kf2=[empty] * n, ep=np.zeros((n, 2), np.float32), F12=np.zeros((n, 9), np.float32),
                    Tcw=np.tile(sc['Tcw'][:1], (n + 1, 1, 1)), Ow=np.tile(sc['Ow'][:1], (n + 1, 1)), cam=np.tile(sc['cam'][:1], (n + 1, 1)))
    matcher.create_new_map_points_batch([item(*specs(7)[0])])
    r = _Raw(orb, [NP._In(specs(7)[0][0]), NP._In(wide(32768)), NP._In(_no_features(wide(40000))), NP._In(wide(32768))])
    assert L.orbm_create_new_map_points_batch(matcher._h, 4, r.arr) == orb.ORB_ERR_CAPACITY
    assert 'item 3' in L.orb_last_error().decode()
    assert r.untouched() and matcher.last_launch_count() == 3


def _digest(res):
    h = 14695981039346656037
    for rec, nm, nc in res:
        for b in rec.tobytes() + nm.tobytes() + nc.tobytes():
            h = ((h ^ b) * 1099511628211) & 0xFFFFFFFFFFFFFFFF
    return h


def test_cpp_create_new_map_points_batch_equals_python(orb, tmp_path):
    """ORBmatcher::CreateNewMapPointsBatch (include/orb_b200/orb_slam3.hpp) from a g++-built caller: seven keyframes, an empty neighbour
    list and a KF1 without features among them, give the Python binding's digest in 3 launches."""
    sp = specs(7)
    lines = ['%d' % len(sp)]
    for j, (sc, coarse, inertial, th_far) in enumerate(sp):
        kfs = [sc['kf1']] + list(sc['kf2'])
        dims = [len(sc['kf1']['kps']), len(sc['kf1']['fv'][0]), len(sc['kf2']), len(sc['sf']), repr(float(sc['scale_factor'])), int(coarse), int(inertial),
                repr(float(th_far))]
        dims += [v for kf in sc['kf2'] for v in (len(kf['kps']), len(kf['fv'][0]))]
        lines.append(' '.join(str(v) for v in dims))
        for k, kf in enumerate(kfs):
            p = 'item%d_kf1' % j if k == 0 else 'item%d_kf2_%d' % (j, k - 1)
            for nm, a, dt in (('kps', kf['kps'], orb.KP_DTYPE), ('desc', kf['desc'], np.uint8), ('mp', kf['has_mp'], np.uint8), ('fvn', kf['fv'][0], np.int32),
                              ('fvf', kf['fv'][1], np.int32)):
                np.ascontiguousarray(a, dt).tofile(str(tmp_path / (p + '_' + nm + '.raw')))
        for nm, key in (('sf', 'sf'), ('sg', 'sigma2'), ('ep', 'ep'), ('F12', 'F12'), ('Tcw', 'Tcw'), ('Ow', 'Ow'), ('cam', 'cam')):
            np.ascontiguousarray(sc[key], np.float32).tofile(str(tmp_path / ('item%d_%s.raw' % (j, nm))))
    (tmp_path / 'dims.txt').write_text('\n'.join(lines) + '\n')
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib = os.path.join(root, 'orb_slam3_modified_b200')
    exe = tmp_path / 'new_map_points_example'
    subprocess.check_call(['g++', '-std=c++14', '-O2', '-Wall', '-I', os.path.join(root, 'include'), os.path.join(root, 'tests', 'new_map_points_example.cpp'),
                           '-o', str(exe), '-L', lib, '-l:liborb_b200.so', '-Wl,-rpath,' + lib, '-lpthread'])
    out = dict(l.split() for l in subprocess.check_output([str(exe), str(tmp_path)]).decode().splitlines())
    m = orb.ORBmatcher(0.6, False, max_batch=1, max_keypoints=2048, max_mappoints=64)
    res = m.create_new_map_points_batch([item(*s) for s in sp])
    assert out['digest'] == '%016x' % _digest(res)
    assert int(out['created']) == sum(len(r[0]) for r in res) > 100
    assert out['launches'] == '3'
