"""GPU tests of orbm_keyframe_culling_batch: per map, status / nMPs / nRedundant / visited equal the oracle's for batches of mono and
inertial maps with empty maps mixed in; a batch equals per-map calls byte for byte; one launch per call; the host replay of the statuses
gives the oracle's final map; the argument errors; the C++ mirror's digest equals the Python binding's."""
import os
import subprocess

import numpy as np
import pytest

import keyframe_culling_lib as K

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def orb():
    import orb_slam3_modified_b200 as m
    m.lib()
    return m


@pytest.fixture(scope='module')
def matcher(orb):
    return orb.ORBmatcher(0.6, True, max_batch=1, max_keypoints=64, max_mappoints=64)


def _no_points(seed):
    """Local keyframes that hold no point: every keyframe is evaluated with nMPs = 0 and kept."""
    cm = K.corridor(seed, n_kf=12)
    for kf in cm.kfs:
        kf.mp[:] = -1
    for p in cm.pts:
        p.obs, p.nObs = {}, 0
    return cm


def _no_local(seed):
    cm = K.corridor(seed, n_kf=8, inertial=bool(seed % 2))
    cm.local = []
    return cm


def _models(B, seed):
    """B maps: seeded corridors (mono and inertial, shuffled or newest-first, some with abortBA or over 100 local keyframes) with a map
    without local keyframes and one whose keyframes hold no point mixed in."""
    out = []
    for s in range(B):
        r = seed * 100 + s
        if B > 1 and s == 1:
            out.append(_no_local(r))
        elif B > 2 and s == 2:
            out.append(_no_points(r))
        elif s % 11 == 5:
            out.append(K.corridor(r, n_kf=120, new_per_kf=5))
        else:
            out.append(K.corridor(r, n_kf=20 + (7 * s) % 30, inertial=s % 2 == 0, order='shuffle' if s % 3 else 'newest', kf_extra=(s % 4) * 4 - 8,
                                  abort=s % 5 == 3, imu_init=s % 3 != 1, ba2=s % 7 == 6))
    return out


def _equal(a, b):
    return all(a[k].tobytes() == b[k].tobytes() for k in ('status', 'nMPs', 'nRedundant')) and a['visited'] == b['visited']


@pytest.mark.parametrize('B', [1, 7, 24])
def test_batch_equals_oracle_and_single_calls(orb, matcher, B):
    models = _models(B, B)
    flat = [K.flatten(cm) for cm in models]
    got = matcher.keyframe_culling_batch(flat)
    assert matcher.last_launch_count() == 1
    statuses = set()
    for cm, m, g in zip(models, flat, got):
        ref, state = K.oracle(m)
        assert _equal(g, ref)
        assert K.same_state(K.replay(cm, g)[0], state)                   # the host replay reproduces the oracle's final map
        statuses |= set(g['status'].tolist())
    for m, g in zip(flat, got):
        one = matcher.keyframe_culling_batch([m])[0]
        assert _equal(one, g)
        assert matcher.last_launch_count() == (1 if len(m['local']) else 0)
    if B == 24:
        assert {K.SKIPPED, K.KEPT, K.CULLED, K.CULLED_TIME, K.KEPT_IMU, K.NOT_VISITED} <= statuses


def test_planted_scenes_equal_oracle(orb, matcher):
    """The CPU tests' planted rules, all in one batch: the cascade, the float boundaries, the guards, the break tests."""
    models = [K.cascade(), K.dense(30, inertial=True, kf_in_map=24), K.dense(40), K.dense(40, inertial=True, kf_in_map=21)]
    models[2].abort = models[3].abort = True
    for n in (10, 20, 90, 250):
        models += [K.boundary(n, n * 9 // 10), K.boundary(n, n * 9 // 10 + 1)]
    for lim, init in ((3.0, True), (0.5, False)):
        models += [K.one_inertial(lim - 1e-9, imu_init=init), K.one_inertial(lim - 1e-6, imu_init=init)]
    models += [K.one_inertial(1.0, gap=0.02 - 1e-5), K.one_inertial(1.0, gap=0.02 + 1e-5)]
    wrap = K.dense(30, inertial=True)
    wrap.local, wrap.current_id = [28, 27], 1
    models.append(wrap)
    flat = [K.flatten(cm) for cm in models]
    got = matcher.keyframe_culling_batch(flat)
    for cm, m, g in zip(models, flat, got):
        ref, state = K.oracle(m)
        assert _equal(g, ref)
        assert K.same_state(K.replay(cm, g)[0], state)


def test_launch_counts(orb, matcher):
    matcher.keyframe_culling_batch([K.flatten(K.corridor(3))])
    assert matcher.last_launch_count() == 1
    out = matcher.keyframe_culling_batch([K.flatten(_no_local(1)), K.flatten(_no_local(2))])
    assert matcher.last_launch_count() == 0 and [o['visited'] for o in out] == [0, 0]
    matcher.keyframe_culling_batch([])
    assert matcher.last_launch_count() == 0


def test_bad_arguments(orb, matcher):
    L = orb.lib()
    base = [K.flatten(K.corridor(5)), K.flatten(K.corridor(6, inertial=True, kf_extra=5))]
    matcher.keyframe_culling_batch(base)
    assert matcher.last_launch_count() == 1

    def expect(edit, struct_edit=None):
        maps = [{k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in m.items()} for m in base]
        edit(maps)
        built = [orb.culling_struct(m) for m in maps]
        arr = (orb.OrbmCullingMap * len(built))(*[b[0] for b in built])
        if struct_edit:
            struct_edit(arr)
        assert L.orbm_keyframe_culling_batch(matcher._h, len(built), arr) == orb.ORB_ERR_ARG
        assert matcher.last_launch_count() == 1                           # rejected before any launch: the previous call's count stays

    def setv(key, i, v, j=0):
        def f(maps): maps[j][key][i] = v
        return f
    expect(setv('local', 3, 10 ** 6))
    expect(setv('local', 0, -1, 1))
    expect(setv('slotPoint', 7, len(base[0]['pointBad'])))
    expect(setv('obsKF', 2, len(base[1]['kfFlags']), 1))
    expect(setv('slotOctave', 4, 256))
    expect(setv('obsOctave', 9, -1))
    expect(setv('prevKF', 5, len(base[1]['kfFlags']), 1))
    expect(setv('nextKF', 5, -2, 1))
    expect(setv('slotStart', 2, 0))                                       # decreasing
    expect(setv('obsStart', 0, 1, 1))                                     # not starting at 0
    expect(lambda maps: None, lambda a: setattr(a[0], 'nLocal', a[0].nKF + 1))
    expect(lambda maps: None, lambda a: setattr(a[1], 'nPoints', -1))
    for field, j in (('timeStamp', 1), ('imuPosition', 1), ('prevKF', 1), ('status', 0), ('nMPs', 1), ('visited', 0), ('slotPoint', 0),
                     ('obsKF', 1), ('kfFlags', 0), ('mnId', 1), ('pointBad', 0)):
        expect(lambda maps: None, lambda a, f=field, j=j: setattr(a[j], f, None))
    assert L.orbm_keyframe_culling_batch(matcher._h, -1, None) == orb.ORB_ERR_ARG
    assert L.orbm_keyframe_culling_batch(matcher._h, 2, None) == orb.ORB_ERR_ARG
    # the inertial arrays are not needed by a monocular map
    mono = {k: v for k, v in base[0].items() if k not in ('prevKF', 'nextKF', 'timeStamp', 'imuPosition')}
    matcher.keyframe_culling_batch([mono])
    assert matcher.last_launch_count() == 1


def _digest(out):
    h = 14695981039346656037
    for o in out:
        for b in o['status'].tobytes() + o['nMPs'].tobytes() + o['nRedundant'].tobytes() + np.int32(o['visited']).tobytes():
            h = ((h ^ b) * 1099511628211) & 0xFFFFFFFFFFFFFFFF
    return h


def test_cpp_keyframe_culling_batch_equals_python(orb, matcher, tmp_path):
    """ORBmatcher::KeyFrameCullingBatch (include/orb_b200/orb_slam3.hpp) from a g++-built caller gives the Python binding's digest."""
    flat = [K.flatten(cm) for cm in _models(6, 41)]
    lines = [str(len(flat))]
    for j, m in enumerate(flat):
        lines.append(' '.join(str(int(v)) for v in (len(m['kfFlags']), len(m['local']), len(m['pointBad']), m['inertial'], m['imuInitialized'],
                                                    m['inertialBA2'], m['abortBA'], m['keyFramesInMap'], m['currentId'], m['lastId'])))
        for name, dt in orb.CULLING_ARRAYS:
            data = np.ascontiguousarray(m[name], dt).tobytes() if m.get(name) is not None else b''
            (tmp_path / ('map%d_%s.raw' % (j, name))).write_bytes(data)
    (tmp_path / 'dims.txt').write_text('\n'.join(lines) + '\n')
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib = os.path.join(root, 'orb_slam3_modified_b200')
    exe = tmp_path / 'keyframe_culling_example'
    subprocess.check_call(['g++', '-std=c++14', '-O2', '-Wall', '-I', os.path.join(root, 'include'), os.path.join(root, 'tests', 'keyframe_culling_example.cpp'),
                           '-o', str(exe), '-L', lib, '-l:liborb_b200.so', '-Wl,-rpath,' + lib, '-lpthread'])
    out = dict(l.split() for l in subprocess.check_output([str(exe), str(tmp_path)]).decode().splitlines())
    res = matcher.keyframe_culling_batch(flat)
    assert out['digest'] == '%016x' % _digest(res)
    assert int(out['culled']) == sum(int((o['status'] >= K.CULLED).sum()) for o in res) > 10
    assert out['launches'] == '1'
