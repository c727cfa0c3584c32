"""GPU tests of orbm_update_connections_batch: every output equals the oracle's byte for byte (normals and distances bitwise) for batches
mixing both modes with empty items and empty counters; a batch equals per-item calls; one launch per call; the host replay gives the
oracle's final map; a fresh point of orbm_create_new_map_points gets the record's normal and distances; the chosen rows equal
orbm_distinctive_descriptors'; the lockstep SearchInNeighbors driver followed by this call equals the oracle chain; the argument errors
come before any launch; the C++ mirror's digest equals the Python binding's."""
import copy
import os
import subprocess

import numpy as np
import pytest

import new_points_lib as NP
import search_in_neighbors_lib as SN
import update_connections_lib as U

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def orb():
    import orb_slam3_modified_b200 as m
    m.lib()
    return m


@pytest.fixture(scope='module')
def matcher(orb):
    return orb.ORBmatcher(0.6, True, max_batch=1, max_keypoints=2048, max_mappoints=64)


def _scenes(B, seed):
    """B keyframes: seeded scenes of both modes and several sizes, with an item without slots, one with an empty counter and (B = 24)
    one whose table is too large for the shared-memory counter mixed in."""
    out = []
    for s in range(B):
        r = seed * 100 + s
        if B > 1 and s == 1:
            out.append(U.scene(r, U.SIN, n_kf=8, n_slots=0))
        elif B > 2 and s == 2:
            out.append(U.planted()['empty_counter'])
        elif B == 24 and s == 5:
            out.append(U.scene(r, U.PNK, n_kf=4500, n_slots=120, obs_per_point=8))
        else:
            out.append(U.scene(r, U.PNK if s % 2 == 0 else U.SIN, n_kf=20 + (37 * s) % 130, n_slots=100 + (211 * s) % 900,
                               first=s % 3 == 0, init=s % 7 == 3))
    return out


@pytest.mark.parametrize('B', [1, 7, 24])
def test_batch_equals_oracle_and_single_calls(orb, matcher, B):
    scenes = _scenes(B, B)
    flat = [U.flatten(sc) for sc in scenes]
    got = matcher.update_connections_batch(flat)
    assert matcher.last_launch_count() == 1
    for sc, m, g in zip(scenes, flat, got):
        ref, fin = U.oracle(m)
        assert U.same_outputs(g, ref)
        assert U.final_state(U.replay(sc, g)) == fin
    for m, g in zip(flat, got):
        one = matcher.update_connections_batch([m])[0]
        assert U.same_outputs(one, g)
        assert matcher.last_launch_count() == (1 if len(m['slotPoint']) else 0)
    if B == 24:
        assert {g['nConnected'] for g in got} >= {-1} and max(g['nConnected'] for g in got) > 5
        assert any(g['parent'] >= 0 for g in got) and any((g['nbrCount'] >= 0).any() for g in got)


def test_planted_scenes_equal_oracle(orb, matcher):
    scenes = list(U.planted().values())
    flat = [U.flatten(sc) for sc in scenes]
    got = matcher.update_connections_batch(flat)
    for sc, m, g in zip(scenes, flat, got):
        ref, fin = U.oracle(m)
        assert U.same_outputs(g, ref)
        assert U.final_state(U.replay(sc, g)) == fin


def test_launch_counts(orb, matcher):
    empty = [U.flatten(U.scene(s, U.PNK, n_kf=8, n_slots=0)) for s in (1, 2)]
    out = matcher.update_connections_batch(empty)
    assert matcher.last_launch_count() == 0 and [o['nConnected'] for o in out] == [-1, -1]
    matcher.update_connections_batch([U.flatten(U.scene(3, U.SIN, n_kf=30, n_slots=200))] + empty)
    assert matcher.last_launch_count() == 1
    matcher.update_connections_batch([])
    assert matcher.last_launch_count() == 0


def test_fresh_point_of_create_new_map_points(orb, matcher):
    """A point just made by orbm_create_new_map_points: observed by KF1 and KF2, mpRefKF = KF1.  UpdateNormalAndDepth gives it the normal
    and distances of its record, bit for bit."""
    sc = NP.scene(18, (3,))
    recs, _, _ = matcher.CreateNewMapPoints(sc['kf1'], sc['kf2'], sc['sf'], sc['sigma2'], sc['ep'], sc['F12'], sc['Tcw'], sc['Ow'], sc['cam'],
                                             sc['scale_factor'])
    assert len(recs) > 50
    k1, k2 = sc['kf1'], sc['kf2'][0]
    for order in ((0x1000, 0x2000), (0x2000, 0x1000)):
        s = U.Scene(U.SIN, sc['sf'])
        s.add_kf(order[0], 7, sc['Ow'][0], k1['kps']['octave'], k1['desc'])
        s.add_kf(order[1], 8, sc['Ow'][1], k2['kps']['octave'], k2['desc'])
        for r in recs:
            p = s.add_point(r['x3D'], [(0, r['idx1']), (1, r['idx2'])], ref=0)
            s.kfs[0].mp[r['idx1']] = p.id
        g = matcher.update_connections_batch([U.flatten(s)])[0]
        assert g['pointUpdated'].all()
        assert g['normal'].tobytes() == np.ascontiguousarray(recs['normal']).tobytes()
        assert g['minDistance'].tobytes() == recs['minDistance'].tobytes() and g['maxDistance'].tobytes() == recs['maxDistance'].tobytes()


def test_chosen_rows_equal_distinctive_descriptors(orb, matcher):
    for mode in (U.PNK, U.SIN):
        sc = U.scene(21 + mode, mode, n_kf=80, n_slots=600)
        g = matcher.update_connections_batch([U.flatten(sc)])[0]
        after = U.replay(sc, g)
        pids = [p.id for p in after.pts if g['pointUpdated'][p.id] and g['descKF'][p.id] >= 0]
        who = [[t for t in after.key_sorted(after.pts[p].obs) if not after.kfs[t].bad] for p in pids]
        rows = [np.stack([after.kfs[t].desc[after.pts[p].obs[t]] for t in w]) for p, w in zip(pids, who)]
        best = matcher.ComputeDistinctiveDescriptors(rows)
        chosen = [(w[b], after.pts[p].obs[w[b]]) for p, w, b in zip(pids, who, best)]
        assert len(pids) > 200 and chosen == [(int(g['descKF'][p]), int(g['descIdx'][p])) for p in pids]


def test_search_in_neighbors_chain_equals_oracle_chain(orb, matcher):
    """The lockstep SearchInNeighbors driver on the GPU, then this call for the new keyframes, against the oracle's searches and the oracle of
    this call: the same final map (observations, descriptors, normals, distances, counters, ordered lists, parents)."""
    g = SN.globals_()
    jobs = SN.make_jobs(g, 5, 17, [3, 1, 4, 2, 5])
    oracle_jobs = copy.deepcopy(jobs)
    SN.lockstep(SN.GpuBatchBackend(matcher), jobs)
    SN.lockstep(SN.OracleBackend(), oracle_jobs)
    assert [j['map'].state() for j in jobs] == [j['map'].state() for j in oracle_jobs]
    scenes = [U.from_search_in_neighbors(j, seed=s) for s, j in enumerate(jobs)]
    got = matcher.update_connections_batch([U.flatten(sc) for sc in scenes])
    assert matcher.last_launch_count() == 1
    for s, (sc, j, gg) in enumerate(zip(scenes, oracle_jobs, got)):
        ref, fin = U.oracle(U.flatten(U.from_search_in_neighbors(j, seed=s)))
        assert U.same_outputs(gg, ref)
        assert U.final_state(U.replay(sc, gg)) == fin
        assert gg['pointUpdated'].sum() > 20 and gg['nConnected'] >= 1 and gg['parent'] == gg['orderedKF'][0]


def test_bad_arguments(orb, matcher):
    L = orb.lib()
    base = [U.flatten(U.scene(5, U.PNK, n_kf=30, n_slots=200)), U.flatten(U.scene(6, U.SIN, n_kf=30, n_slots=200))]
    matcher.update_connections_batch(base)
    assert matcher.last_launch_count() == 1

    def expect(edit, struct_edit=None, rc=orb.ORB_ERR_ARG):
        items = [{k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in m.items()} for m in base]
        edit(items)
        built = [orb.connections_struct(m) for m in items]
        arr = (orb.OrbmConnectionsItem * len(built))(*[b[0] for b in built])
        if struct_edit:
            struct_edit(arr)
        assert L.orbm_update_connections_batch(matcher._h, len(built), arr) == rc
        assert matcher.last_launch_count() == 1                           # rejected before any launch: the previous call's count stays

    def setv(key, i, v, j=0):
        def f(items): items[j][key][i] = v
        return f
    nK, nP = len(base[0]['order']), len(base[0]['pointBad'])
    good = int(np.nonzero(base[1]['pointBad'] == 0)[0][0])
    expect(setv('slotPoint', 3, nP))
    expect(setv('slotPoint', 4, -2, 1))
    expect(setv('slotOctave', 7, 8))
    expect(setv('obsKF', 2, nK, 1))
    expect(setv('obsOctave', 9, -1))
    expect(setv('obsIdx', 1, -1))
    expect(setv('connKF', 0, nK))
    expect(setv('connStart', 2, 0, 1))                                    # decreasing
    expect(setv('obsStart', 0, 1))                                        # not starting at 0
    expect(setv('order', 3, int(base[0]['order'][4])))                    # keys not distinct
    expect(lambda it: it[1]['obsKF'].__setitem__(slice(0, 2), it[1]['obsKF'][1::-1].copy()))   # not in key order
    expect(setv('pointRefKF', good, int(np.setdiff1d(np.arange(nK), base[1]['obsKF'][base[1]['obsStart'][good]:base[1]['obsStart'][good + 1]])[0]), 1))
    expect(lambda it: None, lambda a: setattr(a[0], 'mode', 2))
    expect(lambda it: None, lambda a: setattr(a[1], 'nKF', 0))
    expect(lambda it: None, lambda a: setattr(a[0], 'nPoints', -1))
    expect(lambda it: None, lambda a: setattr(a[0], 'nlevels', 0))
    for field, j in (('order', 0), ('cameraCenter', 1), ('slotDesc', 0), ('obsDesc', 1), ('pointRefKF', 0), ('counter', 1), ('nbrKF', 0),
                     ('parent', 1), ('slotStatus', 0), ('normal', 1), ('scaleFactors', 0)):
        expect(lambda it: None, lambda a, f=field, j=j: setattr(a[j], f, None))
    assert L.orbm_update_connections_batch(matcher._h, -1, None) == orb.ORB_ERR_ARG
    assert L.orbm_update_connections_batch(matcher._h, 2, None) == orb.ORB_ERR_ARG
    assert matcher.last_launch_count() == 1


def _digest(out):
    h = 14695981039346656037
    for o in out:
        for k in U.OUT_KEYS:
            for b in (np.ascontiguousarray(o[k]).tobytes() if np.ndim(o[k]) else np.int32(o[k]).tobytes()):
                h = ((h ^ b) * 1099511628211) & 0xFFFFFFFFFFFFFFFF
    return h


def test_cpp_update_connections_batch_equals_python(orb, matcher, tmp_path):
    """ORBmatcher::UpdateConnectionsBatch (include/orb_b200/orb_slam3.hpp) from a g++-built caller gives the Python binding's digest."""
    flat = [U.flatten(sc) for sc in _scenes(6, 41)]
    lines = [str(len(flat))]
    for j, m in enumerate(flat):
        lines.append(' '.join(str(int(v)) for v in (m['mode'], m['firstConnection'], len(m['order']), len(m['scaleFactors']), len(m['slotPoint']),
                                                    len(m['pointBad']))))
        for name, dt in orb.CONNECTIONS_ARRAYS:
            (tmp_path / ('item%d_%s.raw' % (j, name))).write_bytes(np.ascontiguousarray(m[name], dt).tobytes())
    (tmp_path / 'dims.txt').write_text('\n'.join(lines) + '\n')
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib = os.path.join(root, 'orb_slam3_modified_b200')
    exe = tmp_path / 'update_connections_example'
    subprocess.check_call(['g++', '-std=c++14', '-O2', '-Wall', '-I', os.path.join(root, 'include'), os.path.join(root, 'tests', 'update_connections_example.cpp'),
                           '-o', str(exe), '-L', lib, '-l:liborb_b200.so', '-Wl,-rpath,' + lib, '-lpthread'])
    out = dict(l.split() for l in subprocess.check_output([str(exe), str(tmp_path)]).decode().splitlines())
    res = matcher.update_connections_batch(flat)
    assert out['digest'] == '%016x' % _digest(res)
    assert int(out['updated']) == sum(int(o['pointUpdated'].sum()) for o in res) > 100
    assert out['launches'] == '1'
