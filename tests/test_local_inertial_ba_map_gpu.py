"""GPU tests of local_inertial_ba_map_batch (Optimizer::LocalInertialBA as a whole) at 1 / 7 / 24 maps mixing normal, bLarge, bRecInit,
popped-predecessor, capped and FAIL maps: the walk's lists against the CPU oracle's, the solver's doubles byte-equal to
local_inertial_ba_batch on the oracle's problem, every finish field byte-equal to the oracle finishing the GPU's doubles, the whole chain
against the CPU oracle chain, batch against per-map calls, the launch count, and the C++ shim's digest against the Python binding's."""
import copy
import os
import subprocess

import numpy as np
import pytest

import local_inertial_ba_map_lib as LM
import oracle_lib as O
import orb_slam3_modified_b200 as orb

pytestmark = pytest.mark.gpu

PLANTED = LM.planted()
NAMES = sorted(PLANTED)
LISTS = ('nLists', 'optKF', 'fixedKF', 'localPoint', 'ieLinked')
FINISH = [n for n, _, _, _ in orb.LIBA_MAP_OUTPUTS if n != 'stats8']


def _maps(count):
    out = []
    for i in range(count):
        item = PLANTED[NAMES[i % len(NAMES)]] if i < 2 * len(NAMES) else LM.seeded(i)
        out.append(LM.flatten(*item))
    return out


def _edge_order(m, r):
    return [o for p in r['localPoint'] for o in range(m['obsStart'][p], m['obsStart'][p + 1]) if r['obsFlag'][o] != orb.LBA_OBS_NO_EDGE]


def _same(a, b, fields):
    for n in fields:
        assert np.asarray(a[n]).tobytes() == np.asarray(b[n]).tobytes(), n


@pytest.mark.parametrize('count', [1, 7, 24])
def test_against_oracle(count):
    maps = _maps(count)
    res = orb.Optimizer.local_inertial_ba_map_batch(maps, debug=True)
    assert orb.Optimizer.local_inertial_ba_map_last_launches() == 3
    for j, (m, r) in enumerate(zip(maps, res)):
        o, pr = LM.oracle(m)
        # the walk
        assert r['status'] == o['status'], j
        _same(r, o, LISTS)
        assert np.array_equal(r['obsFlag'] != orb.LBA_OBS_NO_EDGE, o['obsFlag'] != orb.LBA_OBS_NO_EDGE), j
        # the solve: byte-equal to local_inertial_ba_batch on the oracle walk's problem (the solver sums in a fixed order)
        w = orb.LocalInertialBA([pr])[0]
        order = _edge_order(m, r)
        assert r['edgeChi2'][order].tobytes() == w['chi2'].tobytes(), j
        assert np.array_equal(r['stats8'][:6], [w['err'], w['err_end'], w['failed'], w['lam'], w['trials'], w['iters']], equal_nan=True), j
        if not w['failed']:
            assert r['optState21'].tobytes() == w['state'].tobytes() and r['optTcw12'].tobytes() == w['tcw'].tobytes(), j
            assert r['optPoint'].tobytes() == w['points'].tobytes(), j
        # the finish: byte-equal to the oracle finishing the GPU's doubles
        g, _ = LM.oracle(m, given=LM.padded(r, m))
        assert g['status'] == r['status']
        _same(r, g, FINISH)
        # the whole chain against the CPU oracle chain, within the LocalInertialBA bars
        if r['status'] == orb.LIBA_LOCAL_RAN:
            c2 = r['edgeChi2'][order]
            margin = not (np.abs(c2 - 5.991) < 1e-3).any() and not (np.abs(c2 - 1.5 * 5.991) < 1e-3).any()
            if margin:
                assert np.array_equal(r['obsFlag'], o['obsFlag']), j
            assert np.abs(r['optState21'] - o['optState21']).max() < 1e-8, (j, np.abs(r['optState21'] - o['optState21']).max())
            res_g = O.local_inertial_ba_residuals(pr, r['optTcw12'], r['optPoint'])
            res_o = O.local_inertial_ba_residuals(pr, o['optTcw12'], o['optPoint'])
            sane = np.abs(res_o).max(1) < 1e3
            if sane.any():
                assert np.abs(res_g - res_o)[sane].max() < 1e-4, j


def test_batch_equals_single_calls_and_repeats():
    maps = _maps(9)
    both = orb.Optimizer.local_inertial_ba_map_batch(maps + [maps[0]], debug=True)
    keys = [n for n, _, _, _ in orb.LIBA_MAP_OUTPUTS + orb.LIBA_MAP_DEBUG if n != 'stats8'] + ['status']
    for j, m in enumerate(maps):
        one = orb.Optimizer.local_inertial_ba_map_batch([m], debug=True)[0]
        _same(both[j], one, keys)
        assert np.array_equal(both[j]['stats8'][:6], one['stats8'][:6], equal_nan=True)   # [6] is the CTA's time
    _same(both[0], both[-1], keys)


def test_planted_branches_on_the_device():
    names = ['popped_predecessor', 'cap_200', 'fail', 'large', 'no_preint', 'cascade']
    maps = [LM.flatten(*PLANTED[n]) for n in names]
    res = dict(zip(names, orb.Optimizer.local_inertial_ba_map_batch(maps)))
    assert res['fail']['status'] == orb.LIBA_LOCAL_FAILED and not res['fail']['kfPose7'].any()
    assert len(res['cap_200']['fixedKF']) == 200
    assert res['cascade']['pointBad'].any()
    assert not res['no_preint']['ieLinked'].all()
    for n in names:
        if n != 'fail':
            assert res[n]['status'] == orb.LIBA_LOCAL_RAN, n


def _digest(res):
    """FNV-1a over what tests/local_inertial_ba_map_example.cpp hashes, in its order."""
    h = 14695981039346656037
    for r in res:
        parts = [np.int32(r['status']), np.asarray(r['nLists'], np.int32), r['optKF'], r['fixedKF'], r['localPoint'], r['ieLinked'], r['obsFlag'],
                 r['kfPose7'], r['kfCenter'], r['kfVelocity'], r['kfBias6'], r['pointPos'], r['pointBad'], r['pointRefKF'], r['normal'],
                 r['minDistance'], r['maxDistance']]
        for b in b''.join(np.ascontiguousarray(x).tobytes() for x in parts):
            h = ((h ^ b) * 1099511628211) & 0xFFFFFFFFFFFFFFFF
    return h


def test_cpp_local_inertial_ba_batch_equals_python(tmp_path):
    """Optimizer::LocalInertialBABatch (include/orb_b200/orb_slam3.hpp) from a g++-built caller gives the Python binding's digest."""
    flat = _maps(7)
    lines = ['%d' % len(flat)]
    for j, m in enumerate(flat):
        lines.append('%d %d %d %d %d %d' % (len(m['kfFlags']), len(m['pointFlags']), len(m['scaleFactors']), m['keyFramesInMap'], m['bLarge'], m['bRecInit']))
        for name, dt in orb.LIBA_MAP_ARRAYS:
            (tmp_path / ('map%d_%s.raw' % (j, name))).write_bytes(np.ascontiguousarray(m[name], dt).tobytes())
    (tmp_path / 'dims.txt').write_text('\n'.join(lines) + '\n')
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib = os.path.join(root, 'orb_slam3_modified_b200')
    exe = tmp_path / 'local_inertial_ba_map_example'
    subprocess.check_call(['g++', '-std=c++14', '-O2', '-Wall', '-I', os.path.join(root, 'include'),
                           os.path.join(root, 'tests', 'local_inertial_ba_map_example.cpp'), '-o', str(exe), '-L', lib, '-l:liborb_b200.so',
                           '-Wl,-rpath,' + lib, '-lpthread'])
    out = dict(l.split() for l in subprocess.check_output([str(exe), str(tmp_path)]).decode().splitlines())
    res = orb.Optimizer.local_inertial_ba_map_batch(copy.deepcopy(flat))
    assert out['digest'] == '%016x' % _digest(res)
    assert int(out['erased']) == sum(int((r['obsFlag'] == orb.LBA_OBS_ERASED).sum()) for r in res) > 5
    assert out['launches'] == '3'
