"""GPU tests of the two whole-function map walks on the map_walk_scenes.py cases, byte for byte against the CPU oracle:
lba_local_bundle_adjustment_batch (Optimizer::LocalBundleAdjustment) and local_inertial_ba_map_batch (Optimizer::LocalInertialBA).
- The walk: status, counts / nLists, the lists (localKF / optKF, fixedKF, localPoint, ieLinked) and the edge mask of obsFlag equal the
  oracle's, and every entry past the lists holds the walk's fill value.
- The solve: the solver's doubles equal lba_solve_batch / local_inertial_ba_batch run on the oracle walk's built problem (LBA: the same
  problems in the same slot order, so the same cluster size); the LBA poses and points are matched through the oracle's vertex order,
  which is where the vertex sort shows.
- The finish: every write-back output equals the oracle finishing the GPU's own doubles, and every row past the lists is zero.
Every output starts as a sentinel byte, so an unwritten byte shows.  Each case runs alone, all cases run in one call in two orders, per-map
calls equal the batch, a repeat is byte-identical, LIBA's small maps run after a large one on the same thread, LBA handles fitting a case
exactly run it and one size less refuse it, and an mnId of 2^64 - 1 is refused before anything is staged."""
import numpy as np
import pytest

import local_ba_lib as LB
import local_inertial_ba_map_lib as LM
import map_walk_scenes as S
import orb_slam3_modified_b200 as orb

pytestmark = pytest.mark.gpu

SENT = 0xA5
LBA = S.lba_cases()
LIBA = S.liba_cases()
LBA_CAPS = (1024, 8192, 65536)
LBA_FINISH = ('kfPose7', 'kfCenter', 'pointPos', 'pointBad', 'pointRefKF', 'normal', 'minDistance', 'maxDistance')
LIBA_FINISH = ('kfPose7', 'kfCenter', 'kfVelocity', 'kfBias6', 'pointPos', 'pointBad', 'pointRefKF', 'normal', 'minDistance', 'maxDistance')
_flat = {}


def lba_map(name):
    if ('lba', name) not in _flat:
        _flat['lba', name] = LB.flatten(*LBA[name][0]())
    return _flat['lba', name]


def liba_map(name):
    if ('liba', name) not in _flat:
        _flat['liba', name] = LM.flatten(*LIBA[name][0]())
    return _flat['liba', name]


def _sentinel(packs):
    for _, out, _ in packs:
        for a in out.values():
            a.view(np.uint8)[...] = SENT


def _edge_order(m, localPoint, obsFlag):
    return [o for p in localPoint for o in range(m['obsStart'][p], m['obsStart'][p + 1]) if obsFlag[o] != orb.LBA_OBS_NO_EDGE]


def _tail(a, n, v):
    assert (a[n:] == v).all()


# ---- LBA ----
def lba_call(opt, maps):
    """lba_local_bundle_adjustment_batch with sentinel-filled outputs: (return code, raw output dicts)."""
    packs = [orb.local_ba_struct(m, debug=True) for m in maps]
    _sentinel(packs)
    arr = (orb.LbaLocalMap * len(maps))(*[p[0] for p in packs])
    rc = orb.lib().lba_local_bundle_adjustment_batch(opt._h, len(maps), arr)
    return rc, [p[1] for p in packs]


def lba_check(maps, outs, caps=LBA_CAPS):
    probs, where = [], []
    for j, (m, o) in enumerate(zip(maps, outs)):
        g = orb.local_ba_result({k: v.copy() for k, v in o.items()})
        ref, built = LB.oracle(m)
        nK, nP = len(m['kfFlags']), len(m['pointFlags'])
        # the walk
        assert g['status'] == ref['status'], j
        assert o['counts'].tobytes() == ref['counts'].tobytes() and o['nLists'].tobytes() == ref['nLists'].tobytes(), j
        for k in ('localKF', 'fixedKF', 'localPoint'):
            assert np.array_equal(g[k], ref[k]), (j, k)
            _tail(o[k], len(g[k]), -1)
        assert np.array_equal(o['obsFlag'] != orb.LBA_OBS_NO_EDGE, ref['obsFlag'] != orb.LBA_OBS_NO_EDGE), j
        nLoc, nPt = len(g['localKF']), len(g['localPoint'])
        for k in LBA_FINISH + ('optPose',):
            _tail(o[k], nLoc if k in ('kfPose7', 'kfCenter', 'optPose') else nPt, -1 if k == 'pointRefKF' else 0)
        _tail(o['optPoint'], nPt, 0)
        if g['status'] != orb.LBA_LOCAL_RAN:
            assert g['lmStats'][0] == -1 and not g['lmStats'][1:].any() and not o['obsFlag'].any(), j
            for k in LBA_FINISH + ('optPose', 'optPoint', 'edgeChi2', 'edgeDepthPositive'):
                assert (o[k] == (-1 if k == 'pointRefKF' else 0)).all(), (j, k)
            continue
        # the finish: the oracle finishing the GPU's own doubles
        fin, _ = LB.oracle(m, given={k: o[k].copy() for k in ('optPose', 'optPoint', 'edgeChi2', 'edgeDepthPositive')})
        assert o['obsFlag'].tobytes() == fin['obsFlag'].tobytes(), j
        for k in LBA_FINISH:
            assert g[k].tobytes() == fin[k].tobytes(), (j, k)
        order = _edge_order(m, g['localPoint'], o['obsFlag'])
        assert len(order) == g['num_edges']
        noedge = np.ones(len(o['obsFlag']), bool)
        noedge[order] = False
        assert not o['edgeChi2'][noedge].any() and not o['edgeDepthPositive'][noedge].any(), j
        if g['lmStats'][0] >= 0:
            probs.append(built); where.append((j, g, order))
    # the solver's doubles = lba_solve_batch on the oracle walk's problems, in the same slot order
    if probs:
        solver = orb.Optimizer(*caps, max_batch=len(probs))
        packs = [orb.Optimizer._pack(p, 10, 100.0 if maps[j]['inertial'] else 0.0, None) for p, (j, _, _) in zip(probs, where)]
        P = (orb._LbaProblem * len(packs))(*[k[1] for k in packs])
        R = (orb._LbaResult * len(packs))(*[k[3] for k in packs])
        assert orb.lib().lba_solve_batch(solver._h, len(packs), P, R) == orb.ORB_OK
        for i, ((j, g, order), built) in enumerate(zip(where, probs)):
            w = orb.Optimizer._finish(packs[i][2], R[i])
            assert w['iters'] == int(g['lmStats'][0]) and w['trials'] == int(g['lmStats'][1]), j
            vk = {k: v for v, k in enumerate(built['vert_kf'])}
            vp = {p: v for v, p in enumerate(built['vert_point'])}
            assert w['poses'][[vk[k] for k in g['localKF']]].tobytes() == g['optPose'].tobytes(), j
            assert w['points'][[vp[p] for p in g['localPoint']]].tobytes() == g['optPoint'].tobytes(), j
            assert w['chi2'].tobytes() == g['edgeChi2'][order].tobytes() and w['depth_pos'].tobytes() == g['edgeDepthPositive'][order].tobytes(), j


_handles = {}


def lba_opt(n):
    if n not in _handles:
        _handles[n] = orb.Optimizer(*LBA_CAPS, max_batch=n)
    return _handles[n]


def _by_size(names, flat):
    return sorted(names, key=lambda n: -int(flat(n)['obsStart'][-1]))


@pytest.mark.parametrize('name', sorted(LBA))
def test_lba_case_alone(name):
    m = lba_map(name)
    rc, outs = lba_call(lba_opt(1), [m])
    assert rc == orb.ORB_OK, orb.lib().orb_last_error()
    lba_check([m], outs)


def test_lba_all_cases_in_one_call_two_orders():
    names = _by_size(LBA, lba_map)
    assert names[0] == 'qs_qo_40k'
    for order in (names, names[::-1]):
        maps = [lba_map(n) for n in order]
        rc, outs = lba_call(lba_opt(len(maps)), maps)
        assert rc == orb.ORB_OK
        assert lba_opt(len(maps)).local_last_launches() == 5
        lba_check(maps, outs)


def test_lba_per_map_calls_equal_the_pinned_batch_and_repeat():
    names = _by_size(LBA, lba_map)
    maps = [lba_map(n) for n in names]
    opt = orb.Optimizer(*LBA_CAPS, max_batch=len(maps))
    opt.set_cluster_size(4)                         # the cluster size orders the solver's reductions: the same for both
    rc, batch = lba_call(opt, maps)
    assert rc == orb.ORB_OK
    for n, m, b in zip(names, maps, batch):
        rc, one = lba_call(opt, [m])
        assert rc == orb.ORB_OK
        for k in b:
            assert one[0][k].tobytes() == b[k].tobytes(), (n, k)
    rc, again = lba_call(opt, maps)
    assert rc == orb.ORB_OK
    for n, a, b in zip(names, again, batch):
        for k in b:
            assert a[k].tobytes() == b[k].tobytes(), (n, k)


@pytest.mark.parametrize('name', ['np_65', 'nl_4097', 'fixed_500'])
def test_lba_capacity_exact_and_one_less(name):
    m, small = lba_map(name), lba_map('np_1')
    _, built = LB.oracle(m)
    exact = (len(built['poses']), len(built['points']), len(built['edge_point']))
    opt = orb.Optimizer(*exact, max_batch=2)
    rc, outs = lba_call(opt, [small, m])
    assert rc == orb.ORB_OK, orb.lib().orb_last_error()
    lba_check([small, m], outs, exact)
    for i in range(3):
        less = list(exact)
        less[i] -= 1
        h = orb.Optimizer(*less, max_batch=2)
        rc, _ = lba_call(h, [small, m])
        assert rc == orb.ORB_ERR_CAPACITY and 'map 1' in orb.lib().orb_last_error().decode(), i
        rc, outs = lba_call(h, [small])              # the handle serves a map that fits right after
        assert rc == orb.ORB_OK
        lba_check([small], outs, less)
        rc, outs = lba_call(opt, [m])                # and the exact handle the map
        assert rc == orb.ORB_OK
        lba_check([m], outs, exact)


@pytest.mark.parametrize('field', ['mnId', 'pointId'])
def test_lba_refuses_mnid_2_64_minus_1(field):
    """An mnId of 2^64 - 1 (the vertex sort's padding key) is refused before anything is staged: every output keeps its sentinel and
    the handle keeps the previous call's launch count."""
    good = lba_map('np_17')
    opt = lba_opt(2)
    assert lba_call(opt, [good])[0] == orb.ORB_OK and opt.local_last_launches() == 5
    bad = dict(good)
    bad[field] = np.array(good[field])
    bad[field][len(bad[field]) // 2] = np.uint64(2 ** 64 - 1)
    rc, outs = lba_call(opt, [good, bad])
    assert rc == orb.ORB_ERR_ARG
    msg = orb.lib().orb_last_error().decode()
    assert 'map 1' in msg and '2^64 - 1' in msg, msg
    for o in outs:
        for k, a in o.items():
            assert (a.view(np.uint8) == SENT).all(), k
    assert opt.local_last_launches() == 5


# ---- LIBA ----
def liba_call(maps):
    packs = [orb.liba_map_struct(m, debug=True) for m in maps]
    _sentinel(packs)
    arr = (orb.LocalInertialBAMap * len(maps))(*[p[0] for p in packs])
    rc = orb.lib().local_inertial_ba_map_batch(len(maps), arr, 0)
    return rc, [p[1] for p in packs]


def liba_check(maps, outs):
    for j, (m, o) in enumerate(zip(maps, outs)):
        r = orb.liba_map_result({k: v.copy() for k, v in o.items()})
        ref, pr = LM.oracle(m)
        # the walk
        assert r['status'] == ref['status'] and o['nLists'].tobytes() == ref['nLists'].tobytes(), j
        for k in ('optKF', 'fixedKF', 'localPoint', 'ieLinked'):
            assert r[k].tobytes() == ref[k].tobytes(), (j, k)
            _tail(o[k], len(r[k]), 0 if k == 'ieLinked' else -1)
        assert np.array_equal(o['obsFlag'] != orb.LBA_OBS_NO_EDGE, ref['obsFlag'] != orb.LBA_OBS_NO_EDGE), j
        N, nFix, nPt = r['num_OptKF'], r['num_fixedKF'], r['num_MPs']
        for k in LIBA_FINISH:
            _tail(o[k], N if k.startswith('kf') else nPt, -1 if k == 'pointRefKF' else 0)
        _tail(o['optState21'], N + nFix, 0); _tail(o['optTcw12'], N + nFix, 0); _tail(o['optPoint'], nPt, 0)
        # the solve: local_inertial_ba_batch on the oracle walk's problem
        w = orb.LocalInertialBA([pr])[0]
        order = _edge_order(m, r['localPoint'], o['obsFlag'])
        assert r['edgeChi2'][order].tobytes() == w['chi2'].tobytes(), j
        noedge = np.ones(len(o['obsFlag']), bool)
        noedge[order] = False
        assert not o['edgeChi2'][noedge].any(), j
        assert np.array_equal(r['stats8'][:6], [w['err'], w['err_end'], w['failed'], w['lam'], w['trials'], w['iters']], equal_nan=True), j
        assert not w['failed'], j
        assert r['optState21'].tobytes() == w['state'].tobytes() and r['optTcw12'].tobytes() == w['tcw'].tobytes(), j
        assert r['optPoint'].tobytes() == w['points'].tobytes(), j
        # the finish: the oracle finishing the GPU's own doubles
        g, _ = LM.oracle(m, given=LM.padded(r, m))
        assert g['status'] == r['status'] and o['obsFlag'].tobytes() == g['obsFlag'].tobytes(), j
        for k in LIBA_FINISH:
            assert r[k].tobytes() == g[k].tobytes(), (j, k)


def _raw_equal(a, b, what):
    for k in b:
        x, y = a[k].copy(), b[k].copy()
        if k == 'stats8':
            x[6] = y[6] = 0                          # the solver's %globaltimer span
        assert x.tobytes() == y.tobytes(), (what, k)


@pytest.mark.parametrize('name', sorted(LIBA))
def test_liba_case_alone(name):
    m = liba_map(name)
    rc, outs = liba_call([m])
    assert rc == orb.ORB_OK, orb.lib().orb_last_error()
    assert orb.Optimizer.local_inertial_ba_map_last_launches() == 3
    liba_check([m], outs)


def test_liba_all_cases_in_one_call_two_orders_equal_per_map_calls_and_repeat():
    names = _by_size(LIBA, liba_map)
    maps = [liba_map(n) for n in names]
    alone = {}
    for n, m in zip(names, maps):
        rc, outs = liba_call([m])
        assert rc == orb.ORB_OK
        alone[n] = outs[0]
    for order in (names, names[::-1]):
        rc, outs = liba_call([liba_map(n) for n in order])
        assert rc == orb.ORB_OK
        liba_check([liba_map(n) for n in order], outs)
        for n, o in zip(order, outs):
            _raw_equal(o, alone[n], n)
    rc, again = liba_call(maps)
    assert rc == orb.ORB_OK
    for n, o in zip(names, again):
        _raw_equal(o, alone[n], n)


def test_liba_small_maps_after_a_large_one():
    """The thread's staging holds the large map's leftovers when the small ones run."""
    names = _by_size(LIBA, liba_map)
    small = names[-4:]
    first = {n: liba_call([liba_map(n)])[1][0] for n in small}
    assert liba_call([liba_map(names[0])])[0] == orb.ORB_OK
    for n in small:
        rc, outs = liba_call([liba_map(n)])
        assert rc == orb.ORB_OK
        _raw_equal(outs[0], first[n], n)
    rc, outs = liba_call([liba_map(n) for n in small])
    assert rc == orb.ORB_OK
    liba_check([liba_map(n) for n in small], outs)
