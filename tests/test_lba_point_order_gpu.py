"""LocalBundleAdjustment's internal point order.  The solver sorts the points by the ascending list of their observing free
keyframes (the first four, points seen only by fixed keyframes last), ties by the caller's index, and works in that order; the
caller's order comes back at the boundary.  These tests give it problems whose internal order differs from the caller's -- points
seen only by fixed keyframes, points seen by one free keyframe, runs of identical observer sets, a problem at the handle's point
capacity, more points than one shared-memory tile of the sort -- and the same problem with its points and edges permuted by the
caller.  Every result is held to the oracle in the caller's order with `test_lba_gpu._agrees`' bars (same iterations and trials,
residuals within 1e-4 px), and two runs of one build are byte-identical."""
import numpy as np
import pytest

import lba_scenes as S
import oracle_lib as O
from orb_slam3_modified_b200 import synth
from test_lba_gpu import _agrees

pytestmark = pytest.mark.gpu
SORT_TILE = 2048       # keys per shared-memory tile of the structure kernel's point sort (csrc/lba.cu)


def internal_order(p):
    """The solver's point order, restated: the caller's point indices in internal order."""
    fixed = np.asarray(p['fixed'])
    hidx = np.where(fixed == 0, np.cumsum(fixed == 0) - 1, -1)
    obs = [[] for _ in range(len(p['points']))]
    for j, k in zip(p['edge_point'], p['edge_pose']):
        if hidx[k] >= 0:
            obs[j].append(int(hidx[k]))
    none = 1 << 20
    keys = [tuple((sorted(o) + [none] * 4)[:4]) + (j,) for j, o in enumerate(obs)]
    return np.array(sorted(range(len(keys)), key=lambda j: keys[j]))


def permuted(p, pt_perm, e_perm):
    """p with point i of the result = point pt_perm[i] of p, and edge i = edge e_perm[i] of p."""
    new_of_old = np.empty(len(pt_perm), np.int64)
    new_of_old[pt_perm] = np.arange(len(pt_perm))
    q = {k: p[k] for k in ('poses', 'fixed', 'cam', 'huber_delta')}
    q['points'] = np.ascontiguousarray(p['points'][pt_perm])
    q['edge_point'] = new_of_old[p['edge_point'][e_perm]].astype(np.int32)
    for k in ('edge_pose', 'obs', 'inv_sigma2'):
        q[k] = np.ascontiguousarray(p[k][e_perm])
    return q


def _same(a, b):
    return all(a[k].tobytes() == b[k].tobytes() for k in ('poses', 'points', 'chi2', 'depth_pos')) and \
        (a['iters'], a['trials'], a['final_chi2']) == (b['iters'], b['trials'], b['final_chi2'])


def _opt(p, max_batch=1):
    import orb_slam3_modified_b200 as m
    m.lib()
    return m.Optimizer(max_poses=len(p['poses']), max_points=len(p['points']), max_edges=len(p['edge_point']), max_batch=max_batch)


@pytest.mark.parametrize('scene', ['interleaved', 'observer_sets', 'wide'])
def test_caller_permutations(scene):
    """The same problem in four caller orders, one batch: each agrees with the oracle in its own caller order, and the results map
    onto each other through the permutation (point i of an output is input point i)."""
    if scene == 'interleaved':
        base = S.interleaved(n_kf=10, n_pts=500, obs_per_pt=4, seed=21)
    elif scene == 'observer_sets':
        base = S.observer_sets(n_kf=12, n_single=60, n_fixed_only=40, n_window=400, hub=11, seed=22)
    else:
        base = synth.lba_problem(n_kf=12, n_pts=SORT_TILE + 700, obs_per_pt=5, seed=23)
    nL, nE = len(base['points']), len(base['edge_point'])
    rng = np.random.default_rng(24)
    perms = [(np.arange(nL), np.arange(nE)), (np.arange(nL)[::-1].copy(), np.arange(nE)),
             (rng.permutation(nL), np.arange(nE)), (rng.permutation(nL), rng.permutation(nE))]
    probs = [permuted(base, a, b) for a, b in perms]
    for q in probs[1:]:
        assert not np.array_equal(internal_order(q), np.arange(nL))
    outs = _opt(base, len(probs)).LocalBundleAdjustmentBatch(probs)
    b0 = outs[0]
    for q, out, (pp, ep) in zip(probs, outs, perms):
        _agrees(q, out, O.lba_solve(q))
        assert (out['iters'], out['trials']) == (b0['iters'], b0['trials'])
        assert np.allclose(out['points'], b0['points'][pp], rtol=0, atol=1e-8)
        assert np.allclose(out['poses'], b0['poses'], rtol=0, atol=1e-9)
        assert np.allclose(out['chi2'], b0['chi2'][ep], rtol=1e-6, atol=1e-7)
        assert np.array_equal(out['depth_pos'], b0['depth_pos'][ep])


def test_observer_classes_at_point_capacity():
    """Points seen only by fixed keyframes, by one free keyframe, and runs of identical observer sets, shuffled so that the
    internal order differs from the caller's, on a handle whose point capacity is exactly the problem's; two runs of one
    build are byte-identical."""
    base = S.observer_sets(n_kf=12, n_single=60, n_fixed_only=40, n_window=400, hub=11, seed=31)
    nL = len(base['points'])
    p = permuted(base, np.random.default_rng(32).permutation(nL), np.random.default_rng(33).permutation(len(base['edge_point'])))
    fixed = np.asarray(p['fixed'])
    free_obs = [set() for _ in range(nL)]
    for j, k in zip(p['edge_point'], p['edge_pose']):
        if not fixed[k]:
            free_obs[j].add(int(k))
    sets = [frozenset(s) for s in free_obs]
    assert sum(len(s) == 0 for s in sets) >= 40 and sum(len(s) == 1 for s in sets) >= 30
    assert max(sets.count(s) for s in set(sets) if len(s) >= 2) >= 2             # ties between points with several observers
    order = internal_order(p)
    assert not np.array_equal(order, np.arange(nL))
    assert all(len(sets[j]) == 0 for j in order[-sum(len(s) == 0 for s in sets):])   # fixed-only points sort last
    opt = _opt(p)
    a = opt.LocalBundleAdjustment(p)
    _agrees(p, a, O.lba_solve(p))
    assert _same(a, opt.LocalBundleAdjustment(p))
