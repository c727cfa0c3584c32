"""GPU parity of LocalBundleAdjustment on the layouts that the per-edge passes' pipelining splits unevenly: `phase_build_points`
and `phase_points_trial` give every 8-lane group several points per step and load each lane's first edge of every point ahead,
and `phase_build_poses_partial` loads a few edges per lane of a pose's 128-edge chunk ahead.  So: points with 1, exactly 8,
a non-multiple of 8 and more than 16 edges, point counts that are no multiple of the points per step, free poses with 1,
2, 3, 128, 129, 130 and 131 edges (chunk tails shorter than the items in flight), and a window where all keyframes but one
are fixed; each at every forced cluster size from 1 to 4.

Every result is held to `test_lba_gpu._check`'s bars against the oracle, and a problem that appears twice in one launch
gives byte-identical results both times."""
import functools

import numpy as np
import pytest

import lba_scenes as S
import oracle_lib as O
from test_lba_gpu import _agrees

pytestmark = pytest.mark.gpu

EDGE_COUNTS = (1, 8, 3, 9, 13, 16, 17, 25, 2, 7)


def edge_counts(n_pts, n_kf=26, seed=0):
    """Point j is seen by EDGE_COUNTS[j % 10] consecutive keyframes; keyframes 0 and 13 are fixed."""
    fixed = np.zeros(n_kf, np.uint8)
    fixed[[0, 13]] = 1
    obs = []
    for j in range(n_pts):
        c = EDGE_COUNTS[j % len(EDGE_COUNTS)]
        s = (7 * j) % (n_kf - c + 1)
        obs.append(list(range(s, s + c)))
    p = S.make(S.keyframes(n_kf), S.cameras(n_kf, seed + 6000), fixed, obs, seed=seed)
    counts = np.bincount(p['edge_point'], minlength=n_pts)
    assert set(counts.tolist()) == set(EDGE_COUNTS[:min(n_pts, len(EDGE_COUNTS))])
    return p


def one_free(n_kf=8, free=5, n_pts=300, obs_per_pt=4, seed=0):
    mask = np.ones(n_kf, np.uint8)
    mask[free] = 0
    p = S.masked(mask, n_pts, obs_per_pt, seed)
    assert (p['fixed'] == 0).sum() == 1
    return p


@functools.lru_cache(None)
def problems():
    probs = {
        'edge_counts_301': edge_counts(301, seed=1),        # odd: no multiple of the points per step of any cluster size
        'edge_counts_41': edge_counts(41, seed=2),          # fewer points than 8-lane groups, a prime count
        'chunk_tails': S.chunk_edges(counts=(1, 2, 3, 128, 129, 130, 131), seed=4),
        'one_free': one_free(seed=5),
    }
    return probs


@functools.lru_cache(None)
def ref(name):
    return O.lba_solve(problems()[name])


def _same(a, b):
    """Byte-identical results."""
    return all(a[k].tobytes() == b[k].tobytes() for k in ('poses', 'points', 'chi2', 'depth_pos')) and \
        (a['iters'], a['trials'], a['final_chi2']) == (b['iters'], b['trials'], b['final_chi2'])


def test_edge_count_layouts():
    p = problems()['edge_counts_301']
    counts = np.bincount(p['edge_point'])
    assert (counts == 1).any() and (counts == 8).any() and (counts % 8 != 0).any() and (counts > 16).any()
    assert len(counts) % 2 == 1
    pose_edges = np.bincount(problems()['chunk_tails']['edge_pose'])
    assert {1, 2, 3, 128, 129, 130, 131} <= set(pose_edges[problems()['chunk_tails']['fixed'] == 0].tolist())


@pytest.fixture(scope='module')
def opt():
    import orb_slam3_modified_b200 as m
    m.lib()
    return m.Optimizer(max_poses=32, max_points=2000, max_edges=8000, max_batch=2 * len(problems()))


@pytest.mark.parametrize('cluster', [1, 2, 3, 4])
def test_pipelined_passes_at_forced_cluster_sizes(opt, cluster):
    names = list(problems())
    batch = names + names[::-1]                            # every problem twice in one launch
    opt.set_cluster_size(cluster)
    try:
        outs = opt.LocalBundleAdjustmentBatch([problems()[n] for n in batch])
        assert opt.last_cluster_size() == cluster
    finally:
        opt.set_cluster_size(0)
    for n, out in zip(batch, outs):
        _agrees(problems()[n], out, ref(n))
    k = len(names)
    for i in range(k):
        assert _same(outs[i], outs[2 * k - 1 - i]), names[i]
