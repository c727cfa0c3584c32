"""GPU parity tests of LocalBundleAdjustment: reprojection residuals within 1e-4 px of the oracle (north_star bar),
identical LM control flow (iterations, trials) and identical outlier classification."""
import numpy as np
import pytest

import oracle_lib as O
from orb_slam3_modified_b200 import synth

pytestmark = pytest.mark.gpu
TOL_PX = 1e-4   # BASELINE.json north_star: "LBA reprojection residuals within 1e-4 px"


@pytest.fixture(scope='module')
def opt():
    import orb_slam3_modified_b200 as m
    m.lib()
    return m.Optimizer(max_poses=64, max_points=8192, max_edges=65536)


def _check(opt, p, **kw):
    ref = O.lba_solve(p, **kw)
    out = opt.LocalBundleAdjustment(p, **kw)
    return _agrees(p, out, ref)


def _agrees(p, out, ref):
    """The GPU result `out` of problem p against the oracle's `ref` (the assertions of _check, for batched calls)."""
    assert out['iters'] == ref['iters'], (out['iters'], ref['iters'])
    assert out['trials'] == int(ref['stats'][3])
    r_ref = O.lba_residuals(p, ref['poses'], ref['points'])
    r_gpu = O.lba_residuals(p, out['poses'], out['points'])
    assert np.abs(r_ref - r_gpu).max() < TOL_PX, float(np.abs(r_ref - r_gpu).max())
    assert np.allclose(out['poses'], ref['poses'], atol=1e-9) and np.allclose(out['points'], ref['points'], atol=1e-8)
    assert np.allclose(out['chi2'], ref['chi2'], rtol=1e-6, atol=1e-7)
    near = np.abs(ref['chi2'] - 5.991) < 1e-6
    assert np.array_equal((out['chi2'] > 5.991)[~near], (ref['chi2'] > 5.991)[~near])
    assert np.array_equal(out['depth_pos'], ref['depth_pos'])
    assert abs(out['final_chi2'] - ref['stats'][1]) <= 1e-9 * max(1.0, ref['stats'][1])
    return out


def test_config4_20kf_5000pts_40k_edges(opt):
    """BASELINE config 4."""
    p = synth.lba_problem(n_kf=20, n_pts=5000, obs_per_pt=8, seed=0)
    assert len(p['edge_point']) == 40000
    out = _check(opt, p)
    assert out['iters'] >= 5 and out['launches'] > 0


@pytest.mark.parametrize('seed,n_kf,n_pts,obs,n_fixed', [(1, 8, 600, 5, 1), (2, 6, 300, 6, 2), (5, 30, 2000, 10, 3), (7, 3, 50, 3, 1), (9, 12, 800, 12, 11)])
def test_other_sizes(opt, seed, n_kf, n_pts, obs, n_fixed):
    _check(opt, synth.lba_problem(n_kf=n_kf, n_pts=n_pts, obs_per_pt=obs, seed=seed, n_fixed=n_fixed))


def test_control_flow_variants(opt):
    p = synth.lba_problem(n_kf=8, n_pts=500, obs_per_pt=5, seed=11)
    _check(opt, p, user_lambda_init=100.0)          # inertial map initial lambda
    _check(opt, p, iterations=1)
    _check(opt, p, iterations=0)
    out = opt.LocalBundleAdjustment(p, stop_flag=np.ones(1, np.uint8))
    assert out['iters'] == 0 and np.allclose(out['points'], p['points'])
    # badly perturbed start: forces rejected LM trials (lambda escalation + pop)
    q = synth.lba_problem(n_kf=8, n_pts=500, obs_per_pt=5, seed=12, pose_noise=(0.3, 8.0), point_noise=0.5)
    _check(opt, q)


def test_all_poses_fixed_and_bad_graphs(opt):
    import orb_slam3_modified_b200 as m
    p = synth.lba_problem(n_kf=4, n_pts=80, obs_per_pt=4, seed=13, n_fixed=4)   # only landmarks move
    _check(opt, p)
    bad = dict(p)
    bad['edge_pose'] = p['edge_pose'].copy()
    bad['edge_pose'][0] = 99
    with pytest.raises(m.OrbError):
        opt.LocalBundleAdjustment(bad)


def test_batch_of_problems_one_launch():
    """Several local maps (different sizes) solved by one persistent-kernel launch == individual solves."""
    import orb_slam3_modified_b200 as m
    optb = m.Optimizer(max_poses=32, max_points=6000, max_edges=48000, max_batch=24)
    probs = [synth.lba_problem(n_kf=6 + b % 5, n_pts=200 + 37 * b, obs_per_pt=4 + b % 3, seed=20 + b) for b in range(20)]
    probs[3] = synth.lba_problem(n_kf=20, n_pts=5000, obs_per_pt=8, seed=0)
    outs = optb.LocalBundleAdjustmentBatch(probs)
    assert 1 <= optb.last_cluster_size() <= 8
    for p, out in zip(probs, outs):
        ref = O.lba_solve(p)
        assert out['iters'] == ref['iters'] and out['trials'] == int(ref['stats'][3])
        r_ref = O.lba_residuals(p, ref['poses'], ref['points'])
        r_gpu = O.lba_residuals(p, out['poses'], out['points'])
        assert np.abs(r_ref - r_gpu).max() < TOL_PX
    # resident re-run: upload once, run twice, same answer (state restarts from the uploaded estimates)
    # Different problems than the ones slots 0..3 still hold from the call above, and no host synchronisation between run and
    # download: a download that does not wait for the run (it is on another stream) would return stale or half-written results.
    optb.upload(probs[4:8])
    optb.run_device()
    a = optb.download()
    optb.run_device()
    b = optb.download()
    for x, y, first in zip(a, b, outs[4:8]):
        assert np.array_equal(x['poses'], y['poses']) and np.array_equal(x['points'], y['points']) and np.array_equal(x['chi2'], y['chi2'])
        assert np.array_equal(x['poses'], first['poses']) and np.array_equal(x['chi2'], first['chi2']) and x['trials'] == first['trials']
    import torch
    side = torch.cuda.Stream()                         # run on a caller stream, upload + download on the handle's own
    optb.upload(probs[8:12])
    optb.run_device(side.cuda_stream)
    c = optb.download()
    for x, first in zip(c, outs[8:12]):
        assert np.array_equal(x['poses'], first['poses']) and np.array_equal(x['chi2'], first['chi2'])
    optb.run_device(side.cuda_stream)
    optb.upload(probs[12:16])                          # must not overwrite the arena under the running kernel
    optb.run_device(side.cuda_stream)
    d = optb.download()
    for x, first in zip(d, outs[12:16]):
        assert np.array_equal(x['poses'], first['poses']) and np.array_equal(x['chi2'], first['chi2'])


def test_large_window_matrix_in_global_memory():
    """60 free keyframes: the 360x360 reduced camera system does not fit in shared memory -> global/L2 path."""
    import orb_slam3_modified_b200 as m
    optl = m.Optimizer(max_poses=64, max_points=3000, max_edges=40000)
    p = synth.lba_problem(n_kf=61, n_pts=2500, obs_per_pt=12, seed=31)
    ref = O.lba_solve(p)
    out = optl.LocalBundleAdjustment(p)
    assert out['iters'] == ref['iters'] and out['trials'] == int(ref['stats'][3])
    assert np.abs(O.lba_residuals(p, ref['poses'], ref['points']) - O.lba_residuals(p, out['poses'], out['points'])).max() < TOL_PX


def test_many_fixed_keyframes_and_handle_creation_order():
    """The reference puts no bound on lFixedCameras (src/Optimizer.cc:1166-1186): a window with hundreds of fixed keyframes must
    run (pose caches hold all poses, the LDLT panels only the free ones).  And the shared-memory opt-in of the kernel is a
    per-function attribute: a smaller handle created after a larger one must not break the larger one."""
    import orb_slam3_modified_b200 as m
    big = m.Optimizer(max_poses=300, max_points=2000, max_edges=20000)
    p = synth.lba_problem(n_kf=280, n_pts=1500, obs_per_pt=10, seed=51, n_fixed=268)
    small = m.Optimizer(max_poses=4, max_points=100, max_edges=400)
    q = synth.lba_problem(n_kf=4, n_pts=80, obs_per_pt=4, seed=52)
    for opt_, prob in ((small, q), (big, p), (small, q), (big, p)):
        ref = O.lba_solve(prob)
        out = opt_.LocalBundleAdjustment(prob)
        assert out['iters'] == ref['iters'] and out['trials'] == int(ref['stats'][3])
        assert np.abs(O.lba_residuals(prob, ref['poses'], ref['points']) - O.lba_residuals(prob, out['poses'], out['points'])).max() < TOL_PX
    with pytest.raises(m.OrbError):       # beyond the shared-memory pose caches: a clear capacity error, not a launch failure
        huge = m.Optimizer(max_poses=900, max_points=1000, max_edges=9000)
        huge.LocalBundleAdjustment(synth.lba_problem(n_kf=900, n_pts=900, obs_per_pt=8, seed=53, n_fixed=890))


def test_device_structure_build_any_edge_order_and_rejects_bad_graphs(opt):
    """BlockSolver::buildStructure runs on the device: the caller's edges may come in any order (per-edge outputs come back in the
    caller's order), duplicate (point, keyframe) observations and out-of-range indices are refused."""
    import orb_slam3_modified_b200 as m
    p = synth.lba_problem(n_kf=9, n_pts=700, obs_per_pt=6, seed=41, n_fixed=2)
    perm = np.random.default_rng(5).permutation(len(p['edge_point']))
    q = dict(p)
    for k in ('edge_point', 'edge_pose', 'obs', 'inv_sigma2'):
        q[k] = np.ascontiguousarray(p[k][perm])
    _check(opt, q)
    dup = dict(p)
    e = int(np.flatnonzero(np.asarray(p['fixed'])[p['edge_pose']] == 0)[0])      # an observation by a free keyframe, given twice
    for k in ('edge_point', 'edge_pose', 'obs', 'inv_sigma2'):
        dup[k] = np.concatenate([p[k], p[k][e:e + 1]])
    with pytest.raises(m.OrbError):
        opt.LocalBundleAdjustment(dup)
    bad = dict(p)
    bad['edge_point'] = p['edge_point'].copy()
    bad['edge_point'][5] = len(p['points'])
    with pytest.raises(m.OrbError):
        opt.LocalBundleAdjustment(bad)
    _check(opt, p)      # the handle is usable after a refused graph
