"""GPU parity of LocalBundleAdjustment on the layouts and launch shapes the other LBA tests leave alone: one camera per
keyframe (fx != fy, off-centre principal point), fixed keyframes anywhere in the window, exact observer sets, work-chunk
boundaries, points behind a keyframe, heavy outliers (`lba_scenes`, whose oracle results `test_lba_layouts_cpu.py` checks
against a dense numeric step); every forced and automatic cluster size; the reduced camera system in shared and in global
memory; the bench's own 48-problem resident shape; argument errors; and PoseOptimization with a non-square camera.

Every result is held to `test_lba_gpu._check`'s bars: same iterations and trials, residuals within 1e-4 px, poses 1e-9,
points 1e-8, per-edge chi2, classification, depth flags and final chi2."""
import functools
import math

import numpy as np
import pytest

import lba_scenes as S
import oracle_lib as O
from orb_slam3_modified_b200 import synth
from test_lba_gpu import _agrees, _check

pytestmark = pytest.mark.gpu
PC = 20                # doubles per cached pose in the kernel's shared memory (csrc/lba.cu)


@functools.lru_cache(None)
def scenes():
    return {
        'interleaved': S.interleaved(n_kf=12, n_pts=600, obs_per_pt=5, seed=1),
        'last_fixed': S.last_fixed(n_kf=10, n_pts=500, obs_per_pt=4, seed=2),
        'none_fixed': S.none_fixed(n_kf=8, n_pts=400, obs_per_pt=4, seed=3),
        'observer_sets': S.observer_sets(n_kf=12, n_single=60, n_fixed_only=40, n_window=400, hub=11, seed=4),
        'hub': S.hub(seed=5),
        'chunk_edges': S.chunk_edges(seed=6),
        'depth_edges': S.depth_edges(n_kf=8, n_pts=300, n_far=30, seed=7),
        'outliers': S.outliers(n_kf=10, n_pts=500, obs_per_pt=5, seed=8),
    }


@functools.lru_cache(None)
def small():
    return S.small_layouts(seed=10)


@functools.lru_cache(None)
def ref(key):
    """Oracle result of a named problem: 'scene:<name>', 'small:<name>' or 'config4'."""
    return O.lba_solve(problem(key))


def problem(key):
    if key == 'config4':
        return config4()
    kind, name = key.split(':')
    return (scenes() if kind == 'scene' else small())[name]


@functools.lru_cache(None)
def config4():
    return synth.lba_problem(n_kf=20, n_pts=5000, obs_per_pt=8, seed=0)


SCENES = ('interleaved', 'last_fixed', 'none_fixed', 'observer_sets', 'hub', 'chunk_edges', 'depth_edges', 'outliers')
MIXED = ['scene:' + n for n in SCENES] + ['small:' + n for n in ('interleaved', 'observer_sets', 'depth_edges', 'outliers')]


def _same(a, b):
    """Byte-identical results."""
    return all(a[k].tobytes() == b[k].tobytes() for k in ('poses', 'points', 'chi2', 'depth_pos')) and \
        (a['iters'], a['trials'], a['final_chi2']) == (b['iters'], b['trials'], b['final_chi2'])


@pytest.fixture(scope='module')
def opt():
    import orb_slam3_modified_b200 as m
    m.lib()
    return m.Optimizer(max_poses=40, max_points=1000, max_edges=8000, max_batch=len(MIXED))


@pytest.mark.parametrize('name', SCENES)
def test_layout_alone(opt, name):
    out = opt.LocalBundleAdjustment(problem('scene:' + name))
    _agrees(problem('scene:' + name), out, ref('scene:' + name))
    if name == 'depth_edges':
        assert 0 < out['depth_pos'].sum() < len(out['depth_pos'])


def test_layouts_in_one_batch(opt):
    outs = opt.LocalBundleAdjustmentBatch([problem(k) for k in MIXED])
    for k, out in zip(MIXED, outs):
        _agrees(problem(k), out, ref(k))
    assert sum((out['depth_pos'] == 0).sum() for out in outs) > 0


def test_forced_cluster_sizes_single_problem():
    """Cluster sizes 1..8 forced on a config-4 problem: every one equals the oracle, and a repeat is byte-identical."""
    import orb_slam3_modified_b200 as m
    o4 = m.Optimizer(max_poses=20, max_points=5000, max_edges=40000)
    p = config4()
    for cs in range(1, 9):
        o4.set_cluster_size(cs)
        a = o4.LocalBundleAdjustment(p)
        assert o4.last_cluster_size() == cs
        _agrees(p, a, ref('config4'))
        assert _same(a, o4.LocalBundleAdjustment(p)), cs


def test_forced_cluster_sizes_mixed_batch(opt):
    import orb_slam3_modified_b200 as m
    probs = [problem(k) for k in MIXED]
    opt.set_cluster_size(0)
    opt.LocalBundleAdjustmentBatch(probs)
    auto = opt.last_cluster_size()
    try:
        for cs in range(1, 9):
            opt.set_cluster_size(cs)
            a = opt.LocalBundleAdjustmentBatch(probs)
            assert opt.last_cluster_size() == cs
            for k, out in zip(MIXED, a):
                _agrees(problem(k), out, ref(k))
            b = opt.LocalBundleAdjustmentBatch(probs)
            assert all(_same(x, y) for x, y in zip(a, b)), cs
        for bad in (9, -1):
            with pytest.raises(m.OrbError) as e:
                opt.set_cluster_size(bad)
            assert e.value.code == m.ORB_ERR_ARG
        opt.LocalBundleAdjustmentBatch(probs)
        assert opt.last_cluster_size() == 8              # a refused size leaves the forced one in place
    finally:
        opt.set_cluster_size(0)
    opt.LocalBundleAdjustmentBatch(probs)
    assert opt.last_cluster_size() == auto               # 0 returns to the automatic choice


def test_automatic_cluster_choice_at_its_steps():
    """The batch sizes where the automatic choice changes: every cluster of a launch is resident at once (count x size <= SMs)
    up to SMs problems, clusters of one beyond (more than one wave).  Ten distinct problems, replicated: every replica in a
    launch is byte-identical to its base, and every base equals the oracle."""
    import torch
    import orb_slam3_modified_b200 as m
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    bases = [S.interleaved(n_kf=5, n_pts=50, obs_per_pt=3, seed=40 + i) if i % 2 else S.last_fixed(n_kf=6, n_pts=60, obs_per_pt=3, seed=40 + i)
             for i in range(10)]
    refs = [O.lba_solve(p) for p in bases]
    ob = m.Optimizer(max_poses=6, max_points=60, max_edges=200, max_batch=sms + 8)
    for count in (1, sms // 8, sms // 8 + 1, 48, sms // 2, sms // 2 + 1, sms, sms + 8):
        outs = ob.LocalBundleAdjustmentBatch([bases[i % 10] for i in range(count)])
        cs = ob.last_cluster_size()
        assert 1 <= cs <= 8 and (count * cs <= sms if count <= sms else cs == 1), (count, cs)
        for i, out in enumerate(outs):
            if i < 10:
                _agrees(bases[i], out, refs[i])
            else:
                assert _same(out, outs[i % 10]), (count, i)


def _matrix_in_shared_memory(probs):
    """csrc/lba.cu Solver::run: the pose caches (PC doubles for every pose) and the LDLT panels (78 doubles per free pose) of the
    largest problem come first; the reduced camera system (6 nF)^2 joins them in shared memory only when every problem's fits."""
    mp = max(1, max(len(p['poses']) for p in probs))
    mf = max(1, max(int((np.asarray(p['fixed']) == 0).sum()) for p in probs))
    fixed_smem = 8 * (2 * PC * mp + 78 * mf + 16)
    smem_n = math.floor(math.sqrt((200 * 1024 - fixed_smem) / 8))
    return all(6 * int((np.asarray(p['fixed']) == 0).sum()) <= smem_n for p in probs)


def test_reduced_system_in_shared_and_global_memory():
    """One large problem moves every problem of its launch to the global-memory reduced camera system.  The same code runs on a
    different pointer, so a small problem's result is byte-identical on both sides (same forced cluster size)."""
    import orb_slam3_modified_b200 as m
    fit = S.masked(np.r_[1, np.zeros(25, np.uint8)], n_pts=300, obs_per_pt=5, seed=61)      # 25 free poses: the largest that fits
    over = S.masked(np.r_[1, np.zeros(26, np.uint8)], n_pts=300, obs_per_pt=5, seed=62)     # 26 free poses: global memory
    small_p = problem('small:interleaved')
    all_fixed = S.masked(np.ones(5, np.uint8), n_pts=40, obs_per_pt=3, seed=63)              # nF = 0: only points move
    assert _matrix_in_shared_memory([fit]) and not _matrix_in_shared_memory([over])
    assert _matrix_in_shared_memory([small_p]) and _matrix_in_shared_memory([small_p, fit]) and not _matrix_in_shared_memory([small_p, over])
    ob = m.Optimizer(max_poses=27, max_points=300, max_edges=1500, max_batch=4)
    ob.set_cluster_size(4)
    alone = ob.LocalBundleAdjustment(small_p)
    _agrees(small_p, alone, ref('small:interleaved'))
    for p in (fit, over, all_fixed):
        _check(ob, p)
    with_fit = ob.LocalBundleAdjustmentBatch([small_p, fit])
    assert _same(with_fit[0], alone)
    mixed = ob.LocalBundleAdjustmentBatch([small_p, over, all_fixed])
    assert ob.last_cluster_size() == 4
    assert _same(mixed[0], alone)
    _agrees(all_fixed, mixed[2], O.lba_solve(all_fixed))
    _agrees(over, mixed[1], O.lba_solve(over))


def test_bench_shape_resident_on_a_side_stream():
    """bench.py's LBA work: 48 config-4 problems (4 distinct) uploaded once and run twice with run_device on a side stream."""
    import torch
    import bench
    import orb_slam3_modified_b200 as m
    probs = bench.lba_problems(48)
    cfg = bench.LBA_CFG
    ob = m.Optimizer(max_poses=cfg['n_kf'], max_points=cfg['n_pts'], max_edges=cfg['n_pts'] * cfg['obs_per_pt'], max_batch=48)
    ob.upload(probs)
    side = torch.cuda.Stream()
    ob.run_device(side.cuda_stream)
    ob.run_device(side.cuda_stream)
    outs = ob.download()
    for i in range(4):
        assert probs[i] is not probs[(i + 1) % 4]
        _agrees(probs[i], outs[i], O.lba_solve(probs[i]))
    for i in range(4, 48):
        assert probs[i] is probs[i % 4] and _same(outs[i], outs[i % 4]), i


def test_argument_errors_leave_the_handle_usable():
    import orb_slam3_modified_b200 as m
    ob = m.Optimizer(max_poses=8, max_points=100, max_edges=400, max_batch=2)
    p = S.interleaved(n_kf=6, n_pts=60, obs_per_pt=3, seed=71)
    big = S.interleaved(n_kf=9, n_pts=60, obs_per_pt=3, seed=72)                             # 9 poses > max_poses
    empty = dict(p, fixed=np.ones(6, np.uint8), points=np.zeros((0, 3)), edge_point=np.zeros(0, np.int32), edge_pose=np.zeros(0, np.int32),
                 obs=np.zeros((0, 2)), inv_sigma2=np.zeros(0, np.float32))                  # nF + nL == 0
    refused = [lambda: ob.upload([]), lambda: ob.LocalBundleAdjustmentBatch([p, p, p]), lambda: ob.LocalBundleAdjustment(big),
               lambda: ob.LocalBundleAdjustment(empty), lambda: ob.LocalBundleAdjustmentBatch([p, big])]
    for call in refused:
        with pytest.raises(m.OrbError) as e:
            call()
        assert e.value.code == m.ORB_ERR_ARG
        _check(ob, p)
    # a refused upload leaves nothing to run: the slots it had started to rewrite must not be run or downloaded
    ob.upload([p, p])
    with pytest.raises(m.OrbError):
        ob.upload([p, big])
    for call in (ob.run_device, ob.download):
        with pytest.raises(m.OrbError) as e:
            call()
        assert e.value.code == m.ORB_ERR_ARG
    # download of more problems than were uploaded
    ob.upload([p])
    ob.run_device()
    keep, _, out, r = m.Optimizer._pack(p, 10, 0.0, None)
    R = (m._LbaResult * 2)(r, r)
    assert m.lib().lba_download_batch(ob._h, 2, R) == m.ORB_ERR_ARG
    _agrees(p, ob.download()[0], O.lba_solve(p))
    _check(ob, p)


def test_pose_optimization_non_square_camera():
    """PoseOptimization with fx != fy and the principal point off the centre: observations built from Xw through that camera."""
    import orb_slam3_modified_b200 as m
    frames = [S.pose_opt_frame(n=n, seed=80 + i, outlier_frac=f) for i, (n, f) in enumerate([(300, 0.2), (800, 0.35), (40, 0.1), (500, 0.5)])]
    outs = m.PoseOptimization(frames)
    for f, out in zip(frames, outs):
        r = O.pose_optimization(f)
        assert out['inliers'] == r['inliers'] and np.array_equal(out['outlier'], r['outlier'])
        assert np.allclose(out['pose'], r['pose'], atol=1e-9)
    assert outs[0]['inliers'] > 200
