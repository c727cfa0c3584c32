"""LocalBundleAdjustment with helper clusters: a batch whose own clusters leave SMs idle is launched with extra clusters that
serve the chunked phases (build, point records, Schur partial sums) of any problem.  Whichever CTA serves a chunk, the chunk
gives the same bits, so a run with helpers must be byte-identical to a run without them: on bench.py's 48 problems, on a mixed
batch (different sizes, a problem with no free pose, one with a single free pose and one much larger than the rest, which the
helpers serve after the others finish), on a batch that already fills the GPU, at forced cluster sizes 1 to 4, and over two
runs on one handle with other problems uploaded in between.  A sample is held to the oracle, and a run with its stop flag
set terminates."""
import ctypes as C
import functools

import numpy as np
import pytest

import lba_scenes as S
import oracle_lib as O
from test_lba_gpu import _agrees
from test_lba_pipelined_passes_gpu import _same, one_free

pytestmark = pytest.mark.gpu


@functools.lru_cache(None)
def bench_problems():
    from bench import lba_problems
    return tuple(lba_problems(48))


@functools.lru_cache(None)
def mixed():
    from orb_slam3_modified_b200 import synth
    return (
        synth.lba_problem(n_kf=6, n_pts=300, obs_per_pt=5, seed=3),
        S.masked(np.ones(6, np.uint8), n_pts=200, obs_per_pt=3, seed=7),        # no free pose: no Schur phase
        one_free(seed=5),                                                         # a single free pose
        synth.lba_problem(n_kf=10, n_pts=1000, obs_per_pt=6, seed=11),
        synth.lba_problem(n_kf=20, n_pts=5000, obs_per_pt=8, seed=12),         # much larger than the rest
        S.chunk_edges(counts=(1, 2, 3, 128, 129, 130, 131), seed=4),
    )


def _opt(max_batch, max_poses=32, max_points=5000, max_edges=40000):
    import orb_slam3_modified_b200 as m
    m.lib()
    return m.Optimizer(max_poses=max_poses, max_points=max_points, max_edges=max_edges, max_batch=max_batch)


def _helped(opt, n):
    import orb_slam3_modified_b200 as m
    ns = np.zeros(10)
    out = []
    for i in range(n):
        assert m.lib().lba_get_phase_ns(opt._h, i, ns.ctypes.data_as(C.c_void_p)) == 0
        out.append(int(ns[9]))
    return out


def _with_and_without(opt, probs):
    """Results with helpers (default) and without; the helper clusters and helper-served chunks of the first run."""
    opt.set_helpers(-1)
    a = opt.LocalBundleAdjustmentBatch(list(probs))
    nh, helped = opt.last_helpers(), _helped(opt, len(probs))
    opt.set_helpers(0)
    try:
        b = opt.LocalBundleAdjustmentBatch(list(probs))
        assert opt.last_helpers() == 0 and sum(_helped(opt, len(probs))) == 0
    finally:
        opt.set_helpers(-1)
    for i, (x, y) in enumerate(zip(a, b)):
        assert _same(x, y), i
    return a, nh, helped


def test_bench_batch():
    probs = bench_problems()
    opt = _opt(len(probs), max_poses=20)
    out, nh, helped = _with_and_without(opt, probs)
    assert opt.last_cluster_size() == 2 and nh > 0 and sum(helped) > 0
    _agrees(probs[0], out[0], O.lba_solve(probs[0]))


def test_mixed_batch():
    probs = mixed()
    opt = _opt(len(probs))
    out, nh, helped = _with_and_without(opt, probs)
    assert nh > 0 and helped[4] > 0
    for i in (0, 1, 2, 5):
        _agrees(probs[i], out[i], O.lba_solve(probs[i]))


@pytest.mark.parametrize('cluster', [1, 2, 3, 4])
def test_forced_cluster_sizes(cluster):
    probs = mixed()
    opt = _opt(len(probs))
    opt.set_cluster_size(cluster)
    _, nh, _ = _with_and_without(opt, probs)
    assert opt.last_cluster_size() == cluster and nh > 0


def test_batch_that_fills_the_gpu():
    import torch
    n = torch.cuda.get_device_properties(0).multi_processor_count + 4
    probs = [mixed()[i % 4] for i in range(n)]
    opt = _opt(n, max_points=1000, max_edges=6000)
    a = opt.LocalBundleAdjustmentBatch(probs)
    assert opt.last_cluster_size() == 1 and opt.last_helpers() == 0
    for i in range(4):
        assert _same(a[i], a[i + 4]), i


def test_two_runs_on_one_handle():
    first, second = mixed()[:3], mixed()[3:]
    opt = _opt(3)
    opt.set_helpers(0)
    ref = [opt.LocalBundleAdjustmentBatch(list(first)), opt.LocalBundleAdjustmentBatch(list(second))]
    opt.set_helpers(-1)
    for _ in range(2):
        for probs, r in zip((first, second), ref):
            opt.upload(list(probs))
            opt.run_device()
            out = opt.download()
            assert opt.last_helpers() > 0
            for i, (x, y) in enumerate(zip(out, r)):
                assert _same(x, y), i


def test_stop_flag_terminates():
    p = mixed()[4]
    opt = _opt(1)
    flag = np.ones(1, np.uint8)
    out = opt.LocalBundleAdjustment(p, stop_flag=flag)
    assert opt.last_helpers() > 0
    assert out['iters'] == 0 and np.array_equal(out['poses'], opt.LocalBundleAdjustment(p, stop_flag=flag)['poses'])
