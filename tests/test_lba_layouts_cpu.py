"""The LBA oracle on the layouts of `lba_scenes` (one camera per keyframe with fx != fy and an off-centre principal point,
fixed keyframes anywhere in the window, exact observer sets, points behind a keyframe and 500 m away, 40 % outliers),
checked against independent evidence before the GPU is held to it (`test_lba_paths_gpu.py`): one oracle LM step equals
the dense numeric-Jacobian step of `test_lba_dense_cpu.py`, and the oracle's depth flags equal a numpy depth test."""
import numpy as np
import pytest

import lba_scenes as S
import oracle_lib as O
from test_lba_dense_cpu import _R, _exp, _residuals

LAYOUTS = S.small_layouts()


def _dense_step(p):
    """One Levenberg-Marquardt step over all free poses and points from numerical Jacobians of the reprojection residual
    (test_lba_dense_cpu.py: central differences on the manifold, g2o's robustified normal equations, computeLambdaInit)."""
    nP, nL = len(p['poses']), len(p['points'])
    q = p['poses'][:, :4] / np.linalg.norm(p['poses'][:, :4], axis=1)[:, None]
    Rs = [_R(q[i]) for i in range(nP)]
    ts = [p['poses'][i, 4:].astype(np.float64) for i in range(nP)]
    X = p['points'].astype(np.float64)
    free = [i for i in range(nP) if not p['fixed'][i]]
    col = {i: 6 * k for k, i in enumerate(free)}
    n = 6 * len(free) + 3 * nL
    e0 = _residuals(p, Rs, ts, X)
    J = np.zeros((2 * len(e0), n))
    h = 1e-6
    for i in free:
        for a in range(6):
            d = np.zeros(6); d[a] = h
            out = []
            for s in (+1, -1):
                Rd, td = _exp(s * d)
                Rs2, ts2 = list(Rs), list(ts)
                Rs2[i] = Rd @ Rs[i]; ts2[i] = Rd @ ts[i] + td
                out.append(_residuals(p, Rs2, ts2, X))
            J[:, col[i] + a] = ((out[0] - out[1]) / (2 * h)).reshape(-1)
    for l in range(nL):
        for a in range(3):
            out = []
            for s in (+1, -1):
                X2 = X.copy(); X2[l, a] += s * h
                out.append(_residuals(p, Rs, ts, X2))
            J[:, 6 * len(free) + 3 * l + a] = ((out[0] - out[1]) / (2 * h)).reshape(-1)
    is2 = p['inv_sigma2'].astype(np.float64)
    chi2 = is2 * (e0 ** 2).sum(1)
    delta = float(p['huber_delta'])
    rho1 = np.where(chi2 <= delta * delta, 1.0, delta / np.sqrt(np.maximum(chi2, 1e-300)))
    w = np.repeat(rho1 * is2, 2)
    Hm = J.T @ (w[:, None] * J)
    b = -J.T @ (w * e0.reshape(-1))
    lam = 1e-5 * np.abs(np.diag(Hm)).max()
    dx = np.linalg.solve(Hm + lam * np.eye(n), b)
    poses = {}
    for i in free:
        Rd, td = _exp(dx[col[i]:col[i] + 6])
        poses[i] = (Rd @ Rs[i], Rd @ ts[i] + td)
    return poses, X + dx[6 * len(free):].reshape(nL, 3), X


@pytest.mark.parametrize('name', sorted(LAYOUTS))
def test_one_oracle_step_equals_the_dense_numeric_step(name):
    p = LAYOUTS[name]
    ref = O.lba_solve(p, iterations=1)
    assert ref['iters'] == 1 and int(ref['stats'][3]) == 1            # one iteration, one (accepted) trial
    poses, Xn, X = _dense_step(p)
    for i, (Rn, tn) in poses.items():
        qo = ref['poses'][i, :4]
        assert np.abs(_R(qo / np.linalg.norm(qo)) - Rn).max() < 2e-7, (name, i)
        assert np.abs(ref['poses'][i, 4:] - tn).max() < 2e-7, (name, i)
    assert np.abs(ref['points'] - Xn).max() < 2e-6
    assert np.abs(ref['points'] - X).max() > 1e-3                     # a real step


@pytest.mark.parametrize('name', sorted(LAYOUTS))
def test_depth_flags_equal_a_numpy_depth_test(name):
    p = LAYOUTS[name]
    ref = O.lba_solve(p)
    z = S.depths(p, ref['poses'], ref['points'])
    assert np.array_equal(ref['depth_pos'], (z > 0).astype(np.uint8))
    if name == 'depth_edges':
        assert 0 < ref['depth_pos'].sum() < len(z) and (z[ref['depth_pos'] == 0] < -0.5).all()


def test_layouts_have_what_they_promise():
    """The properties the GPU tests rely on, stated once here for the small instances (each scene also asserts its own counts)."""
    for name, p in LAYOUTS.items():
        assert (np.abs(p['cam'][:, 0] - p['cam'][:, 1]) > 20).all() and len(np.unique(p['cam'], axis=0)) == len(p['cam']), name
        assert set(p) >= {'poses', 'fixed', 'cam', 'points', 'edge_point', 'edge_pose', 'obs', 'inv_sigma2', 'huber_delta'}
        assert p['poses'].dtype == np.float64 and np.array_equal(p['poses'], p['poses'].astype(np.float32).astype(np.float64))
        assert np.array_equal(p['obs'], p['obs'].astype(np.float32).astype(np.float64))
        assert np.all(np.diff(p['edge_point']) >= 0)                  # grouped by point, as synth.lba_problem
    free_after_fixed = [n for n, p in LAYOUTS.items() if p['fixed'].any() and np.flatnonzero(p['fixed'] == 0).max() > np.flatnonzero(p['fixed']).min()]
    assert {'interleaved', 'observer_sets', 'depth_edges', 'outliers'} <= set(free_after_fixed)
    assert not LAYOUTS['none_fixed']['fixed'].any() and LAYOUTS['last_fixed']['fixed'][-2:].all()


def test_gpu_scenes_build_with_their_counts():
    """The larger scenes of test_lba_paths_gpu.py (33-observer point, chunk boundaries, ...) assert their counts when built."""
    from test_lba_paths_gpu import scenes
    sc = scenes()
    assert np.bincount(sc['hub']['edge_point']).max() == 33
    assert (S.depths(sc['depth_edges']) < 0).any()
