"""CPU: the oracle of Optimizer::LocalInertialBA (oracle/local_inertial_ba_oracle.cpp; reference src/Optimizer.cc:2383-2958) is pinned by an
independent derivation, since g2o / G2oTypes need Eigen and cannot be compiled into oracle/_ref:
  * its first Levenberg-Marquardt step (lambda = the reference's setUserLambdaInit value) equals the dense damped normal-equation step built
    from NUMERICAL derivatives of the stacked, whitened residuals (EdgeMono, EdgeInertial incl. the down-weighted link to the fixed keyframe,
    EdgeGyroRW, EdgeAccRW) under the reference's update rules (ImuCamPose::Update, additive velocity / bias / point updates), with all points
    eliminated by nothing but numpy's dense solve (no Schur complement);
  * on noisy data it recovers the window and flags the gross outliers; at the noise-free ground truth it stays put."""
import numpy as np

import oracle_lib as O
from orb_slam3_modified_b200 import synth


def _consistent(pr):
    """camera poses derived from the body poses in double (what ImuCamPose::Update computes), so that a zero update is a fixed point"""
    ex = pr['extr']; Rcb, tcb = ex[:9].reshape(3, 3), ex[9:12]
    for k in range(pr['n_kf']):
        R, p = pr['state'][k, :9].reshape(3, 3), pr['state'][k, 9:12]
        pr['tcw'][k, :9] = (Rcb @ R.T).reshape(9); pr['tcw'][k, 9:] = Rcb @ (-R.T @ p) + tcb
    return pr


def test_first_lm_step_is_the_dense_damped_step_from_numerical_derivatives():
    pr = _consistent(synth.local_inertial_ba_problem(n_opt=3, n_cov_fixed=1, n_pts=30, seed=2, outlier_frac=0.0, perturb=0.05, noise_px=0.2, float_inputs=False))
    P = O.liba_preints(pr)
    nO, nL, nE = pr['n_opt'], len(pr['points']), len(pr['e_pt'])
    ex = pr['extr']; Rcb, tcb = ex[:9].reshape(3, 3), ex[9:12]
    infos = [O.imu_information(P[i]) for i in range(nO)]
    chol = []
    for i, (i9, ig, ia) in enumerate(infos):
        chol.append((np.linalg.cholesky(i9 * pr['ie_info_scale'][i] + 1e-18 * np.eye(9)), np.linalg.cholesky(ig), np.linalg.cholesky(ia)))

    def apply(x):
        st = pr['state'].copy(); pts = pr['points'].copy()
        for k in range(nO):
            d = x[15 * k:15 * k + 15]
            R, t = O.imu_pose_update(st[k, :9].reshape(3, 3), st[k, 9:12], d[:6])
            st[k, :9] = R.reshape(9); st[k, 9:12] = t; st[k, 12:15] += d[6:9]; st[k, 15:18] += d[9:12]; st[k, 18:21] += d[12:15]
        pts += x[15 * nO:].reshape(-1, 3)
        return st, pts

    chi_inertial = []

    def residuals(x):
        st, pts = apply(x)
        out = []
        cams = []
        for k in range(pr['n_kf']):
            R, p = st[k, :9].reshape(3, 3), st[k, 9:12]
            cams.append((Rcb @ R.T, Rcb @ (-R.T @ p) + tcb))
        for e in range(nE):
            Rc, tc = cams[pr['e_kf'][e]]
            Xc = Rc @ pts[pr['e_pt'][e]] + tc
            c = pr['cam'][pr['e_kf'][e]].astype(np.float64)
            out.append(np.sqrt(float(pr['inv_sigma2'][e])) * (pr['obs'][e] - np.array([c[0] * Xc[0] / Xc[2] + c[2], c[1] * Xc[1] / Xc[2] + c[3]])))
        for i in range(nO):
            a, b = st[pr['ie_kf1'][i]], st[pr['ie_kf2'][i]]
            e9 = O.imu_edge_inertial(P[i], dict(Rwb1=a[:9].reshape(3, 3), twb1=a[9:12], v1=a[12:15], bg=a[15:18], ba=a[18:21], Rwb2=b[:9].reshape(3, 3), twb2=b[9:12], v2=b[12:15]),
                                     jac=False)[0]
            chi_inertial.append(float(e9 @ (infos[i][0] * pr['ie_info_scale'][i]) @ e9))
            out.append(chol[i][0].T @ e9)
            out.append(chol[i][1].T @ (b[15:18] - a[15:18]))
            out.append(chol[i][2].T @ (b[18:21] - a[18:21]))
        return np.concatenate(out)
    n = 15 * nO + 3 * nL
    r0 = residuals(np.zeros(n))
    # no Huber weight is active at the linearisation point (mono: sqrt(5.991); inertial link: sqrt(16.92))
    assert (r0[:2 * nE].reshape(-1, 2) ** 2).sum(1).max() < 5.99 and chi_inertial[nO - 1] < 16.9
    J = np.zeros((len(r0), n))
    for k in range(n):
        h = 2e-3 if (k < 15 * nO and k % 15 >= 9) else 1e-6     # bias steps must stand out of the float rounding of the preintegrated terms
        d = np.zeros(n); d[k] = h
        J[:, k] = (residuals(d) - residuals(-d)) / (2 * h)
    lam = pr['lambda_init']
    dx = np.linalg.solve(J.T @ J + lam * np.eye(n), -J.T @ r0)
    want_st, want_pts = apply(dx)
    got = O.local_inertial_ba(pr, P, iterations=1)
    assert got['trials'] == 1 and got['iters'] == 1 and not got['failed']
    assert np.allclose(got['state'], want_st, rtol=0, atol=3e-6), np.abs(got['state'] - want_st).max()
    assert np.allclose(got['points'], want_pts, rtol=0, atol=3e-5), np.abs(got['points'] - want_pts).max()
    # the robust cost the oracle reports before the step is the squared norm of the stacked residuals
    assert abs(got['err'] - float(r0 @ r0)) < 1e-3 * float(r0 @ r0)


def test_recovers_the_window_and_flags_gross_outliers():
    for seed, large in ((1, False), (3, True)):
        pr = synth.local_inertial_ba_problem(n_opt=10 if not large else 14, n_cov_fixed=3, n_pts=500, seed=seed, large=large)
        P = O.liba_preints(pr)
        r = O.local_inertial_ba(pr, P)
        nO = pr['n_opt']
        assert not r['failed'] and r['err_end'] < 0.05 * r['err'] and 1 <= r['iters'] <= pr['iterations']
        before = np.abs(pr['state'][:nO, 9:12] - pr['truth'][:nO, 9:12]).max(); after = np.abs(r['state'][:nO, 9:12] - pr['truth'][:nO, 9:12]).max()
        assert after < 0.5 * before, (before, after)
        assert np.abs(r['state'][:nO, 12:15] - pr['truth'][:nO, 12:15]).max() < 0.02
        # fixed keyframes do not move
        assert np.array_equal(r['state'][nO:], pr['state'][nO:]) and np.array_equal(r['tcw'][nO:], pr['tcw'][nO:])
        # the optimised camera pose is the one ImuCamPose::Update derives from the body pose
        ex = pr['extr']; Rcb, tcb = ex[:9].reshape(3, 3), ex[9:12]
        for k in range(nO):
            R, p = r['state'][k, :9].reshape(3, 3), r['state'][k, 9:12]
            assert np.allclose(r['tcw'][k, :9].reshape(3, 3), Rcb @ R.T, atol=1e-12) and np.allclose(r['tcw'][k, 9:], Rcb @ (-R.T @ p) + tcb, atol=1e-12)
            assert np.allclose(R.T @ R, np.eye(3), atol=1e-6)       # the float rounding of the keyframe's Rwb stays: the reference never renormalises it (G2oTypes.cc:206 discards the result)
        # erased observations: residual test of :2848-2862 on the final state
        res = O.local_inertial_ba_residuals(pr, r['tcw'], r['points'])
        chi = pr['inv_sigma2'] * (res ** 2).sum(1)
        close = pr['track_depth'][pr['e_pt']] < 10
        want = np.where(close, chi > 1.5 * 5.991, chi > 5.991)
        assert (want != r['erase'].astype(bool)).mean() < 0.01          # the edges hold the errors of the last evaluated state; depth is positive here
        assert 0.01 < r['erase'].mean() < 0.12


def test_noise_free_ground_truth_is_a_fixed_point():
    pr = _consistent(synth.local_inertial_ba_problem(n_opt=5, n_cov_fixed=2, n_pts=120, seed=4, outlier_frac=0.0, perturb=0.0, noise_px=0.0, float_inputs=False))
    pr['imu'] = [synth.imu_interval(pr['times'][i + 1], pr['times'][i], rate=2000.0, seed=i, bias=tuple(pr['bias6']), noise=False) for i in range(pr['n_opt'])]
    P = O.liba_preints(pr)
    r = O.local_inertial_ba(pr, P)
    assert not r['failed'] and r['erase'].sum() == 0
    assert np.abs(r['state'][:, 9:12] - pr['truth'][:, 9:12]).max() < 2e-3 and np.abs(r['points'] - pr['points_true']).max() < 2e-2


# ---- the kernel's phase functions, run by a serial executor on the host (tests/liba_emulate.cpp), against the oracle ----
def _emulate(pr, P):
    import ctypes as C
    import os
    import subprocess
    import orb_slam3_modified_b200 as orb
    here = os.path.dirname(os.path.abspath(__file__))
    so, src = os.path.join(here, 'libliba_emulate.so'), os.path.join(here, 'liba_emulate.cpp')
    deps = [src] + [os.path.join(here, '..', 'orb_slam3_modified_b200', 'csrc', f) for f in ('liba_core.cuh', 'liba_pack.h', 'inertial_dev.cuh')]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.check_call(['g++', '-O2', '-std=c++17', '-fPIC', '-shared', '-o', so, src])
    L = C.CDLL(so)
    q = dict(pr); q['preint'] = P
    Pm, Rm, keep, outs = orb._liba_marshal([q])
    err = C.create_string_buffer(256)
    L.liba_emulate.argtypes = [C.c_void_p, C.c_void_p, C.c_char_p, C.c_int]
    it = L.liba_emulate(C.cast(Pm, C.c_void_p), C.cast(Rm, C.c_void_p), err, 256)
    assert it >= 0, err.value
    return orb._liba_finish(outs, [it])[0]


def _same_solve(a, b, pr, tol_state=1e-8):
    assert a['iters'] == b['iters'] and a['trials'] == b['trials'] and a['failed'] == b['failed'], (a['iters'], b['iters'], a['trials'], b['trials'])
    assert abs(a['err'] - b['err']) <= 1e-6 * abs(b['err']) and abs(a['err_end'] - b['err_end']) <= 1e-5 * abs(b['err_end']) + 1e-9
    assert abs(a['lam'] - b['lam']) <= 1e-6 * abs(b['lam'])
    assert np.abs(a['state'] - b['state']).max() < tol_state and np.abs(a['tcw'] - b['tcw']).max() < tol_state
    ra = O.local_inertial_ba_residuals(pr, a['tcw'], a['points']); rb = O.local_inertial_ba_residuals(pr, b['tcw'], b['points'])
    d = np.abs(ra - rb)
    sane = np.abs(rb).max(1) < 1e3                         # unobservable outlier-only points can sit anywhere along their ray
    assert d[sane].max(initial=0.0) < 1e-4, d[sane].max(initial=0.0)     # the north-star bar: reprojection residuals within 1e-4 px
    assert np.array_equal(a['erase'], b['erase'])
    assert np.allclose(a['chi2'][sane], b['chi2'][sane], rtol=1e-6, atol=1e-6)


def test_kernel_phases_on_the_host_equal_the_oracle():
    cases = [dict(n_opt=10, n_cov_fixed=3, n_pts=400, seed=1), dict(n_opt=14, n_cov_fixed=2, n_pts=300, seed=3, large=True), dict(n_opt=1, n_cov_fixed=2, n_pts=60, seed=5),
             dict(n_opt=4, n_cov_fixed=0, n_pts=120, seed=6, rec_init=True), dict(n_opt=6, n_cov_fixed=1, n_pts=200, seed=7, perturb=4.0)]
    for kw in cases:
        pr = synth.local_inertial_ba_problem(**kw)
        P = O.liba_preints(pr)
        _same_solve(_emulate(pr, P), O.local_inertial_ba(pr, P), pr)


def test_kernel_phases_default_lambda_and_rejected_steps():
    pr = synth.local_inertial_ba_problem(n_opt=5, n_cov_fixed=1, n_pts=150, seed=8)
    P = O.liba_preints(pr)
    pr['lambda_init'] = 0.0                                 # computeLambdaInit's tau * max diagonal branch
    _same_solve(_emulate(pr, P), O.local_inertial_ba(pr, P), pr)
    pr['lambda_init'] = 1e-12                               # an (almost) undamped first step on a far-off start: rejected trials, lambda growth
    pr2 = synth.local_inertial_ba_problem(n_opt=5, n_cov_fixed=1, n_pts=150, seed=9, perturb=12.0)
    pr2['lambda_init'] = 1e-12
    P2 = O.liba_preints(pr2)
    a, b = _emulate(pr2, P2), O.local_inertial_ba(pr2, P2)
    assert b['trials'] > b['iters']                         # at least one rejected trial happened
    _same_solve(a, b, pr2, tol_state=1e-7)


def test_threaded_batch_packing_equals_single_packing():
    import ctypes as C
    import os
    import orb_slam3_modified_b200 as orb
    prs = []
    for sd in range(12):
        pr = synth.local_inertial_ba_problem(n_opt=3 + sd % 4, n_cov_fixed=1 + sd % 3, n_pts=2500 if sd % 2 else 700, seed=40 + sd)
        pr['preint'] = O.liba_preints(pr)
        pr['iterations'] = 2                                # the packing is what is tested; two LM iterations keep the serial executor short
        prs.append(pr)
    singles = [_emulate(pr, pr['preint']) for pr in prs]    # (also builds the emulation library)
    L = C.CDLL(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'libliba_emulate.so'))
    Pm, Rm, keep, outs = orb._liba_marshal(prs)
    its = np.zeros(len(prs), np.int32); err = C.create_string_buffer(256)
    L.liba_emulate_batch.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_char_p, C.c_int]
    assert L.liba_emulate_batch(len(prs), C.cast(Pm, C.c_void_p), C.cast(Rm, C.c_void_p), its.ctypes.data, err, 256) == 0, err.value
    got = orb._liba_finish(outs, its)
    for a, b in zip(got, singles):
        assert a['iters'] == b['iters'] and a['state'].tobytes() == b['state'].tobytes() and a['points'].tobytes() == b['points'].tobytes() and np.array_equal(a['erase'], b['erase'])


def test_converged_solution_is_the_minimum_an_independent_optimizer_finds():
    """Without gross outliers and with a mild start no Huber kernel is active near the optimum, so the cost is a plain weighted least-squares problem:
    scipy's trust-region solver (numerical Jacobian, its own global parametrisation: rotation vector relative to the start, world-frame translation)
    must end in the same keyframe states and points as the oracle's Levenberg-Marquardt run to convergence."""
    from scipy.optimize import least_squares
    pr = _consistent(synth.local_inertial_ba_problem(n_opt=3, n_cov_fixed=1, n_pts=25, seed=13, outlier_frac=0.0, perturb=0.3, noise_px=0.3, float_inputs=False))
    P = O.liba_preints(pr)
    nO, nL, nE = pr['n_opt'], len(pr['points']), len(pr['e_pt'])
    ex = pr['extr']; Rcb, tcb = ex[:9].reshape(3, 3), ex[9:12]
    infos = [O.imu_information(P[i]) for i in range(nO)]
    chol = [(np.linalg.cholesky(i9 * pr['ie_info_scale'][i] + 1e-18 * np.eye(9)), np.linalg.cholesky(ig), np.linalg.cholesky(ia)) for i, (i9, ig, ia) in enumerate(infos)]
    st0, pts0 = pr['state'].copy(), pr['points'].copy()

    def unpack(x):
        st = st0.copy()
        for k in range(nO):
            d = x[15 * k:15 * k + 15]
            st[k, :9] = (st0[k, :9].reshape(3, 3) @ synth._rodrigues(d[:3])).reshape(9)
            st[k, 9:12] = st0[k, 9:12] + d[3:6]; st[k, 12:15] = st0[k, 12:15] + d[6:9]; st[k, 15:18] = st0[k, 15:18] + d[9:12]; st[k, 18:21] = st0[k, 18:21] + d[12:15]
        return st, pts0 + x[15 * nO:].reshape(-1, 3)

    def residuals(x):
        st, pts = unpack(x)
        out = []
        cams = [(Rcb @ st[k, :9].reshape(3, 3).T, Rcb @ (-st[k, :9].reshape(3, 3).T @ st[k, 9:12]) + tcb) for k in range(pr['n_kf'])]
        for e in range(nE):
            Rc, tc = cams[pr['e_kf'][e]]
            Xc = Rc @ pts[pr['e_pt'][e]] + tc
            c = pr['cam'][pr['e_kf'][e]].astype(np.float64)
            out.append(np.sqrt(float(pr['inv_sigma2'][e])) * (pr['obs'][e] - np.array([c[0] * Xc[0] / Xc[2] + c[2], c[1] * Xc[1] / Xc[2] + c[3]])))
        for i in range(nO):
            a, b = st[pr['ie_kf1'][i]], st[pr['ie_kf2'][i]]
            e9 = O.imu_edge_inertial(P[i], dict(Rwb1=a[:9].reshape(3, 3), twb1=a[9:12], v1=a[12:15], bg=a[15:18], ba=a[18:21], Rwb2=b[:9].reshape(3, 3), twb2=b[9:12], v2=b[12:15]),
                                     jac=False)[0]
            out += [chol[i][0].T @ e9, chol[i][1].T @ (b[15:18] - a[15:18]), chol[i][2].T @ (b[18:21] - a[18:21])]
        return np.concatenate(out)
    n = 15 * nO + 3 * nL
    # the float preintegration makes the residual piecewise constant at the 1e-7 level in the biases: finite-difference steps must stand out of it
    step = np.full(n, 1e-6)
    for k in range(nO):
        step[15 * k + 9:15 * k + 15] = 2e-3

    def jac(x):
        J = np.zeros((len(residuals(x)), n))
        for k in range(n):
            d = np.zeros(n); d[k] = step[k]
            J[:, k] = (residuals(x + d) - residuals(x - d)) / (2 * step[k])
        return J
    sol = least_squares(residuals, np.zeros(n), method='trf', jac=jac, xtol=1e-15, ftol=1e-15, gtol=1e-12, max_nfev=100)
    got = O.local_inertial_ba(pr, P, iterations=60)
    st_s, pts_s = unpack(sol.x)
    # no Huber weight is active at either solution
    rr = residuals(sol.x)
    assert (rr[:2 * nE].reshape(-1, 2) ** 2).sum(1).max() < 5.99
    cost_scipy = float(rr @ rr)
    assert abs(got['err_end'] - cost_scipy) < 1e-4 * cost_scipy, (got['err_end'], cost_scipy)      # measured 7e-6: g2o's stop rule ends the run a little before the exact minimum
    assert np.abs(got['state'][:nO, 9:12] - st_s[:nO, 9:12]).max() < 2e-4 and np.abs(got['state'][:nO, :9] - st_s[:nO, :9]).max() < 2e-4
    assert np.abs(got['state'][:nO, 12:15] - st_s[:nO, 12:15]).max() < 5e-4
    res_o = O.local_inertial_ba_residuals(pr, got['tcw'], got['points'])
    tcw_s = np.array([np.concatenate([(Rcb @ st_s[k, :9].reshape(3, 3).T).reshape(9), Rcb @ (-st_s[k, :9].reshape(3, 3).T @ st_s[k, 9:12]) + tcb]) for k in range(pr['n_kf'])])
    res_s = O.local_inertial_ba_residuals(pr, tcw_s, pts_s)
    assert np.abs(res_o - res_s).max() < 0.05                      # px: two different optimisers stopped at the same minimum
