"""CPU: the inertial oracle (oracle/inertial_oracle.cpp) is pinned by independent derivations, since G2oTypes / ImuTypes need Eigen
and cannot be compiled into oracle/_ref:
  * the analytic Jacobians of EdgeInertial::linearizeOplus and EdgeMono::linearizeOplus equal numerical derivatives of the residuals
    under the reference's own update rules (ImuCamPose::Update for poses, additive for velocity / biases / points);
  * preintegration of noise-free IMU data of an analytic trajectory reproduces the trajectory's relative motion, and the
    EdgeInertial residual vanishes at the ground truth;
  * NormalizeRotation returns the polar factor (checked against numpy's SVD), Exp / Log / Jr / Jr^-1 satisfy their identities;
  * the information matrix is the symmetric inverse of the covariance."""
import numpy as np

import oracle_lib as O
from orb_slam3_modified_b200 import synth


def test_so3_helpers():
    rng = np.random.default_rng(0)
    for _ in range(50):
        w = rng.normal(0, 0.8, 3)
        R = O.so3('exp', w)
        assert np.allclose(R @ R.T, np.eye(3), atol=1e-12) and np.isclose(np.linalg.det(R), 1)
        assert np.allclose(O.so3('log', R), w, atol=1e-9)
        assert np.allclose(O.so3('Jr', w) @ O.so3('invJr', w), np.eye(3), atol=1e-9)
        M = R + rng.normal(0, 1e-3, (3, 3))
        U, _, Vt = np.linalg.svd(M)
        assert np.allclose(O.so3('normalize', M), U @ Vt, atol=1e-12)
        d = rng.normal(0, 1e-6, 3)     # Exp(w + d) ~ Exp(w) Exp(Jr(w) d)
        assert np.allclose(O.so3('exp', w + d), R @ O.so3('exp', O.so3('Jr', w) @ d), atol=1e-10)


def test_preintegration_reproduces_the_trajectory():
    t0, t1 = 1.0, 1.0 + 1.0 / 3
    bias = (0.02, -0.01, 0.03, 0.002, -0.001, 0.0015)
    acc, gyr, dts = synth.imu_interval(t0, t1, rate=3000.0, bias=bias, noise=False)
    P = O.imu_preintegrate(acc, gyr, dts, bias, synth.IMU_NOISE)
    R1, p1, v1, _, _ = synth.imu_trajectory(t0)
    R2, p2, v2, _, _ = synth.imu_trajectory(t1)
    dt = float(P[0])
    g = np.array([0, 0, -9.81])
    dR, dV, dP = O.imu_delta(P, bias[3:], bias[:3])
    assert np.isclose(dt, t1 - t0, atol=1e-5)
    assert np.allclose(dR, R1.T @ R2, atol=2e-5)
    assert np.allclose(dV, R1.T @ (v2 - v1 - g * dt), atol=2e-4)
    assert np.allclose(dP, R1.T @ (p2 - p1 - v1 * dt - 0.5 * g * dt * dt), atol=1e-4)
    s = synth.inertial_edge_state(t0, t1, perturb=0.0)
    err, _ = O.imu_edge_inertial(P, s)
    assert np.abs(err).max() < 5e-4
    info, ig, ia = O.imu_information(P)
    C9 = P[67:].reshape(15, 15)[:9, :9].astype(np.float64)
    ni = np.linalg.inv(C9); ni = (ni + ni.T) / 2
    assert np.allclose(info, info.T) and np.abs(info - ni).max() < 1e-6 * np.abs(ni).max() and np.linalg.eigvalsh(info).min() > 0
    assert np.allclose(ig @ P[67:].reshape(15, 15)[9:12, 9:12].astype(np.float64), np.eye(3), atol=1e-9)


def _numeric_jacobian_inertial(P, s, h_state=1e-6, h_bias=2e-3):
    J = np.zeros((9, 24))
    e0, _ = O.imu_edge_inertial(P, s, jac=False)

    def col(k, sp, sm, h):
        ep, _ = O.imu_edge_inertial(P, sp, jac=False)
        em, _ = O.imu_edge_inertial(P, sm, jac=False)
        J[:, k] = (ep - em) / (2 * h)
    for which, c0 in (('1', 0), ('2', 15)):
        for k in range(6):
            pu = np.zeros(6); pu[k] = h_state
            sp, sm = dict(s), dict(s)
            sp['Rwb' + which], sp['twb' + which] = O.imu_pose_update(s['Rwb' + which], s['twb' + which], pu)
            sm['Rwb' + which], sm['twb' + which] = O.imu_pose_update(s['Rwb' + which], s['twb' + which], -pu)
            col(c0 + k, sp, sm, h_state)
    for name, c0, h in (('v1', 6, h_state), ('bg', 9, h_bias), ('ba', 12, h_bias), ('v2', 21, h_state)):
        for k in range(3):
            d = np.zeros(3); d[k] = h
            sp, sm = dict(s), dict(s)
            sp[name] = s[name] + d; sm[name] = s[name] - d
            col(c0 + k, sp, sm, h)
    return J


def test_edge_inertial_jacobians_equal_numeric_derivatives():
    for seed in range(4):
        t0 = 0.5 + seed
        acc, gyr, dts = synth.imu_interval(t0, t0 + 0.4, seed=seed)
        P = O.imu_preintegrate(acc, gyr, dts, (0.02, -0.01, 0.03, 0.002, -0.001, 0.0015), synth.IMU_NOISE)
        s = synth.inertial_edge_state(t0, t0 + 0.4, seed=seed)
        err, J = O.imu_edge_inertial(P, s)
        Jn = _numeric_jacobian_inertial(P, s)
        exact = [c for c in range(24) if not 9 <= c < 15]
        assert np.abs(J[:, exact] - Jn[:, exact]).max() < 2e-6, np.abs(J[:, exact] - Jn[:, exact]).max()
        # bias columns: the preintegrated terms are float32 and first order in the bias change -> looser
        assert np.abs(J[:, 9:15] - Jn[:, 9:15]).max() < 5e-3 * max(1.0, np.abs(J[:, 9:15]).max()), np.abs(J[:, 9:15] - Jn[:, 9:15]).max()


def test_edge_mono_jacobians_equal_numeric_derivatives():
    rng = np.random.default_rng(3)
    for _ in range(5):
        Rwb = O.so3('exp', rng.normal(0, 0.4, 3)); twb = rng.normal(0, 1, 3)
        Rbc = O.so3('exp', rng.normal(0, 0.3, 3)); tbc = rng.normal(0, 0.1, 3)
        Rcb = Rbc.T; tcb = -Rcb @ tbc
        cam = np.array([458.0, 457.0, 367.0, 248.0], np.float32)
        Xc = np.array([rng.uniform(-1, 1), rng.uniform(-0.7, 0.7), rng.uniform(2, 8)])
        Xw = Rwb @ (Rbc @ Xc + tbc) + twb
        obs = np.array([cam[0] * Xc[0] / Xc[2] + cam[2], cam[1] * Xc[1] / Xc[2] + cam[3]]) + rng.normal(0, 1.0, 2)
        err, Jp, Jx, dp = O.imu_edge_mono(Rwb, twb, Rcb, tcb, Rbc, tbc, cam, Xw, obs)
        assert dp and np.abs(err).max() < 6
        h = 1e-6
        for k in range(3):
            d = np.zeros(3); d[k] = h
            ep = O.imu_edge_mono(Rwb, twb, Rcb, tcb, Rbc, tbc, cam, Xw + d, obs, jac=False)[0]
            em = O.imu_edge_mono(Rwb, twb, Rcb, tcb, Rbc, tbc, cam, Xw - d, obs, jac=False)[0]
            assert np.allclose((ep - em) / (2 * h), Jp[:, k], rtol=1e-5, atol=1e-5)
        for k in range(6):
            pu = np.zeros(6); pu[k] = h
            Rp, tp = O.imu_pose_update(Rwb, twb, pu)
            Rm, tm = O.imu_pose_update(Rwb, twb, -pu)
            ep = O.imu_edge_mono(Rp, tp, Rcb, tcb, Rbc, tbc, cam, Xw, obs, jac=False)[0]
            em = O.imu_edge_mono(Rm, tm, Rcb, tcb, Rbc, tbc, cam, Xw, obs, jac=False)[0]
            assert np.allclose((ep - em) / (2 * h), Jx[:, k], rtol=1e-5, atol=1e-4)


# ---- Optimizer::PoseInertialOptimizationLastKeyFrame (src/Optimizer.cc:4491-4873): oracle properties ----
def _log(R):
    c = (np.trace(R) - 1) / 2
    th = np.arccos(np.clip(c, -1, 1))
    v = np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]]) / 2
    return v if th < 1e-9 else v * th / np.sin(th)


def _pose_err(a, b):
    Ra, Rb = a[:9].reshape(3, 3), b[:9].reshape(3, 3)
    return np.linalg.norm(_log(Ra.T @ Rb)), np.linalg.norm(a[9:12] - b[9:12]), np.linalg.norm(a[12:15] - b[12:15])


def test_pose_inertial_opt_recovers_the_state_and_rejects_outliers():
    for seed in range(4):
        pr = synth.pose_inertial_problem(seed=seed, n=300, outlier_frac=0.1)
        P = O.imu_preintegrate(pr['acc'], pr['gyr'], pr['dt'], pr['bias6'], synth.IMU_NOISE)
        r = O.pose_inertial_opt_last_kf(pr, P)
        e0, e1 = _pose_err(pr['state'], pr['truth']), _pose_err(r['state'], pr['truth'])
        assert e1[0] < 2e-3 and e1[1] < 6e-3 and e1[0] < e0[0] and e1[1] < e0[1], (seed, e0, e1)
        # every gross outlier is flagged, few inliers are
        assert r['outlier'][pr['gross']].mean() > 0.95 and r['outlier'][~pr['gross']].mean() < 0.08
        assert r['ret'] == len(pr['Xw']) - int(r['outlier'].sum())
        # biases stay at the keyframe's (the random-walk edges are the only edges on them)
        assert np.allclose(r['state'][15:21], pr['kf_state'][15:21], atol=1e-9)
        H = r['H']
        assert np.allclose(H, H.T, rtol=1e-9, atol=1e-6 * np.abs(H).max()) and np.linalg.eigvalsh((H + H.T) / 2).min() > -1e-6 * np.abs(H).max()


def test_pose_inertial_opt_noise_free_fixed_point():
    """Exact observations, exact IMU, start at the truth: the estimate stays (the inertial residual of a 300 Hz midpoint integration is tiny) and
    nothing is an outlier; with fewer than 7 points the rounds stop after the first (edges().size() < 10)."""
    pr = synth.pose_inertial_problem(seed=3, n=200, outlier_frac=0.0, perturb=0.0, noise_px=0.0)
    acc, gyr, dts = synth.imu_interval(1.0, 1.2, seed=3, bias=tuple(pr['bias6']), noise=False)
    P = O.imu_preintegrate(acc, gyr, dts, pr['bias6'], synth.IMU_NOISE)
    r = O.pose_inertial_opt_last_kf(pr, P)
    e = _pose_err(r['state'], pr['truth'])
    assert e[0] < 2e-4 and e[1] < 1e-3 and r['outlier'].sum() == 0 and r['ret'] == 200
    few = {k: (v[:5] if k in ('Xw', 'obs', 'inv_sigma2', 'track_depth', 'gross') else v) for k, v in pr.items()}
    r5 = O.pose_inertial_opt_last_kf(few, P)
    assert r5['ret'] == 5 and np.isfinite(r5['state']).all()


def check_first_step_last_kf(pr, P):
    """One Gauss-Newton step of the oracle = the dense normal-equation step built from NUMERICAL derivatives of the stacked, whitened residuals
    (mono edges without robust weight: inliers only, inertial edge, random-walk edges) under ImuCamPose::Update.  For a frame where no
    Huber weight is active at the start."""
    info9, ig, ia = O.imu_information(P)
    ex = pr['extr']

    def apply(s, dx):
        s = s.copy()
        R, t = O.imu_pose_update(s[:9].reshape(3, 3), s[9:12], dx[:6])
        s[:9] = R.reshape(9); s[9:12] = t; s[12:15] += dx[6:9]; s[15:18] += dx[9:12]; s[18:21] += dx[12:15]
        return s

    def residuals(s):
        out = []
        for i in range(len(pr['Xw'])):
            e = O.imu_edge_mono(s[:9].reshape(3, 3), s[9:12], ex[:9], ex[9:12], ex[12:21], ex[21:24], pr['cam'], pr['Xw'][i].astype(np.float64),
                                pr['obs'][i].astype(np.float64), jac=False)[0]
            out.append(np.sqrt(float(pr['inv_sigma2'][i])) * e)
        k = pr['kf_state']
        e9 = O.imu_edge_inertial(P, dict(Rwb1=k[:9].reshape(3, 3), twb1=k[9:12], v1=k[12:15], bg=k[15:18], ba=k[18:21], Rwb2=s[:9].reshape(3, 3), twb2=s[9:12], v2=s[12:15]),
                                 jac=False)[0]
        Lc = np.linalg.cholesky(info9 + 1e-18 * np.eye(9))
        out.append(Lc.T @ e9)
        out.append(np.linalg.cholesky(ig).T @ (s[15:18] - k[15:18]))
        out.append(np.linalg.cholesky(ia).T @ (s[18:21] - k[18:21]))
        return np.concatenate(out)
    s0 = pr['state']
    r0 = residuals(s0)
    assert (r0[:2 * len(pr['Xw'])].reshape(-1, 2) ** 2).sum(1).max(initial=0.0) < 5.99      # no Huber weight at the linearisation point
    J = np.zeros((len(r0), 15))
    for k in range(15):
        h = 1e-6
        d = np.zeros(15); d[k] = h
        J[:, k] = (residuals(apply(s0, d)) - residuals(apply(s0, -d))) / (2 * h)
    dx = np.linalg.solve(J.T @ J, -J.T @ r0)
    want = apply(s0, dx)
    # the oracle with ONE iteration: emulate by comparing against its first update through a 1-iteration copy (huge Huber never active at this noise level)
    got = O.pose_inertial_opt_one_step(pr, P)
    assert np.allclose(got, want, rtol=0, atol=2e-6), np.abs(got - want).max()


def test_pose_inertial_opt_first_step_is_the_gauss_newton_step():
    pr = synth.pose_inertial_problem(seed=5, n=60, outlier_frac=0.0, perturb=0.05, noise_px=0.2)
    check_first_step_last_kf(pr, O.imu_preintegrate(pr['acc'], pr['gyr'], pr['dt'], pr['bias6'], synth.IMU_NOISE))


# ---- Optimizer::PoseInertialOptimizationLastFrame (src/Optimizer.cc:4875-5289) ----
def _preints(pr):
    return (O.imu_preintegrate(pr['acc'], pr['gyr'], pr['dt'], pr['bias6'], synth.IMU_NOISE),
            O.imu_preintegrate(pr['acc_kf'], pr['gyr_kf'], pr['dt_kf'], pr['bias6'], synth.IMU_NOISE))


def test_pose_inertial_opt_last_frame_recovers_the_state():
    for seed in range(3):
        pr = synth.pose_inertial_problem_last_frame(seed=seed, n=300, outlier_frac=0.1)
        Pf, Pk = _preints(pr)
        r = O.pose_inertial_opt_last_frame(pr, Pf, Pk)
        e0, e1 = _pose_err(pr['state'], pr['truth']), _pose_err(r['state'], pr['truth'])
        assert e1[0] < 2e-3 and e1[1] < 8e-3 and e1[0] < e0[0] and e1[1] < e0[1], (seed, e0, e1)
        assert r['outlier'][pr['gross']].mean() > 0.95 and r['outlier'][~pr['gross']].mean() < 0.08 and r['ret'] == len(pr['Xw']) - int(r['outlier'].sum())
        ep = _pose_err(r['prev_state'], pr['truth_prev'])
        assert ep[0] < 6e-3 and ep[1] < 2e-2
        H = r['H']
        assert np.allclose(H, H.T, rtol=1e-8, atol=1e-7 * np.abs(H).max()) and np.linalg.eigvalsh((H + H.T) / 2).min() > -1e-6 * np.abs(H).max()
        C2 = O.constraint_pose_imu_information(H)              # ConstraintPoseImu's constructor: symmetric, no negative eigenvalues, equal to H here
        assert np.allclose(C2, (H + H.T) / 2, rtol=1e-8, atol=1e-8 * np.abs(H).max())


def test_pose_inertial_opt_last_frame_with_a_rigid_prior_is_the_last_keyframe_variant():
    """A prior so strong that the previous frame cannot move, at the previous frame's own state: the frame's result and the marginalised
    Hessian must be those of PoseInertialOptimizationLastKeyFrame with the previous frame as the fixed keyframe."""
    pr = synth.pose_inertial_problem_last_frame(seed=4, n=250, outlier_frac=0.1)
    Pf, _ = _preints(pr)
    pr['prior_state'] = pr['kf_state'].copy(); pr['prev_state'] = pr['kf_state'].copy(); pr['prior_H'] = 1e16 * np.eye(15)
    a = O.pose_inertial_opt_last_frame(pr, Pf, Pf)
    b = O.pose_inertial_opt_last_kf(pr, Pf)
    assert np.array_equal(a['outlier'], b['outlier']) and a['ret'] == b['ret']
    assert np.abs(a['state'] - b['state']).max() < 1e-7 and np.abs(a['prev_state'] - pr['kf_state']).max() < 1e-9
    assert np.abs(a['H'] - b['H']).max() < 1e-4 * np.abs(b['H']).max()          # H_cc - H_cb H_bb^-1 H_bc with H_bb ~ 1e16


def check_first_step_last_frame(pr, Pf, Pk):
    """As check_first_step_last_kf over the 30 unknowns of the frame and the previous frame, with the prior edge."""
    info9 = O.imu_information(Pf)[0]; _, ig, ia = O.imu_information(Pk)
    ex = pr['extr']
    Lp = np.linalg.cholesky(pr['prior_H'])

    def apply(s, dx):
        s = s.copy()
        R, t = O.imu_pose_update(s[:9].reshape(3, 3), s[9:12], dx[:6])
        s[:9] = R.reshape(9); s[9:12] = t; s[12:15] += dx[6:9]; s[15:18] += dx[9:12]; s[18:21] += dx[12:15]
        return s

    def residuals(sc, sp):
        out = []
        for i in range(len(pr['Xw'])):
            e = O.imu_edge_mono(sc[:9].reshape(3, 3), sc[9:12], ex[:9], ex[9:12], ex[12:21], ex[21:24], pr['cam'], pr['Xw'][i].astype(np.float64),
                                pr['obs'][i].astype(np.float64), jac=False)[0]
            out.append(np.sqrt(float(pr['inv_sigma2'][i])) * e)
        e9 = O.imu_edge_inertial(Pf, dict(Rwb1=sp[:9].reshape(3, 3), twb1=sp[9:12], v1=sp[12:15], bg=sp[15:18], ba=sp[18:21], Rwb2=sc[:9].reshape(3, 3), twb2=sc[9:12], v2=sc[12:15]),
                                 jac=False)[0]
        out.append(np.linalg.cholesky(info9 + 1e-18 * np.eye(9)).T @ e9)
        out.append(np.linalg.cholesky(ig).T @ (sc[15:18] - sp[15:18]))
        out.append(np.linalg.cholesky(ia).T @ (sc[18:21] - sp[18:21]))
        q = pr['prior_state']
        Rp = q[:9].reshape(3, 3)
        e15 = np.concatenate([_log(Rp.T @ sp[:9].reshape(3, 3)), Rp.T @ (sp[9:12] - q[9:12]), sp[12:15] - q[12:15], sp[15:18] - q[15:18], sp[18:21] - q[18:21]])
        chi2_prior.append(float(e15 @ pr['prior_H'] @ e15))
        out.append(Lp.T @ e15)
        return np.concatenate(out)
    chi2_prior = []
    c0, p0 = pr['state'], pr['prev_state']
    r0 = residuals(c0, p0)
    assert chi2_prior[0] < 25.0 and (r0[:2 * len(pr['Xw'])].reshape(-1, 2) ** 2).sum(1).max(initial=0.0) < 5.99      # no Huber weight at the linearisation point
    J = np.zeros((len(r0), 30))
    for k in range(30):
        h = 2e-3 if k % 15 >= 9 else 1e-6      # the preintegration applies bias changes in float (src/ImuTypes.cc:283-307): a bias step must stand out of its rounding
        d = np.zeros(30); d[k] = h
        J[:, k] = (residuals(apply(c0, d[:15]), apply(p0, d[15:])) - residuals(apply(c0, -d[:15]), apply(p0, -d[15:]))) / (2 * h)
    dx = np.linalg.solve(J.T @ J, -J.T @ r0)
    got = O.pose_inertial_opt_last_frame(pr, Pf, Pk, rounds=1, iters=1)
    assert np.allclose(got['state'], apply(c0, dx[:15]), rtol=0, atol=3e-6), np.abs(got['state'] - apply(c0, dx[:15])).max()
    assert np.allclose(got['prev_state'], apply(p0, dx[15:]), rtol=0, atol=3e-6), np.abs(got['prev_state'] - apply(p0, dx[15:])).max()


def test_pose_inertial_opt_last_frame_first_step_is_the_gauss_newton_step():
    pr = synth.pose_inertial_problem_last_frame(seed=6, n=50, outlier_frac=0.0, perturb=0.05, noise_px=0.2)
    check_first_step_last_frame(pr, *_preints(pr))
