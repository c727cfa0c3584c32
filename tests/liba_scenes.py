"""Optimizer::LocalInertialBA graphs with explicit control over what `synth.local_inertial_ba_problem` leaves fixed: one camera per
keyframe (fx != fy, principal point off the image centre), any window size, any inertial-edge list (no fixed predecessor, a missing
link, none at all, listed out of chain order, either index orientation, one over a single IMU sample), any number of fixed keyframes,
exactly given observer sets, points behind a keyframe or far away, and keyframe edge lists whose lengths sit on the kernel's slice
and thread-count boundaries.

Every problem has `synth.local_inertial_ba_problem`'s keys plus `preint` [nI, 292].  Keyframes are built in time order (index k of the
window = the k-th newest, the fixed predecessor next, then the covisible fixed keyframes) and may then be renumbered.  Observations are
projections through the observing keyframe's own camera, so the problem is consistent.  Each scene asserts the counts it promises."""
import numpy as np

import lba_scenes
import oracle_lib as O
from orb_slam3_modified_b200 import synth

W, H = 640, 480
NT = 512          # threads per CTA of the LocalInertialBA kernel (csrc/liba_core.cuh)
SL = 32           # slices of a free keyframe's edge list in the kernel's pose-block and Schur phases
P_C = 67          # offset of the 15 x 15 covariance in an IMU::Preintegrated record (csrc/inertial_dev.cuh)


def graph(n_opt, n_cov=2, pred=True, observers=None, n_pts=60, obs_per_pt=3, links=None, home=None, depth=None, seed=0, renumber=False,
          renumber_fixed=False, shuffle_links=False, shuffle_edges=False, rec_init=False, large=False, single_sample=(), outlier_frac=0.03,
          noise_px=0.7, perturb=1.0, kf_dt=0.25, t_end=6.0):
    """The graph whose point j is seen by exactly the keyframes observers[j] (indices before any renumbering).  links: the inertial edges
    as (earlier, later) keyframe pairs, default the chain k+1 -> k (+ the fixed predecessor).  single_sample: indices into links whose
    interval is integrated from one IMU sample.  Point j sits at depth depth[j] (default 3..20 m) in front of keyframe home[j]."""
    rng = np.random.default_rng(seed)
    ex = synth.imu_extrinsics()
    Rcb, tcb = ex[:9].reshape(3, 3), ex[9:12]
    n_fix0 = n_opt + (1 if pred else 0)
    nkf = n_fix0 + n_cov
    times = [t_end - kf_dt * k for k in range(n_fix0)] + [t_end - kf_dt * n_fix0 - 0.4 * (j + 1) for j in range(n_cov)]
    bias = np.array([0.02, -0.01, 0.03, 0.002, -0.001, 0.0015])
    cam = lba_scenes.cameras(nkf, seed + 6000)
    truth = np.zeros((nkf, 21)); state = np.zeros((nkf, 21)); tcw = np.zeros((nkf, 12)); tcw_true = np.zeros((nkf, 12))

    def cam_pose(R, p):
        return np.concatenate([(Rcb @ R.T).reshape(9), Rcb @ (-R.T @ p) + tcb])
    for k, t in enumerate(times):
        R, p, v, _, _ = synth.imu_trajectory(t)
        truth[k] = np.concatenate([R.reshape(9), p, v, bias[3:], bias[:3]])
        tcw_true[k] = cam_pose(R, p)
        if k < n_opt:
            Rn = R @ synth._rodrigues(perturb * rng.normal(0, 0.004, 3)); pn = p + perturb * rng.normal(0, 0.01, 3)
            state[k] = np.concatenate([Rn.reshape(9), pn, v + perturb * rng.normal(0, 0.03, 3), bias[3:] + perturb * rng.normal(0, 1e-4, 3),
                                       bias[:3] + perturb * rng.normal(0, 2e-3, 3)])
        else:
            Rn, pn = R, p
            state[k] = truth[k]
        tcw[k] = cam_pose(Rn, pn)
    state = state.astype(np.float32).astype(np.float64)
    tcw = tcw.astype(np.float32).astype(np.float64)
    # points
    if observers is None:
        span = max(1, nkf - obs_per_pt + 1)
        observers = [list(range(j % span, min(nkf, j % span + obs_per_pt))) for j in range(n_pts)]
    n_pts = len(observers)
    home = [min(o) if o else 0 for o in observers] if home is None else list(home)
    depth = rng.uniform(3.0, 20.0, n_pts) if depth is None else np.asarray(depth, np.float64)
    pts = np.zeros((n_pts, 3))
    e_pt, e_kf, obs, isg = [], [], [], []
    for j, kfs in enumerate(observers):
        assert len(set(kfs)) == len(kfs) and all(0 <= k < nkf for k in kfs)
        T, c = tcw_true[home[j]], cam[home[j]].astype(np.float64)
        u, v = rng.uniform(60, W - 60), rng.uniform(60, H - 60)
        z = depth[j]
        Xc = np.array([(u - c[2]) * z / c[0], (v - c[3]) * z / c[1], z])
        pts[j] = T[:9].reshape(3, 3).T @ (Xc - T[9:])
        for k in kfs:
            T, c = tcw_true[k], cam[k].astype(np.float64)
            Xk = T[:9].reshape(3, 3) @ pts[j] + T[9:]
            octv = int(rng.integers(0, 8))
            o = np.array([c[0] * Xk[0] / Xk[2] + c[2], c[1] * Xk[1] / Xk[2] + c[3]]) + rng.normal(0, noise_px, 2) * 1.2 ** octv
            if rng.random() < outlier_frac:
                o += rng.uniform(8, 40, 2) * rng.choice([-1, 1], 2)
            e_pt.append(j); e_kf.append(k); obs.append(o); isg.append(1.0 / 1.44 ** octv)
    points = (pts + perturb * rng.normal(0, 0.02, pts.shape)).astype(np.float32).astype(np.float64)
    # inertial edges (earlier keyframe -> later keyframe)
    if links is None:
        links = [(k + 1, k) for k in range(n_fix0 - 1)]
    imu, preint = [], []
    for i, (a, b) in enumerate(links):
        assert times[a] < times[b]
        iv = synth.imu_interval(times[a], times[b], rate=1.0 if i in single_sample else 300.0, seed=seed * 100 + i, bias=tuple(bias))
        assert (len(iv[2]) == 1) == (i in single_sample)
        imu.append(iv)
        preint.append(O.imu_preintegrate(*iv, bias.astype(np.float32), synth.IMU_NOISE))
    to_fixed = [a >= n_opt or b >= n_opt for a, b in links]
    pr = dict(n_kf=nkf, n_opt=n_opt, state=state, tcw=tcw, cam=cam, extr=ex,
              ie_kf1=np.array([a for a, b in links], np.int32).reshape(-1), ie_kf2=np.array([b for a, b in links], np.int32).reshape(-1),
              imu=imu, bias6=bias.astype(np.float32), preint=np.array(preint, np.float32).reshape(len(links), 292),
              ie_robust=np.array([1 if (f or rec_init) else 0 for f in to_fixed], np.uint8).reshape(-1),
              ie_info_scale=np.array([1e-2 if f else 1.0 for f in to_fixed]).reshape(-1),
              points=points.reshape(-1, 3), track_depth=np.abs(depth).astype(np.float32), e_pt=np.array(e_pt, np.int32), e_kf=np.array(e_kf, np.int32),
              obs=np.array(obs, np.float64).reshape(-1, 2).astype(np.float32).astype(np.float64), inv_sigma2=np.array(isg, np.float32),
              iterations=4 if large else 10, lambda_init=1e-2 if large else 1.0, large=bool(large), truth=truth, points_true=pts, times=np.array(times))
    # renumbering: the window's and / or the fixed keyframes' indices permuted within their ranges
    perm = np.arange(nkf)
    if renumber:
        perm[:n_opt] = rng.permutation(n_opt)
    if renumber_fixed:
        perm[n_opt:] = n_opt + rng.permutation(nkf - n_opt)
    if renumber or renumber_fixed:
        inv = np.argsort(perm)
        for key in ('state', 'tcw', 'cam', 'truth', 'times'):
            pr[key] = np.ascontiguousarray(pr[key][inv])
        for key in ('e_kf', 'ie_kf1', 'ie_kf2'):
            pr[key] = perm[pr[key]].astype(np.int32)
    if shuffle_links:
        o = rng.permutation(len(links))
        for key in ('ie_kf1', 'ie_kf2', 'preint', 'ie_robust', 'ie_info_scale'):
            pr[key] = np.ascontiguousarray(pr[key][o])
        pr['imu'] = [pr['imu'][i] for i in o]
    if shuffle_edges:
        o = rng.permutation(len(pr['e_pt']))
        for key in ('e_pt', 'e_kf', 'obs', 'inv_sigma2'):
            pr[key] = np.ascontiguousarray(pr[key][o])
    return pr


def free_edge_counts(pr):
    return np.bincount(pr['e_kf'][pr['e_kf'] < pr['n_opt']], minlength=pr['n_opt'])


def window(n_opt, n_cov=2, n_pts=None, seed=0, **kw):
    """Sliding observer windows of three over all keyframes."""
    pr = graph(n_opt, n_cov=n_cov, n_pts=n_pts or max(40, 6 * (n_opt + 1 + n_cov)), seed=seed, **kw)
    assert len(pr['ie_kf1']) == n_opt and free_edge_counts(pr).min() > 0
    return pr


def no_fixed_predecessor(n_opt=8, seed=0):
    pr = graph(n_opt, n_cov=2, pred=False, n_pts=70, seed=seed)
    # no inertial link reaches a fixed keyframe: the accelerometer biases are held by lambda and the random walk alone, and after 10
    # iterations the H100's fused multiply-adds and the oracle's rounding part by 5e-5 in lambda; the parity checks stop at 5
    pr['iterations'] = 5
    assert len(pr['ie_kf1']) == n_opt - 1 and (pr['ie_kf1'] < n_opt).all() and (pr['ie_kf2'] < n_opt).all()
    return pr


def missing_link(n_opt=8, seed=0):
    """The chain without the edge 5 -> 4: the window splits into two inertial chains, only the older one reaches the predecessor."""
    links = [(k + 1, k) for k in range(n_opt) if k != n_opt // 2]
    pr = graph(n_opt, n_cov=2, links=links, n_pts=70, seed=seed)
    # the newer chain's accelerometer biases are held by lambda and the random walk alone: after 10 iterations two summation orders part by
    # 1.3e-7 in the states, so the parity checks stop at 5 (1e-10)
    pr['iterations'] = 5
    assert len(pr['ie_kf1']) == n_opt - 1 and not ((pr['ie_kf1'] == n_opt // 2 + 1) & (pr['ie_kf2'] == n_opt // 2)).any()
    return pr


def no_inertial(n_opt=6, seed=0):
    pr = graph(n_opt, n_cov=2, links=[], n_pts=60, seed=seed)
    assert len(pr['ie_kf1']) == 0 and pr['preint'].shape == (0, 292)
    return pr


def links_out_of_order(n_opt=9, seed=0):
    pr = graph(n_opt, n_cov=2, n_pts=70, seed=seed, shuffle_links=True)
    assert not (np.diff(pr['ie_kf2']) > 0).all() and not (np.diff(pr['ie_kf2']) < 0).all()
    return pr


def mixed_orientation(n_opt=9, seed=0):
    """The window renumbered: inertial edges with ieKf1 > ieKf2 and with ieKf1 < ieKf2 in index terms."""
    pr = graph(n_opt, n_cov=2, n_pts=70, seed=seed, renumber=True)
    assert (pr['ie_kf1'] > pr['ie_kf2']).any() and (pr['ie_kf1'] < pr['ie_kf2']).any()
    return pr


def rec_init(n_opt=6, seed=0):
    pr = graph(n_opt, n_cov=2, n_pts=60, seed=seed, rec_init=True)
    assert pr['ie_robust'].all()
    return pr


def no_fixed(n_opt=6, seed=0):
    pr = graph(n_opt, n_cov=0, pred=False, n_pts=60, seed=seed)
    # nothing fixes the gauge (position and yaw): lambda alone holds that null space, and two summation orders drift apart along it
    # (1.3e-8 after two iterations, 4.7e-4 after ten); the parity checks run one iteration (every phase, 9e-10)
    pr['iterations'] = 1
    assert pr['n_kf'] == pr['n_opt']
    return pr


def fixed_200(n_opt=10, n_cov=200, seed=0):
    """200 covisible fixed keyframes (the reference's maxFixKF) that only see points: every point is seen by two keyframes of the
    window and by two of the fixed ones, round robin, so each fixed keyframe sees at least one point."""
    rng = np.random.default_rng(seed)
    nkf = n_opt + 1 + n_cov
    obs = []
    for j in range(n_cov):
        w = sorted(rng.choice(n_opt + 1, 2, replace=False).tolist())
        obs.append(w + [n_opt + 1 + j, n_opt + 1 + (j + 97) % n_cov])
    pr = graph(n_opt, n_cov=n_cov, observers=obs, seed=seed)
    cnt = np.bincount(pr['e_kf'], minlength=nkf)
    assert (cnt[n_opt + 1:] > 0).all() and pr['n_kf'] - pr['n_opt'] == n_cov + 1
    return pr


def fixed_interleaved(n_opt=7, seed=0):
    """Fixed keyframes renumbered and the edge list shuffled: edges of fixed and free keyframes alternate, and a point's edges are
    scattered over the list."""
    pr = graph(n_opt, n_cov=4, n_pts=80, obs_per_pt=4, seed=seed, renumber_fixed=True, shuffle_edges=True)
    fixed = pr['e_kf'] >= n_opt
    assert (np.diff(fixed.astype(int)) != 0).sum() > 20 and not (np.diff(pr['e_pt']) >= 0).all()
    return pr


def observers(n_opt=6, seed=0):
    """Points seen once (by a free and by a fixed keyframe), points seen only by fixed keyframes, points seen by every window keyframe,
    points behind a free keyframe (negative depth), points ~500 m away, and points whose trackDepth is exactly 10.0f (the bClose
    boundary) with one noise-free observation planted 3.0 .. 4.5 px off, so that its final chi2 lands between 5.991 and 1.5 * 5.991."""
    nkf = n_opt + 3
    fx = [n_opt, n_opt + 1, n_opt + 2]
    obs, home, depth = [], [], []
    rng = np.random.default_rng(seed + 17)

    def add(o, d=None, h=None):
        obs.append(o); home.append(min(o) if h is None else h); depth.append(rng.uniform(3, 20) if d is None else d)
    for k in range(n_opt):
        add([k])                                         # seen once by a free keyframe
    add([fx[0]]); add([fx[2]])                           # seen once by a fixed keyframe
    for _ in range(6):
        add([fx[1], fx[2]])                              # fixed keyframes only
    for _ in range(3):
        add(list(range(n_opt)))                          # every window keyframe
    for _ in range(4):
        add([0, 1, fx[0]], d=-rng.uniform(3, 6))         # behind the window's newest keyframes
    for _ in range(4):
        add([1, 3, fx[1]], d=rng.uniform(480, 520))      # ~500 m away
    boundary = len(obs)
    for _ in range(16):
        add([0, 2, 4, fx[2]], d=10.0)                    # trackDepth == 10.0f
    for j in range(40):
        k = j % n_opt
        add(sorted({k, (k + 1) % n_opt, fx[j % 3]}))
    pr = graph(n_opt, n_cov=2, observers=obs, home=home, depth=depth, seed=seed, outlier_frac=0.0)
    # plant the boundary residuals: noise-free octave-0 observations of keyframe 2, shifted in x
    ex = pr['extr']; Rcb, tcb = ex[:9].reshape(3, 3), ex[9:12]
    R, p = pr['truth'][2, :9].reshape(3, 3), pr['truth'][2, 9:12]
    c = pr['cam'][2].astype(np.float64)
    for j in range(boundary, boundary + 16):
        e = np.flatnonzero((pr['e_pt'] == j) & (pr['e_kf'] == 2))[0]
        Xc = Rcb @ (R.T @ (pr['points_true'][j] - p)) + tcb
        pr['inv_sigma2'][e] = 1.0
        pr['obs'][e] = np.float32([c[0] * Xc[0] / Xc[2] + c[2] + 3.0 + 1.5 * (j - boundary) / 15, c[1] * Xc[1] / Xc[2] + c[3]])
    assert nkf == pr['n_kf']
    n_obs = np.bincount(pr['e_pt'], minlength=len(obs))
    assert (n_obs == 1).sum() == n_opt + 2 and (pr['track_depth'] == np.float32(10.0)).sum() == 16
    z = np.array([(pr['tcw'][k, 6:9] @ pr['points'][j] + pr['tcw'][k, 11]) for j, k in zip(pr['e_pt'], pr['e_kf'])])
    assert (z < 0).sum() >= 8 and (z > 400).sum() >= 8
    return pr


def edge_list_lengths(counts=(0, 1, 31, 32, 33, 65, 4), seed=0):
    """Free keyframe k sees exactly counts[k] points, each also seen by the fixed predecessor and one covisible fixed keyframe: edge
    lists that end before, on and after one and two multiples of SL, and a free keyframe with no mono edge at all."""
    n_opt = len(counts)
    obs = [[k, n_opt, n_opt + 1 + (j % 2)] for k, c in enumerate(counts) for j in range(c)]
    pr = graph(n_opt, n_cov=2, observers=obs, seed=seed)
    assert free_edge_counts(pr).tolist() == list(counts)
    return pr


def n_edges(n_e, seed=0):
    """Exactly n_e mono edges (0: no points at all); points with three observers, the last one with one to three."""
    n_opt = 6
    nkf = n_opt + 3
    obs = []
    while sum(map(len, obs)) + 3 < n_e:
        j = len(obs)
        obs.append(sorted({j % nkf, (j + 2) % nkf, (j + 5) % nkf}))
    rest = n_e - sum(map(len, obs))
    if rest:
        obs.append(list(range(rest)))
    pr = graph(n_opt, n_cov=2, observers=obs, seed=seed)
    if n_e <= 1:
        # without (almost) any mono edge the cost falls to 1e-22 and later accept / reject decisions compare rounding noise: 4 iterations
        pr['iterations'] = 4
    assert len(pr['e_pt']) == n_e and len(pr['points']) == len(obs)
    return pr


def single_imu_sample(n_opt=5, seed=24):
    """The inertial edge 3 -> 2 integrated from one IMU sample: its 9 x 9 covariance is exactly singular (dP's rows are 0.5 dt times dV's),
    so the information matrix takes the Jacobi path, on a non-finite inverse: the reference's PartialPivLU divides by the zero pivot.  The
    information is NaN, so is err, and the FAIL test fires."""
    pr = graph(n_opt, n_cov=2, n_pts=60, seed=seed, single_sample=(2,))
    assert len(pr['imu'][2][2]) == 1
    return pr


def indefinite_covariance(n_opt=5, seed=0):
    """The covariance of inertial edge 2 given one slightly negative eigenvalue (-0.5 x its smallest one): it inverts, but the inverse is
    not positive definite, so the information matrix takes the Jacobi path, which clamps that eigenvalue to zero -- a finite information
    matrix of rank 8."""
    pr = graph(n_opt, n_cov=2, n_pts=60, seed=seed)
    C15 = pr['preint'][2, P_C:P_C + 225].reshape(15, 15)
    w, V = np.linalg.eigh(C15[:9, :9].astype(np.float64))
    w[0] *= -0.5
    C15[:9, :9] = ((V * w) @ V.T).astype(np.float32)
    C15[:9, :9] = (C15[:9, :9] + C15[:9, :9].T) / 2
    pr['preint'][2, P_C:P_C + 225] = C15.reshape(-1)
    assert np.linalg.eigvalsh(C15[:9, :9].astype(np.float64))[0] < 0
    return pr


def nan_observation():
    """synth's seed-33 map with one NaN observation: err is NaN, so the FAIL test fires."""
    pr = synth.local_inertial_ba_problem(n_opt=4, n_cov_fixed=1, n_pts=120, seed=33)
    pr['obs'][5, 0] = np.nan
    pr['preint'] = O.liba_preints(pr)
    return pr


def finite_fail(seed=107):
    """A FAIL with finite errors: the ground-truth window with one to three points pulled to 1 .. 10 % of their distance from a camera
    that sees them, and lambda_init = 1e-300.  The undamped first step overshoots; every retry repeats it (lambda * 2^45 is still
    negligible), and after maxTrials rejections the edges hold the errors of the rejected state: err_end > 2 err, both finite."""
    rng = np.random.default_rng(seed)
    pr = graph(3, n_cov=2, n_pts=40, obs_per_pt=3, seed=seed, perturb=0.0, outlier_frac=0.0, noise_px=0.3)
    pr['lambda_init'] = 1e-300
    for j in rng.choice(len(pr['points']), 1 + seed % 3, replace=False):
        T = pr['tcw'][pr['e_kf'][pr['e_pt'] == j][0]]
        c = -T[:9].reshape(3, 3).T @ T[9:]
        pr['points'][j] = c + (pr['points'][j] - c) * rng.uniform(0.01, 0.1) + rng.normal(0, 0.02, 3)
    return pr


LAYOUTS = {
    'window_1': lambda: window(1, n_cov=2, seed=1),
    'window_2': lambda: window(2, n_cov=1, seed=2),
    'window_10': lambda: window(10, n_cov=3, seed=3),
    'window_25_large': lambda: window(25, n_cov=4, n_pts=240, seed=4, large=True),
    'window_34': lambda: window(34, n_cov=2, n_pts=230, seed=5),
    'window_35': lambda: window(35, n_cov=2, n_pts=230, seed=6),
    'window_64': lambda: window(64, n_cov=2, n_pts=420, seed=7),
    'no_fixed_predecessor': lambda: no_fixed_predecessor(seed=8),
    'missing_link': lambda: missing_link(seed=9),
    'no_inertial': lambda: no_inertial(seed=10),
    'links_out_of_order': lambda: links_out_of_order(seed=11),
    'mixed_orientation': lambda: mixed_orientation(seed=12),
    'rec_init': lambda: rec_init(seed=13),
    'no_fixed': lambda: no_fixed(seed=14),
    'fixed_200': lambda: fixed_200(seed=15),
    'fixed_interleaved': lambda: fixed_interleaved(seed=16),
    'observers': lambda: observers(seed=17),
    'edge_list_lengths': lambda: edge_list_lengths(seed=18),
    'n_edges_0': lambda: n_edges(0, seed=19),
    'n_edges_1': lambda: n_edges(1, seed=20),
    'n_edges_511': lambda: n_edges(511, seed=21),
    'n_edges_512': lambda: n_edges(512, seed=22),
    'n_edges_513': lambda: n_edges(513, seed=23),
    'indefinite_covariance': lambda: indefinite_covariance(seed=24),
}
SLOW = ('window_64', 'fixed_200')
