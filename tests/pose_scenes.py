"""Frames for the tracking pose optimisers -- Optimizer::PoseOptimization (one CTA of NT threads per frame, csrc/pose_opt.cu) and
PoseInertialOptimizationLastKeyFrame / LastFrame (one CTA of PI_NT threads, csrc/inertial.cu) -- that reach the branches a synthetic
frame with random noise rarely reaches: the early return and the `edges().size() < 10` break, edge counts around the thread counts,
frames whose every observation is a gross outlier, a noise-free frame at its true pose, a start bad enough to exhaust the
Levenberg-Marquardt trials, points behind the camera or 500 m away, observations on the image border, a non-unit quaternion, the
`nInliers < 30` recovery, the trackDepth == 10 close rule and a prior whose Huber kernel is active.

Built on `synth.pose_opt_problem` / `lba_scenes.pose_opt_frame` and `synth.pose_inertial_problem(_last_frame)`; every builder is
seeded.  Points are moved by re-placing them at a chosen pixel and depth of the frame's true camera, so observations stay
consistent with the map.  Inertial frames carry their preintegrations (`preint`, or `preint_frame` + `preint_kf`) in the keys the
package's wrappers read.  tests/test_pose_layouts_cpu.py asserts from the oracle that each frame reaches the branch it is named for."""
import numpy as np

import lba_scenes
import oracle_lib as O
from orb_slam3_modified_b200 import synth

W, H = 640, 480
NT = 256          # threads per CTA of pose_opt_kernel
PI_NT = 128       # threads per CTA of pose_inertial_opt_kernel


# ---- PoseOptimization ----
def _conj(q):
    return q * np.array([1, -1, -1, -1])


def _reobserve(f, idx, rng, noise_px=1.0, octave=None):
    """Observations of points idx through the frame's true pose and camera, with noise_px * 1.2^octave pixel noise."""
    gt, c = f['gt_pose'], f['cam'].astype(np.float64)
    octave = rng.integers(0, 8, len(idx)) if octave is None else np.asarray(octave)
    xc = synth._qrot(gt[:4], f['Xw'][idx]) + gt[4:]
    uv = np.stack([c[0] * xc[:, 0] / xc[:, 2] + c[2], c[1] * xc[:, 1] / xc[:, 2] + c[3]], 1)
    f['obs'][idx] = (uv + rng.normal(0, noise_px, uv.shape) * (1.2 ** octave)[:, None]).astype(np.float32).astype(np.float64)
    f['inv_sigma2'][idx] = (1.0 / (np.float32(1.2) ** octave.astype(np.float32)) ** 2).astype(np.float32)


def _place(f, idx, u, v, z):
    """Moves points idx to pixel (u, v) at depth z of the true camera (z < 0: behind it; the projection is the same pixel)."""
    gt, c = f['gt_pose'], f['cam'].astype(np.float64)
    Xc = np.stack([(u - c[2]) * z / c[0], (v - c[3]) * z / c[1], z], 1)
    f['Xw'][idx] = synth._qrot(_conj(gt[:4]), Xc - gt[4:]).astype(np.float32).astype(np.float64)


def depth(f, pose=None):
    """Depth of every point in the camera at pose (default the true pose)."""
    p = f['gt_pose'] if pose is None else np.asarray(pose, np.float64)
    q = p[:4] / np.linalg.norm(p[:4])
    return (synth._qrot(q, f['Xw']) + p[4:])[:, 2]


def po_count(n, seed, outlier_frac=0.15):
    return synth.pose_opt_problem(n=n, seed=seed, outlier_frac=outlier_frac)


def po_all_gross(n=120, seed=0):
    """Every observation 100..200 px off: round one flags them all, no edge is active from round two on."""
    rng = np.random.default_rng(seed + 500)
    f = synth.pose_opt_problem(n=n, seed=seed, outlier_frac=0.0)
    ang = rng.uniform(0, 2 * np.pi, n)
    f['obs'] = (f['obs'] + rng.uniform(100, 200, n)[:, None] * np.stack([np.cos(ang), np.sin(ang)], 1)).astype(np.float32).astype(np.float64)
    return f


def po_noise_free(n=150, seed=0):
    """Exact observations (double, not rounded to float) of the frame's own initial pose with its quaternion normalised in double: every
    round's first step leaves the cost unchanged, rho == 0 ends the round."""
    f = synth.pose_opt_problem(n=n, seed=seed, outlier_frac=0.0, pose_noise=(0.0, 0.0))
    f['pose'][:4] /= np.linalg.norm(f['pose'][:4])
    f['gt_pose'] = f['pose'].copy()
    c = f['cam'].astype(np.float64)
    xc = synth._qrot(f['pose'][:4], f['Xw']) + f['pose'][4:]
    f['obs'] = np.stack([c[0] * xc[:, 0] / xc[:, 2] + c[2], c[1] * xc[:, 1] / xc[:, 2] + c[3]], 1)
    return f


def po_bad_start(seed=3):
    """A start 0.5 m / 12 deg off the truth: at least one iteration ends after 10 rejected trials (qmax == 10)."""
    return synth.pose_opt_problem(n=200, seed=seed, pose_noise=(0.5, 12.0))


def po_behind_and_far(n=200, seed=0):
    """12 points behind the camera (they project to the pixel they are observed at) and 12 points 480..520 m away."""
    rng = np.random.default_rng(seed + 600)
    f = synth.pose_opt_problem(n=n, seed=seed, outlier_frac=0.1)
    idx = rng.choice(n, 24, replace=False)
    _place(f, idx, rng.uniform(20, W - 20, 24), rng.uniform(20, H - 20, 24), np.concatenate([-rng.uniform(3, 8, 12), rng.uniform(480, 520, 12)]))
    _reobserve(f, idx, rng)
    return f


def po_border(n=160, seed=0):
    """40 observations exactly on the image border (columns 0 and W - 1, rows 0 and H - 1, the four corners)."""
    rng = np.random.default_rng(seed + 700)
    f = synth.pose_opt_problem(n=n, seed=seed, outlier_frac=0.1)
    idx = rng.choice(n, 40, replace=False)
    u = np.concatenate([np.zeros(9), np.full(9, W - 1.0), rng.uniform(0, W - 1, 18), [0, W - 1, 0, W - 1]])
    v = np.concatenate([rng.uniform(0, H - 1, 18), np.zeros(9), np.full(9, H - 1.0), [0, 0, H - 1, H - 1]])
    _place(f, idx, u, v, rng.uniform(3, 12, 40))
    f['obs'][idx] = np.stack([u, v], 1).astype(np.float32).astype(np.float64)
    return f


def po_non_unit_quaternion(n=150, seed=0):
    """The initial quaternion scaled by 1.37: the SE3Quat constructor normalises it."""
    f = synth.pose_opt_problem(n=n, seed=seed, outlier_frac=0.15)
    f['pose'][:4] *= 1.37
    return f


def po_octaves(n=96, seed=0):
    """Octave i % 8 for observation i: every level's 1 / 1.44^octave weight and noise scale."""
    rng = np.random.default_rng(seed + 800)
    f = synth.pose_opt_problem(n=n, seed=seed, outlier_frac=0.0)
    _reobserve(f, np.arange(n), rng, octave=np.arange(n) % 8)
    gross = rng.choice(n, 12, replace=False)
    f['obs'][gross] += rng.uniform(8, 30, (12, 2)) * rng.choice([-1, 1], (12, 2))
    return f


PO_LAYOUTS = {
    'n_0': lambda: po_count(0, 1), 'n_1': lambda: po_count(1, 2), 'n_2': lambda: po_count(2, 3),
    'n_3': lambda: po_count(3, 4, 0.0), 'n_9': lambda: po_count(9, 5, 0.0), 'n_10': lambda: po_count(10, 6, 0.1),
    'n_31': lambda: po_count(31, 7), 'n_32': lambda: po_count(32, 8), 'n_33': lambda: po_count(33, 9),
    'n_255': lambda: po_count(255, 10), 'n_256': lambda: po_count(256, 11), 'n_257': lambda: po_count(257, 12),
    'n_511': lambda: po_count(511, 13), 'n_512': lambda: po_count(512, 14), 'n_513': lambda: po_count(513, 15),
    'n_4000': lambda: po_count(4000, 16, 0.3),
    'all_gross': lambda: po_all_gross(seed=17),
    'noise_free': lambda: po_noise_free(seed=18),
    'bad_start': lambda: po_bad_start(seed=3),
    'behind_and_far': lambda: po_behind_and_far(seed=19),
    'border': lambda: po_border(seed=20),
    'non_unit_quaternion': lambda: po_non_unit_quaternion(seed=21),
    'octaves': lambda: po_octaves(seed=22),
    'non_square_camera': lambda: lba_scenes.pose_opt_frame(n=300, seed=23, outlier_frac=0.2),
}


# ---- PoseInertialOptimizationLastKeyFrame ('kf') / LastFrame ('lf') ----
def _with_preint(pr, variant):
    if variant == 'kf':
        pr['preint'] = O.imu_preintegrate(pr['acc'], pr['gyr'], pr['dt'], pr['bias6'], synth.IMU_NOISE)
    else:
        pr['preint_frame'] = O.imu_preintegrate(pr['acc'], pr['gyr'], pr['dt'], pr['bias6'], synth.IMU_NOISE)
        pr['preint_kf'] = O.imu_preintegrate(pr['acc_kf'], pr['gyr_kf'], pr['dt_kf'], pr['bias6'], synth.IMU_NOISE)
    return pr


def _base(variant, n, seed, **kw):
    return (synth.pose_inertial_problem if variant == 'kf' else synth.pose_inertial_problem_last_frame)(n=n, seed=seed, **kw)


def camera_pose(pr, state=None):
    """Rcw, tcw of the frame's camera at a body state (default the truth)."""
    s = pr['truth'] if state is None else state
    ex = pr['extr']
    Rcb, tcb = ex[:9].reshape(3, 3), ex[9:12]
    R, p = s[:9].reshape(3, 3), s[9:12]
    return Rcb @ R.T, Rcb @ (-R.T @ p) + tcb


def _pi_place(pr, idx, u, v, z, offset=None, track_depth=None):
    """Points idx at pixel (u, v), depth z of the true camera, observed noise-free at octave 0 (plus offset [k, 2] px)."""
    Rcw, tcw = camera_pose(pr)
    c = pr['cam'].astype(np.float64)
    Xc = np.stack([(u - c[2]) * z / c[0], (v - c[3]) * z / c[1], z], 1)
    pr['Xw'][idx] = ((Xc - tcw) @ Rcw).astype(np.float32)
    xc = pr['Xw'][idx].astype(np.float64) @ Rcw.T + tcw
    uv = np.stack([c[0] * xc[:, 0] / xc[:, 2] + c[2], c[1] * xc[:, 1] / xc[:, 2] + c[3]], 1)
    pr['obs'][idx] = (uv + (0 if offset is None else offset)).astype(np.float32)
    pr['inv_sigma2'][idx] = 1.0
    pr['track_depth'][idx] = np.abs(z).astype(np.float32) if track_depth is None else track_depth


def chi2(pr, state, idx=None):
    """EdgeMonoOnlyPose chi2 and depth sign of observations idx at a body state."""
    ex = pr['extr']
    idx = np.arange(len(pr['Xw'])) if idx is None else np.asarray(idx)
    c2, dp = [], []
    for i in idx:
        e, _, _, d = O.imu_edge_mono(state[:9].reshape(3, 3), state[9:12], ex[:9], ex[9:12], ex[12:21], ex[21:24], pr['cam'], pr['Xw'][i].astype(np.float64),
                                     pr['obs'][i].astype(np.float64), jac=False)
        c2.append(float(pr['inv_sigma2'][i]) * float(e @ e)); dp.append(bool(d))
    return np.array(c2), np.array(dp, bool)


def _log(R):
    c = (np.trace(R) - 1) / 2
    th = np.arccos(np.clip(c, -1, 1))
    v = np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]]) / 2
    return v if th < 1e-9 else v * th / np.sin(th)


def prior_chi2(pr, prev_state):
    """EdgePriorPoseImu's chi2 e^T H e at the previous frame's state (src/G2oTypes.cc:731-745)."""
    q = pr['prior_state']
    Rp = q[:9].reshape(3, 3)
    e15 = np.concatenate([_log(Rp.T @ prev_state[:9].reshape(3, 3)), Rp.T @ (prev_state[9:12] - q[9:12]), prev_state[12:21] - q[12:21]])
    return float(e15 @ pr['prior_H'] @ e15)


def pi_count(variant, n, seed, clean=False):
    """n observations; clean: no gross outlier, 0.05 x synth's start perturbation and 0.2 px noise, so that no Huber weight is active
    at the start (the first-step check of tests/test_pose_layouts_cpu.py runs on these)."""
    kw = dict(outlier_frac=0.0, perturb=0.05, noise_px=0.2) if clean else dict(outlier_frac=0.1)
    return _with_preint(_base(variant, n, seed, **kw), variant)


def pi_inliers(variant, n_in, seed, n_mod=6):
    """n_in clean observations and n_mod planted 3.2 px off at octave 0 (chi2 ~ 10: above every round's threshold in the last round,
    below the recovery's 18) with trackDepth >= 10: exactly n_in final inliers, and with n_in < 30 the recovery brings the others back."""
    rng = np.random.default_rng(seed + 900)
    pr = _base(variant, n_in + n_mod, seed, outlier_frac=0.0, noise_px=0.3)
    idx = np.arange(n_in, n_in + n_mod)
    ang = rng.uniform(0, 2 * np.pi, n_mod)
    _pi_place(pr, idx, rng.uniform(60, W - 60, n_mod), rng.uniform(60, H - 60, n_mod), rng.uniform(10.5, 20, n_mod),
              offset=3.2 * np.stack([np.cos(ang), np.sin(ang)], 1))
    return _with_preint(pr, variant)


def pi_close(variant, track_depth, seed, n=60, n_plant=8):
    """n noise-free observations and n_plant planted 2.72 px off at octave 0 (final chi2 ~ 7.4, between 5.991 and 1.5 x 5.991) whose
    trackDepth is track_depth: 10.0f is not close (outliers), nextafterf(10, 0) is (inliers)."""
    rng = np.random.default_rng(seed + 1000)
    pr = _base(variant, n + n_plant, seed, outlier_frac=0.0, noise_px=0.0)
    idx = np.arange(n, n + n_plant)
    ang = rng.uniform(0, 2 * np.pi, n_plant)
    _pi_place(pr, idx, rng.uniform(60, W - 60, n_plant), rng.uniform(60, H - 60, n_plant), np.full(n_plant, 10.0),
              offset=2.72 * np.stack([np.cos(ang), np.sin(ang)], 1), track_depth=np.float32(track_depth))
    return _with_preint(pr, variant)


def pi_behind(variant, seed, n=80, n_behind=8):
    """n_behind points behind the camera, observed noise-free where they project: a small chi2, but not isDepthPositive()."""
    rng = np.random.default_rng(seed + 1100)
    pr = _base(variant, n, seed, outlier_frac=0.0, perturb=0.05, noise_px=0.2)
    idx = rng.choice(n, n_behind, replace=False)
    _pi_place(pr, idx, rng.uniform(60, W - 60, n_behind), rng.uniform(60, H - 60, n_behind), -rng.uniform(3, 8, n_behind))
    return _with_preint(pr, variant)


def pi_all_gross(variant, seed, n=60):
    """Every observation 100..200 px off: only the inertial edges move the state."""
    rng = np.random.default_rng(seed + 1200)
    pr = _base(variant, n, seed, outlier_frac=0.0)
    ang = rng.uniform(0, 2 * np.pi, n)
    pr['obs'] = (pr['obs'] + rng.uniform(100, 200, n)[:, None] * np.stack([np.cos(ang), np.sin(ang)], 1)).astype(np.float32)
    return _with_preint(pr, variant)


def lf_prior_huber(seed, n=200):
    """The previous frame starts at its true state and the prior sits 5 cm away from it: the prior's chi2 exceeds 25 (Huber delta 5)."""
    pr = _base('lf', n, seed, outlier_frac=0.1)
    pr['prev_state'] = pr['truth_prev'].copy()
    pr['prior_state'] = pr['truth_prev'].copy()
    pr['prior_state'][9:12] += np.array([0.04, -0.03, 0.0])
    return _with_preint(pr, 'lf')


def _both(variant, s):
    return {
        'n_127': lambda: pi_count(variant, 127, s + 1, clean=True), 'n_128': lambda: pi_count(variant, 128, s + 2, clean=True),
        'n_129': lambda: pi_count(variant, 129, s + 3, clean=True), 'n_256': lambda: pi_count(variant, 256, s + 4),
        'n_257': lambda: pi_count(variant, 257, s + 5), 'n_2000': lambda: pi_count(variant, 2000, s + 6),
        'inliers_29': lambda: pi_inliers(variant, 29, s + 7), 'inliers_30': lambda: pi_inliers(variant, 30, s + 8),
        'depth_10': lambda: pi_close(variant, 10.0, s + 9), 'depth_below_10': lambda: pi_close(variant, np.nextafter(np.float32(10), np.float32(0)), s + 9),
        'behind': lambda: pi_behind(variant, s + 10), 'all_gross': lambda: pi_all_gross(variant, s + 11),
    }


KF_LAYOUTS = {
    'n_0': lambda: pi_count('kf', 0, 1, clean=True), 'n_6': lambda: pi_count('kf', 6, 2, clean=True), 'n_7': lambda: pi_count('kf', 7, 3, clean=True),
    **_both('kf', 10),
}
LF_LAYOUTS = {
    'n_5': lambda: pi_count('lf', 5, 31, clean=True), 'n_6': lambda: pi_count('lf', 6, 32, clean=True),
    **_both('lf', 40),
    'prior_huber': lambda: lf_prior_huber(seed=60),
}
# the layouts with no Huber weight active at the start: the first-step check
KF_CLEAN = ('n_0', 'n_6', 'n_7', 'n_127', 'n_128', 'n_129', 'behind')
LF_CLEAN = ('n_5', 'n_6', 'n_127', 'n_128', 'n_129', 'behind')


def run_oracle(variant, pr, rec_init=False, rounds=4):
    if variant == 'kf':
        return O.pose_inertial_opt_last_kf(pr, pr['preint'], rec_init=rec_init, rounds=rounds)
    return O.pose_inertial_opt_last_frame(pr, pr['preint_frame'], pr['preint_kf'], rec_init=rec_init, rounds=rounds)
