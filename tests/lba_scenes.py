"""LocalBundleAdjustment problems with explicit control over what `synth.lba_problem` leaves fixed: one camera per keyframe
(fx != fy, principal point off the image centre), any fixed-keyframe mask, exactly given observer sets, points behind a
keyframe or far away, and pose pairs / poses whose shared points / edges sit on the kernel's work-chunk boundaries.

Every problem has `synth.lba_problem`'s layout (same keys, float32-rounded inputs, `huber_delta`, edges grouped by point),
and its observations are projections through the observing keyframe's own camera, so the problem is consistent.  Each
scene asserts the counts it promises."""
import numpy as np

from orb_slam3_modified_b200 import synth

W, H = 640, 480
LBA_SCH = 128          # items per chunk of the LBA kernel's pose / pose-pair work lists (csrc/lba.cu)
AHEAD_Z = 12.0         # camera centre of an "ahead" keyframe: 12 m down the common viewing direction


def keyframes(n_kf, ahead=()):
    """Ground-truth poses (qw qx qy qz t, Tcw) of `synth.lba_problem`'s sideways arc.  The keyframes in `ahead` have their
    centre moved to z = AHEAD_Z, so that points in front of the other keyframes (z of 4..10 m) lie behind them."""
    gt = np.zeros((n_kf, 7))
    for i in range(n_kf):
        q = synth._quat_from_rotvec(np.array([0.03 * np.sin(0.4 * i), 0.02 * i - 0.2, 0.02 * np.cos(0.3 * i)]))
        c = np.array([0.25 * i - 0.125 * n_kf, 0.05 * np.sin(0.5 * i), AHEAD_Z if i in ahead else 0.1 * np.cos(0.2 * i)])
        qc = q * np.array([1, -1, -1, -1])
        gt[i, :4] = qc
        gt[i, 4:] = -synth._qrot(qc, c)
    return gt


def cameras(n_kf, seed):
    """One pinhole camera per keyframe: fx, fy at least 20 px apart, principal point 15..60 px off the image centre."""
    rng = np.random.default_rng(seed)
    fx = rng.uniform(400, 560, n_kf)
    fy = fx * rng.uniform(0.8, 0.92, n_kf)
    cx = W / 2 + rng.choice([-1, 1], n_kf) * rng.uniform(15, 60, n_kf)
    cy = H / 2 + rng.choice([-1, 1], n_kf) * rng.uniform(15, 60, n_kf)
    cam = np.stack([fx, fy, cx, cy], 1).astype(np.float32)
    assert (np.abs(cam[:, 0] - cam[:, 1]) > 20).all() and (np.abs(cam[:, 2] - W / 2) > 10).all() and (np.abs(cam[:, 3] - H / 2) > 10).all()
    return cam


def make(gt, cam, fixed, observers, home=None, depth=None, seed=0, outlier_frac=0.05, pose_noise=(0.01, 0.5), point_noise=0.02):
    """The problem whose point j is seen by exactly the keyframes observers[j].  Point j is placed at depth depth[j] (default
    4..10 m) in front of keyframe home[j] (default its middle observer) at a random pixel of that keyframe's image."""
    rng = np.random.default_rng(seed)
    n_kf, n_pts = len(gt), len(observers)
    home = [obs[len(obs) // 2] for obs in observers] if home is None else home
    depth = rng.uniform(4.0, 10.0, n_pts) if depth is None else np.asarray(depth, np.float64)
    inv_sigma2_tab = (1.0 / (np.float32(1.2) ** np.arange(8, dtype=np.float32)) ** 2).astype(np.float32)
    level_p = np.array([217, 181, 151, 126, 105, 87, 73, 60], np.float64)
    level_p /= level_p.sum()
    cam64 = cam.astype(np.float64)
    pts = np.zeros((n_pts, 3))
    e_pt, e_kf, obs, isg = [], [], [], []
    for j, kfs in enumerate(observers):
        assert len(set(kfs)) == len(kfs) and all(0 <= k < n_kf for k in kfs)
        h, z = home[j], depth[j]
        fx, fy, cx, cy = cam64[h]
        u, v = rng.uniform(60, W - 60), rng.uniform(60, H - 60)
        pc = np.array([(u - cx) * z / fx, (v - cy) * z / fy, z])
        pts[j] = synth._qrot(gt[h, :4] * np.array([1, -1, -1, -1]), pc - gt[h, 4:])
        for k in kfs:
            xc = synth._qrot(gt[k, :4], pts[j]) + gt[k, 4:]
            fx, fy, cx, cy = cam64[k]
            oct_ = rng.choice(8, p=level_p)
            uv = np.array([fx * xc[0] / xc[2] + cx, fy * xc[1] / xc[2] + cy]) + rng.normal(0, 1.2 ** oct_, 2)
            if rng.random() < outlier_frac:
                uv += rng.choice([-1, 1], 2) * rng.uniform(10, 20, 2)
            e_pt.append(j); e_kf.append(k); obs.append(uv.astype(np.float32).astype(np.float64)); isg.append(inv_sigma2_tab[oct_])
    fixed = np.asarray(fixed, np.uint8)
    poses = gt.copy()
    for i in np.flatnonzero(fixed == 0):
        poses[i, :4] = synth._qmul(synth._quat_from_rotvec(rng.normal(0, np.deg2rad(pose_noise[1]), 3)), gt[i, :4])
        poses[i, 4:] = gt[i, 4:] + rng.normal(0, pose_noise[0], 3)
    return dict(poses=poses.astype(np.float32).astype(np.float64), fixed=fixed, cam=cam,
                points=(pts + rng.normal(0, point_noise, pts.shape)).astype(np.float32).astype(np.float64),
                edge_point=np.array(e_pt, np.int32), edge_pose=np.array(e_kf, np.int32), obs=np.array(obs, np.float64).reshape(-1, 2),
                inv_sigma2=np.array(isg, np.float32), gt_poses=gt, gt_points=pts, huber_delta=float(np.float32(np.sqrt(5.991))))


def depths(p, poses=None, points=None):
    """Depth of every edge's point in its keyframe (poses / points default to the problem's initial estimates)."""
    poses = p['poses'] if poses is None else poses
    points = p['points'] if points is None else points
    q = poses[:, :4] / np.linalg.norm(poses[:, :4], axis=1)[:, None]
    out = np.zeros(len(p['edge_point']))
    for e, (j, k) in enumerate(zip(p['edge_point'], p['edge_pose'])):
        out[e] = synth._qrot(q[k], points[j])[2] + poses[k, 6]
    return out


def _windows(n_kf, n_pts, obs_per_pt, first=0):
    span = max(1, n_kf - first - obs_per_pt + 1)
    return [list(range(first + j % span, min(n_kf, first + j % span + obs_per_pt))) for j in range(n_pts)]


def masked(mask, n_pts=40, obs_per_pt=3, seed=0, **kw):
    """Sliding observer windows over len(mask) keyframes with per-keyframe cameras; keyframe i is fixed when mask[i]."""
    n_kf = len(mask)
    p = make(keyframes(n_kf), cameras(n_kf, seed + 1000), mask, _windows(n_kf, n_pts, obs_per_pt), seed=seed, **kw)
    assert np.bincount(p['edge_pose'], minlength=n_kf).min() > 0
    return p


def interleaved(n_kf=6, n_pts=40, obs_per_pt=3, seed=0, **kw):
    """Keyframes 1 and n_kf-2 fixed: free poses before, between and after the fixed ones."""
    mask = np.zeros(n_kf, np.uint8)
    mask[[1, n_kf - 2]] = 1
    return masked(mask, n_pts, obs_per_pt, seed, **kw)


def last_fixed(n_kf=6, n_pts=40, obs_per_pt=3, seed=0, **kw):
    mask = np.zeros(n_kf, np.uint8)
    mask[-2:] = 1
    return masked(mask, n_pts, obs_per_pt, seed, **kw)


def none_fixed(n_kf=6, n_pts=40, obs_per_pt=3, seed=0, **kw):
    return masked(np.zeros(n_kf, np.uint8), n_pts, obs_per_pt, seed, **kw)


def outliers(n_kf=6, n_pts=40, obs_per_pt=4, seed=0, frac=0.4):
    """About 40 % gross outliers (10..20 px): the Huber kernel is active on a large share of the edges."""
    mask = np.zeros(n_kf, np.uint8)
    mask[[0, n_kf // 2]] = 1
    p = masked(mask, n_pts, obs_per_pt, seed, outlier_frac=frac)
    res = gt_residuals(p)
    share = float((p['inv_sigma2'] * (res ** 2).sum(1) > p['huber_delta'] ** 2).mean())
    assert share > 0.3, share
    return p


def gt_residuals(p):
    """Reprojection residuals at the ground truth (the noise and outliers the generator put in)."""
    cam = p['cam'].astype(np.float64)
    out = np.zeros((len(p['edge_point']), 2))
    for e, (j, k) in enumerate(zip(p['edge_point'], p['edge_pose'])):
        xc = synth._qrot(p['gt_poses'][k, :4], p['gt_points'][j]) + p['gt_poses'][k, 4:]
        out[e] = p['obs'][e] - [cam[k, 0] * xc[0] / xc[2] + cam[k, 2], cam[k, 1] * xc[1] / xc[2] + cam[k, 3]]
    return out


def observer_sets(n_kf=6, n_single=8, n_fixed_only=8, n_window=30, hub=5, seed=0):
    """Exactly given observer sets: points seen by one keyframe (free ones and fixed ones), points seen only by fixed
    keyframes, one point seen by `hub` keyframes, and a free keyframe (the second to last) no point observes.  Fixed
    keyframes: 1 and the last one, so free poses lie on both sides of a fixed one."""
    assert n_kf >= 5 and hub <= n_kf - 1
    fixed = np.zeros(n_kf, np.uint8)
    fixed[[1, n_kf - 1]] = 1
    idle = n_kf - 2
    seen = [k for k in range(n_kf) if k != idle]
    rng = np.random.default_rng(seed)
    obs = [[seen[i % len(seen)]] for i in range(n_single)]
    obs += [[1, n_kf - 1] for _ in range(n_fixed_only)]
    obs += [sorted(rng.choice(seen, 3, replace=False).tolist()) for _ in range(n_window)]
    obs.append(seen[:hub])
    p = make(keyframes(n_kf), cameras(n_kf, seed + 2000), fixed, obs, seed=seed)
    # the counts the scene promises
    n_obs = np.bincount(p['edge_point'], minlength=len(obs))
    fixed_only = np.array([all(fixed[k] for k in o) for o in obs])
    assert (n_obs == 1).sum() >= n_single and fixed_only.sum() >= n_fixed_only and n_obs.max() == hub
    assert np.bincount(p['edge_pose'], minlength=n_kf)[idle] == 0 and not fixed[idle]
    assert any(not fixed[k] and k > 1 for k in range(n_kf))
    return p


def hub(n_kf=36, n_pts=200, seed=0):
    """One point seen by 33 keyframes: more than four rounds of the kernel's 8-lane point loops.  Every third keyframe
    is fixed, so the 33 observers mix free and fixed poses; the rest of the points use sliding windows of 4."""
    fixed = (np.arange(n_kf) % 3 == 2).astype(np.uint8)
    obs = _windows(n_kf, n_pts - 1, 4) + [list(range(1, 34))]
    p = make(keyframes(n_kf), cameras(n_kf, seed + 3000), fixed, obs, seed=seed)
    assert np.bincount(p['edge_point']).max() == 33 and (np.bincount(p['edge_point']) > 8 * 4).sum() == 1
    return p


def chunk_edges(counts=(127, 128, 129, 256, 257), seed=0):
    """Free keyframe pairs (2i+1, 2i+2) sharing exactly counts[i] points, each point also seen by the fixed keyframe 0:
    pose pairs whose shared-point lists end just before, on and just after a multiple of LBA_SCH, and free poses with
    exactly that many edges."""
    n_kf = 1 + 2 * len(counts)
    fixed = np.zeros(n_kf, np.uint8)
    fixed[0] = 1
    obs = [[0, 2 * i + 1, 2 * i + 2] for i, c in enumerate(counts) for _ in range(c)]
    p = make(keyframes(n_kf), cameras(n_kf, seed + 4000), fixed, obs, seed=seed, outlier_frac=0.02)
    # shared points of every free pair, counted from the edge list
    vis = np.zeros((n_kf, len(obs)), bool)
    vis[p['edge_pose'], p['edge_point']] = True
    shared = vis[1:].astype(np.int64) @ vis[1:].T.astype(np.int64)
    for i, c in enumerate(counts):
        assert shared[2 * i, 2 * i + 1] == c
        assert np.bincount(p['edge_pose'], minlength=n_kf)[2 * i + 1] == c
    off = shared - np.diag(np.diag(shared))
    assert set(np.unique(off).tolist()) == {0} | set(counts)
    return p


def depth_edges(n_kf=6, n_pts=40, n_far=6, seed=0):
    """Keyframe 3 (free) and keyframe 0 (fixed) sit AHEAD_Z down the viewing direction: the points in front of the others
    are behind them (depth -10..-1 m), so edges with a negative depth reach the optimiser and its final depth test.  The
    last n_far points are about 500 m away."""
    ahead = (0, 3)
    fixed = np.zeros(n_kf, np.uint8)
    fixed[[0, n_kf - 1]] = 1
    rng = np.random.default_rng(seed)
    front = [k for k in range(n_kf) if k not in ahead]
    obs, home = [], []
    for j in range(n_pts):
        o = sorted(set(rng.choice(front, 2, replace=False).tolist()) | ({3} if j % 2 == 0 else set()) | ({0} if j % 5 == 0 else set()))
        obs.append(o)
        home.append(min(k for k in o if k in front))
    depth = rng.uniform(4.0, 10.0, n_pts)
    depth[-n_far:] = rng.uniform(480, 520, n_far)
    p = make(keyframes(n_kf, ahead), cameras(n_kf, seed + 5000), fixed, obs, home=home, depth=depth, seed=seed)
    z = depths(dict(p, poses=p['gt_poses'], points=p['gt_points']))
    behind = np.isin(p['edge_pose'], ahead) & (p['edge_point'] < n_pts - n_far)
    assert behind.sum() >= n_pts // 2 and (z[behind] >= -10).all() and (z[behind] <= -1).all()
    assert (z[~np.isin(p['edge_pose'], ahead)] > 3).all()
    far = np.isin(p['edge_point'], np.arange(n_pts - n_far, n_pts)) & ~np.isin(p['edge_pose'], ahead)
    assert far.sum() >= 2 * n_far and (z[far] > 400).all()
    return p


def small_layouts(seed=0):
    """The layouts at the size of a dense check (6 keyframes, up to about 60 points)."""
    return {'interleaved': interleaved(seed=seed), 'last_fixed': last_fixed(seed=seed + 1), 'none_fixed': none_fixed(seed=seed + 2),
            'observer_sets': observer_sets(seed=seed + 3), 'depth_edges': depth_edges(seed=seed + 4), 'outliers': outliers(seed=seed + 5)}


def pose_opt_frame(n=300, seed=0, outlier_frac=0.2, pose_noise=(0.03, 1.5)):
    """`synth.pose_opt_problem` with fx != fy and the principal point off the centre; observations through that camera."""
    rng = np.random.default_rng(seed)
    cam = np.array([470.0, 410.0, W / 2 + 37.0, H / 2 - 29.0], np.float32)
    fx, fy, cx, cy = cam.astype(np.float64)
    gt = np.concatenate([synth._quat_from_rotvec(rng.normal(0, 0.1, 3)), rng.normal(0, 0.3, 3)])
    z = rng.uniform(3, 12, n)
    u, v = rng.uniform(20, W - 20, n), rng.uniform(20, H - 20, n)
    Xw = synth._qrot(gt[:4] * np.array([1, -1, -1, -1]), np.stack([(u - cx) * z / fx, (v - cy) * z / fy, z], 1) - gt[4:])
    Xw = Xw.astype(np.float32).astype(np.float64)
    xc = synth._qrot(gt[:4], Xw) + gt[4:]
    octv = rng.integers(0, 8, n)
    obs = np.stack([fx * xc[:, 0] / xc[:, 2] + cx, fy * xc[:, 1] / xc[:, 2] + cy], 1) + rng.normal(0, 1, (n, 2)) * (1.2 ** octv)[:, None]
    bad = rng.random(n) < outlier_frac
    obs[bad] += rng.uniform(8, 30, (int(bad.sum()), 2)) * rng.choice([-1, 1], (int(bad.sum()), 2))
    pose = gt.copy()
    pose[:4] = synth._qmul(synth._quat_from_rotvec(rng.normal(0, np.deg2rad(pose_noise[1]), 3)), gt[:4])
    pose[4:] += rng.normal(0, pose_noise[0], 3)
    return dict(pose=pose.astype(np.float32).astype(np.float64), cam=cam, Xw=Xw, obs=obs.astype(np.float32).astype(np.float64),
                inv_sigma2=(1.0 / (np.float32(1.2) ** octv.astype(np.float32)) ** 2).astype(np.float32), gt_pose=gt)
