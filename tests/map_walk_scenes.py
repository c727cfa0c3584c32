"""Seeded maps that drive the two whole-function map walks (lba_local_bundle_adjustment_batch: Optimizer::LocalBundleAdjustment,
local_inertial_ba_map_batch: Optimizer::LocalInertialBA) to the shapes where their kernels branch (csrc/map_walk.cuh, local_ba.cu,
local_inertial_ba_map.cu), all one CTA of WT = 512 threads per map:
- the first-appearance numbering (compact / block_prefix) over the local keyframes' slots (Qs), the local points' observations (Qo), the
  local points (nL), LBA's nCov + 1 candidate lists and LIBA's candidates, one 512-wide tile at a time with a carry between tiles;
- segment over empty segments: local keyframes without slots, local points without observations;
- LBA's bitonic vertex sort over n2 = the power of two at or above nP (keyframe vertices) and nL (point vertices), inside sortCap;
- LIBA's lFixedKeyFrames probe (one 512-candidate tile at a time, the f == INT_MAX skip, the stop at maxFixKF = 200) and its window -> edge
  CSR per 512-edge tile for 25-keyframe (bLarge) windows;
- the EraseObservation cascade.
The maps are local_ba_lib / local_inertial_ba_map_lib models with real projections; observations added here are projections of the point's
position through the observer's pose and camera.  lba_shape / liba_shape compute each quantity from a flattened map and a call's record.
lba_cases() / liba_cases(): name -> (builder, wanted shape)."""
import numpy as np

import liba_scenes
import local_ba_lib as LB
import local_inertial_ba_map_lib as LM
import orb_slam3_modified_b200 as orb
from track_lib import pose_matrices

F32 = np.float32
WT = 512
MAXFIX = 200


# ---- model edits (both models: LB.Map and its LM subclass) ----
def observe(M, k, pid, octave=0):
    """Keyframe k observes point pid in a new slot, at the projection of the point through k's pose and camera."""
    f, q = M.kfs[k], M.pts[pid]
    R, t, _ = pose_matrices(f.Tcw)
    X = R.astype(np.float64) @ q.pos.astype(np.float64) + t.astype(np.float64)
    fx, fy, cx, cy = f.cam.astype(np.float64)
    uv = np.array([fx * X[0] / X[2] + cx, fy * X[1] / X[2] + cy], F32)
    f.mp = np.append(f.mp, pid)
    f.pt = np.vstack([f.pt.reshape(-1, 2), uv[None]]).astype(F32)
    f.octave = np.append(f.octave, octave).astype(np.int32)
    q.obs[k] = len(f.mp) - 1
    q.nObs += 1
    if q.ref < 0:
        q.ref = k


def unobserve(M, pid, k):
    """Keyframe k's slot of point pid becomes NULL and the observation goes; mpRefKF moves to the first observer left."""
    q = M.pts[pid]
    M.kfs[k].mp[q.obs.pop(k)] = -1
    q.nObs -= 1
    if q.ref == k:
        q.ref = min(q.obs) if q.obs else -1


def pad(M, k, n):
    """n NULL slots appended to keyframe k."""
    f = M.kfs[k]
    f.mp = np.append(f.mp, np.full(n, -1, np.int64))
    f.pt = np.vstack([f.pt.reshape(-1, 2), np.zeros((n, 2), F32)]).astype(F32)
    f.octave = np.append(f.octave, np.zeros(n, np.int32)).astype(np.int32)


def empty_keyframe(M, k):
    """Keyframe k keeps its place in the lists but has no slot."""
    for pid in [int(p) for p in M.kfs[k].mp if p >= 0]:
        unobserve(M, pid, k)
    f = M.kfs[k]
    f.mp, f.pt, f.octave = np.zeros(0, np.int64), np.zeros((0, 2), F32), np.zeros(0, np.int32)


def no_observations(M, pid):
    """Point pid stays in its slots with an empty observation list (and no mpRefKF)."""
    q = M.pts[pid]
    q.obs, q.nObs, q.ref = {}, 0, -1


def plant_behind(M, pid):
    """Point pid moved behind its observers (reflected through the first one's centre), observed at its exact projections: the solver
    keeps it there and every one of its edges fails the depth test."""
    q = M.pts[pid]
    c = M.kfs[min(q.obs)].Ow.astype(np.float64)
    q.pos = (2 * c - q.pos.astype(np.float64)).astype(F32)
    for k in sorted(q.obs):
        f = M.kfs[k]
        R, t, _ = pose_matrices(f.Tcw)
        X = R.astype(np.float64) @ q.pos.astype(np.float64) + t.astype(np.float64)
        assert X[2] < 0
        fx, fy, cx, cy = f.cam.astype(np.float64)
        f.pt[q.obs[k]] = np.array([fx * X[0] / X[2] + cx, fy * X[1] / X[2] + cy], F32)


def plant_cascade(M, pids, plant):
    """The cascade's cases on points pids (each good with >= 4 observers, the first with exactly 3 after the trim): nObs 3 with an erase
    that turns the point bad and a later erase that finds nothing; the mpRefKF observation erased first; every observation erased."""
    p3, pr, pa = pids
    while len(M.pts[p3].obs) > 3:
        unobserve(M, p3, max(M.pts[p3].obs))
    ks = sorted(M.pts[p3].obs)
    M.pts[p3].ref = ks[1]
    plant(M, p3, [ks[0], ks[2]], px=150.0)
    M.pts[pr].ref = min(M.pts[pr].obs)
    plant(M, pr, [M.pts[pr].ref], px=60.0)
    plant_behind(M, pa)


# ---- LBA: the walk on the model, for tuning ----
def lba_walk(M, pkf):
    K, P = M.kfs, M.pts
    local = [pkf] + [k for k in M.cov[pkf] if not K[k].bad and not K[k].other]
    pts, seen = [], set()
    for k in local:
        for p in K[k].mp:
            if p >= 0 and not P[p].bad and not P[p].other and p not in seen:
                seen.add(int(p)); pts.append(int(p))
    return local, pts


def set_qs(M, pkf, target):
    local, _ = lba_walk(M, pkf)
    qs = sum(len(M.kfs[k].mp) for k in local)
    assert qs <= target, (qs, target)
    pad(M, pkf, target - qs)


def set_qo(M, pkf, target):
    """Observations of local points by keyframes outside the local ones added or removed until Qo == target."""
    local, pts = lba_walk(M, pkf)
    loc = set(local) | set(M.cov[pkf])
    qo = sum(len(M.pts[p].obs) for p in pts)
    others = [k for k in sorted(M.kfs) if k not in loc]
    i = 0
    while qo > target:
        p = pts[-1 - i % len(pts)]
        far = [k for k in sorted(M.pts[p].obs) if k not in loc]
        if far and len(M.pts[p].obs) > 3:
            unobserve(M, p, far[0]); qo -= 1
        i += 1
        assert i < 100 * len(pts)
    while qo < target:
        p = pts[i % len(pts)]
        new = [k for k in others if k not in M.pts[p].obs]
        if new:
            observe(M, new[i % len(new)], p); qo += 1
        i += 1
        assert i < 100 * len(pts)


def set_nl(M, pkf, target):
    """The local points past the first target turned bad: nL == target (the bad points stay in the table and the slots)."""
    _, pts = lba_walk(M, pkf)
    assert len(pts) >= target
    for p in pts[target:]:
        M.pts[p].bad = True


def add_fixed_cameras(M, pkf, n, seed, bad_every=0, other_every=0):
    """n keyframes near pKF that each observe a few local points late in the local list (so their first observation is past Qo's first
    tile); every bad_every-th is bad and every other_every-th of another map, interleaved with the good ones in key order."""
    rng = np.random.default_rng(seed)
    _, pts = lba_walk(M, pkf)
    base = M.kfs[pkf]
    k0 = max(M.kfs) + 1
    mn = max(f.mnId for f in M.kfs.values()) + 1 + rng.permutation(n) * 5
    for i in range(n):
        T = base.Tcw.copy()
        T[4:] += F32(0.01) * np.array([i % 7 - 3, i % 5 - 2, 0], F32)
        kf = LB.KeyFrame(k0 + i, int(mn[i]), T, base.cam, np.zeros((0, 2), F32), np.zeros(0, np.int32))
        kf.bad = bool(bad_every and i % bad_every == 1)
        kf.other = bool(other_every and i % other_every == 2)
        M.kfs[k0 + i] = kf
        for p in rng.choice(pts[len(pts) // 2:], 2, replace=False):
            observe(M, k0 + i, int(p))


# ---- LBA cases ----
def _tiles_qs(seed, target):
    M, k = LB.scene(seed, n_kf=10, n_pts=150, obs_per_pt=3, n_cov=3, slots_extra=0)
    # the slots of pKF's covisibles interleave with NULLs, so that points recur across tiles
    for c in M.cov[k]:
        pad(M, c, 60)
        f = M.kfs[c]
        order = np.random.default_rng(seed + c).permutation(len(f.mp))
        inv = np.argsort(order)
        f.mp, f.pt, f.octave = f.mp[order], f.pt[order], f.octave[order]
        for p, q in M.pts.items():
            if c in q.obs:
                q.obs[c] = int(inv[q.obs[c]])
    set_qs(M, k, target)
    return M, k


def _tiles_qo(seed, target):
    n_pts = {511: 200, 512: 200, 513: 200}.get(target, 400)
    M, k = LB.scene(seed, n_kf=12, n_pts=n_pts, obs_per_pt=4, n_cov=3)
    set_qo(M, k, target)
    return M, k


def _large(seed):
    M, k = LB.scene(seed, n_kf=20, n_pts=6000, obs_per_pt=8, n_cov=10, outlier_frac=0.03, slots_extra=1100)
    return M, k


def _nl(seed, target):
    n_pts = int(target * 1.6) + 40
    M, k = LB.scene(seed, n_kf=12, n_pts=n_pts, obs_per_pt=3, n_cov=6, outlier_frac=0.03)
    set_nl(M, k, target)
    return M, k


def _np_one(seed):
    """pKF alone: no covisible, every point seen only by it, pKF the init keyframe: nP = 1, the one vertex fixed."""
    M, k = LB.scene(seed, n_kf=1, n_pts=80, obs_per_pt=1, n_cov=0)
    M.kfs[k].init = True
    return M, k


def _np(seed, target, huge_ids=False):
    """nP = nLocal + nFix = (n_cov + 1) + 3 with observer windows of 4."""
    n_cov = target - 4
    M, k = LB.scene(seed, n_kf=target + 4, n_pts=12 * (target + 4), obs_per_pt=4, n_cov=n_cov)
    if huge_ids:              # mnIds just below 2^64 - 1, the sort's padding key
        top = (1 << 64) - 2
        for i, f in enumerate(sorted(M.kfs.values(), key=lambda f: f.mnId)):
            f.mnId = top - 3 * (len(M.kfs) - 1 - i)
        for i, q in enumerate(sorted(M.pts.values(), key=lambda q: q.mnId)):
            q.mnId = top - 2 * (len(M.pts) - 1 - i)
    return M, k


def _fixed_many(seed):
    M, k = LB.scene(seed, n_kf=10, n_pts=600, obs_per_pt=3, n_cov=3)
    add_fixed_cameras(M, k, 500, seed, bad_every=3, other_every=5)
    return M, k


def _cov600(seed):
    M, k = LB.scene(seed, n_kf=605, n_pts=1300, obs_per_pt=2, n_cov=600, slots_extra=1)
    for i, c in enumerate(M.cov[k]):
        if i % 97 == 13:
            M.kfs[c].bad = True
        elif i % 89 == 40:
            M.kfs[c].other = True
    M.stop = True
    return M, k


def _empty_cascade(seed):
    M, k = LB.scene(seed, n_kf=14, n_pts=700, obs_per_pt=5, n_cov=7, outlier_frac=0.0)
    cov = M.cov[k]
    empty_keyframe(M, cov[1])                       # between full local keyframes
    empty_keyframe(M, cov[3])
    _, pts = lba_walk(M, k)
    for p in (pts[len(pts) // 3], pts[len(pts) // 3 + 1], pts[2 * len(pts) // 3]):
        no_observations(M, p)                       # in the middle of the local list, two of them consecutive
    local = set(lba_walk(M, k)[0])
    hub = [p for p in pts[5:] if len(M.pts[p].obs) >= 4 and set(M.pts[p].obs) <= local][:3]   # observers the solver moves
    plant_cascade(M, hub, LB.plant_outliers)
    return M, k


# The case whose chi2 are not all 1e-3 clear of 5.991: at about 40,000 edges some chi2 always lands that close.  Its GPU checks do not need
# the margin, since the finish is compared with the oracle finishing the GPU's own doubles.
NO_MARGIN = {'qs_qo_40k'}


def lba_cases():
    """name -> (builder, wanted shape) for lba_local_bundle_adjustment_batch; lba_shape gives the shape of a case."""
    c = {}
    for t in (511, 512, 513, 1023, 1024, 1025):
        c['qs_%d' % t] = (lambda t=t: _tiles_qs(20 + t, t), dict(Qs=t))
        c['qo_%d' % t] = (lambda t=t: _tiles_qo(40 + t, t), dict(Qo=t))
    c['qs_qo_40k'] = (lambda: _large(61), dict(Qs_min=38000, Qo_min=38000))
    for t in (511, 512, 513, 4095, 4096, 4097):
        c['nl_%d' % t] = (lambda t=t: _nl(70 + t + 1000 * (t == 513), t), dict(nL=t))
    c['np_1'] = (lambda: _np_one(81), dict(nP=1))
    for t in (16, 17, 32, 33, 64, 65):
        c['np_%d' % t] = (lambda t=t: _np(90 + t + 1000 * (t == 65), t, huge_ids=t == 17), dict(nP=t))
    c['fixed_500'] = (lambda: _fixed_many(101), dict(nFix_min=250, fix_late=True, fix_skipped=True))
    c['cov_600'] = (lambda: _cov600(102), dict(lists_min=601))
    c['empty_cascade'] = (lambda: _empty_cascade(104), dict(empty_kf=2, empty_pt=3, cascade=True))
    return c


def next_pow2(n):
    n2 = 1
    while n2 < n:
        n2 <<= 1
    return n2


def lba_shape(m, r):
    """The walk's quantities of flattened map m from a record r of it (localKF, fixedKF, localPoint): Qs, Qo, nL, nP, nFix, n2 of the
    two sorts, sortCap, the covisible lists, empty segments, and where first appearances fall in the 512-wide tiles."""
    ss, os_ = m['slotStart'], m['obsStart']
    loc, fix, pts = [int(k) for k in r['localKF']], [int(k) for k in r['fixedKF']], [int(p) for p in r['localPoint']]
    sl = [int(ss[k + 1] - ss[k]) for k in loc]
    ol = [int(os_[p + 1] - os_[p]) for p in pts]
    skip = orb.KF_BAD | orb.KF_OTHER_MAP
    # the positions of the local points in Qs: a point seen in several tiles, and a first appearance in a later tile after a repeat
    first, tiles, repeat, late_first, q = {}, {}, set(), False, 0
    for k in loc:
        for s in range(ss[k], ss[k + 1]):
            p = int(m['slotPoint'][s])
            if p >= 0 and not m['pointFlags'][p] & skip:
                if p in first:
                    repeat.add(q // WT)
                else:
                    first[p] = q
                    late_first |= q // WT in repeat and q >= WT
                tiles.setdefault(p, set()).add(q // WT)
            q += 1
    split = any(len(t) > 1 for t in tiles.values())
    # first observation of each fixed keyframe in Qo
    ffirst, q = {}, 0
    for p in pts:
        for o in range(os_[p], os_[p + 1]):
            ffirst.setdefault(int(m['obsKF'][o]), q)
            q += 1
    fixed_first = [ffirst[k] for k in fix]
    kf = m['kfFlags']
    reached = set(ffirst) - set(range(len(m['cov']) + 1))
    return dict(Qs=sum(sl), Qo=sum(ol), nL=len(pts), nLocal=len(loc), nFix=len(fix), nP=len(loc) + len(fix), n2P=next_pow2(len(loc) + len(fix)),
                n2L=next_pow2(len(pts)), sortCap=next_pow2(max(len(kf), len(m['pointFlags']))), lists=len(m['cov']) + 1,
                empty_kf=sum(1 for i, n in enumerate(sl) if n == 0 and 0 < i < len(sl) - 1),
                empty_pt=sum(1 for i, n in enumerate(ol) if n == 0 and 0 < i < len(ol) - 1),
                split=split, late_first=late_first, fix_late=any(f >= WT for f in fixed_first),
                fix_skipped=any(kf[k] & skip for k in reached))


# ---- LIBA cases ----
def _liba_candidates(seed, cand_obs, n_cov, bad=(), n_opt=4, n_window_pts=60):
    """Candidates in a chosen order: candidate j is seen by pKF, one other window keyframe and the covisibles cand_obs[j] (indices into
    the n_cov covisibles), so that its unmarked observers are exactly those.  pKF's slots are sorted by point, which makes the local
    list (and the candidate list) follow j.  n_window_pts points seen only by the window come after them.  bad: covisibles flagged bad."""
    w = n_opt - 1
    obs = [sorted([0, 1 + j % w] + [n_opt + 1 + c for c in co]) for j, co in enumerate(cand_obs)]
    obs += [sorted({1 + j % w, 1 + (j + 1) % w}) for j in range(n_window_pts)]
    pr = liba_scenes.graph(n_opt, n_cov=n_cov, observers=obs, seed=seed)
    M, ids = LM.from_graph(pr, seed + 500)
    f = M.kfs[ids[0]]
    order = sorted(range(len(f.mp)), key=lambda i: (f.mp[i] < 0, f.mp[i]))
    f.mp, f.pt, f.octave = f.mp[order], f.pt[order], f.octave[order]
    for i, p in enumerate(f.mp):
        if p >= 0:
            M.pts[int(p)].obs[ids[0]] = i
    for c in bad:
        M.kfs[ids[n_opt + 1 + c]].bad = True
    return (M, ids[0], 100, False, False)


def _probe_skip(seed):
    """Candidate 0's step marks covisible 0, which every candidate of the next tile shares: the probe finds none there and moves on a
    tile.  Candidate 513's unmarked observers are both bad: it marks them and adds none."""
    cand = [[0]] * 513 + [[1, 2]] + [[3 + i] for i in range(90)]
    return _liba_candidates(seed, cand, 93, bad=(1, 2))


def _cap_at(seed, at, total):
    """The 200th fixed keyframe (the predecessor, then 199 from candidates) added at candidate `at`; total candidates."""
    cand = [[i] for i in range(198)] + [[0]] * (at - 198) + [[198]] + [[199 + i] for i in range(total - at - 1)]
    return _liba_candidates(seed, cand, 199 + max(0, total - at - 1))


def _fix199(seed):
    """198 candidates add a keyframe, the 402 after them add none: 199 fixed keyframes and the candidates run out."""
    cand = [[i] for i in range(198)] + [[i % 198] for i in range(402)]
    return _liba_candidates(seed, cand, 198)


def _liba_edges(seed, n_edges):
    """A 25-keyframe bLarge window whose points are seen by two window keyframes each (one by a single one when n_edges is odd), the
    keyframes of consecutive edges far apart: nE == n_edges, every window keyframe's edges spread over every 512-edge tile."""
    obs = []
    for j in range(n_edges // 2):
        a = j % 25
        b = (7 * j + 3 + j // 25) % 25
        obs.append(sorted({a, b if b != a else (a + 1) % 25}))
    if n_edges % 2:
        obs.append([n_edges % 25])
    pr = liba_scenes.graph(25, n_cov=2, observers=obs, seed=seed, large=True)
    M, ids = LM.from_graph(pr, seed + 500)
    return (M, ids[0], 60, True, False)


def _liba_nl(seed, n_pts):
    M, k, ids = LM.scene(seed, n_opt=6, n_cov=3, n_pts=n_pts, obs_per_pt=3)
    return (M, k, 40, False, False)


def _liba_empty_cascade(seed):
    M, k, ids = LM.scene(seed, n_opt=6, n_cov=3, n_pts=400, obs_per_pt=4, outlier_frac=0.0)
    empty_keyframe(M, ids[2])                       # a window keyframe between full ones
    win = [ids[i] for i in range(6)]
    pts, seen = [], set()
    for kk in win:
        for p in M.kfs[kk].mp:
            if p >= 0 and int(p) not in seen:
                seen.add(int(p)); pts.append(int(p))
    for p in (pts[len(pts) // 3], pts[len(pts) // 3 + 1], pts[2 * len(pts) // 3]):
        no_observations(M, p)
    hub = [p for p in pts[5:] if len(M.pts[p].obs) >= 4][:3]
    plant_cascade(M, hub, LM.plant_outliers)
    return (M, k, 40, False, False)


def liba_cases():
    """name -> (builder, wanted shape) for local_inertial_ba_map_batch; liba_shape gives the shape of a case."""
    c = {}
    c['probe_skip'] = (lambda: _probe_skip(201), dict(nCand_min=WT + 1, skips_min=1, bad_step=True))
    c['cap_at_511'] = (lambda: _cap_at(202, 511, 612), dict(cap_at=511))
    c['cap_at_512'] = (lambda: _cap_at(203, 512, 612), dict(cap_at=512))
    c['cap_at_last'] = (lambda: _cap_at(204, 399, 400), dict(cap_at=399, nCand=400))
    c['fix_199'] = (lambda: _fix199(205), dict(nFix=199, nCand=600, skips_min=1))
    for t in (511, 512, 513, 5000):
        c['ne_%d' % t] = (lambda t=t: _liba_edges(210 + t, t), dict(nE=t, N=25))
    c['nl_600'] = (lambda: _liba_nl(221, 800), dict(nL_min=WT + 1))
    c['nl_1100'] = (lambda: _liba_nl(222, 1500), dict(nL_min=2 * WT + 1))
    c['empty_cascade'] = (lambda: _liba_empty_cascade(223), dict(empty_kf=1, empty_pt=3, cascade=True))
    return c


def liba_shape(m, r):
    """The walk's quantities of flattened map m from a record r of it (optKF, fixedKF, localPoint, nLists): Qs, Qo, nL, N, nE, the
    candidates and the probe's steps (the candidate of each added keyframe, tile skips, a step that adds none), empty segments."""
    ss, os_, kf = m['slotStart'], m['obsStart'], m['kfFlags']
    nd = LM.nd(int(m['keyFramesInMap']), bool(m['bLarge']))
    chain = [0]
    for _ in range(1, nd):
        if m['prevKF'][chain[-1]] < 0:
            break
        chain.append(int(m['prevKF'][chain[-1]]))
    pts = [int(p) for p in r['localPoint']]
    mark = set(chain) | {int(r['fixedKF'][0])}
    unm = lambda p: any(int(m['obsKF'][o]) not in mark for o in range(os_[p], os_[p + 1]))
    cand = [p for p in pts if unm(p)]
    fixed, steps, skips, bad_step, c0 = [int(r['fixedKF'][0])], [], 0, False, 0
    while c0 < len(cand) and len(fixed) < MAXFIX:
        f = next((c for c in range(c0, min(c0 + WT, len(cand))) if unm(cand[c])), None)
        if f is None:
            skips += 1
            c0 += WT
            continue
        added = False
        for o in range(os_[cand[f]], os_[cand[f] + 1]):
            k = int(m['obsKF'][o])
            if k in mark:
                continue
            mark.add(k)
            if not kf[k] & orb.KF_BAD:
                fixed.append(k); steps.append(f); added = True
                break
        bad_step |= not added
        c0 = f + 1
    sl = [int(ss[k + 1] - ss[k]) for k in chain]
    ol = [int(os_[p + 1] - os_[p]) for p in pts]
    return dict(Qs=sum(sl), Qo=sum(ol), nL=len(pts), N=int(r['nLists'][0]), nE=int(r['nLists'][3]), nCand=len(cand), fixed=fixed,
                nFix=len(fixed), cap_at=steps[-1] if len(fixed) == MAXFIX else None, skips=skips, bad_step=bad_step,
                empty_kf=sum(1 for i, n in enumerate(sl) if n == 0 and 0 < i < len(sl) - 1),
                empty_pt=sum(1 for i, n in enumerate(ol) if n == 0 and 0 < i < len(ol) - 1))


def meets(shape, want):
    """Whether a shape has every wanted value (name_min: at least; cascade is checked by the caller)."""
    for k, v in want.items():
        if k == 'cascade':
            continue
        if k.endswith('_min'):
            if shape[k[:-4]] < v:
                return False
        elif shape[k] != v:
            return False
    return True
