"""Tracking's per-frame loops after the last-frame search, written out literally (monocular, IMU not initialised), over pluggable
backends: TrackWithMotionModel from PoseOptimization through the "discard outliers" loop, and TrackLocalMap from SearchLocalPoints through
the statistics loop.  With the CPU oracle's functions (is_in_frustum, search_local_map, pose_optimization) they are the oracle chain; with
the library's single-frame entry points (orbm_frustum_project, orbm_search_local_map, pose_optimization_batch) they are the per-frame chain
the batched calls replace.  The glue -- index remapping, the visible / found counts, Frame::SetPose / UpdatePoseMatrices -- is the host's.
Also: seeded batch scenes with every rule of that glue planted."""
import numpy as np

F32 = np.float32


# ---- Frame::SetPose / UpdatePoseMatrices in float32, one rounding per operation (csrc/frame_pose.cuh) ----
def set_pose(pose7):
    """Sophus::SE3f(q.cast<float>(), t.cast<float>()) of a double (w, x, y, z, t) pose: the float quaternion normalised with
    n = ((x*x + y*y) + z*z) + w*w and a division of every coefficient by sqrt(n)."""
    w, x, y, z = (F32(v) for v in pose7[:4])
    n = F32(F32(F32(x * x) + F32(y * y)) + F32(z * z)) + F32(w * w)
    s = np.sqrt(F32(n))
    return np.array([w / s, x / s, y / s, z / s, pose7[4], pose7[5], pose7[6]], F32)


def pose_matrices(T):
    """(Rcw row-major [3,3], tcw, Ow) of a float (w, x, y, z, t) pose: Eigen's toRotationMatrix and -(q^-1 * t) with Sophus' rotation."""
    T = np.asarray(T, F32)
    qw, qx, qy, qz = T[:4]
    two = F32(2)
    tx, ty, tz = two * qx, two * qy, two * qz
    twx, twy, twz, txx, txy, txz = tx * qw, ty * qw, tz * qw, tx * qx, ty * qx, tz * qx
    tyy, tyz, tzz = ty * qy, tz * qy, tz * qz
    one = F32(1)
    R = np.array([[one - (tyy + tzz), txy - twz, txz + twy], [txy + twz, one - (txx + tzz), tyz - twx], [txz - twy, tyz + twx, one - (txx + tyy)]], F32)
    ix, iy, iz = -qx, -qy, -qz
    px, py, pz = T[4], T[5], T[6]
    ux, uy, uz = iy * pz - iz * py, iz * px - ix * pz, ix * py - iy * px
    ux, uy, uz = ux + ux, uy + uy, uz + uz
    cx, cy, cz = iy * uz - iz * uy, iz * ux - ix * uz, ix * uy - iy * ux
    Ow = -np.array([(px + qw * ux) + cx, (py + qw * uy) + cy, (pz + qw * uz) + cz], F32)
    return R, T[4:].copy(), Ow


# ---- the two Tracking loops over backends ----
class OracleBackend:
    def __init__(self):
        import oracle_lib as O
        self.O = O

    def frustum(self, pts, R, t, Ow, g):
        return self.O.is_in_frustum(pts, R, t, Ow, g['cam'], g['bounds'], g['logScaleFactor'], len(g['scaleFactors']), g['viewingCosLimit'], g['mbf'])

    def search(self, kps, desc, mp, g, th, match, claimed):
        return self.O.search_local_map(kps, desc, g['bounds'], g['scaleFactors'], mp, th, g['nnratio'], g['bFarPoints'], g['thFarPoints'], match, claimed)

    def pose(self, frame):
        return self.O.pose_optimization(frame)


class GpuChainBackend:
    """The library's existing single-frame entry points, each with its own upload and download."""
    def __init__(self, orb, matcher):
        self.orb, self.m = orb, matcher

    def frustum(self, pts, R, t, Ow, g):
        if len(pts['maxDistance']) == 0:
            return {k: np.zeros(0, dt) for k, dt in (('inView', np.uint8), ('projX', F32), ('projY', F32), ('depth', F32), ('level', np.int32),
                                                      ('viewCos', F32))}
        return self.m.isInFrustum(pts, R, t, Ow, g['cam'], g['bounds'], g['logScaleFactor'], len(g['scaleFactors']), g['viewingCosLimit'], g['mbf'])

    def search(self, kps, desc, mp, g, th, match, claimed):
        F = self.orb.Frame(kps, desc, g['bounds'], g['scaleFactors'])
        F.match[:] = match; F.claimed[:] = claimed
        self.m.mfNNratio = g['nnratio']
        n = self.m.SearchByProjection(F, mp, th, bool(g['bFarPoints']), g['thFarPoints'])
        match[:] = F.match; claimed[:] = F.claimed
        return n

    def pose(self, frame):
        return self.orb.PoseOptimization([frame])[0]


def _pose_frame(st, g, match, xyz, Tcw7):
    edges = np.nonzero(match >= 0)[0]
    kps = st['kps']
    return edges, dict(pose=np.asarray(Tcw7, F32).astype(np.float64), cam=np.asarray(g['cam'], F32), Xw=xyz[match[edges]].astype(np.float64),
                       obs=np.stack([kps['x'][edges], kps['y'][edges]], 1).astype(np.float64),
                       inv_sigma2=g['invLevelSigma2'][kps['octave'][edges]].astype(F32))


def motion_model_step(be, st, g, match, claimed, nmatches):
    """Optimizer::PoseOptimization(&mCurrentFrame), then the "discard outliers" loop.  match / claimed (last-frame indices) are updated
    in place; returns dict(pose7, Tcw7, discarded, nmatchesMap, nmatches)."""
    edges, frame = _pose_frame(st, g, match, st['last_xyz'], st['Tcw7'])
    r = be.pose(frame)
    Tcw7 = set_pose(r['pose']) if len(edges) >= 3 else np.asarray(st['Tcw7'], F32).copy()   # no SetPose when PoseOptimization returns early
    discarded = np.zeros(st['mcapLast'], np.uint8)
    nmatchesMap = 0
    for e, i in enumerate(edges):
        if r['outlier'][e]:
            discarded[match[i]] = 1                       # pMP->mnLastFrameSeen = mCurrentFrame.mnId
            match[i] = -1; claimed[i] = 0
            nmatches -= 1
        elif st['last_hasObs'][match[i]]:
            nmatchesMap += 1
    return dict(pose7=np.asarray(r['pose'], np.float64), Tcw7=Tcw7, discarded=discarded, nmatchesMap=nmatchesMap, nmatches=nmatches)


def local_map_step(be, st, g, match_last, discarded, Tcw7, th):
    """SearchLocalPoints, PoseOptimization, SetPose and the statistics loop of TrackLocalMap.  match_last: the frame's matches in
    last-frame indices (st['lastToLocal'] maps them); discarded: the motion-model step's marks.  Returns the batched call's outputs."""
    K, M = len(st['kps']), st['nM']
    l2l, bad, hasObs = st['lastToLocal'], st['bad'][:M], st['hasObs'][:M]
    match = np.full(K, -1, np.int32)
    visible = np.zeros(M, np.int32); found = np.zeros(M, np.int32); seen = np.zeros(M, bool)
    for i in range(K):                                    # SearchLocalPoints: the frame's own points
        m = match_last[i]
        if m < 0:
            continue
        p = l2l[m]
        if p < 0 or bad[p]:
            continue                                      # *vit = NULL
        match[i] = p; visible[p] += 1; seen[p] = True     # IncreaseVisible, mnLastFrameSeen, mbTrackInView = false
    for j in np.nonzero(discarded)[0]:
        if l2l[j] >= 0:
            seen[l2l[j]] = True
    R, t, Ow = pose_matrices(Tcw7)
    pts = {k: st[k][:M] for k in ('worldPos', 'normal', 'minDistInv', 'maxDistInv', 'maxDistance')}
    fr = be.frustum(pts, R, t, Ow, g)
    inView = (fr['inView'].astype(bool) & ~seen & ~bad.astype(bool)).astype(np.uint8)
    visible += inView
    nToMatch = int(inView.sum())
    claimed = np.zeros(K, np.uint8)
    claimed[match >= 0] = hasObs[match[match >= 0]]
    nmatches = 0
    if nToMatch > 0:
        mp = dict(inView=inView, bad=bad, depth=fr['depth'], projX=fr['projX'], projY=fr['projY'], level=np.maximum(fr['level'], 0),
                  viewCos=fr['viewCos'], hasObs=hasObs, descriptors=st['mpDesc'][:M])
        nmatches = be.search(st['kps'], st['desc'], mp, g, float(th), match, claimed)
    edges, frame = _pose_frame(st, g, match, st['worldPos'], Tcw7)
    r = be.pose(frame)
    Tout = set_pose(r['pose']) if len(edges) >= 3 else np.asarray(Tcw7, F32).copy()
    outlier = np.zeros(K, np.uint8)
    nMI = 0
    for e, i in enumerate(edges):                         # the statistics loop
        outlier[i] = r['outlier'][e]
        if not outlier[i]:
            found[match[i]] += 1
            nMI += int(hasObs[match[i]] != 0)
    return dict(match=match, claimed=claimed, outlier=outlier, visible=visible, found=found, nToMatch=nToMatch, nmatches=nmatches,
                nInliers=int(r['inliers']), nMatchesInliers=nMI, pose7=np.asarray(r['pose'], np.float64), Tcw7=Tout)


# ---- scenes ----
def _quat(rng, scale):
    w = rng.normal(0, scale, 3)
    q = np.concatenate([[1.0], 0.5 * w])
    return q / np.linalg.norm(q)


def _R(q):
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def globals_(W=640, H=480):
    sf = (1.2 ** np.arange(8)).astype(F32)
    return dict(cam=(F32(480.0), F32(482.0), F32(W / 2 - 1.5), F32(H / 2 + 2.5)), bounds=(0.0, 0.0, float(W), float(H)), scaleFactors=sf,
                invLevelSigma2=(1.0 / (sf.astype(np.float64) ** 2)).astype(F32), logScaleFactor=F32(np.log(F32(1.2))), mbf=0.0, nnratio=0.8,
                bFarPoints=0, thFarPoints=0.0, viewingCosLimit=0.5)


def stream(seed, g, M=600, K_extra=60, frac_kp=0.7, frac_last=0.6, n_wrong=12, kind='normal'):
    """One stream: local map of M points, a current frame whose keypoints sit near the projections of ~frac_kp of them, a last frame
    holding ~frac_last of those (plus points outside the local map, lastToLocal = -1), and the last-frame search's matches planted with
    n_wrong wrong ones (outliers of PoseOptimization).  Planted: a wrong match whose point has its own unmatched keypoint (the discarded
    point the local search would take), a matched point that went bad, a last-frame point without a local index, one point held at two
    keypoints.  kind: 'normal', 'empty' (no local point), 'all_seen' (every local point matched), 'few' (2 matches), 'nine' (9 matches)."""
    rng = np.random.default_rng(seed)
    W, H = g['bounds'][2], g['bounds'][3]
    fx, fy, cx, cy = (float(v) for v in g['cam'])
    if kind == 'empty':
        M = 0
    q = _quat(rng, 0.2); R = _R(q); t = rng.normal(0, 0.3, 3)
    pc = np.stack([rng.uniform(-4.5, 4.5, M), rng.uniform(-3.4, 3.4, M), rng.uniform(2.5, 12, M)], 1)
    Xw = (pc - t) @ R                                     # world = R^T (pc - t)
    Ow = -R.T @ t
    PO = Xw - Ow
    dist = np.linalg.norm(PO, axis=1)
    lvl = rng.integers(0, 8, M)
    maxD = (dist * 1.2 ** lvl * rng.uniform(1.0, 1.15, M)).astype(F32)
    normal = PO / np.maximum(dist, 1e-9)[:, None] + rng.normal(0, 0.3, (M, 3))
    normal /= np.maximum(np.linalg.norm(normal, axis=1), 1e-9)[:, None]
    normal[rng.random(M) < 0.05] *= -1
    mpDesc = rng.integers(0, 256, (M, 32), dtype=np.uint8)
    u = fx * pc[:, 0] / pc[:, 2] + cx; v = fy * pc[:, 1] / pc[:, 2] + cy
    vis = (u > 2) & (u < W - 2) & (v > 2) & (v < H - 2)
    own = np.nonzero(vis & (rng.random(M) < (1.0 if kind == 'all_seen' else frac_kp)))[0]
    own = rng.permutation(own)
    # keypoints: one per owned point (+ a duplicate of the first), plus clutter
    src = np.concatenate([own, own[:1]]) if len(own) else own
    Kp = len(src) + K_extra
    kps = np.zeros(Kp, _kp_dtype())
    kps['x'][:len(src)] = np.clip(u[src] + rng.normal(0, 0.7, len(src)), 0.5, W - 0.5)
    kps['y'][:len(src)] = np.clip(v[src] + rng.normal(0, 0.7, len(src)), 0.5, H - 0.5)
    kps['octave'][:len(src)] = lvl[src]
    kps['x'][len(src):] = rng.uniform(1, W - 1, K_extra); kps['y'][len(src):] = rng.uniform(1, H - 1, K_extra)
    kps['octave'][len(src):] = rng.integers(0, 8, K_extra)
    kps['size'] = 31; kps['angle'] = rng.uniform(0, 360, Kp); kps['response'] = 1; kps['class_id'] = -1
    desc = rng.integers(0, 256, (Kp, 32), dtype=np.uint8)
    desc[:len(src)] = mpDesc[src]
    for i in range(len(src)):
        for b in rng.integers(0, 256, rng.integers(0, 20)):
            desc[i, b >> 3] ^= np.uint8(1 << (b & 7))
    perm = rng.permutation(Kp)
    kps, desc = kps[perm], desc[perm]
    kp_src = np.full(Kp, -1); kp_src[np.argsort(perm)[:len(src)]] = src      # local point each keypoint was made from
    # last frame: a subset of the owned points, then points outside the local map
    in_last = own[: int(len(own) * (1.0 if kind == 'all_seen' else frac_last))]
    n_out = 0 if kind == 'all_seen' else 8
    mcapLast = len(in_last) + n_out
    lastToLocal = np.concatenate([in_last, np.full(n_out, -1)]).astype(np.int32)
    lperm = rng.permutation(mcapLast)
    lastToLocal = lastToLocal[lperm]
    last_xyz = np.zeros((mcapLast, 3), F32)
    loc = lastToLocal >= 0
    last_xyz[loc] = Xw[lastToLocal[loc]]
    last_xyz[~loc] = Xw[rng.integers(0, max(M, 1), (~loc).sum())] if M else rng.normal(0, 1, ((~loc).sum(), 3)) + [0, 0, 5]
    last_hasObs = (rng.random(mcapLast) > 0.1).astype(np.uint8)
    local_of_last = {int(p): j for j, p in enumerate(lastToLocal) if p >= 0}
    match = np.full(Kp, -1, np.int32)
    for i in range(Kp):
        if kp_src[i] >= 0 and kp_src[i] in local_of_last:
            match[i] = local_of_last[kp_src[i]]
    # wrong matches: keypoints of points NOT in the last frame matched to last-frame points far away whose own keypoint the search
    # left unmatched (after the discard, only the local search could give them that keypoint)
    free_kp = [i for i in range(Kp) if match[i] < 0 and kp_src[i] >= 0]
    if kind == 'normal' and len(free_kp) > n_wrong and mcapLast:
        targets = rng.choice(np.nonzero(lastToLocal >= 0)[0], n_wrong, replace=False)
        match[np.isin(match, targets)] = -1
        for i, j in zip(rng.choice(free_kp, n_wrong, replace=False), targets):
            match[i] = j
        nolocal = np.nonzero(lastToLocal < 0)[0]          # consistent matches of last-frame points without a local index (went bad)
        cand = [i for i in range(Kp) if match[i] < 0 and kp_src[i] >= 0]
        for i, j in zip(rng.choice(cand, min(3, len(cand)), replace=False), nolocal):
            match[i] = j
            last_xyz[j] = Xw[kp_src[i]]
    if kind in ('few', 'nine'):
        keep = np.nonzero(match >= 0)[0][: (2 if kind == 'few' else 9)]
        m2 = np.full(Kp, -1, np.int32); m2[keep] = match[keep]; match = m2
    bad = (rng.random(M) < 0.04).astype(np.uint8)
    if kind == 'all_seen':                                # the frame holds every good local point
        bad[:] = 1; bad[own] = 0
    hasObs = (rng.random(M) > 0.08).astype(np.uint8)
    if M and kind == 'normal':                            # a matched point that went bad
        mm = [local_of_last_j for local_of_last_j in lastToLocal[match[match >= 0]] if local_of_last_j >= 0]
        if mm:
            bad[mm[0]] = 1
    claimed = np.zeros(Kp, np.uint8)
    claimed[match >= 0] = last_hasObs[match[match >= 0]]
    Tt = np.concatenate([q, t])
    T0 = Tt.copy(); T0[4:] += rng.normal(0, 0.01, 3); qq = T0[:4] + rng.normal(0, 0.002, 4); T0[:4] = qq / np.linalg.norm(qq)
    return dict(kps=kps, desc=desc, nM=M, worldPos=Xw.astype(F32), normal=normal.astype(F32), minDistInv=(F32(0.8) * (maxD / F32(1.2 ** 7))).astype(F32),
                maxDistInv=(F32(1.2) * maxD).astype(F32), maxDistance=maxD, mpDesc=mpDesc, hasObs=hasObs, bad=bad, lastToLocal=lastToLocal,
                mcapLast=mcapLast, last_xyz=last_xyz, last_hasObs=last_hasObs, match=match, claimed=claimed, nmatches=int((match >= 0).sum()),
                Tcw7=T0.astype(F32))


def _kp_dtype():
    return np.dtype([('x', 'f4'), ('y', 'f4'), ('size', 'f4'), ('angle', 'f4'), ('response', 'f4'), ('octave', 'i4'), ('class_id', 'i4')])


def batch(streams, g, th, active=None, kcap=None, mcap=None, mcapLast=None):
    """Pads per-stream dicts into the [batch][cap] slabs of the batched calls.  Returns (motion dict, local-map dict, state) where state
    holds match / claimed / nmatches [B, kcap]."""
    B = len(streams)
    kcap = kcap or max(1, max(len(s['kps']) for s in streams))
    mcap = mcap or max(1, max(s['nM'] for s in streams))
    mL = mcapLast or max(1, max(s['mcapLast'] for s in streams))
    kps = np.zeros((B, kcap), _kp_dtype()); desc = np.zeros((B, kcap, 32), np.uint8)
    match = np.full((B, kcap), -1, np.int32); claimed = np.zeros((B, kcap), np.uint8)
    lx = np.zeros((B, mL, 3), F32); lo = np.zeros((B, mL), np.uint8); l2l = np.full((B, mL), -1, np.int32)
    arr = {k: np.zeros((B, mcap) + sh, dt) for k, sh, dt in (('worldPos', (3,), F32), ('normal', (3,), F32), ('minDistInv', (), F32), ('maxDistInv', (), F32),
                                                              ('maxDistance', (), F32), ('mpDesc', (32,), np.uint8), ('hasObs', (), np.uint8), ('bad', (), np.uint8))}
    for b, s in enumerate(streams):
        K, M, ML = len(s['kps']), s['nM'], s['mcapLast']
        kps[b, :K] = s['kps']; desc[b, :K] = s['desc']; match[b, :K] = s['match']; claimed[b, :K] = s['claimed']
        lx[b, :ML] = s['last_xyz']; lo[b, :ML] = s['last_hasObs']; l2l[b, :ML] = s['lastToLocal']
        for k in arr:
            arr[k][b, :M] = s[k][:M]
    nK = np.array([len(s['kps']) for s in streams], np.int32)
    nM = np.array([s['nM'] for s in streams], np.int32)
    T = np.stack([s['Tcw7'] for s in streams]).astype(F32)
    motion = dict(batch=B, kcap=kcap, mcap=mL, nlevels=8, kps=kps, nK=nK, xyz=lx, hasObs=lo, Tcw7=T, cam=tuple(float(c) for c in g['cam']))
    local = dict(batch=B, kcap=kcap, mcap=mcap, mcapLast=mL, nlevels=8, kps=kps, desc=desc, nK=nK, bounds=g['bounds'], scaleFactors=g['scaleFactors'],
                 invLevelSigma2=g['invLevelSigma2'], cam=tuple(float(c) for c in g['cam']), mbf=g['mbf'], logScaleFactor=g['logScaleFactor'], Tcw7=T.copy(),
                 lastToLocal=l2l, discarded=None, nM=nM, th=np.asarray(th, F32), nnratio=g['nnratio'], bFarPoints=g['bFarPoints'],
                 thFarPoints=g['thFarPoints'], viewingCosLimit=g['viewingCosLimit'], active=active, **arr)
    state = dict(match=match, claimed=claimed, nmatches=np.array([s['nmatches'] for s in streams], np.int32))
    return motion, local, state
