"""Tracking::TrackReferenceKeyFrame (monocular), written out literally over the backends of tests/track_lib.py: with the CPU oracle's
functions (bow_transform, search_by_bow, pose_optimization) it is the oracle chain; with the library's existing entry points
(orbv_transform_batch, orbm_search_by_bow, pose_optimization_batch) it is the per-frame chain orbm_track_reference_keyframe_batch*
replaces.  Also: seeded scenes of a reference keyframe and a frame with every rule of the glue planted, their [batch][cap] slabs, and the
index space [keyframe features | last-frame points] in which such a stream joins orbm_track_local_map_batch*."""
import numpy as np

import track_lib as T
from track_lib import F32, _kp_dtype, _pose_frame, _quat, _R, set_pose


class OracleBackend(T.OracleBackend):
    """track_lib's oracle backend plus Frame::ComputeBoW and SearchByBoW with ORBmatcher(0.7, true)."""
    def __init__(self, voc=None):
        super().__init__()
        self.voc = voc

    def feature_vector(self, desc):
        return self.O.bow_transform(self.voc, desc, 4)[2:]

    def search_bow(self, kf_kps, kf_desc, kf_point, kf_fv, kps, desc, fv):
        return self.O.search_by_bow(kf_kps, kf_desc, kf_point, kf_fv, kps, desc, fv, nnratio=0.7, check_ori=True)


class GpuChainBackend(T.GpuChainBackend):
    """track_lib's per-frame GPU chain plus orbv_transform_batch and orbm_search_by_bow, each with its own upload and download."""
    def __init__(self, orb, matcher, voc=None):
        super().__init__(orb, matcher)
        self.voc = None if voc is None else orb.ORBVocabulary(voc['L'], voc['child_start'], voc['children'], voc['desc'], voc['weight'], voc['word_id'])

    def feature_vector(self, desc):
        return self.voc.transform([desc], 4)[0][2:]                   # orbv_transform_batch

    def search_bow(self, kf_kps, kf_desc, kf_point, kf_fv, kps, desc, fv):
        self.m.mfNNratio, self.m.mbCheckOrientation = 0.7, True       # ORBmatcher matcher(0.7, true)
        return self.m.SearchByBoW(kf_kps, kf_desc, kf_point, kf_fv, kps, desc, fv)


# ---- Tracking::TrackReferenceKeyFrame ----
REF_MIN_MATCHES = 15                                      # if(nmatches<15) return false;


def reference_keyframe_step(be, st, g):
    """Frame::ComputeBoW, then TrackReferenceKeyFrame: SearchByBoW(mpReferenceKF, mCurrentFrame) with ORBmatcher(0.7, true); below 15
    matches the frame is left as it was; otherwise mvpMapPoints = the matches, SetPose(mLastFrame.GetPose()), PoseOptimization and the
    "discard outliers" loop (pMP->mnLastFrameSeen = current frame for an outlier's point).  Returns dict(nmatches (the search's return
    value, which the call returns), match (keyframe feature indices), gated) and, for a gated stream, pose7, Tcw7, discarded [nKF] and
    nmatchesMap."""
    fv, kf_fv = be.feature_vector(st['desc']), be.feature_vector(st['kf_desc'])
    n, match = be.search_bow(st['kf_kps'], st['kf_desc'], st['kfPoint'], kf_fv, st['kps'], st['desc'], fv)
    out = dict(nmatches=int(n), match=np.asarray(match, np.int32).copy(), gated=n >= REF_MIN_MATCHES, fv=fv, kf_fv=kf_fv)
    if not out['gated']:
        return out
    match = out['match']
    edges, frame = _pose_frame(st, g, match, st['kf_xyz'], st['Tcw7_last'])
    r = be.pose(frame)
    Tcw7 = set_pose(r['pose']) if len(edges) >= 3 else np.asarray(st['Tcw7_last'], F32).copy()
    discarded = np.zeros(len(st['kf_kps']), np.uint8)
    nmatchesMap = 0
    for e, i in enumerate(edges):
        if r['outlier'][e]:
            discarded[match[i]] = 1                       # mvpMapPoints[i] = NULL, pMP->mnLastFrameSeen = mCurrentFrame.mnId
            match[i] = -1
        elif st['kf_hasObs'][match[i]]:
            nmatchesMap += 1
    out.update(pose7=np.asarray(r['pose'], np.float64), Tcw7=Tcw7, discarded=discarded, nmatchesMap=nmatchesMap)
    return out


def ref_vocabulary():
    """L = 6, k = 5 (~20k nodes): with levelsup = 4 the FeatureVector groups features at level 2, as ORBvoc does."""
    import oracle_lib as O
    return O.synthetic_vocabulary(5, 6, seed=56)


def _flip(rng, d, nmax):
    d = d.copy()
    for b in rng.integers(0, 256, rng.integers(0, nmax + 1)):
        d[b >> 3] ^= np.uint8(1 << (b & 7))
    return d


def ref_kf_stream(seed, g, voc, kind='normal', M=500, K_extra=60, kf_clutter=40, n_wrong=8, n_rot=5, frac_kf=0.7, frac_seen=0.75):
    """One stream of the reference-keyframe path: a local map of M points, a reference keyframe observing ~frac_kf of the visible ones
    (plus features without a point and features of bad points), a frame with keypoints near the projections of ~frac_seen of the
    keyframe's points (descriptors a few bits from the keyframe's), of the local points the keyframe does not see, and clutter.  Planted:
    n_wrong keyframe descriptors copied to keypoints far from their point (PoseOptimization's outliers), n_rot matches rotated into a
    minority histogram bin, points without observations.  A last frame holds some of the frame's points (the motion-model step's input).
    kind: 'normal'; 'n14' / 'n15' (exactly 14 / 15 matches); 'map9' (gate passed, nmatchesMap < 10); 'fallback' (the motion-model step
    ran PoseOptimization, failed with nmatchesMap < 10 and discarded points the BoW search cannot rematch: the keyframe does not see them,
    and each has its own keypoint the local search would take)."""
    import oracle_lib as O
    rng = np.random.default_rng(seed)
    W, H = g['bounds'][2], g['bounds'][3]
    fx, fy, cx, cy = (float(v) for v in g['cam'])
    q = _quat(rng, 0.2); R = _R(q); t = rng.normal(0, 0.3, 3)
    pc = np.stack([rng.uniform(-4.5, 4.5, M) * W / 640, rng.uniform(-3.4, 3.4, M) * H / 480, rng.uniform(2.5, 12, M)], 1)
    Xw = (pc - t) @ R
    Ow = -R.T @ t
    PO = Xw - Ow
    dist = np.linalg.norm(PO, axis=1)
    lvl = rng.integers(0, 8, M)
    maxD = (dist * 1.2 ** lvl * rng.uniform(1.0, 1.15, M)).astype(F32)
    normal = PO / dist[:, None]
    mpDesc = rng.integers(0, 256, (M, 32), dtype=np.uint8)
    hasObs = (rng.random(M) > 0.1).astype(np.uint8)
    u = fx * pc[:, 0] / pc[:, 2] + cx; v = fy * pc[:, 1] / pc[:, 2] + cy
    vis = np.nonzero((u > 2) & (u < W - 2) & (v > 2) & (v < H - 2))[0]
    vis = rng.permutation(vis)
    kf_pts, extra = vis[: int(frac_kf * len(vis))], vis[int(frac_kf * len(vis)):]
    if kind in ('n14', 'n15'):
        kf_pts = kf_pts[:40]; n_wrong = n_rot = 0
    if kind == 'map9':
        hasObs[kf_pts[5:]] = 0
    # keyframe features: its points, bad points, features without a point
    n_bad = 6
    nKF = len(kf_pts) + n_bad + kf_clutter
    kf_src = np.concatenate([kf_pts, np.full(n_bad + kf_clutter, -1)]).astype(np.int64)
    kfPoint = np.concatenate([np.ones(len(kf_pts)), np.full(n_bad, 2), np.zeros(kf_clutter)]).astype(np.uint8)
    kf_desc = rng.integers(0, 256, (nKF, 32), dtype=np.uint8)
    for j in range(len(kf_pts)):
        kf_desc[j] = _flip(rng, mpDesc[kf_pts[j]], 4)
    kf_kps = np.zeros(nKF, _kp_dtype())
    kf_kps['x'] = rng.uniform(1, W - 1, nKF); kf_kps['y'] = rng.uniform(1, H - 1, nKF); kf_kps['octave'] = rng.integers(0, 8, nKF)
    kf_kps['angle'] = rng.uniform(0, 360, nKF); kf_kps['size'] = 31; kf_kps['response'] = 1; kf_kps['class_id'] = -1
    kf_xyz = np.zeros((nKF, 3), F32); kf_xyz[:len(kf_pts)] = Xw[kf_pts]; kf_xyz[len(kf_pts):len(kf_pts) + n_bad] = rng.normal(0, 2, (n_bad, 3))
    kf_hasObs = np.zeros(nKF, np.uint8); kf_hasObs[:len(kf_pts)] = hasObs[kf_pts]; kf_hasObs[len(kf_pts):len(kf_pts) + n_bad] = 1
    # frame: true correspondences (some rotated), wrong ones, keypoints of points the keyframe does not see, clutter
    n_seen = int(frac_seen * len(kf_pts)) if kind not in ('n14', 'n15') else 21
    seen_j = np.arange(n_seen)
    wrong_j = np.arange(n_seen, min(n_seen + n_wrong, len(kf_pts)))
    rows = []                                             # (x, y, octave, angle, desc, local point or -1)
    for k, j in enumerate(seen_j):
        p = kf_pts[j]
        ang = kf_kps['angle'][j] + rng.normal(0, 3) + (150.0 if k < n_rot else 0.0)
        rows.append((u[p] + rng.normal(0, 0.7), v[p] + rng.normal(0, 0.7), lvl[p], ang % 360, _flip(rng, kf_desc[j], 5), p))
    for j in wrong_j:
        rows.append((rng.uniform(1, W - 1), rng.uniform(1, H - 1), rng.integers(0, 8), (kf_kps['angle'][j] + rng.normal(0, 3)) % 360,
                     _flip(rng, kf_desc[j], 5), -1))
    for p in extra:
        rows.append((u[p] + rng.normal(0, 0.7), v[p] + rng.normal(0, 0.7), lvl[p], rng.uniform(0, 360), _flip(rng, mpDesc[p], 8), p))
    for _ in range(K_extra):
        rows.append((rng.uniform(1, W - 1), rng.uniform(1, H - 1), rng.integers(0, 8), rng.uniform(0, 360), rng.integers(0, 256, 32, dtype=np.uint8), -1))
    perm = rng.permutation(len(rows))
    rows = [rows[i] for i in perm]
    Kp = len(rows)
    kps = np.zeros(Kp, _kp_dtype())
    kps['x'] = np.clip([r[0] for r in rows], 0.5, W - 0.5); kps['y'] = np.clip([r[1] for r in rows], 0.5, H - 0.5)
    kps['octave'] = [r[2] for r in rows]; kps['angle'] = [r[3] for r in rows]; kps['size'] = 31; kps['response'] = 1; kps['class_id'] = -1
    desc = np.stack([r[4] for r in rows]).astype(np.uint8)
    kp_src = np.array([r[5] for r in rows])
    kperm = rng.permutation(nKF)                          # keyframe features in a shuffled order
    kf_kps, kf_desc, kfPoint, kf_xyz, kf_hasObs, kf_src = kf_kps[kperm], kf_desc[kperm], kfPoint[kperm], kf_xyz[kperm], kf_hasObs[kperm], kf_src[kperm]
    fv, kf_fv = O.bow_transform(voc, desc, 4)[2:], O.bow_transform(voc, kf_desc, 4)[2:]
    if kind in ('n14', 'n15'):                            # drop the points of matched keyframe features until the count is exact
        target = 14 if kind == 'n14' else 15
        while True:
            n, match = O.search_by_bow(kf_kps, kf_desc, kfPoint, kf_fv, kps, desc, fv, 0.7, True)
            if n <= target:
                break
            kfPoint[match[match >= 0][: n - target]] = 0
        assert n == target, (kind, n)
    kfToLocal = np.where(kfPoint == 1, kf_src, -1).astype(np.int32)
    # last frame: some of the frame's points; with 'fallback' the motion-model step ran and failed
    own = [p for p in kp_src if p >= 0]
    in_last = np.array(own[:30] + [p for p in extra[:4] if p not in own[:30]], np.int64)
    mcapLast = len(in_last)
    lastToLocal = in_last.astype(np.int32)
    last_xyz = Xw[in_last].astype(F32)
    last_hasObs = hasObs[in_last].copy()
    local_of_last = {int(p): j for j, p in enumerate(in_last)}
    match_mm = np.full(Kp, -1, np.int32)
    if kind == 'fallback':
        last_hasObs[:] = 0; last_hasObs[:5] = 1           # nmatchesMap < 10 after the motion-model PoseOptimization
        for i in range(Kp):
            if kp_src[i] >= 0 and kp_src[i] in local_of_last:
                match_mm[i] = local_of_last[int(kp_src[i])]
        clutter = [i for i in range(Kp) if kp_src[i] < 0 and match_mm[i] < 0]
        for i, p in zip(rng.choice(clutter, 3, replace=False), [p for p in extra[:4] if int(p) in local_of_last][:3]):
            match_mm[match_mm == local_of_last[int(p)]] = -1
            match_mm[i] = local_of_last[int(p)]            # a wrong match: its point is discarded, its own keypoint stays free
    claimed = np.zeros(Kp, np.uint8)
    claimed[match_mm >= 0] = last_hasObs[match_mm[match_mm >= 0]]
    bad = np.zeros(M, np.uint8)
    Tt = np.concatenate([q, t])
    T0 = Tt.copy(); T0[4:] += rng.normal(0, 0.01, 3); qq = T0[:4] + rng.normal(0, 0.002, 4); T0[:4] = qq / np.linalg.norm(qq)
    return dict(kind=kind, kps=kps, desc=desc, fv=fv, kp_src=kp_src, kf_kps=kf_kps, kf_desc=kf_desc, kf_fv=kf_fv, kfPoint=kfPoint, kf_xyz=kf_xyz,
                kf_hasObs=kf_hasObs, kfToLocal=kfToLocal, nM=M, worldPos=Xw.astype(F32), normal=normal.astype(F32),
                minDistInv=(F32(0.8) * (maxD / F32(1.2 ** 7))).astype(F32), maxDistInv=(F32(1.2) * maxD).astype(F32), maxDistance=maxD, mpDesc=mpDesc,
                hasObs=hasObs, bad=bad, lastToLocal=lastToLocal, mcapLast=mcapLast, last_xyz=last_xyz, last_hasObs=last_hasObs, match=match_mm,
                claimed=claimed, nmatches=int((match_mm >= 0).sum()), Tcw7=T0.astype(F32), Tcw7_last=T0.astype(F32))


def ref_batch(streams, g, active=None, kcap=None, mcap=None):
    """Pads reference-keyframe streams into the [batch][cap] slabs of orbm_track_reference_keyframe_batch* (host numpy)."""
    B = len(streams)
    kcap = kcap or max(1, max(len(s['kps']) for s in streams))
    mcap = mcap or max(1, max(len(s['kf_kps']) for s in streams))
    d = dict(batch=B, kcap=kcap, mcap=mcap, nlevels=8, cam=tuple(float(c) for c in g['cam']), invLevelSigma2=g['invLevelSigma2'], active=active,
             kps=np.zeros((B, kcap), _kp_dtype()), desc=np.zeros((B, kcap, 32), np.uint8), nK=np.zeros(B, np.int32),
             fvNode=np.zeros((B, kcap), np.int32), fvFeature=np.zeros((B, kcap), np.int32), nEntries=np.zeros(B, np.int32),
             Tcw7=np.stack([s['Tcw7_last'] for s in streams]).astype(F32), kfN=np.zeros(B, np.int32), kfKps=np.zeros((B, mcap), _kp_dtype()),
             kfDesc=np.zeros((B, mcap, 32), np.uint8), kfFvNode=np.zeros((B, mcap), np.int32), kfFvFeature=np.zeros((B, mcap), np.int32),
             kfNEntries=np.zeros(B, np.int32), kfPoint=np.zeros((B, mcap), np.uint8), xyz=np.zeros((B, mcap, 3), F32), hasObs=np.zeros((B, mcap), np.uint8))
    for b, s in enumerate(streams):
        K, N, e, ek = len(s['kps']), len(s['kf_kps']), len(s['fv'][0]), len(s['kf_fv'][0])
        d['kps'][b, :K] = s['kps']; d['desc'][b, :K] = s['desc']; d['nK'][b] = K
        d['fvNode'][b, :e], d['fvFeature'][b, :e] = s['fv']; d['nEntries'][b] = e
        d['kfKps'][b, :N] = s['kf_kps']; d['kfDesc'][b, :N] = s['kf_desc']; d['kfN'][b] = N
        d['kfFvNode'][b, :ek], d['kfFvFeature'][b, :ek] = s['kf_fv']; d['kfNEntries'][b] = ek
        d['kfPoint'][b, :N] = s['kfPoint']; d['xyz'][b, :N] = s['kf_xyz']; d['hasObs'][b, :N] = s['kf_hasObs']
    return d


def concat_index_space(streams, mcapKF, mcapLast, ref_discarded, mm_discarded):
    """lastToLocal / discarded rows of orbm_track_local_map_batch* for streams that went through the reference keyframe: [keyframe
    features (mcapKF) | last-frame points (mcapLast)].  mm_discarded[b]: the failed motion-model step's marks, or None."""
    B = len(streams)
    l2l = np.full((B, mcapKF + mcapLast), -1, np.int32); dis = np.zeros((B, mcapKF + mcapLast), np.uint8)
    for b, s in enumerate(streams):
        l2l[b, :len(s['kfToLocal'])] = s['kfToLocal']; l2l[b, mcapKF:mcapKF + s['mcapLast']] = s['lastToLocal']
        dis[b, :mcapKF] = ref_discarded[b][:mcapKF]
        if mm_discarded[b] is not None:
            dis[b, mcapKF:mcapKF + s['mcapLast']] = mm_discarded[b]
    return l2l, dis
