"""Tracking's mono-inertial step once the IMU is initialised, written out literally over pluggable backends: PredictStateIMU, then
TrackLocalMap from SearchLocalPoints (the frame holds no point) through PoseInertialOptimizationLast{KeyFrame,Frame}, its write-back
(SetImuPoseVelocity, mImuBias, mpcpi = ConstraintPoseImu) and the statistics loop.  With the CPU oracle's functions it is the oracle chain;
with the library's single-frame entry points (orbm_frustum_project, orbm_search_local_map, pose_inertial_optimization_last_{kf,frame}_batch)
it is the per-frame chain orbm_track_local_map_inertial_batch* replaces.  The float glue is numpy float32 with one rounding per operation,
restating csrc/frame_pose.cuh.  Also: seeded scenes around the synthetic IMU trajectory."""
import numpy as np

import track_lib as T
from orb_slam3_modified_b200 import synth

F32 = np.float32
G = F32(9.81)


# ---- float32 restatements (csrc/frame_pose.cuh, oracle/ref_shim/ref_slam_types.cpp) ----
def _rotate(q, p):
    ux, uy, uz = q[2] * p[2] - q[3] * p[1], q[3] * p[0] - q[1] * p[2], q[1] * p[1] - q[2] * p[0]
    ux, uy, uz = ux + ux, uy + uy, uz + uz
    cx, cy, cz = q[2] * uz - q[3] * uy, q[3] * ux - q[1] * uz, q[1] * uy - q[2] * ux
    return [(p[0] + q[0] * ux) + cx, (p[1] + q[0] * uy) + cy, (p[2] + q[0] * uz) + cz]


def se3_from_matrix(R, t):
    """Sophus::SE3f(Matrix3f, Vector3f): Eigen's quaternion from a rotation matrix, not normalised."""
    R = np.asarray(R, F32).reshape(3, 3)
    tr = (R[0, 0] + R[1, 1]) + R[2, 2]
    q = [F32(0)] * 4
    if tr > 0:
        tr = np.sqrt(tr + F32(1))
        q[0] = F32(0.5) * tr; tr = F32(0.5) / tr
        q[1] = (R[2, 1] - R[1, 2]) * tr; q[2] = (R[0, 2] - R[2, 0]) * tr; q[3] = (R[1, 0] - R[0, 1]) * tr
    else:
        i = 0
        if R[1, 1] > R[0, 0]:
            i = 1
        if R[2, 2] > R[i, i]:
            i = 2
        j, k = (i + 1) % 3, (i + 2) % 3
        tr = np.sqrt(((R[i, i] - R[j, j]) - R[k, k]) + F32(1))
        v = [F32(0)] * 3
        v[i] = F32(0.5) * tr; tr = F32(0.5) / tr
        q[0] = (R[k, j] - R[j, k]) * tr
        v[j] = (R[j, i] + R[i, j]) * tr; v[k] = (R[k, i] + R[i, k]) * tr
        q[1:] = v
    return q + [F32(x) for x in np.asarray(t, F32)]


def se3_inverse(Tq):
    q = [Tq[0], -Tq[1], -Tq[2], -Tq[3]]
    r = _rotate(q, Tq[4:])
    return q + [-r[0], -r[1], -r[2]]


def se3_mul(A, B):
    w, x, y, z = A[:4]
    r = _rotate(A, B[4:])
    return [((w * B[0] - x * B[1]) - y * B[2]) - z * B[3], ((w * B[1] + x * B[0]) + y * B[3]) - z * B[2],
            ((w * B[2] + y * B[0]) + z * B[1]) - x * B[3], ((w * B[3] + z * B[0]) + x * B[2]) - y * B[1],
            r[0] + A[4], r[1] + A[5], r[2] + A[6]]


def set_imu_pose(Tcb7, Rwb, twb):
    """Frame::SetImuPoseVelocity's pose part and what ImuCamPose(Frame*) reads back: (Tcw7, GetImuRotation [9], GetImuPosition [3])."""
    Tcb = [F32(v) for v in np.asarray(Tcb7, F32)]
    Tcw = np.array(se3_mul(Tcb, se3_inverse(se3_from_matrix(Rwb, twb))), F32)
    Rcw, _, Ow = T.pose_matrices(Tcw)
    Rcb, tcb, _ = T.pose_matrices(np.asarray(Tcb7, F32))
    Rimu = np.zeros((3, 3), F32); timu = np.zeros(3, F32)
    for i in range(3):
        for j in range(3):
            Rimu[i, j] = (Rcw[0, i] * Rcb[0, j] + Rcw[1, i] * Rcb[1, j]) + Rcw[2, i] * Rcb[2, j]
        timu[i] = ((Rcw[0, i] * tcb[0] + Rcw[1, i] * tcb[1]) + Rcw[2, i] * tcb[2]) + Ow[i]
    return Tcw, Rimu.reshape(9), timu


def normalize_rotation(M):
    U, _, Vt = np.linalg.svd(np.asarray(M, np.float64).reshape(3, 3))
    return U @ Vt


def predict_state(O, Tcb7, S, P):
    """Tracking::PredictStateIMU from state S [21] (Rwb | twb | v | bg | ba, float) and its preintegration P, then SetImuPoseVelocity.
    The deltas come from the oracle (GetDeltaRotation / Velocity / Position, float); the products are float32 and the outer
    NormalizeRotation a float64 SVD, so this agrees with the device to float rounding, not bit for bit.  Returns (predState21, predTcw7)."""
    S = np.asarray(S, F32)
    dR, dV, dP = O.imu_delta(P, S[15:18].astype(np.float64), S[18:21].astype(np.float64))
    dR, dV, dP = dR.astype(F32), dV.astype(F32), dP.astype(F32)
    R1, t1, V1 = S[:9].reshape(3, 3), S[9:12], S[12:15]
    t12 = F32(P[0])
    Rwb2 = normalize_rotation(R1 @ dR).astype(F32)
    h = (F32(0.5) * t12) * t12
    Gz = np.array([0, 0, -G], F32)
    twb2 = ((t1 + V1 * t12) + h * Gz) + R1 @ dP
    Vwb2 = (V1 + t12 * Gz) + R1 @ dV
    Tcw, Rimu, timu = set_imu_pose(Tcb7, Rwb2, twb2)
    return np.concatenate([Rimu, timu, Vwb2, S[15:21]]).astype(F32), Tcw


def predict_state_f64(S, P, O):
    """The same prediction in float64 throughout (the body state, not the frame read-back): (Rwb2, twb2, Vwb2)."""
    S = np.asarray(S, np.float64)
    dR, dV, dP = O.imu_delta(P, S[15:18], S[18:21])
    R1, t1, V1, t12 = S[:9].reshape(3, 3), S[9:12], S[12:15], float(P[0])
    Gz = np.array([0, 0, -9.81])
    return normalize_rotation(R1 @ dR), t1 + V1 * t12 + 0.5 * t12 * t12 * Gz + R1 @ dP, V1 + t12 * Gz + R1 @ dV


# ---- backends ----
class OracleBackend(T.OracleBackend):
    def pose_kf(self, pr, preint):
        return self.O.pose_inertial_opt_last_kf(pr, preint)

    def pose_lf(self, pr, P_frame, P_kf):
        return self.O.pose_inertial_opt_last_frame(pr, P_frame, P_kf)

    def constraint(self, H):
        return self.O.constraint_pose_imu_information(H)


class GpuChainBackend(T.GpuChainBackend):
    """The library's existing single-frame entry points; ConstraintPoseImu's constructor is the oracle's (no single-frame entry point)."""
    def pose_kf(self, pr, preint):
        return self.orb.PoseInertialOptimizationLastKeyFrame([dict(pr, preint=preint)], pr['extr'])[0]

    def pose_lf(self, pr, P_frame, P_kf):
        return self.orb.PoseInertialOptimizationLastFrame([dict(pr, preint_frame=P_frame, preint_kf=P_kf)], pr['extr'])[0]

    def constraint(self, H):
        import oracle_lib as O
        return O.constraint_pose_imu_information(H)


def local_map_step(be, st, g, rig, mode, pred, predTcw7, th):
    """SearchLocalPoints with the frame holding nothing, the inertial optimiser of `mode` (1: last keyframe, 2: last frame) and the
    write-back.  pred / predTcw7: the frame after PredictStateIMU.  Returns the batched call's outputs for this stream."""
    K, M = len(st['kps']), st['nM']
    bad, hasObs = st['bad'][:M], st['hasObs'][:M]
    R, t, Ow = T.pose_matrices(predTcw7)
    pts = {k: st[k][:M] for k in ('worldPos', 'normal', 'minDistInv', 'maxDistInv', 'maxDistance')}
    fr = be.frustum(pts, R, t, Ow, g)
    inView = (fr['inView'].astype(bool) & ~bad.astype(bool)).astype(np.uint8)   # no point is seen before the frustum test
    visible = inView.astype(np.int32)
    nToMatch = int(inView.sum())
    match = np.full(K, -1, np.int32); claimed = np.zeros(K, np.uint8)
    nmatches = 0
    if nToMatch > 0:
        mp = dict(inView=inView, bad=bad, depth=fr['depth'], projX=fr['projX'], projY=fr['projY'], level=np.maximum(fr['level'], 0),
                  viewCos=fr['viewCos'], hasObs=hasObs, descriptors=st['mpDesc'][:M])
        nmatches = be.search(st['kps'], st['desc'], mp, g, float(th), match, claimed)
    edges = np.nonzero(match >= 0)[0]
    kps = st['kps']
    pr = dict(Xw=st['worldPos'][match[edges]].astype(F32).reshape(-1, 3), obs=np.stack([kps['x'][edges], kps['y'][edges]], 1).astype(F32).reshape(-1, 2),
              inv_sigma2=g['invLevelSigma2'][kps['octave'][edges]].astype(F32), track_depth=fr['depth'][match[edges]].astype(F32),
              cam=np.asarray(g['cam'], F32), extr=rig['extr'], state=np.asarray(pred, F32).astype(np.float64))
    if mode == 1:
        pr['kf_state'] = st['kfState21'].astype(np.float64)
        r = be.pose_kf(pr, st['preintKF'])
    else:
        pr.update(prev_state=st['lastState21'].astype(np.float64), prior_state=st['prior21'], prior_H=st['priorH'])
        r = be.pose_lf(pr, st['preintFrame'], st['preintKF'])
    s = np.asarray(r['state'], np.float64)
    Tcw7, Rimu, timu = set_imu_pose(rig['Tcb7'], s[:9].astype(F32), s[9:12].astype(F32))
    state21 = np.concatenate([Rimu, timu, s[12:21].astype(F32)]).astype(F32)
    outlier = np.zeros(K, np.uint8); found = np.zeros(M, np.int32)
    nMI = 0
    for e, i in enumerate(edges):                          # the statistics loop
        outlier[i] = r['outlier'][e]
        if not outlier[i]:
            found[match[i]] += 1
            nMI += int(hasObs[match[i]] != 0)
    return dict(match=match, claimed=claimed, outlier=outlier, visible=visible, found=found, nToMatch=nToMatch, nmatches=nmatches,
                nInliers=int(r['ret']), nMatchesInliers=nMI, Tcw7=Tcw7, state21=state21, prior21=s.copy(),
                priorH=be.constraint(np.asarray(r['H']).reshape(15, 15)), N=len(edges))


# ---- scenes ----
def rig():
    """Tcb7 (float quaternion + t) of synth's IMU rig and the optimisers' extrinsics24 as the doubles of the same floats."""
    ex = synth.imu_extrinsics()
    Rcb = ex[:9].reshape(3, 3)
    q = np.array(se3_from_matrix(Rcb.astype(F32), ex[9:12].astype(F32)), F32)
    q[:4] /= np.linalg.norm(q[:4].astype(np.float64)).astype(F32)
    Rf, tf, _ = T.pose_matrices(q)
    Rbc = Rf.T
    tbc = -(Rbc.astype(np.float64) @ tf.astype(np.float64)).astype(F32)
    return dict(Tcb7=q, extr=np.concatenate([Rf.reshape(9), tf, Rbc.reshape(9), tbc]).astype(np.float64))


def _state(R, p, v, bias6):
    return np.concatenate([np.asarray(R).reshape(9), p, v, bias6[3:], bias6[:3]]).astype(F32)


def stream(seed, g, rg, mode, M=500, K_extra=60, kind='normal', t2=None, noise=True):
    """One stream at time t2 of synth's IMU trajectory: the source state (last keyframe at t2 - 0.2 or last frame at t2 - 0.05) near the
    truth, its preintegrations, a prior (mode 2), and a local map seen by the true camera.  Keypoints sit near the projections of ~70% of
    the points; planted: wrong descriptors (no match), gross outliers (keypoint displaced 5-7 px, descriptor kept), clutter.
    kind: 'normal', 'empty' (no local point), 'nomatch' (only clutter keypoints: the search finds nothing)."""
    import oracle_lib as O
    rng = np.random.default_rng(seed)
    t2 = 1.0 + 0.37 * (seed % 11) if t2 is None else t2
    bias = np.array([0.02, -0.01, 0.03, 0.002, -0.001, 0.0015])
    tk, tl = t2 - 0.2, t2 - 0.05
    def src(t, pert):
        R, p, v, _, _ = synth.imu_trajectory(t)
        return _state(R @ synth._rodrigues(rng.normal(0, 2e-3 * pert, 3)), p + rng.normal(0, 3e-3 * pert, 3), v + rng.normal(0, 5e-3 * pert, 3),
                      bias + rng.normal(0, 1e-4 * pert, 6))
    kfS, lastS = src(tk, 1.0 if noise else 0.0), src(tl, 1.0 if noise else 0.0)
    pre = lambda a, b, S: O.imu_preintegrate(*synth.imu_interval(a, b, seed=seed, bias=tuple(bias), noise=noise),
                                             np.concatenate([S[18:21], S[15:18]]) + (rng.normal(0, 2e-4, 6) if noise else 0), synth.IMU_NOISE)
    preintKF, preintFrame = pre(tk, t2, kfS), pre(tl, t2, lastS)
    R1, p1, v1, _, _ = synth.imu_trajectory(tl)
    prior = np.concatenate([(R1 @ synth._rodrigues(rng.normal(0, 2e-3, 3))).reshape(9), p1 + rng.normal(0, 5e-3, 3), v1 + rng.normal(0, 1e-2, 3),
                            bias[3:] + rng.normal(0, 1e-4, 3), bias[:3] + rng.normal(0, 1e-3, 3)])
    Hd = np.diag(np.concatenate([np.full(3, 2.5e5), np.full(3, 4e4), np.full(3, 1e4), np.full(3, 1e8), np.full(3, 1e6)]))
    Q, _ = np.linalg.qr(rng.normal(0, 1, (15, 15)))
    Mx = np.eye(15) + 0.05 * (Q - np.eye(15))
    # local map around the true camera
    R2, p2, _, _, _ = synth.imu_trajectory(t2)
    Rcb, tcb = rg['extr'][:9].reshape(3, 3), rg['extr'][9:12]
    Rcw = Rcb @ R2.T; tcw = Rcb @ (-R2.T @ p2) + tcb
    if kind == 'empty':
        M = 0
    W, H = g['bounds'][2], g['bounds'][3]
    fx, fy, cx, cy = (float(v) for v in g['cam'])
    z = rng.uniform(2.0, 16.0, M)
    u, v = rng.uniform(8, W - 8, M), rng.uniform(8, H - 8, M)
    pc = np.stack([(u - cx) * z / fx, (v - cy) * z / fy, z], 1)
    Xw = (pc - tcw) @ Rcw
    Ow = -Rcw.T @ tcw
    PO = Xw - Ow
    dist = np.linalg.norm(PO, axis=1)
    lvl = rng.integers(0, 8, M)
    maxD = (dist * 1.2 ** lvl * rng.uniform(1.0, 1.15, M)).astype(F32)
    normal = PO / np.maximum(dist, 1e-9)[:, None] + rng.normal(0, 0.2, (M, 3))
    normal /= np.maximum(np.linalg.norm(normal, axis=1), 1e-9)[:, None]
    mpDesc = rng.integers(0, 256, (M, 32), dtype=np.uint8)
    own = np.nonzero(rng.random(M) < (0.0 if kind == 'nomatch' else 0.7))[0]
    Kp = len(own) + K_extra
    kps = np.zeros(Kp, T._kp_dtype())
    sig = 1.2 ** lvl[own]
    kps['x'][:len(own)] = np.clip(u[own] + rng.normal(0, 0.5, len(own)) * sig, 0.5, W - 0.5)
    kps['y'][:len(own)] = np.clip(v[own] + rng.normal(0, 0.5, len(own)) * sig, 0.5, H - 0.5)
    gross = rng.random(len(own)) < 0.06
    kps['x'][:len(own)][gross] += rng.uniform(5, 7, gross.sum()) * rng.choice([-1, 1], gross.sum())
    kps['octave'][:len(own)] = lvl[own]
    kps['x'][len(own):] = rng.uniform(1, W - 1, K_extra); kps['y'][len(own):] = rng.uniform(1, H - 1, K_extra)
    kps['octave'][len(own):] = rng.integers(0, 8, K_extra)
    kps['size'] = 31; kps['angle'] = rng.uniform(0, 360, Kp); kps['response'] = 1; kps['class_id'] = -1
    desc = rng.integers(0, 256, (Kp, 32), dtype=np.uint8)
    wrong = rng.random(len(own)) < 0.05
    desc[:len(own)][~wrong] = mpDesc[own][~wrong]
    for i in range(len(own)):
        for b in rng.integers(0, 256, rng.integers(0, 12)):
            desc[i, b >> 3] ^= np.uint8(1 << (b & 7))
    perm = rng.permutation(Kp)
    bad = (rng.random(M) < 0.04).astype(np.uint8)
    hasObs = (rng.random(M) > 0.08).astype(np.uint8)
    return dict(kps=kps[perm], desc=desc[perm], nM=M, worldPos=Xw.astype(F32), normal=normal.astype(F32),
                minDistInv=(F32(0.8) * (maxD / F32(1.2 ** 7))).astype(F32), maxDistInv=(F32(1.2) * maxD).astype(F32), maxDistance=maxD,
                mpDesc=mpDesc, hasObs=hasObs, bad=bad, mode=mode, kfState21=kfS, lastState21=lastS, preintKF=preintKF, preintFrame=preintFrame,
                prior21=prior, priorH=Mx.T @ Hd @ Mx, t2=t2, truth=_state(R2, p2, synth.imu_trajectory(t2)[2], bias), n_gross=int(gross.sum()))


def prior_from_oracle(st, rg, seed):
    """Gives a mode-2 stream the prior the reference would carry: PoseInertialOptimizationLastKeyFrame of the previous frame (at t2 - 0.05,
    synth.pose_inertial_problem with this rig) on the oracle, ConstraintPoseImu's constructor on its H, and the previous frame's float state
    as SetImuPoseVelocity leaves it.  Returns the optimiser's result."""
    import oracle_lib as O
    pr = synth.pose_inertial_problem(st['t2'] - 0.25, st['t2'] - 0.05, n=200, seed=seed)
    pr['extr'] = rg['extr']
    r = O.pose_inertial_opt_last_kf(pr, O.imu_preintegrate(pr['acc'], pr['gyr'], pr['dt'], pr['bias6'], synth.IMU_NOISE))
    s = r['state']
    _, Rimu, timu = set_imu_pose(rg['Tcb7'], s[:9].astype(F32), s[9:12].astype(F32))
    st.update(prior21=s.copy(), priorH=O.constraint_pose_imu_information(r['H']), lastState21=np.concatenate([Rimu, timu, s[12:21].astype(F32)]).astype(F32))
    return r


def batch(streams, g, rg, th, mode=None, kcap=None, mcap=None):
    """Pads per-stream dicts into the slabs of orbm_track_local_map_inertial_batch*: returns (local-map dict, imu dict)."""
    B = len(streams)
    kcap = kcap or max(1, max(len(s['kps']) for s in streams))
    mcap = mcap or max(1, max(s['nM'] for s in streams))
    kps = np.zeros((B, kcap), T._kp_dtype()); desc = np.zeros((B, kcap, 32), np.uint8)
    arr = {k: np.zeros((B, mcap) + sh, dt) for k, sh, dt in (('worldPos', (3,), F32), ('normal', (3,), F32), ('minDistInv', (), F32), ('maxDistInv', (), F32),
                                                              ('maxDistance', (), F32), ('mpDesc', (32,), np.uint8), ('hasObs', (), np.uint8), ('bad', (), np.uint8))}
    for b, s in enumerate(streams):
        K, M = len(s['kps']), s['nM']
        kps[b, :K] = s['kps']; desc[b, :K] = s['desc']
        for k in arr:
            arr[k][b, :M] = s[k][:M]
    local = dict(batch=B, kcap=kcap, mcap=mcap, nlevels=8, kps=kps, desc=desc, nK=np.array([len(s['kps']) for s in streams], np.int32),
                 bounds=g['bounds'], scaleFactors=g['scaleFactors'], invLevelSigma2=g['invLevelSigma2'], cam=tuple(float(c) for c in g['cam']),
                 mbf=g['mbf'], logScaleFactor=g['logScaleFactor'], nM=np.array([s['nM'] for s in streams], np.int32), th=np.asarray(th, F32),
                 nnratio=g['nnratio'], bFarPoints=g['bFarPoints'], thFarPoints=g['thFarPoints'], viewingCosLimit=g['viewingCosLimit'], **arr)
    stk = lambda k, dt: np.stack([np.asarray(s[k], dt).reshape(-1) for s in streams])
    imu = dict(mode=np.array([s['mode'] for s in streams] if mode is None else mode, np.uint8), Tcb7=rg['Tcb7'], extrinsics24=rg['extr'],
               preintKF=stk('preintKF', F32), preintFrame=stk('preintFrame', F32), kfState21=stk('kfState21', F32), lastState21=stk('lastState21', F32),
               prior21=stk('prior21', np.float64), priorH=stk('priorH', np.float64).reshape(B, 15, 15))
    return local, imu
