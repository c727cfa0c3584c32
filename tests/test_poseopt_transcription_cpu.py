"""Optimizer::PoseOptimization (src/Optimizer.cc:814-1113, monocular edges) a second time: the four optimisation rounds -- each
restarting from the frame's pose, 10 LM iterations over the level-0 edges, then re-classification of every observation at
chi2 > 5.991 (errors of excluded edges recomputed, the others as the last LM trial left them), Huber removed after the third round --
in Python with numerical Jacobians on the manifold, against the C++ oracle: same pose, same outlier flags, same inlier count.  (The
number of LM trials is not compared: every round converges after a few iterations and keeps iterating at the optimum, where accepting or
rejecting a step is decided by differences at rounding level.)"""
import numpy as np
import pytest

import oracle_lib as O
import pose_scenes as S
from orb_slam3_modified_b200 import synth
from test_lba_dense_cpu import _R, _exp


def _pose_opt(f):
    cam = f['cam'].astype(np.float64); X = f['Xw'].astype(np.float64); obs = f['obs'].astype(np.float64)
    is2 = f['inv_sigma2'].astype(np.float64); N = len(obs)
    delta = float(np.float32(np.sqrt(5.991))); dsqr = delta * delta
    q = f['pose'][:4] / np.linalg.norm(f['pose'][:4])
    R0, t0 = _R(q), f['pose'][4:].astype(np.float64)
    if N < 3:                                             # if(nInitialCorrespondences<3) return 0; (:996-997)
        return R0, t0, np.zeros(N, bool), 0, 0

    def resid(R, t):
        xc = X @ R.T + t
        return obs - np.stack([cam[0] * xc[:, 0] / xc[:, 2] + cam[2], cam[1] * xc[:, 1] / xc[:, 2] + cam[3]], 1)

    level = np.zeros(N, bool); robust = np.ones(N, bool); outlier = np.zeros(N, bool)
    err = np.zeros((N, 2)); trials = 0; nBad = 0
    R, t = R0, t0

    def rchi(act):
        c = is2[act] * (err[act] ** 2).sum(1)
        big = robust[act] & (c > dsqr)
        s = np.sqrt(np.maximum(c, 1e-300))
        return np.where(big, 2 * s * delta - dsqr, c), np.where(big, delta / s, 1.0)

    for rnd in range(4):
        R, t = R0, t0                                     # Tcw = pFrame->GetPose(): the frame's pose is only set at the very end (:1000-1001)
        act = ~level
        lam = ni = None; nBadLM = 0; ok = True
        it = 0
        while it < 10 and ok and act.any():
            err[act] = resid(R, t)[act]
            r0, r1 = rchi(act)
            currentChi = float(r0.sum()); iniChi = currentChi
            J = np.zeros((2 * int(act.sum()), 6)); h = 1e-6
            for c in range(6):
                d = np.zeros(6); d[c] = h
                Rp, tp = _exp(d); Rm, tm = _exp(-d)
                J[:, c] = ((resid(Rp @ R, Rp @ t + tp)[act] - resid(Rm @ R, Rm @ t + tm)[act]) / (2 * h)).reshape(-1)
            w = np.repeat(r1 * is2[act], 2)
            H = J.T @ (w[:, None] * J); b = -J.T @ (w * err[act].reshape(-1))
            if it == 0:
                lam = 1e-5 * np.abs(np.diag(H)).max(); ni = 2.0; nBadLM = 0
            qmax = 0
            while True:
                x = np.linalg.solve(H + lam * np.eye(6), b)
                Rd, td = _exp(x)
                Rn, tn = Rd @ R, Rd @ t + td
                err[act] = resid(Rn, tn)[act]             # computeActiveErrors: stays even if the trial is rejected
                tempChi = float(rchi(act)[0].sum())
                rho = (currentChi - tempChi) / (float((x * (lam * x + b)).sum()) + 1e-3)
                if rho > 0 and np.isfinite(tempChi):
                    lam *= max(1. / 3., min(1. - (2 * rho - 1) ** 3, 2. / 3.)); ni = 2.0; currentChi = tempChi
                    R, t = Rn, tn
                else:
                    lam *= ni; ni *= 2
                qmax += 1; trials += 1
                if not (rho < 0 and qmax < 10):
                    break
            if qmax == 10 or rho == 0:
                ok = False
            else:
                nBadLM = nBadLM + 1 if (iniChi - currentChi) * 1e3 < iniChi else 0
                if nBadLM >= 3:
                    ok = False
            it += 1
        nBad = 0
        e_now = resid(R, t)
        for e in range(N):
            if outlier[e]:
                err[e] = e_now[e]                         # e->computeError() only for the edges that were excluded (:1020-1023)
            chi2 = np.float32(is2[e] * (err[e] ** 2).sum())      # const float chi2 = e->chi2()
            if chi2 > np.float32(5.991):
                outlier[e] = True; level[e] = True; nBad += 1
            else:
                outlier[e] = False; level[e] = False
            if rnd == 2:
                robust[e] = False
        if N < 10:
            break
    return R, t, outlier, N - nBad, trials


# the layouts of tests/pose_scenes.py, by name
@pytest.mark.parametrize('kw', [dict(n=300, seed=1), dict(n=120, seed=5, outlier_frac=0.3), dict(n=40, seed=9, pose_noise=(0.1, 4.0))] + list(S.PO_LAYOUTS))
def test_pose_optimization_second_transcription(kw):
    f = S.PO_LAYOUTS[kw]() if isinstance(kw, str) else synth.pose_opt_problem(**kw)
    ref = O.pose_optimization(f)
    R, t, outl, inl, trials = _pose_opt(f)
    assert inl == ref['inliers'] and np.array_equal(outl.astype(np.uint8), ref['outlier'])
    assert (trials > 0) == (ref['trials'] > 0) == (len(f['obs']) >= 3)
    qo = ref['pose'][:4]
    assert np.abs(_R(qo / np.linalg.norm(qo)) - R).max() < 1e-6 and np.abs(ref['pose'][4:] - t).max() < 1e-6
