"""The oracle of LocalMapping::CreateNewMapPoints (oracle/mapping_oracle.cpp) against independent evidence: float64 SVDs, the reference's
sequential loop run literally, a float64 numpy restatement of the decision chain, and planted matches that reach every branch."""
import numpy as np
import pytest

import new_points_lib as NP

N30 = tuple(d for a in range(1, 16) for d in (a, -a))
EPS32 = float(np.finfo(np.float32).eps)


def _xn(kp, cam):
    return np.float32((np.float32(kp['x']) - cam[2]) / cam[0]), np.float32((np.float32(kp['y']) - cam[3]) / cam[1])


def _A(x1, y1, x2, y2, T1, T2):
    """Triangulate's A, element by element in float32 (one product, one difference), as the oracle forms it."""
    return np.stack([x1 * T1[2] - T1[0], y1 * T1[2] - T1[1], x2 * T2[2] - T2[0], y2 * T2[2] - T2[1]]).astype(np.float32)


def _svd_bound(A64):
    """|x3D(float Jacobi) - x3D(float64 SVD)| bound: a backward-stable float SVD moves the null vector by at most
    c eps |A| / (s3 - s4) (Wedin); x = v[:3] / v[3] then moves by |dv| (1 + |x|) / |v[3]|.  c = 64 covers the rotations of a few sweeps."""
    _, s, Vt = np.linalg.svd(A64)
    v = Vt[3]
    x = v[:3] / v[3]
    dv = 64 * EPS32 * s[0] / (s[2] - s[3])
    return x, dv * (1 + np.linalg.norm(x)) / abs(v[3])


@pytest.fixture(scope='module')
def sc5():
    return NP.scene(18, (2, -2, 4, -4, 6))


def test_triangulate_vs_float64_svd(sc5):
    """x3D of the oracle's float Jacobi SVD == numpy's float64 SVD of the same float A, within the bound derived from that SVD."""
    rec, _, _, _ = NP.create(sc5)
    assert len(rec) > 100
    worst = 0.0
    for r in rec:
        k = int(r['kf2'])
        kp1, kp2 = sc5['kf1']['kps'][r['idx1']], sc5['kf2'][k]['kps'][r['idx2']]
        x1, y1 = _xn(kp1, sc5['cam'][0]); x2, y2 = _xn(kp2, sc5['cam'][k + 1])
        T1, T2 = sc5['Tcw'][0], sc5['Tcw'][k + 1]
        ok, x, V = NP.triangulate(x1, y1, x2, y2, T1, T2)
        assert ok and np.array_equal(x, r['x3D'])
        x64, tol = _svd_bound(_A(x1, y1, x2, y2, T1, T2).astype(np.float64))
        err = np.abs(x - x64).max()
        assert err <= tol + 4 * EPS32 * np.abs(x64).max(), (err, tol)
        worst = max(worst, err / tol)
        assert np.allclose(V.T @ V, np.eye(4), atol=1e-5)             # V stays orthogonal
    print('worst error / bound: %.3g' % worst)


def test_triangulate_recovers_noise_free_point():
    """Observations projected exactly from a known point (then rounded to float32) give the point back."""
    rng = np.random.default_rng(3)
    T1, _ = NP.pose34(10)
    T2, _ = NP.pose34(16)
    for _ in range(200):
        X = np.array([rng.uniform(-1, 1), rng.uniform(-1, 1), rng.uniform(-0.2, 0.2)])
        p1 = T1[:, :3].astype(np.float64) @ X + T1[:, 3]; p2 = T2[:, :3].astype(np.float64) @ X + T2[:, 3]
        ok, x, _ = NP.triangulate(np.float32(p1[0] / p1[2]), np.float32(p1[1] / p1[2]), np.float32(p2[0] / p2[2]), np.float32(p2[1] / p2[2]), T1, T2)
        assert ok and np.abs(x - X).max() < 2e-4 * np.linalg.norm(X - (-T1[:, :3].T @ T1[:, 3])), (x, X)


@pytest.mark.parametrize('t,dts,coarse,inertial,th_far', [(20, (3,), False, False, 0.0), (20, (1, 2, 3), False, True, 0.0), (12, (2, -2, 4, -4, 6, 8), True, False, 3.3),
                                                          (18, N30[:10], False, False, 0.0), (18, N30, False, True, 0.0), (18, N30, True, True, 3.3),
                                                          (25, N30, False, False, 0.0)])
def test_one_shot_equals_sequential_loop(t, dts, coarse, inertial, th_far):
    """The parallel restatement (static search for all neighbours, first passing neighbour per idx1) == the reference's loop run literally:
    per neighbour, SearchForTriangulation with KF1's CURRENT hasMapPoint, then the checks, then AddMapPoint for the new points."""
    sc = NP.scene(t, dts)
    rec, nm, nc, why = NP.create(sc, coarse, inertial, th_far)
    srec, snm, snc = NP.sequential(sc, NP.oracle_search(sc, coarse), coarse, inertial, th_far)
    assert rec.tobytes() == srec.tobytes() and np.array_equal(nm, snm) and np.array_equal(nc, snc)
    assert nc.sum() == len(rec) and (why == NP.CREATED).sum() == len(rec)
    assert np.array_equal(nm, ((why != NP.NO_MATCH) & (why != NP.TAKEN)).sum(1))
    if len(dts) >= 5:
        assert (why == NP.TAKEN).any()
    kk = rec['kf2'].astype(np.int64) * 100000 + rec['idx1']
    assert (np.diff(kk) > 0).all() and len(np.unique(rec['idx1'])) == len(rec)


def _numpy_chain(sc, k, idx1, idx2, inertial, th_far, rel=1e-4):
    """The decision chain in float64 from the same float inputs: (reason, near) where near = some tested value lies within `rel` of its threshold."""
    kp1, kp2 = sc['kf1']['kps'][idx1], sc['kf2'][k]['kps'][idx2]
    c1, c2 = sc['cam'][0].astype(np.float64), sc['cam'][k + 1].astype(np.float64)
    T1, T2 = sc['Tcw'][0].astype(np.float64), sc['Tcw'][k + 1].astype(np.float64)
    O1, O2 = sc['Ow'][0].astype(np.float64), sc['Ow'][k + 1].astype(np.float64)
    near = False

    def close(v, thr):
        return abs(v - thr) <= rel * max(abs(thr), 1e-30)
    xn1 = np.array([(kp1['x'] - c1[2]) / c1[0], (kp1['y'] - c1[3]) / c1[1], 1.0])
    xn2 = np.array([(kp2['x'] - c2[2]) / c2[0], (kp2['y'] - c2[3]) / c2[1], 1.0])
    r1, r2 = T1[:, :3].T @ xn1, T2[:, :3].T @ xn2
    cp = r1 @ r2 / (np.linalg.norm(r1) * np.linalg.norm(r2))
    lim = 0.9996 if inertial else 0.9998
    near |= close(1 - cp, 1 - lim)
    if not (0 < cp < lim):
        return NP.LOW_PARALLAX, near
    A = np.stack([xn1[0] * T1[2] - T1[0], xn1[1] * T1[2] - T1[1], xn2[0] * T2[2] - T2[0], xn2[1] * T2[2] - T2[1]])
    v = np.linalg.svd(A)[2][3]
    X = v[:3] / v[3]
    for T, c, kp, sig, why_d, why_r in ((T1, c1, kp1, sc['sigma2'], NP.DEPTH1, NP.REPROJ1), (T2, c2, kp2, sc['sigma2'], NP.DEPTH2, NP.REPROJ2)):
        p = T[:, :3] @ X + T[:, 3]
        near |= close(p[2], 0.0) or abs(p[2]) < 1e-6
        if p[2] <= 0:
            return why_d, near
    for T, c, kp, why_r in ((T1, c1, kp1, NP.REPROJ1), (T2, c2, kp2, NP.REPROJ2)):
        p = T[:, :3] @ X + T[:, 3]
        e2 = (c[0] * p[0] / p[2] + c[2] - kp['x']) ** 2 + (c[1] * p[1] / p[2] + c[3] - kp['y']) ** 2
        thr = 5.991 * float(sc['sigma2'][kp['octave']])
        near |= close(e2, thr)
        if e2 > thr:
            return why_r, near
    d1, d2 = np.linalg.norm(X - O1), np.linalg.norm(X - O2)
    if th_far > 0:
        near |= close(d1, th_far) or close(d2, th_far)
        if d1 >= th_far or d2 >= th_far:
            return NP.FAR, near
    rd, ro, rf = d2 / d1, float(sc['sf'][kp1['octave']]) / float(sc['sf'][kp2['octave']]), 1.5 * 1.2
    near |= close(rd * rf, ro) or close(rd, ro * rf)
    if rd * rf < ro or rd > ro * rf:
        return NP.SCALE, near
    return NP.CREATED, near


@pytest.mark.parametrize('t,dts,inertial,th_far', [(18, N30[:12], False, 0.0), (20, (1, 2, 3, 5), True, 3.3), (25, N30, False, 0.0)])
def test_decision_chain_vs_float64_restatement(t, dts, inertial, th_far):
    """Every match of the static search: the oracle's reason == the float64 numpy chain's, except where a tested value lies within 1e-4
    (relative) of its threshold."""
    sc = NP.scene(t, dts)
    _, _, _, why = NP.create(sc, False, inertial, th_far)
    i = NP._In(sc, False, inertial, th_far)
    m12 = [NP.oracle_search(sc)(k, sc['kf1']['has_mp']) for k in range(len(dts))]
    n = excluded = 0
    for k in range(len(dts)):
        for idx1 in np.nonzero(m12[k] >= 0)[0]:
            got, _ = NP.match(sc, k, int(idx1), int(m12[k][idx1]), _in=i)
            want, near = _numpy_chain(sc, k, int(idx1), int(m12[k][idx1]), inertial, th_far)
            n += 1
            if near:
                excluded += 1
                continue
            assert (got == NP.CREATED) == (want == NP.CREATED) and got == want, (k, idx1, NP.REASONS[got], NP.REASONS[want])
    print('%d matches, %d within 1e-4 of a threshold excluded' % (n, excluded))
    assert n > 200 and excluded <= 0.02 * n


def test_every_branch_is_reached():
    """Across scenes and planted matches every reason code occurs; mono and inertial parallax limits and bCoarse are both exercised."""
    seen = set()
    sc = NP.scene(18, N30)
    for coarse in (False, True):
        for inertial in (False, True):
            _, nm, _, why = NP.create(sc, coarse, inertial, 3.3)
            seen |= set(np.unique(why).tolist())
    nm_fine = NP.create(sc, False, False)[1]
    nm_coarse = NP.create(sc, True, False)[1]
    assert (nm_coarse >= nm_fine).all() and nm_coarse.sum() > nm_fine.sum()          # bCoarse drops the epipolar test
    # close frames: low parallax dominates (dt = 1 sits at the 0.9998 limit)
    _, _, _, why1 = NP.create(NP.scene(20, (1,)))
    assert (why1 == NP.LOW_PARALLAX).sum() > 0.5 * (why1 != NP.NO_MATCH).sum()
    seen |= set(np.unique(why1).tolist())
    # mono vs inertial limit: a match with 0.9996 <= cos < 0.9998 passes mono and fails inertial
    sc3 = NP.scene(20, (1, 2, 3))
    mono, inert = NP.create(sc3, False, False)[3], NP.create(sc3, False, True)[3]
    assert ((mono != NP.LOW_PARALLAX) & (mono != NP.NO_MATCH) & (mono != NP.TAKEN) & (inert == NP.LOW_PARALLAX)).any()
    # planted: random pairs fail depth / reprojection
    rng = np.random.default_rng(0)
    i = NP._In(sc3)
    N1, N2 = len(sc3['kf1']['kps']), len(sc3['kf2'][2]['kps'])
    for _ in range(3000):
        seen.add(NP.match(sc3, 2, int(rng.integers(N1)), int(rng.integers(N2)), _in=i)[0])
    # planted: a created point whose KF2 feature is relabelled to the top octave fails the scale test
    rec = NP.create(sc3)[0]
    r = rec[rec['kf2'] == 2][0]
    s_oct = dict(sc3, kf2=list(sc3['kf2']))
    s_oct['kf2'][2] = dict(sc3['kf2'][2], kps=sc3['kf2'][2]['kps'].copy())
    s_oct['kf1'] = dict(sc3['kf1'], kps=sc3['kf1']['kps'].copy())
    s_oct['kf1']['kps']['octave'][r['idx1']] = 0
    s_oct['kf2'][2]['kps']['octave'][r['idx2']] = 7
    why_s = NP.match(s_oct, 2, int(r['idx1']), int(r['idx2']))[0]
    assert why_s == NP.SCALE
    # planted: the camera centre handed in at the point itself gives a zero distance
    s_ow = dict(sc3, Ow=sc3['Ow'].copy())
    s_ow['Ow'][0] = r['x3D']
    assert NP.match(s_ow, 2, int(r['idx1']), int(r['idx2']))[0] == NP.ZERO_DIST
    s_ow['Ow'][0] = sc3['Ow'][0]; s_ow['Ow'][3] = r['x3D']
    assert NP.match(s_ow, 2, int(r['idx1']), int(r['idx2']))[0] == NP.ZERO_DIST
    seen |= {why_s, NP.ZERO_DIST}
    # planted: a degenerate KF2 "pose" whose second row is y2 times its third and whose translation is (0, -100, 0) decouples A's last
    # row and column, so V keeps e4 apart and the smallest singular value's column has V(3, 3) == 0 exactly
    kp1 = np.zeros(1, NP.KP_DTYPE); kp2 = np.zeros(1, NP.KP_DTYPE)
    cam = sc3['cam'][0]
    kp1['x'], kp1['y'] = cam[2] + 0.3 * cam[0], cam[3] + 0.1 * cam[1]
    kp2['x'], kp2['y'] = cam[2] - 0.2 * cam[0], cam[3] + 0.1 * cam[1]
    y2 = _xn(kp2[0], cam)[1]
    T2 = np.array([[1, 0, 0, 0], [0, 0, y2, -100], [0, 0, 1, 0]], np.float32)
    T1 = np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0]], np.float32)
    kf = lambda kp: dict(kps=kp, desc=np.zeros((1, 32), np.uint8), has_mp=np.zeros(1, np.uint8), fv=(np.zeros(0, np.int32), np.zeros(0, np.int32)))
    s_svd = dict(sc3, kf1=kf(kp1), kf2=[kf(kp2)], ep=sc3['ep'][:1], F12=sc3['F12'][:1], Tcw=np.stack([T1, T2]), Ow=sc3['Ow'][:2], cam=sc3['cam'][:2])
    ok, _, V = NP.triangulate(*_xn(kp1[0], cam), *_xn(kp2[0], cam), T1, T2)
    assert not ok and V[3, 3] == 0
    assert NP.match(s_svd, 0, 0, 0)[0] == NP.SVD_W0
    seen.add(NP.SVD_W0)
    missing = set(range(NP.LOW_PARALLAX, NP.TAKEN + 1)) - seen
    assert not missing, [NP.REASONS[m] for m in sorted(missing)]
