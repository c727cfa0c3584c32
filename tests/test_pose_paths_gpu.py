"""GPU: the tracking pose optimisers' C entry points (pose_optimization_batch, pose_inertial_optimization_last_kf_batch /
last_frame_batch) on the frames of tests/pose_scenes.py, in every launch shape: each frame alone against the oracle (outlier flags and
return value equal, PoseOptimization's pose within 1e-9, inertial states within 1e-6, reprojection residuals within 1e-4 px, H within
1e-6 / 1e-5 relative); all frames of an optimiser in one call in two orders and 1,000 frames (several waves of CTAs), repeated, byte-
identical to the single calls; a cap far past every N with NaN in the unused input slots; the outlier slots past N after a call that
flagged every slot; and N[f] outside [0, cap], refused before anything is staged."""
import numpy as np
import pytest

import oracle_lib as O
import pose_scenes as S

pytestmark = pytest.mark.gpu
LAYOUTS = {'po': S.PO_LAYOUTS, 'kf': S.KF_LAYOUTS, 'lf': S.LF_LAYOUTS}
BIG = ('n_4000', 'n_2000')                      # left out of the 1,000-frame calls to keep their slot arrays small


@pytest.fixture(scope='module')
def orb():
    import orb_slam3_modified_b200 as m
    m.lib()
    return m


@pytest.fixture(scope='module')
def frames():
    return {v: {n: f() for n, f in L.items()} for v, L in LAYOUTS.items()}


def _call(orb, variant, frs, cap, fill=0.0, rec=False, N=None, sentinel=0):
    """One direct call of the entry point with `cap` slots per frame, the input slots past N[f] set to `fill`.  Output buffers start
    as `sentinel` bytes.  Returns (rc, dict of the output arrays)."""
    L, p = orb.lib(), orb._ptr
    n = len(frs)
    cnt = np.array([len(f['obs']) for f in frs], np.int32) if N is None else np.asarray(N, np.int32)
    dt = np.float64 if variant == 'po' else np.float32
    Xw = np.full((n, cap, 3), fill, dt); ob = np.full((n, cap, 2), fill, dt); isg = np.full((n, cap), fill, np.float32)
    td = np.full((n, cap), fill, np.float32)
    for i, f in enumerate(frs):
        k = len(f['obs'])
        Xw[i, :k] = f['Xw']; ob[i, :k] = f['obs']; isg[i, :k] = f['inv_sigma2']
        if variant != 'po':
            td[i, :k] = f['track_depth']
    cam = np.stack([np.asarray(f['cam'], np.float32) for f in frs])
    outl = np.full((n, cap), sentinel, np.uint8)
    cnt_out = np.full(n, sentinel * 0x01010101, np.int32)
    if variant == 'po':
        pose = np.stack([np.asarray(f['pose'], np.float64) for f in frs]); out = np.full((n, 7), np.nan)
        rc = L.pose_optimization_batch(n, cap, p(cnt), p(pose), p(cam), p(Xw), p(ob), p(isg), float(np.float32(np.sqrt(5.991))), p(out), p(outl),
                                       p(cnt_out), 0)
        return rc, dict(pose=out, outlier=outl, inliers=cnt_out)
    st = lambda k: np.stack([np.asarray(f[k], np.float64).reshape(-1) for f in frs]).copy()
    ex = np.asarray(frs[0]['extr'], np.float64)
    state = st('state'); H = np.full((n, 15, 15), np.nan)
    if variant == 'kf':
        P = np.stack([np.asarray(f['preint'], np.float32) for f in frs])
        rc = L.pose_inertial_optimization_last_kf_batch(n, cap, p(cnt), p(Xw), p(ob), p(isg), p(td), p(cam), p(ex), p(P), p(st('kf_state')), p(state),
                                                        int(rec), p(outl), p(H), p(cnt_out), 0)
        return rc, dict(state=state, outlier=outl, H=H, ret=cnt_out)
    Pf = np.stack([np.asarray(f['preint_frame'], np.float32) for f in frs]); Pk = np.stack([np.asarray(f['preint_kf'], np.float32) for f in frs])
    prev = st('prev_state')
    rc = L.pose_inertial_optimization_last_frame_batch(n, cap, p(cnt), p(Xw), p(ob), p(isg), p(td), p(cam), p(ex), p(Pf), p(Pk), p(st('prior_state')),
                                                       p(st('prior_H')), p(prev), p(state), int(rec), p(outl), p(H), p(cnt_out), 0)
    return rc, dict(state=state, prev_state=prev, outlier=outl, H=H, ret=cnt_out)


def _run(orb, variant, frs, cap=None, fill=0.0, rec=False):
    """Per-frame results of one call (outlier rows cut at N[f]) and the whole outlier array."""
    cap = cap or max(1, max(len(f['obs']) for f in frs))
    rc, out = _call(orb, variant, frs, cap, fill, rec)
    assert rc == orb.ORB_OK, rc
    res = []
    for i, f in enumerate(frs):
        r = {k: v[i] for k, v in out.items()}
        r['outlier'] = r['outlier'][:len(f['obs'])]
        res.append(r)
    return res, out['outlier']


def _same_bytes(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes(), k


def _oracle(variant, f, rec=False):
    return O.pose_optimization(f) if variant == 'po' else S.run_oracle(variant, f, rec_init=rec)


def _residuals(f, state):
    ex = f['extr']
    return np.array([O.imu_edge_mono(state[:9].reshape(3, 3), state[9:12], ex[:9], ex[9:12], ex[12:21], ex[21:24], f['cam'], f['Xw'][i].astype(np.float64),
                                     f['obs'][i].astype(np.float64), jac=False)[0] for i in range(len(f['Xw']))]).reshape(-1, 2)


def _equals_oracle(variant, got, f, want):
    if variant == 'po':
        assert got['inliers'] == want['inliers'] and np.array_equal(got['outlier'], want['outlier'])
        assert np.abs(got['pose'] - want['pose']).max() <= 1e-9, np.abs(got['pose'] - want['pose']).max()
        if len(f['obs']) < 3:
            assert got['pose'].tobytes() == np.asarray(f['pose'], np.float64).tobytes()
        return
    assert got['ret'] == want['ret'] and np.array_equal(got['outlier'], want['outlier']), (got['ret'], want['ret'])
    assert np.abs(got['state'] - want['state']).max() < 1e-6
    if variant == 'lf':
        assert np.abs(got['prev_state'] - want['prev_state']).max() < 1e-6
    if len(f['Xw']):
        assert np.abs(_residuals(f, got['state']) - _residuals(f, want['state'])).max() < 1e-4       # px
    assert np.abs(got['H'] - want['H']).max() <= (1e-6 if variant == 'kf' else 1e-5) * np.abs(want['H']).max()


PARAMS = [(v, n) for v, L in LAYOUTS.items() for n in L]


@pytest.mark.parametrize('variant,name', PARAMS, ids=['%s-%s' % p for p in PARAMS])
def test_each_layout_alone_equals_the_oracle(orb, frames, variant, name):
    f = frames[variant][name]
    for rec in ((False,) if variant == 'po' else (False, True)):
        got, _ = _run(orb, variant, [f], rec=rec)
        _equals_oracle(variant, got[0], f, _oracle(variant, f, rec))


@pytest.fixture(scope='module')
def single(orb, frames):
    return {v: {n: _run(orb, v, [f])[0][0] for n, f in L.items()} for v, L in frames.items()}


@pytest.mark.parametrize('variant', list(LAYOUTS))
def test_all_layouts_in_one_call_in_two_orders(orb, frames, single, variant):
    names = list(LAYOUTS[variant])
    for order in (names, names[::-1]):
        got, _ = _run(orb, variant, [frames[variant][n] for n in order])
        for n, g in zip(order, got):
            _same_bytes(g, single[variant][n])


@pytest.mark.parametrize('variant', list(LAYOUTS))
def test_more_frames_than_one_wave(orb, frames, single, variant):
    """1,000 frames, one CTA each: both kernels are register-bound to one or two resident CTAs per SM, so on an H100's 132 SMs the call
    runs in several waves.  The same call twice gives the same bytes."""
    names = [n for n in LAYOUTS[variant] if n not in BIG]
    order = [names[i % len(names)] for i in range(1000)]
    frs = [frames[variant][n] for n in order]
    first, a = _run(orb, variant, frs)
    for n, g in zip(order, first):
        _same_bytes(g, single[variant][n])
    again, b = _run(orb, variant, frs)
    assert a.tobytes() == b.tobytes()
    for x, y in zip(first, again):
        _same_bytes(x, y)


@pytest.mark.parametrize('variant', list(LAYOUTS))
def test_cap_past_every_n_with_nan_in_the_unused_slots(orb, frames, single, variant):
    """The kernels read no input slot past N[f]: NaN there changes nothing, and the outlier slots there come back 0."""
    names = list(LAYOUTS[variant])
    frs = [frames[variant][n] for n in names]
    cap = 2 * max(len(f['obs']) for f in frs) + 100
    got, outl = _run(orb, variant, frs, cap=cap, fill=np.nan)
    for n, g in zip(names, got):
        _same_bytes(g, single[variant][n])
    for i, f in enumerate(frs):
        assert not outl[i, len(f['obs']):].any()


def _all_gross(variant, n, seed):
    return S.po_all_gross(n=n, seed=seed) if variant == 'po' else S.pi_all_gross(variant, seed, n=n)


@pytest.mark.parametrize('variant', list(LAYOUTS))
def test_outlier_slots_past_n_are_zero(orb, frames, single, variant):
    """Two calls with the same count and cap lay the staging buffer out the same way.  The first flags every slot of every row (every
    observation a gross outlier, N = cap); the second, with N < cap, must hand back 0 in the slots past N, not the first call's flags."""
    names = [n for n in LAYOUTS[variant] if n not in BIG]
    frs = [frames[variant][n] for n in names]
    cap = max(len(f['obs']) for f in frs) + 40
    gross = [_all_gross(variant, cap, 100 + i) for i in range(len(frs))]
    _, before = _run(orb, variant, gross, cap=cap, rec=True)
    assert before.all()
    got, outl = _run(orb, variant, frs, cap=cap, rec=False)
    for i, (n, f) in enumerate(zip(names, frs)):
        _same_bytes(got[i], single[variant][n])
        assert not outl[i, len(f['obs']):].any(), n


@pytest.mark.parametrize('variant', list(LAYOUTS))
def test_argument_errors(orb, frames, variant):
    """N[f] = cap + 1 or -1 in one frame of a batch: ORB_ERR_ARG, and no output byte written (the call returns before staging); the
    next valid call on this thread still equals the oracle."""
    names = [n for n in LAYOUTS[variant] if n not in BIG][:6]
    frs = [frames[variant][n] for n in names]
    cap = max(len(f['obs']) for f in frs)
    for bad in (cap + 1, -1):
        N = [len(f['obs']) for f in frs]
        N[3] = bad
        rc, out = _call(orb, variant, frs, cap, N=N, sentinel=0x5A)
        assert rc == orb.ORB_ERR_ARG, rc
        assert (out['outlier'] == 0x5A).all() and (out['inliers' if variant == 'po' else 'ret'] == 0x5A5A5A5A).all()
        for k in ('pose', 'H'):
            if k in out:
                assert np.isnan(out[k]).all()
        for k in ('state', 'prev_state'):
            if k in out:
                assert out[k].tobytes() == np.stack([np.asarray(f[k], np.float64).reshape(-1) for f in frs]).tobytes()
    got, _ = _run(orb, variant, frs)
    for g, f in zip(got, frs):
        _equals_oracle(variant, g, f, _oracle(variant, f))
