"""GPU tests of orbm_update_local_map_batch*: every output equals the oracle's byte for byte for batches of both vote branches, monocular and
inertial streams, TrackReferenceKeyFrame index spaces and empty streams; a batch equals per-stream calls; the device form equals the host
form; one launch per call; the argument and capacity errors; the planted scenes of the kernel's long paths; and the device chains
motion-model step -> UpdateLocalMap -> TrackLocalMap and UpdateLocalMap -> inertial TrackLocalMap equal the host forms fed the oracle's
UpdateLocalMap."""
import numpy as np
import pytest

import local_map_lib as L
import track_lib as T

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def orb():
    import orb_slam3_modified_b200 as m
    m.lib()
    return m


@pytest.fixture(scope='module')
def matcher(orb):
    return orb.ORBmatcher(0.8, False, max_batch=240, max_keypoints=2048, max_mappoints=2048, device=0)


def _empty(seed):
    sc = L.scene(seed, n_kf=6)
    sc.src, sc.match = [None] * 5, [-1, 2, -1]          # nothing votes: an empty table
    return sc


def _scenes(B, seed):
    out = []
    for s in range(B):
        r = seed * 1000 + s
        if B > 1 and s % 7 == 1:
            out.append(_empty(r))
        else:
            out.append(L.scene(r, n_kf=15 + (11 * s) % 60, n_pts=200 + (97 * s) % 900, vote_last=s % 3 == 2, inertial=s % 2 == 0,
                               trk_space=s % 5 == 3, n_src=60 + (31 * s) % 300))
    return out


def _same(a, b, what):
    for k in a:
        assert np.ascontiguousarray(a[k]).tobytes() == np.ascontiguousarray(b[k]).tobytes(), (what, k)


@pytest.mark.parametrize('B', [1, 7, 240])
def test_batch_equals_oracle(orb, matcher, B):
    d, ref, _ = L.run_oracle(_scenes(B, B), mcap=2048)
    got = matcher.update_local_map_batch(d)
    assert matcher.last_launch_count() == 1
    _same(got, ref, 'batch')
    assert (ref['nLocalKF'] > 0).any() and (ref['nM'] > 0).any()
    if B > 1:
        assert (ref['nLocalKF'] == 0).any()
    if B == 7:                                          # per-stream calls give the same bytes
        scenes = _scenes(B, B)
        for b in range(B):
            d1, ref1, _ = L.run_oracle([scenes[b]], mcap=2048, kcap=d['kcap'], mcapLast=d['mcapLast'])
            one = matcher.update_local_map_batch(d1)
            _same(one, ref1, ('single', b))
            k0, k1 = d['kfStart'][b], d['kfStart'][b + 1]
            assert one['localKF'].tobytes() == got['localKF'][k0:k1].tobytes()
            for k in ('localPoint', 'worldPos', 'mpDesc', 'lastToLocal', 'nM', 'refKF'):
                assert one[k][0].tobytes() == got[k][b].tobytes(), k


def test_planted_scenes_equal_oracle(orb, matcher):
    """The kernel's long paths against the oracle on the device: more than 80 voters, the cap ending the expansion at 81, the parent
    break, children in a second 32-wide chunk, tables of 400 rows (a three-chunk voter scan, pKFmax in a later chunk and tied across
    chunks), the stalled walk, duplicate votes and shared points -- in one batch with seeded streams, then each alone."""
    import torch
    scenes = L.planted() + _scenes(5, 77)
    d, ref, _ = L.run_oracle(scenes, mcap=4096)
    assert (np.diff(d['kfStart']) > 256).sum() >= 2 and (ref['nLocalKF'] == 81).any() and (ref['nLocalKF'] > 256).any()
    got = matcher.update_local_map_batch(d)
    _same(got, ref, 'planted batch')
    dd = {k: (torch.from_numpy(np.ascontiguousarray(v)).cuda() if isinstance(v, np.ndarray) else v) for k, v in d.items()}
    out = orb.local_map_outputs(d, lambda shape, dt: torch.full(shape, 3, dtype=getattr(torch, np.dtype(dt).name), device='cuda'))
    matcher.update_local_map_batch_device(dd, out, stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    _same({k: v.cpu().numpy() for k, v in out.items()}, ref, 'planted device')
    for sc in L.planted():
        d1, ref1, _ = L.run_oracle([sc], mcap=4096)
        _same(matcher.update_local_map_batch(d1), ref1, 'planted single')


def test_device_form_equals_host_form(orb, matcher):
    import torch
    d, ref, _ = L.run_oracle(_scenes(24, 5), mcap=2048)
    host = matcher.update_local_map_batch(d)
    dd = {k: (torch.from_numpy(np.ascontiguousarray(v)).cuda() if isinstance(v, np.ndarray) else v) for k, v in d.items()}
    out = orb.local_map_outputs(d, lambda shape, dt: torch.full(shape, 7, dtype=getattr(torch, np.dtype(dt).name), device='cuda'))
    matcher.update_local_map_batch_device(dd, out, stream=torch.cuda.current_stream().cuda_stream)
    assert matcher.last_launch_count() == 1
    torch.cuda.synchronize()
    _same({k: v.cpu().numpy() for k, v in out.items()}, host, 'device')
    _same(host, ref, 'host')


def test_launch_counts(orb, matcher):
    d, _, _ = L.run_oracle([_empty(1), _empty(2)], mcap=64)
    out = matcher.update_local_map_batch(d)
    assert matcher.last_launch_count() == 0
    assert (out['nM'] == 0).all() and (out['refKF'] == -1).all() and (out['lastToLocal'] == -1).all() and (out['localPoint'] == -1).all()
    d, _, _ = L.run_oracle([_empty(1), L.scene(4)], mcap=2048)
    matcher.update_local_map_batch(d)
    assert matcher.last_launch_count() == 1


def test_argument_and_capacity_errors(orb, matcher):
    base, _, _ = L.run_oracle([L.scene(8, inertial=True), L.scene(9, vote_last=True)], mcap=2048)
    matcher.update_local_map_batch(base)
    assert matcher.last_launch_count() == 1

    def expect(edit, code=orb.ORB_ERR_ARG):
        d = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in base.items()}
        edit(d)
        out = orb.local_map_outputs(d)
        for v in out.values():
            v.fill(5)
        with pytest.raises(orb.OrbError) as e:
            matcher.update_local_map_batch(d, out)
        assert e.value.code == code
        if code == orb.ORB_ERR_ARG:                     # rejected before any launch: outputs and the launch count untouched
            assert all((v == 5).all() for v in out.values()) and matcher.last_launch_count() == 1
        return str(e.value), out

    def setv(key, i, v):
        def f(d): d[key].reshape(-1)[i] = v
        return f
    n0 = int(base['kfStart'][1])
    expect(setv('covKF', 0, n0 + 500))
    expect(setv('childKF', 0, -1))
    expect(setv('slotPoint', 3, 10 ** 6))
    expect(setv('obsKF', 1, -5))
    expect(setv('parent', 2, n0))
    expect(setv('prevKF', 2, -2))
    expect(setv('lastKF', 0, n0))
    expect(setv('srcPoint', 4, -2))
    expect(setv('match', 0, int(base['nSrc'][0])))
    expect(setv('match', 1, -2))
    expect(setv('nSrc', 0, base['mcapLast'] + 1))
    expect(lambda d: d['covStart'].__setitem__(-1, d['covStart'][-2] - 1))   # decreasing
    expect(setv('obsStart', 0, 1))                      # not starting at 0
    expect(setv('kfStart', 2, base['nKF'] - 1))         # not ending at nKF

    def many_cov(d):
        d['covStart'][1:] += 11
        d['covKF'] = np.concatenate([np.zeros(11, np.int32), d['covKF']])
    expect(many_cov)
    kids = [k for k in range(base['nKF']) if base['childStart'][k + 1] - base['childStart'][k] >= 2]

    def unsorted(d):
        s = d['childStart'][kids[0]]
        d['childKF'][s], d['childKF'][s + 1] = d['childKF'][s + 1], d['childKF'][s]
    expect(unsorted)
    msg, out = expect(lambda d: d.update(mcap=30), orb.ORB_ERR_CAPACITY)
    assert 'stream 0' in msg and (out['nM'] > 30).all() and (out['localPoint'] == -1).all() and (out['lastToLocal'] == -1).all()


def _dev(a):
    import torch
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.uint8) if a.dtype.fields else a).cuda()


def _chain_scene(st, seed, inertial=False):
    """A keyframe model whose points are a tracking stream `st`'s local points (its bad ones included).  Monocular: src is the last
    frame's slots (track_lib), a bad point for each entry without a local index, and match the last-frame search's.  Inertial (the last
    frame votes): src is a random subset of the points with NULL entries and bad points, and the mPrevKF walk starts at the newest
    keyframe."""
    sc = L.Scene(seed)
    rng = sc.rng
    n_kf = 9
    for j, key in enumerate(rng.permutation(n_kf) * 8 + 64):
        sc.add_kf(int(key))
        if j:
            sc.kfs[j].prev = j - 1
            sc.set_parent(j, int(rng.integers(0, j)))
    for p in range(st['nM']):
        q = sc.add_point([int(k) for k in rng.choice(n_kf, int(rng.integers(1, 4)), replace=False)], bad=bool(st['bad'][p]))
        mp = sc.pts[q]
        mp.worldPos, mp.normal, mp.desc, mp.hasObs = st['worldPos'][p], st['normal'][p], st['mpDesc'][p], st['hasObs'][p]
        mp.minDistInv, mp.maxDistInv, mp.maxDistance = st['minDistInv'][p], st['maxDistInv'][p], st['maxDistance'][p]
    for kf in sc.kfs:
        kf.cov = [int(k) for k in rng.permutation(n_kf) if k != kf.id][:int(rng.integers(0, 9))]
    if inertial:
        M = st['nM']
        sc.src = [int(rng.integers(0, M)) if M and rng.random() < 0.8 else None for _ in range(int(rng.integers(40, 200)))]
        sc.src += [sc.add_point([int(rng.integers(0, n_kf))], bad=True) for _ in range(3)]
        sc.vote_last, sc.inertial, sc.last_kf = True, True, n_kf - 1
        return sc
    sc.src = [int(l) if l >= 0 else sc.add_point([int(rng.integers(0, n_kf))], bad=True) for l in st['lastToLocal']]
    sc.match = [int(m) for m in st['match']]
    return sc


def test_device_chain_equals_oracle_chain(orb, matcher):
    """motion-model step -> UpdateLocalMap -> TrackLocalMap, all device forms on one stream, against the host forms with the oracle's
    UpdateLocalMap in between (byte for byte), and against the CPU oracle chain of tests/track_lib.py with the oracle's UpdateLocalMap in
    front (matches and counts equal, poses to 1e-8)."""
    import torch
    g = T.globals_()
    B = 7
    kinds = ('normal', 'normal', 'empty', 'all_seen', 'few', 'nine', 'normal')
    streams = [T.stream(4000 + b, g, M=300 + 97 * b, K_extra=20 + 13 * (b % 5), kind=kinds[b]) for b in range(B)]
    th = np.array([1, 2, 5, 10, 15, 1, 1], np.float32)
    mo, lo, state = T.batch(streams, g, th, mcap=2048)
    items = [L.flatten(_chain_scene(st, b))[0] for b, st in enumerate(streams)]
    d = orb.local_map_batch(items, 2048, kcap=mo['kcap'], mcapLast=mo['mcap'])
    # host chain with the oracle's UpdateLocalMap
    match, claimed, nm = state['match'].copy(), state['claimed'].copy(), state['nmatches'].copy()
    r1 = matcher.motion_model_pose_batch(mo, g['invLevelSigma2'], match, claimed, nm)
    ref = L.oracle(dict(d, match=match))
    assert (ref['nM'] > 0).sum() >= 5
    lh = dict(lo, Tcw7=r1['Tcw7'], discarded=r1['discarded'], **{k: ref[k] for k in ('lastToLocal', 'nM', 'worldPos', 'normal', 'minDistInv',
                                                                                     'maxDistInv', 'maxDistance', 'mpDesc', 'hasObs', 'bad')})
    match_host = match.copy()
    r2 = matcher.track_local_map_batch(lh, match_host)
    assert (r2['nmatches'] > 0).any()
    # device chain
    st = torch.cuda.current_stream().cuda_stream
    md = {k: (_dev(v) if isinstance(v, np.ndarray) else v) for k, v in mo.items()}
    dm, dc, dn = _dev(state['match']), _dev(state['claimed']), _dev(state['nmatches'])
    zeros = lambda shape, dt: torch.zeros(shape, dtype=getattr(torch, np.dtype(dt).name), device='cuda')   # noqa: E731
    p7, t7, dd, nmm = zeros((B, 7), np.float64), zeros((B, 7), np.float32), zeros((B, mo['mcap']), np.uint8), zeros(B, np.int32)
    matcher.motion_model_pose_batch_device(md, _dev(g['invLevelSigma2']), dm, dc, dn, p7, t7, dd, nmm, stream=st)
    ud = {k: (_dev(v) if isinstance(v, np.ndarray) else v) for k, v in d.items()}
    ud['match'] = dm
    uo = orb.local_map_outputs(d, zeros)
    matcher.update_local_map_batch_device(ud, uo, stream=st)
    ld = {k: (_dev(v) if isinstance(v, np.ndarray) else v) for k, v in lo.items()}
    ld.update(Tcw7=t7, discarded=dd, **{k: uo[k] for k in ('lastToLocal', 'nM', 'worldPos', 'normal', 'minDistInv', 'maxDistInv', 'maxDistance',
                                                          'mpDesc', 'hasObs', 'bad')})
    K, M = lo['kcap'], lo['mcap']
    out = dict(match=dm, claimed=zeros((B, K), np.uint8), outlier=zeros((B, K), np.uint8), visible=zeros((B, M), np.int32),
               found=zeros((B, M), np.int32), pose7=zeros((B, 7), np.float64), Tcw7=zeros((B, 7), np.float32),
               **{k: zeros(B, np.int32) for k in ('nToMatch', 'nmatches', 'nInliers', 'nMatchesInliers')})
    matcher.track_local_map_batch_device(ld, out, stream=st)
    torch.cuda.synchronize()
    _same({k: v.cpu().numpy() for k, v in uo.items()}, ref, 'UpdateLocalMap')
    assert out['match'].cpu().numpy().tobytes() == match_host.tobytes()
    _same({k: out[k].cpu().numpy() for k in r2}, r2, 'TrackLocalMap')
    assert t7.cpu().numpy().tobytes() == r1['Tcw7'].tobytes()
    # and directly against the CPU oracle chain: the oracle's motion-model step, its UpdateLocalMap, its TrackLocalMap (tests/track_lib.py);
    # matches and counts equal, poses to 1e-8 (the oracle's FP64 sums are ordered differently, as in tests/test_track_batch_gpu.py)
    ob, R = T.OracleBackend(), {k: v.cpu().numpy() for k, v in out.items()}
    for b, s in enumerate(streams):
        K, ML = len(s['kps']), s['mcapLast']
        m_, c_ = s['match'].copy(), s['claimed'].copy()
        mm = T.motion_model_step(ob, s, g, m_, c_, s['nmatches'])
        assert m_.tobytes() == match[b, :K].tobytes(), b        # so `ref` is the oracle's UpdateLocalMap on the oracle's matches
        row = ref
        s2 = dict(s, nM=int(row['nM'][b]), lastToLocal=row['lastToLocal'][b, :ML],
                  **{k: row[k][b] for k in ('worldPos', 'normal', 'minDistInv', 'maxDistInv', 'maxDistance', 'mpDesc', 'hasObs', 'bad')})
        lm = T.local_map_step(ob, s2, g, m_, mm['discarded'], mm['Tcw7'], th[b])
        assert R['match'][b, :K].tobytes() == lm['match'].tobytes() and R['claimed'][b, :K].tobytes() == lm['claimed'].tobytes(), b
        for k in ('nToMatch', 'nmatches', 'nInliers', 'nMatchesInliers'):
            assert R[k][b] == lm[k], (k, b)
        assert np.abs(R['pose7'][b] - lm['pose7']).max() < 1e-8, b


def test_inertial_device_chain_equals_host_flattened_path(orb, matcher):
    """UpdateLocalMap's device slabs fed straight to orbm_track_local_map_inertial_batch_device equal that call's host form fed the
    oracle's flattened local map (tests/test_track_inertial_gpu.py ties the host form to the per-frame chain and the CPU oracle chain)."""
    import torch
    import track_inertial_lib as TI
    g, rg = T.globals_(), TI.rig()
    B = 6
    kinds = ('normal', 'empty', 'nomatch', 'normal', 'normal', 'normal')
    streams = [TI.stream(5000 + b, g, rg, 1 + b % 2, M=300 + 97 * b, K_extra=20 + 13 * (b % 5), kind=kinds[b]) for b in range(B)]
    th = np.array([2, 6, 5, 15, 2, 6], np.float32)
    lo, imu = TI.batch(streams, g, rg, th, mcap=2048)
    items = [L.flatten(_chain_scene(st, 50 + b, inertial=True))[0] for b, st in enumerate(streams)]
    d = orb.local_map_batch(items, 2048, kcap=lo['kcap'])
    slabs = ('nM', 'worldPos', 'normal', 'minDistInv', 'maxDistInv', 'maxDistance', 'mpDesc', 'hasObs', 'bad')
    ref = L.oracle(d)
    assert (ref['nM'] > 0).sum() >= 4 and (ref['lastToLocal'] >= 0).any()
    R = matcher.track_local_map_inertial_batch(dict(lo, **{k: ref[k] for k in slabs}), imu)
    assert (R['nmatches'] > 0).any() and (R['nInliers'] > 0).any()
    st = torch.cuda.current_stream().cuda_stream
    zeros = lambda shape, dt: torch.zeros(shape, dtype=getattr(torch, np.dtype(dt).name), device='cuda')   # noqa: E731
    ud = {k: (_dev(v) if isinstance(v, np.ndarray) else v) for k, v in d.items()}
    uo = orb.local_map_outputs(d, zeros)
    matcher.update_local_map_batch_device(ud, uo, stream=st)
    dl = {k: (_dev(v) if isinstance(v, np.ndarray) else v) for k, v in lo.items()}
    dl.update({k: uo[k] for k in slabs})
    di = {k: (_dev(v) if isinstance(v, np.ndarray) and k not in ('mode', 'Tcb7') else v) for k, v in imu.items()}
    out = {k: zeros(v.shape, v.dtype) for k, v in R.items()}
    out['pose7'] = None
    matcher.track_local_map_inertial_batch_device(dl, di, out, stream=st)
    torch.cuda.synchronize()
    _same({k: v.cpu().numpy() for k, v in uo.items()}, ref, 'UpdateLocalMap')
    _same({k: out[k].cpu().numpy() for k in R}, R, 'inertial TrackLocalMap')


def test_cpp_update_local_map_batch_equals_python(orb, matcher, tmp_path):
    """ORBmatcher::UpdateLocalMapBatch (include/orb_b200/orb_slam3.hpp) from a g++-built caller gives the Python binding's digest."""
    import os
    import subprocess
    d, _, _ = L.run_oracle(_scenes(9, 41), mcap=2048)
    (tmp_path / 'dims.txt').write_text(' '.join(str(int(d[n])) for n in orb.LOCAL_MAP_SIZES) + '\n')
    for name, dt in orb.LOCAL_MAP_ARRAYS:
        (tmp_path / (name + '.raw')).write_bytes(np.ascontiguousarray(d[name], dt).tobytes())
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib = os.path.join(root, 'orb_slam3_modified_b200')
    exe = tmp_path / 'local_map_example'
    subprocess.check_call(['g++', '-std=c++14', '-O2', '-Wall', '-I', os.path.join(root, 'include'), os.path.join(root, 'tests', 'local_map_example.cpp'),
                           '-o', str(exe), '-L', lib, '-l:liborb_b200.so', '-Wl,-rpath,' + lib, '-lpthread'])
    out = dict(l.split() for l in subprocess.check_output([str(exe), str(tmp_path)]).decode().splitlines())
    res = matcher.update_local_map_batch(d)
    h = 14695981039346656037
    for n, _, _, _ in orb.LOCAL_MAP_OUTPUTS:
        for b in res[n].tobytes():
            h = ((h ^ b) * 1099511628211) & 0xFFFFFFFFFFFFFFFF
    assert out['digest'] == '%016x' % h
    assert int(out['points']) == int(res['nM'].sum()) > 100 and out['launches'] == '1'
