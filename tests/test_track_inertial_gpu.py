"""GPU tests of orbm_track_local_map_inertial_batch*: byte for byte equal to the per-frame chain of the library's existing entry points fed
with the call's own prediction (tests/track_inertial_lib.py), equal to the CPU oracle chain in the matches, chained over three frames on
the device, and the host / device / resident forms agree."""
import numpy as np
import pytest

import oracle_lib as O
import track_inertial_lib as TI
import track_lib as T

pytestmark = pytest.mark.gpu
KINDS = ('normal', 'empty', 'nomatch', 'normal', 'normal', 'normal', 'normal')
THS = (2.0, 6.0, 5.0, 15.0)


@pytest.fixture(scope='module')
def orb():
    import orb_slam3_modified_b200 as m
    return m


def _streams(B, seed, g, rg, modes=None):
    return [TI.stream(seed * 1000 + b, g, rg, (modes[b] if modes is not None else 1 + b % 2), M=300 + 97 * (b % 9), K_extra=20 + 13 * (b % 5),
                      kind=KINDS[b] if b < len(KINDS) else 'normal') for b in range(B)]


def _same(a, b, what):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    assert a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes(), what


def _chain(be, streams, g, rg, R, th):
    return [TI.local_map_step(be, st, g, rg, st['mode'], R['predState21'][b], R['predTcw7'][b], th[b]) for b, st in enumerate(streams)]


def _residuals(st, g, rg, match, state):
    """Reprojection residuals (px) of a stream's matches at the camera of a double state (Rwb | twb ...): Rcw = Rcb Rwb^T, tcw = Rcb (-Rwb^T twb) + tcb."""
    e = np.nonzero(match >= 0)[0]
    Rwb, twb = state[:9].reshape(3, 3), state[9:12]
    Rcb, tcb = rg['extr'][:9].reshape(3, 3), rg['extr'][9:12]
    Xc = st['worldPos'][match[e]].astype(np.float64) @ (Rcb @ Rwb.T).T + (Rcb @ (-Rwb.T @ twb) + tcb)
    fx, fy, cx, cy = (float(c) for c in g['cam'])
    return np.stack([st['kps']['x'][e] - (fx * Xc[:, 0] / Xc[:, 2] + cx), st['kps']['y'][e] - (fy * Xc[:, 1] / Xc[:, 2] + cy)], 1)


def _compare(R, chain, streams, exact=True, g=None, rg=None):
    for b, lm in enumerate(chain):
        K, M = len(streams[b]['kps']), streams[b]['nM']
        _same(R['match'][b, :K], lm['match'], ('match', b)); _same(R['claimed'][b, :K], lm['claimed'], ('claimed', b))
        _same(R['outlier'][b, :K], lm['outlier'], ('outlier', b))
        _same(R['visible'][b, :M], lm['visible'], ('visible', b)); _same(R['found'][b, :M], lm['found'], ('found', b))
        for k in ('nToMatch', 'nmatches', 'nInliers', 'nMatchesInliers'):
            assert R[k][b] == lm[k], (k, b, R[k][b], lm[k])
        if exact:
            for k in ('Tcw7', 'state21', 'prior21', 'priorH'):
                _same(R[k][b], np.asarray(lm[k]).reshape(R[k][b].shape), (k, b))
        else:
            assert np.abs(R['prior21'][b] - lm['prior21']).max() < 1e-8, (b, np.abs(R['prior21'][b] - lm['prior21']).max())
            if rg is not None and lm['N']:
                dr = np.abs(_residuals(streams[b], g, rg, lm['match'], R['prior21'][b]) - _residuals(streams[b], g, rg, lm['match'], lm['prior21'])).max()
                assert dr < 1e-4, (b, dr)


@pytest.mark.parametrize('B,far', [(1, False), (7, False), (7, True), (240, False)])
def test_equals_per_frame_chain_of_existing_entry_points(orb, B, far):
    g, rg = T.globals_(), TI.rig()
    if far:
        g.update(bFarPoints=1, thFarPoints=9.0)
    streams = _streams(B, 3 + B + int(far), g, rg)
    th = np.array([THS[b % len(THS)] for b in range(B)], np.float32)
    m = orb.ORBmatcher(0.8, False, max_batch=B, max_keypoints=1024, max_mappoints=2048, device=0)
    d, imu = TI.batch(streams, g, rg, th)
    R = m.track_local_map_inertial_batch(d, imu)
    assert m.last_launch_count() == (7 if B > 1 else 6)
    mt1 = orb.ORBmatcher(0.8, False, max_batch=1, max_keypoints=1024, max_mappoints=2048)
    _compare(R, _chain(TI.GpuChainBackend(orb, mt1), streams, g, rg, R, th), streams)
    assert (R['nmatches'] > 0).any() and (R['outlier'] > 0).any()
    if B == 7:
        assert R['nToMatch'][1] == 0 and R['nmatches'][2] == 0 and R['nToMatch'][2] > 0      # empty local map; a search that finds nothing
        _compare(R, _chain(TI.OracleBackend(), streams, g, rg, R, th), streams, exact=False, g=g, rg=rg)
        # the prediction against the oracle restatement (float rounding: device NormalizeRotation and sinf / cosf differ in the last bits)
        worst = 0.0
        for b, st in enumerate(streams):
            S, P = (st['kfState21'], st['preintKF']) if st['mode'] == 1 else (st['lastState21'], st['preintFrame'])
            pred, Tcw = TI.predict_state(O, rg['Tcb7'], S, P)
            worst = max(worst, np.abs(R['predState21'][b].astype(np.float64) - pred).max(), np.abs(R['predTcw7'][b].astype(np.float64) - Tcw).max())
        print('prediction: max |device - oracle restatement| = %.2e' % worst)
        assert worst < 1e-5
    R2 = m.track_local_map_inertial_batch(d, imu)                 # two calls give the same bytes
    for k in R:
        _same(R[k], R2[k], k)


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8) if a.dtype.fields else np.ascontiguousarray(a)).cuda()


def _dev_inputs(d, imu):
    return ({k: (_dev(v) if isinstance(v, np.ndarray) else v) for k, v in d.items()},
            {k: (_dev(v) if isinstance(v, np.ndarray) and k not in ('mode', 'Tcb7') else v) for k, v in imu.items()})


def _dev_out(like, fill=0):
    import torch
    return {k: torch.full(v.shape, fill, dtype=getattr(torch, str(v.dtype)), device='cuda') for k, v in like.items()}


def test_three_frames_chained_on_device(orb):
    """Three consecutive frames 50 ms apart per stream: the device form's state21 / prior21 / priorH tensors are the next call's
    lastState21 / prior21 / priorH without leaving the device; the per-frame chain carries its own outputs on the host."""
    import torch
    g, rg = T.globals_(), TI.rig()
    patterns = [(1, 2, 2), (2, 2, 1), (1, 1, 2), (2, 1, 2), (2, 2, 2)]
    B = len(patterns)
    th = np.full(B, 2.0, np.float32)
    frames = [[TI.stream(60 + 10 * b + f, g, rg, patterns[b][f], M=400, t2=1.0 + 0.37 * b + 0.05 * f) for b in range(B)] for f in range(3)]
    kcap = max(len(s['kps']) for fr in frames for s in fr); mcap = max(s['nM'] for fr in frames for s in fr)
    m = orb.ORBmatcher(0.8, False, max_batch=B, max_keypoints=1024, max_mappoints=2048, device=0)
    be = TI.GpuChainBackend(orb, orb.ORBmatcher(0.8, False, max_batch=1, max_keypoints=1024, max_mappoints=2048))
    prev_dev = prev_chain = None
    for f in range(3):
        if f:
            for b, st in enumerate(frames[f]):
                st.update(lastState21=prev_chain[b]['state21'], prior21=prev_chain[b]['prior21'], priorH=prev_chain[b]['priorH'])
        d, imu = TI.batch(frames[f], g, rg, th, kcap=kcap, mcap=mcap)
        dd, di = _dev_inputs(d, imu)
        if f:
            di.update(lastState21=prev_dev['state21'], prior21=prev_dev['prior21'], priorH=prev_dev['priorH'])
        like = dict(match=np.zeros((B, kcap), np.int32), claimed=np.zeros((B, kcap), np.uint8), outlier=np.zeros((B, kcap), np.uint8),
                    visible=np.zeros((B, mcap), np.int32), found=np.zeros((B, mcap), np.int32), Tcw7=np.zeros((B, 7), np.float32),
                    predState21=np.zeros((B, 21), np.float32), predTcw7=np.zeros((B, 7), np.float32), state21=np.zeros((B, 21), np.float32),
                    prior21=np.zeros((B, 21)), priorH=np.zeros((B, 15, 15)), **{k: np.zeros(B, np.int32) for k in ('nToMatch', 'nmatches', 'nInliers', 'nMatchesInliers')})
        out = _dev_out(like)
        m.track_local_map_inertial_batch_device(dd, di, out, stream=torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        R = {k: v.cpu().numpy() for k, v in out.items()}
        chain = _chain(be, frames[f], g, rg, R, th)
        _compare(R, chain, frames[f])
        assert (R['nInliers'] > 0).any() and (R['nmatches'] > 0).any()
        prev_dev, prev_chain = out, chain


def test_forms_agree_and_skipped_streams_untouched(orb):
    import torch
    g, rg = T.globals_(), TI.rig()
    streams = _streams(7, 5, g, rg)
    th = np.array([2, 6, 15, 2, 5, 2, 6], np.float32)
    m = orb.ORBmatcher(0.8, False, max_batch=7, max_keypoints=1024, max_mappoints=2048, device=0)
    d, imu = TI.batch(streams, g, rg, th)
    full = m.track_local_map_inertial_batch(d, imu)
    mode = imu['mode'].copy(); mode[[1, 4]] = 0
    R = m.track_local_map_inertial_batch(d, dict(imu, mode=mode))
    for b in range(7):
        for k in R:
            if mode[b]:
                _same(R[k][b], full[k][b], (k, b))
            elif k != 'match':
                assert not R[k][b].any(), (k, b)
            else:
                assert (R[k][b] == -1).all()
    one = imu['mode'].copy(); one[:] = 2
    m.track_local_map_inertial_batch(d, dict(imu, mode=one))
    assert m.last_launch_count() == 6
    # device form (torch) and resident form agree with the host form byte for byte
    dd, di = _dev_inputs(d, imu)
    out = _dev_out(full)
    m.track_local_map_inertial_batch_device(dd, di, out, stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    for k in full:
        _same(out[k].cpu().numpy(), full[k], ('device', k))
    # device form with skipped streams: their rows keep what the caller had there (a sentinel), the others equal the full call
    out = _dev_out(full, fill=7)
    m.track_local_map_inertial_batch_device(dd, dict(di, mode=mode), out, stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    for k in full:
        o = out[k].cpu().numpy()
        for b in range(7):
            if mode[b]:
                _same(o[b], full[k][b], ('device skip', k, b))
            else:
                assert (o[b] == 7).all(), ('device skip untouched', k, b)
    res = (dd['kps'].data_ptr(), dd['desc'].data_ptr(), dd['nK'].data_ptr(), d['kcap'])
    r3 = m.track_local_map_inertial_batch(d, imu, resident=res)
    for k in full:
        _same(r3[k], full[k], ('resident', k))


def test_launch_count_independent_of_batch(orb):
    g, rg = T.globals_(), TI.rig()
    for B in (2, 240):
        streams = _streams(B, 9, g, rg)
        m = orb.ORBmatcher(0.8, False, max_batch=B, max_keypoints=1024, max_mappoints=2048, device=0)
        d, imu = TI.batch(streams, g, rg, np.full(B, 2.0, np.float32))
        m.track_local_map_inertial_batch(d, imu)
        assert m.last_launch_count() == 7
        m.track_local_map_inertial_batch(d, dict(imu, mode=np.ones(B, np.uint8)))
        assert m.last_launch_count() == 6


def test_bad_arguments_and_capacity(orb):
    g, rg = T.globals_(), TI.rig()
    streams = _streams(2, 13, g, rg)
    m = orb.ORBmatcher(0.8, False, max_batch=2, max_keypoints=1024, max_mappoints=2048, device=0)

    def expect(code, fd=None, fi=None, mt=m):
        d, imu = TI.batch(streams, g, rg, [2, 2])
        if fd:
            fd(d)
        if fi:
            fi(imu)
        with pytest.raises(orb.OrbError) as ei:
            mt.track_local_map_inertial_batch(d, imu)
        assert ei.value.code == code

    def oct_(d): d['kps']['octave'][0, 0] = 8
    for k in ('Tcw7', 'lastToLocal', 'discarded', 'active'):
        expect(orb.ORB_ERR_ARG, fd=lambda d, k=k: d.__setitem__(k, np.zeros((2, 7), np.float32) if k == 'Tcw7' else np.zeros((2, 4), np.uint8 if k != 'lastToLocal' else np.int32)))
    expect(orb.ORB_ERR_ARG, fd=oct_)
    expect(orb.ORB_ERR_ARG, fi=lambda i: i['mode'].__setitem__(0, 3))
    for k in ('lastState21', 'prior21', 'priorH', 'preintFrame'):
        expect(orb.ORB_ERR_ARG, fi=lambda i, k=k: i.__setitem__(k, None))
    small = orb.ORBmatcher(0.8, False, max_batch=2, max_keypoints=1024, max_mappoints=100, device=0)
    expect(orb.ORB_ERR_CAPACITY, mt=small)
    # a non-NULL pose7 through the C ABI
    import ctypes as C
    d, imu = TI.batch(streams, g, rg, [2, 2])
    keep = {k: np.ascontiguousarray(d[k], dt) for k, dt in m._LOCAL_MAP_DT.items() if d.get(k) is not None}
    s = m._local_map_struct(d, lambda k: keep[k].ctypes.data if k in keep else None)
    ik = {k: np.ascontiguousarray(imu[k], dt) for k, dt in dict(m._IMU_DT, extrinsics24=np.float64).items()}
    si = m._imu_struct(imu, imu['mode'], lambda k: ik[k].ctypes.data)
    bufs = [np.zeros(4096, np.float64) for _ in range(16)]
    r = orb._OrbmLocalMapResult(*[b.ctypes.data for b in bufs[:11]])
    ri = orb._OrbmImuTrackResult(*[b.ctypes.data for b in bufs[11:]])
    L = orb.lib()
    assert L.orbm_track_local_map_inertial_batch(m._h, C.byref(s), C.byref(si), C.byref(r), C.byref(ri)) == orb.ORB_ERR_ARG


def _build_cpp(exe):
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib = os.path.join(root, 'orb_slam3_modified_b200')
    subprocess.check_call(['g++', '-std=c++14', '-O2', '-Wall', '-I', os.path.join(root, 'include'), os.path.join(root, 'tests', 'track_inertial_example.cpp'),
                           '-o', str(exe), '-L', lib, '-l:liborb_b200.so', '-Wl,-rpath,' + lib, '-lpthread'])


def test_cpp_batch_tracker_equals_python(orb, tmp_path):
    """BatchTracker::TrackLocalMapInertial (include/orb_b200/orb_slam3.hpp) from a g++-built caller: two chained calls, byte for byte the
    Python binding's."""
    import subprocess
    g, rg = T.globals_(), TI.rig()
    streams = _streams(5, 17, g, rg)
    th = np.array([2, 6, 15, 2, 5], np.float32)
    d, imu = TI.batch(streams, g, rg, th)
    B, K, M = d['batch'], d['kcap'], d['mcap']
    with open(tmp_path / 'dims.txt', 'w') as f:
        vals = [B, K, M, d['nlevels'], *d['bounds'], *d['cam'], d['mbf'], float(d['logScaleFactor']), d['nnratio'], d['bFarPoints'], d['thFarPoints'],
                d['viewingCosLimit'], *[float(v) for v in rg['Tcb7']]]
        f.write(' '.join(repr(float(v)) if isinstance(v, (float, np.floating)) else str(v) for v in vals))
    m = orb.ORBmatcher(0.8, False, max_batch=B, max_keypoints=K, max_mappoints=M, device=0)
    for k, dt in m._LOCAL_MAP_DT.items():
        if d.get(k) is not None:
            (tmp_path / (k + '.raw')).write_bytes(np.ascontiguousarray(d[k], dt).tobytes())
    for k, dt in dict(m._IMU_DT, extrinsics24=np.float64, mode=np.uint8).items():
        (tmp_path / (k + '.raw')).write_bytes(np.ascontiguousarray(imu[k], dt).tobytes())
    exe = tmp_path / 'track_inertial_example'
    _build_cpp(exe)
    out = subprocess.check_output([str(exe), str(tmp_path)]).decode()
    assert 'launches 7' in out
    R = m.track_local_map_inertial_batch(d, imu)
    R1 = m.track_local_map_inertial_batch(d, dict(imu, lastState21=R['state21'], prior21=R['prior21'], priorH=R['priorH']))
    for call, r in enumerate((R, R1)):
        for k in ('match', 'claimed', 'outlier', 'visible', 'found', 'Tcw7', 'predState21', 'predTcw7', 'state21', 'prior21', 'priorH'):
            assert (tmp_path / ('%s%d.out' % (k, call))).read_bytes() == np.ascontiguousarray(r[k]).tobytes(), (k, call)
        counts = np.concatenate([r[k] for k in ('nToMatch', 'nmatches', 'nInliers', 'nMatchesInliers')])
        assert (tmp_path / ('counts%d.out' % call)).read_bytes() == counts.tobytes(), call
