"""GPU tests of Frame::UndistortKeyPoints / Frame::ComputeImageBounds (orbx_undistort_keypoints[_device], orbx_image_bounds): the kernel
against the CPU oracle and cv2 byte for byte on the extractor's own slabs at 1, 7 and 240 frames, the untouched rows, the k1 == 0 copy, the
host / resident form, the bounds, every argument error, the device tracking chain on frames rendered through EuRoC's distortion against the
oracle chain, and a g++-built C++ caller."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import oracle_lib as O
import track_lib as T
import undistort_lib as U

pytestmark = pytest.mark.gpu
SENTINEL = 0xA5
TH = 15.0


@pytest.fixture(scope='module')
def orb():
    import orb_slam3_modified_b200 as m
    m.lib()
    return m


@pytest.fixture(scope='module')
def frames():
    """Six distinct distorted frames per calibration (t = 0..5)."""
    return {name: np.stack([U.distorted_frame(t, W, H, K, D) for t in range(6)]) for name, (K, D, W, H) in U.CALIBRATIONS.items()}


def _extract_device(orb, ex, imgs):
    import torch
    B = len(imgs)
    cap = ex.max_keypoints
    d_img = torch.from_numpy(np.ascontiguousarray(imgs)).cuda()
    d_kps = torch.zeros((B, cap, 7), dtype=torch.float32, device='cuda')
    d_desc = torch.zeros((B, cap, 32), dtype=torch.uint8, device='cuda')
    d_n = torch.zeros(B, dtype=torch.int32, device='cuda'); d_mono = torch.zeros(B, dtype=torch.int32, device='cuda')
    ex.extract_batch_device(d_img, d_kps, d_desc, d_n, d_mono, (0, 1000))
    return d_kps, d_desc, d_n


def _sentinel_like(d_kps):
    import torch
    return torch.full(d_kps.shape, 0, dtype=torch.float32, device='cuda').view(torch.uint8).fill_(SENTINEL).view(torch.float32)


def _host_kps(d):
    B, cap = d.shape[:2]
    return d.cpu().numpy().view(np.uint8).reshape(B, cap, 28).copy().view(O.KP_DTYPE).reshape(B, cap)


@pytest.mark.parametrize('name', sorted(U.CALIBRATIONS))
@pytest.mark.parametrize('B', [1, 7, 240])
def test_kernel_equals_oracle_and_cv2(orb, frames, name, B):
    import torch
    K, D, W, H = U.CALIBRATIONS[name]
    imgs = frames[name][np.arange(B) % 6]
    ex = orb.ORBextractor(1000, 1.2, 8, 20, 7, W, H, B)
    d_kps, _, d_n = _extract_device(orb, ex, imgs)
    n = d_n.clone()
    if B > 1:       # an empty frame beside full ones, and an overflowing frame (n > cap) the kernel must leave alone
        n[1] = 0
    if B > 2:
        n[2] = ex.max_keypoints + 1
    d_un = _sentinel_like(d_kps)
    ex.undistort_keypoints_device(K, D, d_kps, n, d_un)
    torch.cuda.synchronize()
    assert orb.undistort_last_launch_count() == 1
    kin, kun, nn = _host_kps(d_kps), _host_kps(d_un), n.cpu().numpy()
    raw = d_un.cpu().numpy().view(np.uint8).reshape(B, -1, 28)
    cam = U.cam9(K, D)
    for f in range(B):
        k = int(nn[f])
        if k > ex.max_keypoints:
            assert (raw[f] == SENTINEL).all(), f
            continue
        assert kun[f, :k].tobytes() == U.oracle_keypoints(kin[f, :k], cam).tobytes(), f
        for fld in ('size', 'angle', 'response', 'octave', 'class_id'):
            assert kun[f, :k][fld].tobytes() == kin[f, :k][fld].tobytes(), (f, fld)
        if f < 6 and k:
            xy = np.ascontiguousarray(np.stack([kun[f, :k]['x'], kun[f, :k]['y']], 1))
            assert xy.tobytes() == U.cv2_undistort(np.stack([kin[f, :k]['x'], kin[f, :k]['y']], 1), K, D).tobytes(), f
        assert (raw[f, k:] == SENTINEL).all(), f
    assert int(nn.max()) > 900


@pytest.mark.parametrize('k1', [0.0, -0.0])
def test_k1_zero_is_a_byte_copy(orb, frames, k1):
    import torch
    K, D, W, H = U.CALIBRATIONS['euroc']
    ex = orb.ORBextractor(1000, 1.2, 8, 20, 7, W, H, 3)
    d_kps, _, d_n = _extract_device(orb, ex, frames['euroc'][:3])
    d_un = _sentinel_like(d_kps)
    ex.undistort_keypoints_device(K, (k1, 0.5, 0.001, -0.002, 0.3), d_kps, d_n, d_un)
    torch.cuda.synchronize()
    a, b, nn = d_kps.cpu().numpy().view(np.uint8), d_un.cpu().numpy().view(np.uint8), d_n.cpu().numpy()
    for f in range(3):
        k = int(nn[f]) * 7 * 4
        assert a[f].ravel()[:k].tobytes() == b[f].ravel()[:k].tobytes() and (b[f].ravel()[k:] == SENTINEL).all()


def test_host_and_resident_forms_equal_device_form(orb, frames):
    import torch
    K, D, W, H = U.CALIBRATIONS['tum1']
    B = 5
    imgs = frames['tum1'][:B]
    ex = orb.ORBextractor(1000, 1.2, 8, 20, 7, W, H, B)
    d_kps, _, d_n = _extract_device(orb, ex, imgs)
    d_un = _sentinel_like(d_kps)
    ex.undistort_keypoints_device(K, D, d_kps, d_n, d_un)
    torch.cuda.synchronize()
    want, nn = _host_kps(d_un), d_n.cpu().numpy()
    ex.extract_batch(imgs, (0, 1000))
    ptr, got = ex.undistort_keypoints(K, D, batch=B)
    assert ptr and orb.undistort_last_launch_count() == 1
    for f in range(B):
        assert got[f, :nn[f]].tobytes() == want[f, :nn[f]].tobytes(), f
    ptr2, none = ex.undistort_keypoints(K, D, batch=2, host=False)
    assert ptr2 == ptr and none is None
    assert ex.resident_slabs()[0] != ptr          # mvKeys stays where it was
    _, zero = ex.undistort_keypoints(K, D, batch=0)
    assert orb.undistort_last_launch_count() == 0 and zero.shape == (0, ex.max_keypoints)


def test_image_bounds_equal_oracle(orb):
    rng = np.random.default_rng(9)
    cams = [U.CALIBRATIONS['euroc'][:2], U.CALIBRATIONS['tum1'][:2], ((500.0, 500.0, 320.0, 240.0), (-1.2, 0.0, 0.0, 0.0)),
            ((458.654, 457.296, 367.215, 248.375), (0.0, 0.3, 0.01, 0.01, 0.2)), ((458.654, 457.296, 367.215, 248.375), (-0.0, 0.3, 0.0, 0.0))]
    cams += [U.random_calibration(rng)[:2] for _ in range(8)]
    for K, D in cams:
        for W, H in ((640, 480), (752, 480), (1280, 720)):
            b = U.oracle_bounds(U.cam9(K, D), W, H)
            got = np.array(orb.image_bounds(K, D, W, H), np.float32)
            assert got.tobytes() == np.array([b[0], b[2], b[1], b[3]], np.float32).tobytes(), (K, D, W, H, got, b)
            assert orb.undistort_last_launch_count() == 1


def test_argument_errors_launch_nothing_and_change_nothing(orb, frames):
    import torch
    L = orb.lib()
    K, D, W, H = U.CALIBRATIONS['euroc']
    ex = orb.ORBextractor(1000, 1.2, 8, 20, 7, W, H, 2)
    d_kps, _, d_n = _extract_device(orb, ex, frames['euroc'][:2])
    d_un = _sentinel_like(d_kps)
    torch.cuda.synchronize()
    cap = ex.max_keypoints
    good = orb.pinhole_camera(K, D)

    def cam(**kw):
        c = orb.pinhole_camera(K, D)
        for k, v in kw.items():
            setattr(c, k, v)
        return C.byref(c)

    def call(h=ex._h, c=C.byref(good), batch=2, kps=d_kps.data_ptr(), n=d_n.data_ptr(), cap_=cap, out=d_un.data_ptr()):
        return L.orbx_undistort_keypoints_device(h, c, batch, kps, n, cap_, out, None)

    ok = L.orbx_undistort_keypoints_device(ex._h, C.byref(good), 2, d_kps.data_ptr(), d_n.data_ptr(), cap, d_un.data_ptr(), None)
    assert ok == orb.ORB_OK and orb.undistort_last_launch_count() == 1
    torch.cuda.synchronize()
    ref = d_un.clone()
    d_un.view(torch.uint8).fill_(SENTINEL)
    torch.cuda.synchronize()
    bad = dict(null_handle=dict(h=None), null_cam=dict(c=None), null_kps=dict(kps=None), null_n=dict(n=None), null_out=dict(out=None),
               neg_batch=dict(batch=-1), cap0=dict(cap_=0), fx0=dict(c=cam(fx=0.0)), fy0=dict(c=cam(fy=-0.0)), fx_inf=dict(c=cam(fx=float('inf'))),
               cx_nan=dict(c=cam(cx=float('nan'))), k2_nan=dict(c=cam(k2=float('nan'))), k3_inf=dict(c=cam(k3=float('-inf'))),
               p1_nan=dict(c=cam(p1=float('nan'))), same=dict(out=d_kps.data_ptr()), overlap=dict(out=d_kps.data_ptr() + 28 * (cap + 3)),
               overlap_before=dict(out=d_kps.data_ptr() - 28 * 5))
    for what, kw in bad.items():
        ok = call()      # a launch first, so that a refusal visibly resets the count
        assert ok == orb.ORB_OK
        torch.cuda.synchronize()
        d_un.view(torch.uint8).fill_(SENTINEL)
        torch.cuda.synchronize()
        assert call(**kw) == orb.ORB_ERR_ARG, what
        assert orb.undistort_last_launch_count() == 0, what
        torch.cuda.synchronize()
        assert (d_un.view(torch.uint8) == SENTINEL).all(), what
    assert call(batch=0) == orb.ORB_OK and orb.undistort_last_launch_count() == 0
    torch.cuda.synchronize()
    assert (d_un.view(torch.uint8) == SENTINEL).all()
    assert call() == orb.ORB_OK and orb.undistort_last_launch_count() == 1
    torch.cuda.synchronize()
    assert torch.equal(d_un.view(torch.uint8), ref.view(torch.uint8))
    # the host form: the last call was a device-slab extraction, a batch larger than the last call's, a wrong cap
    host = np.full((2, cap), 7, orb.KP_DTYPE)
    out_ptr = C.c_void_p(123)
    assert L.orbx_undistort_keypoints(ex._h, C.byref(good), 1, host.ctypes.data, cap, C.byref(out_ptr)) == orb.ORB_ERR_ARG
    ex.extract_batch(frames['euroc'][:1], (0, 1000))
    for args in ((2, cap), (1, cap - 1), (-1, cap)):
        assert L.orbx_undistort_keypoints(ex._h, C.byref(good), args[0], host.ctypes.data, args[1], C.byref(out_ptr)) == orb.ORB_ERR_ARG
        assert orb.undistort_last_launch_count() == 0
    assert L.orbx_undistort_keypoints(ex._h, cam(fx=0.0), 1, host.ctypes.data, cap, C.byref(out_ptr)) == orb.ORB_ERR_ARG
    assert L.orbx_undistort_keypoints(None, C.byref(good), 1, host.ctypes.data, cap, C.byref(out_ptr)) == orb.ORB_ERR_ARG
    assert (host.view(np.uint8).reshape(-1) == np.full((2, cap), 7, orb.KP_DTYPE).view(np.uint8).reshape(-1)).all() and out_ptr.value == 123
    assert L.orbx_undistort_keypoints(ex._h, C.byref(good), 1, host.ctypes.data, cap, C.byref(out_ptr)) == orb.ORB_OK and out_ptr.value
    # orbx_image_bounds
    b4 = np.full(4, 7.0, np.float32)
    for args in ((C.byref(good), 0, 480), (C.byref(good), 752, 0), (None, 752, 480), (cam(fy=0.0), 752, 480), (cam(k1=float('nan')), 752, 480)):
        assert L.orbx_image_bounds(args[0], args[1], args[2], b4.ctypes.data, 0) == orb.ORB_ERR_ARG
        assert orb.undistort_last_launch_count() == 0 and (b4 == 7.0).all()
    assert L.orbx_image_bounds(C.byref(good), 752, 480, None, 0) == orb.ORB_ERR_ARG
    assert L.orbx_image_bounds(C.byref(good), 752, 480, b4.ctypes.data, 0) == orb.ORB_OK and b4[0] < -100


# ---- the device tracking chain on distorted frames ----
def _scene(orb, K, D, W, H, ts, seed):
    """Per stream: the last frame t (oracle extraction, undistorted, its keypoints back-projected onto the synthetic plane) and the
    current frame t + 1 (distorted image), with the pose prior the motion model would give (true pose, perturbed)."""
    from orb_slam3_modified_b200 import synth
    rng = np.random.default_rng(seed)
    oe = O.OracleExtractor(1000, 1.2, 8, 20, 7)
    cam = U.cam9(K, D)
    out = []
    for t in ts:
        _, lk, ld = oe(U.distorted_frame(t, W, H, K, D), (0, 1000))
        lk = U.oracle_keypoints(lk, cam)
        xyz = synth.backproject(U.ideal_to_synth(np.stack([lk['x'], lk['y']], 1), K, W, H), t, width=W, height=H).astype(np.float32)
        img = U.distorted_frame(t + 1, W, H, K, D)
        true = synth.pose(t + 1)
        T0 = true.copy(); T0[4:] += rng.normal(0, 0.01, 3); q = T0[:4] + rng.normal(0, 0.002, 4); T0[:4] = q / np.linalg.norm(q)
        out.append(dict(lk=lk, ld=ld, xyz=xyz, img=img, true=true, Tcw7=T0.astype(np.float32), hasObs=(rng.random(len(lk)) > 0.1).astype(np.uint8)))
    return out


def _last_slabs(scene, mcap):
    B = len(scene)
    L = dict(nM=np.zeros(B, np.int32), valid=np.zeros((B, mcap), np.uint8), xyz=np.zeros((B, mcap, 3), np.float32), octave=np.zeros((B, mcap), np.int32),
             angle=np.zeros((B, mcap), np.float32), hasObs=np.zeros((B, mcap), np.uint8), mpDesc=np.zeros((B, mcap, 32), np.uint8))
    for b, s in enumerate(scene):
        m = len(s['lk'])
        L['nM'][b] = m; L['valid'][b, :m] = 1; L['xyz'][b, :m] = s['xyz']; L['octave'][b, :m] = s['lk']['octave']
        L['angle'][b, :m] = s['lk']['angle']; L['hasObs'][b, :m] = s['hasObs']; L['mpDesc'][b, :m] = s['ld']
    return L


def _device_chain(orb, K, D, W, H, scene, undistort):
    """extract_batch_device -> [undistort_keypoints_device] -> search_last_frame_batch_device -> motion_model_pose_batch_device."""
    import torch
    B = len(scene)
    ex = orb.ORBextractor(1000, 1.2, 8, 20, 7, W, H, B)
    cap = ex.max_keypoints
    d_kps, d_desc, d_n = _extract_device(orb, ex, np.stack([s['img'] for s in scene]))
    if undistort:
        d_cur = torch.empty_like(d_kps)
        ex.undistort_keypoints_device(K, D, d_kps, d_n, d_cur)
        bounds = orb.image_bounds(K, D, W, H)
    else:
        d_cur, bounds = d_kps, (0.0, 0.0, float(W), float(H))
    Ls = _last_slabs(scene, cap)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    sf = ex.GetScaleFactors()
    d = dict(batch=B, kcap=cap, mcap=cap, nlevels=8, kps=d_cur, desc=d_desc, nK=d_n, scaleFactors=dev(sf), Tcw7=dev(np.stack([s['Tcw7'] for s in scene])),
             cam=[float(c) for c in K], bounds=bounds, reset=1, **{k: dev(v) for k, v in Ls.items()})
    m = orb.ORBmatcher(0.9, True, max_batch=B, max_keypoints=cap, max_mappoints=cap)
    match = torch.zeros((B, cap), dtype=torch.int32, device='cuda'); claimed = torch.zeros((B, cap), dtype=torch.uint8, device='cuda')
    nm = torch.zeros(B, dtype=torch.int32, device='cuda')
    m.search_last_frame_batch_device(d, TH, match, claimed, nm)
    nm1 = nm.clone()
    p7 = torch.zeros((B, 7), dtype=torch.float64, device='cuda'); t7 = torch.zeros((B, 7), dtype=torch.float32, device='cuda')
    disc = torch.zeros((B, cap), dtype=torch.uint8, device='cuda'); nmm = torch.zeros(B, dtype=torch.int32, device='cuda')
    m.motion_model_pose_batch_device(d, dev((1.0 / (sf.astype(np.float64) ** 2)).astype(np.float32)), match, claimed, nm, p7, t7, disc, nmm)
    torch.cuda.synchronize()
    return dict(kps=_host_kps(d_cur), desc=d_desc.cpu().numpy(), n=d_n.cpu().numpy(), nm_search=nm1.cpu().numpy(), match=match.cpu().numpy(),
                claimed=claimed.cpu().numpy(), nmatches=nm.cpu().numpy(), pose7=p7.cpu().numpy(), Tcw7=t7.cpu().numpy(), discarded=disc.cpu().numpy(),
                nmatchesMap=nmm.cpu().numpy(), bounds=bounds, sf=sf, cap=cap)


def _globals(K, bounds, sf):
    g = T.globals_()
    g.update(cam=tuple(np.float32(c) for c in K), bounds=bounds, scaleFactors=sf, invLevelSigma2=(1.0 / (sf.astype(np.float64) ** 2)).astype(np.float32))
    return g


def _oracle_chain(K, D, W, H, scene, bounds, sf):
    """Oracle extraction, orbo_undistort_keypoints, the oracle last-frame search and PoseOptimization with the discard loop."""
    oe = O.OracleExtractor(1000, 1.2, 8, 20, 7)
    g = _globals(K, bounds, sf)
    out = []
    for s in scene:
        _, kps, desc = oe(s['img'], (0, 1000))
        kps = U.oracle_keypoints(kps, U.cam9(K, D))
        m = len(s['lk'])
        last = dict(valid=np.ones(m, np.uint8), xyz=s['xyz'], octave=s['lk']['octave'].astype(np.int32), angle=s['lk']['angle'].astype(np.float32),
                    hasObs=s['hasObs'], descriptors=s['ld'])
        match = np.full(len(kps), -1, np.int32); claimed = np.zeros(len(kps), np.uint8)
        n = O.search_last_frame(kps, desc, bounds, sf, s['Tcw7'], [float(c) for c in K], last, TH, True, match, claimed)
        st = dict(kps=kps, last_xyz=s['xyz'], Tcw7=s['Tcw7'], mcapLast=m, last_hasObs=s['hasObs'])
        mm = T.motion_model_step(T.OracleBackend(), st, g, match, claimed, n)
        out.append(dict(kps=kps, desc=desc, n_search=n, match=match, claimed=claimed, **mm))
    return out


def _pose_error(pose7, true):
    """Rotation angle (rad) + translation distance (m) between two (w, x, y, z, t) poses."""
    q = np.asarray(pose7[:4], np.float64) / np.linalg.norm(pose7[:4])
    return 2 * np.arccos(min(1.0, abs(float(np.dot(q, true[:4]))))) + float(np.linalg.norm(np.asarray(pose7[4:7], np.float64) - true[4:]))


@pytest.fixture(scope='module')
def chain(orb):
    K, D, W, H = U.CALIBRATIONS['euroc']
    scene = _scene(orb, K, D, W, H, ts=(0, 7, 15), seed=11)
    gpu = _device_chain(orb, K, D, W, H, scene, undistort=True)
    return K, D, W, H, scene, gpu


def test_device_chain_on_distorted_frames_equals_oracle_chain(orb, chain):
    K, D, W, H, scene, R = chain
    b = U.oracle_bounds(U.cam9(K, D), W, H)
    assert np.array(R['bounds'], np.float32).tobytes() == np.array([b[0], b[2], b[1], b[3]], np.float32).tobytes()
    ref = _oracle_chain(K, D, W, H, scene, R['bounds'], R['sf'])
    for f, o in enumerate(ref):
        k = int(R['n'][f])
        assert k == len(o['kps']) and R['kps'][f, :k].tobytes() == o['kps'].tobytes(), f
        assert np.array_equal(R['desc'][f, :k], o['desc']), f
        assert R['nm_search'][f] == o['n_search'] > 200, (f, R['nm_search'][f], o['n_search'])
        assert R['match'][f, :k].tobytes() == o['match'].tobytes() and R['claimed'][f, :k].tobytes() == o['claimed'].tobytes(), f
        assert R['nmatches'][f] == o['nmatches'] and R['nmatchesMap'][f] == o['nmatchesMap'], f
        m = len(scene[f]['lk'])
        assert R['discarded'][f, :m].tobytes() == o['discarded'].tobytes(), f
        assert np.abs(R['pose7'][f] - o['pose7']).max() < 1e-8, f


def test_track_local_map_resident_with_undistorted_slab(orb, chain):
    """orbm_track_local_map_batch_resident reading the handle's undistorted slab (orbx_undistort_keypoints) equals TrackLocalMap's
    oracle chain on the oracle's undistorted keypoints.  The local map holds the last frame's points."""
    K, D, W, H, scene, R = chain
    B, cap = len(scene), R['cap']
    ex = orb.ORBextractor(1000, 1.2, 8, 20, 7, W, H, B)
    ex.extract_batch(np.stack([s['img'] for s in scene]), (0, 1000))
    ptr, host = ex.undistort_keypoints(K, D, batch=B)
    _, d_desc, d_n, rcap = ex.resident_slabs()
    assert rcap == cap
    g = _globals(K, R['bounds'], R['sf'])
    M = max(len(s['lk']) for s in scene)
    lo_arr = {k: np.zeros((B, M) + sh, dt) for k, sh, dt in (('worldPos', (3,), np.float32), ('normal', (3,), np.float32), ('minDistInv', (), np.float32),
                                                              ('maxDistInv', (), np.float32), ('maxDistance', (), np.float32), ('mpDesc', (32,), np.uint8),
                                                              ('hasObs', (), np.uint8), ('bad', (), np.uint8))}
    sts, th = [], np.full(B, 1.0, np.float32)
    for b, s in enumerate(scene):
        m = len(s['lk'])
        _, _, Ow = T.pose_matrices(R['Tcw7'][b])
        P = s['xyz'].astype(np.float64)
        PO = P - Ow.astype(np.float64)
        dist = np.linalg.norm(PO, axis=1)
        dmax = (dist * 1.2 ** s['lk']['octave']).astype(np.float32)
        st = dict(kps=host[b, :R['n'][b]], desc=R['desc'][b, :R['n'][b]], nM=m, lastToLocal=np.arange(m, dtype=np.int32), bad=np.zeros(m, np.uint8),
                  hasObs=s['hasObs'], worldPos=s['xyz'], normal=(PO / dist[:, None]).astype(np.float32), minDistInv=(np.float32(0.8) * dmax / np.float32(1.2 ** 7)).astype(np.float32),
                  maxDistInv=(np.float32(1.2) * dmax).astype(np.float32), maxDistance=dmax, mpDesc=s['ld'])
        sts.append(st)
        for k in lo_arr:
            lo_arr[k][b, :m] = st[k]
    l2l = np.full((B, cap), -1, np.int32); disc = np.zeros((B, cap), np.uint8)
    for b, s in enumerate(scene):
        l2l[b, :len(s['lk'])] = np.arange(len(s['lk'])); disc[b] = R['discarded'][b]
    lo = dict(batch=B, kcap=cap, mcap=M, mcapLast=cap, nlevels=8, kps=host, desc=R['desc'], nK=R['n'], bounds=R['bounds'], scaleFactors=R['sf'],
              invLevelSigma2=g['invLevelSigma2'], cam=tuple(float(c) for c in K), mbf=0.0, logScaleFactor=g['logScaleFactor'], Tcw7=R['Tcw7'].copy(),
              lastToLocal=l2l, discarded=disc, nM=np.array([len(s['lk']) for s in scene], np.int32), th=th, nnratio=g['nnratio'], bFarPoints=0,
              thFarPoints=0.0, viewingCosLimit=g['viewingCosLimit'], active=None, **lo_arr)
    m = orb.ORBmatcher(0.8, False, max_batch=B, max_keypoints=cap, max_mappoints=cap)
    match = R['match'].copy()
    r2 = m.track_local_map_batch(lo, match, resident=(ptr, d_desc, d_n, cap))
    for b, st in enumerate(sts):
        k = int(R['n'][b])
        lm = T.local_map_step(T.OracleBackend(), st, g, R['match'][b, :k].copy(), R['discarded'][b, :st['nM']], R['Tcw7'][b], th[b])
        assert match[b, :k].tobytes() == lm['match'].tobytes() and r2['claimed'][b, :k].tobytes() == lm['claimed'].tobytes(), b
        for key in ('nToMatch', 'nmatches', 'nInliers', 'nMatchesInliers'):
            assert r2[key][b] == lm[key], (key, b, r2[key][b], lm[key])
        assert r2['visible'][b, :st['nM']].tobytes() == lm['visible'].tobytes() and r2['found'][b, :st['nM']].tobytes() == lm['found'].tobytes(), b
        assert np.abs(r2['pose7'][b] - lm['pose7']).max() < 1e-8, b
    assert (r2['nInliers'] > 200).all()


def test_undistorted_chain_tracks_better_than_the_distorted_slab(orb, chain):
    """Against the render's true poses: the chain fed mvKeysUn beats the same chain fed the distorted slab, the gap this closes."""
    K, D, W, H, scene, R = chain
    Rd = _device_chain(orb, K, D, W, H, scene, undistort=False)
    err_un = [_pose_error(R['pose7'][b], s['true']) for b, s in enumerate(scene)]
    err_d = [_pose_error(Rd['pose7'][b], s['true']) for b, s in enumerate(scene)]
    assert max(err_un) < 0.01, err_un
    assert all(u < d for u, d in zip(err_un, err_d)), (err_un, err_d)
    assert (R['nmatches'] > Rd['nmatches']).all(), (R['nmatches'], Rd['nmatches'])


def test_cpp_undistort_equals_python(orb, frames, tmp_path):
    """FrameView::UndistortKeyPoints / ComputeImageBounds (include/orb_b200/orb_slam3.hpp) from a g++-built caller equal the Python binding."""
    K, D, W, H = U.CALIBRATIONS['tum1']
    img = frames['tum1'][2]
    (tmp_path / 'image.raw').write_bytes(np.ascontiguousarray(img).tobytes())
    (tmp_path / 'dims.txt').write_text('%d %d %s\n' % (H, W, ' '.join('%.9g' % v for v in U.cam9(K, D))))
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib = os.path.join(root, 'orb_slam3_modified_b200')
    exe = tmp_path / 'undistort_example'
    subprocess.check_call(['g++', '-std=c++14', '-O2', '-Wall', '-I', os.path.join(root, 'include'), os.path.join(root, 'tests', 'undistort_example.cpp'),
                           '-o', str(exe), '-L', lib, '-l:liborb_b200.so', '-Wl,-rpath,' + lib, '-lpthread'])
    out = dict(l.split() for l in subprocess.check_output([str(exe), str(tmp_path)]).decode().splitlines())
    ex = orb.ORBextractor(1000, 1.2, 8, 20, 7, W, H, 1)
    _, kps, _ = ex(img, (0, 1000))
    _, un = ex.undistort_keypoints(K, D, batch=1)
    assert int(out['n']) == len(kps) > 800
    assert (tmp_path / 'kpsUn.raw').read_bytes() == un[0, :len(kps)].tobytes()
    b = orb.image_bounds(K, D, W, H)
    want = np.array([b[0], b[2], b[1], b[3]], np.float32).view(np.uint32)
    assert out['bounds'] == ','.join('%08x' % v for v in want)
