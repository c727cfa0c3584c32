"""GPU tests of orbm_track_reference_keyframe_batch*: byte for byte equal to the per-frame chain of the library's existing entry points
(orbv_transform_batch + SearchByBoW + PoseOptimization, tests/track_ref_lib.py), equal to the CPU oracle chain, the host / device / resident
forms agree, and the device outputs chain into orbm_track_local_map_batch_device through the index space [keyframe features |
last-frame points]."""
import numpy as np
import pytest

import track_lib as T
import track_ref_lib as TR

pytestmark = pytest.mark.gpu
KINDS = ('normal', 'n14', 'n15', 'map9', 'fallback', 'normal', 'normal')


@pytest.fixture(scope='module')
def orb():
    import orb_slam3_modified_b200 as m
    return m


@pytest.fixture(scope='module')
def voc():
    return TR.ref_vocabulary()


def _streams(B, seed, g, voc):
    return [TR.ref_kf_stream(seed * 1000 + b, g, voc, kind=KINDS[b] if b < len(KINDS) else 'normal', M=300 + 37 * (b % 7), K_extra=20 + 11 * (b % 5))
            for b in range(B)]


def _same_bytes(a, b, what):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    assert a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes(), what


def _compare(R, chain, streams, exact=True):
    for b, r in enumerate(chain):
        K, N = len(streams[b]['kps']), len(streams[b]['kf_kps'])
        assert R['nmatches'][b] == r['nmatches'], (b, R['nmatches'][b], r['nmatches'])
        _same_bytes(R['match'][b, :K], r['match'], ('match', b))
        assert (R['match'][b, K:] == -1).all()
        if not r['gated']:                                # below the gate: the pose outputs are not written
            assert not R['pose7'][b].any() and not R['Tcw7'][b].any() and not R['discarded'][b].any() and R['nmatchesMap'][b] == 0, b
            continue
        assert R['nmatchesMap'][b] == r['nmatchesMap'], b
        _same_bytes(R['discarded'][b, :N], r['discarded'], ('discarded', b))
        assert not R['discarded'][b, N:].any()
        if exact:
            _same_bytes(R['pose7'][b], r['pose7'], ('pose7', b))
            _same_bytes(R['Tcw7'][b], r['Tcw7'], ('Tcw7', b))
        else:
            assert np.allclose(R['pose7'][b], r['pose7'], atol=1e-9), b   # PoseOptimization's parity test (tests/test_poseopt_gpu.py)
            assert np.abs(R['Tcw7'][b].astype(np.float64) - r['Tcw7']).max() < 1e-6, b


@pytest.mark.parametrize('B', [1, 7, 240])
def test_equals_per_frame_chain_of_existing_entry_points(orb, voc, B):
    g = T.globals_()
    streams = _streams(B, 3 + B, g, voc)
    m = orb.ORBmatcher(0.8, False, max_batch=B, max_keypoints=2048, max_mappoints=2048, device=0)
    d = TR.ref_batch(streams, g)
    R = m.track_reference_keyframe_batch(d)
    assert m.last_launch_count() == 4
    gpu = TR.GpuChainBackend(orb, orb.ORBmatcher(0.7, True, max_batch=1, max_keypoints=2048, max_mappoints=2048), voc)
    chain = [TR.reference_keyframe_step(gpu, st, g) for st in streams]
    for st, r in zip(streams, chain):                     # the library's transform is the oracle's
        assert all(np.array_equal(a, b) for a, b in zip(r['fv'] + r['kf_fv'], st['fv'] + st['kf_fv']))
    _compare(R, chain, streams)
    if B >= 7:                                            # the planted cases are reached
        assert R['nmatches'][1] == 14 and R['nmatches'][2] == 15 and R['nmatchesMap'][3] < 10 <= R['nmatches'][3]
        assert (R['discarded'].sum(1) > 0).any()
        _compare(R, [TR.reference_keyframe_step(TR.OracleBackend(voc), st, g) for st in streams], streams, exact=False)
    R2 = m.track_reference_keyframe_batch(d)
    for k in R:
        _same_bytes(R[k], R2[k], ('repeat', k))


def test_inactive_streams_untouched_and_forms_agree(orb, voc):
    import torch
    g = T.globals_()
    streams = _streams(7, 5, g, voc)
    m = orb.ORBmatcher(0.8, False, max_batch=7, max_keypoints=2048, max_mappoints=2048, device=0)
    d = TR.ref_batch(streams, g)
    full = m.track_reference_keyframe_batch(d)
    active = np.array([1, 1, 1, 0, 1, 0, 1], np.uint8)
    R = m.track_reference_keyframe_batch(dict(d, active=active))
    for b in range(7):
        for k in R:
            if active[b]:
                _same_bytes(R[k][b], full[k][b], (k, b))
            else:                                         # the wrapper's initial values: match -1, the rest 0
                assert (R[k][b] == (-1 if k == 'match' else 0)).all(), (k, b)
    # device form on torch tensors prefilled with a sentinel: inactive streams and streams below the gate keep it
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8) if a.dtype.fields else np.ascontiguousarray(a)).cuda()
    dd = {k: (dev(v) if isinstance(v, np.ndarray) else v) for k, v in dict(d, active=active).items()}
    B, K, M = d['batch'], d['kcap'], d['mcap']
    out = dict(nmatches=torch.full((B,), 77, dtype=torch.int32, device='cuda'), match=torch.full((B, K), 77, dtype=torch.int32, device='cuda'),
               pose7=torch.full((B, 7), 77.0, dtype=torch.float64, device='cuda'), Tcw7=torch.full((B, 7), 77.0, dtype=torch.float32, device='cuda'),
               discarded=torch.full((B, M), 77, dtype=torch.uint8, device='cuda'), nmatchesMap=torch.full((B,), 77, dtype=torch.int32, device='cuda'))
    m.track_reference_keyframe_batch_device(dd, out, stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert m.last_launch_count() == 4
    o = {k: v.cpu().numpy() for k, v in out.items()}
    for b in range(7):
        gated = active[b] and full['nmatches'][b] >= 15
        for k in o:
            if k in ('nmatches', 'match') and active[b] or k not in ('nmatches', 'match') and gated:
                _same_bytes(o[k][b], full[k][b], ('device', k, b))
            else:
                assert (o[k][b] == 77).all(), ('device untouched', k, b)
    assert active[1] and full['nmatches'][1] == 14            # an active stream below the gate
    # resident form: the current frame (keypoints, descriptors, FeatureVector) from device slabs
    res = tuple(dd[k].data_ptr() for k in ('kps', 'desc', 'nK', 'fvNode', 'fvFeature', 'nEntries'))
    R3 = m.track_reference_keyframe_batch(d, resident=res)
    for k in R3:
        _same_bytes(R3[k], full[k], ('resident', k))


def test_bad_arguments_and_capacity(orb, voc):
    g = T.globals_()
    streams = _streams(2, 9, g, voc)
    m = orb.ORBmatcher(0.8, False, max_batch=2, max_keypoints=2048, max_mappoints=2048, device=0)
    m.track_reference_keyframe_batch(TR.ref_batch(streams, g))
    assert m.last_launch_count() == 4
    m.SearchByBoW(*[streams[0][k] for k in ('kf_kps', 'kf_desc', 'kfPoint', 'kf_fv', 'kps', 'desc', 'fv')])
    n0 = m.last_launch_count()
    assert n0 == 1

    def expect(code, f, handle=m):
        d = TR.ref_batch(streams, g)
        f(d)
        with pytest.raises(orb.OrbError) as ei:
            handle.track_reference_keyframe_batch(d)
        assert ei.value.code == code, f
        assert m.last_launch_count() == n0                # rejected before any launch

    def octave(d): d['kps']['octave'][1, 0] = 8
    def unsorted(d): d['fvNode'][0, 0] = d['fvNode'][0, 1] + 1
    def kf_unsorted(d): d['kfFvNode'][1, 0] = d['kfFvNode'][1, 1] + 1
    def feat_range(d): d['fvFeature'][0, 0] = d['nK'][0]
    def kf_feat_range(d): d['kfFvFeature'][0, 0] = -1
    def kf_n(d): d['kfN'][1] = d['mcap'] + 1
    def n_entries(d): d['nEntries'][0] = d['nK'][0] + 1
    def n_k(d): d['nK'][1] = d['kcap'] + 1
    def batch(d):
        d['batch'] = 3
    for f in (octave, unsorted, kf_unsorted, feat_range, kf_feat_range, kf_n, n_entries, n_k, batch):
        expect(orb.ORB_ERR_ARG, f)
    small = orb.ORBmatcher(0.8, False, max_batch=2, max_keypoints=2048, max_mappoints=100, device=0)
    expect(orb.ORB_ERR_CAPACITY, lambda d: None, small)
    narrow = orb.ORBmatcher(0.8, False, max_batch=2, max_keypoints=100, max_mappoints=2048, device=0)
    expect(orb.ORB_ERR_CAPACITY, lambda d: None, narrow)


@pytest.mark.parametrize('B', [1, 24, 240])
def test_launch_count_independent_of_batch(orb, voc, B):
    g = T.globals_()
    m = orb.ORBmatcher(0.8, False, max_batch=B, max_keypoints=2048, max_mappoints=2048, device=0)
    streams = [TR.ref_kf_stream(40 + (b % 3), g, voc) for b in range(B)]
    m.track_reference_keyframe_batch(TR.ref_batch(streams, g))
    assert m.last_launch_count() == 4


def test_chains_into_track_local_map_on_the_device(orb, voc):
    """Device outputs -> orbm_track_local_map_batch_device with lastToLocal = [kfToLocal | last-frame map] and discarded = [this call's
    marks | the failed motion-model step's marks] concatenated on the device; equal to the oracle's TrackReferenceKeyFrame ->
    TrackLocalMap chain, the fallback stream included."""
    import torch
    g = T.globals_()
    streams = _streams(7, 13, g, voc)
    B = len(streams)
    th = np.array([1, 1, 5, 1, 2, 1, 15], np.float32)
    m = orb.ORBmatcher(0.8, False, max_batch=B, max_keypoints=2048, max_mappoints=2048, device=0)
    d = TR.ref_batch(streams, g)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8) if a.dtype.fields else np.ascontiguousarray(a)).cuda()
    dd = {k: (dev(v) if isinstance(v, np.ndarray) else v) for k, v in d.items()}
    K, MK = d['kcap'], d['mcap']
    out = dict(nmatches=torch.zeros(B, dtype=torch.int32, device='cuda'), match=torch.full((B, K), -1, dtype=torch.int32, device='cuda'),
               pose7=torch.zeros((B, 7), dtype=torch.float64, device='cuda'), Tcw7=torch.zeros((B, 7), dtype=torch.float32, device='cuda'),
               discarded=torch.zeros((B, MK), dtype=torch.uint8, device='cuda'), nmatchesMap=torch.zeros(B, dtype=torch.int32, device='cuda'))
    st_ = torch.cuda.current_stream().cuda_stream
    m.track_reference_keyframe_batch_device(dd, out, stream=st_)
    # the oracle chain: the fallback stream's motion-model step first, then TrackReferenceKeyFrame
    oracle = TR.OracleBackend(voc)
    mm_dis = [None] * B
    for b, s in enumerate(streams):
        if s['kind'] == 'fallback':
            match, claimed = s['match'].copy(), s['claimed'].copy()
            mm = T.motion_model_step(oracle, s, g, match, claimed, s['nmatches'])
            assert mm['nmatchesMap'] < 10 and mm['discarded'].any()
            mm_dis[b] = mm['discarded']
    ref = [TR.reference_keyframe_step(oracle, s, g) for s in streams]
    ok = np.array([r['gated'] and r['nmatchesMap'] >= 10 for r in ref], np.uint8)   # the host's success test, monocular
    assert ok.sum() >= 4 and not ok[1] and not ok[3]
    _, lo, _ = T.batch(streams, g, th, active=ok)
    mL = lo['mcapLast']
    l2l, mm_rows = TR.concat_index_space(streams, MK, mL, [np.zeros(MK, np.uint8)] * B, mm_dis)
    lo.update(mcapLast=MK + mL, lastToLocal=l2l)
    dl = {k: (dev(v) if isinstance(v, np.ndarray) else v) for k, v in lo.items()}
    dl['Tcw7'] = out['Tcw7']
    dl['discarded'] = torch.cat([out['discarded'], dev(mm_rows[:, MK:])], 1).contiguous()   # on the device: no host round trip
    M = lo['mcap']
    lm = dict(match=out['match'].clone(), claimed=torch.zeros((B, K), dtype=torch.uint8, device='cuda'), outlier=torch.zeros((B, K), dtype=torch.uint8, device='cuda'),
              visible=torch.zeros((B, M), dtype=torch.int32, device='cuda'), found=torch.zeros((B, M), dtype=torch.int32, device='cuda'),
              pose7=torch.zeros((B, 7), dtype=torch.float64, device='cuda'), Tcw7=torch.zeros((B, 7), dtype=torch.float32, device='cuda'),
              **{k: torch.zeros(B, dtype=torch.int32, device='cuda') for k in ('nToMatch', 'nmatches', 'nInliers', 'nMatchesInliers')})
    m.track_local_map_batch_device(dl, lm, stream=st_)
    torch.cuda.synchronize()
    o = {k: v.cpu().numpy() for k, v in lm.items()}
    Rr = {k: v.cpu().numpy() for k, v in out.items()}
    _compare(Rr, ref, streams, exact=False)
    for b, s in enumerate(streams):
        if not ok[b]:
            continue
        dis = np.zeros(MK + mL, np.uint8)                 # the same index space, built on the host for the oracle
        dis[:len(ref[b]['discarded'])] = ref[b]['discarded']
        if mm_dis[b] is not None:
            dis[MK:MK + len(mm_dis[b])] = mm_dis[b]
        r = T.local_map_step(oracle, dict(s, lastToLocal=l2l[b]), g, ref[b]['match'], dis, ref[b]['Tcw7'], th[b])
        Kb, Mb = len(s['kps']), s['nM']
        _same_bytes(o['match'][b, :Kb], r['match'], ('local match', b))
        _same_bytes(o['outlier'][b, :Kb], r['outlier'], ('outlier', b))
        _same_bytes(o['visible'][b, :Mb], r['visible'], ('visible', b))
        _same_bytes(o['found'][b, :Mb], r['found'], ('found', b))
        for k in ('nToMatch', 'nmatches', 'nInliers', 'nMatchesInliers'):
            assert o[k][b] == r[k], (k, b, o[k][b], r[k])
        assert np.abs(o['pose7'][b] - r['pose7']).max() < 1e-8, b


def test_cpp_batch_tracker_equals_python(orb, voc, tmp_path):
    """BatchTracker::TrackReferenceKeyFrame (include/orb_b200/orb_slam3.hpp) from a g++-built caller: byte for byte the Python binding's."""
    import os
    import subprocess
    g = T.globals_()
    streams = _streams(5, 17, g, voc)
    d = TR.ref_batch(streams, g, active=np.array([1, 1, 1, 0, 1], np.uint8))
    m = orb.ORBmatcher(0.8, False, max_batch=5, max_keypoints=d['kcap'], max_mappoints=d['mcap'], device=0)
    (tmp_path / 'dims.txt').write_text(' '.join(str(v) for v in (d['batch'], d['kcap'], d['mcap'], d['nlevels']) + tuple(repr(float(c)) for c in d['cam'])))
    for k, dt in m._REF_KF_DT.items():
        (tmp_path / (k + '.raw')).write_bytes(np.ascontiguousarray(d[k], dt).tobytes())
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib = os.path.join(root, 'orb_slam3_modified_b200')
    exe = tmp_path / 'track_reference_kf_example'
    subprocess.check_call(['g++', '-std=c++14', '-O2', '-Wall', '-I', os.path.join(root, 'include'), os.path.join(root, 'tests', 'track_reference_kf_example.cpp'),
                           '-o', str(exe), '-L', lib, '-l:liborb_b200.so', '-Wl,-rpath,' + lib, '-lpthread'])
    out = subprocess.check_output([str(exe), str(tmp_path)]).decode()
    assert 'launches 4' in out
    R = m.track_reference_keyframe_batch(d)
    for k in R:
        assert (tmp_path / (k + '.out')).read_bytes() == np.ascontiguousarray(R[k]).tobytes(), k
