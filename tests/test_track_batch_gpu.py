"""GPU tests of orbm_motion_model_pose_batch* and orbm_track_local_map_batch*: byte for byte equal to the per-frame chain of the library's
existing entry points (tests/track_lib.py), equal to the CPU oracle chain in the matches, and the batch / host / device / resident
forms agree."""
import numpy as np
import pytest

import track_lib as T

pytestmark = pytest.mark.gpu
KINDS = ('normal', 'normal', 'empty', 'all_seen', 'few', 'nine', 'normal')
THS = (1.0, 2.0, 5.0, 10.0, 15.0)


@pytest.fixture(scope='module')
def orb():
    import orb_slam3_modified_b200 as m
    return m


def torch_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _streams(B, seed, g):
    out = []
    for b in range(B):
        kind = KINDS[b] if b < len(KINDS) else 'normal'
        out.append(T.stream(seed * 1000 + b, g, M=300 + 97 * (b % 9), K_extra=20 + 13 * (b % 5), kind=kind))
    return out


def _batched(m, streams, g, th, active=None):
    mo, lo, state = T.batch(streams, g, th, active=active)
    match, claimed, nm = state['match'].copy(), state['claimed'].copy(), state['nmatches'].copy()
    r1 = m.motion_model_pose_batch(mo, g['invLevelSigma2'], match, claimed, nm, active=active)
    lo['Tcw7'] = r1['Tcw7']; lo['discarded'] = r1['discarded']
    match_last = match.copy()
    r2 = m.track_local_map_batch(lo, match)
    return dict(mo=mo, lo=lo, r1=r1, r2=r2, match_last=match_last, claimed1=claimed, nmatches1=nm, match=match)


def _chain(be, streams, g, th):
    res = []
    for b, st in enumerate(streams):
        match, claimed = st['match'].copy(), st['claimed'].copy()
        mm = T.motion_model_step(be, st, g, match, claimed, st['nmatches'])
        disc = mm['discarded']
        lm = T.local_map_step(be, st, g, match, disc, mm['Tcw7'], th[b])
        res.append((match, claimed, mm, lm))
    return res


def _same_bytes(a, b, what):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    assert a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes(), what


def _compare(R, chain, streams, exact=True):
    for b, (match_last, claimed1, mm, lm) in enumerate(chain):
        K, M, ML = len(streams[b]['kps']), streams[b]['nM'], streams[b]['mcapLast']
        _same_bytes(R['match_last'][b, :K], match_last, ('motion match', b))
        _same_bytes(R['claimed1'][b, :K], claimed1, ('motion claimed', b))
        assert R['nmatches1'][b] == mm['nmatches'] and R['r1']['nmatchesMap'][b] == mm['nmatchesMap'], b
        _same_bytes(R['r1']['discarded'][b, :ML], mm['discarded'], ('discarded', b))
        _same_bytes(R['match'][b, :K], lm['match'], ('local match', b))
        _same_bytes(R['r2']['claimed'][b, :K], lm['claimed'], ('local claimed', b))
        r2 = R['r2']
        for k in ('nToMatch', 'nmatches', 'nInliers', 'nMatchesInliers'):
            assert r2[k][b] == lm[k], (k, b, r2[k][b], lm[k])
        if exact:
            _same_bytes(r2['outlier'][b, :K], lm['outlier'], ('outlier', b))
            _same_bytes(r2['visible'][b, :M], lm['visible'], ('visible', b))
            _same_bytes(r2['found'][b, :M], lm['found'], ('found', b))
            _same_bytes(R['r1']['pose7'][b], mm['pose7'], ('motion pose7', b))
            _same_bytes(R['r1']['Tcw7'][b], mm['Tcw7'], ('motion Tcw7', b))
            _same_bytes(r2['pose7'][b], lm['pose7'], ('pose7', b))
            _same_bytes(r2['Tcw7'][b], lm['Tcw7'], ('Tcw7', b))
        else:
            assert np.abs(r2['pose7'][b] - lm['pose7']).max() < 1e-8 and np.abs(R['r1']['pose7'][b] - mm['pose7']).max() < 1e-8


@pytest.mark.parametrize('B,far', [(1, False), (7, False), (7, True), (37, False), (88, True), (240, False)])
def test_equals_per_frame_chain_of_existing_entry_points(orb, B, far):
    """B = 37, 88 and 240 run the local-map search with clusters of fewer than 8 CTAs (batch x size <= 2 x SMs)."""
    g = T.globals_()
    if far:
        g.update(bFarPoints=1, thFarPoints=7.0)
    streams = _streams(B, 7 + B + int(far), g)
    th = np.array([THS[b % len(THS)] for b in range(B)], np.float32)
    m = orb.ORBmatcher(0.8, False, max_batch=B, max_keypoints=2048, max_mappoints=2048, device=0)
    R = _batched(m, streams, g, th)
    assert m.last_launch_count() == 5
    assert B * m.last_cluster_size() <= 2 * torch_sms() and (B <= 33 or m.last_cluster_size() < 8), m.last_cluster_size()
    _compare(R, _chain(T.GpuChainBackend(orb, orb.ORBmatcher(0.8, False, max_batch=1, max_keypoints=2048, max_mappoints=2048)), streams, g, th), streams)
    assert (R['r2']['nmatches'] > 0).any() and (R['r1']['discarded'] > 0).any()
    if B > 1:   # the scene with one point held at two keypoints is among them
        assert (R['r2']['visible'] >= 2).any() and (R['r2']['nToMatch'] == 0).any() and (R['r2']['nInliers'] == 0).any()
    if B == 7:   # the CPU oracle chain: matches equal, poses within 1e-8 (the FP64 sums are ordered differently there)
        _compare(R, _chain(T.OracleBackend(), streams, g, th), streams, exact=False)
    # two calls give the same bytes
    R2 = _batched(m, streams, g, th)
    for k in R['r2']:
        _same_bytes(R['r2'][k], R2['r2'][k], k)
    for k in R['r1']:
        _same_bytes(R['r1'][k], R2['r1'][k], k)


def test_inactive_streams_untouched_and_forms_agree(orb):
    import torch
    g = T.globals_()
    streams = _streams(7, 5, g)
    th = np.array([1, 5, 15, 2, 10, 1, 1], np.float32)
    m = orb.ORBmatcher(0.8, False, max_batch=7, max_keypoints=2048, max_mappoints=2048, device=0)
    full = _batched(m, streams, g, th)
    active = np.array([1, 0, 1, 1, 0, 1, 0], np.uint8)
    mo, lo, state = T.batch(streams, g, th, active=active)
    match, claimed, nm = state['match'].copy(), state['claimed'].copy(), state['nmatches'].copy()
    r1 = m.motion_model_pose_batch(mo, g['invLevelSigma2'], match, claimed, nm, active=active)
    for b in range(7):
        if active[b]:
            _same_bytes(match[b], full['match_last'][b], b); _same_bytes(r1['Tcw7'][b], full['r1']['Tcw7'][b], b)
        else:
            _same_bytes(match[b], state['match'][b], b); _same_bytes(claimed[b], state['claimed'][b], b)
            assert nm[b] == state['nmatches'][b] and not r1['Tcw7'][b].any()
    lo['Tcw7'] = full['r1']['Tcw7']; lo['discarded'] = full['r1']['discarded']
    match2 = full['match_last'].copy()
    r2 = m.track_local_map_batch(lo, match2)
    for b in range(7):
        if active[b]:
            _same_bytes(match2[b], full['match'][b], b)
            for k in r2:
                _same_bytes(r2[k][b], full['r2'][k][b], (k, b))
        else:
            _same_bytes(match2[b], full['match_last'][b], b)
            assert all(not r2[k][b].any() for k in r2)
    # device form (torch) and resident form agree with the host form byte for byte
    lo['active'] = None
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8) if a.dtype.fields else np.ascontiguousarray(a)).cuda()
    dl = {k: (dev(v) if isinstance(v, np.ndarray) else v) for k, v in lo.items()}
    B, K, M = lo['batch'], lo['kcap'], lo['mcap']
    out = dict(match=dev(full['match_last']), claimed=torch.zeros((B, K), dtype=torch.uint8, device='cuda'), outlier=torch.zeros((B, K), dtype=torch.uint8, device='cuda'),
               visible=torch.zeros((B, M), dtype=torch.int32, device='cuda'), found=torch.zeros((B, M), dtype=torch.int32, device='cuda'),
               pose7=torch.zeros((B, 7), dtype=torch.float64, device='cuda'), Tcw7=torch.zeros((B, 7), dtype=torch.float32, device='cuda'),
               **{k: torch.zeros(B, dtype=torch.int32, device='cuda') for k in ('nToMatch', 'nmatches', 'nInliers', 'nMatchesInliers')})
    m.track_local_map_batch_device(dl, out, stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    _same_bytes(out['match'].cpu().numpy(), full['match'], 'device match')
    for k in full['r2']:
        _same_bytes(out[k].cpu().numpy(), full['r2'][k], ('device', k))
    # resident: the frame from an extractor-like device slab
    res = (dl['kps'].data_ptr(), dl['desc'].data_ptr(), dl['nK'].data_ptr(), K)
    match3 = full['match_last'].copy()
    r3 = m.track_local_map_batch(lo, match3, resident=res)
    _same_bytes(match3, full['match'], 'resident match')
    for k in r3:
        _same_bytes(r3[k], full['r2'][k], ('resident', k))
    # motion-model device form
    mo_full, _, st0 = T.batch(streams, g, th)
    md = {k: (dev(v) if isinstance(v, np.ndarray) else v) for k, v in mo_full.items()}
    dm, dc, dn = dev(st0['match']), dev(st0['claimed']), dev(st0['nmatches'])
    p7 = torch.zeros((B, 7), dtype=torch.float64, device='cuda'); t7 = torch.zeros((B, 7), dtype=torch.float32, device='cuda')
    dd = torch.zeros((B, mo_full['mcap']), dtype=torch.uint8, device='cuda'); nmm = torch.zeros(B, dtype=torch.int32, device='cuda')
    m.motion_model_pose_batch_device(md, dev(g['invLevelSigma2']), dm, dc, dn, p7, t7, dd, nmm, stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    _same_bytes(dm.cpu().numpy(), full['match_last'], 'device motion match')
    _same_bytes(t7.cpu().numpy(), full['r1']['Tcw7'], 'device motion Tcw7')
    _same_bytes(p7.cpu().numpy(), full['r1']['pose7'], 'device motion pose7')
    _same_bytes(dd.cpu().numpy(), full['r1']['discarded'], 'device discarded')


def test_bad_arguments_and_capacity(orb):
    g = T.globals_()
    streams = _streams(2, 9, g)
    m = orb.ORBmatcher(0.8, False, max_batch=2, max_keypoints=2048, max_mappoints=2048, device=0)
    m.track_local_map_batch(*(lambda mo, lo, st: (lo, st['match']))(*T.batch(streams, g, [1, 1])))
    n0 = m.last_launch_count()
    def expect(code, **kw):
        mo, lo, st = T.batch(streams, g, [1, 1])
        for k, v in kw.items():
            v(lo, st)
        with pytest.raises(orb.OrbError) as ei:
            m.track_local_map_batch(lo, st['match'])
        assert ei.value.code == code
    def oct_(lo, st): lo['kps']['octave'][0, 0] = 8
    def l2l(lo, st): lo['lastToLocal'][0, 0] = 10 ** 6
    def match(lo, st): st['match'][1, 0] = lo['mcapLast']
    def nm(lo, st): lo['nM'][0] = lo['mcap'] + 1
    def nk(lo, st): lo['nK'][1] = lo['kcap'] + 1
    def batch(lo, st):                                   # more streams than the handle's max_batch
        lo['batch'] = 3; st['match'] = np.full((3, lo['kcap']), -1, np.int32)
    for f in (oct_, l2l, match, nm, nk, batch):
        expect(orb.ORB_ERR_ARG, f=f)
    small = orb.ORBmatcher(0.8, False, max_batch=2, max_keypoints=2048, max_mappoints=100, device=0)
    mo, lo, st = T.batch(streams, g, [1, 1])            # local maps of 300+ points
    with pytest.raises(orb.OrbError) as ei:
        small.track_local_map_batch(lo, st['match'])
    assert ei.value.code == orb.ORB_ERR_CAPACITY
    def mm_oct(mo, st): mo['kps']['octave'][0, 0] = -1
    def mm_nk(mo, st): mo['nK'][1] = mo['kcap'] + 1
    def mm_match(mo, st): st['match'][1, 0] = mo['mcap']
    for f in (mm_oct, mm_nk, mm_match):
        mo, lo, st = T.batch(streams, g, [1, 1])
        f(mo, st)
        with pytest.raises(orb.OrbError) as ei:
            m.motion_model_pose_batch(mo, g['invLevelSigma2'], st['match'], st['claimed'], st['nmatches'])
        assert ei.value.code == orb.ORB_ERR_ARG, f
    assert m.last_launch_count() == n0 == 5


def test_launch_count_independent_of_batch(orb):
    g = T.globals_()
    counts = []
    for B in (1, 240):
        m = orb.ORBmatcher(0.8, False, max_batch=B, max_keypoints=2048, max_mappoints=2048, device=0)
        mo, lo, st = T.batch(_streams(B, 3, g), g, np.ones(B, np.float32))
        m.motion_model_pose_batch(mo, g['invLevelSigma2'], st['match'], st['claimed'], st['nmatches'])
        c1 = m.last_launch_count()
        m.track_local_map_batch(lo, st['match'])
        counts.append((c1, m.last_launch_count()))
    assert counts[0] == counts[1] == (3, 5)
