"""CPU tests of the reference-keyframe path's reference: the oracle chain of tests/track_ref_lib.py (bow_transform + search_by_bow +
pose_optimization, then TrackLocalMap) on planted scenes, checked against a literal restatement that follows mnLastFrameSeen and
mbTrackInView per map point through TrackWithMotionModel (when it failed) -> TrackReferenceKeyFrame -> SearchLocalPoints.  No GPU needed."""

import numpy as np
import pytest

import track_lib as T
import track_ref_lib as TR

CUR = 7                                                   # mCurrentFrame.mnId


@pytest.fixture(scope='module')
def voc():
    return TR.ref_vocabulary()


def _restatement(st, g, mm, ref):
    """SearchLocalPoints' bookkeeping over map points (local indices) as the reference writes it: returns (frame points, lastFrameSeen,
    trackInView, visible before the search, nToMatch)."""
    M = st['nM']
    lastFrameSeen = np.full(M, -1); trackInView = np.zeros(M, bool); visible = np.zeros(M, np.int32)
    if mm is not None:                                    # TrackWithMotionModel's discard loop (it then failed)
        for j in np.nonzero(mm['discarded'])[0]:
            p = st['lastToLocal'][j]
            if p >= 0:
                trackInView[p] = False; lastFrameSeen[p] = CUR
    for j in np.nonzero(ref['discarded'])[0]:             # TrackReferenceKeyFrame's discard loop
        p = st['kfToLocal'][j]
        if p >= 0:
            trackInView[p] = False; lastFrameSeen[p] = CUR
    frame = {}
    for i, j in enumerate(ref['match']):                  # mCurrentFrame.mvpMapPoints = the BoW matches after the loop
        if j >= 0 and st['kfToLocal'][j] >= 0 and not st['bad'][st['kfToLocal'][j]]:
            p = st['kfToLocal'][j]
            frame[i] = p; visible[p] += 1; lastFrameSeen[p] = CUR; trackInView[p] = False
    R, t, Ow = T.pose_matrices(ref['Tcw7'])
    pts = {k: st[k][:M] for k in ('worldPos', 'normal', 'minDistInv', 'maxDistInv', 'maxDistance')}
    fr = T.OracleBackend().frustum(pts, R, t, Ow, g)
    n = 0
    for p in range(M):
        if lastFrameSeen[p] == CUR or st['bad'][p]:
            continue
        if fr['inView'][p]:
            trackInView[p] = True; visible[p] += 1; n += 1
    return frame, lastFrameSeen, trackInView, visible, n


def _chain(st, g, voc, th=1.0):
    be = TR.OracleBackend(voc)
    mm = None
    if st['kind'] == 'fallback':
        match, claimed = st['match'].copy(), st['claimed'].copy()
        mm = T.motion_model_step(be, st, g, match, claimed, st['nmatches'])
    ref = TR.reference_keyframe_step(be, st, g)
    if not ref['gated']:
        return mm, ref, None, None
    NK = len(st['kf_kps'])
    l2l, dis = TR.concat_index_space([st], NK, st['mcapLast'], [ref['discarded']], [None if mm is None else mm['discarded']])
    lm = T.local_map_step(be, dict(st, lastToLocal=l2l[0]), g, ref['match'], dis[0], ref['Tcw7'], th)
    return mm, ref, lm, (l2l[0], dis[0])


@pytest.mark.parametrize('kind', ['normal', 'fallback', 'map9'])
def test_concatenated_index_space_equals_the_per_point_restatement(voc, kind):
    g = T.globals_()
    st = TR.ref_kf_stream(21, g, voc, kind=kind)
    mm, ref, lm, (l2l, dis) = _chain(st, g, voc)
    frame, seen, inview, visible, n = _restatement(st, g, mm, ref)
    # the same frame points, the same "seen" set, the same points in view and the same visible counts before the search
    held = {i: int(p) for i, p in enumerate(lm['match']) if p >= 0}
    assert {i: p for i, p in held.items() if i in frame} == frame
    assert lm['nToMatch'] == n
    assert np.array_equal(lm['visible'], visible)         # TrackLocalMap counts visible before its search only
    assert ref['gated'] and (ref['discarded'].any() or kind == 'map9')
    if kind == 'map9':
        assert ref['nmatchesMap'] < 10 <= ref['nmatches']    # the host's success test fails although the gate passed
    if kind == 'fallback':
        # the failed motion-model step discarded points the keyframe does not see; each has its own keypoint, which the local search
        # takes once the motion-model marks are dropped from the index space, and not with them
        assert mm['nmatchesMap'] < 10 and mm['discarded'].any()
        gone = {int(st['lastToLocal'][j]) for j in np.nonzero(mm['discarded'])[0]}
        assert gone and not gone & set(st['kfToLocal'].tolist()) and all(seen[p] == CUR and not inview[p] for p in gone)
        NK = len(st['kf_kps'])
        lm2 = T.local_map_step(TR.OracleBackend(voc), dict(st, lastToLocal=l2l), g, ref['match'], np.concatenate([dis[:NK], np.zeros_like(dis[NK:])]),
                               ref['Tcw7'], 1.0)
        took = set(lm2['match'][lm2['match'] >= 0].tolist()) - set(lm['match'][lm['match'] >= 0].tolist())
        assert gone & took


def test_gate_and_planted_cases(voc):
    g = T.globals_()
    be = TR.OracleBackend(voc)
    r14 = TR.reference_keyframe_step(be, TR.ref_kf_stream(22, g, voc, kind='n14'), g)
    r15 = TR.reference_keyframe_step(be, TR.ref_kf_stream(23, g, voc, kind='n15'), g)
    assert r14['nmatches'] == 14 and not r14['gated'] and 'pose7' not in r14
    assert r15['nmatches'] == 15 and r15['gated']
    st = TR.ref_kf_stream(24, g, voc)
    r = TR.reference_keyframe_step(be, st, g)
    # keyframe features without a point or with a bad one are never matched
    assert (st['kfPoint'][r['match'][r['match'] >= 0]] == 1).all()
    # the wrong matches (keypoints far from their point) are PoseOptimization's outliers: discarded, not held
    wrong = [i for i in range(len(st['kps'])) if st['kp_src'][i] < 0 and r['match'][i] < 0]
    assert r['discarded'].sum() >= 4 and r['nmatches'] - int(r['discarded'].sum()) == int((r['match'] >= 0).sum()) and wrong
    # the rotated matches fall into minority bins of the rotation histogram and are dropped by the search
    n_rot, _ = be.search_bow(st['kf_kps'], st['kf_desc'], st['kfPoint'], st['kf_fv'], st['kps'], st['desc'], st['fv'])
    n_nori, _ = be.O.search_by_bow(st['kf_kps'], st['kf_desc'], st['kfPoint'], st['kf_fv'], st['kps'], st['desc'], st['fv'], nnratio=0.7, check_ori=False)
    assert n_nori > n_rot
    # points without observations do not count towards nmatchesMap
    held = r['match'][r['match'] >= 0]
    assert r['nmatchesMap'] == int(st['kf_hasObs'][held].sum()) < len(held)
    # one level-2 node per group: with L = 6 and levelsup = 4 the FeatureVector has at most k^2 = 25 distinct nodes and more than one
    assert 1 < len(np.unique(st['fv'][0])) <= 25


def test_new_symbols_exported_and_no_silent_path():
    import torch
    import orb_slam3_modified_b200 as orb
    L = orb.lib()
    for n in ('orbm_track_reference_keyframe_batch', 'orbm_track_reference_keyframe_batch_device', 'orbm_track_reference_keyframe_batch_resident'):
        assert hasattr(L, n), n
        fn = getattr(L, n)
        assert fn(*[None] * len(fn.argtypes)) == orb.ORB_ERR_ARG
    if torch.cuda.is_available():
        pytest.skip('GPU present')
    with pytest.raises(orb.OrbError) as ei:
        orb.ORBmatcher(0.8, False, max_batch=4)
    assert ei.value.code == orb.ORB_ERR_CUDA
