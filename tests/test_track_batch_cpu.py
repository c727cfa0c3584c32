"""CPU tests of the batched tracking calls' reference: the float32 pose hand-off against float64, and the oracle chain of
tests/track_lib.py on planted scenes that reach every rule of Tracking's glue.  No GPU needed."""

import numpy as np
import pytest

import track_lib as T


def test_pose_handoff_agrees_with_float64_to_float_rounding():
    rng = np.random.default_rng(3)
    for _ in range(500):
        q = rng.normal(0, 1, 4)
        q /= np.linalg.norm(q) * rng.uniform(0.999, 1.001)    # the optimiser's quaternion is normalised up to rounding
        pose = np.concatenate([q, rng.normal(0, 3, 3)])
        Tf = T.set_pose(pose)
        qn = pose[:4] / np.linalg.norm(pose[:4])
        assert Tf.dtype == np.float32
        assert np.abs(Tf[:4].astype(np.float64) - qn).max() < 4e-7 and np.array_equal(Tf[4:], pose[4:].astype(np.float32))
        R, t, Ow = T.pose_matrices(Tf)
        R64 = T._R(Tf[:4].astype(np.float64))
        assert np.abs(R.astype(np.float64) - R64).max() < 1e-6
        Ow64 = -R64.T @ Tf[4:].astype(np.float64)
        assert np.abs(Ow.astype(np.float64) - Ow64).max() < 2e-6 * max(1.0, np.abs(Ow64).max())
        assert np.array_equal(t, Tf[4:])


def _chain(st, g, th, discarded_override=None):
    be = T.OracleBackend()
    match, claimed = st['match'].copy(), st['claimed'].copy()
    mm = T.motion_model_step(be, st, g, match, claimed, st['nmatches'])
    disc = mm['discarded'] if discarded_override is None else discarded_override
    lm = T.local_map_step(be, st, g, match, disc, mm['Tcw7'], th)
    return match, mm, lm


def test_oracle_chain_reaches_every_rule():
    g = T.globals_()
    st = T.stream(11, g)
    match_last, mm, lm = _chain(st, g, 1.0)
    l2l = st['lastToLocal']
    # outliers of the motion-model PoseOptimization were discarded, and one of their points has its own keypoint that the local search
    # takes when the discard marks are ignored, but not with them
    disc_local = {int(l2l[j]) for j in np.nonzero(mm['discarded'])[0] if l2l[j] >= 0}
    assert mm['nmatches'] < st['nmatches'] and disc_local
    _, _, lm_nomark = _chain(st, g, 1.0, discarded_override=np.zeros_like(mm['discarded']))
    assert disc_local & set(lm_nomark['match'][lm_nomark['match'] >= 0].tolist()) - set(lm['match'][lm['match'] >= 0].tolist())
    # a matched point that went bad and a last-frame point without a local index are dropped from the frame
    held = match_last[match_last >= 0]
    assert (l2l[held] < 0).any()
    assert any(l2l[j] >= 0 and st['bad'][l2l[j]] for j in held)
    # one point held at two keypoints: counted twice
    assert lm['visible'].max() >= 2 and lm['found'].max() >= 2
    assert lm['nToMatch'] > 0 and lm['nmatches'] > 0 and lm['nInliers'] > 10 and 0 < lm['nMatchesInliers'] <= lm['nInliers']
    assert np.array_equal(lm['visible'] >= lm['found'], np.ones_like(lm['found'], bool))
    # the optimised pose moved towards the truth and SetPose is its float form
    assert np.abs(lm['Tcw7'].astype(np.float64) - lm['pose7']).max() < 1e-6


def test_oracle_chain_degenerate_streams():
    g = T.globals_()
    empty = T.stream(12, g, kind='empty')
    _, mm, lm = _chain(empty, g, 1.0)
    assert lm['nToMatch'] == 0 and lm['nmatches'] == 0 and len(lm['visible']) == 0 and lm['nInliers'] == 0
    assert np.array_equal(lm['Tcw7'], mm['Tcw7']) and np.array_equal(mm['Tcw7'], empty['Tcw7'])     # fewer than 3 edges: no SetPose
    all_seen = T.stream(13, g, kind='all_seen', K_extra=20)
    _, mm, lm = _chain(all_seen, g, 1.0)
    assert lm['nToMatch'] == 0 and lm['nmatches'] == 0 and lm['nInliers'] > 0
    few = T.stream(14, g, kind='few')
    _, mm, lm = _chain(few, g, 1.0)
    assert np.array_equal(mm['Tcw7'], few['Tcw7']) and np.array_equal(mm['pose7'], few['Tcw7'].astype(np.float64)) and mm['nmatchesMap'] <= 2


def test_new_symbols_exported_and_no_silent_path():
    import torch
    import orb_slam3_modified_b200 as orb
    L = orb.lib()
    names = ('orbm_motion_model_pose_batch', 'orbm_motion_model_pose_batch_device', 'orbm_track_local_map_batch',
             'orbm_track_local_map_batch_device', 'orbm_track_local_map_batch_resident')
    for n in names:
        assert hasattr(L, n), n
        fn = getattr(L, n)
        assert fn(*[None] * len(fn.argtypes)) == orb.ORB_ERR_ARG       # no handle: rejected before anything runs
    if torch.cuda.is_available():
        pytest.skip('GPU present')
    with pytest.raises(orb.OrbError) as ei:
        orb.ORBmatcher(0.8, False, max_batch=4)
    assert ei.value.code == orb.ORB_ERR_CUDA
