"""CPU tests of the mono-inertial tracking call's reference (tests/track_inertial_lib.py): the PredictStateIMU restatement against float64
and the truth, the oracle chain on scenes that reach every rule of the glue, and no silent path without a device.  No GPU needed."""

import numpy as np
import pytest

import oracle_lib as O
import track_inertial_lib as TI
import track_lib as T


def test_prediction_restatement_agrees_with_float64_and_truth():
    rg = T.globals_(), TI.rig()
    g, rg = rg
    for seed in range(6):
        for mode in (1, 2):
            st = TI.stream(seed, g, rg, mode, M=10, noise=False)
            S, P = (st['kfState21'], st['preintKF']) if mode == 1 else (st['lastState21'], st['preintFrame'])
            pred, Tcw = TI.predict_state(O, rg['Tcb7'], S, P)
            R64, t64, v64 = TI.predict_state_f64(S, P, O)
            # the float read-back through mTcw equals the float64 body state to float rounding
            Rb, tb = pred[:9].reshape(3, 3).astype(np.float64), pred[9:12].astype(np.float64)
            assert np.abs(Rb - R64).max() < 2e-6 and np.abs(tb - t64).max() < 2e-5 * max(1, np.abs(t64).max()) and np.abs(pred[12:15] - v64).max() < 1e-5
            assert np.array_equal(pred[15:], np.asarray(S, np.float32)[15:])
            # noise-free IMU from the true source state: the prediction is the truth up to integration error
            tr = st['truth']
            assert np.abs(Rb - tr[:9].reshape(3, 3)).max() < 2e-3 and np.abs(tb - tr[9:12]).max() < 2e-3 and np.abs(pred[12:15] - tr[12:15]).max() < 5e-3
            # Tcw is the camera pose of that body pose: Tcw = Tcb Twb^-1
            Rcw, tcw, _ = T.pose_matrices(Tcw)
            Rcb, tcb = rg['extr'][:9].reshape(3, 3), rg['extr'][9:12]
            assert np.abs(Rcw - Rcb @ R64.T).max() < 2e-6 and np.abs(tcw - (Rcb @ (-R64.T @ t64) + tcb)).max() < 2e-5


def _run(st, g, rg, th):
    be = TI.OracleBackend()
    S, P = (st['kfState21'], st['preintKF']) if st['mode'] == 1 else (st['lastState21'], st['preintFrame'])
    pred, Tcw = TI.predict_state(O, rg['Tcb7'], S, P)
    return pred, Tcw, TI.local_map_step(be, st, g, rg, st['mode'], pred, Tcw, th)


def test_oracle_chain_reaches_every_rule():
    g, rg = T.globals_(), TI.rig()
    g.update(bFarPoints=1, thFarPoints=12.0)
    res = {}
    for name, mode, kind, th in (('kf', 1, 'normal', 6.0), ('lf', 2, 'normal', 2.0), ('lost', 2, 'normal', 15.0), ('empty', 1, 'empty', 6.0),
                                 ('nomatch', 2, 'nomatch', 2.0)):
        st = TI.stream(31 + len(res), g, rg, mode, kind=kind)
        if name == 'lf':                                  # the prior the reference carries: the oracle optimiser of the previous frame
            prev = TI.prior_from_oracle(st, rg, 77)
            assert prev['ret'] > 100 and np.abs(st['priorH'] - st['priorH'].T).max() <= 1e-9 * np.abs(st['priorH']).max()
        res[name] = (st,) + _run(st, g, rg, th)
    for name in ('kf', 'lf', 'lost'):
        st, pred, Tcw, r = res[name]
        assert r['nToMatch'] > 100 and r['nmatches'] > 50 and r['nInliers'] > 30 and 0 < r['nMatchesInliers'] <= r['nInliers']
        assert r['outlier'].sum() > 0                                 # the planted gross outliers are flagged
        assert (r['visible'] >= r['found']).all() and r['found'].max() >= 1
        # the optimised pose moved towards the truth, and its float state is the write-back of the double estimate
        assert np.abs(r['state21'][9:12] - st['truth'][9:12]).max() < np.abs(pred[9:12] - st['truth'][9:12]).max() + 1e-3
        assert np.abs(r['state21'][12:21].astype(np.float64) - r['prior21'][12:21]).max() < 1e-6
        H = r['priorH']
        assert np.array_equal(H, O.constraint_pose_imu_information(H.copy())) or np.abs(H - H.T).max() < 1e-6 * np.abs(H).max()
    # far points and th = 15: the lost stream searched a wider window
    assert res['lost'][3]['nmatches'] >= 1
    # an empty local map and a search that finds nothing still run the optimiser, with the inertial edges only (N = 0)
    for name in ('empty', 'nomatch'):
        st, pred, Tcw, r = res[name]
        assert r['nmatches'] == 0 and r['N'] == 0 and r['nInliers'] == 0 and not r['found'].any()
        assert not np.array_equal(r['state21'], pred)              # the inertial edges moved the state
        assert np.abs(r['priorH']).max() > 0
    assert res['nomatch'][3]['nToMatch'] > 0 and res['empty'][3]['nToMatch'] == 0


def test_new_symbols_exported_and_no_silent_path():
    import torch
    import orb_slam3_modified_b200 as orb
    L = orb.lib()
    for n, nargs in (('orbm_track_local_map_inertial_batch', 5), ('orbm_track_local_map_inertial_batch_device', 6),
                     ('orbm_track_local_map_inertial_batch_resident', 5)):
        assert hasattr(L, n), n
        assert getattr(L, n)(*[None] * nargs) == orb.ORB_ERR_ARG     # no handle: rejected before anything runs
    # without a device the handle these calls need cannot be made: creating it fails with ORB_ERR_CUDA, so nothing runs on the CPU
    if torch.cuda.is_available():
        pytest.skip('GPU present')
    with pytest.raises(orb.OrbError) as ei:
        orb.ORBmatcher(0.8, False, max_batch=4)
    assert ei.value.code == orb.ORB_ERR_CUDA


def test_cpp_batch_tracker_caller_compiles(tmp_path):
    """The C++ caller of BatchTracker::TrackLocalMapInertial builds with plain g++ against the C ABI (it runs in the GPU tests)."""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib = os.path.join(root, 'orb_slam3_modified_b200')
    exe = tmp_path / 'track_inertial_example'
    subprocess.check_call(['g++', '-std=c++14', '-O2', '-Wall', '-I', os.path.join(root, 'include'), os.path.join(root, 'tests', 'track_inertial_example.cpp'),
                           '-o', str(exe), '-L', lib, '-l:liborb_b200.so', '-Wl,-rpath,' + lib, '-lpthread'])
    assert exe.exists()
