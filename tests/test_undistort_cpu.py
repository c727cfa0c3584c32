"""CPU tests of Frame::UndistortKeyPoints / Frame::ComputeImageBounds: the oracle (orbo_undistort_points, orbo_undistort_keypoints,
orbo_image_bounds) and the host build of the kernel's per-point function (csrc/undistort.h) are pinned to cv2.undistortPoints bit for bit,
on the EuRoC cam0 and TUM1 calibrations, seeded strong calibrations, 4 and 5 coefficients, OpenCV's icdist < 0 reset, the principal point,
the image border and extracted keypoints.  The integer IEEE division of undistort.h equals the host's division."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import oracle_lib as O
import undistort_lib as U

cv2 = pytest.importorskip('cv2')

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def host(tmp_path_factory):
    """tests/undistort_host.cpp built like the other host checks: g++ -ffp-contract=off with FMA available."""
    so = str(tmp_path_factory.mktemp('undistort_host') / 'libundistort_host.so')
    subprocess.check_call(['g++', '-O2', '-std=c++17', '-fPIC', '-ffp-contract=off', '-mfma', '-shared', '-o', so,
                           os.path.join(ROOT, 'tests', 'undistort_host.cpp')])
    return C.CDLL(so)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def host_points(L, pts, cam9):
    pts = np.ascontiguousarray(pts, np.float32)
    out = np.zeros_like(pts)
    L.uh_undistort_points(_p(pts), len(pts), _p(np.asarray(cam9, np.float32)), _p(out))
    return out


def _grid_points(W, H, rng, n=20000):
    """Random points over the image, the four corners, the principal-point neighbourhood and the border."""
    border = np.concatenate([np.stack([np.arange(0, W + 1, 7), np.zeros_like(np.arange(0, W + 1, 7))], 1),
                             np.stack([np.arange(0, W + 1, 7), np.full_like(np.arange(0, W + 1, 7), H)], 1),
                             np.stack([np.zeros_like(np.arange(0, H + 1, 5)), np.arange(0, H + 1, 5)], 1),
                             np.stack([np.full_like(np.arange(0, H + 1, 5), W), np.arange(0, H + 1, 5)], 1)])
    return np.concatenate([rng.uniform([0, 0], [W, H], (n, 2)), [[0, 0], [W, 0], [0, H], [W, H]], border]).astype(np.float32)


def _check(host, pts, K, D, what):
    ref = U.cv2_undistort(pts, K, D)
    got = U.oracle_points(pts, K, D)
    assert ref.tobytes() == got.tobytes(), (what, 'oracle', int((ref != got).any(1).sum()))
    hc = host_points(host, pts, U.cam9(K, D))
    assert ref.tobytes() == hc.tobytes(), (what, 'undistort.h', int((ref != hc).any(1).sum()))


@pytest.mark.parametrize('name', sorted(U.CALIBRATIONS))
def test_shipped_calibrations_random_points(host, name):
    K, D, W, H = U.CALIBRATIONS[name]
    pts = _grid_points(W, H, np.random.default_rng(1))
    _check(host, pts, K, D, name)
    pp = np.array([[K[2], K[3]], [np.nextafter(np.float32(K[2]), np.float32(0)), K[3]], [K[2], np.nextafter(np.float32(K[3]), np.float32(1e9))]], np.float32)
    _check(host, pp, K, D, name + ' principal point')
    out = U.cv2_undistort(pp[:1], K, D)
    assert out.tobytes() == pp[:1].tobytes()            # the principal point does not move


@pytest.mark.parametrize('name', sorted(U.CALIBRATIONS))
def test_shipped_calibrations_extracted_keypoints(host, name):
    K, D, W, H = U.CALIBRATIONS[name]
    img = U.distorted_frame(0, W, H, K, D)
    _, kps, _ = O.OracleExtractor(1000, 1.2, 8, 20, 7)(img, (0, 1000))
    assert len(kps) > 800
    _check(host, np.stack([kps['x'], kps['y']], 1), K, D, name + ' keypoints')


@pytest.mark.parametrize('seed', range(12))
def test_seeded_strong_calibrations_4_and_5_coefficients(host, seed):
    rng = np.random.default_rng(100 + seed)
    K, D, W, H = U.random_calibration(rng)
    pts = _grid_points(W, H, rng, 4000)
    _check(host, pts, K, D, (seed, 5))
    _check(host, pts, K, D[:4], (seed, 4))
    # four coefficients are the same arithmetic as k3 = 0
    assert U.cv2_undistort(pts, K, D[:4]).tobytes() == U.cv2_undistort(pts, K, list(D[:4]) + [0.0]).tobytes()


def test_icdist_reset_returns_the_input():
    """k1 = -1.2, f = 500 on 640 x 480: the corners' iterates grow until a denominator turns negative, OpenCV resets them to the
    normalised input, and the result is the pixel itself (without the reset they would move outwards)."""
    K, D = (500.0, 500.0, 320.0, 240.0), (-1.2, 0.0, 0.0, 0.0)
    corners = np.array([[0, 0], [640, 0], [0, 480], [640, 480]], np.float32)
    ref = U.cv2_undistort(corners, K, D)
    assert ref.tobytes() == corners.tobytes()
    assert U.oracle_points(corners, K, D).tobytes() == ref.tobytes()


def test_icdist_reset_host_and_mixed_points(host):
    K, D = (500.0, 500.0, 320.0, 240.0), (-1.2, 0.0, 0.0, 0.0)
    pts = _grid_points(640, 480, np.random.default_rng(3), 3000)
    _check(host, pts, K, D, 'reset')


@pytest.mark.parametrize('k1', [0.0, -0.0])
def test_frame_wrapper_copies_when_k1_is_zero(host, k1):
    """The reference copies mvKeys when mDistCoef.at<float>(0) == 0 whatever k2, p1, p2 and k3 are; cv2 itself would move the points."""
    K, D = (458.654, 457.296, 367.215, 248.375), (k1, 0.5, 0.001, -0.002, 0.3)
    rng = np.random.default_rng(4)
    kps = U.random_keypoints(rng, 500, 752, 480)
    out = U.oracle_keypoints(kps, U.cam9(K, D))
    assert out.tobytes() == kps.tobytes()
    assert U.cv2_undistort(np.stack([kps['x'], kps['y']], 1), K, D).tobytes() != np.stack([kps['x'], kps['y']], 1).astype(np.float32).tobytes()
    b = U.oracle_bounds(U.cam9(K, D), 752, 480)
    assert b.tolist() == [0.0, 752.0, 0.0, 480.0]
    hb = np.zeros(4, np.float32)
    host.uh_image_bounds(_p(np.asarray(U.cam9(K, D), np.float32)), 752, 480, _p(hb))
    assert hb.tobytes() == b.tobytes()


def test_frame_wrapper_keeps_every_other_field():
    K, D, W, H = U.CALIBRATIONS['euroc']
    kps = U.random_keypoints(np.random.default_rng(5), 700, W, H)
    out = U.oracle_keypoints(kps, U.cam9(K, D))
    for f in ('size', 'angle', 'response', 'octave', 'class_id'):
        assert out[f].tobytes() == kps[f].tobytes(), f
    xy = np.ascontiguousarray(np.stack([out['x'], out['y']], 1))
    assert xy.tobytes() == U.cv2_undistort(np.stack([kps['x'], kps['y']], 1), K, D).tobytes()


@pytest.mark.parametrize('size', [(640, 480), (752, 480), (1280, 720)])
def test_image_bounds_are_cv2_corner_extremes(host, size):
    W, H = size
    rng = np.random.default_rng(W)
    cams = [U.CALIBRATIONS['euroc'][:2], U.CALIBRATIONS['tum1'][:2]] + [U.random_calibration(rng)[:2] for _ in range(6)]
    for K, D in cams:
        c = U.cv2_undistort(np.array([[0, 0], [W, 0], [0, H], [W, H]], np.float32), K, D)
        want = np.array([min(c[0, 0], c[2, 0]), max(c[1, 0], c[3, 0]), min(c[0, 1], c[1, 1]), max(c[2, 1], c[3, 1])], np.float32)
        got = U.oracle_bounds(U.cam9(K, D), W, H)
        assert got.tobytes() == want.tobytes(), (K, D, got, want)
        hb = np.zeros(4, np.float32)
        host.uh_image_bounds(_p(np.asarray(U.cam9(K, D), np.float32)), W, H, _p(hb))
        assert hb.tobytes() == want.tobytes()
    # EuRoC cam0's undistorted corners reach well outside the image
    b = U.oracle_bounds(U.cam9(*U.CALIBRATIONS['euroc'][:2]), 752, 480)
    assert b[0] < -100 and b[1] > 850


def test_integer_division_equals_ieee_division(host):
    """ddiv_rn (undistort.h) against the host's divsd: random operands over the whole exponent range, subnormals, signed zeros,
    infinities, results that overflow or underflow, and ties of the rounding."""
    rng = np.random.default_rng(6)
    n = 400000
    bits = rng.integers(0, 2 ** 63, (2, n), dtype=np.int64).astype(np.uint64) | (rng.integers(0, 2, (2, n)).astype(np.uint64) << np.uint64(63))
    a, b = bits.view(np.float64)
    near = rng.uniform(-4, 4, (2, n // 4)) * 2.0 ** rng.integers(-30, 30, (2, n // 4))     # the operands undistortion meets
    sub = (rng.integers(1, 2 ** 52, (2, n // 8), dtype=np.int64)).view(np.float64) * rng.choice([-1.0, 1.0], (2, n // 8))
    special = np.array([0.0, -0.0, np.inf, -np.inf, 1.0, -1.0, 3.0, 5e-324, 2.2250738585072014e-308, 1.7976931348623157e308, 0.5, 2.0 ** -1074, 1e300, 1e-300])
    sa, sb = np.meshgrid(special, special)
    a = np.concatenate([a, near[0], sub[0], sa.ravel(), [1.0, 1.0, 2.0 ** -1022]])
    b = np.concatenate([b, near[1], sub[1], sb.ravel(), [3.0, 1.0 + 2.0 ** -52, 3.0]])
    out = np.zeros_like(a)
    host.uh_ddiv_n(_p(a), _p(b), _p(out), len(a))
    with np.errstate(all='ignore'):
        want = a / b
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(out), nan)
    assert out[~nan].view(np.uint64).tobytes() == want[~nan].view(np.uint64).tobytes(), int((out[~nan] != want[~nan]).sum())
    assert (np.abs(want) < 2.2250738585072014e-308).sum() > 1000 and np.isinf(want).sum() > 1000
