"""Shared pieces of the undistortion tests: the calibrations, cv2.undistortPoints as the reference computes it, the CPU oracle's entry points
(orbo_undistort_points / _keypoints / orbo_image_bounds) and frames rendered through a lens distortion."""
import ctypes as C

import numpy as np

import oracle_lib as O

# (fx, fy, cx, cy), distortion coefficients, width, height
CALIBRATIONS = {
    'euroc': ((458.654, 457.296, 367.215, 248.375), (-0.28340811, 0.07395907, 0.00019359, 1.76187114e-05), 752, 480),   # EuRoC cam0
    'tum1': ((517.306408, 516.469215, 318.643040, 255.313989), (0.262383, -0.953104, -0.005358, 0.002628, 1.163314), 640, 480),
}


def cam9(K, D):
    """fx fy cx cy k1 k2 p1 p2 k3 as float32 (k3 = 0 for four coefficients)."""
    D = list(D) + [0.0] * (5 - len(D))
    return np.array(list(K) + D, np.float32)


def cv2_undistort(pts, K, D):
    """cv2.undistortPoints(pts, K, D, None, K) with K and D as CV_32F, as Frame::UndistortKeyPoints calls it."""
    import cv2
    pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 1, 2)
    Km = np.array([[K[0], 0, K[2]], [0, K[1], K[3]], [0, 0, 1]], np.float32)
    return cv2.undistortPoints(pts, Km, np.array(D, np.float32).reshape(-1, 1), None, Km).reshape(-1, 2)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def oracle_points(pts, K, D):
    pts = np.ascontiguousarray(pts, np.float32)
    out = np.zeros_like(pts)
    O.lib().orbo_undistort_points(_p(pts), len(pts), _p(np.asarray(K, np.float32)), _p(np.asarray(D, np.float32)), len(D), _p(out))
    return out


def oracle_keypoints(kps, cam):
    """Frame::UndistortKeyPoints on a KP_DTYPE array."""
    kps = np.ascontiguousarray(kps, O.KP_DTYPE)
    out = np.zeros_like(kps)
    O.lib().orbo_undistort_keypoints(_p(kps), len(kps), _p(np.asarray(cam, np.float32)), _p(out))
    return out


def oracle_bounds(cam, cols, rows):
    """Frame::ComputeImageBounds: mnMinX, mnMaxX, mnMinY, mnMaxY."""
    out = np.zeros(4, np.float32)
    O.lib().orbo_image_bounds(_p(np.asarray(cam, np.float32)), int(cols), int(rows), _p(out))
    return out


def random_calibration(rng):
    """A seeded pinhole calibration with strong barrel (k1 < 0) or pincushion (k1 > 0) distortion and non-zero p1 / p2."""
    W, H = [(640, 480), (752, 480), (1280, 720)][int(rng.integers(0, 3))]
    f = rng.uniform(0.7, 1.2) * W
    K = (f, f * rng.uniform(0.98, 1.02), W / 2 + rng.normal(0, 8), H / 2 + rng.normal(0, 8))
    k1 = rng.choice([-1.0, 1.0]) * rng.uniform(0.1, 0.5)
    D = (k1, rng.uniform(-0.2, 0.2), rng.uniform(-0.005, 0.005), rng.uniform(-0.005, 0.005), rng.uniform(-0.1, 0.1))
    return K, D, W, H


def random_keypoints(rng, n, W, H):
    kps = np.zeros(n, O.KP_DTYPE)
    kps['x'] = rng.uniform(0, W, n); kps['y'] = rng.uniform(0, H, n)
    kps['size'] = 31 * 1.2 ** rng.integers(0, 8, n); kps['angle'] = rng.uniform(0, 360, n); kps['response'] = rng.uniform(0, 100, n)
    kps['octave'] = rng.integers(0, 8, n); kps['class_id'] = rng.integers(-1, 5, n)
    return kps


PAD_X, PAD_Y = 256, 192


def ideal_to_synth(xy, K, W, H):
    """Pixel positions of the undistorted camera K as pixels of synth.frame(t, W, H): the synthetic frame is the pinhole
    (F_PIX, F_PIX, W / 2, H / 2) looking at the same plane."""
    from orb_slam3_modified_b200 import synth
    xy = np.asarray(xy, np.float64)
    return np.stack([synth.F_PIX * (xy[:, 0] - K[2]) / K[0] + W / 2, synth.F_PIX * (xy[:, 1] - K[3]) / K[1] + H / 2], 1)


def distorted_frame(t, W, H, K, D):
    """Frame t of the synthetic trajectory as a camera with calibration (K, D) sees it: cv2.remap of a wider synth.frame whose map sends
    every pixel of the W x H distorted image to cv2.undistortPoints of it.  The camera pose is synth.pose(t)."""
    import cv2
    from orb_slam3_modified_b200 import synth
    big = synth.frame(t, W + 2 * PAD_X, H + 2 * PAD_Y)
    ys, xs = np.mgrid[0:H, 0:W]
    und = cv2_undistort(np.stack([xs.ravel(), ys.ravel()], 1).astype(np.float32), K, D)
    s = ideal_to_synth(und, K, W, H) + [PAD_X, PAD_Y]
    mx = s[:, 0].reshape(H, W).astype(np.float32); my = s[:, 1].reshape(H, W).astype(np.float32)
    return cv2.remap(big, mx, my, cv2.INTER_LINEAR, borderMode=cv2.BORDER_REFLECT)
