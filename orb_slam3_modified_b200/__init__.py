"""H100-native ORB-SLAM3 hot path: Python mirror of the reference class surfaces over the C-ABI.

The compute lives in ``liborb_b200.so`` (hand-written sm_90a CUDA, ``csrc/``); this module only
marshals numpy / torch buffers to the ``extern "C"`` entry points declared in ``include/orb_b200.h``.
There is no CPU fallback: importing works anywhere, but creating any object without the built
library or without an sm_90 (H100) GPU raises.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get('ORB_B200_LIB', os.path.join(_HERE, 'liborb_b200.so'))   # override: kernel-variant experiments

ORB_OK, ORB_ERR_EMPTY, ORB_ERR_ARG, ORB_ERR_CAPACITY, ORB_ERR_CUDA, ORB_ERR_ASPECT = 0, -1, -2, -3, -4, -5

#: numpy view of OrbKeyPoint / cv::KeyPoint (28 bytes)
KP_DTYPE = np.dtype([('x', 'f4'), ('y', 'f4'), ('size', 'f4'), ('angle', 'f4'), ('response', 'f4'),
                     ('octave', 'i4'), ('class_id', 'i4')])
#: numpy view of OrbmNewPoint (44 bytes): one map point made by LocalMapping::CreateNewMapPoints
NEW_POINT_DTYPE = np.dtype([('kf2', 'i4'), ('idx1', 'i4'), ('idx2', 'i4'), ('x3D', 'f4', 3), ('normal', 'f4', 3), ('minDistance', 'f4'),
                            ('maxDistance', 'f4')])
assert NEW_POINT_DTYPE.itemsize == 44


class OrbmTriFrame(C.Structure):
    """A keyframe for the triangulation search (include/orb_b200.h)."""
    _fields_ = [('N', C.c_int), ('keypoints', C.c_void_p), ('descriptors', C.c_void_p), ('hasMapPoint', C.c_void_p), ('nEntries', C.c_int),
                ('fvNode', C.c_void_p), ('fvFeature', C.c_void_p)]


class OrbmNewPointsIn(C.Structure):
    """Input of orbm_create_new_map_points (include/orb_b200.h)."""
    _fields_ = [('KF1', C.POINTER(OrbmTriFrame)), ('nKF2', C.c_int), ('KF2', C.POINTER(OrbmTriFrame)), ('ep2', C.c_void_p), ('F12', C.c_void_p),
                ('scaleFactors', C.c_void_p), ('levelSigma2', C.c_void_p), ('nlevels', C.c_int), ('Tcw', C.c_void_p), ('Ow', C.c_void_p),
                ('cam', C.c_void_p), ('scaleFactor', C.c_float), ('bCoarse', C.c_int), ('bInertial', C.c_int), ('thFarPoints', C.c_float)]


class OrbmNewPointsItem(C.Structure):
    """One new keyframe of orbm_create_new_map_points_batch (include/orb_b200.h); ``in_`` is the header's ``in``."""
    _fields_ = [('in_', OrbmNewPointsIn), ('out', C.c_void_p), ('nNew', C.c_void_p), ('nmatches', C.c_void_p), ('ncreated', C.c_void_p)]


class OrbPinholeCamera(C.Structure):
    """Pinhole calibration with lens distortion (include/orb_b200.h): fx fy cx cy, then k1 k2 p1 p2 k3 (k3 = 0 for 4 coefficients)."""
    _fields_ = [(n, C.c_float) for n in ('fx', 'fy', 'cx', 'cy', 'k1', 'k2', 'p1', 'p2', 'k3')]


def pinhole_camera(K, D):
    """OrbPinholeCamera from (fx, fy, cx, cy) and 4 or 5 distortion coefficients (k1, k2, p1, p2[, k3])."""
    D = list(D)
    if len(D) not in (4, 5):
        raise ValueError('4 or 5 distortion coefficients expected (k1 k2 p1 p2 [k3])')
    return OrbPinholeCamera(*[float(v) for v in K], *[float(v) for v in D + [0.0] * (5 - len(D))])


def image_bounds(K, D, cols, rows, device=0):
    """``Frame::ComputeImageBounds``: (mnMinX, mnMinY, mnMaxX, mnMaxY) -- the order the matchers' ``bounds`` take -- of a cols x rows
    image from its four corners undistorted on the GPU.  With k1 == 0 they are (0, 0, cols, rows)."""
    cam = pinhole_camera(K, D)
    out = np.zeros(4, np.float32)
    rc = lib().orbx_image_bounds(C.byref(cam), int(cols), int(rows), _ptr(out), device)
    if rc != ORB_OK:
        raise OrbError(rc, 'orbx_image_bounds')
    return float(out[0]), float(out[2]), float(out[1]), float(out[3])


def undistort_last_launch_count():
    """Launches of this thread's last undistort_keypoints[_device] / image_bounds call."""
    return lib().orbx_undistort_last_launch_count()


_vp, _i, _f, _d, _sz, _out = C.c_void_p, C.c_int, C.c_float, C.c_double, C.c_size_t, C.POINTER(C.c_void_p)

#: (restype, argtypes) of every liborb_b200.so function the package, its tests and its tools call, as include/orb_b200.h declares it.
#: lib() applies it once when it loads the library; tests/test_abi_layout_cpu.py checks it against the header.
SIGNATURES = {
    'orb_last_error': (C.c_char_p, []),
    'orb_abi_version': (_i, []),
    'orb_compiled_sm': (_i, []),
    # ORBextractor
    'orbx_create': (_i, [_out, _i, _f, _i, _i, _i, _i, _i, _i, _i]),
    'orbx_destroy': (None, [_vp]),
    'orbx_get_levels': (_i, [_vp]),
    'orbx_get_tables': (_i, [_vp] * 6),
    'orbx_max_keypoints': (_i, [_vp]),
    'orbx_extract': (_i, [_vp, _vp, _i, _i, _sz, _i, _i, _vp, _vp, _i, _vp, _vp]),
    'orbx_extract_batch': (_i, [_vp, _vp, _i, _i, _i, _sz, _sz, _i, _i, _vp, _vp, _i, _vp, _vp]),
    'orbx_extract_batch_device': (_i, [_vp, _vp, _i, _i, _i, _sz, _sz, _i, _i, _vp, _vp, _i, _vp, _vp, _vp]),
    'orbx_resident_slabs': (_i, [_vp] * 5),
    'orbx_stereo_matches': (_i, [_vp, _vp, _i, _f, _f, _vp, _vp, _i]),
    'orbx_stereo_matches_device': (_i, [_vp, _vp, _i, _vp, _vp, _vp, _i, _vp, _vp, _vp, _i, _f, _f, _vp, _vp, _vp]),
    'orbx_copy_level_bordered': (_i, [_vp, _i, _i, _i, _vp]),
    'orbx_get_level_size': (_i, [_vp, _i, _vp, _vp]),
    'orbx_copy_level': (_i, [_vp, _i, _i, _i, _vp]),
    'orbx_copy_candidates': (_i, [_vp, _i, _i, _vp, _i]),
    'orbx_last_launch_count': (_i, [_vp]),
    'orbx_set_profiling': (_i, [_vp, _i]),
    'orbx_get_stage_ms': (_i, [_vp, _vp]),
    'orbx_undistort_keypoints_device': (_i, [_vp, _vp, _i, _vp, _vp, _i, _vp, _vp]),
    'orbx_undistort_keypoints': (_i, [_vp, _vp, _i, _vp, _i, _out]),
    'orbx_image_bounds': (_i, [_vp, _i, _i, _vp, _i]),
    'orbx_undistort_last_launch_count': (_i, []),
    # ORBmatcher
    'orbm_create': (_i, [_out, _i, _i, _i, _i]),
    'orbm_destroy': (None, [_vp]),
    'orbm_search_local_map': (_i, [_vp, _vp, _vp, _f, _f, _i, _f, _vp, _vp, _vp]),
    'orbm_search_last_frame': (_i, [_vp, _vp, _vp, _vp, _vp, _f, _i, _vp, _vp, _vp]),
    'orbm_frustum_project': (_i, [_vp] * 9),
    'orbm_search_last_frame_batch_device': (_i, [_vp, _vp, _f, _i, _vp, _vp, _vp, _vp]),
    'orbm_search_last_frame_batch': (_i, [_vp, _vp, _f, _i, _vp, _vp, _vp]),
    'orbm_search_last_frame_batch_resident': (_i, [_vp, _vp, _f, _i, _vp, _vp, _vp]),
    'orbm_motion_model_pose_batch_device': (_i, [_vp] * 12),
    'orbm_motion_model_pose_batch': (_i, [_vp] * 11),
    'orbm_track_local_map_batch_device': (_i, [_vp] * 4),
    'orbm_track_local_map_batch': (_i, [_vp] * 3),
    'orbm_track_local_map_batch_resident': (_i, [_vp] * 3),
    'orbm_track_local_map_inertial_batch_device': (_i, [_vp] * 6),
    'orbm_track_local_map_inertial_batch': (_i, [_vp] * 5),
    'orbm_track_local_map_inertial_batch_resident': (_i, [_vp] * 5),
    'orbm_track_reference_keyframe_batch_device': (_i, [_vp] * 4),
    'orbm_track_reference_keyframe_batch': (_i, [_vp] * 3),
    'orbm_track_reference_keyframe_batch_resident': (_i, [_vp] * 3),
    'orbm_search_for_initialization': (_i, [_vp, _vp, _vp, _vp, _i, _f, _i, _vp, _vp]),
    'orbm_search_by_bow': (_i, [_vp, _vp, _vp, _vp, _f, _i, _vp, _vp]),
    'orbm_search_by_bow_kf': (_i, [_vp, _vp, _vp, _vp, _vp, _f, _i, _vp, _vp]),
    'orbm_common_regions_bow_batch': (_i, [_vp, _i, _vp]),
    'orbm_fuse_search': (_i, [_vp, _vp, _vp, _f, _vp, _vp, _vp, _vp, _f, _vp, _vp]),
    'orbm_fuse_search_batch': (_i, [_vp, _i, _vp]),
    'orbm_fuse_search_sim3': (_i, [_vp, _vp, _f, _vp, _vp, _vp, _vp, _f, _vp, _vp]),
    'orbm_search_by_sim3': (_i, [_vp] * 5 + [_f, _vp, _f, _vp, _vp, _vp]),
    'orbm_search_for_triangulation': (_i, [_vp, _vp, _i, _vp, _vp, _vp, _i, _vp, _vp, _i, _i, _vp, _vp]),
    'orbm_create_new_map_points': (_i, [_vp] * 6),
    'orbm_create_new_map_points_batch': (_i, [_vp, _i, _vp]),
    'orbm_distinctive_descriptors': (_i, [_vp, _i, _vp, _vp, _vp]),
    'orbm_keyframe_culling_batch': (_i, [_vp, _i, _vp]),
    'orbm_update_connections_batch': (_i, [_vp, _i, _vp]),
    'orbm_update_local_map_batch_device': (_i, [_vp] * 4),
    'orbm_update_local_map_batch': (_i, [_vp] * 3),
    'orbm_bf_knn2': (_i, [_vp, _vp, _i, _vp, _i, _vp, _vp]),
    'orbm_descriptor_distance': (_i, [_vp, _vp, _vp, _i, _vp]),
    'orbm_last_launch_count': (_i, [_vp]),
    'orbm_last_cluster_size': (_i, [_vp]),
    # Optimizer
    'lba_create': (_i, [_out, _i, _i, _i, _i]),
    'lba_create_batch': (_i, [_out, _i, _i, _i, _i, _i]),
    'lba_destroy': (None, [_vp]),
    'lba_solve': (_i, [_vp] * 3),
    'lba_solve_batch': (_i, [_vp, _i, _vp, _vp]),
    'lba_upload_batch': (_i, [_vp, _i, _vp]),
    'lba_run_batch_device': (_i, [_vp, _vp]),
    'lba_download_batch': (_i, [_vp, _i, _vp]),
    'lba_last_cluster_size': (_i, [_vp]),
    'lba_set_cluster_size': (_i, [_vp, _i]),
    'lba_last_helpers': (_i, [_vp]),
    'lba_set_helpers': (_i, [_vp, _i]),
    'lba_get_phase_ns': (_i, [_vp, _i, _vp]),
    'lba_local_bundle_adjustment_batch': (_i, [_vp, _i, _vp]),
    'lba_local_last_launches': (_i, [_vp]),
    'pose_optimization_batch': (_i, [_i, _i] + [_vp] * 6 + [_d] + [_vp] * 3 + [_i]),
    'imu_preintegrate_batch': (_i, [_i, _vp, _i] + [_vp] * 6 + [_i]),
    'imu_information_batch': (_i, [_i] + [_vp] * 4 + [_i]),
    'imu_inertial_edges': (_i, [_i, _vp, _vp, _vp, _d, _vp, _vp, _vp, _vp, _i]),
    'imu_mono_edges': (_i, [_vp] * 7 + [_i]),
    'pose_inertial_optimization_last_kf_batch': (_i, [_i, _i] + [_vp] * 10 + [_i, _vp, _vp, _vp, _i]),
    'pose_inertial_optimization_last_frame_batch': (_i, [_i, _i] + [_vp] * 13 + [_i, _vp, _vp, _vp, _i]),
    'local_inertial_ba_batch': (_i, [_i, _vp, _vp, _vp, _i]),
    'local_inertial_ba_map_batch': (_i, [_i, _vp, _i]),
    'local_inertial_ba_map_last_launches': (_i, []),
    # ORBVocabulary
    'orbv_create': (_i, [_out, _vp, _i]),
    'orbv_destroy': (None, [_vp]),
    'orbv_transform_batch': (_i, [_vp, _i, _vp, _vp, _i, _i] + [_vp] * 6),
    'orbv_transform_batch_device': (_i, [_vp, _i, _vp, _vp, _i, _i] + [_vp] * 10),
    # KeyFrameDatabase
    'orbv_db_create': (_i, [_out, _i, _i, _i, _i, _i]),
    'orbv_db_destroy': (None, [_vp]),
    'orbv_db_add_batch': (_i, [_vp, _i] + [_vp] * 5),
    'orbv_db_erase_batch': (_i, [_vp, _i, _vp, _vp]),
    'orbv_db_clear': (_i, [_vp, _i]),
    'orbv_db_size': (_i, [_vp, _i]),
    'orbv_db_query_batch': (_i, [_vp, _i, _vp]),
    'orbv_db_last_launch_count': (_i, [_vp]),
}

_lib = None


class OrbError(RuntimeError):
    def __init__(self, code, where):
        self.code = code
        msg = lib().orb_last_error().decode() if _lib is not None else ''
        super().__init__('%s failed with status %d: %s' % (where, code, msg))


def lib():
    """Load liborb_b200.so (built by ``__graft_entry__.build()``); raise if it is missing."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError('liborb_b200.so is not built (run `python -c "import __graft_entry__ as g; g.build()"`); '
                               'this package has no fallback path')
        L = C.CDLL(LIB_PATH)
        for name, (restype, argtypes) in SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype, fn.argtypes = restype, argtypes
        _lib = L
    return _lib


def _ptr(a):
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return a.ctypes.data_as(C.c_void_p)
    return C.c_void_p(a.data_ptr())  # torch tensor


class ORBextractor:
    """Mirror of ``ORB_SLAM3::ORBextractor`` (reference include/ORBextractor.h:43-109).

    ``ORBextractor(nfeatures, scaleFactor, nlevels, iniThFAST, minThFAST)``; calling the object is
    ``operator()``: ``mono_index, keypoints, descriptors = ex(image, vLappingArea)``.
    """

    def __init__(self, nfeatures=1000, scaleFactor=1.2, nlevels=8, iniThFAST=20, minThFAST=7,
                 max_width=640, max_height=480, max_batch=1, device=0):
        L = lib()
        self._h = C.c_void_p()
        self.nlevels = nlevels
        self.max_batch = max_batch
        rc = L.orbx_create(C.byref(self._h), nfeatures, scaleFactor, nlevels, iniThFAST, minThFAST,
                           max_width, max_height, max_batch, device)
        if rc != ORB_OK:
            self._h = None
            raise OrbError(rc, 'orbx_create')
        self.max_keypoints = L.orbx_max_keypoints(self._h)

    def close(self):
        if getattr(self, '_h', None):
            lib().orbx_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:      # interpreter shutdown: module globals may already be gone
            pass

    # --- getters (include/ORBextractor.h:60-82) ---
    def GetLevels(self):
        return lib().orbx_get_levels(self._h)

    def _tables(self):
        n = self.nlevels
        s, i, g, ig = (np.zeros(n, np.float32) for _ in range(4))
        f = np.zeros(n, np.int32)
        lib().orbx_get_tables(self._h, _ptr(s), _ptr(i), _ptr(g), _ptr(ig), _ptr(f))
        return s, i, g, ig, f

    def GetScaleFactors(self):
        return self._tables()[0]

    def GetScaleFactor(self):
        return float(self._tables()[0][1]) if self.nlevels > 1 else 1.0

    def GetInverseScaleFactors(self):
        return self._tables()[1]

    def GetScaleSigmaSquares(self):
        return self._tables()[2]

    def GetInverseScaleSigmaSquares(self):
        return self._tables()[3]

    def features_per_level(self):
        return self._tables()[4]

    # --- operator() ---
    def __call__(self, image, vLappingArea=(0, 0)):
        """Returns (monoIndex, keypoints[K] as KP_DTYPE, descriptors[K,32] u8); monoIndex == -1 for an empty image."""
        if image is None or image.size == 0:
            return -1, np.zeros(0, KP_DTYPE), np.zeros((0, 32), np.uint8)
        assert image.dtype == np.uint8 and image.ndim == 2, 'CV_8UC1 expected (reference src/ORBextractor.cc:1094)'
        if image.strides[1] != 1:
            image = np.ascontiguousarray(image)
        cap = self.max_keypoints
        kps = np.zeros(cap, KP_DTYPE)
        desc = np.zeros((cap, 32), np.uint8)
        n, mono = C.c_int(0), C.c_int(0)
        rc = lib().orbx_extract(self._h, _ptr(image), image.shape[0], image.shape[1], image.strides[0],
                                int(vLappingArea[0]), int(vLappingArea[1]), _ptr(kps), _ptr(desc), cap,
                                C.byref(n), C.byref(mono))
        if rc == ORB_ERR_EMPTY:
            return -1, kps[:0], desc[:0]
        if rc != ORB_OK:
            raise OrbError(rc, 'orbx_extract')
        return mono.value, kps[:n.value].copy(), desc[:n.value].copy()

    def extract_batch(self, images, vLappingArea=(0, 0)):
        """images: [B, rows, cols] u8 host array.  Returns lists (mono, kps, desc) per frame."""
        images = np.ascontiguousarray(images, np.uint8)
        B, rows, cols = images.shape
        cap = self.max_keypoints
        kps = np.zeros((B, cap), KP_DTYPE)
        desc = np.zeros((B, cap, 32), np.uint8)
        n = np.zeros(B, np.int32)
        mono = np.zeros(B, np.int32)
        rc = lib().orbx_extract_batch(self._h, _ptr(images), B, rows, cols, images.strides[1], images.strides[0],
                                      int(vLappingArea[0]), int(vLappingArea[1]), _ptr(kps), _ptr(desc), cap,
                                      _ptr(n), _ptr(mono))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbx_extract_batch')
        return ([int(m) for m in mono], [kps[b, :n[b]].copy() for b in range(B)], [desc[b, :n[b]].copy() for b in range(B)])

    def extract_batch_slabs(self, images, kps, desc, n, mono, vLappingArea=(0, 0)):
        """Batched operator() into caller-owned fixed-capacity slabs (numpy, ideally pinned): kps [B, cap] KP_DTYPE,
        desc [B, cap, 32] u8, n / mono [B] i32 with cap == max_keypoints.  No per-frame copies."""
        B, rows, cols = images.shape
        assert kps.shape[1] == self.max_keypoints and images.strides[2] == 1
        rc = lib().orbx_extract_batch(self._h, _ptr(images), B, rows, cols, images.strides[1], images.strides[0],
                                      int(vLappingArea[0]), int(vLappingArea[1]), _ptr(kps), _ptr(desc), self.max_keypoints,
                                      _ptr(n), _ptr(mono))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbx_extract_batch')

    def resident_slabs(self):
        """Device addresses (ints) of the slabs the last host-buffer call left in the handle: (kps, desc, n, cap)."""
        k, d, n, cap = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_int()
        rc = lib().orbx_resident_slabs(self._h, C.byref(k), C.byref(d), C.byref(n), C.byref(cap))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbx_resident_slabs')
        return k.value, d.value, n.value, cap.value

    def extract_batch_device(self, d_images, d_kps, d_desc, d_n, d_mono, vLappingArea=(0, 0), stream=0):
        """All-device variant (torch CUDA tensors): d_images [B, rows, cols] u8; slabs d_kps [B, cap, 7] (28-byte rows),
        d_desc [B, cap, 32] u8, d_n / d_mono [B] i32.  Enqueues on ``stream`` and returns immediately."""
        B, rows, cols = d_images.shape
        cap = d_desc.shape[1]
        rc = lib().orbx_extract_batch_device(self._h, _ptr(d_images), B, rows, cols, d_images.stride(1), d_images.stride(0),
                                             int(vLappingArea[0]), int(vLappingArea[1]), _ptr(d_kps), _ptr(d_desc), cap,
                                             _ptr(d_n), _ptr(d_mono), C.c_void_p(stream))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbx_extract_batch_device')

    # --- inspection taps (mvImagePyramid is public in the reference, include/ORBextractor.h:84) ---
    def level(self, level, frame=0, blurred=False):
        w, h = C.c_int(), C.c_int()
        rc = lib().orbx_get_level_size(self._h, level, C.byref(w), C.byref(h))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbx_get_level_size')
        out = np.zeros((h.value, w.value), np.uint8)
        rc = lib().orbx_copy_level(self._h, frame, level, int(blurred), _ptr(out))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbx_copy_level')
        return out

    def level_bordered(self, level, frame=0, border=19):
        """mvImagePyramid[level] with the reflected frame ComputePyramid keeps around it (src/ORBextractor.cc:1185-1191)."""
        w, h = C.c_int(), C.c_int()
        lib().orbx_get_level_size(self._h, level, C.byref(w), C.byref(h))
        out = np.zeros((h.value + 2 * border, w.value + 2 * border), np.uint8)
        rc = lib().orbx_copy_level_bordered(self._h, frame, level, border, _ptr(out))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbx_copy_level_bordered')
        return out

    def ComputeStereoMatches(self, right, mb, mbf, batch=1):
        """``Frame::ComputeStereoMatches`` (src/Frame.cc:811-982) for the pairs both extractors processed in their last host-buffer call
        (self = left).  Returns (mvuRight, mvDepth) as [batch, cap] float32, -1 = no match."""
        cap = self.max_keypoints
        ur = np.zeros((batch, cap), np.float32); dep = np.zeros((batch, cap), np.float32)
        rc = lib().orbx_stereo_matches(self._h, right._h, batch, mb, mbf, _ptr(ur), _ptr(dep), cap)
        if rc != ORB_OK:
            raise OrbError(rc, 'orbx_stereo_matches')
        return ur, dep

    def ComputeStereoMatchesDevice(self, right, d_kpsL, d_descL, d_nL, d_kpsR, d_descR, d_nR, mb, mbf, d_uRight, d_depth, stream=0):
        """All-device ComputeStereoMatches (torch CUDA tensors) for the pairs both extractors processed in their last call (self = left):
        the slabs as extract_batch_device wrote them (d_kps* [B, cap, 7], d_desc* [B, cap, 32] u8, d_n* [B] i32); d_uRight / d_depth
        [B, capL] float32 receive mvuRight / mvDepth (-1 = no match).  Enqueues on ``stream`` and returns immediately."""
        B, capL = d_descL.shape[:2]
        capR = d_descR.shape[1]
        rc = lib().orbx_stereo_matches_device(self._h, right._h, B, _ptr(d_kpsL), _ptr(d_descL), _ptr(d_nL), capL, _ptr(d_kpsR), _ptr(d_descR),
                                              _ptr(d_nR), capR, mb, mbf, _ptr(d_uRight), _ptr(d_depth), C.c_void_p(stream))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbx_stereo_matches_device')

    def candidates(self, level, frame=0, cap=400000):
        out = np.zeros((cap, 3), np.int32)
        n = lib().orbx_copy_candidates(self._h, frame, level, _ptr(out), cap)
        if n < 0:
            raise OrbError(n, 'orbx_copy_candidates')
        return out[:n].copy()

    def last_launch_count(self):
        return lib().orbx_last_launch_count(self._h)

    # --- Frame::UndistortKeyPoints (src/Frame.cc:747) ---
    def undistort_keypoints_device(self, K, D, d_kps, d_n, d_kpsUn, stream=0):
        """mvKeysUn for the slabs extract_batch_device wrote (torch CUDA tensors): d_kps / d_kpsUn [B, cap, 7] (28-byte rows, not
        overlapping), d_n [B] i32; K = (fx, fy, cx, cy), D = 4 or 5 coefficients.  Rows past n[f] and overflowing frames are not touched;
        k1 == 0 copies.  Enqueues one launch on ``stream`` and returns immediately."""
        cam = pinhole_camera(K, D)
        B, cap = d_kps.shape[:2]
        rc = lib().orbx_undistort_keypoints_device(self._h, C.byref(cam), B, _ptr(d_kps), _ptr(d_n), cap, _ptr(d_kpsUn), C.c_void_p(stream))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbx_undistort_keypoints_device')

    def undistort_keypoints(self, K, D, batch=1, host=True):
        """mvKeysUn for the frames of the last extract / extract_batch call, into a slab the handle owns.  Returns (device address of
        that [max_batch, max_keypoints] slab -- the ``kps`` of the matchers' resident forms --, and with ``host`` its [batch, cap]
        KP_DTYPE rows; rows at or past n[f] are unspecified)."""
        cam = pinhole_camera(K, D)
        cap = self.max_keypoints
        out = np.zeros((batch, cap), KP_DTYPE) if host else None
        d = C.c_void_p()
        rc = lib().orbx_undistort_keypoints(self._h, C.byref(cam), batch, _ptr(out), cap, C.byref(d))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbx_undistort_keypoints')
        return d.value, out

    STAGES = ('pyramid', 'blur', 'fast_cells', 'quadtree_orient', 'assemble', 'brief')

    def set_profiling(self, on):
        lib().orbx_set_profiling(self._h, int(on))

    def stage_ms(self):
        ms = np.zeros(6, np.float32)
        rc = lib().orbx_get_stage_ms(self._h, _ptr(ms))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbx_get_stage_ms')
        return dict(zip(self.STAGES, (float(m) for m in ms)))


# =============================================================================================
# ORBmatcher (reference include/ORBmatcher.h:36-103)
# =============================================================================================
class _OrbmFrame(C.Structure):
    _fields_ = [('K', C.c_int), ('keypoints', C.c_void_p), ('descriptors', C.c_void_p), ('minX', C.c_float), ('minY', C.c_float),
                ('maxX', C.c_float), ('maxY', C.c_float), ('scaleFactors', C.c_void_p), ('nlevels', C.c_int)]


class _OrbmBowFrame(C.Structure):
    _fields_ = [('N', C.c_int), ('keypoints', C.c_void_p), ('descriptors', C.c_void_p), ('nEntries', C.c_int), ('fvNode', C.c_void_p),
                ('fvFeature', C.c_void_p)]


class _OrbmLocalPoints(C.Structure):
    _fields_ = [('M', C.c_int)] + [(n, C.c_void_p) for n in ('inView', 'bad', 'depth', 'projX', 'projY', 'level', 'viewCos', 'hasObs', 'descriptors')]


class _OrbmFrustumIn(C.Structure):
    _fields_ = ([('M', C.c_int)] + [(n, C.c_void_p) for n in ('worldPos', 'normal', 'minDistInv', 'maxDistInv', 'maxDistance')] +
                [('Rcw', C.c_float * 9), ('tcw', C.c_float * 3), ('Ow', C.c_float * 3), ('cam', C.c_float * 4),
                 ('minX', C.c_float), ('minY', C.c_float), ('maxX', C.c_float), ('maxY', C.c_float), ('mbf', C.c_float),
                 ('logScaleFactor', C.c_float), ('nScaleLevels', C.c_int), ('viewingCosLimit', C.c_float)])


class _OrbmLastFrame(C.Structure):
    _fields_ = [('M', C.c_int)] + [(n, C.c_void_p) for n in ('valid', 'xyz', 'octave', 'angle', 'hasObs', 'descriptors')]


class _OrbmBatchDevice(C.Structure):
    _fields_ = [('batch', C.c_int), ('kcap', C.c_int), ('mcap', C.c_int), ('nlevels', C.c_int),
                ('kps', C.c_void_p), ('desc', C.c_void_p), ('nK', C.c_void_p),
                ('minX', C.c_float), ('minY', C.c_float), ('maxX', C.c_float), ('maxY', C.c_float),
                ('scaleFactors', C.c_void_p), ('nM', C.c_void_p),
                ('valid', C.c_void_p), ('xyz', C.c_void_p), ('octave', C.c_void_p), ('angle', C.c_void_p), ('hasObs', C.c_void_p),
                ('mpDesc', C.c_void_p), ('Tcw7', C.c_void_p), ('cam', C.c_float * 4), ('resetState', C.c_int)]


class _OrbmLocalMapBatch(C.Structure):
    _fields_ = ([(n, C.c_int) for n in ('batch', 'kcap', 'mcap', 'mcapLast', 'nlevels')] + [(n, C.c_void_p) for n in ('kps', 'desc', 'nK')] +
                [(n, C.c_float) for n in ('minX', 'minY', 'maxX', 'maxY')] + [('scaleFactors', C.c_void_p), ('invLevelSigma2', C.c_void_p),
                 ('cam', C.c_float * 4), ('mbf', C.c_float), ('logScaleFactor', C.c_float)] +
                [(n, C.c_void_p) for n in ('Tcw7', 'lastToLocal', 'discarded', 'nM', 'worldPos', 'normal', 'minDistInv', 'maxDistInv', 'maxDistance',
                                           'mpDesc', 'hasObs', 'bad', 'th')] +
                [('nnratio', C.c_float), ('bFarPoints', C.c_int), ('thFarPoints', C.c_float), ('viewingCosLimit', C.c_float), ('active', C.c_void_p)])


_LOCAL_MAP_OUT = ('match', 'claimed', 'outlier', 'visible', 'found', 'nToMatch', 'nmatches', 'nInliers', 'nMatchesInliers', 'pose7', 'Tcw7')


class _OrbmLocalMapResult(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in _LOCAL_MAP_OUT]


class _OrbmImuTrackBatch(C.Structure):
    _fields_ = [('mode', C.c_void_p), ('Tcb7', C.c_float * 7)] + [(n, C.c_void_p) for n in ('extrinsics24', 'preintKF', 'preintFrame', 'kfState21',
                                                                                            'lastState21', 'prior21', 'priorH')]


_IMU_TRACK_OUT = ('predState21', 'predTcw7', 'state21', 'prior21', 'priorH')


class _OrbmImuTrackResult(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in _IMU_TRACK_OUT]


_REF_KF_FRAME = ('kps', 'desc', 'nK', 'fvNode', 'fvFeature', 'nEntries')
_REF_KF_IN = _REF_KF_FRAME + ('Tcw7', 'kfN', 'kfKps', 'kfDesc', 'kfFvNode', 'kfFvFeature', 'kfNEntries', 'kfPoint', 'xyz', 'hasObs')


class _OrbmRefKeyFrameBatch(C.Structure):
    _fields_ = ([(n, C.c_int) for n in ('batch', 'kcap', 'mcap', 'nlevels')] + [(n, C.c_void_p) for n in _REF_KF_IN] +
                [('cam', C.c_float * 4), ('invLevelSigma2', C.c_void_p), ('active', C.c_void_p)])


_REF_KF_OUT = ('nmatches', 'match', 'pose7', 'Tcw7', 'discarded', 'nmatchesMap')


class _OrbmRefKeyFrameResult(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in _REF_KF_OUT]


class _OrbmFusePoints(C.Structure):
    _fields_ = [('M', C.c_int)] + [(n, C.c_void_p) for n in ('state', 'worldPos', 'normal', 'minDistance', 'maxDistance', 'descriptors')]


class _OrbmFuseItem(C.Structure):
    _fields_ = [('KF', _OrbmFrame), ('invLevelSigma2', C.c_void_p), ('logScaleFactor', C.c_float), ('Tcw7', C.c_float * 7), ('Ow', C.c_float * 3),
                ('cam', C.c_float * 4), ('th', C.c_float), ('pts', _OrbmFusePoints), ('bestIdx', C.c_void_p), ('bestDist', C.c_void_p)]


#: OrbmCommonRegionsQuery's candidate statuses (ORBM_CR_*) and the length of vpCovKFi's rows (include/orb_b200.h)
CR_SKIPPED, CR_ABORTED_NEAR, CR_RAN = range(3)
CR_MAX_COV = 11


class OrbmCommonRegionsKF(C.Structure):
    """One keyframe of an OrbmCommonRegionsQuery's table (include/orb_b200.h)."""
    _fields_ = [('frame', _OrbmBowFrame), ('point', C.c_void_p), ('bad', C.c_int), ('connected', C.c_int)]


class OrbmCommonRegionsQuery(C.Structure):
    """One place-recognition query of orbm_common_regions_bow_batch (include/orb_b200.h)."""
    _fields_ = [('nKF', C.c_int), ('kf', C.POINTER(OrbmCommonRegionsKF)), ('nPoints', C.c_int), ('pointBad', C.c_void_p), ('nCand', C.c_int)] + \
               [(n, C.c_void_p) for n in ('cand', 'covStart', 'cov', 'status', 'covList', 'nmatches', 'numBoWMatches', 'matchedCov', 'matchedPoint')]


def common_regions_struct(q):
    """OrbmCommonRegionsQuery over query dict `q` with fresh outputs: (struct, out dict, objects to keep alive).  `q`: kfs = [dict(kps,
    desc, fv=(nodes, features), point, bad, connected)] (entry 0 the current keyframe), pointBad [nPoints], cand [nCand] (-1 = NULL),
    cov = one list of table indices per candidate (GetBestCovisibilityKeyFrames(10))."""
    keep = []
    table = (OrbmCommonRegionsKF * max(len(q['kfs']), 1))()
    for e, kf in enumerate(q['kfs']):
        a = [_c(kf['kps'], KP_DTYPE), _c(kf['desc'], np.uint8).reshape(-1, 32), _c(kf['fv'][0], np.int32), _c(kf['fv'][1], np.int32),
             _c(kf['point'], np.int32)]
        keep.append(a)
        table[e] = OrbmCommonRegionsKF(_OrbmBowFrame(len(a[0]), a[0].ctypes.data, a[1].ctypes.data, len(a[2]), a[2].ctypes.data, a[3].ctypes.data),
                                       a[4].ctypes.data, int(kf['bad']), int(kf['connected']))
    pbad, cand = _c(q['pointBad'], np.uint8), _c(q['cand'], np.int32)
    cov_start = np.zeros(len(cand) + 1, np.int32)
    cov_start[1:] = np.cumsum([len(c) for c in q['cov']])
    cov = np.array([e for c in q['cov'] for e in c], np.int32)
    nC, N0 = len(cand), len(q['kfs'][0]['kps']) if q['kfs'] else 0
    out = dict(status=np.zeros(nC, np.uint8), covList=np.zeros((nC, CR_MAX_COV), np.int32), nmatches=np.zeros((nC, CR_MAX_COV), np.int32),
               numBoWMatches=np.zeros(nC, np.int32), matchedCov=np.zeros((nC, N0), np.int32), matchedPoint=np.zeros((nC, N0), np.int32))
    keep += [table, pbad, cand, cov_start, cov]
    s = OrbmCommonRegionsQuery(len(q['kfs']), C.cast(table, C.POINTER(OrbmCommonRegionsKF)), len(pbad), _ptr(pbad), nC, _ptr(cand), _ptr(cov_start),
                               _ptr(cov), *[_ptr(out[n]) for n in ('status', 'covList', 'nmatches', 'numBoWMatches', 'matchedCov', 'matchedPoint')])
    return s, out, keep


#: OrbmCullingMap's statuses (ORBM_KFC_*, include/orb_b200.h), by code
KFC_STATUS = ('not visited', 'skipped', 'kept', 'kept: few keyframes', 'kept: recent', 'kept: no link', 'kept: imu', 'culled', 'culled: time',
              'culled: still', 'not erase')
KFC_NOT_VISITED, KFC_SKIPPED, KFC_KEPT, KFC_KEPT_FEW_KFS, KFC_KEPT_RECENT, KFC_KEPT_NO_LINK, KFC_KEPT_IMU, KFC_CULLED, KFC_CULLED_TIME, \
    KFC_CULLED_STILL, KFC_NOT_ERASE = range(11)
KF_BAD, KF_INIT, KF_NOT_ERASE = 1, 2, 4
#: the arrays of one map of ORBmatcher.keyframe_culling_batch, with their dtypes (OrbmCullingMap)
CULLING_ARRAYS = (('mnId', np.uint64), ('kfFlags', np.uint8), ('prevKF', np.int32), ('nextKF', np.int32), ('timeStamp', np.float64),
                  ('imuPosition', np.float32), ('local', np.int32), ('slotStart', np.int32), ('slotPoint', np.int32), ('slotOctave', np.int32),
                  ('pointBad', np.uint8), ('obsStart', np.int32), ('obsKF', np.int32), ('obsOctave', np.int32))
CULLING_SCALARS = ('inertial', 'imuInitialized', 'inertialBA2', 'abortBA', 'keyFramesInMap', 'currentId', 'lastId')


class OrbmCullingMap(C.Structure):
    """One map of orbm_keyframe_culling_batch (include/orb_b200.h)."""
    _fields_ = [('nKF', C.c_int)] + [(n, C.c_void_p) for n in ('mnId', 'kfFlags', 'prevKF', 'nextKF', 'timeStamp', 'imuPosition')] + \
               [('nLocal', C.c_int)] + [(n, C.c_void_p) for n in ('local', 'slotStart', 'slotPoint', 'slotOctave')] + \
               [('nPoints', C.c_int)] + [(n, C.c_void_p) for n in ('pointBad', 'obsStart', 'obsKF', 'obsOctave')] + \
               [(n, C.c_int) for n in ('inertial', 'imuInitialized', 'inertialBA2', 'abortBA', 'keyFramesInMap')] + \
               [('currentId', C.c_uint64), ('lastId', C.c_uint64)] + [(n, C.c_void_p) for n in ('status', 'nMPs', 'nRedundant', 'visited')]


def culling_struct(m):
    """OrbmCullingMap over map dict `m` (keys CULLING_ARRAYS + CULLING_SCALARS) with fresh outputs: (struct, out dict, arrays to keep alive).
    The inertial arrays may be missing when m['inertial'] is false."""
    a = {n: (_c(m[n], dt) if m.get(n) is not None else None) for n, dt in CULLING_ARRAYS}
    nL = len(a['local'])
    out = dict(status=np.zeros(nL, np.uint8), nMPs=np.zeros(nL, np.int32), nRedundant=np.zeros(nL, np.int32), visited=np.zeros(1, np.int32))
    s = OrbmCullingMap(len(a['kfFlags']), *[_ptr(a[n]) for n in ('mnId', 'kfFlags', 'prevKF', 'nextKF', 'timeStamp', 'imuPosition')],
                       nL, *[_ptr(a[n]) for n in ('local', 'slotStart', 'slotPoint', 'slotOctave')],
                       len(a['pointBad']), *[_ptr(a[n]) for n in ('pointBad', 'obsStart', 'obsKF', 'obsOctave')],
                       *[int(m[n]) for n in ('inertial', 'imuInitialized', 'inertialBA2', 'abortBA', 'keyFramesInMap')], int(m['currentId']),
                       int(m['lastId']), *[_ptr(out[n]) for n in ('status', 'nMPs', 'nRedundant', 'visited')])
    return s, out, a


#: OrbmConnectionsItem's modes and slot statuses (ORBM_UC_*), and the keyframe flag of another map (include/orb_b200.h)
UC_PROCESS_NEW_KEYFRAME, UC_SEARCH_IN_NEIGHBORS = 0, 1
UC_SLOT_NONE, UC_SLOT_ADDED, UC_SLOT_IN_KEYFRAME, UC_SLOT_UPDATED = range(4)
KF_OTHER_MAP = 8
#: the arrays of one item of ORBmatcher.update_connections_batch, with their dtypes (OrbmConnectionsItem)
CONNECTIONS_ARRAYS = (('order', np.uint64), ('mnId', np.uint64), ('kfFlags', np.uint8), ('cameraCenter', np.float32), ('connStart', np.int32),
                      ('connKF', np.int32), ('connWeight', np.int32), ('scaleFactors', np.float32), ('slotPoint', np.int32), ('slotOctave', np.int32),
                      ('slotDesc', np.uint8), ('pointBad', np.uint8), ('pointPos', np.float32), ('pointRefKF', np.int32), ('obsStart', np.int32),
                      ('obsKF', np.int32), ('obsIdx', np.int32), ('obsOctave', np.int32), ('obsDesc', np.uint8))
CONNECTIONS_SCALARS = ('mode', 'firstConnection')
#: its outputs, with their dtypes
CONNECTIONS_OUTPUTS = (('slotStatus', np.uint8), ('pointUpdated', np.uint8), ('normal', np.float32), ('minDistance', np.float32),
                       ('maxDistance', np.float32), ('descKF', np.int32), ('descIdx', np.int32), ('counter', np.int32), ('nConnected', np.int32),
                       ('orderedKF', np.int32), ('orderedWeight', np.int32), ('parent', np.int32), ('nbrCount', np.int32), ('nbrKF', np.int32),
                       ('nbrWeight', np.int32))


class OrbmConnectionsItem(C.Structure):
    """One keyframe of orbm_update_connections_batch (include/orb_b200.h)."""
    _fields_ = [('mode', C.c_int), ('nKF', C.c_int)] + \
               [(n, C.c_void_p) for n in ('order', 'mnId', 'kfFlags', 'cameraCenter', 'connStart', 'connKF', 'connWeight')] + \
               [('firstConnection', C.c_int), ('nlevels', C.c_int), ('scaleFactors', C.c_void_p), ('nSlots', C.c_int)] + \
               [(n, C.c_void_p) for n in ('slotPoint', 'slotOctave', 'slotDesc')] + [('nPoints', C.c_int)] + \
               [(n, C.c_void_p) for n in ('pointBad', 'pointPos', 'pointRefKF', 'obsStart', 'obsKF', 'obsIdx', 'obsOctave', 'obsDesc')] + \
               [(n, C.c_void_p) for n, _ in CONNECTIONS_OUTPUTS]


def connections_struct(m):
    """OrbmConnectionsItem over item dict `m` (keys CONNECTIONS_ARRAYS + CONNECTIONS_SCALARS) with fresh outputs: (struct, out dict, arrays
    to keep alive).  Outputs: slotStatus [nSlots], pointUpdated / minDistance / maxDistance / descKF / descIdx [nPoints], normal [nPoints, 3],
    counter / orderedKF / orderedWeight / nbrCount [nKF], nConnected / parent [1], nbrKF / nbrWeight [connStart[-1] + nKF]."""
    a = {n: (_c(m[n], dt) if m.get(n) is not None else None) for n, dt in CONNECTIONS_ARRAYS}
    nK, nS, nP = len(a['order']), len(a['slotPoint']), len(a['pointBad'])
    a['cameraCenter'] = a['cameraCenter'].reshape(-1, 3)
    sizes = dict(slotStatus=nS, pointUpdated=nP, normal=(nP, 3), minDistance=nP, maxDistance=nP, descKF=nP, descIdx=nP, counter=nK, nConnected=1,
                 orderedKF=nK, orderedWeight=nK, parent=1, nbrCount=nK, nbrKF=int(a['connStart'][-1]) + nK, nbrWeight=int(a['connStart'][-1]) + nK)
    out = {n: np.zeros(sizes[n], dt) for n, dt in CONNECTIONS_OUTPUTS}
    s = OrbmConnectionsItem(int(m['mode']), nK, *[_ptr(a[n]) for n in ('order', 'mnId', 'kfFlags', 'cameraCenter', 'connStart', 'connKF', 'connWeight')],
                            int(m['firstConnection']), len(a['scaleFactors']), _ptr(a['scaleFactors']), nS,
                            *[_ptr(a[n]) for n in ('slotPoint', 'slotOctave', 'slotDesc')], nP,
                            *[_ptr(a[n]) for n in ('pointBad', 'pointPos', 'pointRefKF', 'obsStart', 'obsKF', 'obsIdx', 'obsOctave', 'obsDesc')],
                            *[_ptr(out[n]) for n, _ in CONNECTIONS_OUTPUTS])
    return s, out, a


def _connections_result(out):
    return dict(out, nConnected=int(out['nConnected'][0]), parent=int(out['parent'][0]))


#: the arrays of orbm_update_local_map_batch*'s input with their dtypes (OrbmUpdateLocalMapBatch, after its six sizes)
LOCAL_MAP_ARRAYS = (('kfStart', np.int32), ('kfFlags', np.uint8), ('covStart', np.int32), ('covKF', np.int32), ('childStart', np.int32),
                    ('childKF', np.int32), ('parent', np.int32), ('prevKF', np.int32), ('slotStart', np.int32), ('slotPoint', np.int32),
                    ('pointStart', np.int32), ('pointBad', np.uint8), ('obsStart', np.int32), ('obsKF', np.int32), ('worldPos', np.float32),
                    ('normal', np.float32), ('minDistInv', np.float32), ('maxDistInv', np.float32), ('maxDistance', np.float32),
                    ('mpDesc', np.uint8), ('hasObs', np.uint8), ('nSrc', np.int32), ('srcPoint', np.int32), ('voteLastFrame', np.uint8),
                    ('match', np.int32), ('nK', np.int32), ('inertial', np.uint8), ('lastKF', np.int32))
LOCAL_MAP_SIZES = ('batch', 'kcap', 'mcap', 'mcapLast', 'nKF', 'nPoints')
#: its outputs: (name, dtype, row shape); rows are 'kf' = [nKF], 'b' = [batch], 'm' = [batch, mcap], 'l' = [batch, mcapLast]
LOCAL_MAP_OUTPUTS = (('localKF', np.int32, 'kf', ()), ('nLocalKF', np.int32, 'b', ()), ('refKF', np.int32, 'b', ()), ('localPoint', np.int32, 'm', ()),
                     ('nM', np.int32, 'b', ()), ('worldPos', np.float32, 'm', (3,)), ('normal', np.float32, 'm', (3,)), ('minDistInv', np.float32, 'm', ()),
                     ('maxDistInv', np.float32, 'm', ()), ('maxDistance', np.float32, 'm', ()), ('mpDesc', np.uint8, 'm', (32,)),
                     ('hasObs', np.uint8, 'm', ()), ('bad', np.uint8, 'm', ()), ('lastToLocal', np.int32, 'l', ()))


class OrbmUpdateLocalMapBatch(C.Structure):
    """Input of orbm_update_local_map_batch* (include/orb_b200.h)."""
    _fields_ = [(n, C.c_int) for n in LOCAL_MAP_SIZES] + [(n, C.c_void_p) for n, _ in LOCAL_MAP_ARRAYS]


class OrbmUpdateLocalMapResult(C.Structure):
    """Output of orbm_update_local_map_batch* (include/orb_b200.h)."""
    _fields_ = [(n, C.c_void_p) for n, _, _, _ in LOCAL_MAP_OUTPUTS]


def local_map_batch(items, mcap, kcap=None, mcapLast=None):
    """The batch dict of orbm_update_local_map_batch from one dict per stream: its keyframe table (kfFlags, parent, prevKF [nk]; covStart /
    covKF, childStart / childKF, slotStart / slotPoint as CSR), its points (pointBad, minDistInv, maxDistInv, maxDistance, hasObs [np];
    worldPos, normal [np, 3]; mpDesc [np, 32]; obsStart / obsKF as CSR), its vote source (srcPoint [nSrc], voteLastFrame, match [nK] when
    voteLastFrame is 0) and inertial / lastKF.  Indices stay stream-local; the CSR offsets become offsets into the concatenated arrays."""
    B = len(items)
    kcap = kcap or max([1] + [len(it.get('match', ())) for it in items])
    mcapLast = mcapLast or max([1] + [len(it['srcPoint']) for it in items])
    cat = lambda name, dt, shape=(): np.concatenate([np.asarray(it[name], dt).reshape((-1,) + shape) for it in items])   # noqa: E731

    def csr(start, vals):
        off, starts = 0, [np.zeros(1, np.int32)]
        for it in items:
            s = np.asarray(it[start], np.int32)
            starts.append(s[1:] + off)
            off += int(s[-1])
        return np.concatenate(starts).astype(np.int32), cat(vals, np.int32)
    d = dict(batch=B, kcap=kcap, mcap=mcap, mcapLast=mcapLast)
    d['kfStart'] = np.concatenate([[0], np.cumsum([len(it['kfFlags']) for it in items])]).astype(np.int32)
    d['pointStart'] = np.concatenate([[0], np.cumsum([len(it['pointBad']) for it in items])]).astype(np.int32)
    d['nKF'], d['nPoints'] = int(d['kfStart'][-1]), int(d['pointStart'][-1])
    for n in ('kfFlags', 'pointBad', 'hasObs'):
        d[n] = cat(n, np.uint8)
    for n in ('parent', 'prevKF'):
        d[n] = cat(n, np.int32)
    for n in ('minDistInv', 'maxDistInv', 'maxDistance'):
        d[n] = cat(n, np.float32)
    d['worldPos'], d['normal'], d['mpDesc'] = cat('worldPos', np.float32, (3,)), cat('normal', np.float32, (3,)), cat('mpDesc', np.uint8, (32,))
    for start, vals in (('covStart', 'covKF'), ('childStart', 'childKF'), ('slotStart', 'slotPoint'), ('obsStart', 'obsKF')):
        d[start], d[vals] = csr(start, vals)
    d['nSrc'] = np.array([len(it['srcPoint']) for it in items], np.int32)
    d['srcPoint'] = np.full((B, mcapLast), -1, np.int32)
    d['match'] = np.full((B, kcap), -1, np.int32)
    d['nK'] = np.zeros(B, np.int32)
    for b, it in enumerate(items):
        d['srcPoint'][b, :len(it['srcPoint'])] = it['srcPoint']
        if it.get('match') is not None:
            d['match'][b, :len(it['match'])] = it['match']
            d['nK'][b] = len(it['match'])
    for n in ('voteLastFrame', 'inertial'):
        d[n] = np.array([int(it[n]) for it in items], np.uint8)
    d['lastKF'] = np.array([int(it['lastKF']) for it in items], np.int32)
    return d


def local_map_outputs(d, alloc=None):
    """Fresh output arrays for batch dict ``d`` (``alloc(shape, dtype)``: numpy zeros by default)."""
    alloc = alloc or (lambda shape, dt: np.zeros(shape, dt))
    rows = dict(kf=(d['nKF'],), b=(d['batch'],), m=(d['batch'], d['mcap']), l=(d['batch'], d['mcapLast']))
    return {n: alloc(rows[r] + sh, dt) for n, dt, r, sh in LOCAL_MAP_OUTPUTS}


def local_map_structs(d, out, get):
    """(OrbmUpdateLocalMapBatch, OrbmUpdateLocalMapResult) over batch dict ``d`` and outputs ``out``; ``get(k)`` gives an array's address."""
    s = OrbmUpdateLocalMapBatch(*[int(d[n]) for n in LOCAL_MAP_SIZES], *[get(n) for n, _ in LOCAL_MAP_ARRAYS])
    r = OrbmUpdateLocalMapResult(*[_ptr(out[n]) for n, _, _, _ in LOCAL_MAP_OUTPUTS])
    return s, r


def local_map_split(d, out):
    """Per stream: dict(localKF (table rows of the stream, in mvpLocalKeyFrames order), refKF, localPoint, nM, lastToLocal [nSrc])."""
    res = []
    for b in range(d['batch']):
        k0, n = int(d['kfStart'][b]), int(out['nLocalKF'][b])
        nM = int(out['nM'][b])
        res.append(dict(localKF=out['localKF'][k0:k0 + n].copy(), refKF=int(out['refKF'][b]), nM=nM,
                        localPoint=out['localPoint'][b, :min(nM, d['mcap'])].copy(), lastToLocal=out['lastToLocal'][b, :int(d['nSrc'][b])].copy()))
    return res


def _c(a, dt):
    return np.ascontiguousarray(a, dt)


def _host_call(d, dtypes, name, resident, frame_keys):
    """(pointer getter, C function) of a batched call's host form.  The getter gives the address of ``d[k]`` made contiguous as
    ``dtypes[k]`` (None for a missing key) and holds those arrays, so keep it until the call returns.  With ``resident``, device
    pointers of the current frame in the order of ``frame_keys``, it gives those for the frame and the function is the _resident form."""
    keep = {k: _c(d[k], dt) for k, dt in dtypes.items() if d.get(k) is not None}
    if resident is not None:
        keep.update(zip(frame_keys, resident))

    def get(k):
        return (keep[k] if isinstance(keep[k], int) else keep[k].ctypes.data) if k in keep else None
    return get, getattr(lib(), name + '_resident' if resident is not None else name)


class Frame:
    """The slice of ``ORB_SLAM3::Frame`` the matchers read: mvKeysUn, mDescriptors, image bounds, mvScaleFactors,
    and the in/out ``mvpMapPoints`` state as (match index, claimed flag) per keypoint."""

    def __init__(self, keypoints, descriptors, bounds, scale_factors):
        self.keypoints = _c(keypoints, KP_DTYPE)
        self.descriptors = _c(descriptors, np.uint8).reshape(-1, 32)
        self.bounds = tuple(float(b) for b in bounds)   # mnMinX, mnMinY, mnMaxX, mnMaxY
        self.scale_factors = _c(scale_factors, np.float32)
        self.match = np.full(len(self.keypoints), -1, np.int32)     # mvpMapPoints[i] as an index, -1 = NULL
        self.claimed = np.zeros(len(self.keypoints), np.uint8)      # mvpMapPoints[i]->Observations() > 0

    def _struct(self):
        return _OrbmFrame(len(self.keypoints), _ptr(self.keypoints), _ptr(self.descriptors), *self.bounds,
                          _ptr(self.scale_factors), len(self.scale_factors))


class ORBmatcher:
    """Mirror of ``ORB_SLAM3::ORBmatcher`` (reference include/ORBmatcher.h:36-103) for the per-frame hot functions."""
    TH_HIGH, TH_LOW, HISTO_LENGTH = 100, 50, 30   # src/ORBmatcher.cc:35-37

    def __init__(self, nnratio=0.6, checkOri=True, max_batch=1, max_keypoints=2048, max_mappoints=8192, device=0):
        self.mfNNratio, self.mbCheckOrientation = float(nnratio), bool(checkOri)
        self._h = C.c_void_p()
        rc = lib().orbm_create(C.byref(self._h), max_batch, max_keypoints, max_mappoints, device)
        if rc != ORB_OK:
            self._h = None
            raise OrbError(rc, 'orbm_create')

    def close(self):
        if getattr(self, '_h', None):
            lib().orbm_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:      # interpreter shutdown: module globals may already be gone
            pass

    def DescriptorDistance(self, a, b):
        """ORBmatcher::DescriptorDistance for one pair or for n pairs ([n,32] arrays)."""
        a = _c(a, np.uint8).reshape(-1, 32)
        b = _c(b, np.uint8).reshape(-1, 32)
        out = np.zeros(len(a), np.int32)
        rc = lib().orbm_descriptor_distance(self._h, _ptr(a), _ptr(b), len(a), _ptr(out))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbm_descriptor_distance')
        return int(out[0]) if len(out) == 1 else out

    def isInFrustum(self, pts, Rcw, tcw, Ow, cam, bounds, log_scale_factor, n_levels, viewingCosLimit=0.5, mbf=0.0):
        """``Frame::isInFrustum`` + ``MapPoint::PredictScale`` (src/Frame.cc:512-574, src/MapPoint.cc:531-546) for all local map
        points of one frame. ``pts``: worldPos [M,3], normal [M,3], minDistInv, maxDistInv, maxDistance [M]. Returns the tracking
        fields (inView, projX, projY, projXR, depth, level, viewCos) that the local-map SearchByProjection reads."""
        keep = {k: _c(pts[k], np.float32) for k in ('worldPos', 'normal', 'minDistInv', 'maxDistInv', 'maxDistance')}
        M = len(keep['minDistInv'])
        s = _OrbmFrustumIn(M, *[_ptr(keep[k]) for k in ('worldPos', 'normal', 'minDistInv', 'maxDistInv', 'maxDistance')],
                           (C.c_float * 9)(*[float(v) for v in np.asarray(Rcw, np.float32).reshape(9)]),
                           (C.c_float * 3)(*[float(v) for v in np.asarray(tcw, np.float32).reshape(3)]),
                           (C.c_float * 3)(*[float(v) for v in np.asarray(Ow, np.float32).reshape(3)]),
                           (C.c_float * 4)(*[float(v) for v in cam]), *[float(b) for b in bounds], float(mbf),
                           float(np.float32(log_scale_factor)), int(n_levels), float(viewingCosLimit))
        out = dict(inView=np.zeros(M, np.uint8), projX=np.zeros(M, np.float32), projY=np.zeros(M, np.float32), projXR=np.zeros(M, np.float32),
                   depth=np.zeros(M, np.float32), level=np.zeros(M, np.int32), viewCos=np.zeros(M, np.float32))
        rc = lib().orbm_frustum_project(self._h, C.byref(s), *[_ptr(out[k]) for k in ('inView', 'projX', 'projY', 'projXR', 'depth', 'level', 'viewCos')])
        if rc != ORB_OK:
            raise OrbError(rc, 'orbm_frustum_project')
        return out

    def SearchByProjection(self, F, *args, **kw):
        """Overloads by argument type as in the reference: (F, map_points: dict, th, bFarPoints=False, thFarPoints=50)
        or (CurrentFrame, last_frame: dict, th, bMono, Tcw=..., cam=...)."""
        pts = args[0]
        if 'projX' in pts:
            return self._search_local_map(F, pts, *args[1:], **kw)
        return self._search_last_frame(F, pts, *args[1:], **kw)

    def _search_local_map(self, F, pts, th=1.0, bFarPoints=False, thFarPoints=50.0):
        M = len(pts['projX'])
        keep = dict(inView=_c(pts['inView'], np.uint8), bad=_c(pts['bad'], np.uint8), depth=_c(pts['depth'], np.float32),
                    projX=_c(pts['projX'], np.float32), projY=_c(pts['projY'], np.float32), level=_c(pts['level'], np.int32),
                    viewCos=_c(pts['viewCos'], np.float32), hasObs=_c(pts['hasObs'], np.uint8),
                    descriptors=_c(pts['descriptors'], np.uint8))
        s = _OrbmLocalPoints(M, *[_ptr(keep[k]) for k in ('inView', 'bad', 'depth', 'projX', 'projY', 'level', 'viewCos', 'hasObs', 'descriptors')])
        fs = F._struct()
        n = C.c_int(0)
        rc = lib().orbm_search_local_map(self._h, C.byref(fs), C.byref(s), th, self.mfNNratio, int(bFarPoints), thFarPoints,
                                         _ptr(F.match), _ptr(F.claimed), C.byref(n))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbm_search_local_map')
        return n.value

    def _search_last_frame(self, F, last, th, bMono=True, Tcw=None, cam=None):
        assert bMono, 'only the monocular branch is on the hot path (SURVEY.md 8a row a10)'
        M = len(last['valid'])
        keep = dict(valid=_c(last['valid'], np.uint8), xyz=_c(last['xyz'], np.float32), octave=_c(last['octave'], np.int32),
                    angle=_c(last['angle'], np.float32), hasObs=_c(last['hasObs'], np.uint8), descriptors=_c(last['descriptors'], np.uint8))
        s = _OrbmLastFrame(M, *[_ptr(keep[k]) for k in ('valid', 'xyz', 'octave', 'angle', 'hasObs', 'descriptors')])
        T = _c(Tcw, np.float32)
        cm = _c(cam, np.float32)
        fs = F._struct()
        n = C.c_int(0)
        rc = lib().orbm_search_last_frame(self._h, C.byref(fs), C.byref(s), _ptr(T), _ptr(cm), th, int(self.mbCheckOrientation),
                                          _ptr(F.match), _ptr(F.claimed), C.byref(n))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbm_search_last_frame')
        return n.value

    _BATCH_DT = dict(kps=KP_DTYPE, desc=np.uint8, nK=np.int32, scaleFactors=np.float32, nM=np.int32, valid=np.uint8, xyz=np.float32, octave=np.int32,
                     angle=np.float32, hasObs=np.uint8, mpDesc=np.uint8, Tcw7=np.float32)
    _MOTION_IN = ('kps', 'nK', 'xyz', 'hasObs', 'Tcw7')
    _MOTION_DT = dict(kps=KP_DTYPE, nK=np.int32, xyz=np.float32, hasObs=np.uint8, Tcw7=np.float32, invLevelSigma2=np.float32, active=np.uint8)

    @staticmethod
    def _batch_struct(d, get, keys, search=True):
        """OrbmBatchDevice of ``d`` with the arrays ``keys`` at ``get(k)``; the bounds and the reset flag only for the last-frame search."""
        s = _OrbmBatchDevice()
        s.batch, s.kcap, s.mcap, s.nlevels = d['batch'], d['kcap'], d['mcap'], d['nlevels']
        for k in keys:
            setattr(s, k, get(k))
        s.cam = (C.c_float * 4)(*d['cam'])
        if search:
            s.minX, s.minY, s.maxX, s.maxY = d['bounds']
            s.resetState = int(d.get('reset', 0))
        return s

    def search_last_frame_batch_device(self, d, th, d_match, d_claimed, d_nmatches, stream=0):
        """Device-resident batch (torch CUDA tensors in dict ``d``; see OrbmBatchDevice in include/orb_b200.h)."""
        s = self._batch_struct(d, lambda k: d[k].data_ptr(), self._BATCH_DT)
        rc = lib().orbm_search_last_frame_batch_device(self._h, C.byref(s), th, int(self.mbCheckOrientation), _ptr(d_match),
                                                       _ptr(d_claimed), _ptr(d_nmatches), C.c_void_p(stream))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbm_search_last_frame_batch_device')

    def search_last_frame_batch(self, d, th, match, claimed, nmatches, resident=None):
        """Host-buffer batch (numpy arrays in dict ``d``, same keys as the device variant); in/out arrays are numpy.
        ``resident`` = ``ORBextractor.resident_slabs()`` of the extractor that just produced the frames: the current frame is then read
        from the device slabs (d['kps'], d['desc'], d['nK'] are ignored) instead of being uploaded again."""
        assert resident is None or resident[3] == d['kcap']
        get, fn = _host_call(d, self._BATCH_DT, 'orbm_search_last_frame_batch', resident, ('kps', 'desc', 'nK'))
        s = self._batch_struct(d, get, self._BATCH_DT)
        rc = fn(self._h, C.byref(s), th, int(self.mbCheckOrientation), _ptr(match), _ptr(claimed), _ptr(nmatches))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbm_search_last_frame_batch')

    # --- Tracking's per-frame steps after the last-frame search, batched over streams (include/orb_b200.h) ---
    def motion_model_pose_batch(self, d, inv_level_sigma2, match, claimed, nmatches, active=None):
        """TrackWithMotionModel from PoseOptimization through the "discard outliers" loop for ``d['batch']`` streams (host numpy).
        ``d``: the dict ``search_last_frame_batch`` took (kps, nK, xyz, hasObs, Tcw7, cam, kcap, mcap, nlevels are read); ``match`` /
        ``claimed`` [B, kcap] and ``nmatches`` [B] are what the search wrote and are updated in place; ``active`` [B] u8 or None.
        Returns dict(pose7 [B,7] f64, Tcw7 [B,7] f32, discarded [B,mcap] u8, nmatchesMap [B] i32); rows of inactive streams are zero."""
        B, M = d['batch'], d['mcap']
        get, fn = _host_call(dict(d, invLevelSigma2=inv_level_sigma2, active=active), self._MOTION_DT, 'orbm_motion_model_pose_batch', None, ())
        s = self._batch_struct(d, get, self._MOTION_IN, search=False)
        out = dict(pose7=np.zeros((B, 7)), Tcw7=np.zeros((B, 7), np.float32), discarded=np.zeros((B, M), np.uint8), nmatchesMap=np.zeros(B, np.int32))
        for a, dt in ((match, np.int32), (claimed, np.uint8), (nmatches, np.int32)):
            assert a.dtype == dt and a.flags.c_contiguous
        rc = fn(self._h, C.byref(s), get('invLevelSigma2'), get('active'), _ptr(match), _ptr(claimed), _ptr(nmatches),
                *[_ptr(out[k]) for k in ('pose7', 'Tcw7', 'discarded', 'nmatchesMap')])
        if rc != ORB_OK:
            raise OrbError(rc, 'orbm_motion_model_pose_batch')
        return out

    def motion_model_pose_batch_device(self, d, inv_level_sigma2, match, claimed, nmatches, pose7, Tcw7, discarded, nmatchesMap, active=None,
                                       stream=0):
        """Device form of :meth:`motion_model_pose_batch`: torch CUDA tensors in ``d`` and as arguments; enqueues on ``stream``."""
        s = self._batch_struct(d, lambda k: d[k].data_ptr(), self._MOTION_IN, search=False)
        rc = lib().orbm_motion_model_pose_batch_device(self._h, C.byref(s), _ptr(inv_level_sigma2), _ptr(active), _ptr(match), _ptr(claimed),
                                                       _ptr(nmatches), _ptr(pose7), _ptr(Tcw7), _ptr(discarded), _ptr(nmatchesMap),
                                                       C.c_void_p(stream))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbm_motion_model_pose_batch_device')

    @staticmethod
    def _local_map_struct(d, get):
        s = _OrbmLocalMapBatch()
        s.batch, s.kcap, s.mcap, s.nlevels = d['batch'], d['kcap'], d['mcap'], d['nlevels']
        s.mcapLast = d.get('mcapLast', 0)
        s.minX, s.minY, s.maxX, s.maxY = d['bounds']
        s.cam = (C.c_float * 4)(*d['cam'])
        s.mbf, s.logScaleFactor = float(d.get('mbf', 0.0)), float(np.float32(d['logScaleFactor']))
        s.nnratio, s.bFarPoints, s.thFarPoints = float(d.get('nnratio', 0.8)), int(d.get('bFarPoints', 0)), float(d.get('thFarPoints', 0.0))
        s.viewingCosLimit = float(d.get('viewingCosLimit', 0.5))
        for k in ('kps', 'desc', 'nK', 'scaleFactors', 'invLevelSigma2', 'Tcw7', 'lastToLocal', 'discarded', 'nM', 'worldPos', 'normal', 'minDistInv',
                  'maxDistInv', 'maxDistance', 'mpDesc', 'hasObs', 'bad', 'th', 'active'):
            setattr(s, k, get(k))
        return s

    _LOCAL_MAP_DT = dict(kps=KP_DTYPE, desc=np.uint8, nK=np.int32, scaleFactors=np.float32, invLevelSigma2=np.float32, Tcw7=np.float32,
                         lastToLocal=np.int32, discarded=np.uint8, nM=np.int32, worldPos=np.float32, normal=np.float32, minDistInv=np.float32,
                         maxDistInv=np.float32, maxDistance=np.float32, mpDesc=np.uint8, hasObs=np.uint8, bad=np.uint8, th=np.float32, active=np.uint8)

    def track_local_map_batch(self, d, match, resident=None):
        """TrackLocalMap from SearchLocalPoints through the statistics loop for ``d['batch']`` streams (host numpy; see OrbmLocalMapBatch in
        include/orb_b200.h for the keys; 'lastToLocal', 'discarded' and 'active' may be None or absent).  ``match`` [B, kcap] i32 is updated
        in place (local indices afterwards).  ``resident`` = ``ORBextractor.resident_slabs()``: the current frame is read from the device.
        Returns dict(claimed, outlier [B,kcap] u8, visible, found [B,mcap] i32, nToMatch, nmatches, nInliers, nMatchesInliers [B] i32,
        pose7 [B,7] f64, Tcw7 [B,7] f32); rows of inactive streams are zero."""
        B, K, M = d['batch'], d['kcap'], d['mcap']
        assert resident is None or resident[3] == K
        get, fn = _host_call(d, self._LOCAL_MAP_DT, 'orbm_track_local_map_batch', resident, ('kps', 'desc', 'nK'))
        s = self._local_map_struct(d, get)
        assert match.dtype == np.int32 and match.flags.c_contiguous and match.shape == (B, K)
        out = dict(match=match, claimed=np.zeros((B, K), np.uint8), outlier=np.zeros((B, K), np.uint8), visible=np.zeros((B, M), np.int32),
                   found=np.zeros((B, M), np.int32), nToMatch=np.zeros(B, np.int32), nmatches=np.zeros(B, np.int32), nInliers=np.zeros(B, np.int32),
                   nMatchesInliers=np.zeros(B, np.int32), pose7=np.zeros((B, 7)), Tcw7=np.zeros((B, 7), np.float32))
        r = _OrbmLocalMapResult(*[_ptr(out[k]) for k in _LOCAL_MAP_OUT])
        rc = fn(self._h, C.byref(s), C.byref(r))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbm_track_local_map_batch')
        del out['match']
        return out

    def track_local_map_batch_device(self, d, out, stream=0):
        """Device form of :meth:`track_local_map_batch`: torch CUDA tensors in ``d`` and ``out`` (keys of OrbmLocalMapResult; out['match']
        is in / out); enqueues on ``stream``."""
        s = self._local_map_struct(d, lambda k: d[k].data_ptr() if d.get(k) is not None else None)
        r = _OrbmLocalMapResult(*[_ptr(out[k]) for k in _LOCAL_MAP_OUT])
        rc = lib().orbm_track_local_map_batch_device(self._h, C.byref(s), C.byref(r), C.c_void_p(stream))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbm_track_local_map_batch_device')

    _IMU_DT = dict(preintKF=np.float32, preintFrame=np.float32, kfState21=np.float32, lastState21=np.float32, prior21=np.float64, priorH=np.float64)

    @staticmethod
    def _imu_struct(imu, mode, get):
        s = _OrbmImuTrackBatch()
        s.mode = mode.ctypes.data
        s.Tcb7 = (C.c_float * 7)(*[float(v) for v in np.asarray(imu['Tcb7'], np.float32)])
        for k in ('extrinsics24',) + tuple(ORBmatcher._IMU_DT):
            setattr(s, k, get(k))
        return s

    def track_local_map_inertial_batch(self, d, imu, resident=None):
        """Tracking::Track for monocular-inertial frames once the IMU is initialised (PredictStateIMU, SearchLocalPoints, the inertial pose
        optimiser and its write-back) for ``d['batch']`` streams, host numpy.  ``d``: the keys of :meth:`track_local_map_batch` without
        Tcw7 / lastToLocal / discarded / active; ``imu``: mode [B] u8 (0 skip, 1 map updated, 2 not), Tcb7 [7], extrinsics24 [24], preintKF /
        preintFrame [B, IMU_PREINT_FLOATS], kfState21 / lastState21 [B, 21] f32, prior21 [B, 21] / priorH [B, 15, 15] f64 (see
        OrbmImuTrackBatch in include/orb_b200.h; arrays a call does not need may be None).  Returns dict(match, claimed, outlier [B, kcap],
        visible, found [B, mcap], nToMatch, nmatches, nInliers, nMatchesInliers [B], Tcw7 [B, 7], predState21 [B, 21], predTcw7 [B, 7],
        state21 [B, 21], prior21 [B, 21], priorH [B, 15, 15]); rows of mode-0 streams keep their initial values (match -1, the rest 0)."""
        B, K, M = d['batch'], d['kcap'], d['mcap']
        assert resident is None or resident[3] == K
        get, fn = _host_call(d, self._LOCAL_MAP_DT, 'orbm_track_local_map_inertial_batch', resident, ('kps', 'desc', 'nK'))
        s = self._local_map_struct(d, get)
        ik = {k: _c(imu[k], dt) for k, dt in dict(self._IMU_DT, extrinsics24=np.float64).items() if imu.get(k) is not None}
        mode = _c(imu['mode'], np.uint8)
        si = self._imu_struct(imu, mode, lambda k: ik[k].ctypes.data if k in ik else None)
        out = dict(match=np.full((B, K), -1, np.int32), claimed=np.zeros((B, K), np.uint8), outlier=np.zeros((B, K), np.uint8),
                   visible=np.zeros((B, M), np.int32), found=np.zeros((B, M), np.int32), nToMatch=np.zeros(B, np.int32), nmatches=np.zeros(B, np.int32),
                   nInliers=np.zeros(B, np.int32), nMatchesInliers=np.zeros(B, np.int32), pose7=None, Tcw7=np.zeros((B, 7), np.float32))
        io = dict(predState21=np.zeros((B, 21), np.float32), predTcw7=np.zeros((B, 7), np.float32), state21=np.zeros((B, 21), np.float32),
                  prior21=np.zeros((B, 21)), priorH=np.zeros((B, 15, 15)))
        r = _OrbmLocalMapResult(*[_ptr(out[k]) for k in _LOCAL_MAP_OUT])
        ri = _OrbmImuTrackResult(*[_ptr(io[k]) for k in _IMU_TRACK_OUT])
        rc = fn(self._h, C.byref(s), C.byref(si), C.byref(r), C.byref(ri))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbm_track_local_map_inertial_batch')
        del out['pose7']
        out.update(io)
        return out

    def track_local_map_inertial_batch_device(self, d, imu, out, stream=0):
        """Device form of :meth:`track_local_map_inertial_batch`: torch CUDA tensors in ``d``, ``imu`` (imu['mode'] stays a host numpy
        array) and ``out`` (keys of OrbmLocalMapResult without pose7, and of OrbmImuTrackResult); enqueues on ``stream``."""
        s = self._local_map_struct(d, lambda k: d[k].data_ptr() if d.get(k) is not None else None)
        mode = _c(imu['mode'], np.uint8)
        si = self._imu_struct(imu, mode, lambda k: imu[k].data_ptr() if imu.get(k) is not None else None)
        r = _OrbmLocalMapResult(*[_ptr(out[k]) if k != 'pose7' else None for k in _LOCAL_MAP_OUT])
        ri = _OrbmImuTrackResult(*[_ptr(out[k]) for k in _IMU_TRACK_OUT])
        rc = lib().orbm_track_local_map_inertial_batch_device(self._h, C.byref(s), C.byref(si), C.byref(r), C.byref(ri), C.c_void_p(stream))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbm_track_local_map_inertial_batch_device')

    @staticmethod
    def _ref_kf_struct(d, get):
        s = _OrbmRefKeyFrameBatch()
        s.batch, s.kcap, s.mcap, s.nlevels = d['batch'], d['kcap'], d['mcap'], d['nlevels']
        for k in _REF_KF_IN + ('invLevelSigma2', 'active'):
            setattr(s, k, get(k))
        s.cam = (C.c_float * 4)(*d['cam'])
        return s

    _REF_KF_DT = dict(kps=KP_DTYPE, desc=np.uint8, nK=np.int32, fvNode=np.int32, fvFeature=np.int32, nEntries=np.int32, Tcw7=np.float32, kfN=np.int32,
                      kfKps=KP_DTYPE, kfDesc=np.uint8, kfFvNode=np.int32, kfFvFeature=np.int32, kfNEntries=np.int32, kfPoint=np.uint8, xyz=np.float32,
                      hasObs=np.uint8, invLevelSigma2=np.float32, active=np.uint8)

    def track_reference_keyframe_batch(self, d, resident=None):
        """Tracking::TrackReferenceKeyFrame after Frame::ComputeBoW for ``d['batch']`` streams, host numpy (see OrbmRefKeyFrameBatch in
        include/orb_b200.h for the keys; 'active' may be None or absent).  SearchByBoW with ORBmatcher(0.7, true) and, for streams with
        at least 15 matches, PoseOptimization from Tcw7 (mLastFrame's pose) and the "discard outliers" loop.  ``resident`` = (kps, desc, nK,
        fvNode, fvFeature, nEntries) device pointers of the current frame with stride d['kcap'] (d's frame keys are then ignored).
        Returns dict(nmatches [B], match [B, kcap] i32, pose7 [B, 7] f64, Tcw7 [B, 7] f32, discarded [B, mcap] u8, nmatchesMap [B] i32);
        rows the call does not write keep their initial values (match -1, the rest 0)."""
        B, K, M = d['batch'], d['kcap'], d['mcap']
        get, fn = _host_call(d, self._REF_KF_DT, 'orbm_track_reference_keyframe_batch', resident, _REF_KF_FRAME)
        s = self._ref_kf_struct(d, get)
        out = dict(nmatches=np.zeros(B, np.int32), match=np.full((B, K), -1, np.int32), pose7=np.zeros((B, 7)), Tcw7=np.zeros((B, 7), np.float32),
                   discarded=np.zeros((B, M), np.uint8), nmatchesMap=np.zeros(B, np.int32))
        r = _OrbmRefKeyFrameResult(*[_ptr(out[k]) for k in _REF_KF_OUT])
        rc = fn(self._h, C.byref(s), C.byref(r))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbm_track_reference_keyframe_batch')
        return out

    def track_reference_keyframe_batch_device(self, d, out, stream=0):
        """Device form of :meth:`track_reference_keyframe_batch`: torch CUDA tensors in ``d`` and ``out`` (keys of OrbmRefKeyFrameResult);
        enqueues on ``stream``."""
        s = self._ref_kf_struct(d, lambda k: d[k].data_ptr() if d.get(k) is not None else None)
        r = _OrbmRefKeyFrameResult(*[_ptr(out[k]) for k in _REF_KF_OUT])
        rc = lib().orbm_track_reference_keyframe_batch_device(self._h, C.byref(s), C.byref(r), C.c_void_p(stream))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbm_track_reference_keyframe_batch_device')

    def SearchForInitialization(self, F1, F2, vbPrevMatched, windowSize=10):
        """``int ORBmatcher::SearchForInitialization(F1, F2, vbPrevMatched, vnMatches12, windowSize)`` (src/ORBmatcher.cc:648-763).
        ``vbPrevMatched`` [K1, 2] float32 is updated in place; returns (nmatches, vnMatches12 [K1] i32, -1 = none)."""
        assert vbPrevMatched.dtype == np.float32 and vbPrevMatched.flags.c_contiguous and vbPrevMatched.shape == (len(F1.keypoints), 2)
        m12 = np.full(len(F1.keypoints), -1, np.int32)
        n = C.c_int(0)
        f1, f2 = F1._struct(), F2._struct()
        L = lib()
        rc = L.orbm_search_for_initialization(self._h, C.byref(f1), C.byref(f2), _ptr(vbPrevMatched), int(windowSize), self.mfNNratio,
                                              int(self.mbCheckOrientation), _ptr(m12), C.byref(n))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbm_search_for_initialization')
        return n.value, m12

    def SearchByBoW(self, kf_kps, kf_desc, kf_point, kf_fv, f_kps, f_desc, f_fv):
        """``int ORBmatcher::SearchByBoW(KeyFrame*, Frame&, vector<MapPoint*>&)`` (src/ORBmatcher.cc:223-425).  ``*_fv`` = (node ids, feature indices) of
        the DBoW2 FeatureVector; ``kf_point`` [nKF]: 0 none / 1 map point / 2 bad.  Returns (nmatches, match [nF] = keyframe feature index or -1)."""
        keep = [_c(kf_kps, KP_DTYPE), _c(kf_desc, np.uint8), _c(kf_fv[0], np.int32), _c(kf_fv[1], np.int32), _c(f_kps, KP_DTYPE), _c(f_desc, np.uint8),
                _c(f_fv[0], np.int32), _c(f_fv[1], np.int32), _c(kf_point, np.uint8)]
        a = _OrbmBowFrame(len(keep[0]), keep[0].ctypes.data, keep[1].ctypes.data, len(keep[2]), keep[2].ctypes.data, keep[3].ctypes.data)
        b = _OrbmBowFrame(len(keep[4]), keep[4].ctypes.data, keep[5].ctypes.data, len(keep[6]), keep[6].ctypes.data, keep[7].ctypes.data)
        match = np.full(len(keep[4]), -1, np.int32)
        n = C.c_int(0)
        L = lib()
        rc = L.orbm_search_by_bow(self._h, C.byref(a), _ptr(keep[8]), C.byref(b), self.mfNNratio, int(self.mbCheckOrientation), _ptr(match), C.byref(n))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbm_search_by_bow')
        return n.value, match

    def FuseSearch(self, kf_kps, kf_desc, bounds, scale_factors, inv_level_sigma2, log_scale_factor, Tcw7, Ow, cam4, state, xyz, normal, min_d, max_d,
                   mp_desc, th=3.0):
        """The search of ``int ORBmatcher::Fuse(KeyFrame*, const vector<MapPoint*>&, th)`` (src/ORBmatcher.cc:1148-1338): (bestIdx [M], bestDist [M]);
        Fuse's return value is ``(bestDist <= 50).sum()``; see include/orb_b200.h: orbm_fuse_search."""
        k = [_c(kf_kps, KP_DTYPE), _c(kf_desc, np.uint8), _c(scale_factors, np.float32), _c(inv_level_sigma2, np.float32)]
        m = [_c(state, np.uint8), _c(xyz, np.float32), _c(normal, np.float32), _c(min_d, np.float32), _c(max_d, np.float32), _c(mp_desc, np.uint8)]
        o = [_c(Tcw7, np.float32), _c(Ow, np.float32), _c(cam4, np.float32)]
        fr = _OrbmFrame(len(k[0]), k[0].ctypes.data, k[1].ctypes.data, *[float(b) for b in bounds], k[2].ctypes.data, len(k[2]))
        pt = _OrbmFusePoints(len(m[0]), *[a.ctypes.data for a in m])
        bi = np.zeros(len(m[0]), np.int32); bd = np.zeros(len(m[0]), np.int32)
        L = lib()
        rc = L.orbm_fuse_search(self._h, C.byref(fr), _ptr(k[3]), float(log_scale_factor), _ptr(o[0]), _ptr(o[1]), _ptr(o[2]), C.byref(pt), float(th), _ptr(bi), _ptr(bd))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbm_fuse_search')
        return bi, bd

    def FuseSearchSim3(self, kf_kps, kf_desc, bounds, scale_factors, log_scale_factor, Tcw7, Ow, cam4, state, xyz, normal, min_d, max_d, mp_desc, th=3.0):
        """The search of ``ORBmatcher::Fuse(pKF, Scw, vpPoints, th, vpReplacePoint)`` (src/ORBmatcher.cc:1340-1455): (bestIdx, bestDist)."""
        k = [_c(kf_kps, KP_DTYPE), _c(kf_desc, np.uint8), _c(scale_factors, np.float32)]
        m = [_c(state, np.uint8), _c(xyz, np.float32), _c(normal, np.float32), _c(min_d, np.float32), _c(max_d, np.float32), _c(mp_desc, np.uint8)]
        o = [_c(Tcw7, np.float32), _c(Ow, np.float32), _c(cam4, np.float32)]
        fr = _OrbmFrame(len(k[0]), k[0].ctypes.data, k[1].ctypes.data, *[float(b) for b in bounds], k[2].ctypes.data, len(k[2]))
        pt = _OrbmFusePoints(len(m[0]), *[a.ctypes.data for a in m])
        bi = np.zeros(len(m[0]), np.int32); bd = np.zeros(len(m[0]), np.int32)
        L = lib()
        rc = L.orbm_fuse_search_sim3(self._h, C.byref(fr), float(log_scale_factor), _ptr(o[0]), _ptr(o[1]), _ptr(o[2]), C.byref(pt), float(th), _ptr(bi), _ptr(bd))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbm_fuse_search_sim3')
        return bi, bd

    FUSE_ITEM_KEYS = ('kps', 'desc', 'bounds', 'sf', 'isg', 'log_sf', 'Tcw', 'Ow', 'cam', 'state', 'xyz', 'normal', 'min_d', 'max_d', 'mp_desc')

    def fuse_search_batch(self, items, th=3.0):
        """The searches of several ``ORBmatcher::Fuse(KeyFrame*, const vector<MapPoint*>&, th)`` calls in one launch (orbm_fuse_search_batch).
        Each item is a dict with the keys of ``FUSE_ITEM_KEYS`` (the arguments of :meth:`FuseSearch`) and optionally its own ``th``.  Returns
        [(bestIdx [M], bestDist [M])] in item order, each equal to :meth:`FuseSearch` of that item.  The items must not depend on each other's
        bookkeeping: at most one keyframe per map (see include/orb_b200.h)."""
        keep, out = [], []
        arr = (_OrbmFuseItem * max(len(items), 1))()
        for j, it in enumerate(items):
            k = [_c(it['kps'], KP_DTYPE), _c(it['desc'], np.uint8), _c(it['sf'], np.float32), _c(it['isg'], np.float32)]
            m = [_c(it[n], dt) for n, dt in (('state', np.uint8), ('xyz', np.float32), ('normal', np.float32), ('min_d', np.float32), ('max_d', np.float32),
                                             ('mp_desc', np.uint8))]
            M = len(m[0])
            bi = np.zeros(M, np.int32); bd = np.zeros(M, np.int32)
            keep.append(k + m); out.append((bi, bd))
            s = arr[j]
            s.KF = _OrbmFrame(len(k[0]), k[0].ctypes.data, k[1].ctypes.data, *[float(b) for b in it['bounds']], k[2].ctypes.data, len(k[2]))
            s.invLevelSigma2 = k[3].ctypes.data
            s.logScaleFactor = float(it['log_sf'])
            s.Tcw7[:] = [float(v) for v in np.asarray(it['Tcw'], np.float32)]
            s.Ow[:] = [float(v) for v in np.asarray(it['Ow'], np.float32)]
            s.cam[:] = [float(v) for v in np.asarray(it['cam'], np.float32)]
            s.th = float(it.get('th', th))
            s.pts = _OrbmFusePoints(M, *[a.ctypes.data for a in m])
            s.bestIdx, s.bestDist = bi.ctypes.data, bd.ctypes.data
        L = lib()
        rc = L.orbm_fuse_search_batch(self._h, len(items), arr)
        if rc != ORB_OK:
            raise OrbError(rc, 'orbm_fuse_search_batch')
        return out

    def SearchBySim3(self, kf1, kf2, bounds, scale_factors, log_scale_factor, cam4, pre12, th=7.5):
        """``int ORBmatcher::SearchBySim3(pKF1, pKF2, vpMatches12, S12, th)`` (src/ORBmatcher.cc:1457-1674).  kf = dict(kps, desc, state, pcam (the map points
        in the OTHER keyframe's camera frame), min_d, max_d, mp_desc).  Returns (nFound, match12)."""
        keep = []

        def side(kf):
            a = [_c(kf['kps'], KP_DTYPE), _c(kf['desc'], np.uint8), _c(scale_factors, np.float32), _c(kf['state'], np.uint8), _c(kf['pcam'], np.float32),
                 _c(kf['min_d'], np.float32), _c(kf['max_d'], np.float32), _c(kf['mp_desc'], np.uint8)]
            keep.append(a)
            fr = _OrbmFrame(len(a[0]), a[0].ctypes.data, a[1].ctypes.data, *[float(b) for b in bounds], a[2].ctypes.data, len(a[2]))
            pt = _OrbmFusePoints(len(a[3]), a[3].ctypes.data, a[4].ctypes.data, None, a[5].ctypes.data, a[6].ctypes.data, a[7].ctypes.data)
            return fr, pt
        f1, p1 = side(kf1); f2, p2 = side(kf2)
        cam = _c(cam4, np.float32); pre = _c(pre12, np.int32)
        m12 = np.zeros(f1.K, np.int32); n = C.c_int(0)
        L = lib()
        rc = L.orbm_search_by_sim3(self._h, C.byref(f1), C.byref(p1), C.byref(f2), C.byref(p2), float(log_scale_factor), _ptr(cam), float(th), _ptr(pre), _ptr(m12), C.byref(n))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbm_search_by_sim3')
        return n.value, m12

    def SearchByBoWKF(self, k1, d1, point1, fv1, k2, d2, point2, fv2):
        """``int ORBmatcher::SearchByBoW(KeyFrame*, KeyFrame*, vector<MapPoint*>&)`` (src/ORBmatcher.cc:765-905): (nmatches, match12 [N1] = KF2 feature or -1)."""
        keep = [_c(k1, KP_DTYPE), _c(d1, np.uint8), _c(fv1[0], np.int32), _c(fv1[1], np.int32), _c(k2, KP_DTYPE), _c(d2, np.uint8),
                _c(fv2[0], np.int32), _c(fv2[1], np.int32), _c(point1, np.uint8), _c(point2, np.uint8)]
        a = _OrbmBowFrame(len(keep[0]), keep[0].ctypes.data, keep[1].ctypes.data, len(keep[2]), keep[2].ctypes.data, keep[3].ctypes.data)
        b = _OrbmBowFrame(len(keep[4]), keep[4].ctypes.data, keep[5].ctypes.data, len(keep[6]), keep[6].ctypes.data, keep[7].ctypes.data)
        m12 = np.full(len(keep[0]), -1, np.int32)
        n = C.c_int(0)
        L = lib()
        rc = L.orbm_search_by_bow_kf(self._h, C.byref(a), _ptr(keep[8]), C.byref(b), _ptr(keep[9]), self.mfNNratio, int(self.mbCheckOrientation), _ptr(m12), C.byref(n))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbm_search_by_bow_kf')
        return n.value, m12

    def common_regions_bow_batch(self, queries):
        """``LoopClosing::DetectCommonRegionsFromBoW`` up to the Sim3Solver for several place-recognition queries in two launches
        (orbm_common_regions_bow_batch): per candidate its status (CR_*), vpCovKFi, SearchByBoW's count per entry, numBoWMatches and the merged
        vpKeyFrameMatchedMP (as j) / vpMatchedPoints (as point index).  Each query is a dict as :func:`common_regions_struct` takes it.  The
        searches use the reference's ``ORBmatcher(0.9, true)``, not this matcher's settings.  Returns one dict of arrays per query (the
        header's output names)."""
        built = [common_regions_struct(q) for q in queries]
        arr = (OrbmCommonRegionsQuery * max(len(queries), 1))(*[b[0] for b in built])
        rc = lib().orbm_common_regions_bow_batch(self._h, len(queries), arr)
        if rc != ORB_OK:
            raise OrbError(rc, 'orbm_common_regions_bow_batch')
        return [b[1] for b in built]

    @staticmethod
    def _tri_frame(kf, keep):
        """OrbmTriFrame of keyframe dict ``kf`` (kps, desc, has_mp, fv=(nodes, features)); its arrays are appended to ``keep``."""
        a = [_c(kf['kps'], KP_DTYPE), _c(kf['desc'], np.uint8), _c(kf['has_mp'], np.uint8), _c(kf['fv'][0], np.int32), _c(kf['fv'][1], np.int32)]
        keep.append(a)
        return OrbmTriFrame(len(a[0]), a[0].ctypes.data, a[1].ctypes.data, a[2].ctypes.data, len(a[3]), a[3].ctypes.data, a[4].ctypes.data)

    def SearchForTriangulation(self, kf1, kf2_list, scale_factors, level_sigma2, ep, F12, coarse=False):
        """``int ORBmatcher::SearchForTriangulation(pKF1, pKF2, vMatchedPairs, false, bCoarse)`` (src/ORBmatcher.cc:907-1146) for one keyframe against
        several neighbours.  A keyframe is a dict(kps, desc, has_mp, fv=(nodes, features)); ep [n, 2], F12 [n, 9].  Returns (nmatches [n], matches12 [n, N1])."""
        keep = []
        f1 = self._tri_frame(kf1, keep)
        n2 = len(kf2_list)
        f2 = (OrbmTriFrame * max(n2, 1))(*[self._tri_frame(k, keep) for k in kf2_list])
        sf, sg = _c(scale_factors, np.float32), _c(level_sigma2, np.float32)
        epa, Fa = _c(ep, np.float32).reshape(-1, 2), _c(F12, np.float32).reshape(-1, 9)
        m12 = np.full((n2, f1.N), -1, np.int32); nm = np.zeros(n2, np.int32)
        L = lib()
        rc = L.orbm_search_for_triangulation(self._h, C.byref(f1), n2, f2, _ptr(sf), _ptr(sg), len(sf), _ptr(epa), _ptr(Fa), int(coarse), int(self.mbCheckOrientation),
                                             _ptr(m12), _ptr(nm))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbm_search_for_triangulation')
        return nm, m12

    def CreateNewMapPoints(self, kf1, kf2_list, scale_factors, level_sigma2, ep, F12, Tcw, Ow, cam, scale_factor, coarse=False, inertial=False,
                           th_far_points=0.0):
        """``LocalMapping::CreateNewMapPoints`` (src/LocalMapping.cc, the vpNeighKFs loop from :296; monocular keyframes) after the neighbour
        selection: the new map points of keyframe ``kf1`` triangulated against the neighbours ``kf2_list`` (in vpNeighKFs order), exactly as
        the reference's loop creates them.  Keyframes as in :meth:`SearchForTriangulation`; ``Tcw`` [1 + n, 3, 4] (KF1 first), ``Ow`` [1 + n, 3],
        ``cam`` [1 + n, 4]; ``th_far_points`` 0 = off.  Returns (records, nmatches [n], ncreated [n]): ``records`` is a ``NEW_POINT_DTYPE``
        array in creation order.  The matcher's own settings are not used: the reference builds ``ORBmatcher(0.6f, false)`` here."""
        keep = []
        inp = self._new_points_in(kf1, kf2_list, scale_factors, level_sigma2, ep, F12, Tcw, Ow, cam, scale_factor, coarse, inertial, th_far_points, keep)
        out, nm, nc = self._new_points_out(inp)
        n = C.c_int(0)
        L = lib()
        rc = L.orbm_create_new_map_points(self._h, C.byref(inp), _ptr(out), C.byref(n), _ptr(nm), _ptr(nc))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbm_create_new_map_points')
        return out[:n.value].copy(), nm, nc

    def create_new_map_points_batch(self, items):
        """:meth:`CreateNewMapPoints` for several new keyframes in one call of 3 launches (orbm_create_new_map_points_batch).  Each item is a
        dict of :meth:`CreateNewMapPoints`' arguments by name (``kf1``, ``kf2_list``, ``scale_factors``, ... ; ``coarse``, ``inertial`` and
        ``th_far_points`` optional).  Returns [(records, nmatches, ncreated)] in item order, each byte-identical to :meth:`CreateNewMapPoints`
        of that item.  At most one keyframe per map (see include/orb_b200.h)."""
        keep, res = [], []
        arr = (OrbmNewPointsItem * max(len(items), 1))()
        for j, it in enumerate(items):
            inp = self._new_points_in(it['kf1'], it['kf2_list'], it['scale_factors'], it['level_sigma2'], it['ep'], it['F12'], it['Tcw'], it['Ow'],
                                      it['cam'], it['scale_factor'], it.get('coarse', False), it.get('inertial', False), it.get('th_far_points', 0.0), keep)
            out, nm, nc = self._new_points_out(inp)
            n = np.zeros(1, np.int32)
            res.append((out, nm, nc, n))
            arr[j] = OrbmNewPointsItem(inp, out.ctypes.data, n.ctypes.data, nm.ctypes.data, nc.ctypes.data)
        L = lib()
        rc = L.orbm_create_new_map_points_batch(self._h, len(items), arr)
        if rc != ORB_OK:
            raise OrbError(rc, 'orbm_create_new_map_points_batch')
        return [(out[:n[0]].copy(), nm, nc) for out, nm, nc, n in res]

    def _new_points_in(self, kf1, kf2_list, scale_factors, level_sigma2, ep, F12, Tcw, Ow, cam, scale_factor, coarse, inertial, th_far_points, keep):
        """OrbmNewPointsIn of one CreateNewMapPoints call; every array it points to is appended to ``keep``."""
        f1 = self._tri_frame(kf1, keep)
        n2 = len(kf2_list)
        f2 = (OrbmTriFrame * max(n2, 1))(*[self._tri_frame(k, keep) for k in kf2_list])
        arrs = [_c(scale_factors, np.float32), _c(level_sigma2, np.float32), _c(ep, np.float32).reshape(-1, 2), _c(F12, np.float32).reshape(-1, 9),
                _c(Tcw, np.float32).reshape(-1, 12), _c(Ow, np.float32).reshape(-1, 3), _c(cam, np.float32).reshape(-1, 4)]
        assert len(arrs[4]) == len(arrs[5]) == len(arrs[6]) == n2 + 1 and len(arrs[2]) == len(arrs[3]) == n2
        f1p = C.pointer(f1)
        keep.append((f1p, f2, arrs))
        return OrbmNewPointsIn(f1p, n2, C.cast(f2, C.POINTER(OrbmTriFrame)), arrs[2].ctypes.data, arrs[3].ctypes.data, arrs[0].ctypes.data,
                               arrs[1].ctypes.data, len(arrs[0]), arrs[4].ctypes.data, arrs[5].ctypes.data, arrs[6].ctypes.data, float(scale_factor),
                               int(coarse), int(inertial), float(th_far_points))

    @staticmethod
    def _new_points_out(inp):
        """(records [max(KF1.N, 1)], nmatches [nKF2], ncreated [nKF2]) buffers for ``inp``."""
        return np.zeros(max(inp.KF1.contents.N, 1), NEW_POINT_DTYPE), np.zeros(inp.nKF2, np.int32), np.zeros(inp.nKF2, np.int32)

    def keyframe_culling_batch(self, maps):
        """``LocalMapping::KeyFrameCulling()`` (monocular and mono-inertial) for several maps in one launch (orbm_keyframe_culling_batch).
        Each map is a dict with the arrays of ``CULLING_ARRAYS`` (the keyframe table, the local keyframes and their slots in CSR form, the
        points and their observations in CSR form) and the scalars of ``CULLING_SCALARS``.  Returns, per map, dict(status [nLocal] (KFC_*),
        nMPs [nLocal], nRedundant [nLocal], visited); the caller replays the culls in ``status`` order (INTEGRATION.md §2).  The maps must
        share nothing (see include/orb_b200.h)."""
        built = [culling_struct(m) for m in maps]
        arr = (OrbmCullingMap * max(len(maps), 1))(*[b[0] for b in built])
        L = lib()
        rc = L.orbm_keyframe_culling_batch(self._h, len(maps), arr)
        if rc != ORB_OK:
            raise OrbError(rc, 'orbm_keyframe_culling_batch')
        return [dict(b[1], visited=int(b[1]['visited'][0])) for b in built]

    def update_connections_batch(self, items):
        """``LocalMapping::ProcessNewKeyFrame``'s map-point loop (mode UC_PROCESS_NEW_KEYFRAME) or the tail of ``SearchInNeighbors`` (mode
        UC_SEARCH_IN_NEIGHBORS), each followed by ``KeyFrame::UpdateConnections``, for several keyframes in one launch
        (orbm_update_connections_batch).  Each item is a dict with the arrays of ``CONNECTIONS_ARRAYS`` (the keyframe table, current keyframe
        first; its slots; the points and their observations in CSR form, key order) and the scalars of ``CONNECTIONS_SCALARS``.  Returns, per
        item, the outputs of :func:`connections_struct` with ``nConnected`` and ``parent`` as ints; the caller replays them on the host
        (INTEGRATION.md §2).  At most one keyframe per map, and the items share no keyframe or point (see include/orb_b200.h)."""
        built = [connections_struct(m) for m in items]
        arr = (OrbmConnectionsItem * max(len(items), 1))(*[b[0] for b in built])
        rc = lib().orbm_update_connections_batch(self._h, len(items), arr)
        if rc != ORB_OK:
            raise OrbError(rc, 'orbm_update_connections_batch')
        return [_connections_result(b[1]) for b in built]

    def update_local_map_batch(self, d, out=None):
        """``Tracking::UpdateLocalMap``'s UpdateLocalKeyFrames and UpdateLocalPoints for ``d['batch']`` streams in one launch
        (orbm_update_local_map_batch; host numpy).  ``d``: the batch dict of :func:`local_map_batch`.  Returns the outputs of
        :func:`local_map_outputs` (written into ``out`` when given): the local keyframes and points, and the local map in the slabs
        ``track_local_map_batch*`` takes (:func:`local_map_split` cuts them per stream).  The caller replays the marks, mpReferenceKF and the
        NULLing of the voting frame's bad points (INTEGRATION.md §2)."""
        out = local_map_outputs(d) if out is None else out
        keep = {n: _c(d[n], dt) for n, dt in LOCAL_MAP_ARRAYS if d.get(n) is not None}
        s, r = local_map_structs(d, out, lambda n: keep[n].ctypes.data if n in keep else None)
        rc = lib().orbm_update_local_map_batch(self._h, C.byref(s), C.byref(r))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbm_update_local_map_batch')
        return out

    def update_local_map_batch_device(self, d, out, stream=0):
        """Device form of :meth:`update_local_map_batch`: torch CUDA tensors in ``d`` (the sizes stay ints) and ``out`` (the keys of
        :func:`local_map_outputs`); enqueues on ``stream``."""
        s, r = local_map_structs(d, out, lambda n: d[n].data_ptr() if d.get(n) is not None else None)
        rc = lib().orbm_update_local_map_batch_device(self._h, C.byref(s), C.byref(r), C.c_void_p(stream))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbm_update_local_map_batch_device')

    def ComputeDistinctiveDescriptors(self, obs_list):
        """``MapPoint::ComputeDistinctiveDescriptors`` for a list of map points (each an [n, 32] u8 array of observed descriptors): index of the chosen row."""
        start = np.zeros(len(obs_list) + 1, np.int32)
        for i, o in enumerate(obs_list):
            start[i + 1] = start[i] + len(o)
        desc = np.concatenate([_c(o, np.uint8).reshape(-1, 32) for o in obs_list]) if start[-1] else np.zeros((0, 32), np.uint8)
        desc = np.ascontiguousarray(desc)
        best = np.zeros(len(obs_list), np.int32)
        L = lib()
        rc = L.orbm_distinctive_descriptors(self._h, len(obs_list), _ptr(start), _ptr(desc), _ptr(best))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbm_distinctive_descriptors')
        return best

    def knnMatch2(self, query, train):
        """cv::BFMatcher(NORM_HAMMING).knnMatch(query, train, k=2) (src/Frame.cc:1144): (idx[Q,2], dist[Q,2])."""
        q = _c(query, np.uint8).reshape(-1, 32)
        t = _c(train, np.uint8).reshape(-1, 32)
        idx = np.full((len(q), 2), -1, np.int32)
        dist = np.full((len(q), 2), -1, np.int32)
        rc = lib().orbm_bf_knn2(self._h, _ptr(q), len(q), _ptr(t), len(t), _ptr(idx), _ptr(dist))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbm_bf_knn2')
        return idx, dist

    def last_launch_count(self):
        return lib().orbm_last_launch_count(self._h)

    def last_cluster_size(self):
        """CTAs per frame of the last SearchByProjection / SearchForInitialization launch (1..8)."""
        return lib().orbm_last_cluster_size(self._h)


# =============================================================================================
# Optimizer (reference include/Optimizer.h:46-102)
# =============================================================================================
class _LbaProblem(C.Structure):
    _fields_ = [('nPoses', C.c_int), ('poses', C.c_void_p), ('poseFixed', C.c_void_p), ('cam', C.c_void_p),
                ('nPoints', C.c_int), ('points', C.c_void_p), ('nEdges', C.c_int), ('edgePoint', C.c_void_p),
                ('edgePose', C.c_void_p), ('obs', C.c_void_p), ('invSigma2', C.c_void_p), ('huberDelta', C.c_double),
                ('iterations', C.c_int), ('userLambdaInit', C.c_double), ('stopFlag', C.c_void_p)]


class _LbaResult(C.Structure):
    _fields_ = [('poses', C.c_void_p), ('points', C.c_void_p), ('edgeChi2', C.c_void_p), ('edgeDepthPositive', C.c_void_p),
                ('iterations', C.c_int), ('trials', C.c_int), ('lambda_', C.c_double), ('chi2', C.c_double),
                ('initialChi2', C.c_double), ('gpuLaunches', C.c_int)]


#: lba_local_bundle_adjustment_batch's map statuses and observation flags (LBA_LOCAL_*, LBA_OBS_*; include/orb_b200.h)
LBA_LOCAL_RAN, LBA_LOCAL_NO_FIXED, LBA_LOCAL_STOPPED = 0, 1, 2
LBA_OBS_NO_EDGE, LBA_OBS_KEPT, LBA_OBS_ERASED = 0, 1, 2
#: the input arrays of one LbaLocalMap, with their dtypes
LOCAL_BA_ARRAYS = (('mnId', np.uint64), ('kfFlags', np.uint8), ('pose7', np.float32), ('cameraCenter', np.float32), ('cam4', np.float32),
                   ('cov', np.int32), ('slotStart', np.int32), ('slotPoint', np.int32), ('pointId', np.uint64), ('pointFlags', np.uint8),
                   ('worldPos', np.float32), ('refKF', np.int32), ('obsStart', np.int32), ('obsKF', np.int32), ('obsIdx', np.int32),
                   ('obsPt', np.float32), ('obsOctave', np.int32), ('invLevelSigma2', np.float32), ('scaleFactors', np.float32))
#: its outputs: (name, dtype, rows, row shape); rows 'kf' = [nKF], 'pt' = [nPoints], 'obs' = [obsStart[-1]], or a fixed count
LOCAL_BA_OUTPUTS = (('counts', np.int32, 4, ()), ('nLists', np.int32, 3, ()), ('localKF', np.int32, 'kf', ()), ('fixedKF', np.int32, 'kf', ()),
                    ('localPoint', np.int32, 'pt', ()), ('obsFlag', np.uint8, 'obs', ()), ('kfPose7', np.float32, 'kf', (7,)),
                    ('kfCenter', np.float32, 'kf', (3,)), ('pointPos', np.float32, 'pt', (3,)), ('pointBad', np.uint8, 'pt', ()),
                    ('pointRefKF', np.int32, 'pt', ()), ('normal', np.float32, 'pt', (3,)), ('minDistance', np.float32, 'pt', ()),
                    ('maxDistance', np.float32, 'pt', ()), ('lmStats', np.float64, 5, ()))
#: the optional outputs (the solver's own results)
LOCAL_BA_DEBUG = (('optPose', np.float64, 'kf', (7,)), ('optPoint', np.float64, 'pt', (3,)), ('edgeChi2', np.float64, 'obs', ()),
                  ('edgeDepthPositive', np.uint8, 'obs', ()))


class LbaLocalMap(C.Structure):
    """One map of lba_local_bundle_adjustment_batch (include/orb_b200.h)."""
    _fields_ = [('nKF', C.c_int)] + [(n, C.c_void_p) for n in ('mnId', 'kfFlags', 'pose7', 'cameraCenter', 'cam4')] + [('nCov', C.c_int)] + \
               [(n, C.c_void_p) for n in ('cov', 'slotStart', 'slotPoint')] + [('nPoints', C.c_int)] + \
               [(n, C.c_void_p) for n in ('pointId', 'pointFlags', 'worldPos', 'refKF', 'obsStart', 'obsKF', 'obsIdx', 'obsPt', 'obsOctave')] + \
               [('nlevels', C.c_int), ('invLevelSigma2', C.c_void_p), ('scaleFactors', C.c_void_p), ('inertial', C.c_int), ('stopFlag', C.c_void_p),
                ('status', C.c_void_p)] + [(n, C.c_void_p) for n, _, _, _ in LOCAL_BA_OUTPUTS] + \
               [(n, C.c_void_p) for n, _, _, _ in LOCAL_BA_DEBUG]


def local_ba_struct(m, debug=False, given=None):
    """LbaLocalMap over map dict `m` (keys LOCAL_BA_ARRAYS, 'inertial' and optionally 'stop' = a one-byte uint8 array) with fresh outputs:
    (struct, out dict, arrays to keep alive).  debug: also the optional outputs.  given: a dict of LOCAL_BA_DEBUG arrays to point them at
    instead (the CPU oracle reads them as the optimiser's results)."""
    a = {n: _c(m[n] if m.get(n) is not None else np.zeros(0), dt) for n, dt in LOCAL_BA_ARRAYS}
    nK, nP, nC = len(a['kfFlags']), len(a['pointFlags']), len(a['cov'])
    nO = int(a['obsStart'][-1]) if nP else 0
    rows = dict(kf=nK, pt=nP, obs=nO)
    out = {n: np.zeros((r if isinstance(r, int) else rows[r],) + sh, dt) for n, dt, r, sh in LOCAL_BA_OUTPUTS}
    out['status'] = np.zeros(1, np.int32)
    if given is not None:
        out.update({n: _c(given[n], dt) for n, dt, _, _ in LOCAL_BA_DEBUG})
    elif debug:
        out.update({n: np.zeros((rows[r],) + sh, dt) for n, dt, r, sh in LOCAL_BA_DEBUG})
    stop = m.get('stop')
    s = LbaLocalMap(nK, *[_ptr(a[n]) for n in ('mnId', 'kfFlags', 'pose7', 'cameraCenter', 'cam4')], nC,
                    *[_ptr(a[n]) for n in ('cov', 'slotStart', 'slotPoint')], nP,
                    *[_ptr(a[n]) for n in ('pointId', 'pointFlags', 'worldPos', 'refKF', 'obsStart', 'obsKF', 'obsIdx', 'obsPt', 'obsOctave')],
                    len(a['scaleFactors']), _ptr(a['invLevelSigma2']), _ptr(a['scaleFactors']), int(m.get('inertial', 0)), _ptr(stop),
                    _ptr(out['status']), *[_ptr(out[n]) for n, _, _, _ in LOCAL_BA_OUTPUTS], *[_ptr(out.get(n)) for n, _, _, _ in LOCAL_BA_DEBUG])
    a['stop'] = stop
    return s, out, a


def local_ba_result(out):
    """The output dict with the scalars unpacked and the lists cut to their lengths."""
    nLoc, nFix, nPt = (int(v) for v in out['nLists'])
    r = dict(out, status=int(out['status'][0]), num_fixedKF=int(out['counts'][0]), num_OptKF=int(out['counts'][1]), num_MPs=int(out['counts'][2]),
             num_edges=int(out['counts'][3]))
    r['localKF'], r['fixedKF'], r['localPoint'] = out['localKF'][:nLoc].copy(), out['fixedKF'][:nFix].copy(), out['localPoint'][:nPt].copy()
    for n in ('kfPose7', 'kfCenter', 'optPose'):
        if n in r:
            r[n] = out[n][:nLoc].copy()
    for n in ('pointPos', 'pointBad', 'pointRefKF', 'normal', 'minDistance', 'maxDistance', 'optPoint'):
        if n in r:
            r[n] = out[n][:nPt].copy()
    return r


class Optimizer:
    """Mirror of the static ``ORB_SLAM3::Optimizer`` functions on the hot path.  ``LocalBundleAdjustment`` runs the numeric core
    on flat arrays (``synth.lba_problem`` has the layout) and returns what the write-back / outlier test reads, the caller keeping the
    pointer-graph walk (src/Optimizer.cc:1125-1403); ``local_bundle_adjustment_batch`` runs the whole function, walk, erase cascade and
    write-back included, from flattened maps and returns the record the caller replays."""

    def __init__(self, max_poses=64, max_points=8192, max_edges=65536, max_batch=1, device=0):
        L = lib()
        self._h = C.c_void_p()
        rc = L.lba_create_batch(C.byref(self._h), max_poses, max_points, max_edges, max_batch, device)
        if rc != ORB_OK:
            self._h = None
            raise OrbError(rc, 'lba_create')

    def close(self):
        if getattr(self, '_h', None):
            lib().lba_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:      # interpreter shutdown: module globals may already be gone
            pass

    @staticmethod
    def _pack(prob, iterations, user_lambda_init, stop_flag):
        keep = dict(poses=_c(prob['poses'], np.float64), fixed=_c(prob['fixed'], np.uint8), cam=_c(prob['cam'], np.float32),
                    points=_c(prob['points'], np.float64), ep=_c(prob['edge_point'], np.int32), ek=_c(prob['edge_pose'], np.int32),
                    obs=_c(prob['obs'], np.float64), isg=_c(prob['inv_sigma2'], np.float32))
        nP, nL, nE = len(keep['poses']), len(keep['points']), len(keep['ep'])
        p = _LbaProblem(nP, _ptr(keep['poses']), _ptr(keep['fixed']), _ptr(keep['cam']), nL, _ptr(keep['points']), nE, _ptr(keep['ep']),
                        _ptr(keep['ek']), _ptr(keep['obs']), _ptr(keep['isg']), float(prob['huber_delta']), iterations, user_lambda_init,
                        _ptr(stop_flag) if stop_flag is not None else None)
        out = dict(poses=np.zeros((nP, 7)), points=np.zeros((nL, 3)), chi2=np.zeros(nE), depth_pos=np.zeros(nE, np.uint8))
        r = _LbaResult(_ptr(out['poses']), _ptr(out['points']), _ptr(out['chi2']), _ptr(out['depth_pos']))
        return keep, p, out, r

    @staticmethod
    def _finish(out, r):
        out.update(iters=r.iterations, trials=r.trials, lambda_=r.lambda_, final_chi2=r.chi2, initial_chi2=r.initialChi2, launches=r.gpuLaunches)
        return out

    def LocalBundleAdjustmentBatch(self, probs, iterations=10, user_lambda_init=0.0):
        """One LocalBundleAdjustment per stream / local map, all solved by one kernel launch."""
        packs = [self._pack(p, iterations, user_lambda_init, None) for p in probs]
        P = (_LbaProblem * len(probs))(*[k[1] for k in packs])
        R = (_LbaResult * len(probs))(*[k[3] for k in packs])
        rc = lib().lba_solve_batch(self._h, len(probs), P, R)
        if rc != ORB_OK:
            raise OrbError(rc, 'lba_solve_batch')
        return [self._finish(k[2], R[i]) for i, k in enumerate(packs)]

    def upload(self, probs, iterations=10, user_lambda_init=0.0):
        self._packs = [self._pack(p, iterations, user_lambda_init, None) for p in probs]
        P = (_LbaProblem * len(probs))(*[k[1] for k in self._packs])
        rc = lib().lba_upload_batch(self._h, len(probs), P)
        if rc != ORB_OK:
            raise OrbError(rc, 'lba_upload_batch')

    def run_device(self, stream=0):
        rc = lib().lba_run_batch_device(self._h, C.c_void_p(stream))
        if rc != ORB_OK:
            raise OrbError(rc, 'lba_run_batch_device')

    def download(self):
        R = (_LbaResult * len(self._packs))(*[k[3] for k in self._packs])
        rc = lib().lba_download_batch(self._h, len(self._packs), R)
        if rc != ORB_OK:
            raise OrbError(rc, 'lba_download_batch')
        return [self._finish(k[2], R[i]) for i, k in enumerate(self._packs)]

    def last_cluster_size(self):
        return lib().lba_last_cluster_size(self._h)

    def set_cluster_size(self, ctas):
        rc = lib().lba_set_cluster_size(self._h, ctas)
        if rc != ORB_OK:
            raise OrbError(rc, 'lba_set_cluster_size')

    def last_helpers(self):
        return lib().lba_last_helpers(self._h)

    def set_helpers(self, clusters):
        rc = lib().lba_set_helpers(self._h, clusters)
        if rc != ORB_OK:
            raise OrbError(rc, 'lba_set_helpers')

    def local_bundle_adjustment_batch(self, maps, debug=False):
        """``Optimizer::LocalBundleAdjustment`` as a whole -- walk, solve, erase cascade, write-back -- for one map per item (dicts as
        ``local_ba_struct`` reads them), in one call.  Returns one ``local_ba_result`` dict per map; debug adds the solver's own results."""
        packs = [local_ba_struct(m, debug=debug) for m in maps]
        arr = (LbaLocalMap * max(1, len(maps)))(*[p[0] for p in packs])
        rc = lib().lba_local_bundle_adjustment_batch(self._h, len(maps), arr)
        if rc != ORB_OK:
            raise OrbError(rc, 'lba_local_bundle_adjustment_batch')
        return [local_ba_result(p[1]) for p in packs]

    def local_last_launches(self):
        return lib().lba_local_last_launches(self._h)

    @staticmethod
    def local_inertial_ba_map_batch(maps, debug=False, device=0):
        """``Optimizer::LocalInertialBA`` as a whole -- window walk, solve, erase cascade, write-back -- for one map per item (dicts as
        ``liba_map_struct`` reads them), in one call on `device`; like ``LocalInertialBA`` it needs no handle.  Returns one
        ``liba_map_result`` dict per map; debug adds the solver's own results."""
        packs = [liba_map_struct(m, debug=debug) for m in maps]
        arr = (LocalInertialBAMap * max(1, len(maps)))(*[p[0] for p in packs])
        rc = lib().local_inertial_ba_map_batch(len(maps), arr, device)
        if rc != ORB_OK:
            raise OrbError(rc, 'local_inertial_ba_map_batch')
        return [liba_map_result(p[1]) for p in packs]

    @staticmethod
    def local_inertial_ba_map_last_launches():
        """Launches of this thread's last local_inertial_ba_map_batch call."""
        return lib().local_inertial_ba_map_last_launches()

    def LocalBundleAdjustment(self, prob, iterations=10, user_lambda_init=0.0, stop_flag=None):
        keep = dict(poses=_c(prob['poses'], np.float64), fixed=_c(prob['fixed'], np.uint8), cam=_c(prob['cam'], np.float32),
                    points=_c(prob['points'], np.float64), ep=_c(prob['edge_point'], np.int32), ek=_c(prob['edge_pose'], np.int32),
                    obs=_c(prob['obs'], np.float64), isg=_c(prob['inv_sigma2'], np.float32))
        nP, nL, nE = len(keep['poses']), len(keep['points']), len(keep['ep'])
        p = _LbaProblem(nP, _ptr(keep['poses']), _ptr(keep['fixed']), _ptr(keep['cam']), nL, _ptr(keep['points']), nE, _ptr(keep['ep']),
                        _ptr(keep['ek']), _ptr(keep['obs']), _ptr(keep['isg']), float(prob['huber_delta']), iterations, user_lambda_init,
                        _ptr(stop_flag) if stop_flag is not None else None)
        out = dict(poses=np.zeros((nP, 7)), points=np.zeros((nL, 3)), chi2=np.zeros(nE), depth_pos=np.zeros(nE, np.uint8))
        r = _LbaResult(_ptr(out['poses']), _ptr(out['points']), _ptr(out['chi2']), _ptr(out['depth_pos']))
        rc = lib().lba_solve(self._h, C.byref(p), C.byref(r))
        if rc != ORB_OK:
            raise OrbError(rc, 'lba_solve')
        out.update(iters=r.iterations, trials=r.trials, lambda_=r.lambda_, final_chi2=r.chi2, initial_chi2=r.initialChi2, launches=r.gpuLaunches)
        return out


def PoseOptimization(frames, device=0):
    """``Optimizer::PoseOptimization`` for a list of frames (dicts: pose [7], cam [4], Xw [N,3], obs [N,2], inv_sigma2 [N]).
    Returns a list of dicts(pose, outlier, inliers)."""
    count = len(frames)
    cap = max(1, max(len(f['obs']) for f in frames))
    N = np.array([len(f['obs']) for f in frames], np.int32)
    pose = np.stack([_c(f['pose'], np.float64) for f in frames])
    cam = np.stack([_c(f['cam'], np.float32) for f in frames])
    Xw = np.zeros((count, cap, 3)); obs = np.zeros((count, cap, 2)); isg = np.ones((count, cap), np.float32)
    for i, f in enumerate(frames):
        Xw[i, :N[i]] = f['Xw']; obs[i, :N[i]] = f['obs']; isg[i, :N[i]] = f['inv_sigma2']
    out_pose = np.zeros((count, 7)); outl = np.zeros((count, cap), np.uint8); ninl = np.zeros(count, np.int32)
    L = lib()
    rc = L.pose_optimization_batch(count, cap, _ptr(N), _ptr(pose), _ptr(cam), _ptr(Xw), _ptr(obs), _ptr(isg),
                                   float(np.float32(np.sqrt(5.991))), _ptr(out_pose), _ptr(outl), _ptr(ninl), device)
    if rc != ORB_OK:
        raise OrbError(rc, 'pose_optimization_batch')
    return [dict(pose=out_pose[i], outlier=outl[i, :N[i]].copy(), inliers=int(ninl[i])) for i in range(count)]


# =============================================================================================
# Inertial edges (reference src/G2oTypes.cc, src/ImuTypes.cc; SURVEY.md 8f rank 1)
# =============================================================================================
IMU_PREINT_FLOATS = 292


class _ImuMonoEdges(C.Structure):
    _fields_ = [('nPoses', C.c_int), ('poses', C.c_void_p), ('extrinsics', C.c_void_p), ('cam', C.c_void_p), ('nPoints', C.c_int), ('points', C.c_void_p),
                ('nEdges', C.c_int), ('edgePoint', C.c_void_p), ('edgePose', C.c_void_p), ('obs', C.c_void_p), ('invSigma2', C.c_void_p), ('huberDelta', C.c_double)]


def imu_preintegrate(acc, gyr, dt, n_meas, bias6, noise4, device=0):
    """``IMU::Preintegrated`` of `count` intervals: acc / gyr [count, maxMeas, 3], dt [count, maxMeas], n_meas [count], bias6 [count, 6]."""
    acc = _c(acc, np.float32); gyr = _c(gyr, np.float32); dt = _c(dt, np.float32); n = _c(n_meas, np.int32); b = _c(bias6, np.float32); nz = _c(noise4, np.float32)
    count, mm = dt.shape
    out = np.zeros((count, IMU_PREINT_FLOATS), np.float32)
    L = lib()
    rc = L.imu_preintegrate_batch(count, _ptr(n), mm, _ptr(acc), _ptr(gyr), _ptr(dt), _ptr(b), _ptr(nz), _ptr(out), device)
    if rc != ORB_OK:
        raise OrbError(rc, 'imu_preintegrate_batch')
    return out


def imu_information(preint, device=0):
    P = _c(preint, np.float32).reshape(-1, IMU_PREINT_FLOATS)
    n = len(P)
    info = np.zeros((n, 9, 9)); ig = np.zeros((n, 3, 3)); ia = np.zeros((n, 3, 3))
    L = lib()
    rc = L.imu_information_batch(n, _ptr(P), _ptr(info), _ptr(ig), _ptr(ia), device)
    if rc != ORB_OK:
        raise OrbError(rc, 'imu_information_batch')
    return info, ig, ia


def imu_inertial_edges(preint, states36, info9=None, huber_delta=0.0, jac=True, device=0):
    """``EdgeInertial::computeError`` / ``linearizeOplus`` for n edges.  Returns dict(err [n,9], J [n,9,24] | None, chi2, rho)."""
    P = _c(preint, np.float32).reshape(-1, IMU_PREINT_FLOATS); S = _c(states36, np.float64).reshape(-1, 36)
    n = len(S)
    err = np.zeros((n, 9)); J = np.zeros((n, 9, 24)) if jac else None
    info = _c(info9, np.float64) if info9 is not None else None
    chi2 = np.zeros(n); rho = np.zeros(n)
    L = lib()
    rc = L.imu_inertial_edges(n, _ptr(P), _ptr(S), _ptr(info), float(huber_delta), _ptr(err), _ptr(J), _ptr(chi2), _ptr(rho), device)
    if rc != ORB_OK:
        raise OrbError(rc, 'imu_inertial_edges')
    return dict(err=err, J=J, chi2=chi2 if info is not None else None, rho=rho if info is not None else None)


def imu_mono_edges(poses12, extrinsics24, cam, points, edge_point, edge_pose, obs, inv_sigma2, huber_delta=0.0, jac=True, device=0):
    """``EdgeMono`` over ``ImuCamPose`` vertices.  Returns dict(err [n,2], Jpoint [n,2,3], Jpose [n,2,6], chi2, rho, depth_pos)."""
    po = _c(poses12, np.float64).reshape(-1, 12); ex = _c(extrinsics24, np.float64).reshape(24); cm = _c(cam, np.float32).reshape(-1, 4)
    pt = _c(points, np.float64).reshape(-1, 3); ep = _c(edge_point, np.int32); ek = _c(edge_pose, np.int32); ob = _c(obs, np.float64).reshape(-1, 2)
    isg = _c(inv_sigma2, np.float32)
    n = len(ep)
    s = _ImuMonoEdges(len(po), po.ctypes.data, ex.ctypes.data, cm.ctypes.data, len(pt), pt.ctypes.data, n, ep.ctypes.data, ek.ctypes.data, ob.ctypes.data,
                      isg.ctypes.data, float(huber_delta))
    err = np.zeros((n, 2)); Jp = np.zeros((n, 2, 3)) if jac else None; Jx = np.zeros((n, 2, 6)) if jac else None
    chi2 = np.zeros(n); rho = np.zeros(n); dp = np.zeros(n, np.uint8)
    L = lib()
    rc = L.imu_mono_edges(C.byref(s), _ptr(err), _ptr(Jp), _ptr(Jx), _ptr(chi2), _ptr(rho), _ptr(dp), device)
    if rc != ORB_OK:
        raise OrbError(rc, 'imu_mono_edges')
    return dict(err=err, Jpoint=Jp, Jpose=Jx, chi2=chi2, rho=rho, depth_pos=dp)


def PoseInertialOptimizationLastKeyFrame(frames, extrinsics24, rec_init=False, device=0):
    """``int Optimizer::PoseInertialOptimizationLastKeyFrame(Frame*, bool bRecInit)`` (src/Optimizer.cc:4491-4873) for a list of frames, one CTA each.
    frame = dict(Xw [N,3], obs [N,2], inv_sigma2 [N], track_depth [N], cam [4], preint [IMU_PREINT_FLOATS], kf_state [21], state [21]).
    Returns a list of dict(state [21], outlier [N], H [15,15], ret)."""
    n = len(frames)
    cap = max(1, max(len(f['Xw']) for f in frames))
    N = np.array([len(f['Xw']) for f in frames], np.int32)
    Xw = np.zeros((n, cap, 3), np.float32); ob = np.zeros((n, cap, 2), np.float32); isg = np.zeros((n, cap), np.float32); td = np.zeros((n, cap), np.float32)
    for i, f in enumerate(frames):
        Xw[i, :N[i]] = f['Xw']; ob[i, :N[i]] = f['obs']; isg[i, :N[i]] = f['inv_sigma2']; td[i, :N[i]] = f['track_depth']
    cam = np.stack([_c(f['cam'], np.float32) for f in frames]); P = np.stack([_c(f['preint'], np.float32) for f in frames])
    kf = np.stack([_c(f['kf_state'], np.float64) for f in frames]); st = np.stack([_c(f['state'], np.float64) for f in frames]).copy()
    ex = _c(extrinsics24, np.float64)
    out = np.zeros((n, cap), np.uint8); H = np.zeros((n, 15, 15)); ret = np.zeros(n, np.int32)
    L = lib()
    rc = L.pose_inertial_optimization_last_kf_batch(n, cap, _ptr(N), _ptr(Xw), _ptr(ob), _ptr(isg), _ptr(td), _ptr(cam), _ptr(ex), _ptr(P), _ptr(kf), _ptr(st), int(rec_init),
                                                    _ptr(out), _ptr(H), _ptr(ret), device)
    if rc != ORB_OK:
        raise OrbError(rc, 'pose_inertial_optimization_last_kf_batch')
    return [dict(state=st[i], outlier=out[i, :N[i]], H=H[i], ret=int(ret[i])) for i in range(n)]


def PoseInertialOptimizationLastFrame(frames, extrinsics24, rec_init=False, device=0):
    """``int Optimizer::PoseInertialOptimizationLastFrame(Frame*, bool bRecInit)`` (src/Optimizer.cc:4875-5289) for a list of frames.
    frame = dict(Xw, obs, inv_sigma2, track_depth, cam, preint_frame, preint_kf, prior_state [21], prior_H [15,15], prev_state [21], state [21]).
    Returns a list of dict(state, prev_state, outlier, H [15,15], ret)."""
    n = len(frames)
    cap = max(1, max(len(f['Xw']) for f in frames))
    N = np.array([len(f['Xw']) for f in frames], np.int32)
    Xw = np.zeros((n, cap, 3), np.float32); ob = np.zeros((n, cap, 2), np.float32); isg = np.zeros((n, cap), np.float32); td = np.zeros((n, cap), np.float32)
    for i, f in enumerate(frames):
        Xw[i, :N[i]] = f['Xw']; ob[i, :N[i]] = f['obs']; isg[i, :N[i]] = f['inv_sigma2']; td[i, :N[i]] = f['track_depth']
    st64 = lambda k: np.stack([_c(f[k], np.float64).reshape(-1) for f in frames]).copy()
    cam = np.stack([_c(f['cam'], np.float32) for f in frames]); Pf = np.stack([_c(f['preint_frame'], np.float32) for f in frames]); Pk = np.stack([_c(f['preint_kf'], np.float32) for f in frames])
    prior, pH, pv, st = st64('prior_state'), st64('prior_H'), st64('prev_state'), st64('state')
    ex = _c(extrinsics24, np.float64)
    out = np.zeros((n, cap), np.uint8); H = np.zeros((n, 15, 15)); ret = np.zeros(n, np.int32)
    L = lib()
    rc = L.pose_inertial_optimization_last_frame_batch(n, cap, _ptr(N), _ptr(Xw), _ptr(ob), _ptr(isg), _ptr(td), _ptr(cam), _ptr(ex), _ptr(Pf), _ptr(Pk), _ptr(prior), _ptr(pH),
                                                       _ptr(pv), _ptr(st), int(rec_init), _ptr(out), _ptr(H), _ptr(ret), device)
    if rc != ORB_OK:
        raise OrbError(rc, 'pose_inertial_optimization_last_frame_batch')
    return [dict(state=st[i], prev_state=pv[i], outlier=out[i, :N[i]], H=H[i], ret=int(ret[i])) for i in range(n)]


# =============================================================================================
# DBoW2 vocabulary transform (reference Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h; SURVEY.md 8f rank 3)
# =============================================================================================
class _LocalInertialBAProblem(C.Structure):
    _fields_ = [('nKF', C.c_int32), ('nOpt', C.c_int32), ('kfState21', C.c_void_p), ('kfTcw12', C.c_void_p), ('cam4', C.c_void_p), ('extrinsics24', C.c_void_p),
                ('nInertial', C.c_int32), ('ieKf1', C.c_void_p), ('ieKf2', C.c_void_p), ('preint', C.c_void_p), ('ieRobust', C.c_void_p), ('ieInfoScale', C.c_void_p),
                ('nPoints', C.c_int32), ('points3', C.c_void_p), ('trackDepth', C.c_void_p),
                ('nEdges', C.c_int32), ('edgePoint', C.c_void_p), ('edgeKf', C.c_void_p), ('obs2', C.c_void_p), ('invSigma2', C.c_void_p),
                ('iterations', C.c_int32), ('bLarge', C.c_int32), ('lambdaInit', C.c_double)]


class _LocalInertialBAResult(C.Structure):
    _fields_ = [('kfState21', C.c_void_p), ('kfTcw12', C.c_void_p), ('points3', C.c_void_p), ('erase', C.c_void_p), ('edgeChi2', C.c_void_p), ('stats8', C.c_void_p), ('profile8', C.c_void_p)]


def _liba_marshal(probs):
    """ctypes arrays of LocalInertialBAProblem / LocalInertialBAResult for a list of problem dicts (synth.local_inertial_ba_problem layout + 'preint')."""
    n = len(probs)
    P = (_LocalInertialBAProblem * n)(); R = (_LocalInertialBAResult * n)()
    keep, outs = [], []
    for i, pr in enumerate(probs):
        a = dict(st=_c(pr['state'], np.float64), tc=_c(pr['tcw'], np.float64), cam=_c(pr['cam'], np.float32), ex=_c(pr['extr'], np.float64),
                 k1=_c(pr['ie_kf1'], np.int32), k2=_c(pr['ie_kf2'], np.int32), pre=_c(pr['preint'], np.float32), rob=_c(pr['ie_robust'], np.uint8),
                 sc=_c(pr['ie_info_scale'], np.float64), pts=_c(pr['points'], np.float64), td=_c(pr['track_depth'], np.float32), ep=_c(pr['e_pt'], np.int32),
                 ek=_c(pr['e_kf'], np.int32), ob=_c(pr['obs'], np.float64), isg=_c(pr['inv_sigma2'], np.float32))
        nE = len(a['ep'])
        o = dict(state=np.zeros_like(a['st']), tcw=np.zeros_like(a['tc']), points=np.zeros_like(a['pts']), erase=np.zeros(nE, np.uint8), chi2=np.zeros(nE), stats=np.zeros(8), prof=np.zeros(8))
        P[i] = _LocalInertialBAProblem(int(pr['n_kf']), int(pr['n_opt']), a['st'].ctypes.data, a['tc'].ctypes.data, a['cam'].ctypes.data, a['ex'].ctypes.data, len(a['k1']), a['k1'].ctypes.data, a['k2'].ctypes.data,
                                       a['pre'].ctypes.data, a['rob'].ctypes.data, a['sc'].ctypes.data, len(a['pts']), a['pts'].ctypes.data, a['td'].ctypes.data, nE, a['ep'].ctypes.data, a['ek'].ctypes.data,
                                       a['ob'].ctypes.data, a['isg'].ctypes.data, int(pr['iterations']), int(bool(pr['large'])), float(pr['lambda_init']))
        R[i] = _LocalInertialBAResult(o['state'].ctypes.data, o['tcw'].ctypes.data, o['points'].ctypes.data, o['erase'].ctypes.data, o['chi2'].ctypes.data, o['stats'].ctypes.data, o['prof'].ctypes.data)
        keep.append(a); outs.append(o)
    return P, R, keep, outs


def _liba_finish(outs, iters):
    return [dict(state=o['state'], tcw=o['tcw'], points=o['points'], erase=o['erase'], chi2=o['chi2'], iters=int(iters[i]), err=float(o['stats'][0]),
                 err_end=float(o['stats'][1]), failed=bool(o['stats'][2]), lam=float(o['stats'][3]), trials=int(o['stats'][4]), kernel_ms=float(o['stats'][6]) * 1e-6, phase_ms=o['prof'] * 1e-6)
            for i, o in enumerate(outs)]


def LocalInertialBA(probs, device=0):
    """``void Optimizer::LocalInertialBA(KeyFrame*, bool*, Map*, int&, int&, int&, int&, bool bLarge, bool bRecInit)`` (src/Optimizer.cc:2383-2958): the
    numeric core for a list of local maps, one persistent CTA each (``local_inertial_ba_batch``).  A problem is the dict of
    ``synth.local_inertial_ba_problem`` plus ``preint`` [nI, IMU_PREINT_FLOATS]: n_kf, n_opt, state [nKF,21], tcw [nKF,12], cam [nKF,4], extr [24], ie_kf1 / ie_kf2 /
    ie_robust / ie_info_scale [nI], points [nL,3], track_depth [nL], e_pt / e_kf / obs / inv_sigma2 [nE], iterations, lambda_init, large.
    Returns a list of dict(state, tcw, points, erase, chi2, iters, err, err_end, failed, lam, trials)."""
    P, R, keep, outs = _liba_marshal(probs)
    iters = np.zeros(len(probs), np.int32)
    L = lib()
    rc = L.local_inertial_ba_batch(len(probs), C.cast(P, C.c_void_p), C.cast(R, C.c_void_p), _ptr(iters), device)
    if rc != ORB_OK:
        raise OrbError(rc, 'local_inertial_ba_batch')
    return _liba_finish(outs, iters)


#: local_inertial_ba_map_batch's keyframe flags (besides KF_BAD / KF_OTHER_MAP) and map statuses (include/orb_b200.h)
KF_IMU, KF_PREINT = 16, 32
LIBA_LOCAL_RAN, LIBA_LOCAL_FAILED = 0, 1
#: the input arrays of one LocalInertialBAMap, with their dtypes
LIBA_MAP_ARRAYS = (('kfFlags', np.uint8), ('prevKF', np.int32), ('state21', np.float32), ('tcw12', np.float32), ('cameraCenter', np.float32),
                   ('cam4', np.float32), ('preint', np.float32), ('extrinsics24', np.float64), ('slotStart', np.int32), ('slotPoint', np.int32),
                   ('pointFlags', np.uint8), ('worldPos', np.float32), ('trackDepth', np.float32), ('refKF', np.int32), ('obsStart', np.int32),
                   ('obsKF', np.int32), ('obsIdx', np.int32), ('obsPt', np.float32), ('obsOctave', np.int32), ('invLevelSigma2', np.float32),
                   ('scaleFactors', np.float32))
#: its outputs: (name, dtype, rows, row shape); rows 'kf' = [nKF], 'pt' = [nPoints], 'obs' = [obsStart[-1]], or a fixed count
LIBA_MAP_OUTPUTS = (('nLists', np.int32, 4, ()), ('optKF', np.int32, 'kf', ()), ('fixedKF', np.int32, 'kf', ()), ('localPoint', np.int32, 'pt', ()),
                    ('ieLinked', np.uint8, 'kf', ()), ('obsFlag', np.uint8, 'obs', ()), ('kfPose7', np.float32, 'kf', (7,)),
                    ('kfCenter', np.float32, 'kf', (3,)), ('kfVelocity', np.float32, 'kf', (3,)), ('kfBias6', np.float32, 'kf', (6,)),
                    ('pointPos', np.float32, 'pt', (3,)), ('pointBad', np.uint8, 'pt', ()), ('pointRefKF', np.int32, 'pt', ()),
                    ('normal', np.float32, 'pt', (3,)), ('minDistance', np.float32, 'pt', ()), ('maxDistance', np.float32, 'pt', ()),
                    ('stats8', np.float64, 8, ()))
#: the optional outputs (the solver's own results)
LIBA_MAP_DEBUG = (('optState21', np.float64, 'kf', (21,)), ('optTcw12', np.float64, 'kf', (12,)), ('optPoint', np.float64, 'pt', (3,)),
                  ('edgeChi2', np.float64, 'obs', ()))


class LocalInertialBAMap(C.Structure):
    """One map of local_inertial_ba_map_batch (include/orb_b200.h)."""
    _fields_ = [('nKF', C.c_int32)] + [(n, C.c_void_p) for n, _ in LIBA_MAP_ARRAYS[:10]] + [('nPoints', C.c_int32)] + \
               [(n, C.c_void_p) for n, _ in LIBA_MAP_ARRAYS[10:19]] + [('nlevels', C.c_int32)] + [(n, C.c_void_p) for n, _ in LIBA_MAP_ARRAYS[19:]] + \
               [('keyFramesInMap', C.c_int32), ('bLarge', C.c_int32), ('bRecInit', C.c_int32), ('status', C.c_void_p)] + \
               [(n, C.c_void_p) for n, _, _, _ in LIBA_MAP_OUTPUTS + LIBA_MAP_DEBUG]


def liba_map_struct(m, debug=False, given=None):
    """LocalInertialBAMap over map dict `m` (keys LIBA_MAP_ARRAYS, 'keyFramesInMap', 'bLarge', 'bRecInit') with fresh outputs: (struct, out
    dict, arrays to keep alive).  debug: also the optional outputs.  given: a dict of LIBA_MAP_DEBUG arrays and 'stats8' to point them at
    instead (the CPU oracle finishes from them)."""
    a = {n: _c(m[n] if m.get(n) is not None else np.zeros(0), dt) for n, dt in LIBA_MAP_ARRAYS}
    nK, nP = len(a['kfFlags']), len(a['pointFlags'])
    nO = int(a['obsStart'][-1]) if nP else 0
    rows = dict(kf=nK, pt=nP, obs=nO)
    out = {n: np.zeros((r if isinstance(r, int) else rows[r],) + sh, dt) for n, dt, r, sh in LIBA_MAP_OUTPUTS}
    out['status'] = np.zeros(1, np.int32)
    if given is not None:
        out.update({n: _c(given[n], dt).copy() for n, dt, _, _ in LIBA_MAP_DEBUG + (('stats8', np.float64, 8, ()),)})
    elif debug:
        out.update({n: np.zeros((rows[r],) + sh, dt) for n, dt, r, sh in LIBA_MAP_DEBUG})
    p = lambda n: _ptr(a[n])
    s = LocalInertialBAMap(nK, *[p(n) for n, _ in LIBA_MAP_ARRAYS[:10]], nP, *[p(n) for n, _ in LIBA_MAP_ARRAYS[10:19]], len(a['scaleFactors']),
                           *[p(n) for n, _ in LIBA_MAP_ARRAYS[19:]], int(m['keyFramesInMap']), int(m.get('bLarge', 0)), int(m.get('bRecInit', 0)),
                           _ptr(out['status']), *[_ptr(out.get(n)) for n, _, _, _ in LIBA_MAP_OUTPUTS + LIBA_MAP_DEBUG])
    return s, out, a


def liba_map_result(out):
    """The output dict with the status unpacked and the lists cut to their lengths."""
    N, nFix, nPt, nE = (int(v) for v in out['nLists'])
    r = dict(out, status=int(out['status'][0]), num_OptKF=N, num_fixedKF=nFix, num_MPs=nPt, num_edges=nE)
    r['optKF'], r['fixedKF'], r['localPoint'], r['ieLinked'] = out['optKF'][:N].copy(), out['fixedKF'][:nFix].copy(), out['localPoint'][:nPt].copy(), \
        out['ieLinked'][:N].copy()
    for n in ('kfPose7', 'kfCenter', 'kfVelocity', 'kfBias6'):
        r[n] = out[n][:N].copy()
    for n in ('optState21', 'optTcw12'):
        if n in r:
            r[n] = out[n][:N + nFix].copy()
    for n in ('pointPos', 'pointBad', 'pointRefKF', 'normal', 'minDistance', 'maxDistance', 'optPoint'):
        if n in r:
            r[n] = out[n][:nPt].copy()
    return r


class _OrbVocabulary(C.Structure):
    _fields_ = [('nNodes', C.c_int), ('L', C.c_int), ('weighting', C.c_int), ('norm', C.c_int), ('childStart', C.c_void_p), ('children', C.c_void_p),
                ('descriptors', C.c_void_p), ('weight', C.c_void_p), ('wordId', C.c_void_p)]


class ORBVocabulary:
    """Mirror of ``ORB_SLAM3::ORBVocabulary`` (= ``DBoW2::TemplatedVocabulary<FORB::TDescriptor, FORB>``) for ``transform``: the tree is
    given as flat arrays (child_start, children, desc, weight, word_id) and stays on the device."""

    def __init__(self, L, child_start, children, desc, weight, word_id, weighting=0, norm=1, device=0):
        self._keep = [_c(child_start, np.int32), _c(children, np.int32), _c(desc, np.uint8), _c(weight, np.float64), _c(word_id, np.int32)]
        self.n_words = int((self._keep[4] >= 0).sum())     # mpVoc->size()
        s = _OrbVocabulary(len(self._keep[4]), int(L), int(weighting), int(norm), *[a.ctypes.data for a in self._keep])
        self._h = C.c_void_p()
        rc = lib().orbv_create(C.byref(self._h), C.byref(s), device)
        if rc != ORB_OK:
            self._h = None
            raise OrbError(rc, 'orbv_create')

    def close(self):
        if getattr(self, '_h', None):
            lib().orbv_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def transform(self, desc_list, levelsup=4):
        """``transform(features, BowVector, FeatureVector, levelsup)`` for a list of frames (each [n, 32] u8).  Returns per frame
        (word_id [w] i32, word_value [w] f64, fv_node [e] i32, fv_feature [e] i32) in the reference's std::map order."""
        B = len(desc_list)
        cap = max(1, max(len(d) for d in desc_list))
        desc = np.zeros((B, cap, 32), np.uint8); n = np.zeros(B, np.int32)
        for b, d in enumerate(desc_list):
            n[b] = len(d); desc[b, :len(d)] = d
        wid = np.zeros((B, cap), np.int32); wv = np.zeros((B, cap)); nw = np.zeros(B, np.int32)
        fn = np.zeros((B, cap), np.int32); ff = np.zeros((B, cap), np.int32); ne = np.zeros(B, np.int32)
        L = lib()
        rc = L.orbv_transform_batch(self._h, B, _ptr(desc), _ptr(n), cap, int(levelsup), _ptr(wid), _ptr(wv), _ptr(nw), _ptr(fn), _ptr(ff), _ptr(ne))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbv_transform_batch')
        return [(wid[b, :nw[b]].copy(), wv[b, :nw[b]].copy(), fn[b, :ne[b]].copy(), ff[b, :ne[b]].copy()) for b in range(B)]

    def transform_device(self, d_desc, d_n, levelsup, scratch, out, stream=0):
        """Device form of :meth:`transform` (orbv_transform_batch_device) on torch CUDA tensors: d_desc [B, cap, 32] u8, d_n [B] i32;
        ``scratch`` = (word i32, weight f64, node i32), each [B, cap]; ``out`` = (word_id [B, cap] i32, word_value [B, cap] f64,
        n_words [B] i32, fv_node [B, cap] i32, fv_feature [B, cap] i32, n_entries [B] i32), rows laid out as :meth:`transform` returns
        them.  Enqueues on ``stream`` and returns immediately."""
        import torch
        if len(scratch) != 3 or len(out) != 6:
            raise ValueError('transform_device: scratch takes 3 tensors and out 6')
        B, cap = d_desc.shape[0], d_desc.shape[1]
        want = [(d_desc, torch.uint8, (B, cap, 32)), (d_n, torch.int32, (B,))] + \
            [(t, dt, (B, cap)) for t, dt in zip(scratch, (torch.int32, torch.float64, torch.int32))] + \
            [(t, dt, sh) for t, dt, sh in zip(out, (torch.int32, torch.float64, torch.int32, torch.int32, torch.int32, torch.int32),
                                              ((B, cap), (B, cap), (B,), (B, cap), (B, cap), (B,)))]
        for k, (t, dt, sh) in enumerate(want):
            if not t.is_cuda or t.dtype != dt or tuple(t.shape) != sh or not t.is_contiguous():
                raise ValueError('transform_device: operand %d must be a contiguous CUDA %s tensor of shape %s' % (k, dt, sh))
        rc = lib().orbv_transform_batch_device(self._h, B, _ptr(d_desc), _ptr(d_n), cap, int(levelsup), *[_ptr(t) for t in scratch],
                                               *[_ptr(t) for t in out], C.c_void_p(stream))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbv_transform_batch_device')


#: OrbvDbQuery's kinds (ORBV_DB_*, include/orb_b200.h)
DB_RELOC, DB_NBEST = 0, 1


class OrbvDbQuery(C.Structure):
    """One query of orbv_db_query_batch (include/orb_b200.h)."""
    _fields_ = [('dbIndex', C.c_int32), ('kind', C.c_int32), ('nWords', C.c_int32), ('wordId', C.c_void_p), ('wordValue', C.c_void_p),
                ('nConnected', C.c_int32), ('connected', C.c_void_p), ('cap', C.c_int32)] + \
               [(n, C.c_void_p) for n in ('key', 'words', 'scored', 'score', 'nSharing', 'maxCommonWords')]


def db_query_struct(q, cap):
    """OrbvDbQuery over query dict `q` (db, kind, word_id, word_value, connected = keys or None) with fresh outputs of width `cap`:
    (struct, out dict, arrays to keep alive)."""
    wid, wv = _c(q['word_id'], np.int32), _c(q['word_value'], np.float64)
    conn = _c(q['connected'] if q.get('connected') is not None else np.zeros(0), np.uint64)
    out = dict(key=np.zeros(cap, np.uint64), words=np.zeros(cap, np.int32), scored=np.zeros(cap, np.uint8), score=np.zeros(cap, np.float32),
               nSharing=np.zeros(1, np.int32), maxCommonWords=np.zeros(1, np.int32))
    s = OrbvDbQuery(int(q['db']), int(q['kind']), len(wid), _ptr(wid), _ptr(wv), len(conn), _ptr(conn), cap,
                    *[_ptr(out[n]) for n in ('key', 'words', 'scored', 'score', 'nSharing', 'maxCommonWords')])
    return s, out, (wid, wv, conn)


class KeyFrameDatabase:
    """Mirror of ``ORB_SLAM3::KeyFrameDatabase`` over keys: the inverted file on the device (orbv_db_*), ``maxDatabases`` databases in one
    handle.  ``voc`` is the vocabulary's word count (``mpVoc->size()``) or an :class:`ORBVocabulary`.  A BowVector is (word ids ascending,
    values), as :meth:`ORBVocabulary.transform` returns it.  :meth:`query_batch` runs phase 1 of ``DetectRelocalizationCandidates`` /
    ``DetectNBestCandidates``; phase 2 stays with the caller (INTEGRATION.md §2)."""

    def __init__(self, voc, max_databases=1, max_keyframes=1024, max_words=2048, device=0):
        words = voc.n_words if isinstance(voc, ORBVocabulary) else int(voc)
        self.max_keyframes = int(max_keyframes)
        self._h = C.c_void_p()
        rc = lib().orbv_db_create(C.byref(self._h), words, int(max_databases), self.max_keyframes, int(max_words), device)
        if rc != ORB_OK:
            self._h = None
            raise OrbError(rc, 'orbv_db_create')

    def close(self):
        if getattr(self, '_h', None):
            lib().orbv_db_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def add(self, db, keys, bows):
        """``add(pKF)`` for each keyframe in order: ``db`` an index or one per key, ``keys`` uint64, ``bows`` [(word ids, values)]."""
        keys = _c(keys, np.uint64)
        dbs = _c(np.broadcast_to(np.asarray(db, np.int32), keys.shape), np.int32)
        start = np.zeros(len(keys) + 1, np.int32)
        start[1:] = np.cumsum([len(b[0]) for b in bows]) if len(bows) else []
        wid = _c(np.concatenate([np.asarray(b[0], np.int32) for b in bows]) if len(bows) else np.zeros(0), np.int32)
        wv = _c(np.concatenate([np.asarray(b[1], np.float64) for b in bows]) if len(bows) else np.zeros(0), np.float64)
        rc = lib().orbv_db_add_batch(self._h, len(keys), _ptr(dbs), _ptr(keys), _ptr(start), _ptr(wid), _ptr(wv))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbv_db_add_batch')

    def erase(self, db, keys):
        """``erase(pKF)`` for each key (absent keys are no-ops); ``clearMap(pMap)`` is this with the map's keyframes."""
        keys = _c(keys, np.uint64)
        dbs = _c(np.broadcast_to(np.asarray(db, np.int32), keys.shape), np.int32)
        rc = lib().orbv_db_erase_batch(self._h, len(keys), _ptr(dbs), _ptr(keys))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbv_db_erase_batch')

    def clear(self, db=0):
        rc = lib().orbv_db_clear(self._h, int(db))
        if rc != ORB_OK:
            raise OrbError(rc, 'orbv_db_clear')

    def size(self, db=0):
        n = lib().orbv_db_size(self._h, int(db))
        if n < 0:
            raise OrbError(n, 'orbv_db_size')
        return n

    def last_launch_count(self):
        return lib().orbv_db_last_launch_count(self._h)

    def query_batch(self, queries, cap=None):
        """Phase 1 of every query in one call (orbv_db_query_batch).  Each query is a dict(db, kind = DB_RELOC or DB_NBEST, word_id,
        word_value, connected = the keys of GetConnectedKeyFrames() for DB_NBEST).  Returns per query dict(key, words, scored, score) in
        lKFsSharingWords order, nSharing and maxCommonWords.  ``cap`` defaults to max_keyframes (never exceeded)."""
        cap = self.max_keyframes if cap is None else int(cap)
        built = [db_query_struct(q, cap) for q in queries]
        arr = (OrbvDbQuery * max(len(built), 1))(*[b[0] for b in built])
        rc = lib().orbv_db_query_batch(self._h, len(built), arr)
        if rc != ORB_OK:
            raise OrbError(rc, 'orbv_db_query_batch')
        res = []
        for _, out, _ in built:
            n = int(out['nSharing'][0])
            r = {k: out[k][:n].copy() for k in ('key', 'words', 'scored', 'score')}
            r.update(nSharing=n, maxCommonWords=int(out['maxCommonWords'][0]))
            res.append(r)
        return res
