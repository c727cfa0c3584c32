/* orb_b200.h -- C-ABI of the H100-native ORB-SLAM3 hot path (liborb_b200.so).
 *
 * Drop-in boundary for three class surfaces of lturing/ORB_SLAM3_modified (SURVEY.md 8b):
 *   ORBextractor::operator()            include/ORBextractor.h:56-58,  src/ORBextractor.cc:1086
 *   ORBmatcher::SearchByProjection x2,  include/ORBmatcher.h:47-52,    src/ORBmatcher.cc:43,1676
 *   ORBmatcher::DescriptorDistance,     include/ORBmatcher.h:43,       src/ORBmatcher.cc:2058
 *   cv::BFMatcher(NORM_HAMMING).knnMatch(k=2) as used at src/Frame.cc:1144
 *   Optimizer::LocalBundleAdjustment    include/Optimizer.h:71,        src/Optimizer.cc:1116
 *   Optimizer::PoseOptimization         include/Optimizer.h:62,        src/Optimizer.cc:814
 *
 * Conventions: extern "C", plain pointers and sizes, caller-owned output buffers with a capacity
 * and a returned count, int status (0 = ok, <0 = error enum below), no exceptions cross the
 * boundary, one call at a time per handle (the reference's extractor is stateful in the same way,
 * SURVEY.md 8b "Ownership").  Functions suffixed _device take device pointers and a cudaStream_t
 * (passed as void*), enqueue work and return without synchronising; all others take host pointers
 * and return when the results are in the caller's buffers.
 * There is no CPU fallback: every entry point fails with ORB_ERR_CUDA when no sm_90 device exists.
 */
#ifndef ORB_B200_H
#define ORB_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum {
    ORB_OK = 0,
    ORB_ERR_EMPTY = -1,     /* empty image: ORBextractor::operator() returns -1 (src/ORBextractor.cc:1090) */
    ORB_ERR_ARG = -2,       /* bad argument (null pointer, size out of the configured range, ...) */
    ORB_ERR_CAPACITY = -3,  /* caller buffer or an internal slab too small; nothing was truncated silently */
    ORB_ERR_CUDA = -4,      /* CUDA runtime failure or no usable device; see orb_last_error() */
    ORB_ERR_ASPECT = -5     /* bordered aspect ratio < 0.5: the reference divides by zero (src/ORBextractor.cc:559-561) */
};

/* Byte-compatible with cv::KeyPoint (28 bytes): pt.x, pt.y, size, angle, response, octave, class_id. */
typedef struct OrbKeyPoint {
    float x, y;
    float size;
    float angle;
    float response;
    int32_t octave;
    int32_t class_id;
} OrbKeyPoint;

const char* orb_last_error(void);
/* Library/ABI version and the SM architecture the kernels were compiled for (100). */
int orb_abi_version(void);
int orb_compiled_sm(void);

/* ------------------------------------------------------------------------------------------
 * ORBextractor (reference include/ORBextractor.h:43-109)
 * ------------------------------------------------------------------------------------------ */
typedef struct orbx_handle orbx_handle;

/* ORBextractor::ORBextractor(nfeatures, scaleFactor, nlevels, iniThFAST, minThFAST)
 * (src/ORBextractor.cc:409-469) plus the device-side sizing: the largest image and the number
 * of frames one batched call may carry. */
int orbx_create(orbx_handle** out, int nfeatures, float scaleFactor, int nlevels, int iniThFAST, int minThFAST,
                int max_width, int max_height, int max_batch, int device);
void orbx_destroy(orbx_handle* h);

/* GetLevels / GetScaleFactor(s) / GetInverseScaleFactors / GetScaleSigmaSquares /
 * GetInverseScaleSigmaSquares (include/ORBextractor.h:60-82) + mnFeaturesPerLevel. Arrays hold nlevels entries. */
int orbx_get_levels(const orbx_handle* h);
int orbx_get_tables(const orbx_handle* h, float* scaleFactors, float* invScaleFactors, float* levelSigma2,
                    float* invLevelSigma2, int* featuresPerLevel);
/* Upper bound of keypoints one frame can return (sum over levels of N_l + 3, SURVEY.md 7.1). */
int orbx_max_keypoints(const orbx_handle* h);

/* int ORBextractor::operator()(image, mask [ignored], keypoints, descriptors, vLappingArea)
 * image: CV_8UC1, rows x cols, `step` bytes between rows (host memory).
 * keypoints[cap], descriptors[cap*32]; *nkeypoints receives K; returns in *monoIndex what the
 * reference returns (the count of keypoints outside [lap0, lap1], filled from the front; the others
 * are filled from the back, src/ORBextractor.cc:1120-1164).  Status ORB_ERR_EMPTY mirrors `return -1`. */
int orbx_extract(orbx_handle* h, const uint8_t* image, int rows, int cols, size_t step, int lap0, int lap1,
                 OrbKeyPoint* keypoints, uint8_t* descriptors, int cap, int* nkeypoints, int* monoIndex);

/* The same call for `batch` independent frames (one per stream), host buffers.
 * images: batch frames, `frame_stride` bytes apart.  keypoints: batch x cap, descriptors: batch x cap x 32,
 * nkeypoints/monoIndex: batch entries. */
int orbx_extract_batch(orbx_handle* h, const uint8_t* images, int batch, int rows, int cols, size_t step,
                       size_t frame_stride, int lap0, int lap1, OrbKeyPoint* keypoints, uint8_t* descriptors,
                       int cap, int* nkeypoints, int* monoIndex);

/* Device-resident variant: every pointer is a device pointer, work is enqueued on `stream`
 * (cudaStream_t) and the call returns without synchronising.  Slabs have fixed capacity `cap`
 * per frame so that they can be all-gathered as-is (SURVEY.md 8e).
 * Capacity: a frame with K > cap keypoints gets no rows at all (its keypoint and descriptor rows
 * keep what they held); d_nkeypoints[f] still receives K and d_monoIndex[f] the monoIndex, so
 * d_nkeypoints[f] > cap is how the caller sees the overflow.  The other frames are written as usual
 * and the call itself returns ORB_OK. */
int orbx_extract_batch_device(orbx_handle* h, const uint8_t* d_images, int batch, int rows, int cols, size_t step,
                              size_t frame_stride, int lap0, int lap1, OrbKeyPoint* d_keypoints,
                              uint8_t* d_descriptors, int cap, int* d_nkeypoints, int* d_monoIndex, void* stream);

/* The host-buffer calls above also leave their results in the handle's device slabs ([batch][cap] keypoints, [batch][cap][32]
 * descriptors, [batch] counts, cap = orbx_max_keypoints()).  These pointers stay valid until the next call on the handle, so a
 * matcher call that follows (orbm_search_last_frame_batch_resident) does not have to ship the current frame back to the device. */
int orbx_resident_slabs(const orbx_handle* h, const OrbKeyPoint** d_keypoints, const uint8_t** d_descriptors, const int** d_nkeypoints,
                        int* cap);

/* void Frame::ComputeStereoMatches() (reference src/Frame.cc:811-982), the stereo consumer of ORBextractor::mvImagePyramid
 * (src/Frame.cc:122-125 runs two extractors on the left / right image, then :126 calls this): for every left keypoint the best right
 * keypoint on its row band by Hamming distance, an 11 x 11 SAD refinement over 11 shifts on the two pyramids, parabola fit, and the
 * 1.5 * 1.4 * median SAD outlier cut.  `left` and `right` must have extracted the pair's images in their last call (`batch` pairs, pair f =
 * frame f of both); mb / mbf as in Frame.  uRight / depth [batch][cap] receive mvuRight / mvDepth (-1 = no match).
 * Host form: keypoints come from both handles' resident slabs (last call = orbx_extract[_batch]); cap = orbx_max_keypoints(left). */
int orbx_stereo_matches(orbx_handle* left, orbx_handle* right, int batch, float mb, float mbf, float* uRight, float* depth, int cap);
/* Device form: keypoint / descriptor / count slabs as written by orbx_extract_batch_device of the two handles; enqueues on `stream`
 * (the stream both extractions were enqueued on, or one that waits for them). */
int orbx_stereo_matches_device(orbx_handle* left, orbx_handle* right, int batch, const OrbKeyPoint* d_kpsL, const uint8_t* d_descL, const int* d_nL,
                               int capL, const OrbKeyPoint* d_kpsR, const uint8_t* d_descR, const int* d_nR, int capR, float mb, float mbf,
                               float* d_uRight, float* d_depth, void* stream);
/* mvImagePyramid[level] of frame `frame` of the last call including the reflected frame of `border` pixels (19 in the reference,
 * src/ORBextractor.cc:1185-1191) that ComputePyramid keeps around every level: (w + 2 border) x (h + 2 border) bytes, tightly packed. */
int orbx_copy_level_bordered(orbx_handle* h, int frame, int level, int border, uint8_t* dst);

/* Debug/inspection taps used by the parity tests (mvImagePyramid is a public member of the reference class,
 * include/ORBextractor.h:84).  Copies level `level` of frame `frame` of the last call, unbordered, tightly packed.
 * Level 0 unblurred is read from the plane the last call read: after orbx_extract_batch_device with 16-byte aligned frames that
 * is the caller's own device frames, which must then still hold the images; `frame` must be below that call's batch. */
int orbx_get_level_size(const orbx_handle* h, int level, int* width, int* height);
int orbx_copy_level(orbx_handle* h, int frame, int level, int blurred, uint8_t* dst);
/* FAST candidates of one level of the last call as (x, y, score) int triples in the order the reference
 * feeds them to DistributeOctTree (src/ORBextractor.cc:863-871). Returns the count or <0. */
int orbx_copy_candidates(orbx_handle* h, int frame, int level, int* xys, int cap);
/* Number of kernels launched by the last extract call (for bench.py's gpu_launches). */
int orbx_last_launch_count(const orbx_handle* h);
/* Per-kernel device times of the pipeline (the reference's REGISTER_TIMES analogue, include/Settings.h:24): with profiling on,
 * CUDA events bracket each stage on the launching stream (the blur then runs in line instead of on its forked stream).
 * ms6 = pyramid, blur, FAST cells, quadtree, assemble, orientation + BRIEF of the last profiled call. */
int orbx_set_profiling(orbx_handle* h, int on);
int orbx_get_stage_ms(orbx_handle* h, float* ms6);

/* Frame::UndistortKeyPoints (reference src/Frame.cc:747) and Frame::ComputeImageBounds (called at src/Frame.cc:793) for a pinhole camera
 * with lens distortion (mK, mDistCoef).  A 4-coefficient calibration (k1 k2 p1 p2) passes k3 = 0, which OpenCV treats identically. */
typedef struct OrbPinholeCamera {
    float fx, fy, cx, cy;
    float k1, k2, p1, p2, k3;
} OrbPinholeCamera;
/* mvKeysUn from mvKeys for `batch` frames: d_kps / d_kpsUn are [batch][cap] device slabs (as orbx_extract_batch_device writes them),
 * d_n the [batch] counts.  Rows [0, n[f]) of frame f become copies of mvKeys[i] with pt replaced by cv::undistortPoints(pt, K, mDistCoef,
 * cv::Mat(), K), bit for bit; size, angle, response, octave and class_id are kept.  With k1 == 0 (either sign) the rows are copied byte for
 * byte, as the reference's `if(mDistCoef.at<float>(0)==0.0)` does whatever k2, p1, p2 and k3 are.  Rows past n[f], and every row of a frame
 * with n[f] > cap (the extractor's overflow), are not touched.  d_kpsUn must not overlap d_kps: the stereo matcher and the last-frame search
 * (OrbmLastFrame.octave) still read mvKeys.  Enqueues ONE launch on `stream` (none for batch == 0) and returns without synchronising.
 * ORB_ERR_ARG before any launch: a null pointer, batch < 0, cap < 1, overlapping slabs, fx or fy zero, a non-finite camera member. */
int orbx_undistort_keypoints_device(orbx_handle* h, const OrbPinholeCamera* cam, int batch, const OrbKeyPoint* d_kps, const int* d_n, int cap,
                                    OrbKeyPoint* d_kpsUn, void* stream);
/* The same for the frames of the handle's last orbx_extract / orbx_extract_batch call (its resident slabs, orbx_resident_slabs): mvKeysUn
 * goes to a second [max_batch][orbx_max_keypoints] slab the handle owns (allocated on first use), whose device address *d_kpsUn receives
 * when d_kpsUn is not NULL -- the `kps` to give the matchers' _resident forms.  It stays valid until the handle is destroyed and is
 * rewritten by the next call.  When kpsUn is not NULL it receives that slab's [batch][cap] rows (cap must equal orbx_max_keypoints; rows
 * at or past n[f] are unspecified).  Synchronises.  ORB_ERR_ARG before any launch: the errors of the device form, or a last call that was
 * not a host-buffer extraction of at least `batch` frames. */
int orbx_undistort_keypoints(orbx_handle* h, const OrbPinholeCamera* cam, int batch, OrbKeyPoint* kpsUn, int cap, const OrbKeyPoint** d_kpsUn);
/* mnMinX, mnMaxX, mnMinY, mnMaxY of a cols x rows image into bounds4, computed on `device` with the same device function from the four
 * undistorted corners (0, cols, 0, rows when k1 == 0).  ONE launch; host pointers.  ORB_ERR_ARG: the camera errors above, cols or rows < 1,
 * a null pointer. */
int orbx_image_bounds(const OrbPinholeCamera* cam, int cols, int rows, float* bounds4, int device);
/* Launches of the calling thread's last orbx_undistort_keypoints[_device] or orbx_image_bounds call (0 after a refused call or an empty
 * batch).  orbx_last_launch_count() keeps counting extraction launches only. */
int orbx_undistort_last_launch_count(void);

/* ------------------------------------------------------------------------------------------
 * ORBmatcher (reference include/ORBmatcher.h:36-103): the per-frame projection matchers, the Hamming
 * primitive and the brute-force kNN used by the reference.  All inputs are flat arrays: the host shim
 * flattens Frame / MapPoint fields exactly as listed in SURVEY.md 8a' ("Matcher in").
 * ------------------------------------------------------------------------------------------ */
typedef struct orbm_handle orbm_handle;

/* Scratch for up to max_batch frames of max_keypoints keypoints matched against max_mappoints map points (both <= 65535).
 * One call in flight per handle: the per-frame scratch (candidate lists, queries) belongs to the handle, so two concurrent calls --
 * also on different streams -- need two handles (bench.py gives every stream group its own).  Device-side octave / level values
 * outside [0, nlevels) are clamped; the host entry points reject them. */
int orbm_create(orbm_handle** out, int max_batch, int max_keypoints, int max_mappoints, int device);
void orbm_destroy(orbm_handle* h);

/* Current frame as seen by the matchers (Frame::mvKeysUn, mDescriptors, image bounds mnMinX.., mvScaleFactors;
 * the 64x48 grid of Frame::AssignFeaturesToGrid, src/Frame.cc:385-416, is rebuilt on the device). */
typedef struct OrbmFrame {
    int K;                        /* number of keypoints */
    const OrbKeyPoint* keypoints; /* K */
    const uint8_t* descriptors;   /* K x 32 */
    float minX, minY, maxX, maxY; /* mnMinX, mnMinY, mnMaxX, mnMaxY */
    const float* scaleFactors;    /* mvScaleFactors, nlevels entries */
    int nlevels;
} OrbmFrame;

/* Map points for ORBmatcher::SearchByProjection(Frame&, const vector<MapPoint*>&, th, bFarPoints, thFarPoints)
 * (src/ORBmatcher.cc:43-213, mono branch): the tracking fields Frame::isInFrustum wrote (src/Frame.cc:563-571). */
typedef struct OrbmLocalPoints {
    int M;
    const uint8_t* inView;     /* mbTrackInView */
    const uint8_t* bad;        /* isBad() */
    const float* depth;        /* mTrackDepth */
    const float* projX;        /* mTrackProjX */
    const float* projY;        /* mTrackProjY */
    const int32_t* level;      /* mnTrackScaleLevel */
    const float* viewCos;      /* mTrackViewCos */
    const uint8_t* hasObs;     /* Observations() > 0 */
    const uint8_t* descriptors;/* GetDescriptor(), M x 32 */
} OrbmLocalPoints;

/* Last-frame map points for ORBmatcher::SearchByProjection(Frame&, const Frame&, th, bMono=true)
 * (src/ORBmatcher.cc:1676-1887): index i runs over LastFrame.N. */
typedef struct OrbmLastFrame {
    int M;
    const uint8_t* valid;      /* LastFrame.mvpMapPoints[i] != NULL && !LastFrame.mvbOutlier[i] */
    const float* xyz;          /* GetWorldPos(), M x 3 */
    const int32_t* octave;     /* LastFrame.mvKeys[i].octave */
    const float* angle;        /* LastFrame.mvKeysUn[i].angle */
    const uint8_t* hasObs;     /* Observations() > 0 */
    const uint8_t* descriptors;/* GetDescriptor(), M x 32 */
} OrbmLastFrame;

/* Both searches return the reference's `int nmatches` in *nmatches and update, per keypoint of the current frame,
 * match[K] (index of the assigned map point in the input arrays, -1 = none; the host re-attaches MapPoint*) and
 * claimed[K] (assigned point has Observations()>0: such keypoints are skipped by later candidates,
 * src/ORBmatcher.cc:84-86,1747-1749).  Both arrays are in/out (the reference reads Frame::mvpMapPoints). Host pointers. */
int orbm_search_local_map(orbm_handle* h, const OrbmFrame* frame, const OrbmLocalPoints* pts, float th, float nnratio,
                          int bFarPoints, float thFarPoints, int32_t* match, uint8_t* claimed, int* nmatches);
/* Tcw: unit quaternion (w,x,y,z) + translation (CurrentFrame.GetPose()); cam: fx, fy, cx, cy (Pinhole). */
int orbm_search_last_frame(orbm_handle* h, const OrbmFrame* frame, const OrbmLastFrame* last, const float* Tcw7,
                           const float* cam4, float th, int checkOrientation, int32_t* match, uint8_t* claimed,
                           int* nmatches);

/* Frame::isInFrustum (src/Frame.cc:512-574, monocular branch Nleft == -1) with MapPoint::PredictScale
 * (src/MapPoint.cc:531-546) for the M local map points of one frame: what Tracking::SearchLocalPoints
 * (src/Tracking.cc:3346) runs before the local-map SearchByProjection.  Host pointers. */
typedef struct OrbmFrustumIn {
    int M;
    const float* worldPos;        /* GetWorldPos(), M x 3 */
    const float* normal;          /* GetNormal(), M x 3 */
    const float* minDistInv;      /* GetMinDistanceInvariance() = 0.8f * mfMinDistance */
    const float* maxDistInv;      /* GetMaxDistanceInvariance() = 1.2f * mfMaxDistance */
    const float* maxDistance;     /* mfMaxDistance (PredictScale divides it by the current distance) */
    float Rcw[9], tcw[3], Ow[3];  /* mRcw (row-major), mtcw, mOw */
    float cam[4];                 /* fx fy cx cy (Pinhole::project) */
    float minX, minY, maxX, maxY; /* mnMinX ... mnMaxY */
    float mbf;                    /* for mTrackProjXR */
    float logScaleFactor;         /* Frame::mfLogScaleFactor */
    int nScaleLevels;             /* Frame::mnScaleLevels */
    float viewingCosLimit;        /* 0.5 in SearchLocalPoints */
} OrbmFrustumIn;
/* Outputs, one per map point: inView = mbTrackInView (the return value); projX / projY = mTrackProjX / Y (-1 when the
 * point is behind the camera or outside the image; set as soon as the bounds test passes, like the reference);
 * projXR, depth (= |Pc|), level (mnTrackScaleLevel), viewCos are written only for points in view (0 / -1 otherwise: the
 * reference leaves those fields untouched).  M <= max_mappoints of the handle (ORB_ERR_CAPACITY otherwise). */
int orbm_frustum_project(orbm_handle* h, const OrbmFrustumIn* in, uint8_t* inView, float* projX, float* projY, float* projXR,
                         float* depth, int32_t* level, float* viewCos);

/* Device-resident, batched last-frame search: `batch` independent streams.  All pointers are device pointers into
 * fixed-capacity slabs (stride = capacity per stream): current frame slabs as written by orbx_extract_batch_device
 * (kps[batch][kcap], desc[batch][kcap][32], nK[batch]); last-frame slabs [batch][mcap]; Tcw [batch][7].
 * match/claimed [batch][kcap] must be initialised by the caller (e.g. -1 / 0); nmatches [batch].  Enqueues on `stream`. */
typedef struct OrbmBatchDevice {
    int batch, kcap, mcap, nlevels;
    const OrbKeyPoint* kps; const uint8_t* desc; const int32_t* nK;
    float minX, minY, maxX, maxY;
    const float* scaleFactors;          /* device, nlevels */
    const int32_t* nM;                  /* [batch] */
    const uint8_t* valid; const float* xyz; const int32_t* octave; const float* angle; const uint8_t* hasObs;
    const uint8_t* mpDesc;
    const float* Tcw7;                  /* [batch][7] */
    float cam[4];
    int resetState;                     /* 1: start from match = -1, claimed = 0 (fill(mvpMapPoints, NULL), Tracking.cc:2876) instead of reading them */
} OrbmBatchDevice;
int orbm_search_last_frame_batch_device(orbm_handle* h, const OrbmBatchDevice* in, float th, int checkOrientation,
                                        int32_t* d_match, uint8_t* d_claimed, int32_t* d_nmatches, void* stream);

/* Same batched search with HOST pointers in `in` and in match / claimed / nmatches (copies in, runs, copies back). */
int orbm_search_last_frame_batch(orbm_handle* h, const OrbmBatchDevice* in, float th, int checkOrientation,
                                 int32_t* match, uint8_t* claimed, int32_t* nmatches);

/* Tracking::TrackWithMotionModel (reference src/Tracking.cc) from Optimizer::PoseOptimization(&mCurrentFrame) (:2912) through the "discard
 * outliers" loop, for `batch` streams in three launches; monocular, IMU not initialised.  The caller keeps the nmatches < 20 retry and the
 * success thresholds (it passes only the streams it wants optimised in `active`, [batch] or NULL = all).
 * in: the slabs orbm_search_last_frame_batch* took (kps / nK of the current frame, xyz / hasObs of the last frame, cam, nlevels; in->Tcw7 =
 * the pose the search used); invLevelSigma2 [nlevels] = mvInvLevelSigma2.  match / claimed [batch][kcap] and nmatches [batch] are what the
 * search wrote and are updated in place.  PoseOptimization's edges are the keypoints i with match[i] >= 0 in ascending i, with
 * Xw = (double)xyz[match[i]], obs = (double)kps[i].(x, y), invSigma2 = invLevelSigma2[kps[i].octave] (src/Optimizer.cc:877-884), the
 * initial pose (double) of in->Tcw7, exactly pose_optimization_batch's algorithm.
 * Out: pose7 [batch][7] (double, what pose_optimization_batch returns), Tcw7 [batch][7] the float pose after SetPose (may alias in->Tcw7;
 * unchanged with fewer than 3 edges, where the reference returns before SetPose), discarded [batch][mcap] = 1 for the last-frame points of
 * the outliers (their mnLastFrameSeen = current frame; 0 elsewhere), and for every outlier match = -1, claimed = 0, nmatches - 1;
 * nmatchesMap [batch] = inliers whose point has observations.  Streams not in `active` are left untouched. */
int orbm_motion_model_pose_batch_device(orbm_handle* h, const OrbmBatchDevice* in, const float* d_invLevelSigma2, const uint8_t* d_active,
                                        int32_t* d_match, uint8_t* d_claimed, int32_t* d_nmatches, double* d_pose7, float* d_Tcw7,
                                        uint8_t* d_discarded, int32_t* d_nmatchesMap, void* stream);
/* Same with HOST pointers everywhere (one upload, three launches, one download); octaves and match indices out of range are rejected. */
int orbm_motion_model_pose_batch(orbm_handle* h, const OrbmBatchDevice* in, const float* invLevelSigma2, const uint8_t* active, int32_t* match,
                                 uint8_t* claimed, int32_t* nmatches, double* pose7, float* Tcw7, uint8_t* discarded, int32_t* nmatchesMap);

/* Tracking::TrackLocalMap (reference src/Tracking.cc:2952) from SearchLocalPoints (:3346) through the statistics loop that sets
 * mnMatchesInliers, for `batch` streams; monocular, IMU not initialised (so PoseOptimization runs), not only-tracking.  The local map and
 * lastToLocal come from UpdateLocalMap (orbm_update_local_map_batch*, or the caller's own); the caller keeps the thresholds, and the IncreaseVisible / IncreaseFound calls (visible /
 * found say how many).  Precondition: every non-bad point the frame holds is in its local map (true on this path: UpdateLocalKeyFrames votes
 * with the frame's matches), so a match without a local index is one the reference dropped.  On the device, per stream:
 *   1. SearchLocalPoints' first loop: match[i] is remapped to its local index (lastToLocal[match[i]]; -1 or a bad point: match = -1);
 *      a kept point gets visible += 1 and is "seen"; a point TrackWithMotionModel discarded is seen too (no visible count).
 *   2. UpdatePoseMatrices from Tcw7; 3. isInFrustum + PredictScale (viewingCosLimit) for points neither seen nor bad: in view -> visible += 1;
 *      nToMatch = the number in view.  4. SearchByProjection (local map; th[stream], nnratio, bFarPoints / thFarPoints): a keypoint is
 *      claimed at entry when its point has observations; nmatches = its return value (0 when nToMatch == 0).
 *   5. PoseOptimization over all matches (Xw = local worldPos) and SetPose; 6. found += 1 per inlier, mnMatchesInliers = inliers whose
 *      point has observations.
 * Five launches whatever the batch size. */
typedef struct OrbmLocalMapBatch {
    int batch, kcap, mcap, mcapLast, nlevels;
    const OrbKeyPoint* kps; const uint8_t* desc; const int32_t* nK;   /* current frame [batch][kcap], [batch][kcap][32], [batch] */
    float minX, minY, maxX, maxY;
    const float* scaleFactors; const float* invLevelSigma2;          /* mvScaleFactors, mvInvLevelSigma2 [nlevels] */
    float cam[4]; float mbf; float logScaleFactor;                    /* fx fy cx cy; mbf; mfLogScaleFactor */
    const float* Tcw7;                                                /* [batch][7] the frame's pose (after the motion-model step) */
    const int32_t* lastToLocal;   /* [batch][mcapLast]: local index of each last-frame point, -1 = bad; NULL: match is in local indices */
    const uint8_t* discarded;     /* [batch][mcapLast] from the motion-model step ([batch][mcap] local indices without lastToLocal); may be NULL */
    const int32_t* nM;            /* [batch] local points (mvpLocalMapPoints.size()) */
    const float *worldPos, *normal;                                   /* [batch][mcap][3] */
    const float *minDistInv, *maxDistInv, *maxDistance;               /* [batch][mcap]: GetMin/MaxDistanceInvariance(), mfMaxDistance */
    const uint8_t *mpDesc, *hasObs, *bad;                             /* [batch][mcap][32], Observations() > 0, isBad() */
    const float* th;              /* [batch]: 1 on the plain monocular path, 5 right after relocalisation, 15 when lost */
    float nnratio; int bFarPoints; float thFarPoints; float viewingCosLimit;   /* 0.8, mbFarPoints, mThFarPoints, 0.5 */
    const uint8_t* active;        /* [batch] or NULL = all; inactive streams are left untouched */
} OrbmLocalMapBatch;
typedef struct OrbmLocalMapResult {
    int32_t* match;                /* [batch][kcap] in: as the motion-model step left it (last-frame or local indices); out: local indices */
    uint8_t* claimed; uint8_t* outlier;                               /* [batch][kcap]: Observations() > 0 of the match, mvbOutlier */
    int32_t* visible; int32_t* found;                                 /* [batch][mcap]: IncreaseVisible / IncreaseFound counts */
    int32_t *nToMatch, *nmatches, *nInliers, *nMatchesInliers;        /* [batch] */
    double* pose7; float* Tcw7;                                       /* [batch][7]: optimised pose (double) and SetPose's float pose */
} OrbmLocalMapResult;
int orbm_track_local_map_batch_device(orbm_handle* h, const OrbmLocalMapBatch* in, const OrbmLocalMapResult* out, void* stream);
/* HOST pointers in `in` and `out` (one upload, five launches, one download); out-of-range octaves, match and lastToLocal indices are
 * rejected; a slab wider than max_mappoints is ORB_ERR_CAPACITY. */
int orbm_track_local_map_batch(orbm_handle* h, const OrbmLocalMapBatch* in, const OrbmLocalMapResult* out);
/* Same with the current frame on the device (in->kps, in->desc, in->nK from orbx_resident_slabs, stride in->kcap). */
int orbm_track_local_map_batch_resident(orbm_handle* h, const OrbmLocalMapBatch* in, const OrbmLocalMapResult* out);

/* Tracking::Track for a monocular-inertial frame once the IMU is initialised and the frame is past the relocalisation reset window, for
 * `batch` streams (RECENTLY_LOST streams too, with th = 15): TrackWithMotionModel's PredictStateIMU and TrackLocalMap through the
 * statistics loop.  The local map comes from UpdateLocalMap (orbm_update_local_map_batch*, or the caller's own).  The caller keeps
 * PreintegrateIMU, the thresholds, IncreaseVisible / IncreaseFound and the choice of
 * the streams that take this path (imu->mode).  On the device, per stream with mode 1 (mbMapUpdated: from the last keyframe) or 2 (from
 * the last frame):
 *   1. PredictStateIMU in float (source state, its bias and preintegration by mode; gravity (0, 0, -9.81f)) and
 *      Frame::SetImuPoseVelocity: predState21 / predTcw7.
 *   2. SearchLocalPoints with the frame holding no point (match starts at -1): isInFrustum + PredictScale for every non-bad local point,
 *      visible += 1 when in view, then the local-map SearchByProjection with th[stream] (as orbm_track_local_map_batch*).
 *   3. PoseInertialOptimizationLastKeyFrame (mode 1) or PoseInertialOptimizationLastFrame (mode 2), bRecInit = false, over the matches
 *      in ascending keypoint order: Xw = local worldPos, obs = keypoint, invSigma2 = invLevelSigma2[octave], trackDepth = the depth the
 *      frustum test just computed; the current frame's vertices are the double of predState21 (ImuCamPose(Frame*)), the fixed last
 *      keyframe / free previous frame the double of kfState21 / lastState21, the prior (mode 2) prior21 / priorH.  A stream without
 *      matches runs it with the inertial edges only.
 *   4. SetImuPoseVelocity of the float estimate and mImuBias = the optimised bias (Tcw7, state21), mvbOutlier (outlier), mpcpi =
 *      ConstraintPoseImu(double estimate, H) (prior21, priorH: symmetrised, eigenvalues below 1e-12 clamped), found += 1 per inlier,
 *      nMatchesInliers = inliers whose point has observations, nInliers = the optimiser's return value.
 * in: as orbm_track_local_map_batch* with in->Tcw7, in->lastToLocal, in->discarded and in->active NULL.  out: out->pose7 NULL,
 * out->match output only.  Outputs of one call feed the next unchanged (state21 -> lastState21, prior21 / priorH -> the same fields).
 * Streams with mode 0 are left untouched.  At most seven launches whatever the batch size (six with one optimiser variant). */
typedef struct OrbmImuTrackBatch {
    const uint8_t* mode;          /* HOST [batch] in every form: 0 skip, 1 map updated (last keyframe), 2 not updated (last frame) */
    float Tcb7[7];                /* mImuCalib.mTcb as Sophus keeps it: unit quaternion (w, x, y, z) + t (one rig per call) */
    const double* extrinsics24;   /* Rcb | tcb | Rbc | tbc, as the inertial optimisers take it */
    const float* preintKF;        /* [batch][IMU_PREINT_FLOATS] mpImuPreintegratedFromLastKF (= mCurrentFrame.mpImuPreintegrated) */
    const float* preintFrame;     /* [batch][IMU_PREINT_FLOATS] mCurrentFrame.mpImuPreintegratedFrame (mode 2) */
    const float* kfState21;       /* [batch][21] mpLastKeyFrame: GetImuRotation | GetImuPosition | GetVelocity | gyro bias | acc bias (mode 1) */
    const float* lastState21;     /* [batch][21] mLastFrame, same layout (mode 2) */
    const double *prior21, *priorH;  /* [batch][21], [batch][225]: mLastFrame.mpcpi (mode 2) */
} OrbmImuTrackBatch;
typedef struct OrbmImuTrackResult {
    float* predState21;           /* [batch][21] the frame after PredictStateIMU */
    float* predTcw7;              /* [batch][7] its mTcw: the pose SearchLocalPoints projected with */
    float* state21;               /* [batch][21] the frame after the write-back: the next call's lastState21 */
    double *prior21, *priorH;     /* [batch][21], [batch][225]: the new mpcpi */
} OrbmImuTrackResult;
int orbm_track_local_map_inertial_batch_device(orbm_handle* h, const OrbmLocalMapBatch* in, const OrbmImuTrackBatch* imu,
                                               const OrbmLocalMapResult* out, const OrbmImuTrackResult* imuOut, void* stream);
/* HOST pointers in `in`, `imu`, `out` and `imuOut` (one upload, the launches, one download); out-of-range octaves are rejected; a slab
 * wider than max_mappoints is ORB_ERR_CAPACITY. */
int orbm_track_local_map_inertial_batch(orbm_handle* h, const OrbmLocalMapBatch* in, const OrbmImuTrackBatch* imu, const OrbmLocalMapResult* out,
                                        const OrbmImuTrackResult* imuOut);
/* Same with the current frame on the device (in->kps, in->desc, in->nK from orbx_resident_slabs, stride in->kcap). */
int orbm_track_local_map_inertial_batch_resident(orbm_handle* h, const OrbmLocalMapBatch* in, const OrbmImuTrackBatch* imu,
                                                 const OrbmLocalMapResult* out, const OrbmImuTrackResult* imuOut);

/* Tracking::UpdateLocalMap's UpdateLocalKeyFrames and UpdateLocalPoints (reference src/Tracking.cc; monocular and mono-inertial, Nleft == -1)
 * for `batch` streams, one CTA per stream in ONE launch.  Its outputs are the local map in exactly the slabs OrbmLocalMapBatch takes, so
 * orbm_track_local_map_batch_device and orbm_track_local_map_inertial_batch_device can read them with no host step in between.  Per stream:
 *   1. Votes: every good point of the vote source adds 1 to each of its observers (a point held twice votes twice).  voteLastFrame = 0:
 *      the current frame's mvpMapPoints, i.e. srcPoint[match[i]] for i < nK with match[i] >= 0; voteLastFrame = 1 (IMU initialised, past
 *      the relocalisation window): mLastFrame.mvpMapPoints, i.e. every srcPoint entry.
 *   2. The voters that are not bad, in table order (= the std::map's key order), are the first local keyframes; refKF (pKFmax) is the
 *      first of them with the largest count.
 *   3. For each voter, while there are at most 80 local keyframes: the first good unmarked keyframe of its covisibles, the first good
 *      unmarked child, then the parent if unmarked (not tested for isBad()), which ends the loop.
 *   4. Inertial streams with fewer than 80 local keyframes: up to 20 steps from lastKF along prevKF; an unmarked keyframe is added and the
 *      walk moves on, a marked one stalls it.
 *   5. UpdateLocalPoints: the local keyframes in reverse order, each one's slots in slot order; a good point not yet taken is appended.
 * The caller keeps SetReferenceMapPoints, sets the marks (mnTrackReferenceForFrame) and mpReferenceKF, and NULLs the bad points of the
 * voting frame (INTEGRATION.md §2).  Precondition: no keyframe or point is marked for this frame at the call.
 *
 * Keyframe table: stream b's keyframes are rows [kfStart[b], kfStart[b + 1]) in ascending (uint64_t)KeyFrame* order: every observer of a
 * srcPoint entry's point, each observer's covisibles, children and parent, and (inertial) the mPrevKF chain of lastKF, at most 20 entries.
 * Every keyframe index (covKF, childKF, parent, prevKF, obsKF, lastKF, localKF) is relative to the stream's first row; every point index
 * (slotPoint, srcPoint, localPoint) to its first point row pointStart[b].  covKF / childKF / parent are read for the voters only, prevKF
 * for the chain only; the others may be empty / -1.  obsKF is read for the points that vote; which of the srcPoint entries vote is decided
 * by `match`, on the device when the pose step runs there, so give the observations of every srcPoint entry (and put their observers in
 * the table); other points may have none.
 * Output rows past nM are zero (localPoint -1); a stream whose local map has more than mcap points gets its true count in nM, no rows
 * (every row zero, localPoint and lastToLocal -1) and makes the host form return ORB_ERR_CAPACITY naming the stream. */
typedef struct OrbmUpdateLocalMapBatch {
    int batch, kcap, mcap, mcapLast;  /* match [batch][kcap]; output slabs [batch][mcap]; srcPoint / lastToLocal [batch][mcapLast] */
    int nKF, nPoints;                 /* table rows and point rows over the batch (host ints in both forms) */
    const int32_t* kfStart;           /* [batch + 1] */
    const uint8_t* kfFlags;           /* [nKF] ORBM_KF_BAD: isBad() */
    const int32_t* covStart;          /* [nKF + 1] */
    const int32_t* covKF;             /* [covStart[nKF]] GetBestCovisibilityKeyFrames(10): at most 10 per keyframe, in order */
    const int32_t* childStart;        /* [nKF + 1] */
    const int32_t* childKF;           /* [childStart[nKF]] GetChilds(), ascending */
    const int32_t* parent;            /* [nKF] GetParent(), -1 = NULL */
    const int32_t* prevKF;            /* [nKF] mPrevKF, -1 = NULL */
    const int32_t* slotStart;         /* [nKF + 1] */
    const int32_t* slotPoint;         /* [slotStart[nKF]] the non-NULL slots of GetMapPointMatches(), in slot order */
    const int32_t* pointStart;        /* [batch + 1] */
    const uint8_t* pointBad;          /* [nPoints] isBad() */
    const int32_t* obsStart;          /* [nPoints + 1] */
    const int32_t* obsKF;             /* [obsStart[nPoints]] the keyframes of GetObservations(): for every point of srcPoint */
    const float *worldPos, *normal;   /* [nPoints][3] */
    const float *minDistInv, *maxDistInv, *maxDistance;   /* [nPoints] as OrbmLocalMapBatch */
    const uint8_t *mpDesc, *hasObs;   /* [nPoints][32], [nPoints] as OrbmLocalMapBatch */
    const int32_t* nSrc;              /* [batch] entries of the frame's match index space: last-frame slots, or [keyframe features |
                                         last-frame slots] after TrackReferenceKeyFrame (INTEGRATION.md §2); <= mcapLast */
    const int32_t* srcPoint;          /* [batch][mcapLast] point of each entry, -1 = NULL */
    const uint8_t* voteLastFrame;     /* [batch] 0: the frame's match row votes; 1: every srcPoint entry votes */
    const int32_t* match;             /* [batch][kcap] the frame's matches in the index space (what the pose step wrote), values in [-1, nSrc) */
    const int32_t* nK;                /* [batch] keypoints of the frame (read for voteLastFrame = 0) */
    const uint8_t* inertial;          /* [batch] 1: IMU sensor (the temporal walk of step 4) */
    const int32_t* lastKF;            /* [batch] mCurrentFrame.mpLastKeyFrame, -1 = NULL */
} OrbmUpdateLocalMapBatch;
typedef struct OrbmUpdateLocalMapResult {
    int32_t* localKF;                 /* [nKF] mvpLocalKeyFrames of stream b at rows [kfStart[b], kfStart[b] + nLocalKF[b]), -1 after them */
    int32_t* nLocalKF;                /* [batch] */
    int32_t* refKF;                   /* [batch] pKFmax, -1 = none (mpReferenceKF unchanged) */
    int32_t* localPoint;              /* [batch][mcap] mvpLocalMapPoints */
    int32_t* nM;                      /* [batch] mvpLocalMapPoints.size() */
    float *worldPos, *normal;         /* [batch][mcap][3] */
    float *minDistInv, *maxDistInv, *maxDistance;         /* [batch][mcap] */
    uint8_t *mpDesc, *hasObs, *bad;   /* [batch][mcap][32], [batch][mcap], [batch][mcap] (0: local points are good) */
    int32_t* lastToLocal;             /* [batch][mcapLast] local index of srcPoint[j], -1 when NULL, bad or past nSrc */
} OrbmUpdateLocalMapResult;
/* Device pointers everywhere; enqueues on `stream`, one launch, and returns without waiting for it.  Its scratch is a device buffer of the
 * handle's own (grown by the call), shared by every device-form call on the handle: as for the other device forms, the caller orders the
 * calls on one handle on one stream.  The inputs are trusted as the host form checks them. */
int orbm_update_local_map_batch_device(orbm_handle* h, const OrbmUpdateLocalMapBatch* in, const OrbmUpdateLocalMapResult* out, void* stream);
/* HOST pointers (one upload, one launch, one download; no launch when every stream's table is empty).  ORB_ERR_ARG before any launch,
 * with the outputs and orbm_last_launch_count() unchanged: an index or CSR offset out of range, a CSR not starting at 0 or decreasing,
 * kfStart[batch] != nKF or pointStart[batch] != nPoints, more than 10 covisibles, children not ascending, nSrc outside [0, mcapLast], nK
 * outside [0, kcap], a match outside [-1, nSrc), or a null pointer.  ORB_ERR_CAPACITY: a local map larger than mcap (outputs written). */
int orbm_update_local_map_batch(orbm_handle* h, const OrbmUpdateLocalMapBatch* in, const OrbmUpdateLocalMapResult* out);

/* int ORBmatcher::SearchForInitialization(Frame &F1, Frame &F2, vector<cv::Point2f> &vbPrevMatched, vector<int> &vnMatches12,
 * int windowSize) (include/ORBmatcher.h:74, src/ORBmatcher.cc:648-763): the windowed brute-force search of the monocular
 * initialiser (Tracking::MonocularInitialization, src/Tracking.cc:2494-2495, nnratio 0.9, window 100).  F1.K <= max_mappoints and
 * F2.K <= max_keypoints of the handle.  prevMatched [F1.K][2] is vbPrevMatched (in/out, updated like :757-759); matches12 [F1.K] is
 * vnMatches12 (-1 = none); *nmatches is the return value.  Host pointers. */
int orbm_search_for_initialization(orbm_handle* h, const OrbmFrame* F1, const OrbmFrame* F2, float* prevMatched, int windowSize,
                                   float nnratio, int checkOrientation, int32_t* matches12, int* nmatches);

/* Same with the CURRENT FRAME already on the device (in->kps, in->desc, in->nK are device pointers with stride in->kcap, e.g. from
 * orbx_resident_slabs()); everything else as in orbm_search_last_frame_batch (host pointers). */
int orbm_search_last_frame_batch_resident(orbm_handle* h, const OrbmBatchDevice* in, float th, int checkOrientation, int32_t* match,
                                          uint8_t* claimed, int32_t* nmatches);

/* int ORBmatcher::SearchByBoW(KeyFrame* pKF, Frame& F, vector<MapPoint*>& vpMapPointMatches) (include/ORBmatcher.h:68, src/ORBmatcher.cc:223-425,
 * monocular branch): Tracking::TrackReferenceKeyFrame (src/Tracking.cc:2730) and relocalisation.  A frame / keyframe is its keypoints,
 * descriptors and DBoW2::FeatureVector as parallel (node id, feature index) arrays in map order (what orbv_transform_batch returns).
 * kfPoint [KF.N]: 0 = no map point at that keyframe feature, 1 = a map point, 2 = a bad one.  match [F.N] receives the index of the keyframe
 * feature whose map point is assigned to each frame feature (-1 = none), *nmatches the return value.  KF.N <= max_mappoints and
 * F.N <= max_keypoints of the handle.  Host pointers. */
typedef struct OrbmBowFrame {
    int N; const OrbKeyPoint* keypoints; const uint8_t* descriptors;
    int nEntries; const int32_t* fvNode; const int32_t* fvFeature;
} OrbmBowFrame;
int orbm_search_by_bow(orbm_handle* h, const OrbmBowFrame* KF, const uint8_t* kfPoint, const OrbmBowFrame* F, float nnratio, int checkOrientation,
                       int32_t* match, int* nmatches);
/* int ORBmatcher::SearchByBoW(KeyFrame* pKF1, KeyFrame* pKF2, vector<MapPoint*>& vpMatches12) (include/ORBmatcher.h:69, src/ORBmatcher.cc:765-905;
 * LoopClosing): both sides are keyframes (point1 / point2: 0 none, 1 map point, 2 bad), the distance test is strict (bestDist1 < TH_LOW).
 * match12 [KF1.N] = feature of KF2 whose map point goes to vpMatches12[idx1] (-1 = NULL).  KF1.N <= max_mappoints, KF2.N <= max_keypoints. */
int orbm_search_by_bow_kf(orbm_handle* h, const OrbmBowFrame* KF1, const uint8_t* point1, const OrbmBowFrame* KF2, const uint8_t* point2, float nnratio,
                          int checkOrientation, int32_t* match12, int* nmatches);
/* LoopClosing::DetectCommonRegionsFromBoW (src/LoopClosing.cc, v1.0) up to the Sim3Solver, for several place-recognition queries: per
 * candidate pKFi of vpBowCand, in order,
 *   1. NULL or isBad(): SKIPPED;
 *   2. vpCovKFi = pKFi->GetBestCovisibilityKeyFrames(10), [pKFi] when empty, else [pKFi, cov1, ..., cov(n-1), cov0];
 *   3. an entry of vpCovKFi in mpCurrentKF->GetConnectedKeyFrames(): ABORTED_NEAR (bAbortByNearKF);
 *   4. otherwise RAN: ORBmatcher(0.9, true).SearchByBoW(mpCurrentKF, vpCovKFi[j], vvpMatchedMPs[j]) for every non-bad entry j;
 *   5. the merge: for j, k ascending, a good point vvpMatchedMPs[j][k] not yet in spMatchedMPi is inserted, counted in numBoWMatches and
 *      written to vpMatchedPoints[k] / vpKeyFrameMatchedMP[k] (a later j overwrites slot k only with a point not seen before).
 * The caller keeps `if(numBoWMatches >= nBoWMatches)` and everything after it (Sim3Solver, SearchByProjection, OptimizeSim3).  The map is
 * read once, at the call; candidates do not change anything another candidate's sweep reads, so a query may hold the loop candidates and
 * the merge candidates of one keyframe.  Two launches whatever nQueries (the sweep: one CTA per (current keyframe, entry)
 * pair; the merge: one CTA per RAN candidate), ONE upload through the handle's staging and ONE download; orbm_last_launch_count() is 2,
 * or 0 when no candidate is RAN.  Host pointers.
 * ORB_ERR_ARG before any launch, the outputs unchanged: a negative count, nKF < 1, a null pointer a query needs, an index out of range
 * (cand in [-1, nKF) without 0, cov in [1, nKF), point in [-1, nPoints)), covStart not starting at 0 or decreasing, more than 10
 * covisibles, nEntries outside [0, N], an unsorted or out-of-range FeatureVector, kf[0].N > max_mappoints or a candidate / covisible
 * with N > max_keypoints.  ORB_ERR_CAPACITY: more than 2^31 - 1 features in the keyframes the call uploads. */
enum { ORBM_CR_SKIPPED = 0, ORBM_CR_ABORTED_NEAR = 1, ORBM_CR_RAN = 2 };
enum { ORBM_CR_MAX_COV = 11 };
typedef struct OrbmCommonRegionsKF {
    OrbmBowFrame frame;            /* N, mvKeysUn, mDescriptors and the FeatureVector as orbv_transform_batch writes it */
    const int32_t* point;          /* [frame.N] GetMapPointMatches() as point-table indices, -1 = NULL */
    int bad;                       /* isBad() */
    int connected;                 /* in mpCurrentKF->GetConnectedKeyFrames() */
} OrbmCommonRegionsKF;
typedef struct OrbmCommonRegionsQuery {
    int nKF;
    const OrbmCommonRegionsKF* kf; /* [nKF] kf[0] = mpCurrentKF, then the candidates and their covisibles */
    int nPoints;
    const uint8_t* pointBad;       /* [nPoints] isBad(); each MapPoint* of the query once */
    int nCand;
    const int32_t* cand;           /* [nCand] vpBowCand as table indices (loop candidates, then merge candidates), -1 = NULL */
    const int32_t* covStart;       /* [nCand + 1] */
    const int32_t* cov;            /* [covStart[nCand]] each candidate's GetBestCovisibilityKeyFrames(10) */
    uint8_t* status;               /* [nCand] out: ORBM_CR_* */
    int32_t* covList;              /* [nCand][11] out: vpCovKFi as table indices, -1 padded (empty unless RAN) */
    int32_t* nmatches;             /* [nCand][11] out: SearchByBoW's return per entry, -1 where skipped or absent */
    int32_t* numBoWMatches;        /* [nCand] out: 0 unless RAN */
    int32_t* matchedCov;           /* [nCand][kf[0].frame.N] out: j of vpKeyFrameMatchedMP[k], -1 = NULL */
    int32_t* matchedPoint;         /* [nCand][kf[0].frame.N] out: point index of vpMatchedPoints[k], -1 = NULL */
} OrbmCommonRegionsQuery;
int orbm_common_regions_bow_batch(orbm_handle* h, int nQueries, const OrbmCommonRegionsQuery* queries);

/* bool Tracking::TrackReferenceKeyFrame() (reference src/Tracking.cc:2723, monocular; the mono-inertial path runs the same body before
 * the IMU is initialised) after Frame::ComputeBoW, for `batch` streams in four launches whatever the batch size.  The caller computes the
 * frame's BoW with orbv_transform_batch* (levelsup 4) and keeps the success test (nmatchesMap >= 10 monocular, true with an IMU).  Per stream:
 *   1. SearchByBoW(mpReferenceKF, mCurrentFrame) with ORBmatcher(0.7, true): nmatches, match.
 *   2. nmatches < 15: the stream stops there (the reference returns false without touching the frame).
 *   3. Otherwise mvpMapPoints = the matches, SetPose(mLastFrame.GetPose()) = Tcw7, PoseOptimization (edges: the frame features i with
 *      match[i] >= 0 in ascending i, Xw = (double)xyz[match[i]], obs = (double)kps[i].(x, y), invSigma2 = invLevelSigma2[kps[i].octave]),
 *      SetPose of the result, and the "discard outliers" loop: an outlier loses its match and its keyframe feature is marked in discarded
 *      (pMP->mnLastFrameSeen = current frame, mbTrackInView = false); nmatchesMap = inliers whose point has observations.
 * Outputs: nmatches and match for every active stream (match after the discard loop for a stream that passed the gate, the search result
 * otherwise); pose7, Tcw7, discarded and nmatchesMap only for active streams with nmatches >= 15.  Streams not in `active` are untouched.
 * match / discarded feed orbm_track_local_map_batch* in the index space [keyframe features | last-frame points] (INTEGRATION.md §2). */
typedef struct OrbmRefKeyFrameBatch {
    int batch, kcap, mcap, nlevels;
    /* current frame [batch][kcap] (device pointers in the resident form): mvKeysUn, mDescriptors, N, and the FeatureVector as
     * orbv_transform_batch* writes it (fvNode / fvFeature [batch][kcap], nEntries [batch]) */
    const OrbKeyPoint* kps; const uint8_t* desc; const int32_t* nK;
    const int32_t* fvNode; const int32_t* fvFeature; const int32_t* nEntries;
    const float* Tcw7;            /* [batch][7] mLastFrame.GetPose(): the pose SetPose gives the frame before PoseOptimization */
    /* reference keyframe [batch][mcap], indexed by keyframe feature (mcap <= max_mappoints) */
    const int32_t* kfN; const OrbKeyPoint* kfKps; const uint8_t* kfDesc;       /* N, mvKeysUn, mDescriptors */
    const int32_t* kfFvNode; const int32_t* kfFvFeature; const int32_t* kfNEntries;  /* its FeatureVector */
    const uint8_t* kfPoint;       /* 0 no map point, 1 a map point, 2 a bad one */
    const float* xyz;             /* [batch][mcap][3] GetWorldPos() of the point at each feature */
    const uint8_t* hasObs;        /* Observations() > 0 of that point */
    float cam[4];                 /* fx fy cx cy */
    const float* invLevelSigma2;  /* mvInvLevelSigma2 [nlevels] */
    const uint8_t* active;        /* [batch] or NULL = all */
} OrbmRefKeyFrameBatch;
typedef struct OrbmRefKeyFrameResult {
    int32_t* nmatches;            /* [batch] SearchByBoW's return value */
    int32_t* match;               /* [batch][kcap] keyframe feature whose point each frame feature holds, -1 = none */
    double* pose7; float* Tcw7;   /* [batch][7] PoseOptimization's pose and the float pose after SetPose */
    uint8_t* discarded;           /* [batch][mcap] 1 = the outlier's point got mnLastFrameSeen = current frame */
    int32_t* nmatchesMap;         /* [batch] */
} OrbmRefKeyFrameResult;
/* All pointers device pointers; enqueues on `stream`.  The FeatureVectors are trusted as orbv_transform_batch_device writes them. */
int orbm_track_reference_keyframe_batch_device(orbm_handle* h, const OrbmRefKeyFrameBatch* in, const OrbmRefKeyFrameResult* out, void* stream);
/* HOST pointers in `in` and `out` (one upload, four launches, one download).  Out-of-range octaves and counts and unsorted or out-of-range
 * FeatureVectors are ORB_ERR_ARG, slabs wider than the handle ORB_ERR_CAPACITY, both before any launch. */
int orbm_track_reference_keyframe_batch(orbm_handle* h, const OrbmRefKeyFrameBatch* in, const OrbmRefKeyFrameResult* out);
/* Same with the current frame on the device (in->kps, desc, nK, fvNode, fvFeature, nEntries: e.g. the extractor's resident slabs and
 * orbv_transform_batch_device's output on them); everything else host pointers. */
int orbm_track_reference_keyframe_batch_resident(orbm_handle* h, const OrbmRefKeyFrameBatch* in, const OrbmRefKeyFrameResult* out);
/* int ORBmatcher::Fuse(KeyFrame* pKF, const vector<MapPoint*>& vpMapPoints, const float th, const bool bRight) (include/ORBmatcher.h:99,
 * src/ORBmatcher.cc:1148-1338, monocular keyframe; LocalMapping::SearchInNeighbors, src/LocalMapping.cc:878-1021): the SEARCH of every map
 * point -- projection with the keyframe pose, KeyFrame::IsInImage, distance / viewing-angle tests, MapPoint::PredictScale, the radius search
 * of KeyFrame::GetFeaturesInArea with the level window and the chi-square gate, best Hamming distance.  bestIdx[i] = keyframe keypoint
 * (-1: none), bestDist[i] its distance (256: none).  Fuse's return value is the number of i with bestDist[i] <= TH_LOW (50); for those the
 * caller applies :1310-1330 in map-point order (Replace the point with fewer observations, or AddObservation + AddMapPoint): that walk
 * mutates the pointer graph and does not feed back into any search.  state[i]: 0 = NULL, 1 = searched, 2 = isBad(), 3 = IsInKeyFrame(pKF).
 * minDistance / maxDistance are the RAW mfMinDistance / mfMaxDistance (the 0.8f / 1.2f of the getters are applied inside).
 * KF.K <= max_keypoints of the handle; M is unbounded.  Host pointers. */
typedef struct OrbmFusePoints {
    int M; const uint8_t* state; const float* worldPos; const float* normal; const float* minDistance; const float* maxDistance;
    const uint8_t* descriptors;
} OrbmFusePoints;
int orbm_fuse_search(orbm_handle* h, const OrbmFrame* KF, const float* invLevelSigma2, float logScaleFactor, const float* Tcw7, const float* Ow3,
                     const float* cam4, const OrbmFusePoints* pts, float th, int32_t* bestIdx, int32_t* bestDist);
/* The searches of several ORBmatcher::Fuse(KeyFrame*, vector<MapPoint*>, th) calls (each exactly orbm_fuse_search's) in ONE upload through the
 * handle's staging, ONE launch and ONE download; orbm_last_launch_count() is 1 (0 when every item is empty).  Items with pts.M == 0 or KF.K == 0
 * get -1 / 256 and take no CTA.  Host pointers.
 * PRECONDITION: the items must not depend on each other's bookkeeping.  LocalMapping::SearchInNeighbors of several keyframes runs in lockstep
 * rounds: round r holds target r of every keyframe (one keyframe per MAP: keyframes of different maps share no keyframe and no map point),
 * with state and descriptors read after round r-1's walk; the Fuse(mpCurrentKeyFrame, vpFuseCandidates) of all keyframes is one more call
 * (INTEGRATION.md §2, DESIGN.md §4).  Two keyframes of the same map in one call are NOT equivalent to the reference.
 * ORB_ERR_ARG: an octave outside [0, nlevels), empty bounds, nlevels outside [1, 256], a null pointer an item needs (invLevelSigma2
 * always; keypoints / descriptors when K > 0; the point arrays and the outputs when M > 0); ORB_ERR_CAPACITY: K > max_keypoints of the handle or
 * a keyframe too large for the shared-memory grid.  Both before any launch. */
typedef struct OrbmFuseItem {
    OrbmFrame KF;                 /* the target keyframe: mvKeysUn, mDescriptors, bounds, mvScaleFactors */
    const float* invLevelSigma2;  /* mvInvLevelSigma2 [KF.nlevels] */
    float logScaleFactor;         /* mfLogScaleFactor */
    float Tcw7[7];                /* GetPose(): unit quaternion (w, x, y, z) + t */
    float Ow[3];                  /* GetCameraCenter() */
    float cam[4];                 /* fx, fy, cx, cy */
    float th;                     /* Fuse's th: 3 in SearchInNeighbors */
    OrbmFusePoints pts;           /* the points to fuse into KF; state as for orbm_fuse_search */
    int32_t* bestIdx;             /* [pts.M] out */
    int32_t* bestDist;            /* [pts.M] out */
} OrbmFuseItem;
int orbm_fuse_search_batch(orbm_handle* h, int nItems, const OrbmFuseItem* items);
/* int ORBmatcher::Fuse(KeyFrame* pKF, Sophus::Sim3f& Scw, const vector<MapPoint*>& vpPoints, float th, vector<MapPoint*>& vpReplacePoint)
 * (include/ORBmatcher.h:102, src/ORBmatcher.cc:1340-1455; LoopClosing::SearchAndFuse): the search of orbm_fuse_search without the chi-square
 * gate.  Tcw7 / Ow3: the caller's decomposition of Scw (:1349-1350: SE3f(Scw.rotationMatrix(), Scw.translation() / Scw.scale()) and its
 * inverse's translation).  state[i]: 1 = searched, 2 = isBad(), 3 = already among the keyframe's map points.  The caller applies :1436-1450
 * (vpReplacePoint / AddObservation) to every bestDist[i] <= TH_LOW. */
int orbm_fuse_search_sim3(orbm_handle* h, const OrbmFrame* KF, float logScaleFactor, const float* Tcw7, const float* Ow3, const float* cam4, const OrbmFusePoints* pts,
                          float th, int32_t* bestIdx, int32_t* bestDist);
/* int ORBmatcher::SearchBySim3(KeyFrame* pKF1, KeyFrame* pKF2, vector<MapPoint*>& vpMatches12, const Sophus::Sim3f& S12, const float th)
 * (include/ORBmatcher.h:95, src/ORBmatcher.cc:1457-1674): both projection searches and the agreement test.  One map-point slot per keyframe
 * feature (pts.M == KF.K; state 0 = none, 1 = good, 2 = bad); pts1.worldPos holds the points of KF1 IN KF2's CAMERA FRAME
 * (S12.inverse() * (T1w * p3Dw), :1507-1508), pts2.worldPos those of KF2 in KF1's (S12 * (T2w * p3Dw), :1586-1587) -- Sophus expressions the
 * caller evaluates; normal is not read.  cam4 = pKF1's intrinsics (the reference uses them for both directions).  pre12[i1] = KF2 feature of
 * an existing vpMatches12[i1] or -1; match12 = pre12 plus the new mutual matches, *nFound = the return value.  Host pointers. */
int orbm_search_by_sim3(orbm_handle* h, const OrbmFrame* KF1, const OrbmFusePoints* pts1, const OrbmFrame* KF2, const OrbmFusePoints* pts2, float logScaleFactor,
                        const float* cam4, float th, const int32_t* pre12, int32_t* match12, int* nFound);
/* int ORBmatcher::SearchForTriangulation(KeyFrame* pKF1, KeyFrame* pKF2, vector<pair<size_t,size_t>>& vMatchedPairs, const bool bOnlyStereo,
 * const bool bCoarse) (include/ORBmatcher.h:84-85, src/ORBmatcher.cc:907-1146; monocular keyframes, bOnlyStereo = false) for ONE new keyframe
 * against nKF2 neighbours in one launch (LocalMapping::CreateNewMapPoints loops over vpNeighKFs, src/LocalMapping.cc:296-344).
 * A keyframe is its undistorted keypoints, descriptors, hasMapPoint[i] (GetMapPoint(i) != NULL) and DBoW2::FeatureVector as (node id, feature
 * index) arrays in map order.  ep2 [nKF2][2]: the epipole pKF2->mpCamera->project(T2w * Cw) (:913-919); F12 [nKF2][9] row-major: the
 * fundamental matrix of Pinhole::epipolarConstrain (src/CameraModels/Pinhole.cpp:109-112) -- both are Eigen / Sophus expressions the caller
 * evaluates.  scaleFactors / levelSigma2: mvScaleFactors / mvLevelSigma2 (the same extractor settings for all keyframes).
 * matches12 [nKF2][KF1.N]: vMatchedPairs scattered (index in KF2 or -1); nmatches [nKF2]: the return values.  Host pointers. */
typedef struct OrbmTriFrame {
    int N; const OrbKeyPoint* keypoints; const uint8_t* descriptors; const uint8_t* hasMapPoint;
    int nEntries; const int32_t* fvNode; const int32_t* fvFeature;
} OrbmTriFrame;
int orbm_search_for_triangulation(orbm_handle* h, const OrbmTriFrame* KF1, int nKF2, const OrbmTriFrame* KF2, const float* scaleFactors, const float* levelSigma2,
                                  int nlevels, const float* ep2, const float* F12, int bCoarse, int checkOrientation, int32_t* matches12, int32_t* nmatches);
/* LocalMapping::CreateNewMapPoints (src/LocalMapping.cc, the vpNeighKFs loop from :296; monocular keyframes) for ONE new keyframe KF1 against
 * its nKF2 neighbours, in vpNeighKFs order: per neighbour ORBmatcher(0.6f, false).SearchForTriangulation (no rotation histogram), then per
 * match the ray parallax test (cos < 0.9998, or < 0.9996 when bInertial), GeometricTools::Triangulate (4x4 SVD), positive depth and the
 * reprojection test in both keyframes, the far-point cut (thFarPoints > 0) and the scale-consistency test.  A feature of KF1 that received a
 * point from neighbour j is skipped by the searches of every later neighbour, as in the reference (the point was added to KF1).
 * Caller's job: picking the neighbours, the baseline / median-depth skip, CheckNewKeyFrames, and the pointer graph (see INTEGRATION.md).
 * Tcw [1 + nKF2][12]: GetPose().matrix3x4() row-major, KF1 first; Ow [1 + nKF2][3]: GetCameraCenter(); cam [1 + nKF2][4]: fx, fy, cx, cy.
 * ep2, F12, scaleFactors, levelSigma2, nlevels, bCoarse: as in orbm_search_for_triangulation.  scaleFactor: mfScaleFactor of KF1. */
typedef struct OrbmNewPointsIn {
    const OrbmTriFrame* KF1; int nKF2; const OrbmTriFrame* KF2;
    const float* ep2; const float* F12;
    const float* scaleFactors; const float* levelSigma2; int nlevels;
    const float* Tcw; const float* Ow; const float* cam;
    float scaleFactor; int bCoarse; int bInertial; float thFarPoints;
} OrbmNewPointsIn;
/* One new map point, observed by KF1 at idx1 and by neighbour kf2 at idx2; normal / minDistance / maxDistance as
 * MapPoint::UpdateNormalAndDepth sets them (reference keyframe KF1). */
typedef struct OrbmNewPoint {
    int32_t kf2, idx1, idx2; float x3D[3]; float normal[3]; float minDistance, maxDistance;
} OrbmNewPoint;
/* out [KF1.N]: the new points in the order the reference creates them ((neighbour, idx1) ascending), *nNew of them.  nmatches [nKF2]: the
 * reference's vMatchedIndices.size() per neighbour; ncreated [nKF2]: points created from each neighbour.  Host pointers; 3 launches. */
int orbm_create_new_map_points(orbm_handle* h, const OrbmNewPointsIn* in, OrbmNewPoint* out, int* nNew, int32_t* nmatches, int32_t* ncreated);
/* orbm_create_new_map_points for several new keyframes (items) in ONE upload through the handle's staging, 3 launches and ONE download; every
 * item's outputs are byte-identical to what orbm_create_new_map_points gives it alone.  Every per-keyframe setting (level tables, nlevels,
 * scaleFactor, bCoarse, bInertial, thFarPoints) is per item.  An item with nKF2 == 0 or KF1.N == 0 gets zero counts and takes no CTA;
 * orbm_last_launch_count() is 3, or 0 when every item is empty.  Host pointers.
 * PRECONDITION: at most one keyframe per MAP.  CreateNewMapPoints of keyframe A calls AddMapPoint on A and on its neighbours, which changes
 * the hasMapPoint another keyframe of the same map may search; keyframes of different maps share no keyframe and no map point.  Two
 * keyframes of the same map in one call are NOT equivalent to the reference.  CheckNewKeyFrames stays with the caller: read it once per item
 * and cut that item's neighbour list to its first entry when a keyframe is queued (INTEGRATION.md §2).
 * ORB_ERR_ARG: any item failing a check of orbm_create_new_map_points, nItems < 0, or items NULL with nItems > 0; ORB_ERR_CAPACITY: more than
 * 65535 (keyframe, neighbour) pairs over the items with KF1.N > 0.  Both before anything is staged; the message names the item. */
typedef struct OrbmNewPointsItem {
    OrbmNewPointsIn in;           /* exactly what orbm_create_new_map_points takes, per keyframe */
    OrbmNewPoint* out;            /* [in.KF1->N] out: records in creation order */
    int* nNew;                    /* [1] out */
    int32_t* nmatches;            /* [in.nKF2] out */
    int32_t* ncreated;            /* [in.nKF2] out */
} OrbmNewPointsItem;
int orbm_create_new_map_points_batch(orbm_handle* h, int nItems, const OrbmNewPointsItem* items);
/* void MapPoint::ComputeDistinctiveDescriptors() (src/MapPoint.cc:329-403) for nPoints map points at once (LocalMapping::ProcessNewKeyFrame /
 * CreateNewMapPoints call it per point): the observed descriptors of point p are rows obsStart[p] .. obsStart[p+1] of `descriptors`;
 * best[p] = row (relative to obsStart[p]) with the least median Hamming distance to the others, -1 for a point without observations. */
int orbm_distinctive_descriptors(orbm_handle* h, int nPoints, const int32_t* obsStart, const uint8_t* descriptors, int32_t* best);
/* LocalMapping::KeyFrameCulling() (src/LocalMapping.cc, monocular and mono-inertial: redundant_th = 0.9, Nd = 21) for several maps: one CTA
 * per map walks the map's local keyframes in GetVectorCovisibleKeyFrames() order, as the reference's loop does, and applies every cull to the
 * map's state (point bad flags, Observations(), culled keyframes, prev / next links, KeyFramesInMap()) before it evaluates the next keyframe.
 * ONE upload through the handle's staging, ONE launch, ONE download; orbm_last_launch_count() is 1 (0 when no map has a local keyframe).
 * The caller replays the result on the host in `status` order (INTEGRATION.md §2): MergePrevious, the relink and SetBadFlag.
 *
 * Keyframe table [nKF]: every keyframe the call can touch -- the local keyframes, every observer of their points, every prev / next neighbour.
 * Points [nPoints]: each point once per map, with isBad() and its observations (mObservations: the observing keyframe's table index and
 * the observing keypoint's mvKeysUn[idx].octave); Observations() is the number of observations (monocular: nObs counts one per keyframe).
 * PRECONDITIONS: a non-bad point in slot i of keyframe k lists k exactly once among its observations, and occupies no other slot of k;
 * `local` holds each keyframe at most once; the maps of one call share nothing (their keyframes and points are distinct objects).
 * Scalars are read once at the call, as the reference reads them before or during its loop: abortBA is mbAbortBA at the call (Tracking
 * may set it while the loop runs; taking it at the start is one of the reference's own interleavings, a loop that ends before the flag
 * is set).  lastId: the mnId reached from the current keyframe by following mPrevKF at most Nd times (inertial only).
 * ORB_ERR_ARG before any launch: an index out of range (local, slotPoint, obsKF, prevKF / nextKF), slotStart / obsStart not starting
 * at 0 or decreasing, an octave outside [0, 256), nLocal > nKF, a negative count, or a null pointer the map needs (the inertial arrays
 * only when `inertial` is set; the outputs always, visited included). */
enum {
    ORBM_KFC_NOT_VISITED = 0,    /* after the loop's break */
    ORBM_KFC_SKIPPED = 1,        /* the map's init keyframe or isBad() */
    ORBM_KFC_KEPT = 2,           /* not redundant */
    ORBM_KFC_KEPT_FEW_KFS = 3,   /* inertial: KeyFramesInMap() <= Nd */
    ORBM_KFC_KEPT_RECENT = 4,    /* inertial: mnId > current mnId - 2 (unsigned) */
    ORBM_KFC_KEPT_NO_LINK = 5,   /* inertial: mPrevKF or mNextKF is NULL */
    ORBM_KFC_KEPT_IMU = 6,       /* inertial: neither the time rule nor the still rule holds */
    ORBM_KFC_CULLED = 7,         /* monocular: SetBadFlag */
    ORBM_KFC_CULLED_TIME = 8,    /* inertial: (bInitImu && mnId < last_ID && t < 3) || t < 0.5; merge, relink, SetBadFlag */
    ORBM_KFC_CULLED_STILL = 9,   /* inertial: !GetIniertialBA2() && |p - p_prev| < 0.02 && t < 3; merge, relink, SetBadFlag */
    ORBM_KFC_NOT_ERASE = 10      /* SetBadFlag called on a keyframe with mbNotErase: mbToBeErased set (inertial: after the relink) */
};
enum { ORBM_KF_BAD = 1, ORBM_KF_INIT = 2, ORBM_KF_NOT_ERASE = 4 };
typedef struct OrbmCullingMap {
    int nKF;
    const uint64_t* mnId;          /* [nKF] */
    const uint8_t* kfFlags;        /* [nKF] ORBM_KF_*: isBad(), mnId == GetMap()->GetInitKFid(), mbNotErase */
    const int32_t* prevKF;         /* [nKF] inertial only: mPrevKF as a table index, -1 = NULL */
    const int32_t* nextKF;         /* [nKF] inertial only: mNextKF */
    const double* timeStamp;       /* [nKF] inertial only: mTimeStamp */
    const float* imuPosition;      /* [nKF][3] inertial only: GetImuPosition() */
    int nLocal;
    const int32_t* local;          /* [nLocal] table indices in GetVectorCovisibleKeyFrames() order */
    const int32_t* slotStart;      /* [nLocal + 1] the non-NULL slots of GetMapPointMatches(), in slot order */
    const int32_t* slotPoint;      /* [slotStart[nLocal]] point index */
    const int32_t* slotOctave;     /* [slotStart[nLocal]] mvKeysUn[i].octave */
    int nPoints;
    const uint8_t* pointBad;       /* [nPoints] isBad() */
    const int32_t* obsStart;       /* [nPoints + 1] */
    const int32_t* obsKF;          /* [obsStart[nPoints]] observing keyframe (table index) */
    const int32_t* obsOctave;      /* [obsStart[nPoints]] its mvKeysUn[idx].octave */
    int inertial, imuInitialized, inertialBA2, abortBA;   /* mbInertial, isImuInitialized(), GetIniertialBA2(), mbAbortBA */
    int keyFramesInMap;            /* mpAtlas->KeyFramesInMap() */
    uint64_t currentId, lastId;    /* mpCurrentKeyFrame->mnId, last_ID */
    uint8_t* status;               /* [nLocal] out: ORBM_KFC_* */
    int32_t* nMPs;                 /* [nLocal] out: -1 where not evaluated */
    int32_t* nRedundant;           /* [nLocal] out: nRedundantObservations, -1 where not evaluated */
    int32_t* visited;              /* [1] out: the reference's `count` when the loop ended */
} OrbmCullingMap;
int orbm_keyframe_culling_batch(orbm_handle* h, int nMaps, const OrbmCullingMap* maps);
/* LocalMapping::ProcessNewKeyFrame's map-point loop followed by KeyFrame::UpdateConnections (mode ORBM_UC_PROCESS_NEW_KEYFRAME), or the
 * tail of LocalMapping::SearchInNeighbors -- ComputeDistinctiveDescriptors and UpdateNormalAndDepth of every good point of the keyframe,
 * then UpdateConnections (mode ORBM_UC_SEARCH_IN_NEIGHBORS) -- for several keyframes (monocular observations), one CTA per item.
 * ONE upload through the handle's staging, ONE launch, ONE download; orbm_last_launch_count() is 1 (0 when every item has nSlots == 0).
 * The caller replays the result on the host (INTEGRATION.md §2): AddObservation for ADDED slots, the point fields of updated points,
 * mlpRecentAddedMapPoints for IN_KEYFRAME slots, the connection maps and lists, AddChild.
 *
 * Keyframe table [nKF]: entry 0 is the current keyframe, then every observer of its points and every keyframe in the connection maps of
 * those observers.  `order` is the std::map key the reference iterates by ((uint64_t)KeyFrame*); keys are distinct.  Observations and
 * connections are listed in key order.  connStart / connKF / connWeight: mConnectedKeyFrameWeights as CSR; only keyframes that can receive
 * AddConnection (good observers of the same map) need theirs, the others may be empty.  Every keyframe shares the current keyframe's
 * mvScaleFactors (one ORB extractor per map).
 * Points [nPoints]: each point of the keyframe's slots once, with isBad(), GetWorldPos(), mpRefKF (a table index: one of its observers)
 * and mObservations as CSR in key order (keyframe, keypoint index, that keypoint's octave and descriptor row).
 * PRECONDITIONS: at most one keyframe per map per call; the items share no keyframe and no point.
 * ORB_ERR_ARG before any launch: an index, an octave or a CSR offset out of range, a CSR not starting at 0 or decreasing, keys not
 * distinct or a list not in key order, a good point whose mpRefKF is not among its observers, a null pointer the item needs, or a
 * negative count.  ORB_ERR_CAPACITY: a point with more than 65534 observations. */
enum { ORBM_UC_PROCESS_NEW_KEYFRAME = 0, ORBM_UC_SEARCH_IN_NEIGHBORS = 1 };
enum {
    ORBM_UC_SLOT_NONE = 0,           /* NULL or isBad() */
    ORBM_UC_SLOT_ADDED = 1,          /* ProcessNewKeyFrame: AddObservation(KF, i), UpdateNormalAndDepth, ComputeDistinctiveDescriptors */
    ORBM_UC_SLOT_IN_KEYFRAME = 2,    /* ProcessNewKeyFrame: IsInKeyFrame(KF), mlpRecentAddedMapPoints.push_back */
    ORBM_UC_SLOT_UPDATED = 3         /* SearchInNeighbors: ComputeDistinctiveDescriptors, UpdateNormalAndDepth */
};
enum { ORBM_KF_OTHER_MAP = 8 };
typedef struct OrbmConnectionsItem {
    int mode;                      /* ORBM_UC_* */
    int nKF;                       /* >= 1 */
    const uint64_t* order;         /* [nKF] the key of std::map<KeyFrame*, ...> */
    const uint64_t* mnId;          /* [nKF] */
    const uint8_t* kfFlags;        /* [nKF] ORBM_KF_BAD, ORBM_KF_OTHER_MAP (GetMap() != the current keyframe's); entry 0: ORBM_KF_INIT when
                                      mnId == mpMap->GetInitKFid() */
    const float* cameraCenter;     /* [nKF][3] GetCameraCenter() */
    const int32_t* connStart;      /* [nKF + 1] */
    const int32_t* connKF;         /* [connStart[nKF]] table index, in key order */
    const int32_t* connWeight;     /* [connStart[nKF]] */
    int firstConnection;           /* mbFirstConnection of the current keyframe */
    int nlevels;                   /* mnScaleLevels */
    const float* scaleFactors;     /* [nlevels] mvScaleFactors */
    int nSlots;                    /* N of the current keyframe */
    const int32_t* slotPoint;      /* [nSlots] point index, -1 = NULL */
    const int32_t* slotOctave;     /* [nSlots] mvKeysUn[i].octave */
    const uint8_t* slotDesc;       /* [nSlots][32] mDescriptors.row(i) */
    int nPoints;
    const uint8_t* pointBad;       /* [nPoints] isBad() */
    const float* pointPos;         /* [nPoints][3] GetWorldPos() */
    const int32_t* pointRefKF;     /* [nPoints] mpRefKF */
    const int32_t* obsStart;       /* [nPoints + 1] */
    const int32_t* obsKF;          /* [obsStart[nPoints]] observing keyframe (table index), in key order */
    const int32_t* obsIdx;         /* [obsStart[nPoints]] its keypoint index */
    const int32_t* obsOctave;      /* [obsStart[nPoints]] that keypoint's octave */
    const uint8_t* obsDesc;        /* [obsStart[nPoints]][32] that keypoint's descriptor row */
    uint8_t* slotStatus;           /* [nSlots] out: ORBM_UC_SLOT_* */
    uint8_t* pointUpdated;         /* [nPoints] out: UpdateNormalAndDepth and ComputeDistinctiveDescriptors ran on the point */
    float* normal;                 /* [nPoints][3] out: mNormalVector of an updated point, 0 otherwise */
    float* minDistance;            /* [nPoints] out: mfMinDistance of an updated point, 0 otherwise */
    float* maxDistance;            /* [nPoints] out: mfMaxDistance of an updated point, 0 otherwise */
    int32_t* descKF;               /* [nPoints] out: the keyframe of the row mDescriptor takes, -1 = unchanged */
    int32_t* descIdx;              /* [nPoints] out: that keyframe's keypoint index */
    int32_t* counter;              /* [nKF] out: KFcounter, the current keyframe's new mConnectedKeyFrameWeights (0 = absent) */
    int32_t* nConnected;           /* [1] out: length of the ordered list; -1 = empty counter, UpdateConnections changed nothing */
    int32_t* orderedKF;            /* [nKF] out: mvpOrderedConnectedKeyFrames, -1 past the end */
    int32_t* orderedWeight;        /* [nKF] out: mvOrderedWeights */
    int32_t* parent;               /* [1] out: the new mpParent (mbFirstConnection becomes false), -1 = unchanged */
    int32_t* nbrCount;             /* [nKF] out: per keyframe, -1 = no AddConnection or an equal weight (nothing changed), else the length
                                      of its new ordered list; its weight for the current keyframe is then counter[k] */
    int32_t* nbrKF;                /* [connStart[nKF] + nKF] out: keyframe k's new ordered list at offset connStart[k] + k */
    int32_t* nbrWeight;            /* [connStart[nKF] + nKF] out: its weights */
} OrbmConnectionsItem;
int orbm_update_connections_batch(orbm_handle* h, int nItems, const OrbmConnectionsItem* items);

/* cv::BFMatcher(NORM_HAMMING).knnMatch(query, train, k=2) as used at src/Frame.cc:1144: idx/dist are Q x 2,
 * ordered by (distance, lower train index); missing neighbours are -1.  Q and T are unbounded.  Host pointers. */
int orbm_bf_knn2(orbm_handle* h, const uint8_t* query, int Q, const uint8_t* train, int T, int32_t* idx, int32_t* dist);
/* ORBmatcher::DescriptorDistance (src/ORBmatcher.cc:2058-2074) for n descriptor pairs a[i], b[i]; n is unbounded.  Host pointers. */
int orbm_descriptor_distance(orbm_handle* h, const uint8_t* a, const uint8_t* b, int n, int32_t* out);
int orbm_last_launch_count(const orbm_handle* h);
/* Thread-block-cluster size (CTAs per frame, 1..8) of the handle's last SearchByProjection or SearchForInitialization launch.  For
 * SearchByProjection it is the largest size with batch x size <= 2 x SMs whose clusters are all resident at once, for the call's batch
 * and shared-memory size; SearchForInitialization always uses 8.  A refused call leaves it unchanged (and orbm_last_launch_count() is 0). */
int orbm_last_cluster_size(const orbm_handle* h);

/* ------------------------------------------------------------------------------------------
 * Optimizer::LocalBundleAdjustment (reference include/Optimizer.h:71, src/Optimizer.cc:1116-1498): the numeric
 * core between graph construction and write-back, i.e. optimizer.initializeOptimization(); optimizer.optimize(10)
 * (:1410-1411) with g2o's BlockSolver_6_3 + Levenberg-Marquardt semantics, and the per-edge values the outlier
 * test reads (:1417-1430).  The host shim flattens the pointer graph exactly as :1213-1403 builds it
 * (SURVEY.md 8a' "LBA in"); arrays are in g2o's Hessian order (poses by id, then points by id).
 * ------------------------------------------------------------------------------------------ */
typedef struct lba_handle lba_handle;

typedef struct LbaProblem {
    int nPoses;                  /* local + fixed keyframes (VertexSE3Expmap) */
    const double* poses;         /* nPoses x 7: unit quaternion (w,x,y,z) + translation of Tcw (float->double cast, :1217-1218) */
    const uint8_t* poseFixed;    /* vSE3->setFixed(...): InitKF or member of lFixedCameras */
    const float* cam;            /* nPoses x 4: fx, fy, cx, cy of pKFi->mpCamera (Pinhole, float parameters) */
    int nPoints;                 /* VertexSBAPointXYZ, all marginalized (:1289) */
    const double* points;        /* nPoints x 3 */
    int nEdges;                  /* EdgeSE3ProjectXYZ (mono observations, :1305-1331) */
    const int32_t* edgePoint;    /* vertex 0 */
    const int32_t* edgePose;     /* vertex 1 */
    const double* obs;           /* nEdges x 2: kpUn.pt (:1307-1309) */
    const float* invSigma2;      /* nEdges: pKFi->mvInvLevelSigma2[kpUn.octave] (:1316) */
    double huberDelta;           /* thHuberMono = (float)sqrt(5.991) (:1275,:1321) */
    int iterations;              /* optimizer.optimize(10) */
    double userLambdaInit;       /* solver->setUserLambdaInit(100.0) for inertial maps (:1197-1198), else 0 */
    const volatile uint8_t* stopFlag; /* bool* pbStopFlag (&mbAbortBA, src/LocalMapping.cc:154): one byte, so that the caller's own bool can be
                                       * handed over as it is; polled like SparseOptimizer::terminate(); may be NULL */
} LbaProblem;

typedef struct LbaResult {
    double* poses;               /* nPoses x 7, optimised (fixed ones unchanged) */
    double* points;              /* nPoints x 3 */
    double* edgeChi2;            /* nEdges: e->chi2() as the outlier test sees it (errors of the last evaluated state) */
    uint8_t* edgeDepthPositive;  /* nEdges: e->isDepthPositive() at the final state */
    int iterations;              /* return value of SparseOptimizer::optimize */
    int trials;                  /* total LM trials */
    double lambda, chi2, initialChi2;
    int gpuLaunches;
} LbaResult;

int lba_create(lba_handle** out, int max_poses, int max_points, int max_edges, int device);
/* Same, sized for up to max_batch independent problems solved by one kernel launch (one per stream / local map). */
int lba_create_batch(lba_handle** out, int max_poses, int max_points, int max_edges, int max_batch, int device);
void lba_destroy(lba_handle* h);
/* Host pointers in and out; edges may come in any order (per-edge results come back in the caller's order); the index structures of
 * BlockSolver::buildStructure are derived on the device.  Returns ORB_OK, or ORB_ERR_ARG for malformed graphs (index out of range,
 * the same point observed twice by one free keyframe, no free vertex), ORB_ERR_CAPACITY for a problem larger than the handle. */
int lba_solve(lba_handle* h, const LbaProblem* problem, LbaResult* result);
int lba_solve_batch(lba_handle* h, int count, const LbaProblem* problems, LbaResult* results);
/* Split form of lba_solve_batch: upload the flattened graphs once (host pointers), run the whole LM loop for all of
 * them from the uploaded initial estimates on `stream` (device-resident, asynchronous, repeatable), download results.
 * Ordering: lba_download_batch and the next lba_upload_batch wait (on the device, through an event) for the last
 * lba_run_batch_device whatever stream it was given, so no synchronisation is required from the caller in between. */
int lba_upload_batch(lba_handle* h, int count, const LbaProblem* problems);
int lba_run_batch_device(lba_handle* h, void* stream);
int lba_download_batch(lba_handle* h, int count, LbaResult* results);
/* Thread-block-cluster size (CTAs per problem) the last run used. */
int lba_last_cluster_size(const lba_handle* h);
/* Force the cluster size (1..8 CTAs per problem; 0 = automatic: the largest for which every problem's cluster is resident at once). */
int lba_set_cluster_size(lba_handle* h, int ctas);
/* Helper clusters: a batch whose clusters leave SMs idle is launched with extra clusters of the same size that serve the chunked
 * phases (build, point records, Schur partial sums) of every problem; results do not depend on them.  -1 (default): as many as
 * are resident beside the batch; 0: none; n > 0: at most n.  lba_last_helpers: helper clusters of the last run. */
int lba_set_helpers(lba_handle* h, int clusters);
int lba_last_helpers(const lba_handle* h);
/* Device-side phase timers (ns, CTA 0) of problem i of the last downloaded run: errors (first iteration), build_points +
 * build_poses partial sums, build_poses combine, point_prep (after a rejected step), schur_partial, ldlt, schur_combine, pose_trial, points_trial
 * (back-substitution + update + residuals), and last a count instead of a time: the chunks helper clusters served for problem i. */
int lba_get_phase_ns(const lba_handle* h, int i, double* ns10);

/* void Optimizer::LocalBundleAdjustment(KeyFrame* pKF, bool* pbStopFlag, Map* pMap, int& num_fixedKF, int& num_OptKF, int& num_MPs,
 * int& num_edges) (src/Optimizer.cc:1116-1498) as a whole, for a batch of maps: the graph walk (:1125-1403), the solve above, the
 * outlier test and the EraseMapPointMatch / EraseObservation cascade (:1417-1460), and the write-back (:1464-1497).  One map per item,
 * at most one keyframe per map, and the maps share no keyframe and no point.  Monocular observations only: the table has no field for
 * right-camera / stereo observations, so it describes mono maps and mono-inertial maps before IMU initialisation (LocalMapping.cc:129-156).
 * Everything is read once at the call.  Keyframes are table indices, points point indices; std::map<KeyFrame*, ...> order is the caller's
 * key order, in which every point's observations are listed.
 *   keyframe table [nKF]: entry 0 is pKF, then its GetVectorCovisibleKeyFrames() and every observer of the points in their slots.
 *     mnId, kfFlags (ORBM_KF_BAD: isBad(), ORBM_KF_OTHER_MAP: GetMap() != pKF->GetMap(), ORBM_KF_INIT: mnId == pMap->GetInitKFid()),
 *     pose7 = GetPose() as (w, x, y, z, tx, ty, tz), cameraCenter = GetCameraCenter(), cam4 = fx, fy, cx, cy.
 *   cov [nCov]: pKF->GetVectorCovisibleKeyFrames() in order (bad and other-map entries included: the walk filters them).
 *   slots of the candidate local keyframes, candidate c = 0 for pKF and 1 + i for cov[i]: slotStart [nCov + 2], slotPoint = the point of
 *     GetMapPointMatches()[s], -1 for NULL.
 *   points [nPoints]: pointId = mnId, pointFlags (ORBM_KF_BAD: isBad(), ORBM_KF_OTHER_MAP: GetMap() != pKF->GetMap()), worldPos = GetWorldPos(),
 *     refKF = mpRefKF; GetObservations() as CSR obsStart [nPoints + 1] / obsKF / obsIdx, with obsPt = mvKeysUn[idx].pt and obsOctave = .octave.
 *   invLevelSigma2 / scaleFactors [nlevels]: the map's extractor tables; inertial = pMap->IsInertial() (setUserLambdaInit(100)); stopFlag =
 *     pbStopFlag, one byte (may be NULL), read after the walk (:1406) and polled by the solver.
 * Outputs (host pointers):
 *   status: LBA_LOCAL_RAN, LBA_LOCAL_NO_FIXED (num_fixedKF == 0: the reference returns after the walk) or LBA_LOCAL_STOPPED (*pbStopFlag at
 *     :1406: nothing is erased or written back); counts = num_fixedKF, num_OptKF, num_MPs, num_edges (the last three 0 for NO_FIXED, which
 *     returns before assigning them); nLists = |lLocalKeyFrames|, |lFixedCameras|, |lLocalMapPoints|.
 *   localKF [nKF], fixedKF [nKF], localPoint [nPoints]: lLocalKeyFrames, lFixedCameras, lLocalMapPoints in the reference's order.
 *   obsFlag [obsStart[nPoints]]: LBA_OBS_NO_EDGE, LBA_OBS_KEPT or LBA_OBS_ERASED (chi2 > 5.991 or depth not positive); vToErase is the
 *     ERASED observations of lLocalMapPoints in list order, each point's in key order.
 *   per local keyframe i (list order): kfPose7 [nKF][7] = the float pose SetPose receives, kfCenter [nKF][3] = its new GetCameraCenter().
 *   per local point i (list order): pointPos [nPoints][3] = SetWorldPos' argument, pointBad = bad after the cascade, pointRefKF = mpRefKF
 *     after it (-1 once no observation remains), normal [nPoints][3] / minDistance / maxDistance as UpdateNormalAndDepth leaves them
 *     (0 for a bad point, which it leaves unchanged).
 *   lmStats [5]: iterations, trials, lambda, chi2, initial chi2 of LbaResult (iterations -1 when nothing was optimised).
 *   optional (may be NULL): optPose [nKF][7] / optPoint [nPoints][3], the solver's double estimates per local keyframe / point in list order;
 *     edgeChi2 / edgeDepthPositive [obsStart[nPoints]] per observation with an edge.
 * Errors: ORB_ERR_ARG for an index, octave or CSR offset out of range, a CSR that does not start at 0 or decreases, repeated keyframe /
 * point ids, a keyframe or point mnId of 2^64 - 1 (ORB-SLAM3 counts mnIds up from 0; the vertex sort pads with that value), a keyframe
 * listed twice among a point's observations, or null arrays a map needs; ORB_ERR_CAPACITY when nMaps > max_batch or a map's built problem exceeds max_poses / max_points /
 * max_edges.  The message names the map.  Launches (lba_local_last_launches): walk, fill, structure, solver and finish whatever nMaps
 * when any map reaches the solver, else walk and finish.  One staging upload, one copy of the built sizes back, three small tables
 * (slot records, fill sources, solve results) to the device, one download. */
enum { LBA_LOCAL_RAN = 0, LBA_LOCAL_NO_FIXED = 1, LBA_LOCAL_STOPPED = 2 };
enum { LBA_OBS_NO_EDGE = 0, LBA_OBS_KEPT = 1, LBA_OBS_ERASED = 2 };
typedef struct LbaLocalMap {
    int32_t nKF;
    const uint64_t* mnId; const uint8_t* kfFlags; const float* pose7; const float* cameraCenter; const float* cam4;
    int32_t nCov;
    const int32_t* cov; const int32_t* slotStart; const int32_t* slotPoint;
    int32_t nPoints;
    const uint64_t* pointId; const uint8_t* pointFlags; const float* worldPos; const int32_t* refKF;
    const int32_t* obsStart; const int32_t* obsKF; const int32_t* obsIdx; const float* obsPt; const int32_t* obsOctave;
    int32_t nlevels;
    const float* invLevelSigma2; const float* scaleFactors;
    int32_t inertial;
    const volatile uint8_t* stopFlag;
    int32_t* status; int32_t* counts; int32_t* nLists;
    int32_t* localKF; int32_t* fixedKF; int32_t* localPoint; uint8_t* obsFlag;
    float* kfPose7; float* kfCenter;
    float* pointPos; uint8_t* pointBad; int32_t* pointRefKF; float* normal; float* minDistance; float* maxDistance;
    double* lmStats;
    double* optPose; double* optPoint; double* edgeChi2; uint8_t* edgeDepthPositive;
} LbaLocalMap;
int lba_local_bundle_adjustment_batch(lba_handle* h, int nMaps, const LbaLocalMap* maps);
int lba_local_last_launches(const lba_handle* h);

/* ------------------------------------------------------------------------------------------
 * int Optimizer::PoseOptimization(Frame* pFrame) (reference include/Optimizer.h:62, src/Optimizer.cc:814-1114), monocular
 * branch, for `count` frames at once (one CTA per frame).  Per frame f (slots of `cap` entries, N[f] used):
 *   pose7 [count][7]: pFrame->GetPose() as unit quaternion (w,x,y,z) + translation, cast to double (:829-830)
 *   cam4  [count][4]: fx, fy, cx, cy;  Xw [count][cap][3]: pMP->GetWorldPos() (:884);  obs [count][cap][2]: mvKeysUn[i].pt
 *   invSigma2 [count][cap]: mvInvLevelSigma2[octave] (:877);  huberDelta = (float)sqrt(5.991)
 * Out: poseOut [count][7] (pFrame->SetPose), outlier [count][cap] (pFrame->mvbOutlier in slots [0, N[f]), 0 in the slots past N[f]),
 * nInliers[count] = the return value nInitialCorrespondences - nBad.  N[f] outside [0, cap] is refused (ORB_ERR_ARG).  Host pointers.
 * ------------------------------------------------------------------------------------------ */
int pose_optimization_batch(int count, int cap, const int32_t* N, const double* pose7, const float* cam4, const double* Xw,
                            const double* obs, const float* invSigma2, double huberDelta, double* poseOut, uint8_t* outlier,
                            int32_t* nInliers, int device);


/* ------------------------------------------------------------------------------------------
 * Inertial edges (SURVEY.md 8f rank 1): what Optimizer::LocalInertialBA (reference include/Optimizer.h:96, src/Optimizer.cc:2383-2958)
 * and PoseInertialOptimizationLast{KeyFrame,Frame} (:4491, :4875) evaluate in every iteration, batched over all streams of a GPU.
 * The 15-DoF block solver around them is not part of this library yet; these entry points return residuals, Jacobians, chi2 and
 * robust weights in g2o's conventions.  Host pointers.
 * ------------------------------------------------------------------------------------------ */
/* One IMU::Preintegrated (reference include/ImuTypes.h:159-240) as 292 floats:
 *   [0] dT | [1..9] dR | [10..12] dV | [13..15] dP | [16..24] JRg | [25..33] JVg | [34..42] JVa | [43..51] JPg | [52..60] JPa |
 *   [61..66] b = (bax, bay, baz, bwx, bwy, bwz) | [67..291] C (15 x 15 covariance, row-major).  3 x 3 blocks are row-major. */
#define IMU_PREINT_FLOATS 292
/* Preintegrated::Initialize(b) + IntegrateNewMeasurement (src/ImuTypes.cc:177-240) for `count` intervals (one per stream / keyframe pair):
 * acc, gyr [count][maxMeas][3], dt [count][maxMeas], nMeas [count], bias6 [count][6] = (bax, bay, baz, bwx, bwy, bwz);
 * noise4 = (ng, na, ngw, naw) as given to IMU::Calib::Set (:395-407).  preint [count][IMU_PREINT_FLOATS]. */
int imu_preintegrate_batch(int count, const int32_t* nMeas, int maxMeas, const float* acc, const float* gyr, const float* dt, const float* bias6,
                           const float* noise4, float* preint, int device);
/* EdgeInertial's information matrix (src/G2oTypes.cc:499-507: inverse of C.block<9,9>, symmetrised, eigenvalues < 1e-12 clamped) and the
 * EdgeGyroRW / EdgeAccRW informations (src/Optimizer.cc:551,559: inverses of C.block<3,3>(9,9) / (12,12)).  info9 [count][81], infoG / infoA [count][9]. */
int imu_information_batch(int count, const float* preint, double* info9, double* infoG, double* infoA, int device);
/* EdgeInertial::computeError + linearizeOplus (src/G2oTypes.cc:514-594) for `count` edges; edge e uses preint[e].
 * states36 [count][36]: Rwb1 9 | twb1 3 | v1 3 | gyro bias 3 | acc bias 3 | Rwb2 9 | twb2 3 | v2 3 (estimates of the six vertices).
 * err9 [count][9] = (er, ev, ep); J9x24 [count][9][24] (may be NULL), columns: pose 1 (rotation 3, translation 3; tangent of
 * ImuCamPose::Update) | velocity 1 | gyro bias | acc bias | pose 2 | velocity 2.  With info9: chi2 [count] = e^T Omega e and, if rho is
 * given, the Huber weight rho'(chi2) for huberDelta (sqrt(16.92) in LocalInertialBA, src/Optimizer.cc:540-542; <= 0: no kernel). */
int imu_inertial_edges(int count, const float* preint, const double* states36, const double* info9, double huberDelta, double* err9, double* J9x24,
                       double* chi2, double* rho, int device);
/* int Optimizer::PoseInertialOptimizationLastKeyFrame(Frame* pFrame, bool bRecInit) (include/Optimizer.h:66, src/Optimizer.cc:4491-4873),
 * monocular frame: the inertial pose optimiser Tracking::TrackLocalMap runs per frame once the IMU is initialised and the map was updated
 * (src/Tracking.cc:2985-2994), for `count` frames at once (one CTA per frame).  Per frame f (slots of `cap` entries, N[f] used):
 *   Xw [count][cap][3] pMP->GetWorldPos(); obs [count][cap][2] mvKeysUn[i].pt; invSigma2 [count][cap] mvInvLevelSigma2[octave] / unc2;
 *   trackDepth [count][cap] pMP->mTrackDepth (the 10 m "close" rule, :4730); cam4 [count][4]; extrinsics24: Rcb 9 | tcb 3 | Rbc 9 | tbc 3;
 *   preint [count][IMU_PREINT_FLOATS]: pFrame->mpImuPreintegrated (from the last keyframe);
 *   kfState21 / state21 [count][21]: Rwb 9 | twb 3 | velocity 3 | gyro bias 3 | acc bias 3 of the last keyframe (fixed) and of the frame
 *   (in: VertexPose / Velocity / GyroBias / AccBias(pFrame); out: what SetImuPoseVelocity / mImuBias receive, :4813-4817).
 * Out: outlier [count][cap] = mvbOutlier in slots [0, N[f]) and 0 in the slots past N[f], H15 [count][225] = the Hessian handed to
 * ConstraintPoseImu (:4819-4870, row-major, order pose 6 | velocity | gyro bias | acc bias), ret [count] = nInitialCorrespondences - nBad.
 * N[f] outside [0, cap] is refused (ORB_ERR_ARG).  Host pointers. */
int pose_inertial_optimization_last_kf_batch(int count, int cap, const int32_t* N, const float* Xw, const float* obs, const float* invSigma2, const float* trackDepth,
                                             const float* cam4, const double* extrinsics24, const float* preint, const double* kfState21, double* state21, int bRecInit,
                                             uint8_t* outlier, double* H15, int32_t* ret, int device);
/* int Optimizer::PoseInertialOptimizationLastFrame(Frame* pFrame, bool bRecInit) (include/Optimizer.h:67, src/Optimizer.cc:4875-5289), monocular
 * frame: the variant Tracking::TrackLocalMap runs when the map was NOT updated since the last frame (src/Tracking.cc:2985-2994).  The previous
 * frame's pose / velocity / biases are free too (30 unknowns) and held by EdgePriorPoseImu: prior21 [count][21] = Rwb | twb | vwb | bg | ba and
 * priorH [count][225] = pFp->mpcpi->H (what ConstraintPoseImu's constructor made of the Hessian the previous call returned: symmetrised,
 * eigenvalues < 1e-12 clamped).  preintFrame = pFrame->mpImuPreintegratedFrame (EdgeInertial), preintKF = pFrame->mpImuPreintegrated (only the
 * covariance blocks of the two random-walk edges, :5068-5078).  prevState21 in: VertexPose / Velocity / GyroBias / AccBias(pFp); out: their
 * estimates afterwards (the reference does not write them back).  H15 = Marginalize(H, 0, 14).block<15,15>(15,15) (:5268-5270), the Hessian
 * handed to the new ConstraintPoseImu.  Everything else as in pose_inertial_optimization_last_kf_batch. */
int pose_inertial_optimization_last_frame_batch(int count, int cap, const int32_t* N, const float* Xw, const float* obs, const float* invSigma2, const float* trackDepth,
                                                const float* cam4, const double* extrinsics24, const float* preintFrame, const float* preintKF, const double* prior21,
                                                const double* priorH, double* prevState21, double* state21, int bRecInit, uint8_t* outlier, double* H15, int32_t* ret,
                                                int device);
/* EdgeMono (include/G2oTypes.h:342-385, src/G2oTypes.cc:349-373) over VertexPose = ImuCamPose (body pose + camera extrinsics, src/G2oTypes.cc:148-220). */
typedef struct ImuMonoEdges {
    int nPoses;  const double* poses;       /* [nPoses][12]: Rwb 9 | twb 3 */
    const double* extrinsics;               /* [24]: Rcb 9 | tcb 3 | Rbc 9 | tbc 3 (camera 0, IMU::Calib mTcb / mTbc) */
    const float* cam;                       /* [nPoses][4]: fx fy cx cy */
    int nPoints; const double* points;      /* [nPoints][3] */
    int nEdges;  const int32_t* edgePoint; const int32_t* edgePose; const double* obs /* [nEdges][2] */; const float* invSigma2 /* [nEdges] */;
    double huberDelta;                      /* thHuberMono = sqrt(5.991); <= 0: no kernel */
} ImuMonoEdges;
/* err2 [nEdges][2]; Jpoint2x3 [nEdges][6] / Jpose2x6 [nEdges][12] (both or neither may be NULL); chi2, rho (may be NULL) [nEdges];
 * depthPositive [nEdges] = EdgeMono::isDepthPositive(). */
int imu_mono_edges(const ImuMonoEdges* in, double* err2, double* Jpoint2x3, double* Jpose2x6, double* chi2, double* rho, uint8_t* depthPositive, int device);


/* void Optimizer::LocalInertialBA(KeyFrame* pKF, bool* pbStopFlag, Map* pMap, int& num_fixedKF, int& num_OptKF, int& num_MPs, int& num_edges,
 * bool bLarge, bool bRecInit) (include/Optimizer.h:62, src/Optimizer.cc:2383-2958; call site LocalMapping::Run, src/LocalMapping.cc:129-151),
 * monocular-inertial: the numeric core between the graph set-up (:2385-2833, the caller's walk over keyframes / map points / observations) and the
 * write-back (:2890-2957), for `count` local maps at once (one persistent CTA per map; LBA-style "replicas" across streams).
 *   keyframes [0, nOpt): the temporal window vpOptimizableKFs (VertexPose + VertexVelocity + VertexGyroBias + VertexAccBias, all free);
 *   keyframes [nOpt, nKF): lFixedKeyFrames (the window's predecessor first when it is linked by an EdgeInertial).
 *   kfState21 [nKF][21]: Rwb 9 | twb 3 | velocity 3 | gyro bias 3 | acc bias 3 (GetImuRotation / GetImuPosition / GetVelocity / GetImuBias, as doubles);
 *   kfTcw12 [nKF][12]: Rcw 9 | tcw 3 = the keyframe's own camera pose (GetRotation / GetTranslation): ImuCamPose(KeyFrame*) loads both and uses the
 *   camera pose as it is until the vertex is first updated (src/G2oTypes.cc:25-47, :213-221);  cam4 [nKF][4];  extrinsics24: Rcb 9 | tcb 3 | Rbc 9 | tbc 3.
 *   inertial edge i (:2593-2656): keyframes ieKf1[i] (mPrevKF) -> ieKf2[i], preint [nInertial][IMU_PREINT_FLOATS] = pKFi->mpImuPreintegrated,
 *   ieRobust[i] = 1 for the Huber kernel sqrt(16.92) (i == N-1 || bRecInit), ieInfoScale[i] = 1e-2 for i == N-1, else 1.  Every inertial edge
 *   brings its EdgeGyroRW and EdgeAccRW (informations from the preintegration covariance).
 *   points3 [nPoints][3] = GetWorldPos(), trackDepth [nPoints] = mTrackDepth;  mono edge e (:2737-2763): edgePoint[e], edgeKf[e], obs2 = mvKeysUn[].pt,
 *   invSigma2 = mvInvLevelSigma2[octave] / unc2; at most one edge per (point, keyframe) (monocular: no right-camera observations).
 *   iterations = opt_it (10, or 4 with bLarge), lambdaInit = setUserLambdaInit's value (1e0, or 1e-2 with bLarge).
 * Results (host pointers, per problem): the optimised kfState21 / kfTcw12 / points3 (what SetPose / SetVelocity / SetNewBias / SetWorldPos receive
 * after the casts of :2905-2950), erase [nEdges] = 1 for the (keyframe, point) pairs of vToErase (:2848-2862), edgeChi2 [nEdges] = e->chi2(),
 * stats8 = err, err_end (:2837-2839, as floats), failed (the "FAIL LOCAL-INERTIAL BA" test :2884: states and points are then returned unchanged),
 * final lambda, LM trials, optimize()'s iteration count, nanoseconds the map's CTA spent in the solver.  iterationsOut [count] (may be NULL). */
typedef struct LocalInertialBAProblem {
    int32_t nKF, nOpt;
    const double* kfState21; const double* kfTcw12; const float* cam4; const double* extrinsics24;
    int32_t nInertial; const int32_t* ieKf1; const int32_t* ieKf2; const float* preint; const uint8_t* ieRobust; const double* ieInfoScale;
    int32_t nPoints; const double* points3; const float* trackDepth;
    int32_t nEdges; const int32_t* edgePoint; const int32_t* edgeKf; const double* obs2; const float* invSigma2;
    int32_t iterations; int32_t bLarge; double lambdaInit;
} LocalInertialBAProblem;
typedef struct LocalInertialBAResult {
    double* kfState21; double* kfTcw12; double* points3; uint8_t* erase; double* edgeChi2; double* stats8;
    double* profile8;   /* may be NULL; diagnostic: nanoseconds in errors | buildSystem | Dinv, Y | Schur | LDL^T | point back-substitution | update / pop | rest */
} LocalInertialBAResult;
int local_inertial_ba_batch(int count, const LocalInertialBAProblem* problems, const LocalInertialBAResult* results, int32_t* iterationsOut, int device);

/* void Optimizer::LocalInertialBA(KeyFrame* pKF, bool* pbStopFlag, Map* pMap, int&, int&, int&, int&, bool bLarge, bool bRecInit)
 * (src/Optimizer.cc:2383-2958, monocular observations) as a whole, for a batch of maps: the window / point / fixed-keyframe walk
 * (:2385-2478), the edge walk (:2593-2763), the solve of local_inertial_ba_batch, the EraseMapPointMatch / EraseObservation cascade
 * (:2848-2902) and the write-back (:2905-2957).  One map per item, at most one keyframe per map, the maps share no keyframe and no point,
 * and no keyframe or point carries a mark (mnBALocalForKF / mnBAFixedForKF) equal to pKF->mnId at the call.  Keyframes are table indices,
 * points point indices; std::map<KeyFrame*, ...> order is the caller's key order, in which every point's observations are listed.
 *   keyframe table [nKF]: entry 0 is pKF, then its mPrevKF chain (at least Nd + 1 links where they exist) and every observer of the points
 *     in the slots of the chain's first Nd keyframes.  kfFlags: ORBM_KF_BAD (isBad()), ORBM_KF_OTHER_MAP (GetMap() != pKF->GetMap()),
 *     ORBM_KF_IMU (bImu), ORBM_KF_PREINT (mpImuPreintegrated != NULL); prevKF = mPrevKF as a table index (-1 = NULL);
 *     state21 = GetImuRotation | GetImuPosition | GetVelocity | GetGyroBias | GetAccBias, tcw12 = GetRotation | GetTranslation,
 *     cameraCenter = GetCameraCenter(), cam4 = fx fy cx cy; preint [nKF][IMU_PREINT_FLOATS] = mpImuPreintegrated (rows read where
 *     ORBM_KF_PREINT; may be NULL when no entry has it); extrinsics24 as local_inertial_ba_batch takes it.
 *   slots [nKF + 1] CSR: slotPoint = the point of GetMapPointMatches()[s], -1 for NULL (only the window candidates' slots are read).
 *   points [nPoints]: pointFlags (ORBM_KF_BAD: isBad()), worldPos, trackDepth = mTrackDepth, refKF = mpRefKF; GetObservations() as CSR
 *     obsStart [nPoints + 1] / obsKF / obsIdx with obsPt = mvKeysUn[idx].pt and obsOctave = .octave (Pinhole: uncertainty2 = 1).
 *   keyFramesInMap = pMap->KeyFramesInMap(); bLarge, bRecInit as the reference takes them.
 * Outputs (host pointers):
 *   status: LIBA_LOCAL_RAN or LIBA_LOCAL_FAILED ("FAIL LOCAL-INERTIAL BA": nothing is erased or written back, and the marks stay set);
 *   nLists [4] = N, |lFixedKeyFrames|, |lLocalMapPoints|, mono edges.
 *   optKF [nKF] = vpOptimizableKFs (newest first), fixedKF [nKF] = lFixedKeyFrames, localPoint [nPoints] = lLocalMapPoints, all in the
 *     reference's order; ieLinked [nKF]: window keyframe i got its inertial edge (and its preintegration SetNewBias(mPrevKF->GetImuBias())).
 *   obsFlag [obsStart[nPoints]]: LBA_OBS_NO_EDGE, LBA_OBS_KEPT or LBA_OBS_ERASED; vToErase is the ERASED observations of localPoint in
 *     list order, each point's in key order (none on FAILED).
 *   per window keyframe i: kfPose7 [nKF][7] = the SE3f SetPose receives, kfCenter [nKF][3] = its GetCameraCenter(), kfVelocity [nKF][3],
 *     kfBias6 [nKF][6] = IMU::Bias (bax, bay, baz, bwx, bwy, bwz).
 *   per local point i: pointPos [nPoints][3], pointBad, pointRefKF, normal [nPoints][3] / minDistance / maxDistance as in
 *     lba_local_bundle_adjustment_batch.  Every per-keyframe and per-point value is 0 on FAILED (pointRefKF -1).
 *   stats8 as LocalInertialBAResult.stats8.
 *   optional (all four or none): optState21 [nKF][21] / optTcw12 [nKF][12] = the solver's doubles per problem keyframe (window, then
 *     lFixedKeyFrames), optPoint [nPoints][3] per local point, edgeChi2 [obsStart[nPoints]] per observation with an edge (0 elsewhere);
 *     the first three are 0 on FAILED.
 * Errors, before the device is touched: ORB_ERR_ARG naming the map for an index, octave or CSR offset out of range, a keyframe that
 * observes a point twice, an mpRefKF of a good point that is not among its observers, pKF of another map or without mPrevKF, a window
 * keyframe without ORBM_KF_IMU, an mPrevKF chain that revisits a keyframe within Nd + 1 steps, or a null array a map needs.  Then
 * ORB_ERR_CUDA without a usable device.  Three launches whatever nMaps (walk, solver, finish; local_inertial_ba_map_last_launches), one
 * staging upload and one download, no host synchronisation in between.  Like local_inertial_ba_batch it uses the thread's staging on device. */
enum { ORBM_KF_IMU = 16, ORBM_KF_PREINT = 32 };
enum { LIBA_LOCAL_RAN = 0, LIBA_LOCAL_FAILED = 1 };
typedef struct LocalInertialBAMap {
    int32_t nKF;
    const uint8_t* kfFlags; const int32_t* prevKF;
    const float* state21; const float* tcw12; const float* cameraCenter; const float* cam4;
    const float* preint; const double* extrinsics24;
    const int32_t* slotStart; const int32_t* slotPoint;
    int32_t nPoints;
    const uint8_t* pointFlags; const float* worldPos; const float* trackDepth; const int32_t* refKF;
    const int32_t* obsStart; const int32_t* obsKF; const int32_t* obsIdx; const float* obsPt; const int32_t* obsOctave;
    int32_t nlevels;
    const float* invLevelSigma2; const float* scaleFactors;
    int32_t keyFramesInMap; int32_t bLarge; int32_t bRecInit;
    int32_t* status; int32_t* nLists;
    int32_t* optKF; int32_t* fixedKF; int32_t* localPoint; uint8_t* ieLinked; uint8_t* obsFlag;
    float* kfPose7; float* kfCenter; float* kfVelocity; float* kfBias6;
    float* pointPos; uint8_t* pointBad; int32_t* pointRefKF; float* normal; float* minDistance; float* maxDistance;
    double* stats8;
    double* optState21; double* optTcw12; double* optPoint; double* edgeChi2;
} LocalInertialBAMap;
int local_inertial_ba_map_batch(int nMaps, const LocalInertialBAMap* maps, int device);
int local_inertial_ba_map_last_launches(void);

/* ------------------------------------------------------------------------------------------
 * DBoW2 transform (SURVEY.md 8f rank 3): Frame::ComputeBoW / KeyFrame::ComputeBoW (reference src/Frame.cc:738-745) call
 * ORBVocabulary::transform(vCurrentDesc, mBowVec, mFeatVec, 4) = DBoW2::TemplatedVocabulary<FORB::TDescriptor, FORB>::transform
 * (Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h:1127-1259).  The vocabulary tree is handed over once as flat arrays (the host shim
 * flattens m_nodes after loadFromTextFile) and stays in HBM; a call transforms the descriptors of `batch` frames.
 * ------------------------------------------------------------------------------------------ */
typedef struct orbv_handle orbv_handle;
typedef struct OrbVocabulary {
    int nNodes;                   /* m_nodes.size(); node 0 is the root */
    int L;                        /* m_L (6 for ORBvoc) */
    int weighting;                /* m_weighting: 0 TF_IDF (ORB-SLAM3), 1 TF, 2 IDF, 3 BINARY */
    int norm;                     /* what m_scoring_object->mustNormalize gives: 0 none, 1 L1 (L1_NORM, ORB-SLAM3), 2 L2 */
    const int32_t* childStart;    /* [nNodes + 1]: children of node n are children[childStart[n] .. childStart[n+1]) */
    const int32_t* children;      /* node ids in the order of m_nodes[n].children */
    const uint8_t* descriptors;   /* [nNodes][32]: m_nodes[n].descriptor */
    const double* weight;         /* [nNodes]: m_nodes[n].weight (idf of a word; 0 = stopped) */
    const int32_t* wordId;        /* [nNodes]: m_nodes[n].word_id for leaves, -1 otherwise */
} OrbVocabulary;
/* ORB_ERR_ARG, before anything is uploaded: nNodes < 2, L < 1, weighting outside [0, 3], norm outside [0, 2], a null pointer, a root
 * (node 0) without children, a childStart that does not start at 0 or decreases, a node with more than 2^20 children, a child index
 * outside [1, nNodes), a node listed as a child more than once (so a table with a cycle is refused: with the root nobody's child and
 * every other node at most one node's, the nodes the descent can reach form a tree), or a leaf with a negative wordId.  A leaf is a node
 * without children; a stopped word is a leaf with weight 0. */
int orbv_create(orbv_handle** out, const OrbVocabulary* voc, int device);
void orbv_destroy(orbv_handle* h);
/* transform() for `batch` frames; frame f has n[f] descriptors in desc [batch][cap][32].  Outputs in the iteration order of the reference's
 * std::map containers: BowVector as wordId / wordValue [batch][cap] (nWords[f] entries, ascending word id; values are DBoW2's doubles bit
 * for bit), FeatureVector as parallel arrays fvNode / fvFeature [batch][cap] (nEntries[f] entries: ascending node id, feature indices
 * ascending within a node).  A feature whose leaf lies above depth L - levelsup is filed under node 0 (the reference leaves that node id
 * unset).  levelsup = 4 in the reference.  Host pointers.  ORB_ERR_ARG before anything is staged: batch < 1, cap outside [1, 16384],
 * levelsup < 0, n[f] outside [0, cap], or a null pointer. */
int orbv_transform_batch(orbv_handle* h, int batch, const uint8_t* desc, const int32_t* n, int cap, int levelsup, int32_t* wordId, double* wordValue,
                         int32_t* nWords, int32_t* fvNode, int32_t* fvFeature, int32_t* nEntries);
/* Device form: all pointers device pointers; d_scratch* are [batch][cap] work arrays owned by the caller; enqueues on `stream`.
 * ORB_ERR_ARG before any launch: batch < 1, cap outside [1, 16384], levelsup < 0, or a null pointer.  d_n is read on the device only,
 * where a count above cap stands for cap and a negative one for 0. */
int orbv_transform_batch_device(orbv_handle* h, int batch, const uint8_t* d_desc, const int* d_n, int cap, int levelsup, int* d_scratchWord,
                                double* d_scratchWeight, int* d_scratchNode, int* d_wordId, double* d_wordValue, int* d_nWords, int* d_fvNode,
                                int* d_fvFeature, int* d_nEntries, void* stream);

/* ------------------------------------------------------------------------------------------
 * KeyFrameDatabase (src/KeyFrameDatabase.cc): the inverted file on the device, and phase 1 of DetectRelocalizationCandidates
 * (Tracking::Relocalization) and DetectNBestCandidates (LoopClosing::NewDetectCommonRegions) -- the walk over the inverted-file lists
 * of the query's words and the L1Scoring::score of the keyframes that share more than minCommonWords -- for a batch of queries.
 * Phase 2 (accumulation over GetBestCovisibilityKeyFrames(10), the sort and the selection) stays with the caller (INTEGRATION.md §2).
 * One handle serves maxDatabases databases (one per SLAM system) from one pool of maxKeyFrames keyframes of at most maxWords words.
 * Scoring is L1Scoring, what ORBvoc.txt's header declares and ORB-SLAM3 uses; vocabularyWords = mpVoc->size() bounds the word ids.
 * A keyframe is a caller key unique within its database, such as (uint64_t)KeyFrame*; a BowVector is its (id, value) pairs with
 * ascending ids, as orbv_transform_batch returns them.  Host pointers throughout.
 * THREADS: the staging buffers, the slot pool and the launch count belong to the handle, not to one database, so the handle serialises
 * its calls: every orbv_db_* entry point holds the handle's mutex for the whole call, and threads of different SLAM systems may call
 * one handle at once.  The caller keeps the reference's per-database mMutex around a detection and the replay of its record (the
 * marks, counters and scores live in its KeyFrame objects; INTEGRATION.md §2).
 * ------------------------------------------------------------------------------------------ */
typedef struct orbv_db_handle orbv_db_handle;
/* ORB_ERR_ARG for a size < 1 or maxWords > 8192; ORB_ERR_CUDA without an sm_90 device. */
int orbv_db_create(orbv_db_handle** out, int vocabularyWords, int maxDatabases, int maxKeyFrames, int maxWords, int device);
void orbv_db_destroy(orbv_db_handle* h);
/* add(pKF) for n keyframes, in array order: keyframe i goes to database dbIndex[i] with the BowVector wordId / wordValue
 * [wordStart[i], wordStart[i + 1]).  One upload, one launch.  ORB_ERR_ARG before anything changes: a database index out of range, a
 * key already in its database or added twice by the call (the reference would list that keyframe twice), more than maxWords words, a
 * word id outside [0, vocabularyWords), ids that do not ascend, a wordStart that does not start at 0 or decreases, a null pointer.
 * ORB_ERR_CAPACITY: fewer than n free slots.  A call that fails leaves the database and the free slots as they were. */
int orbv_db_add_batch(orbv_db_handle* h, int n, const int32_t* dbIndex, const uint64_t* key, const int32_t* wordStart, const int32_t* wordId,
                      const double* wordValue);
/* erase(pKF) for n keyframes: a key not in its database is a no-op, as in the reference.  clearMap(pMap) is this call with the map's
 * keyframes: the entries that remain keep their relative order either way.  No launch. */
int orbv_db_erase_batch(orbv_db_handle* h, int n, const int32_t* dbIndex, const uint64_t* key);
/* clear(): empties one database.  No launch. */
int orbv_db_clear(orbv_db_handle* h, int dbIndex);
/* The number of keyframes in a database (ORB_ERR_ARG for an index out of range). */
int orbv_db_size(const orbv_db_handle* h, int dbIndex);
enum { ORBV_DB_RELOC = 0, ORBV_DB_NBEST = 1 };
/* One query.  kind ORBV_DB_RELOC: DetectRelocalizationCandidates(F, pMap) with F->mBowVec; ORBV_DB_NBEST: DetectNBestCandidates(pKF, ...)
 * with pKF->mBowVec and the keys of pKF->GetConnectedKeyFrames() (keys not in the database are ignored).
 * Outputs: lKFsSharingWords in the reference's order, the first min(nSharing, cap) entries: key, words = the mnRelocWords /
 * mnPlaceRecognitionWords counter, scored = words > minCommonWords (the entry is in lScoreAndMatch), score = the float mRelocScore /
 * mPlaceRecognitionScore of a scored entry (0 otherwise); entries past that are 0.  nSharing = |lKFsSharingWords|,
 * maxCommonWords = the largest counter (0 when the list is empty; minCommonWords = (int)(maxCommonWords * 0.8f)). */
typedef struct OrbvDbQuery {
    int32_t dbIndex;
    int32_t kind;                  /* ORBV_DB_RELOC or ORBV_DB_NBEST */
    int32_t nWords;
    const int32_t* wordId;         /* [nWords] ascending */
    const double* wordValue;       /* [nWords] */
    int32_t nConnected;            /* NBEST only */
    const uint64_t* connected;     /* [nConnected] NBEST only */
    int32_t cap;
    uint64_t* key;                 /* [cap] out */
    int32_t* words;                /* [cap] out */
    uint8_t* scored;               /* [cap] out */
    float* score;                  /* [cap] out */
    int32_t* nSharing;             /* [1] out */
    int32_t* maxCommonWords;       /* [1] out */
} OrbvDbQuery;
/* Phase 1 of every query, mixing kinds and databases: one upload through the handle's staging, three launches whatever nQueries
 * (orbv_db_last_launch_count; 0 for nQueries == 0), one download.  Scores equal L1Scoring::score bit for bit: the common words' terms
 * fabs(vi - wi) - fabs(vi) - fabs(wi) are added in ascending word order in double, then -score / 2.0 is rounded to float.
 * PRECONDITIONS, as the reference's walk needs them: no keyframe of the database carries the query's mark (mnRelocQuery /
 * mnPlaceRecognitionQuery == the query's mnId) at the call, and a keyframe's mBowVec does not change while it is in the database.
 * ORB_ERR_ARG before any launch: nQueries outside [0, 2^24 - 1], a database index out of range, an unknown kind, a negative cap or nConnected, a word id outside
 * [0, vocabularyWords), ids that do not ascend, more than maxWords words, a null pointer.  ORB_ERR_CAPACITY after the call: a query
 * with nSharing > cap (its outputs hold the first cap entries, nSharing and maxCommonWords are exact). */
int orbv_db_query_batch(orbv_db_handle* h, int nQueries, const OrbvDbQuery* q);
/* Kernel launches of the handle's last add / erase / clear / query call. */
int orbv_db_last_launch_count(const orbv_db_handle* h);

#ifdef __cplusplus
}
#endif
#endif /* ORB_B200_H */
