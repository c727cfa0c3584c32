// Host-side C++ mirror of the three reference class surfaces over the C-ABI (orb_b200.h).  Header only, no OpenCV/Eigen:
// cv::KeyPoint / cv::Mat are replaced by layout-compatible PODs (SURVEY.md 8b).  Method names, argument meaning and
// error behaviour follow the reference so that Frame.cc / Tracking.cc / LocalMapping.cc-style callers read the same.
//   ORB_SLAM3::ORBextractor   reference include/ORBextractor.h:43-109
//   ORB_SLAM3::ORBmatcher     reference include/ORBmatcher.h:36-103   (per-frame hot functions)
//   ORB_SLAM3::Optimizer      reference include/Optimizer.h:46-102    (LocalBundleAdjustment numeric core)
//   ORB_SLAM3::KeyFrameDatabase  reference include/KeyFrameDatabase.h  (the inverted file and phase 1 of both detections, over keys)
#pragma once
#include <cstdint>
#include <stdexcept>
#include <string>
#include <cmath>
#include <vector>

#include "../orb_b200.h"

namespace ORB_SLAM3 {

using KeyPoint = OrbKeyPoint;                    // byte-compatible with cv::KeyPoint
struct Descriptors {                             // stands in for a CV_8UC1 cv::Mat with 32 columns
    int rows = 0;
    std::vector<uint8_t> data;
    uint8_t* ptr(int r) { return data.data() + (size_t)r * 32; }
    const uint8_t* ptr(int r) const { return data.data() + (size_t)r * 32; }
    void release() { rows = 0; data.clear(); }
};
struct Image {                                   // stands in for a CV_8UC1 cv::Mat
    const uint8_t* data = nullptr;
    int rows = 0, cols = 0;
    size_t step = 0;
    bool empty() const { return !data || rows <= 0 || cols <= 0; }
};

inline void orb_check(int rc, const char* where) {
    if (rc != ORB_OK) throw std::runtime_error(std::string(where) + ": " + orb_last_error());
}

class ORBextractor {
public:
    enum { HARRIS_SCORE = 0, FAST_SCORE = 1 };
    ORBextractor(int nfeatures, float scaleFactor, int nlevels, int iniThFAST, int minThFAST, int maxWidth = 1920, int maxHeight = 1080,
                 int device = 0)
        : nlevels_(nlevels) {
        orb_check(orbx_create(&h_, nfeatures, scaleFactor, nlevels, iniThFAST, minThFAST, maxWidth, maxHeight, 1, device), "orbx_create");
        mvScaleFactor.resize(nlevels); mvInvScaleFactor.resize(nlevels); mvLevelSigma2.resize(nlevels); mvInvLevelSigma2.resize(nlevels);
        orbx_get_tables(h_, mvScaleFactor.data(), mvInvScaleFactor.data(), mvLevelSigma2.data(), mvInvLevelSigma2.data(), nullptr);
    }
    ~ORBextractor() { orbx_destroy(h_); }
    ORBextractor(const ORBextractor&) = delete;
    ORBextractor& operator=(const ORBextractor&) = delete;

    // int operator()(InputArray image, InputArray mask, vector<KeyPoint>&, OutputArray descriptors, vector<int>& vLappingArea)
    // Returns monoIndex, or -1 for an empty image (src/ORBextractor.cc:1090-1091).  The mask is ignored, as in the reference.
    int operator()(const Image& image, const Image& /*mask*/, std::vector<KeyPoint>& keypoints, Descriptors& descriptors,
                   std::vector<int>& vLappingArea) {
        if (image.empty()) return -1;
        const int cap = orbx_max_keypoints(h_);
        keypoints.resize(cap);
        descriptors.data.resize((size_t)cap * 32);
        int n = 0, mono = 0;
        const int rc = orbx_extract(h_, image.data, image.rows, image.cols, image.step, vLappingArea.at(0), vLappingArea.at(1),
                                    keypoints.data(), descriptors.data.data(), cap, &n, &mono);
        if (rc == ORB_ERR_EMPTY) return -1;
        orb_check(rc, "orbx_extract");
        keypoints.resize(n);
        descriptors.rows = n;
        descriptors.data.resize((size_t)n * 32);
        if (n == 0) descriptors.release();         // _descriptors.release() (:1108-1109)
        return mono;
    }
    int GetLevels() { return nlevels_; }
    float GetScaleFactor() { return nlevels_ > 1 ? mvScaleFactor[1] : 1.0f; }
    std::vector<float> GetScaleFactors() { return mvScaleFactor; }
    std::vector<float> GetInverseScaleFactors() { return mvInvScaleFactor; }
    std::vector<float> GetScaleSigmaSquares() { return mvLevelSigma2; }
    std::vector<float> GetInverseScaleSigmaSquares() { return mvInvLevelSigma2; }
    // mvImagePyramid[level] of the last call (public member in the reference, read by the stereo matcher only)
    std::vector<uint8_t> ImagePyramidLevel(int level, int& width, int& height) {
        orb_check(orbx_get_level_size(h_, level, &width, &height), "orbx_get_level_size");
        std::vector<uint8_t> out((size_t)width * height);
        orb_check(orbx_copy_level(h_, 0, level, 0, out.data()), "orbx_copy_level");
        return out;
    }
    orbx_handle* handle() { return h_; }

private:
    orbx_handle* h_ = nullptr;
    int nlevels_;
    std::vector<float> mvScaleFactor, mvInvScaleFactor, mvLevelSigma2, mvInvLevelSigma2;
};

// The slice of Frame the matchers read (mvKeysUn, mDescriptors, image bounds, mvScaleFactors) plus the in/out
// mvpMapPoints state as (index of the map point in the caller's array, Observations()>0 flag).
struct FrameView {
    std::vector<KeyPoint> mvKeysUn;
    Descriptors mDescriptors;
    float mnMinX = 0, mnMinY = 0, mnMaxX = 0, mnMaxY = 0;
    std::vector<float> mvScaleFactors;
    std::vector<int32_t> mvpMapPoints;     // -1 == NULL
    std::vector<uint8_t> mvbClaimed;
    OrbmFrame c_struct() const {
        OrbmFrame f;
        f.K = (int)mvKeysUn.size(); f.keypoints = mvKeysUn.data(); f.descriptors = mDescriptors.data.data();
        f.minX = mnMinX; f.minY = mnMinY; f.maxX = mnMaxX; f.maxY = mnMaxY;
        f.scaleFactors = mvScaleFactors.data(); f.nlevels = (int)mvScaleFactors.size();
        return f;
    }
    // void Frame::UndistortKeyPoints() (src/Frame.cc:747): mvKeysUn from mvKeys, the keypoints `extractor` returned in its last call, on
    // the GPU (the extractor's resident slab, no upload).  k1 == 0 copies mvKeys.
    void UndistortKeyPoints(ORBextractor& extractor, const OrbPinholeCamera& cam, const std::vector<KeyPoint>& mvKeys) {
        const int cap = orbx_max_keypoints(extractor.handle());
        std::vector<KeyPoint> slab((size_t)cap);
        orb_check(orbx_undistort_keypoints(extractor.handle(), &cam, 1, slab.data(), cap, nullptr), "orbx_undistort_keypoints");
        mvKeysUn.assign(slab.begin(), slab.begin() + (std::ptrdiff_t)mvKeys.size());
    }
    // void Frame::ComputeImageBounds(const cv::Mat& imLeft) (called at src/Frame.cc:793): mnMinX, mnMaxX, mnMinY, mnMaxY from the
    // undistorted image corners (0, cols, 0, rows when k1 == 0).
    void ComputeImageBounds(const OrbPinholeCamera& cam, int cols, int rows, int device = 0) {
        float b[4];
        orb_check(orbx_image_bounds(&cam, cols, rows, b, device), "orbx_image_bounds");
        mnMinX = b[0]; mnMaxX = b[1]; mnMinY = b[2]; mnMaxY = b[3];
    }
};

namespace detail {
// The reference constructs ORBmatcher as a stack temporary per use (src/Tracking.cc:2494,2730,2859,3393,3631) and Optimizer's
// functions are static: neither can own device scratch.  The handles therefore live in per-thread caches (Tracking and
// LocalMapping are different threads, src/System.cc:197) that grow on demand and are reused by every later call.
struct MatcherSlot {
    orbm_handle* h = nullptr; int maxK = 0, maxM = 0, device = -1;
    ~MatcherSlot() { if (h) orbm_destroy(h); }
};
inline orbm_handle* matcher_handle(int needK, int needM, int device) {
    thread_local MatcherSlot s;
    if (!s.h || s.device != device || needK > s.maxK || needM > s.maxM) {
        if (s.h) { orbm_destroy(s.h); s.h = nullptr; }
        s.maxK = needK > s.maxK ? needK + needK / 2 : s.maxK; if (s.maxK < 4096) s.maxK = 4096; if (s.maxK > 65535) s.maxK = 65535;
        s.maxM = needM > s.maxM ? needM + needM / 2 : s.maxM; if (s.maxM < 16384) s.maxM = 16384; if (s.maxM > 65535) s.maxM = 65535;
        s.device = device;
        orb_check(orbm_create(&s.h, 1, s.maxK, s.maxM, device), "orbm_create");
    }
    return s.h;
}
struct LbaSlot {
    lba_handle* h = nullptr; int maxP = 0, maxL = 0, maxE = 0, device = -1;
    ~LbaSlot() { if (h) lba_destroy(h); }
};
inline lba_handle* lba_handle_for(int nP, int nL, int nE, int device) {
    thread_local LbaSlot s;
    if (!s.h || s.device != device || nP > s.maxP || nL > s.maxL || nE > s.maxE) {
        if (s.h) { lba_destroy(s.h); s.h = nullptr; }
        auto grow = [](int need, int have, int floor_) { int v = need > have ? need + need / 2 : have; return v < floor_ ? floor_ : v; };
        s.maxP = grow(nP, s.maxP, 32); s.maxL = grow(nL, s.maxL, 4096); s.maxE = grow(nE, s.maxE, 32768); s.device = device;
        orb_check(lba_create(&s.h, s.maxP, s.maxL, s.maxE, device), "lba_create");
    }
    return s.h;
}
}  // namespace detail

class ORBmatcher {
public:
    static const int TH_LOW = 50, TH_HIGH = 100, HISTO_LENGTH = 30;   // src/ORBmatcher.cc:35-37
    // ORBmatcher(float nnratio=0.6, bool checkOri=true): two scalars, like the reference -- cheap to construct per use
    ORBmatcher(float nnratio = 0.6, bool checkOri = true, int device = 0) : mfNNratio(nnratio), mbCheckOrientation(checkOri), device_(device) {}

    // static int DescriptorDistance(const cv::Mat& a, const cv::Mat& b): the device popcount is exposed for parity checks; a host caller
    // that needs one distance uses this portable form (the reference's SWAR popcount, src/ORBmatcher.cc:2058-2074)
    static int DescriptorDistance(const uint8_t* a, const uint8_t* b) {
        const uint32_t* pa = reinterpret_cast<const uint32_t*>(a); const uint32_t* pb = reinterpret_cast<const uint32_t*>(b);
        int dist = 0;
        for (int i = 0; i < 8; ++i) { uint32_t v = pa[i] ^ pb[i]; v = v - ((v >> 1) & 0x55555555); v = (v & 0x33333333) + ((v >> 2) & 0x33333333);
                                      dist += (((v + (v >> 4)) & 0xF0F0F0F) * 0x1010101) >> 24; }
        return dist;
    }
    // int SearchByProjection(Frame &F, const vector<MapPoint*> &vpMapPoints, const float th, const bool bFarPoints, const float thFarPoints)
    int SearchByProjection(FrameView& F, const OrbmLocalPoints& vpMapPoints, const float th = 3, const bool bFarPoints = false,
                           const float thFarPoints = 50.0f) {
        prepare(F);
        const OrbmFrame f = F.c_struct();
        int n = 0;
        orb_check(orbm_search_local_map(detail::matcher_handle(f.K, vpMapPoints.M, device_), &f, &vpMapPoints, th, mfNNratio, bFarPoints, thFarPoints,
                                        F.mvpMapPoints.data(), F.mvbClaimed.data(), &n), "orbm_search_local_map");
        return n;
    }
    // int SearchByProjection(Frame &CurrentFrame, const Frame &LastFrame, const float th, const bool bMono)  (mono branch)
    int SearchByProjection(FrameView& CurrentFrame, const OrbmLastFrame& LastFrame, const float Tcw[7], const float cam[4], const float th,
                           const bool bMono) {
        if (!bMono) throw std::invalid_argument("only the monocular branch is accelerated");
        prepare(CurrentFrame);
        const OrbmFrame f = CurrentFrame.c_struct();
        int n = 0;
        orb_check(orbm_search_last_frame(detail::matcher_handle(f.K, LastFrame.M, device_), &f, &LastFrame, Tcw, cam, th, mbCheckOrientation,
                                         CurrentFrame.mvpMapPoints.data(), CurrentFrame.mvbClaimed.data(), &n), "orbm_search_last_frame");
        return n;
    }
    // int SearchForInitialization(Frame &F1, Frame &F2, vector<cv::Point2f> &vbPrevMatched, vector<int> &vnMatches12, int windowSize=10)
    // vbPrevMatched: F1.N x 2 floats (x, y), updated like the reference (src/ORBmatcher.cc:757-759)
    int SearchForInitialization(const FrameView& F1, const FrameView& F2, std::vector<float>& vbPrevMatched, std::vector<int>& vnMatches12,
                                int windowSize = 10) {
        const OrbmFrame f1 = F1.c_struct(), f2 = F2.c_struct();
        if (vbPrevMatched.size() != (size_t)f1.K * 2) throw std::invalid_argument("vbPrevMatched must hold one point per keypoint of F1");
        vnMatches12.assign((size_t)f1.K, -1);
        int n = 0;
        orb_check(orbm_search_for_initialization(detail::matcher_handle(f2.K, f1.K, device_), &f1, &f2, vbPrevMatched.data(), windowSize, mfNNratio,
                                                 mbCheckOrientation, vnMatches12.data(), &n), "orbm_search_for_initialization");
        return n;
    }
    // bool Frame::isInFrustum(MapPoint* pMP, float viewingCosLimit) for all local map points of a frame (Tracking::SearchLocalPoints,
    // src/Tracking.cc:3346): fills the per-point tracking fields that the local-map SearchByProjection above reads.
    struct TrackFields { std::vector<uint8_t> inView; std::vector<float> projX, projY, projXR, depth, viewCos; std::vector<int32_t> level; };
    void isInFrustum(const OrbmFrustumIn& points, TrackFields& out) {
        const size_t M = (size_t)(points.M > 0 ? points.M : 0);
        out.inView.assign(M, 0); out.projX.assign(M, -1.f); out.projY.assign(M, -1.f); out.projXR.assign(M, 0.f); out.depth.assign(M, 0.f);
        out.viewCos.assign(M, 0.f); out.level.assign(M, -1);
        if (!M) return;
        orb_check(orbm_frustum_project(detail::matcher_handle(1, points.M, device_), &points, out.inView.data(), out.projX.data(), out.projY.data(),
                                       out.projXR.data(), out.depth.data(), out.level.data(), out.viewCos.data()), "orbm_frustum_project");
    }
    // The searches of int Fuse(KeyFrame* pKF, const vector<MapPoint*>& vpMapPoints, const float th = 3.0) for several keyframes in one launch
    // (orbm_fuse_search_batch): one round of LocalMapping::SearchInNeighbors for keyframes of DIFFERENT maps (INTEGRATION.md §2).  Every
    // item's bestIdx / bestDist receive its search; the caller walks them in map-point order (src/ORBmatcher.cc:1310-1330), re-testing
    // isBad() / IsInKeyFrame(pKF) when it reaches a point.
    void FuseBatch(const std::vector<OrbmFuseItem>& items) {
        int maxK = 1;
        for (const OrbmFuseItem& it : items) if (it.KF.K > maxK) maxK = it.KF.K;
        orb_check(orbm_fuse_search_batch(detail::matcher_handle(maxK, 1, device_), (int)items.size(), items.data()), "orbm_fuse_search_batch");
    }
    // void LocalMapping::CreateNewMapPoints() (monocular, the vpNeighKFs loop) for several new keyframes of DIFFERENT maps in three launches
    // (orbm_create_new_map_points_batch).  Every item's out / nNew / nmatches / ncreated receive exactly what orbm_create_new_map_points
    // gives it alone; the caller picks the neighbours, cuts a list to one entry when CheckNewKeyFrames() holds, and replays the records in
    // order (INTEGRATION.md §2).
    void CreateNewMapPointsBatch(const std::vector<OrbmNewPointsItem>& items) {
        orb_check(orbm_create_new_map_points_batch(detail::matcher_handle(1, 1, device_), (int)items.size(), items.data()),
                  "orbm_create_new_map_points_batch");
    }
    // void LocalMapping::KeyFrameCulling() (monocular and mono-inertial) for several maps that share nothing, in one launch
    // (orbm_keyframe_culling_batch).  Every map's status / nMPs / nRedundant / visited receive its walk; the caller replays the culls in
    // status order: MergePrevious, the relink and SetBadFlag (INTEGRATION.md §2).
    void KeyFrameCullingBatch(const std::vector<OrbmCullingMap>& maps) {
        orb_check(orbm_keyframe_culling_batch(detail::matcher_handle(1, 1, device_), (int)maps.size(), maps.data()), "orbm_keyframe_culling_batch");
    }
    // LoopClosing::DetectCommonRegionsFromBoW up to the Sim3Solver for several place-recognition queries in two launches
    // (orbm_common_regions_bow_batch): every query's outputs receive each candidate's status, vpCovKFi, the SearchByBoW counts, numBoWMatches
    // and the merged vpKeyFrameMatchedMP / vpMatchedPoints; the caller replays them and keeps the reference's text from
    // `if(numBoWMatches >= nBoWMatches)` on (INTEGRATION.md §2).  The searches use the reference's ORBmatcher(0.9, true), whatever this
    // object's settings.
    void CommonRegionsBoWBatch(const std::vector<OrbmCommonRegionsQuery>& queries) {
        int maxK = 1, maxM = 1;
        for (const OrbmCommonRegionsQuery& q : queries)
            for (int e = 0; q.kf && e < q.nKF; ++e) {
                int& need = e == 0 ? maxM : maxK;
                if (q.kf[e].frame.N > need) need = q.kf[e].frame.N;
            }
        orb_check(orbm_common_regions_bow_batch(detail::matcher_handle(maxK, maxM, device_), (int)queries.size(), queries.data()),
                  "orbm_common_regions_bow_batch");
    }
    // Tracking::UpdateLocalMap's UpdateLocalKeyFrames and UpdateLocalPoints for a batch of streams in one launch (orbm_update_local_map_batch).
    // `out` receives every stream's local keyframes, reference keyframe and local points, and the local map in the slabs of
    // OrbmLocalMapBatch; the caller replays the marks, mpReferenceKF and the NULLing of the voting frame's bad points (INTEGRATION.md §2).
    void UpdateLocalMapBatch(const OrbmUpdateLocalMapBatch& in, const OrbmUpdateLocalMapResult& out) {
        orb_check(orbm_update_local_map_batch(detail::matcher_handle(1, 1, device_), &in, &out), "orbm_update_local_map_batch");
    }
    // LocalMapping::ProcessNewKeyFrame's map-point loop or the tail of SearchInNeighbors, each followed by KeyFrame::UpdateConnections, for
    // several keyframes of different maps in one launch (orbm_update_connections_batch).  Every item's outputs receive its result; the caller
    // replays it on the host: AddObservation, the point fields, mlpRecentAddedMapPoints, the connection maps and lists, AddChild
    // (INTEGRATION.md §2).
    void UpdateConnectionsBatch(const std::vector<OrbmConnectionsItem>& items) {
        orb_check(orbm_update_connections_batch(detail::matcher_handle(1, 1, device_), (int)items.size(), items.data()), "orbm_update_connections_batch");
    }
    // cv::BFMatcher(NORM_HAMMING).knnMatch(query, train, matches, 2)
    void knnMatch(const Descriptors& query, const Descriptors& train, std::vector<int32_t>& idx, std::vector<int32_t>& dist) {
        idx.assign((size_t)query.rows * 2, -1); dist.assign((size_t)query.rows * 2, -1);
        orb_check(orbm_bf_knn2(detail::matcher_handle(query.rows, train.rows, device_), query.data.data(), query.rows, train.data.data(), train.rows,
                               idx.data(), dist.data()), "orbm_bf_knn2");
    }

protected:
    static void prepare(FrameView& F) {
        if (F.mvpMapPoints.size() != F.mvKeysUn.size()) F.mvpMapPoints.assign(F.mvKeysUn.size(), -1);
        if (F.mvbClaimed.size() != F.mvKeysUn.size()) F.mvbClaimed.assign(F.mvKeysUn.size(), 0);
    }
    float mfNNratio;
    bool mbCheckOrientation;
    int device_;
};

// Tracking's per-frame steps after the last-frame search for a batch of streams (INTEGRATION.md §2): monocular with the IMU not
// initialised, TrackWithMotionModel's PoseOptimization + "discard outliers" loop, TrackReferenceKeyFrame, and TrackLocalMap from SearchLocalPoints through the
// statistics loop; monocular-inertial with the IMU initialised, PredictStateIMU and TrackLocalMap with the inertial pose optimisers.
// Unlike ORBmatcher above it owns its matcher handle, sized for the batch; host pointers throughout.
class BatchTracker {
public:
    BatchTracker(int max_batch, int max_keypoints, int max_mappoints, int device = 0) {
        orb_check(orbm_create(&h_, max_batch, max_keypoints, max_mappoints, device), "orbm_create");
    }
    ~BatchTracker() { if (h_) orbm_destroy(h_); }
    BatchTracker(const BatchTracker&) = delete;
    BatchTracker& operator=(const BatchTracker&) = delete;
    // in: the slabs of orbm_search_last_frame_batch; match / claimed / nmatches: what that search wrote (updated in place)
    void MotionModelPose(const OrbmBatchDevice& in, const float* invLevelSigma2, const uint8_t* active, int32_t* match, uint8_t* claimed,
                         int32_t* nmatches, double* pose7, float* Tcw7, uint8_t* discarded, int32_t* nmatchesMap) {
        orb_check(orbm_motion_model_pose_batch(h_, &in, invLevelSigma2, active, match, claimed, nmatches, pose7, Tcw7, discarded, nmatchesMap),
                  "orbm_motion_model_pose_batch");
    }
    void TrackLocalMap(const OrbmLocalMapBatch& in, const OrbmLocalMapResult& out) {
        orb_check(orbm_track_local_map_batch(h_, &in, &out), "orbm_track_local_map_batch");
    }
    // Tracking::TrackReferenceKeyFrame after Frame::ComputeBoW (the frame's FeatureVector from orbv_transform_batch): SearchByBoW, the
    // 15-match gate, PoseOptimization from in.Tcw7 and the "discard outliers" loop.  The caller applies nmatchesMap >= 10 (monocular)
    // and feeds out.match / out.discarded to TrackLocalMap in the index space [keyframe features | last-frame points].
    void TrackReferenceKeyFrame(const OrbmRefKeyFrameBatch& in, const OrbmRefKeyFrameResult& out) {
        orb_check(orbm_track_reference_keyframe_batch(h_, &in, &out), "orbm_track_reference_keyframe_batch");
    }
    // Monocular-inertial frames once the IMU is initialised: PredictStateIMU, SearchLocalPoints, PoseInertialOptimizationLast{KeyFrame,Frame}
    // and its write-back for every stream with imu.mode != 0 (in.Tcw7 / lastToLocal / discarded / active and out.pose7 NULL).  Feed
    // imuOut.state21 / prior21 / priorH back as the next call's lastState21 / prior21 / priorH.
    void TrackLocalMapInertial(const OrbmLocalMapBatch& in, const OrbmImuTrackBatch& imu, const OrbmLocalMapResult& out, const OrbmImuTrackResult& imuOut) {
        orb_check(orbm_track_local_map_inertial_batch(h_, &in, &imu, &out, &imuOut), "orbm_track_local_map_inertial_batch");
    }
    int LastLaunchCount() const { return orbm_last_launch_count(h_); }

private:
    orbm_handle* h_ = nullptr;
};

class Optimizer {
public:
    // void static LocalBundleAdjustment(KeyFrame* pKF, bool* pbStopFlag, Map* pMap, int& num_fixedKF, int& num_OptKF, int& num_MPs, int& num_edges)
    // The pointer-graph walk (src/Optimizer.cc:1125-1403) and the write-back (:1464-1497) stay with the caller; this is
    // optimizer.initializeOptimization(); optimizer.optimize(10); and the values the outlier test at :1417-1430 reads.
    // graph.stopFlag takes the caller's own `bool* pbStopFlag` (one byte).  The device arena is kept per thread and reused.
    static void LocalBundleAdjustment(const LbaProblem& graph, LbaResult& out, int device = 0) {
        if (graph.stopFlag && *graph.stopFlag) return;               // :1406-1408
        orb_check(lba_solve(detail::lba_handle_for(graph.nPoses, graph.nPoints > 0 ? graph.nPoints : 1, graph.nEdges > 0 ? graph.nEdges : 1, device),
                            &graph, &out), "lba_solve");
    }
    // The same function as a whole, walk, erase cascade and write-back included, for a batch of maps (one keyframe each): each LbaLocalMap
    // is the flattened map and receives the record the host replays (include/orb_b200.h, INTEGRATION.md §3).  h is sized for the largest
    // built problem and for nMaps (lba_create_batch).
    static void LocalBundleAdjustmentBatch(lba_handle* h, int nMaps, const LbaLocalMap* maps) {
        orb_check(lba_local_bundle_adjustment_batch(h, nMaps, maps), "lba_local_bundle_adjustment_batch");
    }
    // int static PoseOptimization(Frame* pFrame)  (src/Optimizer.cc:814-1113, monocular branch): the caller flattens the frame's map
    // point associations (:862-905); returns nInitialCorrespondences - nBad, writes the pose and the outlier flags.
    static int PoseOptimization(int N, const double pose7[7], const float cam4[4], const double* Xw, const double* obs, const float* invSigma2,
                                double poseOut[7], uint8_t* mvbOutlier, int device = 0) {
        int32_t n = N, inliers = 0;
        orb_check(pose_optimization_batch(1, N > 0 ? N : 1, &n, pose7, cam4, Xw, obs, invSigma2, (double)(float)std::sqrt(5.991) /* deltaMono, :852 */, poseOut, mvbOutlier, &inliers, device),
                  "pose_optimization_batch");
        return inliers;
    }
    // void static LocalInertialBA(KeyFrame* pKF, bool* pbStopFlag, Map* pMap, int& num_fixedKF, int& num_OptKF, int& num_MPs, int& num_edges,
    //                             bool bLarge = false, bool bRecInit = false)   (include/Optimizer.h:62, src/Optimizer.cc:2383-2958)
    // The caller keeps the graph walk (:2385-2478, :2690-2833) and the write-back (:2890-2957); `graph` is the flattened window (LocalInertialBAProblem:
    // the temporal window first, newest keyframe first like vpOptimizableKFs, then lFixedKeyFrames) and `out` receives what SetPose / SetVelocity /
    // SetNewBias / SetWorldPos take plus the vToErase flags.  bLarge / bRecInit choose the iteration count, the initial lambda and which inertial
    // edges carry the Huber kernel exactly as :2387-2394, :2497-2509, :2633-2643 do; the reference sets the stop flag only after optimize() (:2840),
    // so pbStopFlag never interrupts this solve.  Returns false on "FAIL LOCAL-INERTIAL BA" (:2884-2888: nothing is to be written back).
    static bool LocalInertialBA(LocalInertialBAProblem graph, LocalInertialBAResult& out, bool bLarge = false, bool bRecInit = false, int device = 0) {
        const int N = graph.nInertial;
        std::vector<uint8_t> robust((size_t)(N > 0 ? N : 1), 0);
        std::vector<double> scale((size_t)(N > 0 ? N : 1), 1.0);
        for (int i = 0; i < N; ++i) {                                  // i == N-1: the link to the fixed keyframe (vpOptimizableKFs order)
            robust[i] = (i == N - 1 || bRecInit) ? 1 : 0;
            scale[i] = (i == N - 1) ? 1e-2 : 1.0;
        }
        graph.ieRobust = robust.data(); graph.ieInfoScale = scale.data();
        graph.iterations = bLarge ? 4 : 10; graph.lambdaInit = bLarge ? 1e-2 : 1e0; graph.bLarge = bLarge ? 1 : 0;
        double stats[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        LocalInertialBAResult r = out;
        if (!r.stats8) r.stats8 = stats;
        orb_check(local_inertial_ba_batch(1, &graph, &r, nullptr, device), "local_inertial_ba_batch");
        return r.stats8[2] == 0.0;
    }
    // The same function as a whole -- window walk, solve, erase cascade and write-back -- for a batch of maps (one keyframe each): each
    // LocalInertialBAMap is the flattened map and receives the record the host replays (include/orb_b200.h, INTEGRATION.md §3).  Like
    // LocalInertialBA it needs no handle; the staging is the calling thread's.
    static void LocalInertialBABatch(int nMaps, const LocalInertialBAMap* maps, int device = 0) {
        orb_check(local_inertial_ba_map_batch(nMaps, maps, device), "local_inertial_ba_map_batch");
    }
};

// KeyFrameDatabase over caller keys (such as (uint64_t)KeyFrame*), the inverted file resident on the device; one object serves
// maxDatabases databases, one per SLAM system.  add / erase / clear are the reference's members for one database; clearMap(pMap) is
// erase of the map's keyframes.  QueryBatch runs phase 1 of DetectRelocalizationCandidates / DetectNBestCandidates for a batch of
// queries; the caller replays the records onto its keyframes and keeps the reference's phase 2 (INTEGRATION.md §2).  The reference's
// mMutex stays with the caller: Tracking and LoopClosing share one database.
class KeyFrameDatabase {
public:
    struct BowVector { std::vector<int32_t> id; std::vector<double> value; };   // DBoW2::BowVector in map order
    KeyFrameDatabase(int vocabularyWords, int maxDatabases, int maxKeyFrames, int maxWords, int device = 0) {
        orb_check(orbv_db_create(&h_, vocabularyWords, maxDatabases, maxKeyFrames, maxWords, device), "orbv_db_create");
    }
    ~KeyFrameDatabase() { orbv_db_destroy(h_); }
    KeyFrameDatabase(const KeyFrameDatabase&) = delete;
    KeyFrameDatabase& operator=(const KeyFrameDatabase&) = delete;

    void add(int db, uint64_t key, const BowVector& bow) { add(std::vector<int32_t>{db}, std::vector<uint64_t>{key}, std::vector<BowVector>{bow}); }
    // add(pKF) for each keyframe, in order
    void add(const std::vector<int32_t>& db, const std::vector<uint64_t>& keys, const std::vector<BowVector>& bows) {
        std::vector<int32_t> start(1, 0), id;
        std::vector<double> value;
        for (const BowVector& b : bows) {
            id.insert(id.end(), b.id.begin(), b.id.end());
            value.insert(value.end(), b.value.begin(), b.value.end());
            start.push_back((int32_t)id.size());
        }
        orb_check(orbv_db_add_batch(h_, (int)keys.size(), db.data(), keys.data(), start.data(), id.data(), value.data()), "orbv_db_add_batch");
    }
    void erase(int db, uint64_t key) { erase(std::vector<int32_t>{db}, std::vector<uint64_t>{key}); }
    void erase(const std::vector<int32_t>& db, const std::vector<uint64_t>& keys) {
        orb_check(orbv_db_erase_batch(h_, (int)keys.size(), db.data(), keys.data()), "orbv_db_erase_batch");
    }
    void clear(int db) { orb_check(orbv_db_clear(h_, db), "orbv_db_clear"); }
    void QueryBatch(const std::vector<OrbvDbQuery>& queries) {
        orb_check(orbv_db_query_batch(h_, (int)queries.size(), queries.data()), "orbv_db_query_batch");
    }
    orbv_db_handle* handle() { return h_; }

private:
    orbv_db_handle* h_ = nullptr;
};

}  // namespace ORB_SLAM3
