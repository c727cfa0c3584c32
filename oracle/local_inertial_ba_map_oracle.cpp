// TEST INFRASTRUCTURE ONLY -- CPU oracle of Optimizer::LocalInertialBA (src/Optimizer.cc:2383-2958, monocular observations, maxCovKF = 0) as
// a whole, a literal transcription over a small pointer map rebuilt from the flattened input (LocalInertialBAMap, include/orb_b200.h):
// keyframes with mPrevKF, bImu, mpImuPreintegrated, mnBALocalForKF / mnBAFixedForKF and their slots; map points with mObservations (a list
// in the caller's key order, which is the std::map's iteration order), nObs, mpRefKF, mTrackDepth and the bad flag.  The solve is
// orbo_local_inertial_ba (local_inertial_ba_oracle.cpp) on the problem the walk builds (the window newest first, then lFixedKeyFrames; points
// in list order; edges in insertion order).  The erase loop follows MapPoint::EraseObservation / SetBadFlag, the write-back
// Sophus::SE3f(Rcw.cast<float>(), tcw.cast<float>()) (Eigen's matrix-to-quaternion conversion, csrc/frame_pose.cuh), GetCameraCenter,
// SetVelocity, SetNewBias and UpdateNormalAndDepth.  Built with -ffp-contract=off: every float operation rounds once, as the kernels do.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <list>
#include <utility>
#include <vector>

extern "C" int orbo_local_inertial_ba(int nKF, int nOpt, double* kfState21, double* kfTcw12, const float* cam4, const double* extr24, int nI, const int* ieKf1,
                                      const int* ieKf2, const float* preint, const uint8_t* ieRobust, const double* ieInfoScale, int nL, double* points3,
                                      const float* trackDepth, int nE, const int* ePt, const int* eKf, const double* obs2, const float* invSigma2, int iterations,
                                      double lambdaInit, int bLarge, uint8_t* eraseOut, double* edgeChi2Out, double* stats);

extern "C" {
// Layout-compatible with LocalInertialBAMap (include/orb_b200.h).
typedef struct OrboLiMap {
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
} OrboLiMap;

// The LocalInertialBAProblem the walk hands to the optimiser (capacity: nKF keyframes and inertial edges, nPoints points, obsStart[nPoints]
// edges); sizes = nKF, nOpt, nInertial, nPoints, nEdges, iterations; lambdaInit [1].
typedef struct OrboLiBuilt {
    double* kfState21; double* kfTcw12; float* cam4; int32_t* ieKf1; int32_t* ieKf2; float* preint; uint8_t* ieRobust; double* ieInfoScale;
    double* points3; float* trackDepth; int32_t* edgePoint; int32_t* edgeKf; double* obs2; float* invSigma2; int32_t* sizes; double* lambdaInit;
} OrboLiBuilt;
}

namespace {

enum { KF_BAD = 1, KF_OTHER_MAP = 8, KF_IMU = 16, KF_PREINT = 32 };
enum { OBS_NO_EDGE = 0, OBS_KEPT = 1, OBS_ERASED = 2 };
const int P_SIZE = 292;
const uint64_t ID = 1;        // pKF->mnId as the marks carry it (no mark carries it at the call; the reference resets marks to 0)

struct MapPoint;
struct KeyFrame {
    int idx; bool bad, otherMap, bImu, preint;
    KeyFrame* mPrevKF = nullptr;
    float Ow[3];
    uint64_t mnBALocalForKF = 0, mnBAFixedForKF = 0;
    std::vector<MapPoint*> slots;
};
struct MapPoint {
    int idx; bool bad;
    float pos[3], mTrackDepth;
    std::vector<std::pair<KeyFrame*, int>> obs;   // mObservations: keyframe, row of the flattened observation
    int nObs;
    KeyFrame* ref;
    uint64_t mnBALocalForKF = 0;
    float normal[3] = {0, 0, 0}, minD = 0, maxD = 0;
};

float norm3(float x, float y, float z) { return std::sqrt((x * x + y * y) + z * z); }

// Sophus::SE3f(Matrix3f R, Vector3f t): Eigen's quaternion from a rotation matrix (R row-major), T = (w, x, y, z, t); then GetCameraCenter =
// -(q^-1 * t) with Sophus' rotation (csrc/frame_pose.cuh: se3_from_matrix, update_pose_matrices)
void set_pose(const float* R, const float* t, float* T, float* Ow) {
    float tr = (R[0] + R[4]) + R[8];
    if (tr > 0) {
        tr = std::sqrt(tr + 1.0f);
        T[0] = 0.5f * tr; tr = 0.5f / tr;
        T[1] = (R[7] - R[5]) * tr; T[2] = (R[2] - R[6]) * tr; T[3] = (R[3] - R[1]) * tr;
    } else {
        int i = 0;
        if (R[4] > R[0]) i = 1;
        if (R[8] > R[i * 4]) i = 2;
        const int j = (i + 1) % 3, k = (j + 1) % 3;
        tr = std::sqrt(((R[i * 4] - R[j * 4]) - R[k * 4]) + 1.0f);
        float q[3];
        q[i] = 0.5f * tr; tr = 0.5f / tr;
        T[0] = (R[k * 3 + j] - R[j * 3 + k]) * tr;
        q[j] = (R[j * 3 + i] + R[i * 3 + j]) * tr; q[k] = (R[k * 3 + i] + R[i * 3 + k]) * tr;
        T[1] = q[0]; T[2] = q[1]; T[3] = q[2];
    }
    T[4] = t[0]; T[5] = t[1]; T[6] = t[2];
    const float qw = T[0], ix = -T[1], iy = -T[2], iz = -T[3], px = T[4], py = T[5], pz = T[6];
    float ux = iy * pz - iz * py, uy = iz * px - ix * pz, uz = ix * py - iy * px;
    ux = ux + ux; uy = uy + uy; uz = uz + uz;
    const float cx = iy * uz - iz * uy, cy = iz * ux - ix * uz, cz = ix * uy - iy * ux;
    Ow[0] = -((px + qw * ux) + cx); Ow[1] = -((py + qw * uy) + cy); Ow[2] = -((pz + qw * uz) + cz);
}

struct Run {
    const OrboLiMap& m;
    std::vector<KeyFrame> kfs;
    std::vector<MapPoint> pts;
    explicit Run(const OrboLiMap& mm) : m(mm) {
        kfs.resize(m.nKF);
        for (int k = 0; k < m.nKF; ++k) {
            KeyFrame& K = kfs[k];
            K.idx = k; K.bad = m.kfFlags[k] & KF_BAD; K.otherMap = m.kfFlags[k] & KF_OTHER_MAP; K.bImu = m.kfFlags[k] & KF_IMU;
            K.preint = m.kfFlags[k] & KF_PREINT;
            K.mPrevKF = m.prevKF[k] >= 0 ? &kfs[m.prevKF[k]] : nullptr;
            std::memcpy(K.Ow, m.cameraCenter + 3 * k, 12);
        }
        pts.resize(m.nPoints);
        for (int p = 0; p < m.nPoints; ++p) {
            MapPoint& P = pts[p];
            P.idx = p; P.bad = m.pointFlags[p] & KF_BAD; P.mTrackDepth = m.trackDepth[p];
            std::memcpy(P.pos, m.worldPos + 3 * p, 12);
            for (int o = m.obsStart[p]; o < m.obsStart[p + 1]; ++o) P.obs.push_back({&kfs[m.obsKF[o]], o});
            P.nObs = (int)P.obs.size();
            P.ref = m.refKF[p] >= 0 ? &kfs[m.refKF[p]] : nullptr;
        }
        for (int k = 0; k < m.nKF; ++k)
            for (int s = m.slotStart[k]; s < m.slotStart[k + 1]; ++s) kfs[k].slots.push_back(m.slotPoint[s] >= 0 ? &pts[m.slotPoint[s]] : nullptr);
    }
    void EraseObservation(MapPoint* p, KeyFrame* k) {
        bool bBad = false;
        auto it = std::find_if(p->obs.begin(), p->obs.end(), [&](const std::pair<KeyFrame*, int>& e) { return e.first == k; });
        if (it != p->obs.end()) {
            p->nObs--;                                              // monocular observation
            p->obs.erase(it);
            if (p->ref == k) p->ref = p->obs.empty() ? nullptr : p->obs.begin()->first;
            if (p->nObs <= 2) bBad = true;
        }
        if (bBad) { p->bad = true; p->obs.clear(); }               // SetBadFlag (the keyframes' slots are the replay's)
    }
    void UpdateNormalAndDepth(MapPoint* p) {
        if (p->bad || p->obs.empty()) return;
        float normal[3] = {0, 0, 0};
        int n = 0, level = 0;
        for (auto& e : p->obs) {
            const KeyFrame* K = e.first;
            const float v[3] = {p->pos[0] - K->Ow[0], p->pos[1] - K->Ow[1], p->pos[2] - K->Ow[2]};
            const float d = norm3(v[0], v[1], v[2]);
            for (int i = 0; i < 3; ++i) normal[i] = normal[i] + v[i] / d;
            ++n;
            if (K == p->ref) level = m.obsOctave[e.second];
        }
        const KeyFrame* r = p->ref;
        const float dist = norm3(p->pos[0] - r->Ow[0], p->pos[1] - r->Ow[1], p->pos[2] - r->Ow[2]);
        p->maxD = dist * m.scaleFactors[level];
        p->minD = p->maxD / m.scaleFactors[m.nlevels - 1];
        for (int i = 0; i < 3; ++i) p->normal[i] = normal[i] / (float)n;
    }

    int run(bool given, OrboLiBuilt* built) {
        const int nObsAll = m.nPoints ? m.obsStart[m.nPoints] : 0;
        for (int k = 0; k < m.nKF; ++k) {
            m.optKF[k] = m.fixedKF[k] = -1; m.ieLinked[k] = 0;
            for (int c = 0; c < 7; ++c) m.kfPose7[7 * k + c] = 0;
            for (int c = 0; c < 3; ++c) m.kfCenter[3 * k + c] = m.kfVelocity[3 * k + c] = 0;
            for (int c = 0; c < 6; ++c) m.kfBias6[6 * k + c] = 0;
        }
        for (int p = 0; p < m.nPoints; ++p) {
            m.localPoint[p] = -1; m.pointBad[p] = 0; m.pointRefKF[p] = -1; m.minDistance[p] = m.maxDistance[p] = 0;
            for (int c = 0; c < 3; ++c) m.pointPos[3 * p + c] = m.normal[3 * p + c] = 0;
        }
        for (int o = 0; o < nObsAll; ++o) m.obsFlag[o] = OBS_NO_EDGE;
        KeyFrame* pKF = &kfs[0];
        // :2385-2394
        int maxOpt = 10, opt_it = 10;
        if (m.bLarge) { maxOpt = 25; opt_it = 4; }
        const int Nd = std::min(m.keyFramesInMap - 2, maxOpt);
        // :2395-2410
        std::vector<KeyFrame*> vpOptimizableKFs;
        vpOptimizableKFs.push_back(pKF);
        pKF->mnBALocalForKF = ID;
        for (int i = 1; i < Nd; i++) {
            if (vpOptimizableKFs.back()->mPrevKF) {
                vpOptimizableKFs.push_back(vpOptimizableKFs.back()->mPrevKF);
                vpOptimizableKFs.back()->mnBALocalForKF = ID;
            } else
                break;
        }
        int N = (int)vpOptimizableKFs.size();
        // :2413-2428
        std::list<MapPoint*> lLocalMapPoints;
        for (int i = 0; i < N; i++)
            for (MapPoint* pMP : vpOptimizableKFs[i]->slots)
                if (pMP && !pMP->bad && pMP->mnBALocalForKF != ID) { lLocalMapPoints.push_back(pMP); pMP->mnBALocalForKF = ID; }
        // :2431-2442
        std::list<KeyFrame*> lFixedKeyFrames;
        if (vpOptimizableKFs.back()->mPrevKF) {
            lFixedKeyFrames.push_back(vpOptimizableKFs.back()->mPrevKF);
            vpOptimizableKFs.back()->mPrevKF->mnBAFixedForKF = ID;
        } else {
            vpOptimizableKFs.back()->mnBALocalForKF = 0;
            vpOptimizableKFs.back()->mnBAFixedForKF = ID;
            lFixedKeyFrames.push_back(vpOptimizableKFs.back());
            vpOptimizableKFs.pop_back();
        }
        // :2444-2456: maxCovKF = 0, so lpOptVisKFs stays empty.  :2458-2478
        const size_t maxFixKF = 200;
        for (MapPoint* pMP : lLocalMapPoints) {
            for (auto& e : pMP->obs) {
                KeyFrame* pKFi = e.first;
                if (pKFi->mnBALocalForKF != ID && pKFi->mnBAFixedForKF != ID) {
                    pKFi->mnBAFixedForKF = ID;
                    if (!pKFi->bad) { lFixedKeyFrames.push_back(pKFi); break; }
                }
            }
            if (lFixedKeyFrames.size() >= maxFixKF) break;
        }
        // the problem: vertices of the window, then of lFixedKeyFrames (:2512-2590)
        N = (int)vpOptimizableKFs.size();
        std::vector<KeyFrame*> vk(vpOptimizableKFs);
        vk.insert(vk.end(), lFixedKeyFrames.begin(), lFixedKeyFrames.end());
        const int nK = (int)vk.size();
        std::vector<int> kfIndex(m.nKF, -1);
        std::vector<double> state(21 * (size_t)nK), tcw(12 * (size_t)nK);
        std::vector<float> cam(4 * (size_t)nK);
        for (int v = 0; v < nK; ++v) {
            const int k = vk[v]->idx;
            kfIndex[k] = v;
            for (int c = 0; c < 21; ++c) state[21 * v + c] = (double)m.state21[21 * k + c];
            for (int c = 0; c < 12; ++c) tcw[12 * v + c] = (double)m.tcw12[12 * k + c];
            for (int c = 0; c < 4; ++c) cam[4 * v + c] = m.cam4[4 * k + c];
        }
        // inertial edges (:2593-2656), keyed on the window index
        std::vector<int> ie1, ie2;
        std::vector<float> preint;
        std::vector<uint8_t> robust;
        std::vector<double> scale;
        for (int i = 0; i < N; i++) {
            KeyFrame* pKFi = vpOptimizableKFs[i];
            if (!pKFi->mPrevKF) continue;                                      // "NOT INERTIAL LINK TO PREVIOUS FRAME!!!!"
            if (pKFi->bImu && pKFi->mPrevKF->bImu && pKFi->preint) {
                m.ieLinked[i] = 1;                                             // mpImuPreintegrated->SetNewBias(mPrevKF->GetImuBias())
                ie1.push_back(kfIndex[pKFi->mPrevKF->idx]); ie2.push_back(i);
                preint.insert(preint.end(), m.preint + (size_t)P_SIZE * pKFi->idx, m.preint + (size_t)P_SIZE * (pKFi->idx + 1));
                robust.push_back(i == N - 1 || m.bRecInit ? 1 : 0);
                scale.push_back(i == N - 1 ? 1e-2 : 1.0);
            }
        }
        const int nI = (int)ie1.size();
        // points and mono edges (:2690-2763)
        std::vector<MapPoint*> vp(lLocalMapPoints.begin(), lLocalMapPoints.end());
        const int nL = (int)vp.size();
        std::vector<double> points(3 * (size_t)nL);
        std::vector<float> td(nL);
        std::vector<int> ePt, eKf, eObs;
        std::vector<double> obs;
        std::vector<float> isg;
        for (int r = 0; r < nL; ++r) {
            MapPoint* pMP = vp[r];
            for (int c = 0; c < 3; ++c) points[3 * r + c] = (double)pMP->pos[c];
            td[r] = pMP->mTrackDepth;
            for (auto& e : pMP->obs) {
                KeyFrame* pKFi = e.first;
                if (pKFi->mnBALocalForKF != ID && pKFi->mnBAFixedForKF != ID) continue;
                if (pKFi->bad || pKFi->otherMap) continue;
                const int o = e.second;
                ePt.push_back(r); eKf.push_back(kfIndex[pKFi->idx]);
                obs.push_back((double)m.obsPt[2 * o]); obs.push_back((double)m.obsPt[2 * o + 1]);
                isg.push_back(m.invLevelSigma2[m.obsOctave[o]] / 1.0f);         // / uncertainty2, 1 for Pinhole
                eObs.push_back(o);
            }
        }
        const int nE = (int)ePt.size();
        const double lambdaInit = m.bLarge ? 1e-2 : 1e0;
        int i = 0;
        for (KeyFrame* k : vpOptimizableKFs) m.optKF[i++] = k->idx;
        i = 0;
        for (KeyFrame* k : lFixedKeyFrames) m.fixedKF[i++] = k->idx;
        for (int r = 0; r < nL; ++r) m.localPoint[r] = vp[r]->idx;
        m.nLists[0] = N; m.nLists[1] = (int)lFixedKeyFrames.size(); m.nLists[2] = nL; m.nLists[3] = nE;
        if (built) {
            std::memcpy(built->kfState21, state.data(), 8 * state.size()); std::memcpy(built->kfTcw12, tcw.data(), 8 * tcw.size());
            std::memcpy(built->cam4, cam.data(), 4 * cam.size());
            std::memcpy(built->ieKf1, ie1.data(), 4 * (size_t)nI); std::memcpy(built->ieKf2, ie2.data(), 4 * (size_t)nI);
            std::memcpy(built->preint, preint.data(), 4 * preint.size()); std::memcpy(built->ieRobust, robust.data(), nI);
            std::memcpy(built->ieInfoScale, scale.data(), 8 * (size_t)nI);
            std::memcpy(built->points3, points.data(), 8 * points.size()); std::memcpy(built->trackDepth, td.data(), 4 * (size_t)nL);
            std::memcpy(built->edgePoint, ePt.data(), 4 * (size_t)nE); std::memcpy(built->edgeKf, eKf.data(), 4 * (size_t)nE);
            std::memcpy(built->obs2, obs.data(), 8 * obs.size()); std::memcpy(built->invSigma2, isg.data(), 4 * (size_t)nE);
            const int sz[6] = {nK, N, nI, nL, nE, opt_it};
            std::memcpy(built->sizes, sz, sizeof(sz));
            *built->lambdaInit = lambdaInit;
        }
        // the solve (:2836-2839): err, optimize(opt_it), err_end; or the given results
        std::vector<double> chi2(nE, 0.0);
        bool failed;
        if (given) {
            for (int v = 0; v < nK; ++v) {
                for (int c = 0; c < 21; ++c) state[21 * v + c] = m.optState21[21 * v + c];
                for (int c = 0; c < 12; ++c) tcw[12 * v + c] = m.optTcw12[12 * v + c];
            }
            for (int r = 0; r < nL; ++r) for (int c = 0; c < 3; ++c) points[3 * r + c] = m.optPoint[3 * r + c];
            for (int e = 0; e < nE; ++e) chi2[e] = m.edgeChi2[eObs[e]];
            failed = m.stats8[2] != 0.0;
        } else {
            std::vector<uint8_t> erase(nE);
            orbo_local_inertial_ba(nK, N, state.data(), tcw.data(), cam.data(), m.extrinsics24, nI, ie1.data(), ie2.data(), preint.data(), robust.data(),
                                   scale.data(), nL, points.data(), td.data(), nE, ePt.data(), eKf.data(), obs.data(), isg.data(), opt_it, lambdaInit,
                                   m.bLarge, erase.data(), chi2.data(), m.stats8);
            failed = m.stats8[2] != 0.0;
            if (m.edgeChi2) {
                for (int o = 0; o < nObsAll; ++o) m.edgeChi2[o] = 0.0;
                for (int e = 0; e < nE; ++e) m.edgeChi2[eObs[e]] = chi2[e];
                for (int v = 0; v < m.nKF; ++v) {
                    for (int c = 0; c < 21; ++c) m.optState21[21 * v + c] = !failed && v < nK ? state[21 * v + c] : 0.0;
                    for (int c = 0; c < 12; ++c) m.optTcw12[12 * v + c] = !failed && v < nK ? tcw[12 * v + c] : 0.0;
                }
                for (int p = 0; p < m.nPoints; ++p) for (int c = 0; c < 3; ++c) m.optPoint[3 * p + c] = !failed && p < nL ? points[3 * p + c] : 0.0;
            }
        }
        for (int e = 0; e < nE; ++e) m.obsFlag[eObs[e]] = OBS_KEPT;
        // Check inlier observations (:2848-2862)
        const float chi2Mono2 = 5.991f;
        std::vector<std::pair<KeyFrame*, MapPoint*>> vToErase;
        std::vector<int> eraseObs;                     // the flattened observation of each vToErase pair
        for (int e = 0; e < nE; ++e) {
            MapPoint* pMP = vp[ePt[e]];
            const bool bClose = pMP->mTrackDepth < 10.f;
            if (pMP->bad) continue;
            const double* T = &tcw[12 * (size_t)eKf[e]];
            const double* X = &points[3 * (size_t)ePt[e]];
            const bool depthPositive = (T[6] * X[0] + T[7] * X[1] + T[8] * X[2] + T[11]) > 0.0;   // EdgeMono::isDepthPositive
            if ((chi2[e] > chi2Mono2 && !bClose) || (chi2[e] > 1.5f * chi2Mono2 && bClose) || !depthPositive)
            { vToErase.push_back({&kfs[m.obsKF[eObs[e]]], pMP}); eraseObs.push_back(eObs[e]); }
        }
        // :2884-2888: FAIL returns with the lock taken, before anything is erased or written back
        if (failed) { *m.status = 1; return 1; }
        for (size_t j = 0; j < vToErase.size(); ++j) {   // pKFi->EraseMapPointMatch(pMPi) is the replay's; pMPi->EraseObservation(pKFi)
            m.obsFlag[eraseObs[j]] = OBS_ERASED;
            EraseObservation(vToErase[j].second, vToErase[j].first);
        }
        for (KeyFrame* k : lFixedKeyFrames) k->mnBAFixedForKF = 0;
        // Recover optimized data (:2905-2950)
        for (int v = 0; v < N; v++) {
            KeyFrame* pKFi = vpOptimizableKFs[v];
            float R[9], t[3], T[7];
            for (int c = 0; c < 9; ++c) R[c] = (float)tcw[12 * v + c];
            for (int c = 0; c < 3; ++c) t[c] = (float)tcw[12 * v + 9 + c];
            set_pose(R, t, T, pKFi->Ow);
            pKFi->mnBALocalForKF = 0;
            std::memcpy(m.kfPose7 + 7 * v, T, 28); std::memcpy(m.kfCenter + 3 * v, pKFi->Ow, 12);
            if (pKFi->bImu) {
                for (int c = 0; c < 3; ++c) m.kfVelocity[3 * v + c] = (float)state[21 * v + 12 + c];
                for (int c = 0; c < 3; ++c) { m.kfBias6[6 * v + c] = (float)state[21 * v + 18 + c]; m.kfBias6[6 * v + 3 + c] = (float)state[21 * v + 15 + c]; }
            }
        }
        for (int r = 0; r < nL; ++r) {
            MapPoint* pMP = vp[r];
            for (int c = 0; c < 3; ++c) pMP->pos[c] = (float)points[3 * r + c];
            UpdateNormalAndDepth(pMP);
            std::memcpy(m.pointPos + 3 * r, pMP->pos, 12);
            m.pointBad[r] = pMP->bad; m.pointRefKF[r] = pMP->ref ? pMP->ref->idx : -1;
            if (!pMP->bad) { std::memcpy(m.normal + 3 * r, pMP->normal, 12); m.minDistance[r] = pMP->minD; m.maxDistance[r] = pMP->maxD; }
        }
        *m.status = 0;
        return 0;
    }
};

}  // namespace

extern "C" {
// The whole function on one map; returns the status (LIBA_LOCAL_*).  With given the solve is not run: the map's optState21 / optTcw12 (per
// problem keyframe), optPoint (per local point), edgeChi2 (per observation) and stats8 (the FAIL flag, [2]) are read as the optimiser's
// results.  built (may be NULL) receives the problem the optimiser sees.
int orbo_local_inertial_ba_map(const OrboLiMap* m, int given, OrboLiBuilt* built) {
    Run r(*m);
    return r.run(given != 0, built);
}
}
