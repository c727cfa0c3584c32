// TEST INFRASTRUCTURE ONLY -- CPU oracle of Optimizer::LocalBundleAdjustment (src/Optimizer.cc:1116-1498, monocular observations) as a
// whole, a literal transcription over a small pointer map rebuilt from the flattened input (LbaLocalMap, include/orb_b200.h): keyframes
// with mnBALocalForKF / mnBAFixedForKF, map points with mObservations (a list in the caller's key order, which is the std::map's
// iteration order), nObs, mpRefKF and the bad flag.  The solve is orbo_lba_solve (lba_oracle.cpp) on the graph the walk builds, with
// vertices in g2o's order (keyframes by mnId, then points by mnId); the erase loop follows MapPoint::EraseObservation / SetBadFlag, the
// write-back Sophus::SE3f(q.cast<float>(), t.cast<float>()) (the normalisation of csrc/frame_pose.cuh), GetCameraCenter and
// UpdateNormalAndDepth.  Built with -ffp-contract=off: every float operation rounds once, as the kernels evaluate them.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <list>
#include <utility>
#include <vector>

extern "C" int orbo_lba_solve(int nP, double* posesInOut, const uint8_t* fixed, const float* cam4, int nL, double* pointsInOut, int nE,
                              const int* edgePoint, const int* edgePose, const double* obs2, const float* invSigma2, double huberDelta,
                              int iterations, double userLambdaInit, const int* stopFlag, double* edgeChi2Out, uint8_t* edgeDepthPosOut,
                              double* stats);

extern "C" {
// Layout-compatible with LbaLocalMap (include/orb_b200.h).
typedef struct OrboLocalMap {
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
} OrboLocalMap;

// The graph the walk hands to the optimiser (LbaProblem's arrays, capacity nKF poses / nPoints points / obsStart[nPoints] edges) and the
// table entry of every vertex.  sizes = nP, nL, nE.
typedef struct OrboLocalBuilt {
    double* poses; uint8_t* fixed; float* cam; double* points; int32_t* edgePoint; int32_t* edgePose; double* obs; float* invSigma2;
    int32_t* vertKF; int32_t* vertPoint; int32_t* sizes;
} OrboLocalBuilt;
}

namespace {

enum { KF_BAD = 1, KF_INIT = 2, KF_OTHER_MAP = 8 };
const uint64_t NONE = ~0ull;

struct KeyFrame {
    int idx; uint64_t mnId; bool bad, otherMap;
    float Tcw[7], Ow[3], cam[4];
    uint64_t mnBALocalForKF = NONE, mnBAFixedForKF = NONE;
};
struct MapPoint {
    int idx; uint64_t mnId; bool bad, otherMap;
    float pos[3];
    std::vector<std::pair<KeyFrame*, int>> obs;   // mObservations: keyframe, row of the flattened observation
    int nObs;
    KeyFrame* ref;
    uint64_t mnBALocalForKF = NONE;
    float normal[3] = {0, 0, 0}, minD = 0, maxD = 0;
};

float norm3(float x, float y, float z) { return std::sqrt((x * x + y * y) + z * z); }

// Sophus::SE3f(SE3quat.rotation().cast<float>(), SE3quat.translation().cast<float>()) and GetCameraCenter (frame_pose.cuh)
void set_pose(const double* T, float* Tf, float* Ow) {
    const float w = (float)T[0], x = (float)T[1], y = (float)T[2], z = (float)T[3];
    const float n = ((x * x + y * y) + z * z) + w * w;
    const float s = std::sqrt(n);
    Tf[0] = w / s; Tf[1] = x / s; Tf[2] = y / s; Tf[3] = z / s;
    Tf[4] = (float)T[4]; Tf[5] = (float)T[5]; Tf[6] = (float)T[6];
    const float qw = Tf[0], ix = -Tf[1], iy = -Tf[2], iz = -Tf[3], px = Tf[4], py = Tf[5], pz = Tf[6];
    float ux = iy * pz - iz * py, uy = iz * px - ix * pz, uz = ix * py - iy * px;
    ux = ux + ux; uy = uy + uy; uz = uz + uz;
    const float cx = iy * uz - iz * uy, cy = iz * ux - ix * uz, cz = ix * uy - iy * ux;
    Ow[0] = -((px + qw * ux) + cx); Ow[1] = -((py + qw * uy) + cy); Ow[2] = -((pz + qw * uz) + cz);
}

struct Run {
    const OrboLocalMap& m;
    std::vector<KeyFrame> kfs;
    std::vector<MapPoint> pts;
    explicit Run(const OrboLocalMap& mm) : m(mm) {
        kfs.resize(m.nKF);
        for (int k = 0; k < m.nKF; ++k) {
            KeyFrame& K = kfs[k];
            K.idx = k; K.mnId = m.mnId[k]; K.bad = m.kfFlags[k] & KF_BAD; K.otherMap = m.kfFlags[k] & KF_OTHER_MAP;
            std::memcpy(K.Tcw, m.pose7 + 7 * k, 28); std::memcpy(K.Ow, m.cameraCenter + 3 * k, 12); std::memcpy(K.cam, m.cam4 + 4 * k, 16);
        }
        pts.resize(m.nPoints);
        for (int p = 0; p < m.nPoints; ++p) {
            MapPoint& P = pts[p];
            P.idx = p; P.mnId = m.pointId[p]; P.bad = m.pointFlags[p] & KF_BAD; P.otherMap = m.pointFlags[p] & KF_OTHER_MAP;
            std::memcpy(P.pos, m.worldPos + 3 * p, 12);
            for (int o = m.obsStart[p]; o < m.obsStart[p + 1]; ++o) P.obs.push_back({&kfs[m.obsKF[o]], o});
            P.nObs = (int)P.obs.size();
            P.ref = m.refKF[p] >= 0 ? &kfs[m.refKF[p]] : nullptr;
        }
    }
    // the candidate local keyframe's slots: c = 0 for pKF, 1 + i for cov[i]
    std::vector<MapPoint*> GetMapPointMatches(int c) {
        std::vector<MapPoint*> v;
        for (int s = m.slotStart[c]; s < m.slotStart[c + 1]; ++s) v.push_back(m.slotPoint[s] >= 0 ? &pts[m.slotPoint[s]] : nullptr);
        return v;
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

    int run(bool givenLm, OrboLocalBuilt* built) {
        const int nObs = m.nPoints ? m.obsStart[m.nPoints] : 0;
        for (int k = 0; k < m.nKF; ++k) { m.localKF[k] = m.fixedKF[k] = -1; for (int c = 0; c < 7; ++c) m.kfPose7[7 * k + c] = 0; for (int c = 0; c < 3; ++c) m.kfCenter[3 * k + c] = 0; }
        for (int p = 0; p < m.nPoints; ++p) {
            m.localPoint[p] = -1; m.pointBad[p] = 0; m.pointRefKF[p] = -1; m.minDistance[p] = m.maxDistance[p] = 0;
            for (int c = 0; c < 3; ++c) m.pointPos[3 * p + c] = m.normal[3 * p + c] = 0;
        }
        for (int o = 0; o < nObs; ++o) m.obsFlag[o] = 0;
        for (int i = 0; i < 4; ++i) m.counts[i] = 0;
        if (!givenLm) { m.lmStats[0] = -1; for (int i = 1; i < 5; ++i) m.lmStats[i] = 0; }
        KeyFrame* pKF = &kfs[0];
        // Local KeyFrames: First Breath Search from Current Keyframe (:1125-1140)
        std::list<KeyFrame*> lLocalKeyFrames;
        lLocalKeyFrames.push_back(pKF);
        pKF->mnBALocalForKF = pKF->mnId;
        std::vector<int> candOf(m.nKF, -1);
        candOf[0] = 0;
        for (int i = 0; i < m.nCov; ++i) {
            KeyFrame* pKFi = &kfs[m.cov[i]];
            pKFi->mnBALocalForKF = pKF->mnId;
            if (!pKFi->bad && !pKFi->otherMap) { lLocalKeyFrames.push_back(pKFi); candOf[pKFi->idx] = 1 + i; }
        }
        // Local MapPoints seen in Local KeyFrames (:1142-1166)
        int num_fixedKF = 0;
        std::list<MapPoint*> lLocalMapPoints;
        for (KeyFrame* pKFi : lLocalKeyFrames) {
            if (m.kfFlags[pKFi->idx] & KF_INIT) num_fixedKF = 1;
            for (MapPoint* pMP : GetMapPointMatches(candOf[pKFi->idx]))
                if (pMP && !pMP->bad && !pMP->otherMap && pMP->mnBALocalForKF != pKF->mnId) {
                    lLocalMapPoints.push_back(pMP);
                    pMP->mnBALocalForKF = pKF->mnId;
                }
        }
        // Fixed Keyframes (:1168-1184)
        std::list<KeyFrame*> lFixedCameras;
        for (MapPoint* pMP : lLocalMapPoints)
            for (auto& e : pMP->obs) {
                KeyFrame* pKFi = e.first;
                if (pKFi->mnBALocalForKF != pKF->mnId && pKFi->mnBAFixedForKF != pKF->mnId) {
                    pKFi->mnBAFixedForKF = pKF->mnId;
                    if (!pKFi->bad && !pKFi->otherMap) lFixedCameras.push_back(pKFi);
                }
            }
        num_fixedKF = (int)lFixedCameras.size() + num_fixedKF;
        int i = 0;
        for (KeyFrame* k : lLocalKeyFrames) m.localKF[i++] = k->idx;
        i = 0;
        for (KeyFrame* k : lFixedCameras) m.fixedKF[i++] = k->idx;
        i = 0;
        for (MapPoint* p : lLocalMapPoints) m.localPoint[i++] = p->idx;
        m.nLists[0] = (int)lLocalKeyFrames.size(); m.nLists[1] = (int)lFixedCameras.size(); m.nLists[2] = (int)lLocalMapPoints.size();
        if (num_fixedKF == 0) { *m.status = 1; return 1; }
        // vertices in g2o's order: keyframes by mnId, then points by mnId
        std::vector<KeyFrame*> vk(lLocalKeyFrames.begin(), lLocalKeyFrames.end());
        vk.insert(vk.end(), lFixedCameras.begin(), lFixedCameras.end());
        std::sort(vk.begin(), vk.end(), [](const KeyFrame* a, const KeyFrame* b) { return a->mnId < b->mnId; });
        std::vector<MapPoint*> vp(lLocalMapPoints.begin(), lLocalMapPoints.end());
        std::sort(vp.begin(), vp.end(), [](const MapPoint* a, const MapPoint* b) { return a->mnId < b->mnId; });
        const int nP = (int)vk.size(), nL = (int)vp.size();
        std::vector<int> kfVert(m.nKF, -1), ptVert(m.nPoints, -1);
        std::vector<double> poses(7 * (size_t)nP), points(3 * (size_t)nL);
        std::vector<uint8_t> fixed(nP);
        std::vector<float> cam(4 * (size_t)nP);
        for (int v = 0; v < nP; ++v) {
            KeyFrame* K = vk[v];
            kfVert[K->idx] = v;
            for (int c = 0; c < 7; ++c) poses[7 * v + c] = (double)K->Tcw[c];
            for (int c = 0; c < 4; ++c) cam[4 * v + c] = K->cam[c];
            const bool local = K->mnBALocalForKF == pKF->mnId && !K->bad && !K->otherMap;
            fixed[v] = !local || (m.kfFlags[K->idx] & KF_INIT);
        }
        for (int v = 0; v < nL; ++v) {
            ptVert[vp[v]->idx] = v;
            for (int c = 0; c < 3; ++c) points[3 * v + c] = (double)vp[v]->pos[c];
        }
        // edges (:1287-1331)
        std::vector<int> ePt, ePose, eObs;
        std::vector<double> obs;
        std::vector<float> isg;
        std::vector<MapPoint*> vpMapPointEdgeMono;
        std::vector<KeyFrame*> vpEdgeKFMono;
        for (MapPoint* pMP : lLocalMapPoints)
            for (auto& e : pMP->obs) {
                KeyFrame* pKFi = e.first;
                if (pKFi->bad || pKFi->otherMap) continue;
                const int o = e.second;
                ePt.push_back(ptVert[pMP->idx]); ePose.push_back(kfVert[pKFi->idx]);
                obs.push_back((double)m.obsPt[2 * o]); obs.push_back((double)m.obsPt[2 * o + 1]);
                isg.push_back(m.invLevelSigma2[m.obsOctave[o]]);
                eObs.push_back(o); vpMapPointEdgeMono.push_back(pMP); vpEdgeKFMono.push_back(pKFi);
            }
        const int nE = (int)ePt.size();
        m.counts[0] = num_fixedKF; m.counts[1] = (int)lLocalKeyFrames.size(); m.counts[2] = nL; m.counts[3] = nE;
        if (built) {
            std::memcpy(built->poses, poses.data(), 56 * (size_t)nP); std::memcpy(built->fixed, fixed.data(), nP); std::memcpy(built->cam, cam.data(), 16 * (size_t)nP);
            std::memcpy(built->points, points.data(), 24 * (size_t)nL);
            std::memcpy(built->edgePoint, ePt.data(), 4 * (size_t)nE); std::memcpy(built->edgePose, ePose.data(), 4 * (size_t)nE);
            std::memcpy(built->obs, obs.data(), 16 * (size_t)nE); std::memcpy(built->invSigma2, isg.data(), 4 * (size_t)nE);
            for (int v = 0; v < nP; ++v) built->vertKF[v] = vk[v]->idx;
            for (int v = 0; v < nL; ++v) built->vertPoint[v] = vp[v]->idx;
            built->sizes[0] = nP; built->sizes[1] = nL; built->sizes[2] = nE;
        }
        if (m.stopFlag && *m.stopFlag) { *m.status = 2; return 2; }   // :1406-1408
        std::vector<double> chi2(nE, 0.0);
        std::vector<uint8_t> dpos(nE, 1);
        if (givenLm) {
            i = 0;
            for (KeyFrame* k : lLocalKeyFrames) { for (int c = 0; c < 7; ++c) poses[7 * kfVert[k->idx] + c] = m.optPose[7 * i + c]; ++i; }
            i = 0;
            for (MapPoint* p : lLocalMapPoints) { for (int c = 0; c < 3; ++c) points[3 * ptVert[p->idx] + c] = m.optPoint[3 * i + c]; ++i; }
            for (int e = 0; e < nE; ++e) { chi2[e] = m.edgeChi2[eObs[e]]; dpos[e] = m.edgeDepthPositive[eObs[e]]; }
        } else {
            const int stop = 0;
            double stats[8];
            int nF = 0;
            for (int v = 0; v < nP; ++v) nF += !fixed[v];
            if (nF + nL > 0) {
                const int it = orbo_lba_solve(nP, poses.data(), fixed.data(), cam.data(), nL, points.data(), nE, ePt.data(), ePose.data(), obs.data(), isg.data(),
                                              (double)(float)std::sqrt(5.991), 10, m.inertial ? 100.0 : 0.0, &stop, chi2.data(), dpos.data(), stats);
                m.lmStats[0] = it; m.lmStats[1] = stats[3]; m.lmStats[2] = stats[0]; m.lmStats[3] = stats[1]; m.lmStats[4] = stats[2];
            }
        }
        if (!givenLm && m.optPose) {
            i = 0;
            for (KeyFrame* k : lLocalKeyFrames) { for (int c = 0; c < 7; ++c) m.optPose[7 * i + c] = poses[7 * kfVert[k->idx] + c]; ++i; }
            i = 0;
            for (MapPoint* p : lLocalMapPoints) { for (int c = 0; c < 3; ++c) m.optPoint[3 * i + c] = points[3 * ptVert[p->idx] + c]; ++i; }
            for (int e = 0; e < nE; ++e) { m.edgeChi2[eObs[e]] = chi2[e]; m.edgeDepthPositive[eObs[e]] = dpos[e]; }
        }
        // Check inlier observations (:1417-1430), then the erase loop (:1450-1460)
        std::vector<std::pair<KeyFrame*, MapPoint*>> vToErase;
        for (int e = 0; e < nE; ++e) {
            MapPoint* pMP = vpMapPointEdgeMono[e];
            m.obsFlag[eObs[e]] = 1;
            if (pMP->bad) continue;
            if (chi2[e] > 5.991 || !dpos[e]) { vToErase.push_back({vpEdgeKFMono[e], pMP}); m.obsFlag[eObs[e]] = 2; }
        }
        for (auto& te : vToErase) EraseObservation(te.second, te.first);
        // Recover optimized data (:1464-1497)
        i = 0;
        for (KeyFrame* pKFi : lLocalKeyFrames) {
            set_pose(&poses[7 * kfVert[pKFi->idx]], pKFi->Tcw, pKFi->Ow);
            std::memcpy(m.kfPose7 + 7 * i, pKFi->Tcw, 28); std::memcpy(m.kfCenter + 3 * i, pKFi->Ow, 12);
            ++i;
        }
        i = 0;
        for (MapPoint* pMP : lLocalMapPoints) {
            for (int c = 0; c < 3; ++c) pMP->pos[c] = (float)points[3 * ptVert[pMP->idx] + c];
            UpdateNormalAndDepth(pMP);
            std::memcpy(m.pointPos + 3 * i, pMP->pos, 12);
            m.pointBad[i] = pMP->bad; m.pointRefKF[i] = pMP->ref ? pMP->ref->idx : -1;
            if (!pMP->bad) { std::memcpy(m.normal + 3 * i, pMP->normal, 12); m.minDistance[i] = pMP->minD; m.maxDistance[i] = pMP->maxD; }
            ++i;
        }
        *m.status = 0;
        return 0;
    }
};

}  // namespace

extern "C" {
// The whole function on one map; returns the status (LBA_LOCAL_*).  With givenLm the solve is not run: the map's optPose / optPoint
// (per local keyframe / point in list order) and edgeChi2 / edgeDepthPositive (per observation) are read as the optimiser's results,
// and lmStats is left as it is.  built (may be NULL) receives the graph the optimiser sees.
int orbo_local_ba(const OrboLocalMap* m, int givenLm, OrboLocalBuilt* built) {
    Run r(*m);
    return r.run(givenLm != 0, built);
}
}
