// TEST INFRASTRUCTURE ONLY -- CPU oracle of LoopClosing::DetectCommonRegionsFromBoW (src/LoopClosing.cc, v1.0) up to the Sim3Solver:
// the candidate loop's text transcribed over a small pointer model rebuilt from the flattened query -- KeyFrame objects with
// mvpMapPoints, isBad() and their best covisibles, MapPoint objects with isBad(), mpCurrentKF->GetConnectedKeyFrames() as a std::set and
// spMatchedMPi as a std::set<MapPoint*>.  Each SearchByBoW(mpCurrentKF, vpCovKFi[j], vvpMatchedMPs[j]) with ORBmatcher(0.9, true) is
// orbo_search_by_bow_kf (oracle/matcher_oracle.cpp, pinned to the reference's own body); its match12 becomes the vector<MapPoint*>.
#include <cstdint>
#include <set>
#include <vector>

#include "oracle_common.h"

extern "C" {
int orbo_search_by_bow_kf(int N1, const orbo::KeyPoint* kps1, const uint8_t* desc1, const uint8_t* point1, int E1, const int* fvNode1, const int* fvFeat1,
                          int N2, const orbo::KeyPoint* kps2, const uint8_t* desc2, const uint8_t* point2, int E2, const int* fvNode2, const int* fvFeat2,
                          float nnratio, int checkOri, int* match12);

// Layout-compatible with OrbmBowFrame, OrbmCommonRegionsKF and OrbmCommonRegionsQuery (include/orb_b200.h).
typedef struct OrboBowFrame {
    int N; const orbo::KeyPoint* keypoints; const uint8_t* descriptors;
    int nEntries; const int32_t* fvNode; const int32_t* fvFeature;
} OrboBowFrame;
typedef struct OrboCommonRegionsKF {
    OrboBowFrame frame; const int32_t* point; int bad; int connected;
} OrboCommonRegionsKF;
typedef struct OrboCommonRegionsQuery {
    int nKF; const OrboCommonRegionsKF* kf;
    int nPoints; const uint8_t* pointBad;
    int nCand; const int32_t* cand; const int32_t* covStart; const int32_t* cov;
    uint8_t* status; int32_t* covList; int32_t* nmatches; int32_t* numBoWMatches; int32_t* matchedCov; int32_t* matchedPoint;
} OrboCommonRegionsQuery;
}

namespace {

enum { SKIPPED = 0, ABORTED_NEAR = 1, RAN = 2 };
constexpr int MAX_COV = 11;

struct MapPoint {
    int id = -1; bool mbBad = false;
    bool isBad() const { return mbBad; }
};
struct KeyFrame {
    int id = -1; bool mbBad = false;
    const OrboBowFrame* F = nullptr;
    std::vector<MapPoint*> mvpMapPoints;
    std::vector<KeyFrame*> mvpOrderedConnectedKeyFrames;   // the first 10 of them: what GetBestCovisibilityKeyFrames(10) returns
    bool isBad() const { return mbBad; }
    std::vector<MapPoint*> GetMapPointMatches() const { return mvpMapPoints; }
    std::vector<KeyFrame*> GetBestCovisibilityKeyFrames(int N) const {
        return (int)mvpOrderedConnectedKeyFrames.size() < N ? mvpOrderedConnectedKeyFrames
                                                              : std::vector<KeyFrame*>(mvpOrderedConnectedKeyFrames.begin(), mvpOrderedConnectedKeyFrames.begin() + N);
    }
};

// ORBmatcher::SearchByBoW(pKF1, pKF2, vpMatches12) through the pinned oracle: point flags from the keyframes' map points
int SearchByBoW(KeyFrame* pKF1, KeyFrame* pKF2, std::vector<MapPoint*>& vpMatches12) {
    auto flags = [](const KeyFrame* k) {
        std::vector<uint8_t> f(k->mvpMapPoints.size());
        for (size_t i = 0; i < f.size(); ++i) f[i] = !k->mvpMapPoints[i] ? 0 : k->mvpMapPoints[i]->isBad() ? 2 : 1;
        return f;
    };
    const std::vector<uint8_t> p1 = flags(pKF1), p2 = flags(pKF2);
    std::vector<int> m12(pKF1->F->N > 0 ? pKF1->F->N : 1);
    const OrboBowFrame &a = *pKF1->F, &b = *pKF2->F;
    const int n = orbo_search_by_bow_kf(a.N, a.keypoints, a.descriptors, p1.data(), a.nEntries, a.fvNode, a.fvFeature, b.N, b.keypoints, b.descriptors, p2.data(),
                                        b.nEntries, b.fvNode, b.fvFeature, 0.9f, 1, m12.data());
    vpMatches12 = std::vector<MapPoint*>(pKF1->mvpMapPoints.size(), static_cast<MapPoint*>(nullptr));
    for (int i = 0; i < a.N; ++i) if (m12[i] >= 0) vpMatches12[i] = pKF2->mvpMapPoints[m12[i]];
    return n;
}

}  // namespace

extern "C" void orbo_common_regions_bow(const OrboCommonRegionsQuery* q) {
    std::vector<MapPoint> points(q->nPoints);
    for (int p = 0; p < q->nPoints; ++p) { points[p].id = p; points[p].mbBad = q->pointBad[p] != 0; }
    std::vector<KeyFrame> kfs(q->nKF);
    std::set<KeyFrame*> spConnectedKeyFrames;               // mpCurrentKF->GetConnectedKeyFrames()
    for (int e = 0; e < q->nKF; ++e) {
        KeyFrame& k = kfs[e];
        k.id = e; k.mbBad = q->kf[e].bad != 0; k.F = &q->kf[e].frame;
        k.mvpMapPoints.assign(k.F->N, nullptr);
        for (int i = 0; i < k.F->N; ++i) if (q->kf[e].point[i] >= 0) k.mvpMapPoints[i] = &points[q->kf[e].point[i]];
        if (q->kf[e].connected) spConnectedKeyFrames.insert(&k);
    }
    std::vector<KeyFrame*> vpBowCand;
    for (int c = 0; c < q->nCand; ++c) {
        vpBowCand.push_back(q->cand[c] >= 0 ? &kfs[q->cand[c]] : nullptr);
        if (q->cand[c] >= 0)
            for (int i = q->covStart[c]; i < q->covStart[c + 1]; ++i) kfs[q->cand[c]].mvpOrderedConnectedKeyFrames.push_back(&kfs[q->cov[i]]);
    }
    KeyFrame* mpCurrentKF = &kfs[0];
    const int nNumCovisibles = 10;
    for (int c = 0; c < q->nCand; ++c) {
        const int N0 = mpCurrentKF->F->N;
        int32_t *covList = q->covList + (size_t)c * MAX_COV, *nm = q->nmatches + (size_t)c * MAX_COV;
        for (int j = 0; j < MAX_COV; ++j) { covList[j] = -1; nm[j] = -1; }
        q->numBoWMatches[c] = 0;
        for (int k = 0; k < N0; ++k) { q->matchedCov[(size_t)c * N0 + k] = -1; q->matchedPoint[(size_t)c * N0 + k] = -1; }

        KeyFrame* pKFi = vpBowCand[c];
        if (!pKFi || pKFi->isBad()) { q->status[c] = SKIPPED; continue; }

        std::vector<KeyFrame*> vpCovKFi = pKFi->GetBestCovisibilityKeyFrames(nNumCovisibles);
        if (vpCovKFi.empty()) {
            vpCovKFi.push_back(pKFi);
        } else {
            vpCovKFi.push_back(vpCovKFi[0]);
            vpCovKFi[0] = pKFi;
        }
        for (size_t j = 0; j < vpCovKFi.size(); ++j) covList[j] = vpCovKFi[j]->id;

        bool bAbortByNearKF = false;
        for (size_t j = 0; j < vpCovKFi.size(); ++j) {
            if (spConnectedKeyFrames.find(vpCovKFi[j]) != spConnectedKeyFrames.end()) {
                bAbortByNearKF = true;
                break;
            }
        }
        if (bAbortByNearKF) { q->status[c] = ABORTED_NEAR; continue; }
        q->status[c] = RAN;

        std::vector<std::vector<MapPoint*>> vvpMatchedMPs;
        vvpMatchedMPs.resize(vpCovKFi.size());
        std::set<MapPoint*> spMatchedMPi;
        int numBoWMatches = 0;

        std::vector<MapPoint*> vpMatchedPoints = std::vector<MapPoint*>(mpCurrentKF->GetMapPointMatches().size(), static_cast<MapPoint*>(nullptr));
        std::vector<KeyFrame*> vpKeyFrameMatchedMP = std::vector<KeyFrame*>(mpCurrentKF->GetMapPointMatches().size(), static_cast<KeyFrame*>(nullptr));

        for (size_t j = 0; j < vpCovKFi.size(); ++j) {
            if (!vpCovKFi[j] || vpCovKFi[j]->isBad()) continue;
            nm[j] = SearchByBoW(mpCurrentKF, vpCovKFi[j], vvpMatchedMPs[j]);
        }

        for (size_t j = 0; j < vpCovKFi.size(); ++j) {
            for (size_t k = 0; k < vvpMatchedMPs[j].size(); ++k) {
                MapPoint* pMPi_j = vvpMatchedMPs[j][k];
                if (!pMPi_j || pMPi_j->isBad()) continue;
                if (spMatchedMPi.find(pMPi_j) == spMatchedMPi.end()) {
                    spMatchedMPi.insert(pMPi_j);
                    numBoWMatches++;
                    vpMatchedPoints[k] = pMPi_j;
                    vpKeyFrameMatchedMP[k] = vpCovKFi[j];
                    q->matchedCov[(size_t)c * N0 + k] = (int32_t)j;     // the position of vpKeyFrameMatchedMP[k] in vpCovKFi
                }
            }
        }
        q->numBoWMatches[c] = numBoWMatches;
        for (int k = 0; k < N0; ++k) q->matchedPoint[(size_t)c * N0 + k] = vpMatchedPoints[k] ? vpMatchedPoints[k]->id : -1;
    }
}
