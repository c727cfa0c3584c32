// TEST INFRASTRUCTURE ONLY -- CPU oracle of Tracking::UpdateLocalMap's UpdateLocalKeyFrames and UpdateLocalPoints (src/Tracking.cc;
// monocular and mono-inertial, Nleft == -1), a literal transcription over a small pointer model rebuilt from the flattened input of
// orbm_update_local_map_batch, one stream at a time.  A stream's keyframes are allocated in one array in table order, so the std::map and
// std::set below iterate them in table order exactly as the reference iterates its KeyFrame pointers.  Only what the two functions read is
// modelled: isBad(), mnTrackReferenceForFrame, GetObservations(), GetBestCovisibilityKeyFrames(10), GetChilds(), GetParent(), mPrevKF,
// GetMapPointMatches() (the non-NULL slots) and the voting frame's mvpMapPoints.
#include <cstdint>
#include <cstring>
#include <map>
#include <set>
#include <tuple>
#include <unordered_map>
#include <vector>

extern "C" {
// Layout-compatible with OrbmUpdateLocalMapBatch / OrbmUpdateLocalMapResult (include/orb_b200.h).
typedef struct OrboUpdateLocalMapBatch {
    int batch, kcap, mcap, mcapLast;
    int nKF, nPoints;
    const int32_t* kfStart; const uint8_t* kfFlags; const int32_t* covStart; const int32_t* covKF; const int32_t* childStart;
    const int32_t* childKF; const int32_t* parent; const int32_t* prevKF; const int32_t* slotStart; const int32_t* slotPoint;
    const int32_t* pointStart; const uint8_t* pointBad; const int32_t* obsStart; const int32_t* obsKF;
    const float *worldPos, *normal; const float *minDistInv, *maxDistInv, *maxDistance; const uint8_t *mpDesc, *hasObs;
    const int32_t* nSrc; const int32_t* srcPoint; const uint8_t* voteLastFrame; const int32_t* match; const int32_t* nK;
    const uint8_t* inertial; const int32_t* lastKF;
} OrboUpdateLocalMapBatch;
typedef struct OrboUpdateLocalMapResult {
    int32_t* localKF; int32_t* nLocalKF; int32_t* refKF; int32_t* localPoint; int32_t* nM;
    float *worldPos, *normal; float *minDistInv, *maxDistInv, *maxDistance; uint8_t *mpDesc, *hasObs, *bad;
    int32_t* lastToLocal;
} OrboUpdateLocalMapResult;
}

namespace {

struct MapPoint;
struct KeyFrame {
    bool mbBad = false;
    unsigned long mnTrackReferenceForFrame = 0;
    std::vector<KeyFrame*> mvpOrderedConnectedKeyFrames;   // its first <= 10 entries: all the flattened table gives
    std::set<KeyFrame*> mspChildrens;
    KeyFrame* mpParent = nullptr;
    KeyFrame* mPrevKF = nullptr;
    std::vector<MapPoint*> mvpMapPoints;                   // the non-NULL slots, in slot order
    bool isBad() const { return mbBad; }
    std::vector<KeyFrame*> GetBestCovisibilityKeyFrames(const int& N) const {
        if ((int)mvpOrderedConnectedKeyFrames.size() < N) return mvpOrderedConnectedKeyFrames;
        return std::vector<KeyFrame*>(mvpOrderedConnectedKeyFrames.begin(), mvpOrderedConnectedKeyFrames.begin() + N);
    }
    std::set<KeyFrame*> GetChilds() const { return mspChildrens; }
    KeyFrame* GetParent() const { return mpParent; }
    std::vector<MapPoint*> GetMapPointMatches() const { return mvpMapPoints; }
};
struct MapPoint {
    bool mbBad = false;
    unsigned long mnTrackReferenceForFrame = 0;
    std::map<KeyFrame*, std::tuple<int, int>> mObservations;
    bool isBad() const { return mbBad; }
    std::map<KeyFrame*, std::tuple<int, int>> GetObservations() const { return mObservations; }
};
struct Frame {
    unsigned long mnId = 0;
    int N = 0;
    std::vector<MapPoint*> mvpMapPoints;
    KeyFrame* mpLastKeyFrame = nullptr;
    KeyFrame* mpReferenceKF = nullptr;
};

enum { IMU_MONOCULAR = 1, MONOCULAR = 0 };

struct Tracking {
    Frame mCurrentFrame, mLastFrame;
    std::vector<KeyFrame*> mvpLocalKeyFrames;
    std::vector<MapPoint*> mvpLocalMapPoints;
    KeyFrame* mpReferenceKF = nullptr;
    unsigned long mnLastRelocFrameId = 0;
    int mSensor = MONOCULAR;
    bool imuInitialized = false;
    bool isImuInitialized() const { return imuInitialized; }

    void UpdateLocalKeyFrames() {
        // Each map point vote for the keyframes in which it has been observed
        std::map<KeyFrame*, int> keyframeCounter;
        if (!isImuInitialized() || (mCurrentFrame.mnId < mnLastRelocFrameId + 2)) {
            for (int i = 0; i < mCurrentFrame.N; i++) {
                MapPoint* pMP = mCurrentFrame.mvpMapPoints[i];
                if (pMP) {
                    if (!pMP->isBad()) {
                        const std::map<KeyFrame*, std::tuple<int, int>> observations = pMP->GetObservations();
                        for (std::map<KeyFrame*, std::tuple<int, int>>::const_iterator it = observations.begin(), itend = observations.end(); it != itend; it++)
                            keyframeCounter[it->first]++;
                    } else {
                        mCurrentFrame.mvpMapPoints[i] = NULL;
                    }
                }
            }
        } else {
            for (int i = 0; i < mLastFrame.N; i++) {
                // Using lastframe since current frame has not matches yet
                if (mLastFrame.mvpMapPoints[i]) {
                    MapPoint* pMP = mLastFrame.mvpMapPoints[i];
                    if (!pMP) continue;
                    if (!pMP->isBad()) {
                        const std::map<KeyFrame*, std::tuple<int, int>> observations = pMP->GetObservations();
                        for (std::map<KeyFrame*, std::tuple<int, int>>::const_iterator it = observations.begin(), itend = observations.end(); it != itend; it++)
                            keyframeCounter[it->first]++;
                    } else {
                        // MODIFICATION
                        mLastFrame.mvpMapPoints[i] = NULL;
                    }
                }
            }
        }

        int max = 0;
        KeyFrame* pKFmax = static_cast<KeyFrame*>(NULL);

        mvpLocalKeyFrames.clear();
        mvpLocalKeyFrames.reserve(3 * keyframeCounter.size());

        // All keyframes that observe a map point are included in the local map. Also check which keyframe shares most points
        for (std::map<KeyFrame*, int>::const_iterator it = keyframeCounter.begin(), itEnd = keyframeCounter.end(); it != itEnd; it++) {
            KeyFrame* pKF = it->first;
            if (pKF->isBad()) continue;
            if (it->second > max) {
                max = it->second;
                pKFmax = pKF;
            }
            mvpLocalKeyFrames.push_back(pKF);
            pKF->mnTrackReferenceForFrame = mCurrentFrame.mnId;
        }

        // Include also some not-already-included keyframes that are neighbors to already-included keyframes
        for (std::vector<KeyFrame*>::const_iterator itKF = mvpLocalKeyFrames.begin(), itEndKF = mvpLocalKeyFrames.end(); itKF != itEndKF; itKF++) {
            // Limit the number of keyframes
            if (mvpLocalKeyFrames.size() > 80) break;

            KeyFrame* pKF = *itKF;

            const std::vector<KeyFrame*> vNeighs = pKF->GetBestCovisibilityKeyFrames(10);

            for (std::vector<KeyFrame*>::const_iterator itNeighKF = vNeighs.begin(), itEndNeighKF = vNeighs.end(); itNeighKF != itEndNeighKF; itNeighKF++) {
                KeyFrame* pNeighKF = *itNeighKF;
                if (!pNeighKF->isBad()) {
                    if (pNeighKF->mnTrackReferenceForFrame != mCurrentFrame.mnId) {
                        mvpLocalKeyFrames.push_back(pNeighKF);
                        pNeighKF->mnTrackReferenceForFrame = mCurrentFrame.mnId;
                        break;
                    }
                }
            }

            const std::set<KeyFrame*> spChilds = pKF->GetChilds();
            for (std::set<KeyFrame*>::const_iterator sit = spChilds.begin(), send = spChilds.end(); sit != send; sit++) {
                KeyFrame* pChildKF = *sit;
                if (!pChildKF->isBad()) {
                    if (pChildKF->mnTrackReferenceForFrame != mCurrentFrame.mnId) {
                        mvpLocalKeyFrames.push_back(pChildKF);
                        pChildKF->mnTrackReferenceForFrame = mCurrentFrame.mnId;
                        break;
                    }
                }
            }

            KeyFrame* pParent = pKF->GetParent();
            if (pParent) {
                if (pParent->mnTrackReferenceForFrame != mCurrentFrame.mnId) {
                    mvpLocalKeyFrames.push_back(pParent);
                    pParent->mnTrackReferenceForFrame = mCurrentFrame.mnId;
                    break;
                }
            }
        }

        // Add 10 last temporal KFs (mainly for IMU)
        if ((mSensor == IMU_MONOCULAR) && mvpLocalKeyFrames.size() < 80) {
            KeyFrame* tempKeyFrame = mCurrentFrame.mpLastKeyFrame;

            const int Nd = 20;
            for (int i = 0; i < Nd; i++) {
                if (!tempKeyFrame) break;
                if (tempKeyFrame->mnTrackReferenceForFrame != mCurrentFrame.mnId) {
                    mvpLocalKeyFrames.push_back(tempKeyFrame);
                    tempKeyFrame->mnTrackReferenceForFrame = mCurrentFrame.mnId;
                    tempKeyFrame = tempKeyFrame->mPrevKF;
                }
            }
        }

        if (pKFmax) {
            mpReferenceKF = pKFmax;
            mCurrentFrame.mpReferenceKF = mpReferenceKF;
        }
    }

    void UpdateLocalPoints() {
        mvpLocalMapPoints.clear();

        int count_pts = 0;

        for (std::vector<KeyFrame*>::const_reverse_iterator itKF = mvpLocalKeyFrames.rbegin(), itEndKF = mvpLocalKeyFrames.rend(); itKF != itEndKF; ++itKF) {
            KeyFrame* pKF = *itKF;
            const std::vector<MapPoint*> vpMPs = pKF->GetMapPointMatches();

            for (std::vector<MapPoint*>::const_iterator itMP = vpMPs.begin(), itEndMP = vpMPs.end(); itMP != itEndMP; itMP++) {
                MapPoint* pMP = *itMP;
                if (!pMP) continue;
                if (pMP->mnTrackReferenceForFrame == mCurrentFrame.mnId) continue;
                if (!pMP->isBad()) {
                    count_pts++;
                    mvpLocalMapPoints.push_back(pMP);
                    pMP->mnTrackReferenceForFrame = mCurrentFrame.mnId;
                }
            }
        }
    }
};

void one_stream(const OrboUpdateLocalMapBatch& I, const OrboUpdateLocalMapResult& O, int b) {
    const int k0 = I.kfStart[b], nk = I.kfStart[b + 1] - k0, p0 = I.pointStart[b], np = I.pointStart[b + 1] - p0;
    std::vector<KeyFrame> kfs(nk);                       // one array in table order: pointer order == table order
    std::vector<MapPoint> pts(np);
    for (int k = 0; k < nk; ++k) {
        KeyFrame& K = kfs[k];
        const int g = k0 + k;
        K.mbBad = I.kfFlags[g] & 1;
        for (int e = I.covStart[g]; e < I.covStart[g + 1]; ++e) K.mvpOrderedConnectedKeyFrames.push_back(&kfs[I.covKF[e]]);
        for (int e = I.childStart[g]; e < I.childStart[g + 1]; ++e) K.mspChildrens.insert(&kfs[I.childKF[e]]);
        K.mpParent = I.parent[g] >= 0 ? &kfs[I.parent[g]] : nullptr;
        K.mPrevKF = I.prevKF[g] >= 0 ? &kfs[I.prevKF[g]] : nullptr;
        for (int s = I.slotStart[g]; s < I.slotStart[g + 1]; ++s) K.mvpMapPoints.push_back(&pts[I.slotPoint[s]]);
    }
    for (int p = 0; p < np; ++p) {
        pts[p].mbBad = I.pointBad[p0 + p] != 0;
        for (int o = I.obsStart[p0 + p]; o < I.obsStart[p0 + p + 1]; ++o) pts[p].mObservations[&kfs[I.obsKF[o]]] = std::make_tuple(0, -1);
    }
    const int32_t* src = I.srcPoint + (size_t)b * I.mcapLast;
    auto point = [&](int j) { return src[j] >= 0 ? &pts[src[j]] : nullptr; };
    Tracking T;
    T.mCurrentFrame.mnId = 10;                           // past the relocalisation window: the branch is isImuInitialized()
    T.imuInitialized = I.voteLastFrame[b] != 0;
    T.mSensor = I.inertial[b] ? IMU_MONOCULAR : MONOCULAR;
    T.mCurrentFrame.mpLastKeyFrame = I.lastKF[b] >= 0 ? &kfs[I.lastKF[b]] : nullptr;
    if (!T.imuInitialized) {
        T.mCurrentFrame.N = I.nK[b];
        for (int i = 0; i < I.nK[b]; ++i) {
            const int m = I.match[(size_t)b * I.kcap + i];
            T.mCurrentFrame.mvpMapPoints.push_back(m >= 0 ? point(m) : nullptr);
        }
    } else {
        T.mLastFrame.N = I.nSrc[b];
        for (int j = 0; j < I.nSrc[b]; ++j) T.mLastFrame.mvpMapPoints.push_back(point(j));
    }
    T.UpdateLocalKeyFrames();
    T.UpdateLocalPoints();

    for (int k = 0; k < nk; ++k) O.localKF[k0 + k] = k < (int)T.mvpLocalKeyFrames.size() ? (int)(T.mvpLocalKeyFrames[k] - kfs.data()) : -1;
    O.nLocalKF[b] = (int)T.mvpLocalKeyFrames.size();
    O.refKF[b] = T.mpReferenceKF ? (int)(T.mpReferenceKF - kfs.data()) : -1;
    const int nM = (int)T.mvpLocalMapPoints.size();
    O.nM[b] = nM;
    const bool fits = nM <= I.mcap;
    std::unordered_map<const MapPoint*, int> local;
    for (int l = 0; l < I.mcap; ++l) {
        const size_t r = (size_t)b * I.mcap + l;
        const int p = fits && l < nM ? (int)(T.mvpLocalMapPoints[l] - pts.data()) : -1;
        O.localPoint[r] = p;
        const size_t q = (size_t)(p0 + p);
        for (int c = 0; c < 3; ++c) { O.worldPos[3 * r + c] = p >= 0 ? I.worldPos[3 * q + c] : 0.0f; O.normal[3 * r + c] = p >= 0 ? I.normal[3 * q + c] : 0.0f; }
        O.minDistInv[r] = p >= 0 ? I.minDistInv[q] : 0.0f;
        O.maxDistInv[r] = p >= 0 ? I.maxDistInv[q] : 0.0f;
        O.maxDistance[r] = p >= 0 ? I.maxDistance[q] : 0.0f;
        if (p >= 0) memcpy(O.mpDesc + 32 * r, I.mpDesc + 32 * q, 32); else memset(O.mpDesc + 32 * r, 0, 32);
        O.hasObs[r] = p >= 0 ? I.hasObs[q] : 0;
        O.bad[r] = 0;
        if (p >= 0) local[&pts[p]] = l;
    }
    for (int j = 0; j < I.mcapLast; ++j) {
        int v = -1;
        if (j < I.nSrc[b] && src[j] >= 0) {
            auto it = local.find(&pts[src[j]]);
            if (it != local.end()) v = it->second;
        }
        O.lastToLocal[(size_t)b * I.mcapLast + j] = v;
    }
}

}  // namespace

extern "C" void orbo_update_local_map(const OrboUpdateLocalMapBatch* in, const OrboUpdateLocalMapResult* out) {
    for (int b = 0; b < in->batch; ++b) one_stream(*in, *out, b);
}
