// TEST INFRASTRUCTURE ONLY -- CPU oracle of LocalMapping::KeyFrameCulling() (src/LocalMapping.cc; monocular and mono-inertial:
// redundant_th = 0.9, Nd = 21), a literal transcription of the loop over a small pointer map rebuilt from the flattened input:
// keyframes with mvpMapPoints (the local keyframes' slots), map points with their observation map and nObs, the prev / next links,
// KeyFrame::SetBadFlag (init keyframe, mbNotErase, EraseObservation of every point, KeyFramesInMap()), MapPoint::EraseObservation
// (monocular: nObs--) and MapPoint::SetBadFlag (the point leaves every keyframe that holds it).  MergePrevious, the covisibility graph
// and the spanning tree are not modelled: the loop reads none of them.
//
// Float rules (built with -ffp-contract=off, as the kernel evaluates them): redundant_th * nMPs is one float product; t is the double
// difference of the timestamps rounded to float; the norm is sqrtf((dx*dx + dy*dy) + dz*dz) with every operation rounded, compared in
// double with 0.02.  Eigen's Vector3f::norm() under the reference's -march=native may contract the sum of squares; that is not pinned.
#include <cmath>
#include <cstdint>
#include <map>
#include <utility>
#include <vector>

extern "C" {
// Layout-compatible with OrbmCullingMap (include/orb_b200.h).
typedef struct OrboCullingMap {
    int nKF;
    const uint64_t* mnId; const uint8_t* kfFlags; const int32_t* prevKF; const int32_t* nextKF; const double* timeStamp; const float* imuPosition;
    int nLocal;
    const int32_t* local; const int32_t* slotStart; const int32_t* slotPoint; const int32_t* slotOctave;
    int nPoints;
    const uint8_t* pointBad; const int32_t* obsStart; const int32_t* obsKF; const int32_t* obsOctave;
    int inertial, imuInitialized, inertialBA2, abortBA;
    int keyFramesInMap;
    uint64_t currentId, lastId;
    uint8_t* status; int32_t* nMPs; int32_t* nRedundant; int32_t* visited;
} OrboCullingMap;
}

namespace {

enum { NOT_VISITED = 0, SKIPPED, KEPT, KEPT_FEW_KFS, KEPT_RECENT, KEPT_NO_LINK, KEPT_IMU, CULLED, CULLED_TIME, CULLED_STILL, NOT_ERASE };
enum { F_BAD = 1, F_INIT = 2, F_NOT_ERASE = 4, F_TO_BE_ERASED = 8 };

struct MapPoint;
struct KeyFrame {
    unsigned long mnId = 0;
    bool mbBad = false, init = false, mbNotErase = false, mbToBeErased = false;
    KeyFrame *mPrevKF = nullptr, *mNextKF = nullptr;
    double mTimeStamp = 0;
    float imuPos[3] = {0, 0, 0};
    std::vector<MapPoint*> mvpMapPoints;     // the local keyframes' non-NULL slots at the call, in slot order
    std::vector<int> octave;                 // mvKeysUn[i].octave of those slots
    bool isBad() const { return mbBad; }
};
struct MapPoint {
    bool mbBad = false;
    int nObs = 0;
    std::map<KeyFrame*, std::pair<int, int>> mObservations;   // keyframe -> (its slot in mvpMapPoints, -1 when not a local keyframe; octave)
    bool isBad() const { return mbBad; }
    int Observations() const { return nObs; }
};
struct Map { int keyFramesInMap; };

void SetBadFlag(MapPoint* p) {
    p->mbBad = true;
    std::map<KeyFrame*, std::pair<int, int>> obs = p->mObservations;
    p->mObservations.clear();
    for (auto& o : obs)
        if (o.second.first >= 0) o.first->mvpMapPoints[o.second.first] = nullptr;   // EraseMapPointMatch
}
void EraseObservation(MapPoint* p, KeyFrame* pKF) {
    bool bBad = false;
    if (p->mObservations.count(pKF)) {
        p->nObs--;
        p->mObservations.erase(pKF);
        if (p->nObs <= 2) bBad = true;
    }
    if (bBad) SetBadFlag(p);
}
void SetBadFlag(KeyFrame* k, Map& map) {
    if (k->init) return;
    if (k->mbNotErase) { k->mbToBeErased = true; return; }
    for (MapPoint* p : k->mvpMapPoints)
        if (p) EraseObservation(p, k);
    k->mbBad = true;
    map.keyFramesInMap--;
}

}  // namespace

// Runs the loop on map `m`, writes its status / nMPs / nRedundant / visited, and the final state: kfFlagsOut [nKF] (F_*), prevOut /
// nextOut [nKF] (inertial; -1 = NULL), pointBadOut / nObsOut [nPoints], *keyFramesInMapOut.
extern "C" int orbo_keyframe_culling(const OrboCullingMap* m, uint8_t* kfFlagsOut, int32_t* prevOut, int32_t* nextOut, uint8_t* pointBadOut,
                                     int32_t* nObsOut, int* keyFramesInMapOut) {
    std::vector<KeyFrame> kfs((size_t)m->nKF);
    std::vector<MapPoint> pts((size_t)m->nPoints);
    for (int k = 0; k < m->nKF; ++k) {
        KeyFrame& K = kfs[k];
        K.mnId = (unsigned long)m->mnId[k];
        K.mbBad = m->kfFlags[k] & F_BAD; K.init = m->kfFlags[k] & F_INIT; K.mbNotErase = m->kfFlags[k] & F_NOT_ERASE;
        if (m->inertial) {
            K.mPrevKF = m->prevKF[k] >= 0 ? &kfs[m->prevKF[k]] : nullptr;
            K.mNextKF = m->nextKF[k] >= 0 ? &kfs[m->nextKF[k]] : nullptr;
            K.mTimeStamp = m->timeStamp[k];
            for (int c = 0; c < 3; ++c) K.imuPos[c] = m->imuPosition[3 * k + c];
        }
    }
    for (int p = 0; p < m->nPoints; ++p) {
        pts[p].mbBad = m->pointBad[p];
        pts[p].nObs = m->obsStart[p + 1] - m->obsStart[p];
        for (int o = m->obsStart[p]; o < m->obsStart[p + 1]; ++o) pts[p].mObservations[&kfs[m->obsKF[o]]] = std::make_pair(-1, (int)m->obsOctave[o]);
    }
    for (int l = 0; l < m->nLocal; ++l) {
        KeyFrame* K = &kfs[m->local[l]];
        for (int s = m->slotStart[l]; s < m->slotStart[l + 1]; ++s) {
            MapPoint* P = &pts[m->slotPoint[s]];
            auto it = P->mObservations.find(K);
            if (it != P->mObservations.end()) it->second.first = (int)K->mvpMapPoints.size();
            K->mvpMapPoints.push_back(P);
            K->octave.push_back(m->slotOctave[s]);
        }
    }
    Map map{m->keyFramesInMap};
    const unsigned long currentId = (unsigned long)m->currentId, last_ID = (unsigned long)m->lastId;
    const bool mbInertial = m->inertial, bInitImu = m->imuInitialized, inertialBA2 = m->inertialBA2, mbAbortBA = m->abortBA;

    const int Nd = 21;
    const float redundant_th = 0.9f;
    int count = 0;
    for (int l = 0; l < m->nLocal; ++l) {
        m->status[l] = NOT_VISITED; m->nMPs[l] = -1; m->nRedundant[l] = -1;
    }
    for (int l = 0; l < m->nLocal; ++l) {
        count++;
        KeyFrame* pKF = &kfs[m->local[l]];
        if (pKF->init || pKF->isBad()) { m->status[l] = SKIPPED; continue; }
        const std::vector<MapPoint*> vpMapPoints = pKF->mvpMapPoints;     // GetMapPointMatches()
        const int thObs = 3;
        int nRedundantObservations = 0;
        int nMPs = 0;
        for (size_t i = 0, iend = vpMapPoints.size(); i < iend; i++) {
            MapPoint* pMP = vpMapPoints[i];
            if (pMP) {
                if (!pMP->isBad()) {
                    nMPs++;
                    if (pMP->Observations() > thObs) {
                        const int& scaleLevel = pKF->octave[i];
                        const std::map<KeyFrame*, std::pair<int, int>> observations = pMP->mObservations;
                        int nObs = 0;
                        for (auto mit = observations.begin(), mend = observations.end(); mit != mend; mit++) {
                            KeyFrame* pKFi = mit->first;
                            if (pKFi == pKF) continue;
                            const int scaleLeveli = mit->second.second;
                            if (scaleLeveli <= scaleLevel + 1) {
                                nObs++;
                                if (nObs > thObs) break;
                            }
                        }
                        if (nObs > thObs) nRedundantObservations++;
                    }
                }
            }
        }
        m->nMPs[l] = nMPs; m->nRedundant[l] = nRedundantObservations;
        m->status[l] = KEPT;
        if (nRedundantObservations > redundant_th * nMPs) {
            if (mbInertial) {
                if (map.keyFramesInMap <= Nd) { m->status[l] = KEPT_FEW_KFS; continue; }
                if (pKF->mnId > (currentId - 2)) { m->status[l] = KEPT_RECENT; continue; }
                m->status[l] = KEPT_NO_LINK;
                if (pKF->mPrevKF && pKF->mNextKF) {
                    const float t = pKF->mNextKF->mTimeStamp - pKF->mPrevKF->mTimeStamp;
                    m->status[l] = KEPT_IMU;
                    const float dx = pKF->imuPos[0] - pKF->mPrevKF->imuPos[0], dy = pKF->imuPos[1] - pKF->mPrevKF->imuPos[1],
                                dz = pKF->imuPos[2] - pKF->mPrevKF->imuPos[2];
                    if ((bInitImu && (pKF->mnId < last_ID) && (t < 3.)) || (t < 0.5)) {
                        pKF->mNextKF->mPrevKF = pKF->mPrevKF;
                        pKF->mPrevKF->mNextKF = pKF->mNextKF;
                        pKF->mNextKF = nullptr;
                        pKF->mPrevKF = nullptr;
                        m->status[l] = pKF->mbNotErase ? NOT_ERASE : CULLED_TIME;
                        SetBadFlag(pKF, map);
                    } else if (!inertialBA2 && (std::sqrt((dx * dx + dy * dy) + dz * dz) < 0.02) && (t < 3)) {
                        pKF->mNextKF->mPrevKF = pKF->mPrevKF;
                        pKF->mPrevKF->mNextKF = pKF->mNextKF;
                        pKF->mNextKF = nullptr;
                        pKF->mPrevKF = nullptr;
                        m->status[l] = pKF->mbNotErase ? NOT_ERASE : CULLED_STILL;
                        SetBadFlag(pKF, map);
                    }
                }
            } else {
                m->status[l] = pKF->mbNotErase ? NOT_ERASE : CULLED;
                SetBadFlag(pKF, map);
            }
        }
        if ((count > 20 && mbAbortBA) || count > 100) break;
    }
    *m->visited = count;
    for (int k = 0; k < m->nKF; ++k) {
        const KeyFrame& K = kfs[k];
        kfFlagsOut[k] = (K.mbBad ? F_BAD : 0) | (K.init ? F_INIT : 0) | (K.mbNotErase ? F_NOT_ERASE : 0) | (K.mbToBeErased ? F_TO_BE_ERASED : 0);
        if (m->inertial) {
            prevOut[k] = K.mPrevKF ? (int32_t)(K.mPrevKF - kfs.data()) : -1;
            nextOut[k] = K.mNextKF ? (int32_t)(K.mNextKF - kfs.data()) : -1;
        }
    }
    for (int p = 0; p < m->nPoints; ++p) { pointBadOut[p] = pts[p].mbBad; nObsOut[p] = pts[p].nObs; }
    *keyFramesInMapOut = map.keyFramesInMap;
    return 0;
}
