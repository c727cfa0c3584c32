// TEST INFRASTRUCTURE ONLY -- CPU oracle of LocalMapping::ProcessNewKeyFrame's map-point loop and of the tail of
// LocalMapping::SearchInNeighbors (src/LocalMapping.cc; monocular observations), each followed by KeyFrame::UpdateConnections
// (src/KeyFrame.cc), a literal transcription over a small pointer map rebuilt from the flattened input: keyframes with their camera
// centre and mConnectedKeyFrameWeights, map points with mObservations, every std::map<KeyFrame*, ...> ordered by the keyframe's `order`
// key (the stand-in for pointer order).  MapPoint::AddObservation (monocular: nObs += 1), UpdateNormalAndDepth,
// ComputeDistinctiveDescriptors (orbo_distinctive_descriptor), KeyFrame::UpdateConnections, AddConnection, UpdateBestCovisibles.
//
// Float rules (built with -ffp-contract=off, as the kernel evaluates them): |v| = sqrtf((x*x + y*y) + z*z) with every operation
// rounded, the normal summed element-wise in key order from zero, then divided by (float)n.  Eigen's Vector3f::norm() under the
// reference's -march=native may contract the sum of squares; that is not pinned.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <map>
#include <utility>
#include <vector>

extern "C" {
int orbo_distinctive_descriptor(int n, const uint8_t* desc);

// Layout-compatible with OrbmConnectionsItem (include/orb_b200.h).
typedef struct OrboConnectionsItem {
    int mode, nKF;
    const uint64_t* order; const uint64_t* mnId; const uint8_t* kfFlags; const float* cameraCenter;
    const int32_t* connStart; const int32_t* connKF; const int32_t* connWeight;
    int firstConnection, nlevels;
    const float* scaleFactors;
    int nSlots;
    const int32_t* slotPoint; const int32_t* slotOctave; const uint8_t* slotDesc;
    int nPoints;
    const uint8_t* pointBad; const float* pointPos; const int32_t* pointRefKF; const int32_t* obsStart; const int32_t* obsKF; const int32_t* obsIdx;
    const int32_t* obsOctave; const uint8_t* obsDesc;
    uint8_t* slotStatus; uint8_t* pointUpdated; float* normal; float* minDistance; float* maxDistance; int32_t* descKF; int32_t* descIdx;
    int32_t* counter; int32_t* nConnected; int32_t* orderedKF; int32_t* orderedWeight; int32_t* parent; int32_t* nbrCount; int32_t* nbrKF;
    int32_t* nbrWeight;
} OrboConnectionsItem;

// The map after the call: every point's mObservations ([nPoints + 1], [obsStart[nPoints] + nPoints] keyframe / keypoint index, key order),
// every keyframe's mConnectedKeyFrameWeights ([nKF + 1], [connStart[nKF] + 2 nKF] keyframe / weight, key order), mlpRecentAddedMapPoints
// (the points pushed, in order), the current keyframe's mbFirstConnection.
typedef struct OrboConnectionsFinal {
    int32_t* obsStart; int32_t* obsKF; int32_t* obsIdx;
    int32_t* connStart; int32_t* connKF; int32_t* connWeight;
    int32_t* recent; int32_t* nRecent; int32_t* firstConnection;
} OrboConnectionsFinal;
}

namespace {

enum { PROCESS_NEW_KEYFRAME = 0, SEARCH_IN_NEIGHBORS = 1 };
enum { SLOT_NONE = 0, SLOT_ADDED, SLOT_IN_KEYFRAME, SLOT_UPDATED };
enum { F_BAD = 1, F_INIT = 2, F_OTHER_MAP = 8 };

struct KeyFrame;
struct ByOrder { bool operator()(const KeyFrame* a, const KeyFrame* b) const; };
struct Map { int id; };
struct KeyFrame {
    int t = 0;                                       // table index
    uint64_t order = 0;
    unsigned long mnId = 0;
    bool mbBad = false, mbFirstConnection = false, init = false;
    Map* mpMap = nullptr;
    float Ow[3] = {0, 0, 0};
    std::map<KeyFrame*, int, ByOrder> mConnectedKeyFrameWeights;
    std::vector<KeyFrame*> mvpOrderedConnectedKeyFrames;
    std::vector<int> mvOrderedWeights;
    bool resorted = false;                           // UpdateBestCovisibles ran (the list is the call's)
    KeyFrame* mpParent = nullptr;
    std::vector<KeyFrame*> children;
    std::vector<struct MapPoint*> mvpMapPoints;      // the current keyframe's slots
    std::vector<int> octave;                         // mvKeysUn[i].octave of the current keyframe
    std::vector<const uint8_t*> desc;                // mDescriptors.row(i) of the current keyframe
    bool isBad() const { return mbBad; }
    Map* GetMap() const { return mpMap; }
    void AddChild(KeyFrame* k) { children.push_back(k); }
    void UpdateBestCovisibles();
    void AddConnection(KeyFrame* pKF, const int& weight);
    void UpdateConnections();
};
bool ByOrder::operator()(const KeyFrame* a, const KeyFrame* b) const { return a->order < b->order; }

struct Obs { int idx, octave; const uint8_t* desc; };
struct MapPoint {
    bool mbBad = false, updated = false;
    int nObs = 0;
    float pos[3] = {0, 0, 0};
    KeyFrame* mpRefKF = nullptr;
    std::map<KeyFrame*, Obs, ByOrder> mObservations;
    float normal[3] = {0, 0, 0}, mfMinDistance = 0, mfMaxDistance = 0;
    KeyFrame* descKF = nullptr;
    int descIdx = -1;
    bool isBad() const { return mbBad; }
    bool IsInKeyFrame(KeyFrame* k) const { return mObservations.count(k) != 0; }
    void AddObservation(KeyFrame* pKF, int idx, int octave, const uint8_t* d) {
        if (mObservations.count(pKF)) return;
        mObservations[pKF] = Obs{idx, octave, d};
        nObs++;
    }
};

// pair<int, KeyFrame*> in the reference's sort order
bool pair_less(const std::pair<int, KeyFrame*>& a, const std::pair<int, KeyFrame*>& b) {
    return a.first < b.first || (a.first == b.first && a.second->order < b.second->order);
}

void KeyFrame::UpdateBestCovisibles() {
    std::vector<std::pair<int, KeyFrame*>> vPairs;
    for (auto& m : mConnectedKeyFrameWeights) vPairs.push_back(std::make_pair(m.second, m.first));
    std::sort(vPairs.begin(), vPairs.end(), pair_less);
    mvpOrderedConnectedKeyFrames.clear(); mvOrderedWeights.clear();
    for (size_t i = vPairs.size(); i-- > 0;)          // push_front of the ascending pairs
        if (!vPairs[i].second->isBad()) { mvpOrderedConnectedKeyFrames.push_back(vPairs[i].second); mvOrderedWeights.push_back(vPairs[i].first); }
    resorted = true;
}

void KeyFrame::AddConnection(KeyFrame* pKF, const int& weight) {
    if (!mConnectedKeyFrameWeights.count(pKF)) mConnectedKeyFrameWeights[pKF] = weight;
    else if (mConnectedKeyFrameWeights[pKF] != weight) mConnectedKeyFrameWeights[pKF] = weight;
    else return;
    UpdateBestCovisibles();
}

float norm3(float x, float y, float z) { return std::sqrt((x * x + y * y) + z * z); }

struct Ctx { int nlevels; const float* sf; };

void UpdateNormalAndDepth(MapPoint* p, const Ctx& c) {
    if (p->mbBad || p->mObservations.empty()) return;
    float normal[3] = {0, 0, 0};
    int n = 0;
    for (auto& o : p->mObservations) {
        const KeyFrame* k = o.first;
        const float v[3] = {p->pos[0] - k->Ow[0], p->pos[1] - k->Ow[1], p->pos[2] - k->Ow[2]};
        const float d = norm3(v[0], v[1], v[2]);
        for (int i = 0; i < 3; ++i) normal[i] = normal[i] + v[i] / d;
        n++;
    }
    const KeyFrame* r = p->mpRefKF;
    const float dist = norm3(p->pos[0] - r->Ow[0], p->pos[1] - r->Ow[1], p->pos[2] - r->Ow[2]);
    const int level = p->mObservations.at(const_cast<KeyFrame*>(r)).octave;
    p->mfMaxDistance = dist * c.sf[level];
    p->mfMinDistance = p->mfMaxDistance / c.sf[c.nlevels - 1];
    for (int i = 0; i < 3; ++i) p->normal[i] = normal[i] / (float)n;
    p->updated = true;
}

void ComputeDistinctiveDescriptors(MapPoint* p) {
    if (p->mbBad || p->mObservations.empty()) return;
    std::vector<uint8_t> rows;
    std::vector<std::pair<KeyFrame*, int>> who;
    for (auto& o : p->mObservations)
        if (!o.first->isBad()) { rows.insert(rows.end(), o.second.desc, o.second.desc + 32); who.push_back(std::make_pair(o.first, o.second.idx)); }
    if (who.empty()) return;
    const int b = orbo_distinctive_descriptor((int)who.size(), rows.data());
    p->descKF = who[b].first; p->descIdx = who[b].second;
    p->updated = true;
}

void KeyFrame::UpdateConnections() {
    std::map<KeyFrame*, int, ByOrder> KFcounter;
    const std::vector<MapPoint*> vpMP = mvpMapPoints;
    for (MapPoint* pMP : vpMP) {
        if (!pMP || pMP->isBad()) continue;
        const std::map<KeyFrame*, Obs, ByOrder> observations = pMP->mObservations;
        for (auto& mit : observations) {
            if (mit.first->mnId == mnId || mit.first->isBad() || mit.first->GetMap() != mpMap) continue;
            KFcounter[mit.first]++;
        }
    }
    if (KFcounter.empty()) return;
    int nmax = 0;
    KeyFrame* pKFmax = nullptr;
    const int th = 15;
    std::vector<std::pair<int, KeyFrame*>> vPairs;
    for (auto& mit : KFcounter) {
        if (mit.second > nmax) { nmax = mit.second; pKFmax = mit.first; }
        if (mit.second >= th) { vPairs.push_back(std::make_pair(mit.second, mit.first)); mit.first->AddConnection(this, mit.second); }
    }
    if (vPairs.empty()) { vPairs.push_back(std::make_pair(nmax, pKFmax)); pKFmax->AddConnection(this, nmax); }
    std::sort(vPairs.begin(), vPairs.end(), pair_less);
    mvpOrderedConnectedKeyFrames.clear(); mvOrderedWeights.clear();
    for (size_t i = vPairs.size(); i-- > 0;) { mvpOrderedConnectedKeyFrames.push_back(vPairs[i].second); mvOrderedWeights.push_back(vPairs[i].first); }
    mConnectedKeyFrameWeights = KFcounter;
    resorted = true;
    if (mbFirstConnection && !init) {
        mpParent = mvpOrderedConnectedKeyFrames.front();
        mpParent->AddChild(this);
        mbFirstConnection = false;
    }
}

}  // namespace

// Runs item `it` and writes its outputs (as the GPU call does) and the final map `fin`.
extern "C" int orbo_update_connections(const OrboConnectionsItem* it, const OrboConnectionsFinal* fin) {
    const int K = it->nKF, P = it->nPoints;
    Map mine{0}, other{1};
    std::vector<KeyFrame> kfs((size_t)K);
    std::vector<MapPoint> pts((size_t)P);
    for (int k = 0; k < K; ++k) {
        KeyFrame& F = kfs[k];
        F.t = k; F.order = it->order[k]; F.mnId = (unsigned long)it->mnId[k];
        F.mbBad = it->kfFlags[k] & F_BAD;
        F.mpMap = (it->kfFlags[k] & F_OTHER_MAP) ? &other : &mine;
        for (int c = 0; c < 3; ++c) F.Ow[c] = it->cameraCenter[3 * k + c];
    }
    for (int k = 0; k < K; ++k)
        for (int c = it->connStart[k]; c < it->connStart[k + 1]; ++c) kfs[k].mConnectedKeyFrameWeights[&kfs[it->connKF[c]]] = it->connWeight[c];
    KeyFrame* KF = &kfs[0];
    KF->mbFirstConnection = it->firstConnection != 0;
    KF->init = it->kfFlags[0] & F_INIT;
    for (int p = 0; p < P; ++p) {
        MapPoint& M = pts[p];
        M.mbBad = it->pointBad[p];
        for (int c = 0; c < 3; ++c) M.pos[c] = it->pointPos[3 * p + c];
        M.mpRefKF = &kfs[it->pointRefKF[p]];
        for (int o = it->obsStart[p]; o < it->obsStart[p + 1]; ++o)
            M.AddObservation(&kfs[it->obsKF[o]], it->obsIdx[o], it->obsOctave[o], it->obsDesc + (size_t)o * 32);
    }
    for (int s = 0; s < it->nSlots; ++s) {
        KF->mvpMapPoints.push_back(it->slotPoint[s] >= 0 ? &pts[it->slotPoint[s]] : nullptr);
        KF->octave.push_back(it->slotOctave[s]);
        KF->desc.push_back(it->slotDesc + (size_t)s * 32);
    }
    const Ctx ctx{it->nlevels, it->scaleFactors};
    std::vector<MapPoint*> recent;
    const std::vector<MapPoint*> vpMapPointMatches = KF->mvpMapPoints;
    for (size_t i = 0; i < vpMapPointMatches.size(); i++) {
        MapPoint* pMP = vpMapPointMatches[i];
        uint8_t st = SLOT_NONE;
        if (pMP && !pMP->isBad()) {
            if (it->mode == PROCESS_NEW_KEYFRAME) {
                if (!pMP->IsInKeyFrame(KF)) {
                    pMP->AddObservation(KF, (int)i, KF->octave[i], KF->desc[i]);
                    UpdateNormalAndDepth(pMP, ctx);
                    ComputeDistinctiveDescriptors(pMP);
                    st = SLOT_ADDED;
                } else {
                    recent.push_back(pMP);
                    st = SLOT_IN_KEYFRAME;
                }
            } else {
                ComputeDistinctiveDescriptors(pMP);
                UpdateNormalAndDepth(pMP, ctx);
                st = SLOT_UPDATED;
            }
        }
        it->slotStatus[i] = st;
    }
    KF->UpdateConnections();

    // outputs
    for (int p = 0; p < P; ++p) {
        const MapPoint& M = pts[p];
        it->pointUpdated[p] = M.updated;
        for (int c = 0; c < 3; ++c) it->normal[3 * p + c] = M.normal[c];
        it->minDistance[p] = M.mfMinDistance; it->maxDistance[p] = M.mfMaxDistance;
        it->descKF[p] = M.descKF ? M.descKF->t : -1; it->descIdx[p] = M.descKF ? M.descIdx : -1;
    }
    const int nNbr = it->connStart[K] + K;
    std::fill(it->counter, it->counter + K, 0);
    std::fill(it->orderedKF, it->orderedKF + K, -1);
    std::fill(it->orderedWeight, it->orderedWeight + K, 0);
    std::fill(it->nbrKF, it->nbrKF + nNbr, -1);
    std::fill(it->nbrWeight, it->nbrWeight + nNbr, 0);
    *it->nConnected = -1;
    *it->parent = KF->mpParent ? KF->mpParent->t : -1;
    if (KF->resorted) {
        for (auto& m : KF->mConnectedKeyFrameWeights) it->counter[m.first->t] = m.second;
        *it->nConnected = (int32_t)KF->mvpOrderedConnectedKeyFrames.size();
        for (size_t r = 0; r < KF->mvpOrderedConnectedKeyFrames.size(); ++r) {
            it->orderedKF[r] = KF->mvpOrderedConnectedKeyFrames[r]->t; it->orderedWeight[r] = KF->mvOrderedWeights[r];
        }
    }
    for (int k = 0; k < K; ++k) {
        it->nbrCount[k] = -1;
        if (k == 0 || !kfs[k].resorted) continue;
        const KeyFrame& F = kfs[k];
        it->nbrCount[k] = (int32_t)F.mvpOrderedConnectedKeyFrames.size();
        for (size_t r = 0; r < F.mvpOrderedConnectedKeyFrames.size(); ++r) {
            it->nbrKF[it->connStart[k] + k + r] = F.mvpOrderedConnectedKeyFrames[r]->t;
            it->nbrWeight[it->connStart[k] + k + r] = F.mvOrderedWeights[r];
        }
    }
    // the final map
    int n = 0;
    fin->obsStart[0] = 0;
    for (int p = 0; p < P; ++p) {
        for (auto& o : pts[p].mObservations) { fin->obsKF[n] = o.first->t; fin->obsIdx[n] = o.second.idx; ++n; }
        fin->obsStart[p + 1] = n;
    }
    n = 0;
    fin->connStart[0] = 0;
    for (int k = 0; k < K; ++k) {
        for (auto& m : kfs[k].mConnectedKeyFrameWeights) { fin->connKF[n] = m.first->t; fin->connWeight[n] = m.second; ++n; }
        fin->connStart[k + 1] = n;
    }
    for (size_t r = 0; r < recent.size(); ++r) fin->recent[r] = (int32_t)(recent[r] - pts.data());
    *fin->nRecent = (int32_t)recent.size();
    *fin->firstConnection = KF->mbFirstConnection;
    return 0;
}
