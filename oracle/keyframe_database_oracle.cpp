// TEST INFRASTRUCTURE ONLY -- CPU oracle of KeyFrameDatabase (src/KeyFrameDatabase.cc, ORB-SLAM3 v1.0, the base of the fork), a literal
// transcription over a pointer model: mvInvertedFile as vector<list<KeyFrame*>> sized mpVoc->size(), add / erase / clear / clearMap, and
// DetectRelocalizationCandidates / DetectNBestCandidates whole (phase 1: the walk and the scores; phase 2: the covisibility accumulation,
// the sort and the selection).  The phase-1 record (lKFsSharingWords with each keyframe's counter, whether it entered lScoreAndMatch and
// its score) is exposed next to the candidates.  The keyframes' marks (mnRelocQuery / mnPlaceRecognitionQuery), counters and scores
// live in the model across queries, so phase 2 reads a stale score where the reference would.  The scene -- BowVectors, ordered
// covisibility lists (GetBestCovisibilityKeyFrames(10) = their first 10, GetConnectedKeyFrames() = all of them), maps, isBad() and
// Map::IsBad() -- is given at creation.  Scores: mpVoc->score = L1Scoring::score, orbo_bow_score_l1 (bow_oracle.cpp, pinned against
// the reference's DBoW2).  Transcribed from ORB-SLAM3 v1.0 src/KeyFrameDatabase.cc: KeyFrameDatabase::add, erase, clear, clearMap,
// DetectRelocalizationCandidates(Frame*, Map*) and DetectNBestCandidates(KeyFrame*, vector<KeyFrame*>&, vector<KeyFrame*>&, int), with
// the file-static compFirst; compare with the fork's file when a checkout is at hand.  One deviation: the NBEST selection loop's
// `if (pKFi->isBad()) continue;` does not advance its iterator, so the reference spins there forever; this oracle returns ORBO_KFDB_SPIN
// instead.
#include <algorithm>
#include <cstdint>
#include <list>
#include <map>
#include <set>
#include <utility>
#include <vector>

extern "C" double orbo_bow_score_l1(int n1, const int* id1, const double* v1, int n2, const int* id2, const double* v2);

namespace {

struct Map { bool bad = false; bool IsBad() const { return bad; } };

struct KeyFrame {
    std::map<unsigned, double> mBowVec;
    std::vector<int> bowId; std::vector<double> bowVal;      // the same BowVector, flat, for orbo_bow_score_l1
    std::vector<KeyFrame*> ordered;                          // mvpOrderedConnectedKeyFrames
    Map* map = nullptr;
    bool bad = false;
    int index = 0;
    uint64_t mnRelocQuery = 0; int mnRelocWords = 0; float mRelocScore = 0;
    uint64_t mnPlaceRecognitionQuery = 0; int mnPlaceRecognitionWords = 0; float mPlaceRecognitionScore = 0;
    bool isBad() const { return bad; }
    Map* GetMap() const { return map; }
    std::vector<KeyFrame*> GetBestCovisibilityKeyFrames(int N) const {
        return std::vector<KeyFrame*>(ordered.begin(), ordered.begin() + std::min<size_t>(ordered.size(), (size_t)N));
    }
    std::set<KeyFrame*> GetConnectedKeyFrames() const { return std::set<KeyFrame*>(ordered.begin(), ordered.end()); }
};

// The query side: a Frame (RELOC) or a KeyFrame (NBEST) -- mnId, mBowVec, and for NBEST its connected keyframes and map.
struct Query {
    uint64_t mnId;
    std::map<unsigned, double> mBowVec;
    std::vector<int> bowId; std::vector<double> bowVal;
    std::set<KeyFrame*> connected;
    Map* map;
    std::set<KeyFrame*> GetConnectedKeyFrames() const { return connected; }
    Map* GetMap() const { return map; }
};

float score(const Query& a, const KeyFrame& b) {
    return (float)orbo_bow_score_l1((int)a.bowId.size(), a.bowId.data(), a.bowVal.data(), (int)b.bowId.size(), b.bowId.data(), b.bowVal.data());
}
bool compFirst(const std::pair<float, KeyFrame*>& a, const std::pair<float, KeyFrame*>& b) { return a.first > b.first; }

struct Database {
    std::vector<std::list<KeyFrame*>> mvInvertedFile;
    std::vector<KeyFrame> kfs;
    std::vector<Map> maps;

    void add(KeyFrame* pKF) {
        for (auto vit = pKF->mBowVec.begin(), vend = pKF->mBowVec.end(); vit != vend; vit++) mvInvertedFile[vit->first].push_back(pKF);
    }
    void erase(KeyFrame* pKF) {
        for (auto vit = pKF->mBowVec.begin(), vend = pKF->mBowVec.end(); vit != vend; vit++) {
            std::list<KeyFrame*>& lKFs = mvInvertedFile[vit->first];
            for (auto lit = lKFs.begin(), lend = lKFs.end(); lit != lend; lit++)
                if (pKF == *lit) { lKFs.erase(lit); break; }
        }
    }
    void clear() {
        mvInvertedFile.clear();
        mvInvertedFile.resize(vocSize);
    }
    void clearMap(Map* pMap) {
        for (std::list<KeyFrame*>& lKFs : mvInvertedFile)
            for (auto lit = lKFs.begin(); lit != lKFs.end();) {
                if (pMap == (*lit)->GetMap()) lit = lKFs.erase(lit);
                else ++lit;
            }
    }
    size_t vocSize = 0;
};

struct Record {
    int cap; int* kf; int* words; uint8_t* scored; float* score; int* nSharing; int* maxCommon;
    void write(const std::list<KeyFrame*>& l, int minCommon, int maxCommonWords, bool reloc) {
        int j = 0;
        for (KeyFrame* p : l) {
            if (j < cap) {
                const int w = reloc ? p->mnRelocWords : p->mnPlaceRecognitionWords;
                kf[j] = p->index; words[j] = w; scored[j] = w > minCommon;
                score[j] = w > minCommon ? (reloc ? p->mRelocScore : p->mPlaceRecognitionScore) : 0.0f;
            }
            ++j;
        }
        *nSharing = j; *maxCommon = maxCommonWords;
    }
};

Query make_query(Database* D, uint64_t id, int nW, const int* wid, const double* wval, int nConn, const int* conn, int map) {
    Query q;
    q.mnId = id;
    for (int k = 0; k < nW; ++k) q.mBowVec[(unsigned)wid[k]] = wval[k];
    q.bowId.assign(wid, wid + nW); q.bowVal.assign(wval, wval + nW);
    for (int c = 0; c < nConn; ++c) q.connected.insert(&D->kfs[conn[c]]);
    q.map = map >= 0 ? &D->maps[map] : nullptr;
    return q;
}

}  // namespace

extern "C" {

enum { ORBO_KFDB_OK = 0, ORBO_KFDB_SPIN = 1 };

// The scene: nKF keyframes with their BowVectors (CSR, ascending ids), maps, isBad(), and ordered covisibility lists (CSR of keyframe
// indices); nMaps maps with Map::IsBad().  The database starts empty.
void* orbo_kfdb_create(int vocSize, int nKF, const int* bowStart, const int* bowId, const double* bowVal, const int* kfMap, const uint8_t* kfBad,
                       const int* covStart, const int* cov, int nMaps, const uint8_t* mapBad) {
    Database* D = new Database();
    D->vocSize = (size_t)vocSize;
    D->mvInvertedFile.resize(D->vocSize);
    D->maps.resize((size_t)nMaps);
    for (int m = 0; m < nMaps; ++m) D->maps[m].bad = mapBad[m] != 0;
    D->kfs.resize((size_t)nKF);
    for (int k = 0; k < nKF; ++k) {
        KeyFrame& K = D->kfs[k];
        K.index = k;
        for (int i = bowStart[k]; i < bowStart[k + 1]; ++i) { K.mBowVec[(unsigned)bowId[i]] = bowVal[i]; K.bowId.push_back(bowId[i]); K.bowVal.push_back(bowVal[i]); }
        K.map = &D->maps[kfMap[k]];
        K.bad = kfBad[k] != 0;
        for (int i = covStart[k]; i < covStart[k + 1]; ++i) K.ordered.push_back(&D->kfs[cov[i]]);
    }
    return D;
}
void orbo_kfdb_destroy(void* o) { delete (Database*)o; }
void orbo_kfdb_add(void* o, int kf) { Database* D = (Database*)o; D->add(&D->kfs[kf]); }
void orbo_kfdb_erase(void* o, int kf) { Database* D = (Database*)o; D->erase(&D->kfs[kf]); }
void orbo_kfdb_clear(void* o) { ((Database*)o)->clear(); }
void orbo_kfdb_clear_map(void* o, int map) { Database* D = (Database*)o; D->clearMap(&D->maps[map]); }
// The inverted-file list of word w, in list order (returns its length; writes at most cap keyframe indices).
int orbo_kfdb_list(void* o, int w, int cap, int* kf) {
    int j = 0;
    for (KeyFrame* p : ((Database*)o)->mvInvertedFile[w]) { if (j < cap) kf[j] = p->index; ++j; }
    return j;
}

// DetectRelocalizationCandidates(F, pMap): F = (queryId, BowVector), pMap = map index.  Record as described above; cand [nKF] = the
// returned vector.
int orbo_kfdb_detect_reloc(void* o, uint64_t queryId, int nW, const int* wid, const double* wval, int map, int cap, int* recKF, int* recWords,
                           uint8_t* recScored, float* recScore, int* nSharing, int* maxCommon, int* cand, int* nCand) {
    Database* D = (Database*)o;
    const Query Fq = make_query(D, queryId, nW, wid, wval, 0, nullptr, map);
    const Query* F = &Fq;
    Map* pMap = Fq.map;
    Record rec{cap, recKF, recWords, recScored, recScore, nSharing, maxCommon};
    *nCand = 0;
    std::list<KeyFrame*> lKFsSharingWords;
    for (auto vit = F->mBowVec.begin(), vend = F->mBowVec.end(); vit != vend; vit++) {
        std::list<KeyFrame*>& lKFs = D->mvInvertedFile[vit->first];
        for (auto lit = lKFs.begin(), lend = lKFs.end(); lit != lend; lit++) {
            KeyFrame* pKFi = *lit;
            if (pKFi->mnRelocQuery != F->mnId) {
                pKFi->mnRelocWords = 0;
                pKFi->mnRelocQuery = F->mnId;
                lKFsSharingWords.push_back(pKFi);
            }
            pKFi->mnRelocWords++;
        }
    }
    if (lKFsSharingWords.empty()) { rec.write(lKFsSharingWords, 0, 0, true); return ORBO_KFDB_OK; }
    int maxCommonWords = 0;
    for (auto lit = lKFsSharingWords.begin(), lend = lKFsSharingWords.end(); lit != lend; lit++)
        if ((*lit)->mnRelocWords > maxCommonWords) maxCommonWords = (*lit)->mnRelocWords;
    int minCommonWords = maxCommonWords * 0.8f;
    std::list<std::pair<float, KeyFrame*>> lScoreAndMatch;
    int nscores = 0;
    for (auto lit = lKFsSharingWords.begin(), lend = lKFsSharingWords.end(); lit != lend; lit++) {
        KeyFrame* pKFi = *lit;
        if (pKFi->mnRelocWords > minCommonWords) {
            nscores++;
            float si = score(*F, *pKFi);
            pKFi->mRelocScore = si;
            lScoreAndMatch.push_back(std::make_pair(si, pKFi));
        }
    }
    rec.write(lKFsSharingWords, minCommonWords, maxCommonWords, true);
    if (lScoreAndMatch.empty()) return ORBO_KFDB_OK;
    std::list<std::pair<float, KeyFrame*>> lAccScoreAndMatch;
    float bestAccScore = 0;
    for (auto it = lScoreAndMatch.begin(), itend = lScoreAndMatch.end(); it != itend; it++) {
        KeyFrame* pKFi = it->second;
        std::vector<KeyFrame*> vpNeighs = pKFi->GetBestCovisibilityKeyFrames(10);
        float bestScore = it->first;
        float accScore = bestScore;
        KeyFrame* pBestKF = pKFi;
        for (auto vit = vpNeighs.begin(), vend = vpNeighs.end(); vit != vend; vit++) {
            KeyFrame* pKF2 = *vit;
            if (pKF2->mnRelocQuery != F->mnId) continue;
            accScore += pKF2->mRelocScore;
            if (pKF2->mRelocScore > bestScore) { pBestKF = pKF2; bestScore = pKF2->mRelocScore; }
        }
        lAccScoreAndMatch.push_back(std::make_pair(accScore, pBestKF));
        if (accScore > bestAccScore) bestAccScore = accScore;
    }
    float minScoreToRetain = 0.75f * bestAccScore;
    std::set<KeyFrame*> spAlreadyAddedKF;
    std::vector<KeyFrame*> vpRelocCandidates;
    vpRelocCandidates.reserve(lAccScoreAndMatch.size());
    for (auto it = lAccScoreAndMatch.begin(), itend = lAccScoreAndMatch.end(); it != itend; it++) {
        const float& si = it->first;
        if (si > minScoreToRetain) {
            KeyFrame* pKFi = it->second;
            if (pKFi->GetMap() != pMap) continue;
            if (!spAlreadyAddedKF.count(pKFi)) { vpRelocCandidates.push_back(pKFi); spAlreadyAddedKF.insert(pKFi); }
        }
    }
    for (KeyFrame* p : vpRelocCandidates) cand[(*nCand)++] = p->index;
    return ORBO_KFDB_OK;
}

// DetectNBestCandidates(pKF, vpLoopCand, vpMergeCand, nNumCandidates): pKF = (queryId, BowVector, connected keyframe indices, map index).
int orbo_kfdb_detect_nbest(void* o, uint64_t queryId, int nW, const int* wid, const double* wval, int nConn, const int* conn, int map, int nNumCandidates,
                           int cap, int* recKF, int* recWords, uint8_t* recScored, float* recScore, int* nSharing, int* maxCommon, int* loop, int* nLoop,
                           int* merge, int* nMerge) {
    Database* D = (Database*)o;
    const Query Kq = make_query(D, queryId, nW, wid, wval, nConn, conn, map);
    const Query* pKF = &Kq;
    Record rec{cap, recKF, recWords, recScored, recScore, nSharing, maxCommon};
    *nLoop = *nMerge = 0;
    std::list<KeyFrame*> lKFsSharingWords;
    std::set<KeyFrame*> spConnectedKF;
    {
        spConnectedKF = pKF->GetConnectedKeyFrames();
        for (auto vit = pKF->mBowVec.begin(), vend = pKF->mBowVec.end(); vit != vend; vit++) {
            std::list<KeyFrame*>& lKFs = D->mvInvertedFile[vit->first];
            for (auto lit = lKFs.begin(), lend = lKFs.end(); lit != lend; lit++) {
                KeyFrame* pKFi = *lit;
                if (pKFi->mnPlaceRecognitionQuery != pKF->mnId) {
                    pKFi->mnPlaceRecognitionWords = 0;
                    if (!spConnectedKF.count(pKFi)) {
                        pKFi->mnPlaceRecognitionQuery = pKF->mnId;
                        lKFsSharingWords.push_back(pKFi);
                    }
                }
                pKFi->mnPlaceRecognitionWords++;
            }
        }
    }
    if (lKFsSharingWords.empty()) { rec.write(lKFsSharingWords, 0, 0, false); return ORBO_KFDB_OK; }
    int maxCommonWords = 0;
    for (auto lit = lKFsSharingWords.begin(), lend = lKFsSharingWords.end(); lit != lend; lit++)
        if ((*lit)->mnPlaceRecognitionWords > maxCommonWords) maxCommonWords = (*lit)->mnPlaceRecognitionWords;
    int minCommonWords = maxCommonWords * 0.8f;
    std::list<std::pair<float, KeyFrame*>> lScoreAndMatch;
    int nscores = 0;
    for (auto lit = lKFsSharingWords.begin(), lend = lKFsSharingWords.end(); lit != lend; lit++) {
        KeyFrame* pKFi = *lit;
        if (pKFi->mnPlaceRecognitionWords > minCommonWords) {
            nscores++;
            float si = score(*pKF, *pKFi);
            pKFi->mPlaceRecognitionScore = si;
            lScoreAndMatch.push_back(std::make_pair(si, pKFi));
        }
    }
    rec.write(lKFsSharingWords, minCommonWords, maxCommonWords, false);
    if (lScoreAndMatch.empty()) return ORBO_KFDB_OK;
    std::list<std::pair<float, KeyFrame*>> lAccScoreAndMatch;
    float bestAccScore = 0;
    for (auto it = lScoreAndMatch.begin(), itend = lScoreAndMatch.end(); it != itend; it++) {
        KeyFrame* pKFi = it->second;
        std::vector<KeyFrame*> vpNeighs = pKFi->GetBestCovisibilityKeyFrames(10);
        float bestScore = it->first;
        float accScore = bestScore;
        KeyFrame* pBestKF = pKFi;
        for (auto vit = vpNeighs.begin(), vend = vpNeighs.end(); vit != vend; vit++) {
            KeyFrame* pKF2 = *vit;
            if (pKF2->mnPlaceRecognitionQuery != pKF->mnId) continue;
            accScore += pKF2->mPlaceRecognitionScore;
            if (pKF2->mPlaceRecognitionScore > bestScore) { pBestKF = pKF2; bestScore = pKF2->mPlaceRecognitionScore; }
        }
        lAccScoreAndMatch.push_back(std::make_pair(accScore, pBestKF));
        if (accScore > bestAccScore) bestAccScore = accScore;
    }
    lAccScoreAndMatch.sort(compFirst);
    std::vector<KeyFrame*> vpLoopCand, vpMergeCand;
    vpLoopCand.reserve(nNumCandidates);
    vpMergeCand.reserve(nNumCandidates);
    std::set<KeyFrame*> spAlreadyAddedKF;
    size_t i = 0;
    auto it = lAccScoreAndMatch.begin();
    while (i < lAccScoreAndMatch.size() && (vpLoopCand.size() < (size_t)nNumCandidates || vpMergeCand.size() < (size_t)nNumCandidates)) {
        KeyFrame* pKFi = it->second;
        if (pKFi->isBad()) return ORBO_KFDB_SPIN;          // the reference: `continue;` without i++ / it++
        if (!spAlreadyAddedKF.count(pKFi)) {
            if (pKF->GetMap() == pKFi->GetMap() && vpLoopCand.size() < (size_t)nNumCandidates) vpLoopCand.push_back(pKFi);
            else if (pKF->GetMap() != pKFi->GetMap() && vpMergeCand.size() < (size_t)nNumCandidates && !pKFi->GetMap()->IsBad()) vpMergeCand.push_back(pKFi);
            spAlreadyAddedKF.insert(pKFi);
        }
        i++;
        it++;
    }
    for (KeyFrame* p : vpLoopCand) loop[(*nLoop)++] = p->index;
    for (KeyFrame* p : vpMergeCand) merge[(*nMerge)++] = p->index;
    return ORBO_KFDB_OK;
}

}  // extern "C"
