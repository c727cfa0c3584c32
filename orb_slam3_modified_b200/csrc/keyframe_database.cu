// KeyFrameDatabase (src/KeyFrameDatabase.cc, ORB-SLAM3 v1.0) on the device: the inverted file, and phase 1 of
// DetectRelocalizationCandidates / DetectNBestCandidates -- the shared-word walk and the L1Scoring::score of the keyframes that share
// enough words -- for a batch of queries.  Phase 2 (covisibility accumulation, sort, selection) stays with the caller (DESIGN.md §4).
//
// Layout (DESIGN.md §4): one handle serves several databases from one pool of keyframe slots.  A slot holds the keyframe's key and its
// BowVector as one fixed-width row of maxWords (int32 id, double value) pairs, ascending ids; the rows stay resident.  The host keeps, per
// database, key -> (add sequence number, slot) and the live slots in sequence order.  mvInvertedFile[w] is then "the live slots that hold w,
// in add order", so the reference's lKFsSharingWords -- each keyframe at its first encounter in the walk over the query's words in
// ascending order -- is the sharing slots ordered by (rank of the first query word they share, add order).  A query uploads its
// database's slot order (4 bytes per keyframe) and needs no per-word index.
//
// Three launches whatever the query count:
//   kfdb_share_kernel   a warp per (query, slot): words shared with the query and the rank of the first, by binary search of the row's ids
//                       in the query's ids (shared memory); a connected slot of an NBEST query counts as not sharing;
//   kfdb_order_kernel   a CTA per query: compaction of the sharing slots in add order (block_prefix), a stable LSD radix sort on the first
//                       rank by 1-bit splits (block_prefix per bit), max, minCommonWords, the record;
//   kfdb_score_kernel   a warp per scored entry: L1Scoring::score, the common words' terms gathered by the lanes and added in ascending
//                       word order by one running double (as the reference's loop), then -score / 2.0 rounded to float.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <algorithm>
#include <map>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/orb_b200.h"
#include "device_utils.cuh"
#include "staging.h"

using orbx::set_error;

namespace kfdb {

constexpr int MAX_WORDS = 8192;
constexpr int MAX_BLOCKS_PER_QUERY = 128;
constexpr int MAX_QUERIES = (1 << 24) - 1;   // MAX_BLOCKS_PER_QUERY CTAs per query stay within gridDim.x's 2^31 - 1

// One query as the kernels see it: its inputs and its pieces of the staging buffer.
struct DbQuery {
    int kind, nW, n, cap, nConn;
    const int* qWord; const double* qVal;
    const int* order;                // [n] the database's live slots in add order
    const int* conn;                 // [nConn] connected slots, ascending (NBEST)
    int *cnt, *rank, *A, *B, *P;     // [n] scratch
    int* sorted;                     // [n] the list's slots
    unsigned long long* key; int* words; uint8_t* scored; float* score; int* nSharing; int* maxCommon;
};

struct Pool {
    int W;                           // maxWords: row width
    const int* nWords; const unsigned long long* key; const int* word; const double* value;
};

constexpr int SH_NT = 256, SH_WARPS = SH_NT / 32;
__global__ void __launch_bounds__(SH_NT) kfdb_share_kernel(Pool pool, const DbQuery* __restrict__ queries, int blocksPerQuery) {
    extern __shared__ int s_qw[];
    const int bx = blockIdx.x % blocksPerQuery;                     // blocksPerQuery CTAs per query, queries along x
    const DbQuery& Q = queries[blockIdx.x / blocksPerQuery];
    const int nW = Q.nW, n = Q.n;
    for (int i = threadIdx.x; i < nW; i += SH_NT) s_qw[i] = Q.qWord[i];
    __syncthreads();
    const int lane = threadIdx.x & 31;
    for (int i = bx * SH_WARPS + (threadIdx.x >> 5); i < n; i += blocksPerQuery * SH_WARPS) {
        const int slot = Q.order[i];
        bool connected = false;
        if (Q.kind == ORBV_DB_NBEST) {
            const int lo = orbx::lower_bound(Q.conn, 0, Q.nConn, slot);
            connected = lo < Q.nConn && Q.conn[lo] == slot;
        }
        int count = 0;
        unsigned first = 0xFFFFFFFFu;
        if (!connected) {
            const int m = pool.nWords[slot];
            const int* row = pool.word + (size_t)slot * pool.W;
            for (int k = lane; k < m; k += 32) {
                const int w = row[k];
                const int lo = orbx::lower_bound(s_qw, 0, nW, w);
                if (lo < nW && s_qw[lo] == w) { ++count; first = min(first, (unsigned)lo); }
            }
            count = __reduce_add_sync(0xffffffffu, count);
            first = __reduce_min_sync(0xffffffffu, first);
        }
        if (lane == 0) { Q.cnt[i] = count; Q.rank[i] = (int)first; }
    }
}

constexpr int OR_NT = 512;
__global__ void __launch_bounds__(OR_NT) kfdb_order_kernel(Pool pool, const DbQuery* __restrict__ queries) {
    __shared__ int sm[33];
    __shared__ int s_max[OR_NT / 32];
    const DbQuery Q = queries[blockIdx.x];
    const int n = Q.n, tid = threadIdx.x;
    // lKFsSharingWords in add order: position i of the database's list, compacted
    const int nS = orbx::block_prefix<OR_NT>(n, Q.P, sm, [&](int i) { return Q.cnt[i] > 0 ? 1 : 0; });
    int mx = 0;
    for (int i = tid; i < n; i += OR_NT) {
        const int c = Q.cnt[i];
        if (c > 0) Q.A[Q.P[i]] = i;
        mx = max(mx, c);
    }
    mx = __reduce_max_sync(0xffffffffu, mx);
    if ((tid & 31) == 0) s_max[tid >> 5] = mx;
    __syncthreads();
    mx = 0;
    for (int w = 0; w < OR_NT / 32; ++w) mx = max(mx, s_max[w]);
    // stable sort on the first shared rank: the walk meets a keyframe at its first shared word, keyframes of one word in add order
    int *src = Q.A, *dst = Q.B;
    const int bits = Q.nW > 1 ? 32 - __clz(Q.nW - 1) : 0;
    for (int b = 0; b < bits; ++b) {
        const int zeros = orbx::block_prefix<OR_NT>(nS, Q.P, sm, [&](int j) { return ((Q.rank[src[j]] >> b) & 1) ? 0 : 1; });
        for (int j = tid; j < nS; j += OR_NT) {
            const int p = Q.P[j];
            dst[((Q.rank[src[j]] >> b) & 1) ? zeros + j - p : p] = src[j];
        }
        __syncthreads();
        int* t = src; src = dst; dst = t;
    }
    const int minCommon = (int)__fmul_rn((float)mx, 0.8f);          // int minCommonWords = maxCommonWords * 0.8f;
    for (int j = tid; j < nS; j += OR_NT) Q.sorted[j] = Q.order[src[j]];
    for (int j = tid; j < Q.cap; j += OR_NT) {
        if (j < nS) {
            const int i = src[j], c = Q.cnt[i];
            Q.key[j] = pool.key[Q.order[i]]; Q.words[j] = c; Q.scored[j] = c > minCommon;
        } else {
            Q.key[j] = 0; Q.words[j] = 0; Q.scored[j] = 0;
        }
        Q.score[j] = 0.0f;
    }
    if (tid == 0) { *Q.nSharing = nS; *Q.maxCommon = mx; }
}

constexpr int SC_NT = 256, SC_WARPS = SC_NT / 32;
__global__ void __launch_bounds__(SC_NT) kfdb_score_kernel(Pool pool, const DbQuery* __restrict__ queries, int blocksPerQuery) {
    extern __shared__ double s_qv[];                                 // [nW] values, then [nW] ids
    const int bx = blockIdx.x % blocksPerQuery;
    const DbQuery& Q = queries[blockIdx.x / blocksPerQuery];
    const int nW = Q.nW;
    int* s_qw = reinterpret_cast<int*>(s_qv + nW);
    for (int i = threadIdx.x; i < nW; i += SC_NT) { s_qv[i] = Q.qVal[i]; s_qw[i] = Q.qWord[i]; }
    __syncthreads();
    const int m = min(*Q.nSharing, Q.cap), lane = threadIdx.x & 31;
    for (int j = bx * SC_WARPS + (threadIdx.x >> 5); j < m; j += blocksPerQuery * SC_WARPS) {
        if (!Q.scored[j]) continue;
        const int slot = Q.sorted[j], nr = pool.nWords[slot];
        const int* row = pool.word + (size_t)slot * pool.W;
        const double* val = pool.value + (size_t)slot * pool.W;
        double score = 0.0;
        for (int k0 = 0; k0 < nr; k0 += 32) {
            const int k = k0 + lane;
            double term = 0.0;
            bool hit = false;
            if (k < nr) {
                const int w = row[k];
                const int lo = orbx::lower_bound(s_qw, 0, nW, w);
                if (lo < nW && s_qw[lo] == w) {
                    const double vi = s_qv[lo], wi = val[k];
                    term = __dsub_rn(__dsub_rn(fabs(__dsub_rn(vi, wi)), fabs(vi)), fabs(wi));   // fabs(vi-wi) - fabs(vi) - fabs(wi)
                    hit = true;
                }
            }
            unsigned hits = __ballot_sync(0xffffffffu, hit);
            while (hits) {                                           // score += term, in ascending word order (the row's order)
                const int l = __ffs(hits) - 1;
                score = __dadd_rn(score, __shfl_sync(0xffffffffu, term, l));
                hits &= hits - 1;
            }
        }
        if (lane == 0) Q.score[j] = __double2float_rn(-score / 2.0);
    }
}

// add: a CTA per keyframe writes its slot's key, word count and row
constexpr int ADD_NT = 128;
__global__ void __launch_bounds__(ADD_NT) kfdb_add_kernel(int W, int* __restrict__ nWords, unsigned long long* __restrict__ slotKey, int* __restrict__ word,
                                                          double* __restrict__ value, const int* __restrict__ slot, const unsigned long long* __restrict__ key,
                                                          const int* __restrict__ start, const int* __restrict__ id, const double* __restrict__ val) {
    const int i = blockIdx.x, s = slot[i], b = start[i], m = start[i + 1] - b;
    int* row = word + (size_t)s * W;
    double* rowVal = value + (size_t)s * W;
    for (int k = threadIdx.x; k < m; k += ADD_NT) { row[k] = id[b + k]; rowVal[k] = val[b + k]; }
    if (threadIdx.x == 0) { nWords[s] = m; slotKey[s] = key[i]; }
}

}  // namespace kfdb

using namespace kfdb;

struct orbv_db_handle {
    int device = 0, vocabularyWords = 0, maxDatabases = 0, maxKeyFrames = 0, maxWords = 0, launches = 0;
    uint8_t* d_arena = nullptr;
    Pool pool{};
    int* d_nWords = nullptr; unsigned long long* d_key = nullptr; int* d_word = nullptr; double* d_value = nullptr;
    cudaStream_t st = nullptr;
    orbx::Staging staging;
    // Every entry point holds it for the whole call: the staging buffers, the free list, the sequence counter and the launch count belong
    // to the handle, not to one database, so calls for different databases (different SLAM systems) are serialised here.
    mutable std::mutex mu;
    struct Entry { uint64_t seq; int slot; };
    struct Database { std::unordered_map<uint64_t, Entry> byKey; std::map<uint64_t, int> bySeq; };
    std::vector<Database> dbs;
    std::vector<int> freeSlots;      // a stack: the next add takes the back
    uint64_t nextSeq = 0;
    ~orbv_db_handle() {
        staging.release();
        cudaSetDevice(device);
        if (d_arena) cudaFree(d_arena);
        if (st) cudaStreamDestroy(st);
    }
};

namespace {

void release_slots(orbv_db_handle* h, orbv_db_handle::Database& D) {
    for (const auto& e : D.bySeq) h->freeSlots.push_back(e.second);
    D.byKey.clear(); D.bySeq.clear();
}

// A BowVector as the entry points take it: n ascending ids in [0, vocabularyWords), n <= maxWords.
int check_bow(const orbv_db_handle* h, const char* where, int i, int n, const int32_t* id, const double* value) {
    auto bad = [&](const char* what) { set_error(std::string(where) + ": item " + std::to_string(i) + ": " + what); return ORB_ERR_ARG; };
    if (n < 0 || n > h->maxWords) return bad("word count outside [0, maxWords]");
    if (n > 0 && (!id || !value)) return bad("word ids / values are null");
    for (int k = 0; k < n; ++k) {
        if (id[k] < 0 || id[k] >= h->vocabularyWords) return bad("word id outside [0, vocabularyWords)");
        if (k > 0 && id[k] <= id[k - 1]) return bad("word ids do not ascend");
    }
    return ORB_OK;
}

}  // namespace

extern "C" {

int orbv_db_create(orbv_db_handle** out, int vocabularyWords, int maxDatabases, int maxKeyFrames, int maxWords, int device) {
    if (!out || vocabularyWords < 1 || maxDatabases < 1 || maxKeyFrames < 1 || maxWords < 1 || maxWords > MAX_WORDS) {
        set_error("orbv_db_create: bad argument (every size >= 1, maxWords <= " + std::to_string(MAX_WORDS) + ")");
        return ORB_ERR_ARG;
    }
    if (int rc = orbx::check_device(device)) return rc;
    CK(cudaSetDevice(device));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, device));
    if (int rc = orbx::require_sm90(prop.major, prop.minor)) return rc;
    orbv_db_handle* h = new orbv_db_handle();
    h->device = h->staging.device = device;
    h->vocabularyWords = vocabularyWords; h->maxDatabases = maxDatabases; h->maxKeyFrames = maxKeyFrames; h->maxWords = maxWords;
    auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
    const size_t K = maxKeyFrames, W = maxWords;
    const size_t oN = 0, oK = oN + al(4 * K), oW = oK + al(8 * K), oV = oW + al(4 * K * W), total = oV + al(8 * K * W);
    cudaError_t e = cudaMalloc(&h->d_arena, total);
    if (e == cudaSuccess) e = cudaMemset(h->d_arena, 0, total);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&h->st, cudaStreamNonBlocking);
    if (e != cudaSuccess) { set_error(std::string("orbv_db_create: ") + cudaGetErrorString(e)); delete h; return ORB_ERR_CUDA; }
    h->d_nWords = (int*)(h->d_arena + oN); h->d_key = (unsigned long long*)(h->d_arena + oK);
    h->d_word = (int*)(h->d_arena + oW); h->d_value = (double*)(h->d_arena + oV);
    h->pool = Pool{maxWords, h->d_nWords, h->d_key, h->d_word, h->d_value};
    h->dbs.resize((size_t)maxDatabases);
    h->freeSlots.reserve(K);
    for (int s = maxKeyFrames - 1; s >= 0; --s) h->freeSlots.push_back(s);
    *out = h;
    return ORB_OK;
}

void orbv_db_destroy(orbv_db_handle* h) { delete h; }

int orbv_db_last_launch_count(const orbv_db_handle* h) {
    if (!h) return -1;
    std::lock_guard<std::mutex> lock(h->mu);
    return h->launches;
}

int orbv_db_add_batch(orbv_db_handle* h, int n, const int32_t* dbIndex, const uint64_t* key, const int32_t* wordStart, const int32_t* wordId,
                      const double* wordValue) {
    const char* where = "orbv_db_add_batch";
    if (!h || n < 0 || (n > 0 && (!dbIndex || !key || !wordStart))) { set_error(std::string(where) + ": bad argument"); return ORB_ERR_ARG; }
    std::lock_guard<std::mutex> lock(h->mu);
    if (n > 0 && !orbx::csr_ok(n, wordStart)) { set_error(std::string(where) + ": wordStart must start at 0 and not decrease"); return ORB_ERR_ARG; }
    std::vector<std::pair<int, uint64_t>> seen;
    for (int i = 0; i < n; ++i) {
        const int d = dbIndex[i];
        if (d < 0 || d >= h->maxDatabases) { set_error(std::string(where) + ": item " + std::to_string(i) + ": database index out of range"); return ORB_ERR_ARG; }
        if (h->dbs[d].byKey.count(key[i])) { set_error(std::string(where) + ": item " + std::to_string(i) + ": key already in the database"); return ORB_ERR_ARG; }
        if (int rc = check_bow(h, where, i, wordStart[i + 1] - wordStart[i], wordId ? wordId + wordStart[i] : nullptr,
                               wordValue ? wordValue + wordStart[i] : nullptr)) return rc;
        seen.push_back({d, key[i]});
    }
    std::sort(seen.begin(), seen.end());
    if (std::adjacent_find(seen.begin(), seen.end()) != seen.end()) { set_error(std::string(where) + ": a key is added twice to one database"); return ORB_ERR_ARG; }
    if ((size_t)n > h->freeSlots.size()) {
        set_error(std::string(where) + ": " + std::to_string(n) + " keyframes, " + std::to_string(h->freeSlots.size()) + " free slots (maxKeyFrames)");
        return ORB_ERR_CAPACITY;
    }
    h->launches = 0;
    if (n == 0) return ORB_OK;
    CK(cudaSetDevice(h->device));
    std::vector<int> slot((size_t)n);                                // taken from the free list only once the rows are on the device
    for (int i = 0; i < n; ++i) slot[i] = h->freeSlots[h->freeSlots.size() - 1 - (size_t)i];
    const size_t nw = (size_t)wordStart[n];
    orbx::Staging& S = h->staging;
    S.begin();
    const int pSlot = S.in(slot.data(), 4 * (size_t)n), pKey = S.in(key, 8 * (size_t)n), pStart = S.in(wordStart, 4 * (size_t)(n + 1)),
              pId = S.in(wordId, 4 * nw), pVal = S.in(wordValue, 8 * nw);
    if (int rc = S.reserve()) return rc;
    CK(S.upload(h->st));
    const int* dSlot = S.dev<int>(pSlot); const unsigned long long* dKey = S.dev<unsigned long long>(pKey); const int* dStart = S.dev<int>(pStart);
    const int* dId = S.dev<int>(pId); const double* dVal = S.dev<double>(pVal);
    kfdb_add_kernel<<<n, ADD_NT, 0, h->st>>>(h->maxWords, h->d_nWords, h->d_key, h->d_word, h->d_value, dSlot, dKey, dStart, dId, dVal);
    CK(cudaGetLastError());
    h->launches = 1;
    CK(S.download(h->st));
    h->freeSlots.resize(h->freeSlots.size() - (size_t)n);
    for (int i = 0; i < n; ++i) {
        orbv_db_handle::Database& D = h->dbs[dbIndex[i]];
        const uint64_t seq = h->nextSeq++;
        D.byKey[key[i]] = {seq, slot[i]};
        D.bySeq[seq] = slot[i];
    }
    return ORB_OK;
}

int orbv_db_erase_batch(orbv_db_handle* h, int n, const int32_t* dbIndex, const uint64_t* key) {
    if (!h || n < 0 || (n > 0 && (!dbIndex || !key))) { set_error("orbv_db_erase_batch: bad argument"); return ORB_ERR_ARG; }
    std::lock_guard<std::mutex> lock(h->mu);
    for (int i = 0; i < n; ++i)
        if (dbIndex[i] < 0 || dbIndex[i] >= h->maxDatabases) {
            set_error("orbv_db_erase_batch: item " + std::to_string(i) + ": database index out of range");
            return ORB_ERR_ARG;
        }
    h->launches = 0;
    for (int i = 0; i < n; ++i) {
        orbv_db_handle::Database& D = h->dbs[dbIndex[i]];
        auto it = D.byKey.find(key[i]);
        if (it == D.byKey.end()) continue;                            // not in the database: a no-op, as in the reference
        D.bySeq.erase(it->second.seq);
        h->freeSlots.push_back(it->second.slot);
        D.byKey.erase(it);
    }
    return ORB_OK;
}

int orbv_db_clear(orbv_db_handle* h, int dbIndex) {
    if (!h || dbIndex < 0 || dbIndex >= h->maxDatabases) { set_error("orbv_db_clear: bad argument"); return ORB_ERR_ARG; }
    std::lock_guard<std::mutex> lock(h->mu);
    h->launches = 0;
    release_slots(h, h->dbs[dbIndex]);
    return ORB_OK;
}

int orbv_db_size(const orbv_db_handle* h, int dbIndex) {
    if (!h || dbIndex < 0 || dbIndex >= h->maxDatabases) { set_error("orbv_db_size: bad argument"); return ORB_ERR_ARG; }
    std::lock_guard<std::mutex> lock(h->mu);
    return (int)h->dbs[dbIndex].byKey.size();
}

int orbv_db_query_batch(orbv_db_handle* h, int nQueries, const OrbvDbQuery* q) {
    const char* where = "orbv_db_query_batch";
    if (!h || nQueries < 0 || nQueries > MAX_QUERIES || (nQueries > 0 && !q)) {
        set_error(std::string(where) + ": bad argument (nQueries in [0, " + std::to_string(MAX_QUERIES) + "])");
        return ORB_ERR_ARG;
    }
    std::lock_guard<std::mutex> lock(h->mu);
    for (int j = 0; j < nQueries; ++j) {
        const OrbvDbQuery& Q = q[j];
        auto bad = [&](const char* what) { set_error(std::string(where) + ": query " + std::to_string(j) + ": " + what); return ORB_ERR_ARG; };
        if (Q.dbIndex < 0 || Q.dbIndex >= h->maxDatabases) return bad("database index out of range");
        if (Q.kind != ORBV_DB_RELOC && Q.kind != ORBV_DB_NBEST) return bad("kind is neither ORBV_DB_RELOC nor ORBV_DB_NBEST");
        if (Q.cap < 0) return bad("negative cap");
        if (!Q.nSharing || !Q.maxCommonWords || (Q.cap > 0 && (!Q.key || !Q.words || !Q.scored || !Q.score))) return bad("an output is null");
        if (Q.kind == ORBV_DB_NBEST && (Q.nConnected < 0 || (Q.nConnected > 0 && !Q.connected))) return bad("bad connected keys");
        if (int rc = check_bow(h, where, j, Q.nWords, Q.wordId, Q.wordValue)) return rc;
    }
    h->launches = 0;
    if (nQueries == 0) return ORB_OK;
    CK(cudaSetDevice(h->device));
    // each queried database's live slots in add order, once per call
    std::map<int, std::vector<int>> order;
    for (int j = 0; j < nQueries; ++j) {
        auto ins = order.emplace(q[j].dbIndex, std::vector<int>());
        if (ins.second)
            for (const auto& e : h->dbs[q[j].dbIndex].bySeq) ins.first->second.push_back(e.second);
    }
    std::vector<std::vector<int>> conn((size_t)nQueries);
    int maxN = 0, maxW = 0;
    for (int j = 0; j < nQueries; ++j) {
        const OrbvDbQuery& Q = q[j];
        if (Q.kind == ORBV_DB_NBEST) {
            const auto& byKey = h->dbs[Q.dbIndex].byKey;
            for (int c = 0; c < Q.nConnected; ++c) {
                auto it = byKey.find(Q.connected[c]);
                if (it != byKey.end()) conn[j].push_back(it->second.slot);   // keys not in the database are ignored
            }
            std::sort(conn[j].begin(), conn[j].end());
            conn[j].erase(std::unique(conn[j].begin(), conn[j].end()), conn[j].end());
        }
        maxN = std::max(maxN, (int)order[Q.dbIndex].size());
        maxW = std::max(maxW, Q.nWords);
    }
    orbx::Staging& S = h->staging;
    S.begin();
    std::map<int, int> orderPiece;
    for (const auto& o : order) orderPiece[o.first] = S.in(o.second.data(), 4 * o.second.size());
    struct Pieces { int w, v, conn, cnt, rank, A, B, P, sorted, key, words, scored, score, nS, mx; };
    std::vector<Pieces> pc((size_t)nQueries);
    for (int j = 0; j < nQueries; ++j) {
        const OrbvDbQuery& Q = q[j];
        const size_t n = order[Q.dbIndex].size(), cap = (size_t)Q.cap, nw = (size_t)Q.nWords;
        Pieces& p = pc[j];
        p.w = S.in(Q.wordId, 4 * nw); p.v = S.in(Q.wordValue, 8 * nw); p.conn = S.in(conn[j].data(), 4 * conn[j].size());
        p.cnt = S.scratch(4 * n); p.rank = S.scratch(4 * n); p.A = S.scratch(4 * n); p.B = S.scratch(4 * n); p.P = S.scratch(4 * n);
        p.sorted = S.scratch(4 * n);
        p.key = S.out(Q.key, 8 * cap); p.words = S.out(Q.words, 4 * cap); p.scored = S.out(Q.scored, cap); p.score = S.out(Q.score, 4 * cap);
        p.nS = S.out(Q.nSharing, 4); p.mx = S.out(Q.maxCommonWords, 4);
    }
    const int tab = S.in(nullptr, sizeof(DbQuery) * (size_t)nQueries);
    if (int rc = S.reserve()) return rc;
    DbQuery* T = S.host<DbQuery>(tab);
    for (int j = 0; j < nQueries; ++j) {
        const OrbvDbQuery& Q = q[j];
        const Pieces& p = pc[j];
        DbQuery d;
        d.kind = Q.kind; d.nW = Q.nWords; d.n = (int)order[Q.dbIndex].size(); d.cap = Q.cap; d.nConn = (int)conn[j].size();
        d.qWord = S.dev<int>(p.w); d.qVal = S.dev<double>(p.v); d.order = S.dev<int>(orderPiece[Q.dbIndex]); d.conn = S.dev<int>(p.conn);
        d.cnt = S.dev<int>(p.cnt); d.rank = S.dev<int>(p.rank); d.A = S.dev<int>(p.A); d.B = S.dev<int>(p.B); d.P = S.dev<int>(p.P);
        d.sorted = S.dev<int>(p.sorted);
        d.key = S.dev<unsigned long long>(p.key); d.words = S.dev<int>(p.words); d.scored = S.dev(p.scored); d.score = S.dev<float>(p.score);
        d.nSharing = S.dev<int>(p.nS); d.maxCommon = S.dev<int>(p.mx);
        T[j] = d;
    }
    CK(S.upload(h->st));
    const DbQuery* dq = S.dev<DbQuery>(tab);
    const int bpq = std::min(std::max((maxN + SH_WARPS - 1) / SH_WARPS, 1), MAX_BLOCKS_PER_QUERY);
    const unsigned gx = (unsigned)bpq * (unsigned)nQueries;
    const size_t smShare = 4 * (size_t)std::max(maxW, 1), smScore = 12 * (size_t)std::max(maxW, 1);
    if (int rc = orbx::ensure_dynamic_smem(kfdb_share_kernel, smShare, h->device)) return rc;
    if (int rc = orbx::ensure_dynamic_smem(kfdb_score_kernel, smScore, h->device)) return rc;
    kfdb_share_kernel<<<gx, SH_NT, smShare, h->st>>>(h->pool, dq, bpq);
    kfdb_order_kernel<<<(unsigned)nQueries, OR_NT, 0, h->st>>>(h->pool, dq);
    kfdb_score_kernel<<<gx, SC_NT, smScore, h->st>>>(h->pool, dq, bpq);
    CK(cudaGetLastError());
    h->launches = 3;
    CK(S.download(h->st));
    for (int j = 0; j < nQueries; ++j)
        if (*q[j].nSharing > q[j].cap) {
            set_error(std::string(where) + ": query " + std::to_string(j) + ": " + std::to_string(*q[j].nSharing) + " keyframes share words, cap is " +
                      std::to_string(q[j].cap));
            return ORB_ERR_CAPACITY;
        }
    return ORB_OK;
}

}  // extern "C"
