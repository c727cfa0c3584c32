// A C++ caller of ORB_SLAM3::KeyFrameDatabase (include/orb_b200/orb_slam3.hpp), built with plain g++ by tests/test_keyframe_database_gpu.py:
// reads the keyframes and queries written by the test (dims.txt + .raw files), adds the keyframes in one batch, runs the queries as one
// QueryBatch and prints a digest of every query's (key, words, scored, score, nSharing, maxCommonWords) for a comparison with the Python
// binding.
#include <cstdio>
#include <cstring>
#include <fstream>
#include <iterator>
#include <string>
#include <vector>

#include "orb_b200/orb_slam3.hpp"

static std::string dir;
template <class T> static std::vector<T> slurp(const char* name) {
    std::ifstream f(dir + "/" + name + ".raw", std::ios::binary);
    std::vector<char> b((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
    std::vector<T> out(b.size() / sizeof(T));
    if (!out.empty()) std::memcpy(out.data(), b.data(), out.size() * sizeof(T));
    return out;
}
static void fnv1a(unsigned long long& h, const void* p, size_t bytes) {
    const unsigned char* c = (const unsigned char*)p;
    for (size_t i = 0; i < bytes; ++i) { h ^= c[i]; h *= 1099511628211ull; }
}

int main(int argc, char** argv) {
    if (argc < 2) { std::fprintf(stderr, "usage: %s DIR\n", argv[0]); return 2; }
    dir = argv[1];
    std::ifstream dims(dir + "/dims.txt");
    int vocWords = 0, nDb = 0, maxKF = 0, maxWords = 0, cap = 0;
    dims >> vocWords >> nDb >> maxKF >> maxWords >> cap;
    if (!dims) { std::fprintf(stderr, "bad dims.txt\n"); return 2; }
    const std::vector<int32_t> addDb = slurp<int32_t>("add_db"), addStart = slurp<int32_t>("add_start"), addId = slurp<int32_t>("add_id");
    const std::vector<uint64_t> addKey = slurp<uint64_t>("add_key");
    const std::vector<double> addVal = slurp<double>("add_val");
    std::vector<ORB_SLAM3::KeyFrameDatabase::BowVector> bows(addKey.size());
    for (size_t i = 0; i < addKey.size(); ++i) {
        bows[i].id.assign(addId.begin() + addStart[i], addId.begin() + addStart[i + 1]);
        bows[i].value.assign(addVal.begin() + addStart[i], addVal.begin() + addStart[i + 1]);
    }
    ORB_SLAM3::KeyFrameDatabase database(vocWords, nDb, maxKF, maxWords);
    database.add(addDb, addKey, bows);

    const std::vector<int32_t> meta = slurp<int32_t>("q_meta"), qId = slurp<int32_t>("q_id");   // meta: [nQ][4] db, kind, nWords, nConnected
    const std::vector<double> qVal = slurp<double>("q_val");
    const std::vector<uint64_t> qConn = slurp<uint64_t>("q_conn");
    const size_t nQ = meta.size() / 4;
    std::vector<uint64_t> key(nQ * cap);
    std::vector<int32_t> words(nQ * cap), nSharing(nQ), maxCommon(nQ);
    std::vector<uint8_t> scored(nQ * cap);
    std::vector<float> score(nQ * cap);
    std::vector<OrbvDbQuery> queries(nQ);
    size_t w = 0, c = 0;
    for (size_t j = 0; j < nQ; ++j) {
        OrbvDbQuery& q = queries[j];
        q.dbIndex = meta[4 * j]; q.kind = meta[4 * j + 1]; q.nWords = meta[4 * j + 2]; q.nConnected = meta[4 * j + 3];
        q.wordId = qId.data() + w; q.wordValue = qVal.data() + w; q.connected = qConn.data() + c;
        w += (size_t)q.nWords; c += (size_t)q.nConnected;
        q.cap = cap;
        q.key = key.data() + j * cap; q.words = words.data() + j * cap; q.scored = scored.data() + j * cap; q.score = score.data() + j * cap;
        q.nSharing = &nSharing[j]; q.maxCommonWords = &maxCommon[j];
    }
    database.QueryBatch(queries);
    unsigned long long h = 14695981039346656037ull;
    int total = 0;
    for (size_t j = 0; j < nQ; ++j) {
        fnv1a(h, key.data() + j * cap, 8 * (size_t)cap);
        fnv1a(h, words.data() + j * cap, 4 * (size_t)cap);
        fnv1a(h, scored.data() + j * cap, (size_t)cap);
        fnv1a(h, score.data() + j * cap, 4 * (size_t)cap);
        fnv1a(h, &nSharing[j], 4);
        fnv1a(h, &maxCommon[j], 4);
        total += nSharing[j];
    }
    std::printf("digest %016llx\nsharing %d\nlaunches %d\n", h, total, orbv_db_last_launch_count(database.handle()));
    return 0;
}
