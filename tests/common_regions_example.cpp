// A C++ caller of ORBmatcher::CommonRegionsBoWBatch (include/orb_b200/orb_slam3.hpp), built with plain g++ by
// tests/test_common_regions_gpu.py: reads the queries written by the test (dims.txt + one .raw file per query and array), runs them as one
// batch and prints a digest of every query's record (status, covList, nmatches, numBoWMatches, matchedCov, matchedPoint) for a comparison
// with the Python binding.
#include <cstdio>
#include <fstream>
#include <iterator>
#include <string>
#include <vector>

#include "orb_b200/orb_slam3.hpp"

static std::string dir;
static std::vector<char> slurp(const std::string& name) {
    std::ifstream f(dir + "/" + name + ".raw", std::ios::binary);
    return std::vector<char>(std::istreambuf_iterator<char>(f), std::istreambuf_iterator<char>());
}
static void fnv1a(unsigned long long& h, const void* p, size_t bytes) {
    const unsigned char* c = (const unsigned char*)p;
    for (size_t i = 0; i < bytes; ++i) { h ^= c[i]; h *= 1099511628211ull; }
}

struct Query {
    std::vector<std::vector<char>> raw;              // every array read from disk
    std::vector<OrbmCommonRegionsKF> kf;
    std::vector<int32_t> cand, covStart, cov;
    std::vector<uint8_t> status;
    std::vector<int32_t> covList, nmatches, numBoW, matchedCov, matchedPoint;
};

int main(int argc, char** argv) {
    if (argc < 2) { std::fprintf(stderr, "usage: %s DIR\n", argv[0]); return 2; }
    dir = argv[1];
    std::ifstream dims(dir + "/dims.txt");
    int n = 0;
    dims >> n;
    std::vector<Query> Q((size_t)n);
    std::vector<OrbmCommonRegionsQuery> queries((size_t)n);
    for (int i = 0; i < n; ++i) {
        Query& d = Q[i];
        OrbmCommonRegionsQuery& q = queries[i];
        dims >> q.nKF >> q.nPoints >> q.nCand;
        d.cand.resize((size_t)q.nCand);
        for (int32_t& c : d.cand) dims >> c;
        d.covStart.assign((size_t)q.nCand + 1, 0);
        for (int c = 0; c < q.nCand; ++c) { int len = 0; dims >> len; d.covStart[c + 1] = d.covStart[c] + len; }
        d.cov.resize((size_t)d.covStart[q.nCand]);
        for (int32_t& e : d.cov) dims >> e;
        if (!dims) { std::fprintf(stderr, "bad dims.txt\n"); return 2; }
        const std::string qn = "q" + std::to_string(i);
        d.raw.push_back(slurp(qn + "_pointBad"));
        q.pointBad = (const uint8_t*)d.raw.back().data();
        d.kf.resize((size_t)q.nKF);
        d.raw.reserve(2 + 5 * (size_t)q.nKF);
        for (int e = 0; e < q.nKF; ++e) {
            OrbmCommonRegionsKF& k = d.kf[e];
            dims >> k.frame.N >> k.frame.nEntries >> k.bad >> k.connected;
            const std::string kn = qn + "_kf" + std::to_string(e) + "_";
            const char* names[] = {"kps", "desc", "fvNode", "fvFeature", "point"};
            const char* p[5];
            for (int a = 0; a < 5; ++a) { d.raw.push_back(slurp(kn + names[a])); p[a] = d.raw.back().data(); }
            k.frame.keypoints = (const OrbKeyPoint*)p[0]; k.frame.descriptors = (const uint8_t*)p[1];
            k.frame.fvNode = (const int32_t*)p[2]; k.frame.fvFeature = (const int32_t*)p[3]; k.point = (const int32_t*)p[4];
        }
        const size_t C = (size_t)q.nCand, N0 = (size_t)d.kf[0].frame.N;
        d.status.assign(C, 0); d.covList.assign(C * ORBM_CR_MAX_COV, 0); d.nmatches.assign(C * ORBM_CR_MAX_COV, 0); d.numBoW.assign(C, 0);
        d.matchedCov.assign(C * N0, 0); d.matchedPoint.assign(C * N0, 0);
        q.kf = d.kf.data(); q.cand = d.cand.data(); q.covStart = d.covStart.data(); q.cov = d.cov.data();
        q.status = d.status.data(); q.covList = d.covList.data(); q.nmatches = d.nmatches.data(); q.numBoWMatches = d.numBoW.data();
        q.matchedCov = d.matchedCov.data(); q.matchedPoint = d.matchedPoint.data();
    }
    ORB_SLAM3::ORBmatcher matcher;
    matcher.CommonRegionsBoWBatch(queries);
    unsigned long long h = 14695981039346656037ull;
    int ran = 0;
    for (const Query& d : Q) {
        fnv1a(h, d.status.data(), d.status.size());
        fnv1a(h, d.covList.data(), 4 * d.covList.size());
        fnv1a(h, d.nmatches.data(), 4 * d.nmatches.size());
        fnv1a(h, d.numBoW.data(), 4 * d.numBoW.size());
        fnv1a(h, d.matchedCov.data(), 4 * d.matchedCov.size());
        fnv1a(h, d.matchedPoint.data(), 4 * d.matchedPoint.size());
        for (uint8_t s : d.status) ran += s == ORBM_CR_RAN;
    }
    std::printf("digest %016llx\nran %d\nlaunches %d\n", h, ran, orbm_last_launch_count(ORB_SLAM3::detail::matcher_handle(1, 1, 0)));
    return 0;
}
