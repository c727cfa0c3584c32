// A C++ caller of ORBmatcher::UpdateConnectionsBatch (include/orb_b200/orb_slam3.hpp), built with plain g++ by
// tests/test_update_connections_gpu.py: reads the items written by the test (dims.txt + one .raw file per item and array), runs them as
// one batch and prints a digest of every item's outputs, in the order of OrbmConnectionsItem, for a comparison with the Python binding.
#include <cstdio>
#include <fstream>
#include <iterator>
#include <string>
#include <vector>

#include "orb_b200/orb_slam3.hpp"

static std::string dir;
static std::vector<char> slurp(int item, const char* name) {
    std::ifstream f(dir + "/item" + std::to_string(item) + "_" + name + ".raw", std::ios::binary);
    return std::vector<char>(std::istreambuf_iterator<char>(f), std::istreambuf_iterator<char>());
}
static void fnv1a(unsigned long long& h, const void* p, size_t bytes) {
    const unsigned char* c = (const unsigned char*)p;
    for (size_t i = 0; i < bytes; ++i) { h ^= c[i]; h *= 1099511628211ull; }
}

struct Outputs {
    std::vector<uint8_t> slotStatus, pointUpdated;
    std::vector<float> normal, minDistance, maxDistance;
    std::vector<int32_t> descKF, descIdx, counter, nConnected, orderedKF, orderedWeight, parent, nbrCount, nbrKF, nbrWeight;
};

int main(int argc, char** argv) {
    if (argc < 2) { std::fprintf(stderr, "usage: %s DIR\n", argv[0]); return 2; }
    dir = argv[1];
    std::ifstream dims(dir + "/dims.txt");
    int n = 0;
    dims >> n;
    const char* names[] = {"order", "mnId", "kfFlags", "cameraCenter", "connStart", "connKF", "connWeight", "scaleFactors", "slotPoint", "slotOctave",
                           "slotDesc", "pointBad", "pointPos", "pointRefKF", "obsStart", "obsKF", "obsIdx", "obsOctave", "obsDesc"};
    std::vector<std::vector<std::vector<char>>> a((size_t)n);
    std::vector<Outputs> o((size_t)n);
    std::vector<OrbmConnectionsItem> items((size_t)n);
    for (int j = 0; j < n; ++j) {
        OrbmConnectionsItem& it = items[j];
        dims >> it.mode >> it.firstConnection >> it.nKF >> it.nlevels >> it.nSlots >> it.nPoints;
        if (!dims) { std::fprintf(stderr, "bad dims.txt\n"); return 2; }
        for (const char* nm : names) a[j].push_back(slurp(j, nm));
        const std::vector<std::vector<char>>& r = a[j];
        auto ptr = [&](int k) { return r[k].empty() ? nullptr : r[k].data(); };
        it.order = (const uint64_t*)ptr(0); it.mnId = (const uint64_t*)ptr(1); it.kfFlags = (const uint8_t*)ptr(2); it.cameraCenter = (const float*)ptr(3);
        it.connStart = (const int32_t*)ptr(4); it.connKF = (const int32_t*)ptr(5); it.connWeight = (const int32_t*)ptr(6);
        it.scaleFactors = (const float*)ptr(7); it.slotPoint = (const int32_t*)ptr(8); it.slotOctave = (const int32_t*)ptr(9);
        it.slotDesc = (const uint8_t*)ptr(10); it.pointBad = (const uint8_t*)ptr(11); it.pointPos = (const float*)ptr(12);
        it.pointRefKF = (const int32_t*)ptr(13); it.obsStart = (const int32_t*)ptr(14); it.obsKF = (const int32_t*)ptr(15);
        it.obsIdx = (const int32_t*)ptr(16); it.obsOctave = (const int32_t*)ptr(17); it.obsDesc = (const uint8_t*)ptr(18);
        const size_t K = (size_t)it.nKF, S = (size_t)it.nSlots, P = (size_t)it.nPoints, NB = (size_t)it.connStart[it.nKF] + K;
        Outputs& q = o[j];
        q.slotStatus.assign(S, 0); q.pointUpdated.assign(P, 0); q.normal.assign(3 * P, 0.f); q.minDistance.assign(P, 0.f); q.maxDistance.assign(P, 0.f);
        q.descKF.assign(P, 0); q.descIdx.assign(P, 0); q.counter.assign(K, 0); q.nConnected.assign(1, 0); q.orderedKF.assign(K, 0);
        q.orderedWeight.assign(K, 0); q.parent.assign(1, 0); q.nbrCount.assign(K, 0); q.nbrKF.assign(NB, 0); q.nbrWeight.assign(NB, 0);
        it.slotStatus = q.slotStatus.data(); it.pointUpdated = q.pointUpdated.data(); it.normal = q.normal.data(); it.minDistance = q.minDistance.data();
        it.maxDistance = q.maxDistance.data(); it.descKF = q.descKF.data(); it.descIdx = q.descIdx.data(); it.counter = q.counter.data();
        it.nConnected = q.nConnected.data(); it.orderedKF = q.orderedKF.data(); it.orderedWeight = q.orderedWeight.data(); it.parent = q.parent.data();
        it.nbrCount = q.nbrCount.data(); it.nbrKF = q.nbrKF.data(); it.nbrWeight = q.nbrWeight.data();
    }
    ORB_SLAM3::ORBmatcher matcher;
    matcher.UpdateConnectionsBatch(items);
    unsigned long long h = 14695981039346656037ull;
    int updated = 0;
    for (const Outputs& q : o) {
        fnv1a(h, q.slotStatus.data(), q.slotStatus.size()); fnv1a(h, q.pointUpdated.data(), q.pointUpdated.size());
        fnv1a(h, q.normal.data(), 4 * q.normal.size()); fnv1a(h, q.minDistance.data(), 4 * q.minDistance.size());
        fnv1a(h, q.maxDistance.data(), 4 * q.maxDistance.size());
        for (const std::vector<int32_t>* v : {&q.descKF, &q.descIdx, &q.counter, &q.nConnected, &q.orderedKF, &q.orderedWeight, &q.parent, &q.nbrCount,
                                              &q.nbrKF, &q.nbrWeight})
            fnv1a(h, v->data(), 4 * v->size());
        for (uint8_t u : q.pointUpdated) updated += u;
    }
    std::printf("digest %016llx\nupdated %d\nlaunches %d\n", h, updated, orbm_last_launch_count(ORB_SLAM3::detail::matcher_handle(1, 1, 0)));
    return 0;
}
