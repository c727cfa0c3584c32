// A C++ caller of ORBmatcher::KeyFrameCullingBatch (include/orb_b200/orb_slam3.hpp), built with plain g++ by
// tests/test_keyframe_culling_gpu.py: reads the maps written by the test (dims.txt + one .raw file per map and array), runs them as one
// batch and prints a digest of every map's (status, nMPs, nRedundant, visited) for a comparison with the Python binding.
#include <cstdio>
#include <fstream>
#include <iterator>
#include <string>
#include <vector>

#include "orb_b200/orb_slam3.hpp"

static std::string dir;
static std::vector<char> slurp(int map, const char* name) {
    std::ifstream f(dir + "/map" + std::to_string(map) + "_" + name + ".raw", std::ios::binary);
    return std::vector<char>(std::istreambuf_iterator<char>(f), std::istreambuf_iterator<char>());
}
static void fnv1a(unsigned long long& h, const void* p, size_t bytes) {
    const unsigned char* c = (const unsigned char*)p;
    for (size_t i = 0; i < bytes; ++i) { h ^= c[i]; h *= 1099511628211ull; }
}

int main(int argc, char** argv) {
    if (argc < 2) { std::fprintf(stderr, "usage: %s DIR\n", argv[0]); return 2; }
    dir = argv[1];
    std::ifstream dims(dir + "/dims.txt");
    int n = 0;
    dims >> n;
    const char* names[] = {"mnId", "kfFlags", "prevKF", "nextKF", "timeStamp", "imuPosition", "local", "slotStart", "slotPoint", "slotOctave",
                           "pointBad", "obsStart", "obsKF", "obsOctave"};
    std::vector<std::vector<std::vector<char>>> a((size_t)n);
    std::vector<std::vector<uint8_t>> status((size_t)n);
    std::vector<std::vector<int32_t>> nMPs((size_t)n), nRed((size_t)n);
    std::vector<int32_t> visited((size_t)n, -7);
    std::vector<OrbmCullingMap> maps((size_t)n);
    for (int j = 0; j < n; ++j) {
        OrbmCullingMap& m = maps[j];
        unsigned long long cur, last;
        dims >> m.nKF >> m.nLocal >> m.nPoints >> m.inertial >> m.imuInitialized >> m.inertialBA2 >> m.abortBA >> m.keyFramesInMap >> cur >> last;
        if (!dims) { std::fprintf(stderr, "bad dims.txt\n"); return 2; }
        m.currentId = cur; m.lastId = last;
        for (const char* nm : names) a[j].push_back(slurp(j, nm));
        const std::vector<std::vector<char>>& r = a[j];
        auto ptr = [&](int k) { return r[k].empty() ? nullptr : r[k].data(); };
        m.mnId = (const uint64_t*)ptr(0); m.kfFlags = (const uint8_t*)ptr(1); m.prevKF = (const int32_t*)ptr(2); m.nextKF = (const int32_t*)ptr(3);
        m.timeStamp = (const double*)ptr(4); m.imuPosition = (const float*)ptr(5); m.local = (const int32_t*)ptr(6); m.slotStart = (const int32_t*)ptr(7);
        m.slotPoint = (const int32_t*)ptr(8); m.slotOctave = (const int32_t*)ptr(9); m.pointBad = (const uint8_t*)ptr(10); m.obsStart = (const int32_t*)ptr(11);
        m.obsKF = (const int32_t*)ptr(12); m.obsOctave = (const int32_t*)ptr(13);
        status[j].assign((size_t)m.nLocal, 0); nMPs[j].assign((size_t)m.nLocal, 0); nRed[j].assign((size_t)m.nLocal, 0);
        m.status = status[j].data(); m.nMPs = nMPs[j].data(); m.nRedundant = nRed[j].data(); m.visited = &visited[j];
    }
    ORB_SLAM3::ORBmatcher matcher;
    matcher.KeyFrameCullingBatch(maps);
    unsigned long long h = 14695981039346656037ull;
    int culled = 0;
    for (int j = 0; j < n; ++j) {
        fnv1a(h, status[j].data(), status[j].size());
        fnv1a(h, nMPs[j].data(), 4 * nMPs[j].size());
        fnv1a(h, nRed[j].data(), 4 * nRed[j].size());
        fnv1a(h, &visited[j], 4);
        for (uint8_t s : status[j]) culled += s >= ORBM_KFC_CULLED;
    }
    std::printf("digest %016llx\nculled %d\nlaunches %d\n", h, culled, orbm_last_launch_count(ORB_SLAM3::detail::matcher_handle(1, 1, 0)));
    return 0;
}
