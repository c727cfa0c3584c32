// A C++ caller of ORBmatcher::FuseBatch (include/orb_b200/orb_slam3.hpp), built with plain g++ by tests/test_search_in_neighbors_gpu.py:
// reads one round of LocalMapping::SearchInNeighbors written by the test (dims.txt + one .raw file per item and array), runs it as one batch
// and prints a digest of every item's (bestIdx, bestDist) for a comparison with the Python binding.
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

int main(int argc, char** argv) {
    if (argc < 2) { std::fprintf(stderr, "usage: %s DIR\n", argv[0]); return 2; }
    dir = argv[1];
    std::ifstream dims(dir + "/dims.txt");
    int n = 0;
    dims >> n;
    const char* names[] = {"kps", "desc", "sf", "isg", "state", "xyz", "normal", "min_d", "max_d", "mp_desc"};
    std::vector<std::vector<std::vector<char>>> a((size_t)n);
    std::vector<std::vector<int32_t>> bi((size_t)n), bd((size_t)n);
    std::vector<OrbmFuseItem> items((size_t)n);
    for (int j = 0; j < n; ++j) {
        OrbmFuseItem& it = items[j];
        int K, M, nlevels;
        dims >> K >> M >> nlevels >> it.KF.minX >> it.KF.minY >> it.KF.maxX >> it.KF.maxY >> it.logScaleFactor >> it.th;
        for (float& v : it.Tcw7) dims >> v;
        for (float& v : it.Ow) dims >> v;
        for (float& v : it.cam) dims >> v;
        if (!dims) { std::fprintf(stderr, "bad dims.txt\n"); return 2; }
        for (const char* nm : names) a[j].push_back(slurp(j, nm));
        const std::vector<std::vector<char>>& r = a[j];
        it.KF.K = K; it.KF.keypoints = (const OrbKeyPoint*)r[0].data(); it.KF.descriptors = (const uint8_t*)r[1].data();
        it.KF.scaleFactors = (const float*)r[2].data(); it.KF.nlevels = nlevels; it.invLevelSigma2 = (const float*)r[3].data();
        it.pts.M = M; it.pts.state = (const uint8_t*)r[4].data(); it.pts.worldPos = (const float*)r[5].data(); it.pts.normal = (const float*)r[6].data();
        it.pts.minDistance = (const float*)r[7].data(); it.pts.maxDistance = (const float*)r[8].data(); it.pts.descriptors = (const uint8_t*)r[9].data();
        bi[j].assign((size_t)M, 0); bd[j].assign((size_t)M, 0);
        it.bestIdx = bi[j].data(); it.bestDist = bd[j].data();
    }
    ORB_SLAM3::ORBmatcher matcher;
    matcher.FuseBatch(items);
    unsigned long long h = 14695981039346656037ull;
    int fused = 0;
    for (int j = 0; j < n; ++j) {
        fnv1a(h, bi[j].data(), 4 * bi[j].size());
        fnv1a(h, bd[j].data(), 4 * bd[j].size());
        for (int32_t d : bd[j]) fused += d <= ORB_SLAM3::ORBmatcher::TH_LOW;
    }
    int maxK = 1;
    for (const OrbmFuseItem& it : items) if (it.KF.K > maxK) maxK = it.KF.K;
    std::printf("digest %016llx\nfused %d\nlaunches %d\n", h, fused, orbm_last_launch_count(ORB_SLAM3::detail::matcher_handle(maxK, 1, 0)));
    return 0;
}
