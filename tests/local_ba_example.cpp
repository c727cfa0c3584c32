// A C++ caller of Optimizer::LocalBundleAdjustmentBatch (include/orb_b200/orb_slam3.hpp), built with plain g++ by
// tests/test_local_ba_gpu.py: reads the maps written by the test (dims.txt + one .raw file per map and array), runs them as one batch
// and prints a digest of every map's record (status, counts, the three lists, the observation flags, the float write-back and the LM
// statistics) for a comparison with the Python binding.
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

struct Out {
    int32_t status = -1, counts[4] = {0, 0, 0, 0}, nLists[3] = {0, 0, 0};
    std::vector<int32_t> localKF, fixedKF, localPoint, pointRefKF;
    std::vector<uint8_t> obsFlag, pointBad;
    std::vector<float> kfPose7, kfCenter, pointPos, normal, minDistance, maxDistance;
    double lmStats[5] = {0, 0, 0, 0, 0};
};

int main(int argc, char** argv) {
    if (argc < 2) { std::fprintf(stderr, "usage: %s DIR\n", argv[0]); return 2; }
    dir = argv[1];
    std::ifstream dims(dir + "/dims.txt");
    int n = 0, maxP = 0, maxL = 0, maxE = 0;
    dims >> n >> maxP >> maxL >> maxE;
    const char* names[] = {"mnId", "kfFlags", "pose7", "cameraCenter", "cam4", "cov", "slotStart", "slotPoint", "pointId", "pointFlags", "worldPos",
                           "refKF", "obsStart", "obsKF", "obsIdx", "obsPt", "obsOctave", "invLevelSigma2", "scaleFactors", "stop"};
    std::vector<std::vector<std::vector<char>>> a((size_t)n);
    std::vector<Out> out((size_t)n);
    std::vector<LbaLocalMap> maps((size_t)n);
    for (int j = 0; j < n; ++j) {
        LbaLocalMap& m = maps[j];
        Out& o = out[j];
        dims >> m.nKF >> m.nCov >> m.nPoints >> m.nlevels >> m.inertial;
        if (!dims) { std::fprintf(stderr, "bad dims.txt\n"); return 2; }
        for (const char* nm : names) a[j].push_back(slurp(j, nm));
        const std::vector<std::vector<char>>& r = a[j];
        auto ptr = [&](int k) { return r[k].empty() ? nullptr : r[k].data(); };
        m.mnId = (const uint64_t*)ptr(0); m.kfFlags = (const uint8_t*)ptr(1); m.pose7 = (const float*)ptr(2); m.cameraCenter = (const float*)ptr(3);
        m.cam4 = (const float*)ptr(4); m.cov = (const int32_t*)ptr(5); m.slotStart = (const int32_t*)ptr(6); m.slotPoint = (const int32_t*)ptr(7);
        m.pointId = (const uint64_t*)ptr(8); m.pointFlags = (const uint8_t*)ptr(9); m.worldPos = (const float*)ptr(10); m.refKF = (const int32_t*)ptr(11);
        m.obsStart = (const int32_t*)ptr(12); m.obsKF = (const int32_t*)ptr(13); m.obsIdx = (const int32_t*)ptr(14); m.obsPt = (const float*)ptr(15);
        m.obsOctave = (const int32_t*)ptr(16); m.invLevelSigma2 = (const float*)ptr(17); m.scaleFactors = (const float*)ptr(18);
        m.stopFlag = (const volatile uint8_t*)ptr(19);
        const size_t K = (size_t)m.nKF, P = (size_t)m.nPoints, O = P ? (size_t)m.obsStart[m.nPoints] : 0;
        o.localKF.assign(K, 0); o.fixedKF.assign(K, 0); o.localPoint.assign(P, 0); o.pointRefKF.assign(P, 0); o.obsFlag.assign(O, 0);
        o.pointBad.assign(P, 0); o.kfPose7.assign(7 * K, 0.f); o.kfCenter.assign(3 * K, 0.f); o.pointPos.assign(3 * P, 0.f); o.normal.assign(3 * P, 0.f);
        o.minDistance.assign(P, 0.f); o.maxDistance.assign(P, 0.f);
        m.status = &o.status; m.counts = o.counts; m.nLists = o.nLists; m.localKF = o.localKF.data(); m.fixedKF = o.fixedKF.data();
        m.localPoint = o.localPoint.data(); m.obsFlag = o.obsFlag.data(); m.kfPose7 = o.kfPose7.data(); m.kfCenter = o.kfCenter.data();
        m.pointPos = o.pointPos.data(); m.pointBad = o.pointBad.data(); m.pointRefKF = o.pointRefKF.data(); m.normal = o.normal.data();
        m.minDistance = o.minDistance.data(); m.maxDistance = o.maxDistance.data(); m.lmStats = o.lmStats;
        m.optPose = nullptr; m.optPoint = nullptr; m.edgeChi2 = nullptr; m.edgeDepthPositive = nullptr;
    }
    lba_handle* h = nullptr;
    ORB_SLAM3::orb_check(lba_create_batch(&h, maxP, maxL, maxE, n, 0), "lba_create_batch");
    ORB_SLAM3::Optimizer::LocalBundleAdjustmentBatch(h, n, maps.data());
    // the digest: per map the status and counts, then every list and per-list output cut to its length, the observation flags, the
    // LM statistics (tests/test_local_ba_gpu.py::_digest hashes the same bytes)
    unsigned long long d = 14695981039346656037ull;
    int erased = 0;
    for (int j = 0; j < n; ++j) {
        const Out& o = out[j];
        const size_t nl = (size_t)o.nLists[0], nf = (size_t)o.nLists[1], np = (size_t)o.nLists[2];
        fnv1a(d, &o.status, 4); fnv1a(d, o.counts, 16); fnv1a(d, o.nLists, 12);
        fnv1a(d, o.localKF.data(), 4 * nl); fnv1a(d, o.fixedKF.data(), 4 * nf); fnv1a(d, o.localPoint.data(), 4 * np);
        fnv1a(d, o.obsFlag.data(), o.obsFlag.size());
        fnv1a(d, o.kfPose7.data(), 28 * nl); fnv1a(d, o.kfCenter.data(), 12 * nl);
        fnv1a(d, o.pointPos.data(), 12 * np); fnv1a(d, o.pointBad.data(), np); fnv1a(d, o.pointRefKF.data(), 4 * np);
        fnv1a(d, o.normal.data(), 12 * np); fnv1a(d, o.minDistance.data(), 4 * np); fnv1a(d, o.maxDistance.data(), 4 * np);
        fnv1a(d, o.lmStats, 40);
        for (uint8_t f : o.obsFlag) erased += f == LBA_OBS_ERASED;
    }
    std::printf("digest %016llx\nerased %d\nlaunches %d\n", d, erased, lba_local_last_launches(h));
    lba_destroy(h);
    return 0;
}
