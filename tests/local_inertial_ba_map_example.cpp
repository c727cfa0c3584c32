// A C++ caller of Optimizer::LocalInertialBABatch (include/orb_b200/orb_slam3.hpp), built with plain g++ by
// tests/test_local_inertial_ba_map_gpu.py: reads the maps written by the test (dims.txt + one .raw file per map and array), runs them as
// one batch and prints a digest of every map's record (status, the lists, the observation flags and the float write-back) for a
// comparison with the Python binding.
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
    int32_t status = -1, nLists[4] = {0, 0, 0, 0};
    std::vector<int32_t> optKF, fixedKF, localPoint, pointRefKF;
    std::vector<uint8_t> ieLinked, obsFlag, pointBad;
    std::vector<float> kfPose7, kfCenter, kfVelocity, kfBias6, pointPos, normal, minDistance, maxDistance;
    double stats8[8] = {0, 0, 0, 0, 0, 0, 0, 0};
};

int main(int argc, char** argv) {
    if (argc < 2) { std::fprintf(stderr, "usage: %s DIR\n", argv[0]); return 2; }
    dir = argv[1];
    std::ifstream dims(dir + "/dims.txt");
    int n = 0;
    dims >> n;
    const char* names[] = {"kfFlags", "prevKF", "state21", "tcw12", "cameraCenter", "cam4", "preint", "extrinsics24", "slotStart", "slotPoint",
                           "pointFlags", "worldPos", "trackDepth", "refKF", "obsStart", "obsKF", "obsIdx", "obsPt", "obsOctave", "invLevelSigma2",
                           "scaleFactors"};
    std::vector<std::vector<std::vector<char>>> a((size_t)n);
    std::vector<Out> out((size_t)n);
    std::vector<LocalInertialBAMap> maps((size_t)n);
    for (int j = 0; j < n; ++j) {
        LocalInertialBAMap& m = maps[j];
        Out& o = out[j];
        dims >> m.nKF >> m.nPoints >> m.nlevels >> m.keyFramesInMap >> m.bLarge >> m.bRecInit;
        if (!dims) { std::fprintf(stderr, "bad dims.txt\n"); return 2; }
        for (const char* nm : names) a[j].push_back(slurp(j, nm));
        const std::vector<std::vector<char>>& r = a[j];
        auto ptr = [&](int k) { return r[k].empty() ? nullptr : r[k].data(); };
        m.kfFlags = (const uint8_t*)ptr(0); m.prevKF = (const int32_t*)ptr(1); m.state21 = (const float*)ptr(2); m.tcw12 = (const float*)ptr(3);
        m.cameraCenter = (const float*)ptr(4); m.cam4 = (const float*)ptr(5); m.preint = (const float*)ptr(6); m.extrinsics24 = (const double*)ptr(7);
        m.slotStart = (const int32_t*)ptr(8); m.slotPoint = (const int32_t*)ptr(9); m.pointFlags = (const uint8_t*)ptr(10); m.worldPos = (const float*)ptr(11);
        m.trackDepth = (const float*)ptr(12); m.refKF = (const int32_t*)ptr(13); m.obsStart = (const int32_t*)ptr(14); m.obsKF = (const int32_t*)ptr(15);
        m.obsIdx = (const int32_t*)ptr(16); m.obsPt = (const float*)ptr(17); m.obsOctave = (const int32_t*)ptr(18);
        m.invLevelSigma2 = (const float*)ptr(19); m.scaleFactors = (const float*)ptr(20);
        const size_t K = (size_t)m.nKF, P = (size_t)m.nPoints, O = P ? (size_t)m.obsStart[m.nPoints] : 0;
        o.optKF.assign(K, 0); o.fixedKF.assign(K, 0); o.localPoint.assign(P, 0); o.pointRefKF.assign(P, 0); o.ieLinked.assign(K, 0);
        o.obsFlag.assign(O, 0); o.pointBad.assign(P, 0); o.kfPose7.assign(7 * K, 0.f); o.kfCenter.assign(3 * K, 0.f); o.kfVelocity.assign(3 * K, 0.f);
        o.kfBias6.assign(6 * K, 0.f); o.pointPos.assign(3 * P, 0.f); o.normal.assign(3 * P, 0.f); o.minDistance.assign(P, 0.f); o.maxDistance.assign(P, 0.f);
        m.status = &o.status; m.nLists = o.nLists; m.optKF = o.optKF.data(); m.fixedKF = o.fixedKF.data(); m.localPoint = o.localPoint.data();
        m.ieLinked = o.ieLinked.data(); m.obsFlag = o.obsFlag.data(); m.kfPose7 = o.kfPose7.data(); m.kfCenter = o.kfCenter.data();
        m.kfVelocity = o.kfVelocity.data(); m.kfBias6 = o.kfBias6.data(); m.pointPos = o.pointPos.data(); m.pointBad = o.pointBad.data();
        m.pointRefKF = o.pointRefKF.data(); m.normal = o.normal.data(); m.minDistance = o.minDistance.data(); m.maxDistance = o.maxDistance.data();
        m.stats8 = o.stats8; m.optState21 = nullptr; m.optTcw12 = nullptr; m.optPoint = nullptr; m.edgeChi2 = nullptr;
    }
    ORB_SLAM3::Optimizer::LocalInertialBABatch(n, maps.data(), 0);
    // the digest: per map the status and the list lengths, then every list and per-list output cut to its length, and the observation
    // flags (tests/test_local_inertial_ba_map_gpu.py::_digest hashes the same bytes)
    unsigned long long d = 14695981039346656037ull;
    int erased = 0;
    for (int j = 0; j < n; ++j) {
        const Out& o = out[j];
        const size_t nw = (size_t)o.nLists[0], nf = (size_t)o.nLists[1], np = (size_t)o.nLists[2];
        fnv1a(d, &o.status, 4); fnv1a(d, o.nLists, 16);
        fnv1a(d, o.optKF.data(), 4 * nw); fnv1a(d, o.fixedKF.data(), 4 * nf); fnv1a(d, o.localPoint.data(), 4 * np); fnv1a(d, o.ieLinked.data(), nw);
        fnv1a(d, o.obsFlag.data(), o.obsFlag.size());
        fnv1a(d, o.kfPose7.data(), 28 * nw); fnv1a(d, o.kfCenter.data(), 12 * nw); fnv1a(d, o.kfVelocity.data(), 12 * nw); fnv1a(d, o.kfBias6.data(), 24 * nw);
        fnv1a(d, o.pointPos.data(), 12 * np); fnv1a(d, o.pointBad.data(), np); fnv1a(d, o.pointRefKF.data(), 4 * np);
        fnv1a(d, o.normal.data(), 12 * np); fnv1a(d, o.minDistance.data(), 4 * np); fnv1a(d, o.maxDistance.data(), 4 * np);
        for (uint8_t f : o.obsFlag) erased += f == LBA_OBS_ERASED;
    }
    std::printf("digest %016llx\nerased %d\nlaunches %d\n", d, erased, local_inertial_ba_map_last_launches());
    return 0;
}
