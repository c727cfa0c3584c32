// A C++ caller of ORBmatcher::UpdateLocalMapBatch (include/orb_b200/orb_slam3.hpp), built with plain g++ by tests/test_local_map_gpu.py:
// reads the batch written by the test (dims.txt + one .raw file per input array), runs it and prints a digest of every output for a
// comparison with the Python binding.
#include <cstdio>
#include <fstream>
#include <iterator>
#include <string>
#include <vector>

#include "orb_b200/orb_slam3.hpp"

static std::string dir;
static std::vector<char> slurp(const char* name) {
    std::ifstream f(dir + "/" + name + ".raw", std::ios::binary);
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
    OrbmUpdateLocalMapBatch in = {};
    dims >> in.batch >> in.kcap >> in.mcap >> in.mcapLast >> in.nKF >> in.nPoints;
    if (!dims) { std::fprintf(stderr, "bad dims.txt\n"); return 2; }
    const char* names[] = {"kfStart", "kfFlags", "covStart", "covKF", "childStart", "childKF", "parent", "prevKF", "slotStart", "slotPoint",
                           "pointStart", "pointBad", "obsStart", "obsKF", "worldPos", "normal", "minDistInv", "maxDistInv", "maxDistance",
                           "mpDesc", "hasObs", "nSrc", "srcPoint", "voteLastFrame", "match", "nK", "inertial", "lastKF"};
    std::vector<std::vector<char>> a;
    for (const char* nm : names) a.push_back(slurp(nm));
    const void** fields[] = {(const void**)&in.kfStart, (const void**)&in.kfFlags, (const void**)&in.covStart, (const void**)&in.covKF,
                             (const void**)&in.childStart, (const void**)&in.childKF, (const void**)&in.parent, (const void**)&in.prevKF,
                             (const void**)&in.slotStart, (const void**)&in.slotPoint, (const void**)&in.pointStart, (const void**)&in.pointBad,
                             (const void**)&in.obsStart, (const void**)&in.obsKF, (const void**)&in.worldPos, (const void**)&in.normal,
                             (const void**)&in.minDistInv, (const void**)&in.maxDistInv, (const void**)&in.maxDistance, (const void**)&in.mpDesc,
                             (const void**)&in.hasObs, (const void**)&in.nSrc, (const void**)&in.srcPoint, (const void**)&in.voteLastFrame,
                             (const void**)&in.match, (const void**)&in.nK, (const void**)&in.inertial, (const void**)&in.lastKF};
    for (size_t k = 0; k < a.size(); ++k) *fields[k] = a[k].empty() ? nullptr : a[k].data();
    const size_t B = in.batch, M = in.mcap, ML = in.mcapLast, NK = in.nKF;
    std::vector<int32_t> localKF(NK), nLocalKF(B), refKF(B), localPoint(B * M), nM(B), lastToLocal(B * ML);
    std::vector<float> worldPos(3 * B * M), normal(3 * B * M), minD(B * M), maxD(B * M), raw(B * M);
    std::vector<uint8_t> desc(32 * B * M), hasObs(B * M), bad(B * M);
    const OrbmUpdateLocalMapResult out = {localKF.data(), nLocalKF.data(), refKF.data(), localPoint.data(), nM.data(), worldPos.data(), normal.data(),
                                          minD.data(), maxD.data(), raw.data(), desc.data(), hasObs.data(), bad.data(), lastToLocal.data()};
    ORB_SLAM3::ORBmatcher matcher;
    matcher.UpdateLocalMapBatch(in, out);
    unsigned long long h = 14695981039346656037ull;
    fnv1a(h, localKF.data(), 4 * NK); fnv1a(h, nLocalKF.data(), 4 * B); fnv1a(h, refKF.data(), 4 * B); fnv1a(h, localPoint.data(), 4 * B * M);
    fnv1a(h, nM.data(), 4 * B); fnv1a(h, worldPos.data(), 12 * B * M); fnv1a(h, normal.data(), 12 * B * M); fnv1a(h, minD.data(), 4 * B * M);
    fnv1a(h, maxD.data(), 4 * B * M); fnv1a(h, raw.data(), 4 * B * M); fnv1a(h, desc.data(), 32 * B * M); fnv1a(h, hasObs.data(), B * M);
    fnv1a(h, bad.data(), B * M); fnv1a(h, lastToLocal.data(), 4 * B * ML);
    long points = 0;
    for (int32_t n : nM) points += n;
    std::printf("digest %016llx\npoints %ld\nlaunches %d\n", h, points, orbm_last_launch_count(ORB_SLAM3::detail::matcher_handle(1, 1, 0)));
    return 0;
}
