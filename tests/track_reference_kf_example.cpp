// A C++ caller of BatchTracker::TrackReferenceKeyFrame (include/orb_b200/orb_slam3.hpp), built with plain g++ by
// tests/test_track_reference_kf_gpu.py: reads a batch written by the test (dims.txt + one .raw file per slab), runs the call and writes
// every output as <name>.out for a byte-for-byte comparison with the Python binding.
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
static void dump(const std::string& name, const void* p, size_t bytes) {
    std::ofstream f(dir + "/" + name + ".out", std::ios::binary);
    f.write((const char*)p, (std::streamsize)bytes);
}

int main(int argc, char** argv) {
    if (argc < 2) { std::fprintf(stderr, "usage: %s DIR\n", argv[0]); return 2; }
    dir = argv[1];
    std::ifstream dims(dir + "/dims.txt");
    int B, K, M, nlevels;
    double cam[4];
    dims >> B >> K >> M >> nlevels >> cam[0] >> cam[1] >> cam[2] >> cam[3];
    if (!dims) { std::fprintf(stderr, "bad dims.txt\n"); return 2; }
    const char* names[] = {"kps", "desc", "nK", "fvNode", "fvFeature", "nEntries", "Tcw7", "kfN", "kfKps", "kfDesc", "kfFvNode", "kfFvFeature",
                           "kfNEntries", "kfPoint", "xyz", "hasObs", "invLevelSigma2", "active"};
    std::vector<std::vector<char>> a;
    for (const char* n : names) a.push_back(slurp(n));
    OrbmRefKeyFrameBatch in = {};
    in.batch = B; in.kcap = K; in.mcap = M; in.nlevels = nlevels;
    in.kps = (const OrbKeyPoint*)a[0].data(); in.desc = (const uint8_t*)a[1].data(); in.nK = (const int32_t*)a[2].data();
    in.fvNode = (const int32_t*)a[3].data(); in.fvFeature = (const int32_t*)a[4].data(); in.nEntries = (const int32_t*)a[5].data();
    in.Tcw7 = (const float*)a[6].data(); in.kfN = (const int32_t*)a[7].data(); in.kfKps = (const OrbKeyPoint*)a[8].data();
    in.kfDesc = (const uint8_t*)a[9].data(); in.kfFvNode = (const int32_t*)a[10].data(); in.kfFvFeature = (const int32_t*)a[11].data();
    in.kfNEntries = (const int32_t*)a[12].data(); in.kfPoint = (const uint8_t*)a[13].data(); in.xyz = (const float*)a[14].data();
    in.hasObs = (const uint8_t*)a[15].data(); in.invLevelSigma2 = (const float*)a[16].data(); in.active = (const uint8_t*)a[17].data();
    for (int i = 0; i < 4; ++i) in.cam[i] = (float)cam[i];

    const size_t b = B, k = K, m = M;
    std::vector<int32_t> nmatches(b), match(b * k, -1), nmatchesMap(b);
    std::vector<double> pose7(7 * b);
    std::vector<float> Tcw7(7 * b);
    std::vector<uint8_t> discarded(b * m);
    OrbmRefKeyFrameResult out = {nmatches.data(), match.data(), pose7.data(), Tcw7.data(), discarded.data(), nmatchesMap.data()};
    ORB_SLAM3::BatchTracker tracker(B, K, M);
    tracker.TrackReferenceKeyFrame(in, out);
    dump("nmatches", nmatches.data(), 4 * b); dump("match", match.data(), 4 * b * k); dump("pose7", pose7.data(), 56 * b);
    dump("Tcw7", Tcw7.data(), 28 * b); dump("discarded", discarded.data(), b * m); dump("nmatchesMap", nmatchesMap.data(), 4 * b);
    std::printf("launches %d\n", tracker.LastLaunchCount());
    return 0;
}
