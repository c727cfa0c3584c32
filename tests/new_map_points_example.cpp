// A C++ caller of ORBmatcher::CreateNewMapPointsBatch (include/orb_b200/orb_slam3.hpp), built with plain g++ by
// tests/test_new_map_points_batch_gpu.py: reads the new keyframes of several maps written by the test (dims.txt + one .raw file per array),
// runs them as one batch and prints a digest of every item's (records, nmatches, ncreated) for a comparison with the Python binding.
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

struct Keyframe {
    std::vector<char> kps, desc, mp, fvn, fvf;
    OrbmTriFrame frame(int N, int E) const {
        OrbmTriFrame f;
        f.N = N; f.keypoints = (const OrbKeyPoint*)kps.data(); f.descriptors = (const uint8_t*)desc.data(); f.hasMapPoint = (const uint8_t*)mp.data();
        f.nEntries = E; f.fvNode = (const int32_t*)fvn.data(); f.fvFeature = (const int32_t*)fvf.data();
        return f;
    }
};
static Keyframe read_keyframe(const std::string& p) {
    return Keyframe{slurp(p + "_kps"), slurp(p + "_desc"), slurp(p + "_mp"), slurp(p + "_fvn"), slurp(p + "_fvf")};
}

int main(int argc, char** argv) {
    if (argc < 2) { std::fprintf(stderr, "usage: %s DIR\n", argv[0]); return 2; }
    dir = argv[1];
    std::ifstream dims(dir + "/dims.txt");
    int n = 0;
    dims >> n;
    struct Item {
        std::vector<Keyframe> kf;                                  // KF1 first
        std::vector<OrbmTriFrame> f1, f2;
        std::vector<std::vector<char>> a;                          // sf, sg, ep, F12, Tcw, Ow, cam
        std::vector<OrbmNewPoint> out;
        std::vector<int32_t> nm, nc;
        int nNew = 0;
    };
    std::vector<Item> st((size_t)n);
    std::vector<OrbmNewPointsItem> items((size_t)n);
    for (int j = 0; j < n; ++j) {
        Item& s = st[j];
        OrbmNewPointsIn& in = items[j].in;
        int N1, E1, K;
        dims >> N1 >> E1 >> K >> in.nlevels >> in.scaleFactor >> in.bCoarse >> in.bInertial >> in.thFarPoints;
        const std::string p = "item" + std::to_string(j);
        s.kf.push_back(read_keyframe(p + "_kf1"));
        s.f1.push_back(s.kf[0].frame(N1, E1));
        for (int k = 0; k < K; ++k) {
            int N2, E2;
            dims >> N2 >> E2;
            s.kf.push_back(read_keyframe(p + "_kf2_" + std::to_string(k)));
            s.f2.push_back(s.kf.back().frame(N2, E2));
        }
        if (!dims) { std::fprintf(stderr, "bad dims.txt\n"); return 2; }
        for (const char* nm : {"sf", "sg", "ep", "F12", "Tcw", "Ow", "cam"}) s.a.push_back(slurp(p + "_" + nm));
        in.KF1 = s.f1.data(); in.nKF2 = K; in.KF2 = s.f2.data();
        in.scaleFactors = (const float*)s.a[0].data(); in.levelSigma2 = (const float*)s.a[1].data();
        in.ep2 = (const float*)s.a[2].data(); in.F12 = (const float*)s.a[3].data();
        in.Tcw = (const float*)s.a[4].data(); in.Ow = (const float*)s.a[5].data(); in.cam = (const float*)s.a[6].data();
        s.out.resize(N1 > 0 ? N1 : 1); s.nm.assign((size_t)K, -1); s.nc.assign((size_t)K, -1);
        items[j].out = s.out.data(); items[j].nNew = &s.nNew; items[j].nmatches = s.nm.data(); items[j].ncreated = s.nc.data();
    }
    ORB_SLAM3::ORBmatcher matcher(0.6f, false);
    matcher.CreateNewMapPointsBatch(items);
    unsigned long long h = 14695981039346656037ull;
    int created = 0;
    for (const Item& s : st) {
        fnv1a(h, s.out.data(), sizeof(OrbmNewPoint) * (size_t)s.nNew);
        fnv1a(h, s.nm.data(), 4 * s.nm.size());
        fnv1a(h, s.nc.data(), 4 * s.nc.size());
        created += s.nNew;
    }
    std::printf("digest %016llx\ncreated %d\nlaunches %d\n", h, created, orbm_last_launch_count(ORB_SLAM3::detail::matcher_handle(1, 1, 0)));
    return 0;
}
