// A C++ caller of BatchTracker::TrackLocalMapInertial (include/orb_b200/orb_slam3.hpp), built with plain g++ by
// tests/test_track_inertial_gpu.py: reads a batch written by the test (dims.txt + one .raw file per slab), runs two chained calls
// (the first call's state21 / prior21 / priorH are the second call's lastState21 / prior21 / priorH) and writes every output of
// both calls as <name><call>.out for a byte-for-byte comparison with the Python binding.
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
    int B, K, M, nlevels, bFar;
    double minX, minY, maxX, maxY, cam[4], mbf, logSF, nnratio, thFar, cosLimit, Tcb[7];
    dims >> B >> K >> M >> nlevels >> minX >> minY >> maxX >> maxY >> cam[0] >> cam[1] >> cam[2] >> cam[3] >> mbf >> logSF >> nnratio >> bFar >> thFar >> cosLimit;
    for (double& v : Tcb) dims >> v;
    if (!dims) { std::fprintf(stderr, "bad dims.txt\n"); return 2; }
    const char* names[] = {"kps", "desc", "nK", "scaleFactors", "invLevelSigma2", "nM", "worldPos", "normal", "minDistInv", "maxDistInv", "maxDistance",
                           "mpDesc", "hasObs", "bad", "th", "mode", "extrinsics24", "preintKF", "preintFrame", "kfState21", "lastState21", "prior21", "priorH"};
    std::vector<std::vector<char>> a;
    for (const char* n : names) a.push_back(slurp(n));
    OrbmLocalMapBatch in = {};
    in.batch = B; in.kcap = K; in.mcap = M; in.nlevels = nlevels;
    in.kps = (const OrbKeyPoint*)a[0].data(); in.desc = (const uint8_t*)a[1].data(); in.nK = (const int32_t*)a[2].data();
    in.minX = (float)minX; in.minY = (float)minY; in.maxX = (float)maxX; in.maxY = (float)maxY;
    in.scaleFactors = (const float*)a[3].data(); in.invLevelSigma2 = (const float*)a[4].data();
    for (int i = 0; i < 4; ++i) in.cam[i] = (float)cam[i];
    in.mbf = (float)mbf; in.logScaleFactor = (float)logSF;
    in.nM = (const int32_t*)a[5].data(); in.worldPos = (const float*)a[6].data(); in.normal = (const float*)a[7].data();
    in.minDistInv = (const float*)a[8].data(); in.maxDistInv = (const float*)a[9].data(); in.maxDistance = (const float*)a[10].data();
    in.mpDesc = (const uint8_t*)a[11].data(); in.hasObs = (const uint8_t*)a[12].data(); in.bad = (const uint8_t*)a[13].data();
    in.th = (const float*)a[14].data(); in.nnratio = (float)nnratio; in.bFarPoints = bFar; in.thFarPoints = (float)thFar; in.viewingCosLimit = (float)cosLimit;
    OrbmImuTrackBatch imu = {};
    imu.mode = (const uint8_t*)a[15].data();
    for (int i = 0; i < 7; ++i) imu.Tcb7[i] = (float)Tcb[i];
    imu.extrinsics24 = (const double*)a[16].data(); imu.preintKF = (const float*)a[17].data(); imu.preintFrame = (const float*)a[18].data();
    imu.kfState21 = (const float*)a[19].data(); imu.lastState21 = (const float*)a[20].data();
    imu.prior21 = (const double*)a[21].data(); imu.priorH = (const double*)a[22].data();

    const size_t b = B, k = K, m = M;
    std::vector<int32_t> match(b * k, -1), visible(b * m), found(b * m), counts(4 * b);
    std::vector<uint8_t> claimed(b * k), outlier(b * k);
    std::vector<float> Tcw7(7 * b), pred(21 * b), predT(7 * b), state(21 * b), lastState(21 * b);
    std::vector<double> prior(21 * b), priorH(225 * b), lastPrior(21 * b), lastPriorH(225 * b);
    OrbmLocalMapResult out = {match.data(), claimed.data(), outlier.data(), visible.data(), found.data(), counts.data(), counts.data() + b,
                              counts.data() + 2 * b, counts.data() + 3 * b, nullptr, Tcw7.data()};
    OrbmImuTrackResult io = {pred.data(), predT.data(), state.data(), prior.data(), priorH.data()};
    ORB_SLAM3::BatchTracker tracker(B, K, M);
    for (int call = 0; call < 2; ++call) {
        tracker.TrackLocalMapInertial(in, imu, out, io);
        const std::string c = std::to_string(call);
        dump("match" + c, match.data(), 4 * b * k); dump("claimed" + c, claimed.data(), b * k); dump("outlier" + c, outlier.data(), b * k);
        dump("visible" + c, visible.data(), 4 * b * m); dump("found" + c, found.data(), 4 * b * m); dump("counts" + c, counts.data(), 16 * b);
        dump("Tcw7" + c, Tcw7.data(), 28 * b); dump("predState21" + c, pred.data(), 84 * b); dump("predTcw7" + c, predT.data(), 28 * b);
        dump("state21" + c, state.data(), 84 * b); dump("prior21" + c, prior.data(), 168 * b); dump("priorH" + c, priorH.data(), 1800 * b);
        lastState = state; lastPrior = prior; lastPriorH = priorH;
        imu.lastState21 = lastState.data(); imu.prior21 = lastPrior.data(); imu.priorH = lastPriorH.data();
    }
    std::printf("launches %d\n", tracker.LastLaunchCount());
    return 0;
}
