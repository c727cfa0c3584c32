// TEST VEHICLE (never part of the product library): the phase functions of the LocalInertialBA kernel
// (orb_slam3_modified_b200/csrc/liba_core.cuh) instantiated with a SERIAL executor and compiled by g++, so that the kernel's logic --
// phases, task decompositions, the blocked LDL^T, the LM control flow -- is checked against the CPU oracle in the GPU-less container
// (tests/test_local_inertial_ba_cpu.py).  What it cannot see are races between the threads of a phase; those are covered by the
// -m gpu tests and compute-sanitizer racecheck on the GPU.
#include <math.h>

#include <vector>

#include "../orb_slam3_modified_b200/csrc/liba_pack.h"

namespace {
struct HostExec {
    std::vector<double> pnl = std::vector<double>((size_t)liba::MAXN * liba::LW, -1.0);
    double* panel() { return pnl.data(); }
    void tag(int) {}
    template <class F> void par(F f) { for (int t = 0; t < liba::NT; ++t) f(t); }
    // the device's reduction tree: shuffle-down inside each warp (lane 0 holds the warp's sum), then the warp sums in order
    template <class F> double sum(F f) {
        double v[liba::NT];
        for (int t = 0; t < liba::NT; ++t) v[t] = f(t);
        double total = 0;
        for (int w = 0; w < liba::NT / 32; ++w) {
            double* a = v + 32 * w;
            for (int off = 16; off >= 1; off >>= 1) for (int l = 0; l < off; ++l) a[l] += a[l + off];
            total += a[0];
        }
        return total;
    }
    template <class F> double max(F f) { double m = 0; for (int t = 0; t < liba::NT; ++t) m = fmax(m, f(t)); return m; }
};
}  // namespace

extern "C" int liba_emulate(const LocalInertialBAProblem* p, const LocalInertialBAResult* r, char* errText, int errCap) {
    std::string err = liba::check(*p);
    liba::Layout L{};
    std::vector<uint8_t> in, sc, out;
    if (err.empty()) {
        L = liba::make_layout(*p);
        in.assign(L.inBytes + 16, 0); sc.assign(L.scBytes + 16, 0xAB); out.assign(L.outBytes + 16, 0);   // scratch deliberately dirty
        err = liba::pack_inputs(*p, L, in.data());
    }
    if (!err.empty()) { if (errText && errCap > 0) { strncpy(errText, err.c_str(), errCap - 1); errText[errCap - 1] = 0; } return -1; }
    liba::Dev D;
    liba::bind(D, *p, L, in.data(), sc.data(), out.data());
    HostExec ex;
    liba::run(D, ex);
    return liba::unpack_outputs(*p, *r, L, out.data());
}

// Whether information_matrices takes its fast path (no Jacobi sweeps) for one IMU::Preintegrated record.
extern "C" int liba_information_fast_path(const float* P) {
    double A[81];
    return liba::information_fast_path(P, A) ? 1 : 0;
}

// The batch form of the host side (layout, threaded packing into ONE staging buffer, per-problem views) followed by the serial executor per map.
extern "C" int liba_emulate_batch(int count, const LocalInertialBAProblem* p, const LocalInertialBAResult* r, int* iterations, char* errText, int errCap) {
    std::vector<liba::Layout> lay(count);
    std::vector<size_t> inOff(count);
    size_t inTot = 0;
    std::string err;
    for (int i = 0; i < count && err.empty(); ++i) {
        err = liba::check(p[i]);
        if (!err.empty()) break;
        lay[i] = liba::make_layout(p[i]);
        inOff[i] = inTot;
        inTot += (lay[i].inBytes + 255) & ~(size_t)255;
    }
    std::vector<uint8_t> in(inTot + 256, 0);
    if (err.empty()) err = liba::pack_batch(count, p, lay.data(), inOff.data(), in.data());
    if (!err.empty()) { if (errText && errCap > 0) { strncpy(errText, err.c_str(), errCap - 1); errText[errCap - 1] = 0; } return -1; }
    for (int i = 0; i < count; ++i) {
        std::vector<uint8_t> sc(lay[i].scBytes + 32, 0xAB), out(lay[i].outBytes + 32, 0);
        liba::Dev D;
        liba::bind(D, p[i], lay[i], in.data() + inOff[i], sc.data(), out.data());
        HostExec ex;
        liba::run(D, ex);
        iterations[i] = liba::unpack_outputs(p[i], r[i], lay[i], out.data());
    }
    return 0;
}
