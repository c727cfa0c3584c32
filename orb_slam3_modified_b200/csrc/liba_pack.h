// Host-side flattening for local_inertial_ba_batch (and for the host emulation of its kernel, tests/liba_emulate.cpp): argument checks,
// the memory layout of one problem (inputs | scratch | outputs), the CSR lists point -> edges and free keyframe -> edges.  Plain C++.
#pragma once
#include <stdint.h>
#include <string.h>

#include <string>
#include <thread>
#include <vector>

#include "../../include/orb_b200.h"
#include "liba_core.cuh"

namespace liba {

struct Layout {
    // byte offsets inside the three regions of one problem
    size_t kfState, kfTcw, cam, extr, ieKf1, ieKf2, preint, ieRobust, ieInfoScale, pts, trackDepth, ePt, eKf, obs, invSigma2, ptStart, ptEdges, kfStart, kfEdges, inBytes;
    size_t pk, info9, infoG, infoA, errM, errI, errG, errA, ejac, W, Y, Hll, bl, Dinv, db, H, b, Hs, bs, dvec, x, He, be, part, partb, Jin, OJ, Oe, win, kfBk, tcwBk, ptsBk, scBytes;
    size_t outState, outTcw, outPts, erase, chi2, stats, prof, outBytes;
    int nFreeEdges;
};

inline size_t bump(size_t& off, size_t bytes) { const size_t at = off; off = (off + bytes + 31) & ~(size_t)31; return at; }   // 32-byte vector loads

// returns an error text ("" = ok)
inline std::string check(const LocalInertialBAProblem& p) {
    if (p.nKF < 1 || p.nOpt < 0 || p.nOpt > p.nKF || p.nInertial < 0 || p.nPoints < 0 || p.nEdges < 0 || p.iterations < 0) return "LocalInertialBA: negative or inconsistent sizes";
    if (p.nOpt < 1) return "LocalInertialBA: empty temporal window (the reference's window always holds the current keyframe)";
    if (p.nOpt > 64) return "LocalInertialBA: more than 64 keyframes in the temporal window";
    if (!p.kfState21 || !p.kfTcw12 || !p.cam4 || !p.extrinsics24) return "LocalInertialBA: null keyframe arrays";
    if (p.nInertial && (!p.ieKf1 || !p.ieKf2 || !p.preint || !p.ieRobust || !p.ieInfoScale)) return "LocalInertialBA: null inertial-edge arrays";
    if (p.nPoints && (!p.points3 || !p.trackDepth)) return "LocalInertialBA: null point arrays";
    if (p.nEdges && (!p.edgePoint || !p.edgeKf || !p.obs2 || !p.invSigma2)) return "LocalInertialBA: null edge arrays";
    for (int i = 0; i < p.nInertial; ++i)
        if (p.ieKf1[i] < 0 || p.ieKf1[i] >= p.nKF || p.ieKf2[i] < 0 || p.ieKf2[i] >= p.nKF || p.ieKf1[i] == p.ieKf2[i]) return "LocalInertialBA: inertial edge keyframe out of range";
    for (int e = 0; e < p.nEdges; ++e)
        if (p.edgePoint[e] < 0 || p.edgePoint[e] >= p.nPoints || p.edgeKf[e] < 0 || p.edgeKf[e] >= p.nKF) return "LocalInertialBA: edge index out of range";
    return "";
}

// The layout of a problem of at most nKF keyframes, nO of them in the window, nI inertial edges, nL points and nE mono edges of which nFree
// observe a window keyframe.  Every array of a problem within these bounds fits at the same offsets, so local_inertial_ba_map_batch lays
// out the problems its walk kernel builds on the device from bounds the host reads off the map.
inline Layout make_layout(size_t nKF, size_t nO, size_t nI, size_t nL, size_t nE, int nFree) {
    Layout L;
    const size_t n = 15 * nO;
    L.nFreeEdges = nFree;
    size_t o = 0;
    L.kfState = bump(o, nKF * 21 * 8); L.kfTcw = bump(o, nKF * 12 * 8); L.cam = bump(o, nKF * 4 * 4); L.extr = bump(o, 24 * 8);
    L.ieKf1 = bump(o, nI * 4); L.ieKf2 = bump(o, nI * 4); L.preint = bump(o, nI * IMU_PREINT_FLOATS * 4); L.ieRobust = bump(o, nI); L.ieInfoScale = bump(o, nI * 8);
    L.pts = bump(o, nL * 3 * 8); L.trackDepth = bump(o, nL * 4); L.ePt = bump(o, nE * 4); L.eKf = bump(o, nE * 4); L.obs = bump(o, nE * 2 * 8); L.invSigma2 = bump(o, nE * 4);
    L.ptStart = bump(o, (nL + 1) * 4); L.ptEdges = bump(o, nE * 4); L.kfStart = bump(o, (nO + 1) * 4); L.kfEdges = bump(o, (size_t)nFree * 4);
    L.inBytes = o;
    o = 0;
    L.pk = bump(o, nL * nO * 4); L.info9 = bump(o, nI * 81 * 8); L.infoG = bump(o, nI * 9 * 8); L.infoA = bump(o, nI * 9 * 8);
    L.errM = bump(o, nE * 2 * 8); L.errI = bump(o, nI * 9 * 8); L.errG = bump(o, nI * 3 * 8); L.errA = bump(o, nI * 3 * 8);
    L.ejac = bump(o, nE * EJ * 8); L.W = bump(o, nE * WS * 8); L.Y = bump(o, nE * WS * 8);
    L.Hll = bump(o, nL * 9 * 8); L.bl = bump(o, nL * 3 * 8); L.Dinv = bump(o, nL * 9 * 8); L.db = bump(o, nL * 3 * 8);
    L.H = bump(o, n * n * 8); L.b = bump(o, n * 8); L.Hs = bump(o, n * n * 8); L.bs = bump(o, n * 8); L.dvec = bump(o, n * 8); L.x = bump(o, (n + 3 * nL) * 8);
    L.He = bump(o, nI * 900 * 8); L.be = bump(o, nI * 30 * 8);
    L.part = bump(o, nO * (nO + 1) / 2 * SL * 36 * 8); L.partb = bump(o, nO * SL * 6 * 8);
    L.Jin = bump(o, nI * 216 * 8); L.OJ = bump(o, nI * 216 * 8); L.Oe = bump(o, nI * 9 * 8); L.win = bump(o, nI * 8);
    L.kfBk = bump(o, nO * 21 * 8); L.tcwBk = bump(o, nO * 12 * 8); L.ptsBk = bump(o, nL * 3 * 8);
    L.scBytes = o;
    o = 0;
    L.outState = bump(o, nKF * 21 * 8); L.outTcw = bump(o, nKF * 12 * 8); L.outPts = bump(o, nL * 3 * 8); L.erase = bump(o, nE); L.chi2 = bump(o, nE * 8); L.stats = bump(o, 8 * 8); L.prof = bump(o, 8 * 8);
    L.outBytes = o;
    return L;
}

inline Layout make_layout(const LocalInertialBAProblem& p) {
    int nFree = 0;
    for (int e = 0; e < p.nEdges; ++e) nFree += p.edgeKf[e] < p.nOpt;
    return make_layout(p.nKF, p.nOpt, p.nInertial, p.nPoints, p.nEdges, nFree);
}

// fills the input region (host memory); returns an error text when a (point, keyframe) pair is observed twice
inline std::string pack_inputs(const LocalInertialBAProblem& p, const Layout& L, uint8_t* in) {
    const size_t nKF = p.nKF, nI = p.nInertial, nL = p.nPoints, nE = p.nEdges;
    memcpy(in + L.kfState, p.kfState21, nKF * 21 * 8); memcpy(in + L.kfTcw, p.kfTcw12, nKF * 12 * 8); memcpy(in + L.cam, p.cam4, nKF * 16); memcpy(in + L.extr, p.extrinsics24, 24 * 8);
    if (nI) {
        memcpy(in + L.ieKf1, p.ieKf1, nI * 4); memcpy(in + L.ieKf2, p.ieKf2, nI * 4); memcpy(in + L.preint, p.preint, nI * IMU_PREINT_FLOATS * 4);
        memcpy(in + L.ieRobust, p.ieRobust, nI); memcpy(in + L.ieInfoScale, p.ieInfoScale, nI * 8);
    }
    if (nL) { memcpy(in + L.pts, p.points3, nL * 24); memcpy(in + L.trackDepth, p.trackDepth, nL * 4); }
    if (nE) { memcpy(in + L.ePt, p.edgePoint, nE * 4); memcpy(in + L.eKf, p.edgeKf, nE * 4); memcpy(in + L.obs, p.obs2, nE * 16); memcpy(in + L.invSigma2, p.invSigma2, nE * 4); }
    int* ptStart = (int*)(in + L.ptStart); int* ptEdges = (int*)(in + L.ptEdges); int* kfStart = (int*)(in + L.kfStart); int* kfEdges = (int*)(in + L.kfEdges);
    for (size_t i = 0; i <= nL; ++i) ptStart[i] = 0;
    for (int i = 0; i <= p.nOpt; ++i) kfStart[i] = 0;
    for (size_t e = 0; e < nE; ++e) { ++ptStart[p.edgePoint[e] + 1]; if (p.edgeKf[e] < p.nOpt) ++kfStart[p.edgeKf[e] + 1]; }
    for (size_t i = 0; i < nL; ++i) ptStart[i + 1] += ptStart[i];
    for (int i = 0; i < p.nOpt; ++i) kfStart[i + 1] += kfStart[i];
    std::vector<int> pc(ptStart, ptStart + nL), kc(kfStart, kfStart + p.nOpt);
    for (size_t e = 0; e < nE; ++e) { ptEdges[pc[p.edgePoint[e]]++] = (int)e; if (p.edgeKf[e] < p.nOpt) kfEdges[kc[p.edgeKf[e]]++] = (int)e; }
    // one EdgeMono per (point, keyframe): the Schur phase addresses an observation by that pair
    std::vector<int> seen((size_t)p.nKF, -1);
    for (size_t q = 0; q < nL; ++q)
        for (int j = ptStart[q]; j < ptStart[q + 1]; ++j) {
            const int k = p.edgeKf[ptEdges[j]];
            if (seen[k] == (int)q) return "LocalInertialBA: two observations of one point in one keyframe (right-camera edges are not supported)";
            seen[k] = (int)q;
        }
    return "";
}

// pack_inputs for a batch on up to 8 host threads (the copies into the pinned staging buffer dominate the host side of a many-map call);
// returns the first error text ("" = ok)
inline std::string pack_batch(int count, const LocalInertialBAProblem* problems, const Layout* lay, const size_t* inOff, uint8_t* hIn) {
    size_t bytes = 0;
    for (int i = 0; i < count; ++i) bytes += lay[i].inBytes;
    int nth = (int)std::thread::hardware_concurrency();
    if (nth > 8) nth = 8;
    if (nth > count) nth = count;
    if (nth < 2 || bytes < ((size_t)4 << 20)) {
        for (int i = 0; i < count; ++i) { const std::string e = pack_inputs(problems[i], lay[i], hIn + inOff[i]); if (!e.empty()) return e; }
        return "";
    }
    std::vector<std::string> err((size_t)nth);
    std::vector<std::thread> th;
    for (int t = 0; t < nth; ++t)
        th.emplace_back([&, t]() {
            for (int i = t; i < count; i += nth) { const std::string e = pack_inputs(problems[i], lay[i], hIn + inOff[i]); if (!e.empty() && err[t].empty()) err[t] = e; }
        });
    for (auto& x : th) x.join();
    for (const auto& e : err) if (!e.empty()) return e;
    return "";
}

inline void bind(Dev& D, const LocalInertialBAProblem& p, const Layout& L, uint8_t* in, uint8_t* sc, uint8_t* out) {
    D.nKF = p.nKF; D.nOpt = p.nOpt; D.nI = p.nInertial; D.nL = p.nPoints; D.nE = p.nEdges; D.iterations = p.iterations; D.bLarge = p.bLarge; D.lambdaInit = p.lambdaInit;
    D.kfState = (double*)(in + L.kfState); D.kfTcw = (double*)(in + L.kfTcw); D.cam = (const float*)(in + L.cam); D.extr = (const double*)(in + L.extr);
    D.ieKf1 = (const int*)(in + L.ieKf1); D.ieKf2 = (const int*)(in + L.ieKf2); D.preint = (const float*)(in + L.preint); D.ieRobust = in + L.ieRobust;
    D.ieInfoScale = (const double*)(in + L.ieInfoScale); D.pts = (double*)(in + L.pts); D.trackDepth = (const float*)(in + L.trackDepth);
    D.ePt = (const int*)(in + L.ePt); D.eKf = (const int*)(in + L.eKf); D.obs = (const double*)(in + L.obs); D.invSigma2 = (const float*)(in + L.invSigma2);
    D.ptStart = (const int*)(in + L.ptStart); D.ptEdges = (const int*)(in + L.ptEdges); D.kfStart = (const int*)(in + L.kfStart); D.kfEdges = (const int*)(in + L.kfEdges);
    D.pk = (int*)(sc + L.pk); D.info9 = (double*)(sc + L.info9); D.infoG = (double*)(sc + L.infoG); D.infoA = (double*)(sc + L.infoA);
    D.errM = (double*)(sc + L.errM); D.errI = (double*)(sc + L.errI); D.errG = (double*)(sc + L.errG); D.errA = (double*)(sc + L.errA);
    D.ejac = (double*)(sc + L.ejac); D.W = (double*)(sc + L.W); D.Y = (double*)(sc + L.Y);
    D.Hll = (double*)(sc + L.Hll); D.bl = (double*)(sc + L.bl); D.Dinv = (double*)(sc + L.Dinv); D.db = (double*)(sc + L.db);
    D.H = (double*)(sc + L.H); D.b = (double*)(sc + L.b); D.Hs = (double*)(sc + L.Hs); D.bs = (double*)(sc + L.bs); D.dvec = (double*)(sc + L.dvec); D.x = (double*)(sc + L.x);
    D.He = (double*)(sc + L.He); D.be = (double*)(sc + L.be); D.part = (double*)(sc + L.part); D.partb = (double*)(sc + L.partb);
    D.Jin = (double*)(sc + L.Jin); D.OJ = (double*)(sc + L.OJ); D.Oe = (double*)(sc + L.Oe); D.win = (double*)(sc + L.win);
    D.kfBk = (double*)(sc + L.kfBk); D.tcwBk = (double*)(sc + L.tcwBk); D.ptsBk = (double*)(sc + L.ptsBk);
    D.outState = (double*)(out + L.outState); D.outTcw = (double*)(out + L.outTcw); D.outPts = (double*)(out + L.outPts); D.erase = out + L.erase;
    D.chi2 = (double*)(out + L.chi2); D.stats = (double*)(out + L.stats); D.prof = (double*)(out + L.prof);
}

// copies one problem's output region to the caller's arrays; on FAIL the inputs are handed back (the reference returns before its write-back)
inline int unpack_outputs(const LocalInertialBAProblem& p, const LocalInertialBAResult& r, const Layout& L, const uint8_t* out) {
    const double* stats = (const double*)(out + L.stats);
    const bool failed = stats[2] != 0.0;
    if (r.kfState21) memcpy(r.kfState21, failed ? (const void*)p.kfState21 : (const void*)(out + L.outState), (size_t)p.nKF * 21 * 8);
    if (r.kfTcw12) memcpy(r.kfTcw12, failed ? (const void*)p.kfTcw12 : (const void*)(out + L.outTcw), (size_t)p.nKF * 12 * 8);
    if (r.points3 && p.nPoints) memcpy(r.points3, failed ? (const void*)p.points3 : (const void*)(out + L.outPts), (size_t)p.nPoints * 24);
    if (r.erase && p.nEdges) { if (failed) memset(r.erase, 0, p.nEdges); else memcpy(r.erase, out + L.erase, p.nEdges); }
    if (r.edgeChi2 && p.nEdges) memcpy(r.edgeChi2, out + L.chi2, (size_t)p.nEdges * 8);
    if (r.stats8) memcpy(r.stats8, stats, 64);
    if (r.profile8) memcpy(r.profile8, out + L.prof, 64);
    return (int)stats[5];
}

}  // namespace liba
