// Bit-exact scalar building blocks shared by the CUDA kernels and by the host-side
// self-checks (tests compile this header with g++ as well, see tests/hostcheck.cpp).
//
// Everything here must produce the same bits on sm_90a and on an x86-64 host built
// with -ffp-contract=off, because the reference results depend on them:
//   * cvRound          -> round-half-even (OpenCV core/fast_math.hpp)
//   * fast_atan2_deg   -> cv::fastAtan2 (call site reference src/ORBextractor.cc:102)
//   * sincosf_glibc    -> glibc 2.39 sincosf, FMA ifunc variant (what
//                         `(float)cos(angle), (float)sin(angle)` at src/ORBextractor.cc:112
//                         compiles to on an FMA-capable host)
//   * libstdcxx_sort   -> libstdc++ std::sort (introsort + final insertion sort) so that
//                         ties in compareNodes (src/ORBextractor.cc:538-553) fall the same way
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define ORB_HD __host__ __device__ __forceinline__
#else
#define ORB_HD static inline
#include <math.h>
#endif

namespace orbx {

// ---- individually rounded float/double ops (no contraction on either side) ----
#if defined(__CUDA_ARCH__)
ORB_HD float fmul(float a, float b) { return __fmul_rn(a, b); }
ORB_HD float fadd(float a, float b) { return __fadd_rn(a, b); }
ORB_HD float fsub(float a, float b) { return __fsub_rn(a, b); }
ORB_HD float fdiv(float a, float b) { return __fdiv_rn(a, b); }
ORB_HD float ffma(float a, float b, float c) { return __fmaf_rn(a, b, c); }
ORB_HD double dmul(double a, double b) { return __dmul_rn(a, b); }
ORB_HD double dadd(double a, double b) { return __dadd_rn(a, b); }
ORB_HD double dsub(double a, double b) { return __dsub_rn(a, b); }
ORB_HD double dfma(double a, double b, double c) { return __fma_rn(a, b, c); }
ORB_HD int round_half_even(float v) { return __float2int_rn(v); }
ORB_HD float d2f(double v) { return __double2float_rn(v); }
#else
ORB_HD float fmul(float a, float b) { return a * b; }
ORB_HD float fadd(float a, float b) { return a + b; }
ORB_HD float fsub(float a, float b) { return a - b; }
ORB_HD float fdiv(float a, float b) { return a / b; }
ORB_HD float ffma(float a, float b, float c) { return fmaf(a, b, c); }
ORB_HD double dmul(double a, double b) { return a * b; }
ORB_HD double dadd(double a, double b) { return a + b; }
ORB_HD double dsub(double a, double b) { return a - b; }
ORB_HD double dfma(double a, double b, double c) { return fma(a, b, c); }
ORB_HD int round_half_even(float v) { return (int)nearbyintf(v); }
ORB_HD float d2f(double v) { return (float)v; }
#endif

// cv::fastAtan2(y, x) in degrees, [0, 360).  SURVEY.md section 9F.
ORB_HD float fast_atan2_deg(float y, float x) {
    const float scale = 57.295780181884765625f;  // (float)(180/pi)
    // p_i = (float)c_i * scale, each a float x float product (precomputed, exact constants below
    // are checked against the expression form in tests/hostcheck.cpp)
    const float p1 = fmul(0.9997878412794807f, scale), p3 = fmul(-0.3258083974640975f, scale);
    const float p5 = fmul(0.1555786518463281f, scale), p7 = fmul(-0.04432655554792128f, scale);
    const float eps = 2.220446049250313e-16f;  // (float)DBL_EPSILON
    float ax = x < 0 ? -x : x, ay = y < 0 ? -y : y, a, c, c2;
    if (ax >= ay) {
        c = fdiv(ay, fadd(ax, eps));
        c2 = fmul(c, c);
        a = fmul(fadd(fmul(fadd(fmul(fadd(fmul(p7, c2), p5), c2), p3), c2), p1), c);
    } else {
        c = fdiv(ax, fadd(ay, eps));
        c2 = fmul(c, c);
        a = fsub(90.f, fmul(fadd(fmul(fadd(fmul(fadd(fmul(p7, c2), p5), c2), p3), c2), p1), c));
    }
    if (x < 0) a = fsub(180.f, a);
    if (y < 0) a = fsub(360.f, a);
    return a;
}

// glibc 2.39 sincosf (sysdeps/ieee754/flt-32/s_sincosf.c, __sincosf_fma variant: every
// a + b*c of the C source is one fused multiply-add; constants read back from libm.so.6).
// Valid for |y| < 120 (the extractor only passes [0, 2*pi]).
ORB_HD void sincosf_glibc(float y, float* sinp, float* cosp) {
    const double hpi_inv = 0x1.45F306DC9C883p+23;  // 2/pi * 2^24
    const double hpi = 0x1.921FB54442D18p0;
    const double C0 = 0x1p0, C1 = -0x1.ffffffd0c621cp-2, C2 = 0x1.55553e1068f19p-5;
    const double C3 = -0x1.6c087e89a359dp-10, C4 = 0x1.99343027bf8c3p-16;
    const double S1 = -0x1.555545995a603p-3, S2 = 0x1.1107605230bc4p-7, S3 = -0x1.994eb3774cf24p-13;
    double x = (double)y;
    union { float f; uint32_t u; } cv;
    cv.f = y;
    const uint32_t top = (cv.u >> 20) & 0x7ff;
    int n = 0;
    double sgn = 1.0, csg = 1.0;  // csg: sign applied to the cosine polynomial (table[1] when n&2)
    if (top < 0x3f4) {            // |y| < pi/4   (abstop12(y) < abstop12(pio4f) = 0x3f4)
        if (top < 0x398) {        // |y| < 2^-12
            *sinp = y;
            *cosp = 1.0f;
            return;
        }
    } else {
        double r = dmul(x, hpi_inv);
        n = ((int32_t)r + 0x800000) >> 24;
        x = dfma(-(double)n, hpi, x);
        sgn = ((n & 3) == 1 || (n & 3) == 2) ? -1.0 : 1.0;
        if (n & 2) csg = -1.0;
    }
    const double x2 = dmul(x, x);  // note: x*x uses the unsigned reduced x
    const double xs = dmul(x, sgn);
    const double x4 = dmul(x2, x2);
    const double x3 = dmul(x2, xs);
    const double c2 = dfma(x2, dmul(csg, C4), dmul(csg, C3));
    const double s1 = dfma(x2, S3, S2);
    const double c1 = dfma(x2, dmul(csg, C1), dmul(csg, C0));
    const double x5 = dmul(x3, x2);
    const double x6 = dmul(x4, x2);
    const double s = dfma(x3, S1, xs);
    const double c = dfma(x4, dmul(csg, C2), c1);
    const float sv = d2f(dfma(x5, s1, s));
    const float cvv = d2f(dfma(x6, c2, c));
    if (n & 1) { *sinp = cvv; *cosp = sv; }
    else       { *sinp = sv;  *cosp = cvv; }
}

// glibc 2.39 logf (sysdeps/ieee754/flt-32/e_logf.c with logf_data.c, __logf_fma variant: every a*b + c of the C source is
// one fused multiply-add).  `MapPoint::PredictScale` calls it through std::log(float) (src/MapPoint.cc:531-546).
// Valid for positive normal finite x (the caller passes a distance ratio).
ORB_HD float logf_glibc(float x) {
    const double T[16][2] = {
        {0x1.661ec79f8f3bep+0, -0x1.57bf7808caadep-2}, {0x1.571ed4aaf883dp+0, -0x1.2bef0a7c06ddbp-2},
        {0x1.49539f0f010bp+0, -0x1.01eae7f513a67p-2},  {0x1.3c995b0b80385p+0, -0x1.b31d8a68224e9p-3},
        {0x1.30d190c8864a5p+0, -0x1.6574f0ac07758p-3}, {0x1.25e227b0b8eap+0, -0x1.1aa2bc79c81p-3},
        {0x1.1bb4a4a1a343fp+0, -0x1.a4e76ce8c0e5ep-4}, {0x1.12358f08ae5bap+0, -0x1.1973c5a611cccp-4},
        {0x1.0953f419900a7p+0, -0x1.252f438e10c1ep-5}, {0x1p+0, 0x0p+0},
        {0x1.e608cfd9a47acp-1, 0x1.aa5aa5df25984p-5},  {0x1.ca4b31f026aap-1, 0x1.c5e53aa362eb4p-4},
        {0x1.b2036576afce6p-1, 0x1.526e57720db08p-3},  {0x1.9c2d163a1aa2dp-1, 0x1.bc2860d22477p-3},
        {0x1.886e6037841edp-1, 0x1.1058bc8a07ee1p-2},  {0x1.767dcf5534862p-1, 0x1.4043057b6ee09p-2}};
    const double Ln2 = 0x1.62e42fefa39efp-1;
    const double A0 = -0x1.00ea348b88334p-2, A1 = 0x1.5575b0be00b6ap-2, A2 = -0x1.ffffef20a4123p-2;
    union { float f; uint32_t u; } cv;
    cv.f = x;
    const uint32_t ix = cv.u;
    if (ix == 0x3f800000u) return 0.0f;
    // x = 2^k z; z in [OFF, 2 OFF); the range is split into 16 subintervals, the ratio of the endpoints is close to 1 / invc
    const uint32_t tmp = ix - 0x3f330000u;
    const int i = (int)((tmp >> 19) & 15u);
    const int k = (int32_t)tmp >> 23;
    cv.u = ix - (tmp & 0xff800000u);
    const double z = (double)cv.f;
    const double invc = T[i][0], logc = T[i][1];
    const double r = dfma(z, invc, -1.0);
    const double y0 = dfma((double)k, Ln2, logc);
    const double r2 = dmul(r, r);
    double y = dfma(A1, r, A2);
    y = dfma(A0, r2, y);
    y = dfma(y, r2, y0 + r);
    return d2f(y);
}

// ---------------------------------------------------------------------------
// libstdc++ std::sort emulation (bits/stl_algo.h: __sort -> __introsort_loop +
// __final_insertion_sort, _S_threshold = 16, median-of-3 to first, unguarded
// partition, heapsort fallback).  Less(a, b) must be a strict weak order; T is
// a small POD.  Runs sequentially (one thread).
// ---------------------------------------------------------------------------
template <class T, class Less>
ORB_HD void sx_adjust_heap(T* first, int hole, int len, T value, Less less) {
    const int top = hole;
    int child = hole;
    while (child < (len - 1) / 2) {
        child = 2 * (child + 1);
        if (less(first[child], first[child - 1])) child--;
        first[hole] = first[child];
        hole = child;
    }
    if ((len & 1) == 0 && child == (len - 2) / 2) {
        child = 2 * (child + 1);
        first[hole] = first[child - 1];
        hole = child - 1;
    }
    int parent = (hole - 1) / 2;  // __push_heap
    while (hole > top && less(first[parent], value)) {
        first[hole] = first[parent];
        hole = parent;
        parent = (hole - 1) / 2;
    }
    first[hole] = value;
}

template <class T, class Less>
ORB_HD void sx_heapsort(T* first, int n, Less less) {  // __partial_sort(first, last, last)
    if (n >= 2) {                                       // __make_heap
        int parent = (n - 2) / 2;
        while (true) {
            T v = first[parent];
            sx_adjust_heap(first, parent, n, v, less);
            if (parent == 0) break;
            parent--;
        }
    }
    for (int last = n; last > 1;) {                     // __sort_heap
        --last;
        T v = first[last];
        first[last] = first[0];
        sx_adjust_heap(first, 0, last, v, less);
    }
}

template <class T, class Less>
ORB_HD void sx_unguarded_linear_insert(T* last, Less less) {
    T val = *last;
    T* next = last - 1;
    while (less(val, *next)) {
        *last = *next;
        last = next;
        --next;
    }
    *last = val;
}

template <class T, class Less>
ORB_HD void sx_insertion_sort(T* first, T* last, Less less) {
    if (first == last) return;
    for (T* i = first + 1; i != last; ++i) {
        if (less(*i, *first)) {
            T val = *i;
            for (T* p = i; p != first; --p) *p = *(p - 1);
            *first = val;
        } else {
            sx_unguarded_linear_insert(i, less);
        }
    }
}

// __move_median_to_first(first, first+1, mid, last-1) on [lo, hi)
template <class T, class Less>
ORB_HD void sx_median_to_first(T* a, int lo, int hi, Less less) {
    T* first = a + lo;
    T* A = first + 1;
    T* B = first + (hi - lo) / 2;
    T* C = a + hi - 1;
    T* med;
    if (less(*A, *B)) {
        if (less(*B, *C)) med = B;
        else if (less(*A, *C)) med = C;
        else med = A;
    } else if (less(*A, *C)) med = A;
    else if (less(*B, *C)) med = C;
    else med = B;
    { T t = *first; *first = *med; *med = t; }
}

// One __introsort_loop iteration on [lo, hi): sx_median_to_first + __unguarded_partition(first+1, last, pivot = *first); returns the cut.
template <class T, class Less>
ORB_HD int sx_partition_step(T* a, int lo, int hi, Less less) {
    sx_median_to_first(a, lo, hi, less);
    T* first = a + lo;
    const T pivot = *first;   // the loop below never writes *first: l > first, and r stops at first at the latest
    T* l = first + 1;
    T* r = a + hi;
    while (true) {
        while (less(*l, pivot)) ++l;
        --r;
        while (less(pivot, *r)) --r;
        if (!(l < r)) break;
        T t = *l; *l = *r; *r = t;
        ++l;
    }
    return (int)(l - a);
}

template <class T, class Less>
ORB_HD void libstdcxx_sort(T* a, int n, Less less) {
    if (n < 2) return;
    // explicit stack of [lo, hi) ranges with remaining depth (the recursion of
    // __introsort_loop always descends into the right part first and loops on the left)
    int stack_lo[64], stack_hi[64], stack_d[64];
    int sp = 0;
    int depth = 0;
    for (int t = n; t > 1; t >>= 1) depth++;
    depth *= 2;
    stack_lo[sp] = 0; stack_hi[sp] = n; stack_d[sp] = depth; sp++;
    while (sp > 0) {
        sp--;
        int lo = stack_lo[sp], hi = stack_hi[sp], d = stack_d[sp];
        while (hi - lo > 16) {
            if (d == 0) {
                sx_heapsort(a + lo, hi - lo, less);
                break;
            }
            --d;
            const int cut = sx_partition_step(a, lo, hi, less);
            // recurse on [cut, hi) first: emulate by pushing the LEFT part and continuing... no:
            // libstdc++ calls __introsort_loop(cut, last) recursively, then loops on [first, cut).
            // The two parts are disjoint, so the order in which they are finished does not matter;
            // we push the right part and continue with the left.
            stack_lo[sp] = cut; stack_hi[sp] = hi; stack_d[sp] = d; sp++;
            hi = cut;
        }
    }
    // __final_insertion_sort
    if (n > 16) {
        sx_insertion_sort(a, a + 16, less);
        for (T* i = a + 16; i != a + n; ++i) sx_unguarded_linear_insert(i, less);
    } else {
        sx_insertion_sort(a, a + n, less);
    }
}


// ---------------------------------------------------------------------------
// The same sort as a sequence of ROUNDS of independent tasks (what quadtree_kernel runs with one lane per task):
//   round r: every pending range longer than 16 does ONE partition step (or the heapsort fallback when its depth budget is spent) and
//            hands its two parts to the next round; parts of <= 16 elements become leaves;
//   finally every leaf is insertion-sorted on its own.
// Equal to libstdcxx_sort: the parts of a partition are disjoint, so the order in which they are processed is irrelevant; and the final
// insertion sort of std::sort never moves an element across a partition boundary (left part <= pivot <= right part, and it stops at the
// first element that is not greater), so it decomposes into independent insertion sorts of the leaves.  Checked against std::sort on the
// host (tests/hostcheck.cpp: hc_sort_check_rounds).  `task` holds (lo, hi, depth) triples: 2 x capacity ints x 3; `leaf` (lo, hi) pairs.
// ---------------------------------------------------------------------------
struct SxTask { int lo, hi, d; };
template <class T, class Less>
ORB_HD void sx_round_task(T* a, SxTask t, Less less, SxTask* next, int* nNext, SxTask* leaf, int* nLeaf) {
    // sequential helper used by the host model; the device driver inlines the same steps with atomic counters
    if (t.hi - t.lo <= 16) { leaf[(*nLeaf)++] = t; return; }
    if (t.d == 0) { sx_heapsort(a + t.lo, t.hi - t.lo, less); return; }          // sorted: not a leaf, nothing left to do
    const int cut = sx_partition_step(a, t.lo, t.hi, less);
    const SxTask right = {cut, t.hi, t.d - 1}, left = {t.lo, cut, t.d - 1};
    if (right.hi - right.lo > 16) next[(*nNext)++] = right; else leaf[(*nLeaf)++] = right;
    if (left.hi - left.lo > 16) next[(*nNext)++] = left; else leaf[(*nLeaf)++] = left;
}
template <class T, class Less>
inline void libstdcxx_sort_rounds_host(T* a, int n, Less less, SxTask* q0, SxTask* q1, SxTask* leaf) {
    if (n < 2) return;
    int depth = 0;
    for (int t = n; t > 1; t >>= 1) depth++;
    depth *= 2;
    int nCur = 1, nLeaf = 0;
    q0[0] = SxTask{0, n, depth};
    SxTask *cur = q0, *nxt = q1;
    while (nCur) {
        int nNext = 0;
        for (int i = 0; i < nCur; ++i) sx_round_task(a, cur[i], less, nxt, &nNext, leaf, &nLeaf);
        SxTask* t = cur; cur = nxt; nxt = t;
        nCur = nNext;
    }
    for (int i = 0; i < nLeaf; ++i) sx_insertion_sort(a + leaf[i].lo, a + leaf[i].hi, less);
}

}  // namespace orbx
