// H100 kernels + C-ABI for the DBoW2 transform the reference runs per (key)frame (SURVEY.md 8f rank 3):
//   Frame::ComputeBoW / KeyFrame::ComputeBoW (reference src/Frame.cc:738-745) -> mpORBvocabulary->transform(vCurrentDesc, mBowVec, mFeatVec, 4)
//   TemplatedVocabulary::transform   Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h:1127-1197 (frame), :1218-1259 (one feature: tree descent)
//   BowVector::addWeight / addIfNotExist / normalize (BowVector.cpp:35-88), FeatureVector::addFeature (FeatureVector.cpp:30-45)
// The vocabulary tree (k = 10, L = 6, ~1.08 M nodes for ORBvoc: 35 MB of descriptors) lives in HBM once per handle; a call transforms the
// descriptors of `batch` frames:
//   bow_descend_kernel   half a warp per feature: at every level the lanes take the children of the current node, 256-bit Hamming distance,
//                        argmin with ties to the first child (the reference keeps the first minimum), L dependent steps;
//   bow_assemble_kernel  one CTA per frame: bitonic sort of (word id, feature index) and (node id, feature index) keys in shared memory,
//                        per-word weight sums in feature order (= the order std::map::operator+= sees them), L1 / L2 normalisation with the
//                        norm accumulated in ascending word order like BowVector::normalize -- results are bit-identical to DBoW2's doubles.
#include <cuda_runtime.h>
#include <math.h>
#include <string.h>
#include <string>
#include <vector>

#include "../../include/orb_b200.h"
#include "device_utils.cuh"
#include "staging.h"

using orbx::set_error;

namespace bow {

struct Voc {
    int L, weighting, norm, nNodes;
    const int *childStart, *children, *wordId;
    const uint8_t* desc;
    const double* weight;
};

constexpr int BD_NT = 256;
// half a warp per feature
__global__ void __launch_bounds__(BD_NT) bow_descend_kernel(Voc V, int batch, int cap, const uint8_t* __restrict__ feats, const int* __restrict__ nFeat, int levelsup,
                                                            int* __restrict__ fWord, double* __restrict__ fWeight, int* __restrict__ fNode) {
    const int g = (blockIdx.x * BD_NT + threadIdx.x) >> 4, sl = threadIdx.x & 15;
    const unsigned gmask = 0xFFFFu << (threadIdx.x & 16);
    const int f = g / cap, i = g - f * cap;
    if (f >= batch) return;
    const int N = min(nFeat[f], cap);
    if (i >= N) return;                                       // whole half-warp leaves together (same i)
    uint32_t fd[8];
    orbx::load_desc(feats + ((size_t)f * cap + i) * 32, fd);
    const int nid_level = V.L - levelsup;
    int final_id = 0, nid = 0, level = 0;
    for (;;) {
        ++level;
        const int a = V.childStart[final_id], b = V.childStart[final_id + 1];
        unsigned best = 0xFFFFFFFFu;                          // distance << 20 | child rank: the first minimum wins (:1241-1246)
        for (int c = a + sl; c < b; c += 16) {
            const int id = V.children[c];
            uint32_t dd[8];
            orbx::load_desc(V.desc + (size_t)id * 32, dd);
            best = min(best, ((unsigned)orbx::hamming256(fd, dd) << 20) | (unsigned)(c - a));
        }
#pragma unroll
        for (int o = 8; o; o >>= 1) best = min(best, __shfl_xor_sync(gmask, best, o));
        final_id = V.children[a + (int)(best & 0xFFFFFu)];
        if (level == nid_level) nid = final_id;
        if (V.childStart[final_id + 1] <= V.childStart[final_id]) break;      // isLeaf()
    }
    if (sl == 0) {
        const double w = V.weight[final_id];
        const size_t o = (size_t)f * cap + i;
        fWord[o] = w > 0 ? V.wordId[final_id] : -1;           // w == 0: a stopped word, the feature is dropped (:1157, :1182)
        fWeight[o] = w;
        fNode[o] = nid;
    }
}

constexpr int BA_NT = 512;
constexpr int MAX_CAP = 16384;   // bow_assemble_kernel sorts a frame in shared memory: 12 * 16384 B = 192 KiB
__device__ void bitonic_sort(unsigned long long* k, int n2) {   // n2: power of two, all threads of the CTA
    for (int size = 2; size <= n2; size <<= 1)
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int t = threadIdx.x; t < n2 / 2; t += BA_NT) {
                const int lo = 2 * t - (t & (stride - 1)), hi = lo + stride;
                const bool up = (lo & size) == 0;
                const unsigned long long a = k[lo], b = k[hi];
                if ((a > b) == up) { k[lo] = b; k[hi] = a; }
            }
            __syncthreads();
        }
}
__global__ void __launch_bounds__(BA_NT) bow_assemble_kernel(Voc V, int cap, int n2, const int* __restrict__ nFeat, const int* __restrict__ fWord, const double* __restrict__ fWeight,
                                                             const int* __restrict__ fNode, int* __restrict__ outWord, double* __restrict__ outValue, int* __restrict__ nWords,
                                                             int* __restrict__ fvNode, int* __restrict__ fvFeature, int* __restrict__ nEntries) {
    extern __shared__ unsigned long long s_keys[];          // n2 keys
    __shared__ int s_warp[33];
    __shared__ int s_cnt;
    int* s_flag = reinterpret_cast<int*>(s_keys + n2);      // n2 ints
    const int f = blockIdx.x, tid = threadIdx.x;
    const int N = min(nFeat[f], cap);
    const size_t base = (size_t)f * cap;
    // ---- FeatureVector: (node id, feature index) of the kept features, ascending ----
    for (int i = tid; i < n2; i += BA_NT) s_keys[i] = (i < N && fWord[base + i] >= 0) ? (((unsigned long long)(unsigned)fNode[base + i] << 32) | (unsigned)i) : ~0ull;
    __syncthreads();
    bitonic_sort(s_keys, n2);
    if (tid == 0) s_cnt = 0;
    __syncthreads();
    for (int i = tid; i < n2; i += BA_NT) {
        const unsigned long long key = s_keys[i];
        if (key != ~0ull) { fvNode[base + i] = (int)(key >> 32); fvFeature[base + i] = (int)(key & 0xFFFFFFFFu); atomicAdd(&s_cnt, 1); }
    }
    __syncthreads();
    const int kept = s_cnt;
    if (tid == 0) nEntries[f] = kept;
    __syncthreads();
    // ---- BowVector: (word id, feature index) ascending; a word's value = its weights added in feature order ----
    for (int i = tid; i < n2; i += BA_NT) s_keys[i] = (i < N && fWord[base + i] >= 0) ? (((unsigned long long)(unsigned)fWord[base + i] << 32) | (unsigned)i) : ~0ull;
    __syncthreads();
    bitonic_sort(s_keys, n2);
    for (int i = tid; i < n2; i += BA_NT) s_flag[i] = i < kept && (i == 0 || (s_keys[i] >> 32) != (s_keys[i - 1] >> 32));
    __syncthreads();
    const int nw = orbx::block_prefix<BA_NT>(n2, s_flag, s_warp, [&](int i) { return s_flag[i]; });   // s_flag[i] = output slot of the run starting at i (for heads)
    for (int i = tid; i < kept; i += BA_NT) {
        const unsigned word = (unsigned)(s_keys[i] >> 32);
        if (i == 0 || word != (unsigned)(s_keys[i - 1] >> 32)) {
            double v;
            if (V.weighting == 0 || V.weighting == 1) {                  // TF_IDF / TF: addWeight
                v = fWeight[base + (unsigned)(s_keys[i] & 0xFFFFFFFFu)];
                for (int j = i + 1; j < kept && (unsigned)(s_keys[j] >> 32) == word; ++j) v += fWeight[base + (unsigned)(s_keys[j] & 0xFFFFFFFFu)];
            } else v = fWeight[base + (unsigned)(s_keys[i] & 0xFFFFFFFFu)];   // IDF / BINARY: addIfNotExist keeps the first
            outWord[base + s_flag[i]] = (int)word;
            outValue[base + s_flag[i]] = v;
        }
    }
    __syncthreads();
    if (tid == 0) {   // ordered like BowVector::normalize / the !must division (:1164-1170): ascending word id
        nWords[f] = nw;
        double* val = outValue + base;
        if ((V.weighting == 0 || V.weighting == 1) && nw > 0 && V.norm == 0) { const double nd = (double)nw; for (int i = 0; i < nw; ++i) val[i] /= nd; }
        if (V.norm) {
            double nrm = 0.0;
            if (V.norm == 1) for (int i = 0; i < nw; ++i) nrm += fabs(val[i]);
            else { for (int i = 0; i < nw; ++i) nrm = fma(val[i], val[i], nrm); nrm = sqrt(nrm); }   // fused, like the reference build (see oracle)
            if (nrm > 0.0) for (int i = 0; i < nw; ++i) val[i] /= nrm;
        }
    }
}

struct Vocabulary {
    int device = 0;
    Voc V{};
    uint8_t* d_arena = nullptr;
    cudaStream_t st = nullptr;
    orbx::Staging staging;       // the host entry point's operands
    ~Vocabulary() { cudaSetDevice(device); if (d_arena) cudaFree(d_arena); if (st) cudaStreamDestroy(st); }
};

}  // namespace bow

using namespace bow;

struct orbv_handle { Vocabulary v; };

extern "C" {

int orbv_create(orbv_handle** out, const OrbVocabulary* voc, int device) {
    if (!out || !voc || voc->nNodes < 2 || voc->L < 1 || !voc->childStart || !voc->children || !voc->descriptors || !voc->weight || !voc->wordId ||
        voc->weighting < 0 || voc->weighting > 3 || voc->norm < 0 || voc->norm > 2) { set_error("orbv_create: bad argument"); return ORB_ERR_ARG; }
    const int n = voc->nNodes;
    if (voc->childStart[0] != 0 || voc->childStart[1] <= 0) { set_error("orbv_create: node 0 must be the root and have children"); return ORB_ERR_ARG; }
    const int nChildren = voc->childStart[n];
    for (int i = 0; i < n; ++i) if (voc->childStart[i + 1] < voc->childStart[i]) { set_error("orbv_create: childStart must be non-decreasing"); return ORB_ERR_ARG; }
    for (int i = 0; i < n; ++i)    // bow_descend_kernel packs a child's list position into 20 bits
        if (voc->childStart[i + 1] - voc->childStart[i] > (1 << 20)) { set_error("orbv_create: a node has more than 2^20 children"); return ORB_ERR_ARG; }
    for (int c = 0; c < nChildren; ++c) if (voc->children[c] <= 0 || voc->children[c] >= n) { set_error("orbv_create: child index out of range"); return ORB_ERR_ARG; }
    // The root is nobody's child (above) and every other node the child of at most one list entry, so the nodes reachable from the root
    // form a tree and the descent reaches a leaf within nNodes steps.  A table with a cycle fails this test.
    std::vector<uint8_t> listed(n, 0);
    for (int c = 0; c < nChildren; ++c)
        if (listed[voc->children[c]]++) { set_error("orbv_create: a node is listed as a child more than once"); return ORB_ERR_ARG; }
    for (int i = 1; i < n; ++i)    // the kernels would drop a negative word id's features where DBoW2 files them under (unsigned)id
        if (voc->childStart[i + 1] == voc->childStart[i] && voc->wordId[i] < 0) { set_error("orbv_create: a leaf has a negative wordId"); return ORB_ERR_ARG; }
    if (int rc = orbx::check_device(device)) return rc;
    CK(cudaSetDevice(device));
    orbv_handle* h = new orbv_handle();
    Vocabulary& v = h->v;
    v.device = v.staging.device = device;
    auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
    const size_t oCS = 0, oCh = oCS + al(4 * (size_t)(n + 1)), oW = oCh + al(4 * (size_t)nChildren), oD = oW + al(4 * (size_t)n), oWt = oD + al(32 * (size_t)n),
                 total = oWt + al(8 * (size_t)n);
    if (cudaMalloc(&v.d_arena, total) != cudaSuccess) { delete h; set_error("orbv_create: cudaMalloc failed"); return ORB_ERR_CUDA; }
    cudaError_t e = cudaMemcpy(v.d_arena + oCS, voc->childStart, 4 * (size_t)(n + 1), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(v.d_arena + oCh, voc->children, 4 * (size_t)nChildren, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(v.d_arena + oW, voc->wordId, 4 * (size_t)n, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(v.d_arena + oD, voc->descriptors, 32 * (size_t)n, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(v.d_arena + oWt, voc->weight, 8 * (size_t)n, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&v.st, cudaStreamNonBlocking);
    if (e != cudaSuccess) { set_error(cudaGetErrorString(e)); delete h; return ORB_ERR_CUDA; }
    v.V.L = voc->L; v.V.weighting = voc->weighting; v.V.norm = voc->norm; v.V.nNodes = n;
    v.V.childStart = (const int*)(v.d_arena + oCS); v.V.children = (const int*)(v.d_arena + oCh); v.V.wordId = (const int*)(v.d_arena + oW);
    v.V.desc = v.d_arena + oD; v.V.weight = (const double*)(v.d_arena + oWt);
    *out = h;
    return ORB_OK;
}
void orbv_destroy(orbv_handle* h) { delete h; }

int orbv_transform_batch_device(orbv_handle* h, int batch, const uint8_t* d_desc, const int* d_n, int cap, int levelsup, int* d_scratchWord, double* d_scratchWeight,
                                int* d_scratchNode, int* d_wordId, double* d_wordValue, int* d_nWords, int* d_fvNode, int* d_fvFeature, int* d_nEntries, void* stream) {
    if (!h || batch < 1 || cap < 1 || cap > MAX_CAP || !d_desc || !d_n || !d_scratchWord || !d_scratchWeight || !d_scratchNode || !d_wordId || !d_wordValue || !d_nWords ||
        !d_fvNode || !d_fvFeature || !d_nEntries || levelsup < 0) { set_error("orbv_transform_batch_device: bad argument (cap <= 16384)"); return ORB_ERR_ARG; }
    Vocabulary& v = h->v;
    CK(cudaSetDevice(v.device));
    cudaStream_t st = (cudaStream_t)stream;
    const long groups = (long)batch * cap;
    bow_descend_kernel<<<(unsigned)((groups * 16 + BD_NT - 1) / BD_NT), BD_NT, 0, st>>>(v.V, batch, cap, d_desc, d_n, levelsup, d_scratchWord, d_scratchWeight, d_scratchNode);
    int n2 = 1;
    while (n2 < cap) n2 <<= 1;
    const size_t sm = (size_t)n2 * 12;
    if (orbx::ensure_dynamic_smem(bow_assemble_kernel, sm, v.device)) return ORB_ERR_CUDA;
    bow_assemble_kernel<<<batch, BA_NT, sm, st>>>(v.V, cap, n2, d_n, d_scratchWord, d_scratchWeight, d_scratchNode, d_wordId, d_wordValue, d_nWords, d_fvNode, d_fvFeature, d_nEntries);
    CK(cudaGetLastError());
    return ORB_OK;
}

int orbv_transform_batch(orbv_handle* h, int batch, const uint8_t* desc, const int32_t* n, int cap, int levelsup, int32_t* wordId, double* wordValue, int32_t* nWords,
                         int32_t* fvNode, int32_t* fvFeature, int32_t* nEntries) {
    if (!h || batch < 1 || cap < 1 || cap > MAX_CAP || !desc || !n || !wordId || !wordValue || !nWords || !fvNode || !fvFeature || !nEntries || levelsup < 0) {
        set_error("orbv_transform_batch: bad argument (cap <= 16384)"); return ORB_ERR_ARG;
    }
    if (int rc = orbx::check_row_counts("orbv_transform_batch", n, batch, cap)) return rc;
    Vocabulary& v = h->v;
    CK(cudaSetDevice(v.device));
    const size_t B = batch, K = cap;
    orbx::Staging& S = v.staging;
    S.begin();
    const int pD = S.in(desc, 32 * B * K), pN = S.in(n, 4 * B), pSW = S.scratch(4 * B * K), pSWt = S.scratch(8 * B * K), pSN = S.scratch(4 * B * K),
              pW = S.out(wordId, 4 * B * K), pV = S.out(wordValue, 8 * B * K), pNW = S.out(nWords, 4 * B), pFN = S.out(fvNode, 4 * B * K),
              pFF = S.out(fvFeature, 4 * B * K), pNE = S.out(nEntries, 4 * B);
    int rc = S.reserve();
    if (rc) return rc;
    CK(S.upload(v.st));
    rc = orbv_transform_batch_device(h, batch, S.dev(pD), S.dev<int>(pN), cap, levelsup, S.dev<int>(pSW), S.dev<double>(pSWt), S.dev<int>(pSN), S.dev<int>(pW),
                                     S.dev<double>(pV), S.dev<int>(pNW), S.dev<int>(pFN), S.dev<int>(pFF), S.dev<int>(pNE), v.st);
    if (rc) return rc;
    CK(S.download(v.st));
    return ORB_OK;
}

}  // extern "C"
