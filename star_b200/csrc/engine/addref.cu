// addref.cu — C-ABI of the device part of adding references at the mapping stage (include/star_b200.h: star_gpu_addref_*).
// Kernels: addref_kernels.cuh.  No CPU fallback: without a CUDA device star_gpu_addref_open fails.
#include <string>
#include <vector>

#include "addref_kernels.cuh"

namespace starb {
void setLastError(const std::string& m);     // engine_api.cu
void countLaunches(unsigned n);
}
using namespace starb;

struct star_addref {
    int device = 0;
    int nSM = 132;
    u8* dG = nullptr;       // 256 + nGenome + 256 bytes of the grown genome (freed before the merge, which does not read it)
    u64* dSA = nullptr;     // the old rows, re-based in place; (nSA+63)/64 * bits words
    SjdbIndex ix;
    u64 nG = 0, nG1 = 0, nG2 = 0;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
};

namespace {
template <class T> struct DevBuf {   // device allocation released on every exit path
    T* p = nullptr;
    ~DevBuf() { if (p) cudaFree(p); }
    cudaError_t alloc(size_t n) { return cudaMalloc(&p, (n ? n : 1) * sizeof(T)); }
    operator T*() const { return p; }
};
struct AddrefGuard {                 // closes a half-built handle unless released
    star_addref* h;
    ~AddrefGuard() { if (h) star_gpu_addref_close(h); }
};
unsigned gridFor(u64 want, int nSM) { return (unsigned)(want < (u64)nSM * 8 ? (want ? want : 1) : (u64)nSM * 8); }
}  // namespace

#define AR_CK(call)                                                                                                              \
    do {                                                                                                                         \
        cudaError_t e_ = (call);                                                                                                 \
        if (e_ != cudaSuccess) {                                                                                                 \
            setLastError(std::string("CUDA error: ") + cudaGetErrorString(e_) + " at " + __FILE__ + ":" + std::to_string(__LINE__)); \
            return STAR_EXIT_RUNTIME;                                                                                            \
        }                                                                                                                        \
    } while (0)

// device time between the handle's two events
static int elapsed(star_addref* h, float* ms) {
    AR_CK(cudaEventSynchronize(h->e1));
    float t = 0;
    AR_CK(cudaEventElapsedTime(&t, h->e0, h->e1));
    if (ms) *ms = t;
    return 0;
}

extern "C" {

int star_gpu_addref_open(star_addref_t** out, int device, const star_index_view_t* v, uint64_t nG, uint64_t nG1, uint64_t nG2, float* ms) {
    *out = nullptr;
    int nDev = 0;
    cudaError_t e = cudaGetDeviceCount(&nDev);
    if (e != cudaSuccess || nDev == 0) {
        setLastError(std::string("star_b200: no CUDA device available (") + cudaGetErrorString(e) + "); adding references has no CPU fallback");
        return STAR_EXIT_RUNTIME;
    }
    if (device < 0 || device >= nDev) { setLastError("star_b200: bad device ordinal"); return STAR_EXIT_RUNTIME; }
    if (nG + nG1 + nG2 != v->nGenome) { setLastError("star_b200: the grown genome is not nG + nG1 + nG2 bytes"); return STAR_EXIT_BUG; }
    AR_CK(cudaSetDevice(device));
    star_addref* h = new star_addref;
    AddrefGuard guard{h};
    h->device = device;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) h->nSM = prop.multiProcessorCount;
    const u32 bits = v->GstrandBit + 1;
    const u64 nSAnewMax = v->nSA + 2 * nG1;
    const size_t gBytes = 256 + v->nGenome + 256, saWords = (v->nSA + 63) / 64 * bits + 2;
    {   // G + old SA now, the new SA at the merge (G is released by then), and the search's text and insertion points
        size_t fr = 0, tot = 0;
        AR_CK(cudaMemGetInfo(&fr, &tot));
        const size_t need = saWords * 8 + std::max<size_t>(gBytes + (2 * nG1 + 272) + 32 * nG1, ((nSAnewMax + 63) / 64 * bits + 2) * 8 + 32 * nG1);
        if (need > fr) {
            setLastError("star_b200: adding references needs " + std::to_string(need >> 20) + " MiB of device memory, " + std::to_string(fr >> 20) + " MiB are free");
            return STAR_EXIT_MEMORY_ALLOCATION;
        }
    }
    if (cudaMalloc(&h->dG, gBytes) != cudaSuccess || cudaMalloc(&h->dSA, saWords * 8) != cudaSuccess) {
        setLastError("star_b200: out of device memory for adding references");
        return STAR_EXIT_MEMORY_ALLOCATION;
    }
    AR_CK(cudaEventCreate(&h->e0));
    AR_CK(cudaEventCreate(&h->e1));
    AR_CK(cudaMemcpy(h->dG, v->G - 256, gBytes, cudaMemcpyHostToDevice));
    AR_CK(cudaMemset(h->dSA, 0, saWords * 8));
    AR_CK(cudaMemcpy(h->dSA, v->SA, v->nSAbyte, cudaMemcpyHostToDevice));
    h->ix.G = h->dG + 256; h->ix.SA = h->dSA; h->ix.nGenome = v->nGenome; h->ix.nSA = v->nSA;
    h->ix.GstrandBit = v->GstrandBit; h->ix.saBits = bits;
    h->nG = nG; h->nG1 = nG1; h->nG2 = nG2;
    AddrefRebase a{v->nSA, nG, nG1, nG2, v->GstrandBit, bits};
    const u64 tiles = ((v->nSA + 63) / 64 + 31) / 32;
    const size_t smemBytes = (size_t)4 * 32 * bits * 8;
    AR_CK(cudaFuncSetAttribute(addref_rebase_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smemBytes));
    AR_CK(cudaEventRecord(h->e0));
    addref_rebase_kernel<<<gridFor((tiles + 3) / 4, h->nSM), 128, smemBytes>>>(a, h->dSA);
    countLaunches(1);
    AR_CK(cudaGetLastError());
    AR_CK(cudaEventRecord(h->e1));
    if (int rc = elapsed(h, ms)) return rc;
    guard.h = nullptr;
    *out = h;
    return 0;
}

int star_gpu_addref_search(star_addref_t* h, const uint8_t* seq, uint64_t* indArray, float* ms) {
    AR_CK(cudaSetDevice(h->device));
    if (!h->dG) { setLastError("star_b200: star_gpu_addref_search after the merge"); return STAR_EXIT_BUG; }
    const u64 nSuf = 2 * h->nG1;
    DevBuf<u8> dSeq;
    DevBuf<u64> dInd;
    AR_CK(dSeq.alloc(nSuf + 272));
    AR_CK(dInd.alloc(nSuf * 2 + 2));
    AR_CK(cudaMemset(dSeq, 5, nSuf + 272));
    AR_CK(cudaMemcpy(dSeq, seq, nSuf, cudaMemcpyHostToDevice));
    AR_CK(cudaEventRecord(h->e0));
    addref_search_kernel<<<gridFor((nSuf + 255) / 256, h->nSM), 256>>>(h->ix, dSeq, h->nG, h->nG1, dInd);
    countLaunches(1);
    AR_CK(cudaGetLastError());
    AR_CK(cudaEventRecord(h->e1));
    if (int rc = elapsed(h, ms)) return rc;
    AR_CK(cudaMemcpy(indArray, dInd, nSuf * 16, cudaMemcpyDeviceToHost));
    return 0;
}

int star_gpu_addref_merge_sa(star_addref_t* h, const uint64_t* indSorted, uint64_t nInd, uint8_t* SAnew, uint64_t nSAnewByte, float* ms) {
    AR_CK(cudaSetDevice(h->device));
    if (h->dG) { cudaFree(h->dG); h->dG = nullptr; h->ix.G = nullptr; }
    const u64 nSAnew = h->ix.nSA + nInd;
    std::vector<u64> row(nInd + 1), val(nInd + 1);
    sjdbInsertedRows(indSorted, nInd, h->ix.nSA, h->nG1, h->nG, h->ix.GstrandBit, row.data(), val.data(), h->nG2);
    DevBuf<u64> dRow, dVal, dOut;
    const u64 outWords = (nSAnew + 63) / 64 * h->ix.saBits + 2;
    if (nSAnewByte > outWords * 8) { setLastError("star_b200: bad size of the new suffix array"); return STAR_EXIT_BUG; }
    AR_CK(dRow.alloc(nInd + 1));
    AR_CK(dVal.alloc(nInd + 1));
    AR_CK(dOut.alloc(outWords));
    AR_CK(cudaMemcpy(dRow, row.data(), (nInd + 1) * 8, cudaMemcpyHostToDevice));
    AR_CK(cudaMemcpy(dVal, val.data(), (nInd + 1) * 8, cudaMemcpyHostToDevice));
    AddrefMerge m{dRow, dVal, nInd, nSAnew};
    const u64 tiles = ((nSAnew + 63) / 64 + 31) / 32;
    const size_t smemBytes = (size_t)4 * 32 * h->ix.saBits * 8;
    AR_CK(cudaFuncSetAttribute(sjdb_merge_sa_kernel<AddrefMerge>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smemBytes));
    AR_CK(cudaEventRecord(h->e0));
    sjdb_merge_sa_kernel<<<gridFor((tiles + 3) / 4, h->nSM), 128, smemBytes>>>(h->ix, m, dOut);
    countLaunches(1);
    AR_CK(cudaGetLastError());
    AR_CK(cudaEventRecord(h->e1));
    if (int rc = elapsed(h, ms)) return rc;
    AR_CK(cudaMemcpy(SAnew, dOut, nSAnewByte, cudaMemcpyDeviceToHost));
    return 0;
}

void star_gpu_addref_close(star_addref_t* h) {
    if (!h) return;
    cudaFree(h->dG);
    cudaFree(h->dSA);
    if (h->e0) cudaEventDestroy(h->e0);
    if (h->e1) cudaEventDestroy(h->e1);
    delete h;
}

}  // extern "C"
