// sjdb.cu — C-ABI of the device part of the on-the-fly junction insertion (include/star_b200.h: star_gpu_sjdb_*).
// Kernels: sjdb_kernels.cuh.  No CPU fallback: without a CUDA device star_gpu_sjdb_open fails.
#include <string>
#include <vector>

#include "sjdb_kernels.cuh"

namespace starb {
void setLastError(const std::string& m);     // engine_api.cu
void countLaunches(unsigned n);
}
using namespace starb;

struct star_sjdb {
    int device = 0;
    int nSM = 132;
    u8* dG = nullptr;       // 256 + nGenome + 256 bytes
    u64* dSA = nullptr;
    SjdbIndex ix;
    u64 sjGstart = 0, sjdbNold = 0;
};

namespace {
template <class T> struct DevBuf {   // device allocation released on every exit path
    T* p = nullptr;
    ~DevBuf() { if (p) cudaFree(p); }
    cudaError_t alloc(size_t n) { return cudaMalloc(&p, (n ? n : 1) * sizeof(T)); }
    operator T*() const { return p; }
};
struct SjdbGuard {                   // closes a half-built handle unless released
    star_sjdb* h;
    ~SjdbGuard() { if (h) star_gpu_sjdb_close(h); }
};
}  // namespace

#define SJ_CK(call)                                                                                                              \
    do {                                                                                                                         \
        cudaError_t e_ = (call);                                                                                                 \
        if (e_ != cudaSuccess) {                                                                                                 \
            setLastError(std::string("CUDA error: ") + cudaGetErrorString(e_) + " at " + __FILE__ + ":" + std::to_string(__LINE__)); \
            return STAR_EXIT_RUNTIME;                                                                                            \
        }                                                                                                                        \
    } while (0)

extern "C" {

int star_gpu_sjdb_open(star_sjdb_t** out, int device, const star_index_view_t* v) {
    *out = nullptr;
    int nDev = 0;
    cudaError_t e = cudaGetDeviceCount(&nDev);
    if (e != cudaSuccess || nDev == 0) {
        setLastError(std::string("star_b200: no CUDA device available (") + cudaGetErrorString(e) + "); junction insertion has no CPU fallback");
        return STAR_EXIT_RUNTIME;
    }
    if (device < 0 || device >= nDev) { setLastError("star_b200: bad device ordinal"); return STAR_EXIT_RUNTIME; }
    SJ_CK(cudaSetDevice(device));
    star_sjdb* h = new star_sjdb;
    SjdbGuard guard{h};
    h->device = device;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) h->nSM = prop.multiProcessorCount;
    const size_t gBytes = 256 + v->nGenome + 256, saWords = (v->nSAbyte + 7) / 8 + 2;
    if (cudaMalloc(&h->dG, gBytes) != cudaSuccess || cudaMalloc(&h->dSA, saWords * 8) != cudaSuccess) {
        setLastError("star_b200: out of device memory for the junction insertion");
        return STAR_EXIT_MEMORY_ALLOCATION;
    }
    SJ_CK(cudaMemcpy(h->dG, v->G - 256, gBytes, cudaMemcpyHostToDevice));
    SJ_CK(cudaMemset(h->dSA, 0, saWords * 8));
    SJ_CK(cudaMemcpy(h->dSA, v->SA, v->nSAbyte, cudaMemcpyHostToDevice));
    h->ix.G = h->dG + 256; h->ix.SA = h->dSA; h->ix.nGenome = v->nGenome; h->ix.nSA = v->nSA;
    h->ix.GstrandBit = v->GstrandBit; h->ix.saBits = v->GstrandBit + 1;
    h->sjGstart = v->chrStart[v->nChrReal];
    h->sjdbNold = v->sjdbN;
    guard.h = nullptr;
    *out = h;
    return 0;
}

int star_gpu_sjdb_search(star_sjdb_t* h, const uint8_t* Gsj, uint64_t sjdbN, uint64_t sjdbLength, const uint8_t* skipSeq, uint64_t* indArray) {
    SJ_CK(cudaSetDevice(h->device));
    const u64 nSeq = 2 * sjdbN, nSuf = nSeq * sjdbLength;
    DevBuf<u8> dGsj, dSkip;
    DevBuf<u64> dInd;
    SJ_CK(dGsj.alloc(nSuf + 1 + 256));
    SJ_CK(dSkip.alloc(nSeq + 1));
    SJ_CK(dInd.alloc(nSuf * 2 + 2));
    SJ_CK(cudaMemset(dGsj, 5, nSuf + 1 + 256));
    SJ_CK(cudaMemcpy(dGsj, Gsj, nSuf + 1, cudaMemcpyHostToDevice));
    SJ_CK(cudaMemcpy(dSkip, skipSeq, nSeq, cudaMemcpyHostToDevice));
    const u64 want = (nSuf + 255) / 256;
    const unsigned grid = (unsigned)(want < (u64)h->nSM * 8 ? (want ? want : 1) : (u64)h->nSM * 8);   // a multiple of the SM count once the job is large
    sjdb_search_kernel<<<grid, 256>>>(h->ix, dGsj, nSeq, sjdbLength, dSkip, dInd);
    countLaunches(1);
    SJ_CK(cudaGetLastError());
    SJ_CK(cudaMemcpy(indArray, dInd, nSuf * 16, cudaMemcpyDeviceToHost));
    return 0;
}

int star_gpu_sjdb_merge_sa(star_sjdb_t* h, const uint64_t* indSorted, uint64_t nInd, uint64_t nGsj, uint64_t nGsjNew, uint64_t sjdbLength,
                           const uint32_t* oldSJind, uint8_t* SAnew, uint64_t nSAnewByte) {
    SJ_CK(cudaSetDevice(h->device));
    const u64 nSAnew = h->ix.nSA + nInd;
    std::vector<u64> row(nInd + 1), val(nInd + 1);
    sjdbInsertedRows(indSorted, nInd, h->ix.nSA, nGsj, h->sjGstart, h->ix.GstrandBit, row.data(), val.data());
    DevBuf<u64> dRow, dVal, dOut;
    DevBuf<u32> dOld;
    const u64 outWords = (nSAnew + 63) / 64 * h->ix.saBits + 2;
    SJ_CK(dRow.alloc(nInd + 1));
    SJ_CK(dVal.alloc(nInd + 1));
    SJ_CK(dOld.alloc(h->sjdbNold + 1));
    SJ_CK(dOut.alloc(outWords));
    SJ_CK(cudaMemcpy(dRow, row.data(), (nInd + 1) * 8, cudaMemcpyHostToDevice));
    SJ_CK(cudaMemcpy(dVal, val.data(), (nInd + 1) * 8, cudaMemcpyHostToDevice));
    if (h->sjdbNold) SJ_CK(cudaMemcpy(dOld, oldSJind, h->sjdbNold * 4, cudaMemcpyHostToDevice));
    SjdbMerge m;
    m.insRow = dRow; m.insVal = dVal; m.nInd = nInd; m.nSAnew = nSAnew;
    m.nGenomeOld = h->ix.nGenome; m.nGenomeNew = h->sjGstart + nGsj; m.sjGstart = h->sjGstart; m.sjdbLength = sjdbLength; m.sjdbNold = h->sjdbNold;
    m.nGsjNew = nGsjNew; m.oldSJind = dOld;
    const u64 tiles = ((nSAnew + 63) / 64 + 31) / 32, want = (tiles + 3) / 4;   // 4 warps per CTA, one tile of 32 x 64 rows per warp and step
    const unsigned grid = (unsigned)(want < (u64)h->nSM * 8 ? (want ? want : 1) : (u64)h->nSM * 8);
    const size_t smemBytes = (size_t)4 * 32 * h->ix.saBits * 8;
    SJ_CK(cudaFuncSetAttribute(sjdb_merge_sa_kernel<SjdbMerge>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smemBytes));
    sjdb_merge_sa_kernel<<<grid, 128, smemBytes>>>(h->ix, m, dOut);
    countLaunches(1);
    SJ_CK(cudaGetLastError());
    if (nSAnewByte > outWords * 8) { setLastError("star_b200: bad size of the new suffix array"); return STAR_EXIT_BUG; }
    SJ_CK(cudaMemcpy(SAnew, dOut, nSAnewByte, cudaMemcpyDeviceToHost));
    return 0;
}

void star_gpu_sjdb_close(star_sjdb_t* h) {
    if (!h) return;
    cudaFree(h->dG);
    cudaFree(h->dSA);
    delete h;
}

}  // extern "C"
