// dedup.cu — C-ABI of the duplicate marking (include/star_b200.h: star_gpu_dedup_*).  Kernels and the batch loop: dedup_kernels.cuh;
// the sort / scan / compaction primitives are cub's.  No CPU fallback: without a CUDA device star_gpu_dedup_open fails.
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <string>

#include "dev.cuh"

namespace starb {
void setLastError(const std::string& m);     // engine_api.cu
void countLaunches(unsigned n);
static int g_ddSM = 132;
static cudaError_t g_ddErr = cudaSuccess;
static inline void ddNote(cudaError_t e) { if (e != cudaSuccess && g_ddErr == cudaSuccess) g_ddErr = e; }
static inline void* ddAlloc(size_t bytes) { void* p = nullptr; if (cudaMalloc(&p, bytes ? bytes : 1) != cudaSuccess) { cudaGetLastError(); return nullptr; } return p; }
static inline unsigned ddGrid(unsigned long long count) {
    const unsigned long long want = (count + 255) / 256, cap = (unsigned long long)g_ddSM * 8;
    return (unsigned)(want < cap ? (want ? want : 1) : cap);
}
static void* g_ddTmp = nullptr;   // cub's temporary storage, kept between calls
static size_t g_ddTmpBytes = 0;
static void* ddTmp(size_t bytes) {
    if (bytes > g_ddTmpBytes) { cudaFree(g_ddTmp); g_ddTmp = ddAlloc(bytes); g_ddTmpBytes = g_ddTmp ? bytes : 0; if (!g_ddTmp) ddNote(cudaErrorMemoryAllocation); }
    return g_ddTmp;
}
static void ddSortPairs(const u64* kIn, u64* kOut, const u32* vIn, u32* vOut, u64 n, int endBit) {   // LSD radix sort: stable
    size_t tb = 0;
    ddNote(cub::DeviceRadixSort::SortPairs(nullptr, tb, kIn, kOut, vIn, vOut, (long long)n, 0, endBit));
    if (void* t = ddTmp(tb)) ddNote(cub::DeviceRadixSort::SortPairs(t, tb, kIn, kOut, vIn, vOut, (long long)n, 0, endBit));
    countLaunches((endBit + 7) / 8 + 1);
}
static void ddMaxScan(u32* a, u64 n) {
    size_t tb = 0;
    ddNote(cub::DeviceScan::InclusiveScan(nullptr, tb, a, a, cub::Max(), (long long)n));
    if (void* t = ddTmp(tb)) ddNote(cub::DeviceScan::InclusiveScan(t, tb, a, a, cub::Max(), (long long)n));
    countLaunches(2);
}
static void ddSelectIndex(const u8* flags, u32* out, u64 n, u64* nSel) {   // indices i < n with flags[i], in order
    *nSel = 0;
    unsigned long long* dN = (unsigned long long*)ddAlloc(8);
    if (!dN) { ddNote(cudaErrorMemoryAllocation); return; }
    thrust::counting_iterator<u32> it(0);
    size_t tb = 0;
    ddNote(cub::DeviceSelect::Flagged(nullptr, tb, it, flags, out, dN, (long long)n));
    if (void* t = ddTmp(tb)) ddNote(cub::DeviceSelect::Flagged(t, tb, it, flags, out, dN, (long long)n));
    unsigned long long h = 0;
    ddNote(cudaMemcpy(&h, dN, 8, cudaMemcpyDeviceToHost));
    *nSel = h;
    countLaunches(2);
    cudaFree(dN);
}
}  // namespace starb

#define DD_ALLOC(bytes) starb::ddAlloc(bytes)
#define DD_FREE(p) cudaFree(p)
#define DD_ZERO(p, bytes) starb::ddNote(cudaMemset(p, 0, bytes))
#define DD_COPY_TO(dst, src, bytes) starb::ddNote(cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice))
#define DD_COPY_FROM(dst, src, bytes) starb::ddNote(cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost))
#define DD_LAUNCH(count, kernel, ...) do { kernel<<<starb::ddGrid(count), 256>>>(__VA_ARGS__); starb::ddNote(cudaGetLastError()); starb::countLaunches(1); } while (0)
#define DD_SORT_PAIRS_U64(kIn, kOut, vIn, vOut, n, endBit) starb::ddSortPairs(kIn, kOut, vIn, vOut, n, endBit)
#define DD_MAXSCAN_U32(a, n) starb::ddMaxScan(a, n)
#define DD_SELECT_INDEX(flags, out, n, nSel) starb::ddSelectIndex(flags, out, n, nSel)
#define DD_ATOMIC_MIN_U64(p, v) atomicMin((unsigned long long*)(p), (unsigned long long)(v))
#define DD_ATOMIC_MAX_U64(p, v) atomicMax((unsigned long long*)(p), (unsigned long long)(v))
#define DD_SYNC() starb::ddNote(cudaDeviceSynchronize())
#include "dedup_kernels.cuh"

using namespace starb;

struct star_dedup {
    int device = 0;
    u32 mate2N = 0, hashBits = 64;
    u64 maxM = 0;
    DdBufs bufs;
    cudaEvent_t ev[2];
};

extern "C" {

int star_gpu_dedup_open(star_dedup_t** out, int device, uint64_t mate2basesN) {
    *out = nullptr;
    int nDev = 0;
    cudaError_t e = cudaGetDeviceCount(&nDev);
    if (e != cudaSuccess || nDev == 0) {
        setLastError(std::string("star_b200: no CUDA device available (") + cudaGetErrorString(e) + "); duplicate removal has no CPU fallback");
        return STAR_EXIT_RUNTIME;
    }
    if (device < 0 || device >= nDev) { setLastError("star_b200: bad device ordinal"); return STAR_EXIT_RUNTIME; }
    if (cudaSetDevice(device) != cudaSuccess) { setLastError("star_b200: cudaSetDevice failed"); return STAR_EXIT_RUNTIME; }
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) g_ddSM = prop.multiProcessorCount;
    star_dedup* h = new star_dedup;
    h->device = device;
    // mate2basesN beyond any l_seq (2^32-1) always fails the N <= l_seq contract; 2^32-1 keeps that
    h->mate2N = mate2basesN > 0xffffffffULL ? 0xffffffffu : (u32)mate2basesN;
    // Members per sub-batch from the free memory: 80 bytes of per-member arrays plus the sort's scratch, and the record bytes
    // (a few hundred per paired-end record); a quarter of the free memory at 1 KB per member.
    size_t freeB = 0, totalB = 0;
    if (cudaMemGetInfo(&freeB, &totalB) != cudaSuccess) freeB = 1ULL << 30;
    h->maxM = std::min<u64>(1ULL << 31, std::max<u64>(1ULL << 16, freeB / 4 / 1024));
    if (const char* s = getenv("STAR_B200_DEDUP_BATCH_RECS")) h->maxM = std::max<u64>(1, strtoull(s, nullptr, 10));
    if (const char* s = getenv("STAR_B200_DEDUP_HASH_BITS")) h->hashBits = (u32)std::min<u64>(64, strtoull(s, nullptr, 10));
    cudaEventCreate(&h->ev[0]);
    cudaEventCreate(&h->ev[1]);
    *out = h;
    return 0;
}

int star_gpu_dedup_batch(star_dedup_t* h, const uint8_t* bytes, const uint64_t* offsets, const uint32_t* groups, uint64_t n, uint8_t* unmark, float* ms) {
    if (cudaSetDevice(h->device) != cudaSuccess) { setLastError("star_b200: cudaSetDevice failed"); return STAR_EXIT_RUNTIME; }
    for (u64 i = 1; i < n; i++)
        if (groups[i] < groups[i - 1] || offsets[i] <= offsets[i - 1]) {
            setLastError("star_b200: star_gpu_dedup_batch: member " + std::to_string(i) + " is out of file or group order");
            return STAR_EXIT_BUG;
        }
    memset(unmark, 0, n);
    if (ms) *ms = 0;
    if (n == 0) return 0;
    g_ddErr = cudaSuccess;
    u64 errMember = 0;
    u32 errKind = 0;
    cudaEventRecord(h->ev[0]);
    const int rc = dedupBatchRun(h->bufs, bytes, offsets, groups, n, h->mate2N, h->hashBits, h->maxM, unmark, errMember, errKind);
    cudaEventRecord(h->ev[1]);
    cudaEventSynchronize(h->ev[1]);
    if (ms) cudaEventElapsedTime(ms, h->ev[0], h->ev[1]);
    if (rc == 3 || g_ddErr == cudaErrorMemoryAllocation) { setLastError("star_b200: out of device memory for duplicate removal"); return STAR_EXIT_MEMORY_ALLOCATION; }
    if (g_ddErr != cudaSuccess) { setLastError(std::string("CUDA error in duplicate removal: ") + cudaGetErrorString(g_ddErr)); return STAR_EXIT_RUNTIME; }
    if (rc == 1) {
        setLastError("star_b200: duplicate removal: input error (kind " + std::to_string(errKind) + ") at member " + std::to_string(errMember));
        return dedupReportError(unmark, n, errMember, errKind);
    }
    return 0;
}

void star_gpu_dedup_close(star_dedup_t* h) {
    if (!h) return;
    cudaSetDevice(h->device);
    h->bufs.release();
    cudaFree(g_ddTmp);
    g_ddTmp = nullptr;
    g_ddTmpBytes = 0;
    cudaEventDestroy(h->ev[0]);
    cudaEventDestroy(h->ev[1]);
    delete h;
}

}  // extern "C"
