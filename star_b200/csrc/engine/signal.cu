// signal.cu — C-ABI of the signal tracks (include/star_b200.h: star_gpu_signal_*).  Kernels and the window loop: signal_kernels.cuh;
// the scan / sort / compaction primitives are cub's.  No CPU fallback: without a CUDA device star_gpu_signal_open fails.
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>

#include <cstdlib>
#include <string>
#include <vector>

#include "dev.cuh"

namespace starb {
void setLastError(const std::string& m);     // engine_api.cu
void countLaunches(unsigned n);
static int g_sgSM = 132;
static cudaError_t g_sgErr = cudaSuccess;
static inline void sgNote(cudaError_t e) { if (e != cudaSuccess && g_sgErr == cudaSuccess) g_sgErr = e; }
static inline void* sgAlloc(size_t bytes) { void* p = nullptr; if (cudaMalloc(&p, bytes ? bytes : 1) != cudaSuccess) { cudaGetLastError(); return nullptr; } return p; }
static inline unsigned sgGrid(unsigned long long count) {
    const unsigned long long want = (count + 255) / 256, cap = (unsigned long long)g_sgSM * 8;
    return (unsigned)(want < cap ? (want ? want : 1) : cap);
}
// cub's temporary storage, kept between calls
static void* g_sgTmp = nullptr;
static size_t g_sgTmpBytes = 0;
static void* sgTmp(size_t bytes) {
    if (bytes > g_sgTmpBytes) { cudaFree(g_sgTmp); g_sgTmp = sgAlloc(bytes); g_sgTmpBytes = g_sgTmp ? bytes : 0; if (!g_sgTmp) sgNote(cudaErrorMemoryAllocation); }
    return g_sgTmp;
}
static void sgScanU32(u32* a, u64 n) {
    size_t tb = 0;
    sgNote(cub::DeviceScan::InclusiveSum(nullptr, tb, a, a, (long long)n));
    if (void* t = sgTmp(tb)) sgNote(cub::DeviceScan::InclusiveSum(t, tb, a, a, (long long)n));
    countLaunches(2);
}
static void sgExScanU32(u32* a, u64 n) {
    size_t tb = 0;
    sgNote(cub::DeviceScan::ExclusiveSum(nullptr, tb, a, a, (long long)n));
    if (void* t = sgTmp(tb)) sgNote(cub::DeviceScan::ExclusiveSum(t, tb, a, a, (long long)n));
    countLaunches(2);
}
static void sgExScanU64(u64* a, u64 n) {
    size_t tb = 0;
    sgNote(cub::DeviceScan::ExclusiveSum(nullptr, tb, a, a, (long long)n));
    if (void* t = sgTmp(tb)) sgNote(cub::DeviceScan::ExclusiveSum(t, tb, a, a, (long long)n));
    countLaunches(2);
}
static void sgSortPairs(const u32* kIn, u32* kOut, const u32* vIn, u32* vOut, u64 n, int endBit) {   // LSD radix sort: stable
    size_t tb = 0;
    sgNote(cub::DeviceRadixSort::SortPairs(nullptr, tb, kIn, kOut, vIn, vOut, (long long)n, 0, endBit));
    if (void* t = sgTmp(tb)) sgNote(cub::DeviceRadixSort::SortPairs(t, tb, kIn, kOut, vIn, vOut, (long long)n, 0, endBit));
    countLaunches(4);
}
static void sgSelectIndex(const u8* flags, u32* out, u64 n, u64* nSel) {   // indices i < n with flags[i], in order
    *nSel = 0;
    unsigned long long* dN = (unsigned long long*)sgAlloc(8);
    if (!dN) { sgNote(cudaErrorMemoryAllocation); return; }
    thrust::counting_iterator<u32> it(0);
    size_t tb = 0;
    sgNote(cub::DeviceSelect::Flagged(nullptr, tb, it, flags, out, dN, (long long)n));
    if (void* t = sgTmp(tb)) sgNote(cub::DeviceSelect::Flagged(t, tb, it, flags, out, dN, (long long)n));
    unsigned long long h = 0;
    sgNote(cudaMemcpy(&h, dN, 8, cudaMemcpyDeviceToHost));
    *nSel = h;
    countLaunches(2);
    cudaFree(dN);
}
}  // namespace starb

#define SG_ALLOC(bytes) starb::sgAlloc(bytes)
#define SG_FREE(p) cudaFree(p)
#define SG_ZERO(p, bytes) starb::sgNote(cudaMemset(p, 0, bytes))
#define SG_COPY_TO(dst, src, bytes) starb::sgNote(cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice))
#define SG_COPY_FROM(dst, src, bytes) starb::sgNote(cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost))
#define SG_LAUNCH(count, kernel, ...) do { kernel<<<starb::sgGrid(count), 256>>>(__VA_ARGS__); starb::sgNote(cudaGetLastError()); starb::countLaunches(1); } while (0)
#define SG_SCAN_U32(a, n) starb::sgScanU32(a, n)
#define SG_EXSCAN_U32(a, n) starb::sgExScanU32(a, n)
#define SG_EXSCAN_U64(a, n) starb::sgExScanU64(a, n)
#define SG_SORT_PAIRS_U32(kIn, kOut, vIn, vOut, n, endBit) starb::sgSortPairs(kIn, kOut, vIn, vOut, n, endBit)
#define SG_SELECT_INDEX(flags, out, n, nSel) starb::sgSelectIndex(flags, out, n, nSel)
#define SG_SYNC() starb::sgNote(cudaDeviceSynchronize())
#include "signal_kernels.cuh"

using namespace starb;

struct star_signal {
    int device = 0;
    u32 nS = 1;
    u64 maxW = 0, maxPairs = 0;
    SigBufs bufs;
    std::vector<u32> pos[4];
    std::vector<double> val[4];
    cudaEvent_t ev[2];
};

extern "C" {

int star_gpu_signal_open(star_signal_t** out, int device, uint32_t nStrands) {
    *out = nullptr;
    int nDev = 0;
    cudaError_t e = cudaGetDeviceCount(&nDev);
    if (e != cudaSuccess || nDev == 0) {
        setLastError(std::string("star_b200: no CUDA device available (") + cudaGetErrorString(e) + "); the signal tracks have no CPU fallback");
        return STAR_EXIT_RUNTIME;
    }
    if (device < 0 || device >= nDev) { setLastError("star_b200: bad device ordinal"); return STAR_EXIT_RUNTIME; }
    if (nStrands != 1 && nStrands != 2) { setLastError("star_b200: star_gpu_signal_open: nStrands must be 1 or 2"); return STAR_EXIT_BUG; }
    if (cudaSetDevice(device) != cudaSuccess) { setLastError("star_b200: cudaSetDevice failed"); return STAR_EXIT_RUNTIME; }
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) g_sgSM = prop.multiProcessorCount;
    star_signal* h = new star_signal;
    h->device = device;
    h->nS = nStrands;
    // Capacities from the free memory: per window position and strand 20 bytes (two counters, rank, fold) plus per track 13 bytes (flag,
    // index, value); per pair 16 bytes (keys and values, double-buffered for the sort) plus the sort's scratch.  Half of the free memory goes
    // to the positions (a window of 2^28 covers the longest human chromosome), what is left to the pairs.
    size_t freeB = 0, totalB = 0;
    if (cudaMemGetInfo(&freeB, &totalB) != cudaSuccess) freeB = 1ULL << 30;
    const u64 perPos = 20ULL * nStrands + 13ULL * 2 * nStrands;
    h->maxW = std::min<u64>(1ULL << 28, std::max<u64>(1ULL << 16, freeB / 2 / perPos));
    const u64 left = freeB > h->maxW * perPos ? freeB - h->maxW * perPos : 0;
    h->maxPairs = std::min<u64>(1ULL << 30, std::max<u64>(1ULL << 16, left / 2 / 40));
    if (const char* s = getenv("STAR_B200_SIGNAL_WINDOW")) h->maxW = std::max<u64>(1, strtoull(s, nullptr, 10));
    if (const char* s = getenv("STAR_B200_SIGNAL_PAIRS")) h->maxPairs = std::max<u64>(1, strtoull(s, nullptr, 10));
    cudaEventCreate(&h->ev[0]);
    cudaEventCreate(&h->ev[1]);
    *out = h;
    return 0;
}

int star_gpu_signal_segment(star_signal_t* h, uint32_t chrLen, const star_signal_block_t* blocks, uint64_t nBlocks, int mode,
                            star_signal_track_t* tracks, float* ms) {
    if (cudaSetDevice(h->device) != cudaSuccess) { setLastError("star_b200: cudaSetDevice failed"); return STAR_EXIT_RUNTIME; }
    for (u64 i = 0; i < nBlocks; i++)
        if ((u64)blocks[i].start + blocks[i].len > chrLen || blocks[i].nh == 0 || blocks[i].strand >= h->nS) {
            setLastError("star_b200: star_gpu_signal_segment: block " + std::to_string(i) + " is outside the segment or has NH 0 / a bad strand");
            return STAR_EXIT_BUG;
        }
    g_sgErr = cudaSuccess;
    const u32 nT = 2 * h->nS;
    for (u32 t = 0; t < nT; t++) { h->pos[t].clear(); h->val[t].clear(); }
    cudaEventRecord(h->ev[0]);
    const int rc = signalSegmentRun(h->bufs, h->nS, chrLen, blocks, nBlocks, mode, h->maxW, h->maxPairs, h->pos, h->val);
    cudaEventRecord(h->ev[1]);
    cudaEventSynchronize(h->ev[1]);
    if (ms) { *ms = 0; cudaEventElapsedTime(ms, h->ev[0], h->ev[1]); }
    if (rc == 3 || g_sgErr == cudaErrorMemoryAllocation) { setLastError("star_b200: out of device memory for the signal tracks"); return STAR_EXIT_MEMORY_ALLOCATION; }
    if (g_sgErr != cudaSuccess) { setLastError(std::string("CUDA error in the signal tracks: ") + cudaGetErrorString(g_sgErr)); return STAR_EXIT_RUNTIME; }
    for (u32 t = 0; t < nT; t++) { tracks[t].pos = h->pos[t].data(); tracks[t].val = h->val[t].data(); tracks[t].n = h->pos[t].size(); }
    return 0;
}

void star_gpu_signal_close(star_signal_t* h) {
    if (!h) return;
    cudaSetDevice(h->device);
    h->bufs.release();
    cudaFree(g_sgTmp);
    g_sgTmp = nullptr;
    g_sgTmpBytes = 0;
    cudaEventDestroy(h->ev[0]);
    cudaEventDestroy(h->ev[1]);
    delete h;
}

}  // extern "C"
