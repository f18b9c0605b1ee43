// engine_api.cu — C-ABI of the CUDA engine (include/star_b200.h): context, HBM residency of the index,
// per-chunk kernel pipeline, slow-path re-run of reads that exceed a fast-path cap.
//
// Replaces (reference): ReadAlignChunk::mapChunk + the ReadAlign::oneRead loop
// (source/ReadAlignChunk_mapChunk.cpp:7-128, ReadAlign_oneRead.cpp:8-121) and the shared-memory genome
// residency (Genome_genomeLoad.cpp:177-243).  There is NO CPU fallback: every entry point fails with
// STAR_EXIT_RUNTIME when no CUDA device is usable.
//
// Pipeline of one chunk (star_gpu_map_resident), all on one stream:
//   prep_reads -> seed_search (MMP) -> radix sort by number of loci (heaviest first) -> stitch_kernel for reads with < 4 loci
//   -> flat_setup (windows, export) -> flat_dfs_warp (sub-tree tasks) -> flat_record_warp (ordered recording, selection)
//   -> overflow tiers for reads that exceeded a cap (bigger arenas; last tier = the reference's own limits) -> scan + pack
//   -> work counters.  Environment knobs (STAR_B200_*) exist for measurements only; defaults are the measured best.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include <cub/device/device_radix_sort.cuh>

#include "dev.cuh"
#include "seed_types.cuh"
#include "stitch_types.cuh"

namespace starb {
// kernels (seed.cu, stitch.cu)
__global__ void prep_reads_kernel(const char*, const u64*, u32, u32, u8*, u32, ReadInfo*, star_params_t);
void launch_build_sa_keys(int, cudaStream_t, const DevIndex&, u32*);
void launch_seed_chains(int, cudaStream_t, const DevIndex&, const star_params_t&, const u8*, u32, ReadInfo*, u32, const KeyedArgs&);
void launch_seed_keyed_search(int, int, int, cudaStream_t, const DevIndex&, const star_params_t&, const u8*, u32, ReadInfo*, const u32*, const KeyedArgs&);
void launch_seed_replay(int, cudaStream_t, const star_params_t&, ReadInfo*, Piece*, u32, u32, const KeyedArgs&);
void launch_seed_warp(int, int, cudaStream_t, const DevIndex&, const star_params_t&, const u8*, u32, ReadInfo*, Piece*, u32, u32, const u32*, u32*, u32);
__global__ void stitch_kernel(DevIndex, star_params_t, const u8*, u32, ReadInfo*, const Piece*, u32, const u32*, u32*, u8*, Caps,
                              star_read_result_t*, star_align_t*, const u32*, u32, HeavyArgs);
__global__ void stitch_heavy_kernel(DevIndex, star_params_t, const u8*, u32, ReadInfo*, const Piece*, u32, const u32*, const u64*, const u8*, u32*, u8*, Caps,
                                    star_read_result_t*, star_align_t*, u32, u8*, HeavyScratch);
__global__ void count_heavy_kernel(const ReadInfo*, u32, u32, u32*);
__global__ void order_keys_kernel(const ReadInfo*, u32, u32*, u32*);
__global__ void prof_read_kernel(unsigned long long*, int);
__global__ void pack_kernel(const star_read_result_t*, const u64*, const star_align_t*, u32, u32, star_align_t*);
__global__ void scan_partial_kernel(const star_read_result_t*, u32, u32, u64*);
__global__ void scan_top_kernel(u64*, u32, u64*);
__global__ void scan_write_kernel(star_read_result_t*, u64*, u32, u32, const u64*);
__global__ void reduce_counters_kernel(const ReadInfo*, u32, WorkCounters*);

// collects the indices of reads whose ReadInfo.flags has `mask` set
__global__ void collect_flagged_kernel(const ReadInfo* __restrict__ info, u32 nReads, u32 mask, u32* __restrict__ list, u32* __restrict__ count) {
    u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nReads && (info[i].flags & mask)) {
        u32 k = atomicAdd(count, 1u);
        list[k] = i;
    }
}
}  // namespace starb

using namespace starb;

static thread_local std::string g_err;
static unsigned long long g_launches = 0;
namespace starb {   // used by sjdb.cu
void setLastError(const std::string& m) { g_err = m; }
void countLaunches(unsigned n) { g_launches += n; }
}

#define CK(call)                                                                                       \
    do {                                                                                               \
        cudaError_t e_ = (call);                                                                       \
        if (e_ != cudaSuccess) {                                                                       \
            g_err = std::string("CUDA error: ") + cudaGetErrorString(e_) + " at " + __FILE__ + ":" + std::to_string(__LINE__); \
            return STAR_EXIT_RUNTIME;                                                                  \
        }                                                                                              \
    } while (0)

struct star_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    star_params_t P;
    DevIndex ix;
    std::vector<void*> owned;    // device allocations freed in destroy
    u32 maxReads = 0;
    int nSM = 0;
    // per-chunk buffers
    char* d_seq = nullptr; size_t seqCap = 0;
    u64* d_seqOff = nullptr;
    u8* d_reads = nullptr; u8* d_readsBase = nullptr; size_t readsCap = 0;   // d_reads = d_readsBase + 256: the 8-byte gathers of the seed stage touch up to 14 bytes in front of a row
    ReadInfo* d_info = nullptr;
    Piece* d_pieces = nullptr;
    star_read_result_t* d_results = nullptr;
    star_align_t* d_staged = nullptr;
    star_align_t* d_aligns = nullptr;
    u64* d_offsets = nullptr;
    u64* d_total = nullptr;
    u64* d_scanPartial = nullptr;
    u32* d_counter = nullptr;    // [0] ticket, [1] flagged count
    u32* d_list = nullptr;
    u32 *d_keys = nullptr, *d_keys2 = nullptr, *d_vals = nullptr, *d_order = nullptr;
    void* d_sortTmp = nullptr; size_t sortTmpBytes = 0;
    WorkCounters* d_wc = nullptr;
    // heavy-read path (warp per read)
    u8* d_heavyPool = nullptr; u64 heavyPoolBytes = 0;
    unsigned long long* d_heavyBump = nullptr;     // [0] pool bump, [1] (u32) heavy count
    u64* d_heavyOff = nullptr;
    u32* d_heavyList = nullptr;
    u8* d_heavyScratch = nullptr;
    u32 heavyEst = 1024; u32 heavyNA = 64; u32 heavyMaxTasks = 8192, heavyMaxBlocks = 4096;
    Caps heavyCaps; u8* d_arenaHeavy = nullptr;   // per-WARP arenas of the warp-per-read kernel (bigger caps than the per-lane fast arenas)
    u64 heavyScratchBytes = 0; u64 heavyScratchStride = 0; u64 lastHeavy = 0;
    // flattened heavy path (stitch_flat.cuh): setup -> sub-tree tasks -> ordered recording, each over all heavy reads of the chunk
    bool flat = false;
    FlatArgs fa{};
    Caps recCaps; u8* d_arenaRec = nullptr;
    int setupCtas = 3; u8* d_arenaSetup = nullptr; int recCtas = 4; int dfsCtas = 4;
    int seedWarpCtas = 0;   // > 0: seed_search_warp_kernel with this many CTAs per SM for the whole chunk (STAR_B200_SEED_WARP; measurements)
    // keyed seed stage (seed_keyed.cuh): SA keys of the index, chain items, their sort, records
    KeyedArgs ka{};
    u32* d_saKeys = nullptr;
    u32 *d_itemKey2 = nullptr, *d_itemOrder = nullptr;
    void* d_itemSortTmp = nullptr; size_t itemSortTmpBytes = 0;
    int keyedCtas = 8, keyedLanes = 8; int seedSortBits = 16; float msKeys = 0;
    unsigned long long flatUse[4] = {0, 0, 0, 0};   // pool bytes / tasks / blocks / stored words used by the last chunk
    // fast path
    Caps fast; u8* d_arenaFast = nullptr; int gridSeed = 0, gridStitch = 0;
    // overflow tiers (allocated on first use): [0] medium caps on many lanes, [1] the reference's own limits on few lanes
    struct Tier { Caps caps; u8* arena = nullptr; Piece* pieces = nullptr; u32 lanes = 0, batch = 0; Caps recCaps; u8* arenaSetup = nullptr; u8* arenaRec = nullptr; };
    Tier tiers[2];
    u32 tierReads[2] = {0, 0};   // reads redone by each overflow tier in the last chunk
    // state of the resident chunk
    u32 nReads = 0, nMates = 1, stride = 0, smemStride = 0;
    u64 nAligns = 0;
    cudaEvent_t ev[12];
    star_chunk_stats_t last;
};

template <class T>
static int devAlloc(star_ctx* c, T** p, size_t n) {
    void* q = nullptr;
    CK(cudaMalloc(&q, n * sizeof(T) + 64));
    c->owned.push_back(q);
    *p = (T*)q;
    return 0;
}
template <class T>
static int devUpload(star_ctx* c, const T** dst, const T* src, size_t n, size_t padBytes = 64) {
    void* q = nullptr;
    CK(cudaMalloc(&q, n * sizeof(T) + padBytes));
    c->owned.push_back(q);
    CK(cudaMemset(q, 0, n * sizeof(T) + padBytes));
    if (n) CK(cudaMemcpy(q, src, n * sizeof(T), cudaMemcpyHostToDevice));
    *dst = (const T*)q;
    return 0;
}

static u64 arenaSize(const Caps& c) {
    u64 b = 0;
    b += (u64)c.maxW * sizeof(Window);
    b += (u64)c.maxW * c.spw * sizeof(Seed);
    b += (u64)c.maxTr * sizeof(DevTr);
    b += 2 * sizeof(DevTr);
    b += (u64)(c.spw + 2) * 128;     // Frame is 128 bytes (stitch.cu)
    b += (u64)c.maxTr * 2;
    b += (u64)c.maxW * 2 * 2;
    return (b + 255) & ~255ULL;
}

static u32 envU32(const char* name, u32 dflt) {
    const char* e = getenv(name);
    return e ? (u32)strtoul(e, nullptr, 10) : dflt;
}

extern "C" {

const char* star_gpu_last_error(void) { return g_err.c_str(); }
uint64_t star_gpu_launch_count(void) { return g_launches; }

int star_gpu_set_sj_novel(star_ctx_t* c, const uint64_t* sjStart, const uint64_t* sjEnd, uint64_t n) {
    CK(cudaSetDevice(c->device));
    CK(cudaDeviceSynchronize());
    if (devUpload(c, &c->ix.sjNovelStart, (const u64*)sjStart, n)) return STAR_EXIT_RUNTIME;
    if (devUpload(c, &c->ix.sjNovelEnd, (const u64*)sjEnd, n)) return STAR_EXIT_RUNTIME;
    c->ix.sjNovelN = n;
    c->ix.sjNovelOn = 1;
    return 0;
}

void star_gpu_destroy(star_ctx_t* c) {
    if (!c) return;
    cudaSetDevice(c->device);
    cudaDeviceSynchronize();
    for (void* p : c->owned) cudaFree(p);
    if (c->d_seq) cudaFree(c->d_seq);                 // grown on demand (ensureSeq / ensureReads / launchHeavy), not in `owned`
    if (c->d_readsBase) cudaFree(c->d_readsBase);
    if (c->d_heavyScratch) cudaFree(c->d_heavyScratch);
    if (c->stream) cudaStreamDestroy(c->stream);
    for (auto& e : c->ev) if (e) cudaEventDestroy(e);
    delete c;
}

static int initCtx(star_ctx* c, int device, const star_index_view_t* v, const star_params_t* params, uint32_t maxReadsPerChunk);

int star_gpu_init(star_ctx_t** out, int device, const star_index_view_t* v, const star_params_t* params, uint32_t maxReadsPerChunk) {
    *out = nullptr;
    int nDev = 0;
    cudaError_t e = cudaGetDeviceCount(&nDev);
    if (e != cudaSuccess || nDev == 0) {
        g_err = std::string("star_b200: no CUDA device available (") + cudaGetErrorString(e) + "); this engine has no CPU fallback";
        return STAR_EXIT_RUNTIME;
    }
    if (device < 0 || device >= nDev) { g_err = "star_b200: bad device ordinal"; return STAR_EXIT_RUNTIME; }
    if (v->gSAsparseD != 1) { g_err = "star_b200: only genomeSAsparseD 1 indices are supported"; return STAR_EXIT_GENOME_FILES; }
    if (v->gSAindexNbases > 18) { g_err = "star_b200: genomeSAindexNbases > 18 is not supported"; return STAR_EXIT_GENOME_FILES; }
    if (params->seedPerWindowNmax > 50) { g_err = "star_b200: seedPerWindowNmax > 50 is not supported by this build (DFS depth)"; return STAR_EXIT_PARAMETER; }
    if (params->seedPerWindowNmax > 1000 || params->seedPerReadNmax > 60000 || params->alignTranscriptsPerReadNmax > 60000) {
        g_err = "star_b200: seedPerWindowNmax/seedPerReadNmax/alignTranscriptsPerReadNmax exceed the engine's 16-bit index range"; return STAR_EXIT_PARAMETER;
    }
    CK(cudaSetDevice(device));
    star_ctx* c = new star_ctx;
    memset(c->ev, 0, sizeof(c->ev));
    c->device = device;
    const int rc = initCtx(c, device, v, params, maxReadsPerChunk);
    if (rc) {   // nothing allocated so far outlives a failed init; the failed call's error state is consumed here
        const std::string keep = g_err;
        star_gpu_destroy(c);
        cudaGetLastError();
        g_err = keep;
        return rc;
    }
    *out = c;
    return 0;
}

static int initCtx(star_ctx* c, int device, const star_index_view_t* v, const star_params_t* params, uint32_t maxReadsPerChunk) {
    c->P = *params;
    c->maxReads = maxReadsPerChunk;
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, device));
    c->nSM = prop.multiProcessorCount;
    {   // The path is random 32-byte sector access over an index of tens of GB; with 64-byte fills of L2 every miss fetches a neighbour sector
        // that is rarely read.  32-byte fills halve the DRAM bytes of the seed search, but the kernels are latency-bound, not bandwidth-bound,
        // and the neighbour sector is a free prefetch for the key / SA / genome reads that do continue.  Default 64.
        const u32 gran = envU32("STAR_B200_L2_FETCH_BYTES", 64);
        if (gran == 32 || gran == 64 || gran == 128) cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, gran);
        cudaGetLastError();
    }
    CK(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    for (auto& ev : c->ev) CK(cudaEventCreate(&ev));

    // ---- index -> HBM (once) ----
    DevIndex& ix = c->ix;
    memset(&ix, 0, sizeof(ix));
    {
        const size_t PAD = 256;
        u8* g = nullptr;
        CK(cudaMalloc((void**)&g, v->nGenome + 2 * PAD + 64));
        c->owned.push_back(g);
        CK(cudaMemcpy(g, v->G - PAD, v->nGenome + 2 * PAD, cudaMemcpyHostToDevice));
        ix.G = g + PAD;
    }
    ix.nGenome = v->nGenome;
    {
        size_t words = (v->nSAbyte + 7) / 8 + 2;
        std::vector<u64> tmp;   // copy through a zero-padded word buffer only for the tail
        u64* d = nullptr;
        CK(cudaMalloc((void**)&d, words * 8));
        c->owned.push_back(d);
        CK(cudaMemset(d, 0, words * 8));
        CK(cudaMemcpy(d, v->SA, v->nSAbyte, cudaMemcpyHostToDevice));
        ix.SA = d;
        size_t wordsI = (v->nSAibyte + 7) / 8 + 2;
        u64* di = nullptr;
        CK(cudaMalloc((void**)&di, wordsI * 8));
        c->owned.push_back(di);
        CK(cudaMemset(di, 0, wordsI * 8));
        CK(cudaMemcpy(di, v->SAi, v->nSAibyte, cudaMemcpyHostToDevice));
        ix.SAi = di;
    }
    ix.nSA = v->nSA; ix.nSAi = v->nSAi;
    ix.GstrandBit = v->GstrandBit; ix.saBits = v->GstrandBit + 1; ix.saiBits = v->GstrandBit + 3;
    ix.gSAindexNbases = v->gSAindexNbases; ix.gChrBinNbits = v->gChrBinNbits; ix.nChrReal = v->nChrReal;
    ix.GstrandMask = ~(1ULL << v->GstrandBit);
    ix.SAiMarkNmaskC = 1ULL << (v->GstrandBit + 1); ix.SAiMarkNmask = ~ix.SAiMarkNmaskC; ix.SAiMarkAbsentMaskC = 1ULL << (v->GstrandBit + 2);
    for (u32 i = 0; i <= v->gSAindexNbases; i++) ix.genomeSAindexStart[i] = v->genomeSAindexStart[i];
    {   // Genome::chrBinFill Genome.cpp:209-216
        u64 nb = 1ULL << v->gChrBinNbits;
        u64 chrBinN = v->chrStart[v->nChrReal] / nb + 1;
        std::vector<u32> cb(chrBinN);
        for (u64 ii = 0, ichr = 1; ii < chrBinN; ++ii) {
            if (ii * nb >= v->chrStart[ichr]) ichr++;
            cb[ii] = (u32)(ichr - 1);
        }
        if (devUpload(c, &ix.chrBin, cb.data(), chrBinN)) return STAR_EXIT_RUNTIME;
        ix.chrBinN = chrBinN;
    }
    if (devUpload(c, &ix.chrStart, (const u64*)v->chrStart, v->nChrReal + 1)) return STAR_EXIT_RUNTIME;
    if (devUpload(c, &ix.chrLength, (const u64*)v->chrLength, v->nChrReal)) return STAR_EXIT_RUNTIME;
    ix.sjdbN = v->sjdbN; ix.sjdbOverhang = v->sjdbOverhang; ix.sjdbLength = v->sjdbLength; ix.sjGstart = v->sjGstart;
    if (devUpload(c, &ix.sjdbStart, (const u64*)v->sjdbStart, v->sjdbN)) return STAR_EXIT_RUNTIME;
    if (devUpload(c, &ix.sjdbEnd, (const u64*)v->sjdbEnd, v->sjdbN)) return STAR_EXIT_RUNTIME;
    if (devUpload(c, &ix.sjDstart, (const u64*)v->sjDstart, v->sjdbN)) return STAR_EXIT_RUNTIME;
    if (devUpload(c, &ix.sjAstart, (const u64*)v->sjAstart, v->sjdbN)) return STAR_EXIT_RUNTIME;
    if (devUpload(c, &ix.sjdbMotif, v->sjdbMotif, v->sjdbN)) return STAR_EXIT_RUNTIME;
    if (devUpload(c, &ix.sjdbShiftLeft, v->sjdbShiftLeft, v->sjdbN)) return STAR_EXIT_RUNTIME;
    if (devUpload(c, &ix.sjdbShiftRight, v->sjdbShiftRight, v->sjdbN)) return STAR_EXIT_RUNTIME;
    if (devUpload(c, &ix.sjdbStrand, v->sjdbStrand, v->sjdbN)) return STAR_EXIT_RUNTIME;
    {   // step table of int(ceil(log2((double)g)*scale-0.5)) evaluated with the HOST libm exactly as the reference writes it
        // (stitchWindowAligns.cpp:221-225); the function is monotone in g, so change points are found by bisection.
        std::vector<u64> thr; std::vector<int> val;
        const double scale = params->scoreGenomicLengthLog2scale;
        auto f = [&](u64 g) { return int(std::ceil(std::log2((double)g) * scale - 0.5)); };
        const u64 gMax = 1ULL << 40;
        u64 pos = 1;
        thr.push_back(1); val.push_back(f(1));
        while (pos < gMax && thr.size() < 4096) {
            int cur = f(pos);
            if (f(gMax) == cur) break;
            u64 lo = pos, hi = pos + 1;
            while (hi < gMax && f(hi) == cur) { lo = hi; hi = hi * 2 < gMax ? hi * 2 : gMax; }
            if (f(hi) == cur) break;
            while (lo + 1 < hi) { u64 mid = lo + (hi - lo) / 2; if (f(mid) == cur) lo = mid; else hi = mid; }
            thr.push_back(hi); val.push_back(f(hi));
            pos = hi;
        }
        if (devUpload(c, &ix.log2Thr, thr.data(), thr.size())) return STAR_EXIT_RUNTIME;
        if (devUpload(c, &ix.log2Val, val.data(), val.size())) return STAR_EXIT_RUNTIME;
        ix.log2N = (int)thr.size();
    }
    // ---- per-chunk buffers ----
    const u32 N = maxReadsPerChunk;
    const u32 nOut = (u32)(params->outFilterMultimapNmax > 0 ? params->outFilterMultimapNmax : 1);
    c->fast.maxP = envU32("STAR_B200_FAST_MAXP", 128);
    c->fast.maxW = envU32("STAR_B200_FAST_MAXW", 128);
    c->fast.maxTr = envU32("STAR_B200_FAST_MAXTR", 128);
    c->fast.spw = (u32)params->seedPerWindowNmax;
    c->fast.nOut = nOut;
    c->fast.sortMinW = envU32("STAR_B200_SORTED_LOOKUP_MIN", 12);
    c->fast.binFilter = envU32("STAR_B200_BIN_FILTER", 0);   // no gain over the bisection at GRCh38 size: off
    if (c->fast.maxP > params->seedPerReadNmax) c->fast.maxP = (u32)params->seedPerReadNmax;
    if (c->fast.maxW > params->alignWindowsPerReadNmax) c->fast.maxW = (u32)params->alignWindowsPerReadNmax;
    c->fast.maxW = (c->fast.maxW + 1) & ~1u;
    if (c->fast.maxTr > params->alignTranscriptsPerReadNmax) c->fast.maxTr = (u32)params->alignTranscriptsPerReadNmax;
    c->fast.arenaBytes = arenaSize(c->fast);
    {
        star_ctx::Tier& M = c->tiers[0];
        M.caps.maxP = std::min<u32>((u32)params->seedPerReadNmax, envU32("STAR_B200_MID_MAXP", 512));
        M.caps.maxW = (std::min<u32>((u32)params->alignWindowsPerReadNmax, envU32("STAR_B200_MID_MAXW", 2048)) + 1) & ~1u;
        M.caps.maxTr = std::min<u32>((u32)params->alignTranscriptsPerReadNmax, envU32("STAR_B200_MID_MAXTR", 4096));
        M.caps.spw = c->fast.spw; M.caps.nOut = nOut; M.caps.sortMinW = c->fast.sortMinW; M.caps.binFilter = c->fast.binFilter;
        M.caps.arenaBytes = arenaSize(M.caps);
        M.lanes = envU32("STAR_B200_MID_LANES", 8192); M.batch = envU32("STAR_B200_MID_BATCH", 65536);
        star_ctx::Tier& S = c->tiers[1];
        S.caps.maxP = (u32)params->seedPerReadNmax;
        S.caps.maxW = ((u32)params->alignWindowsPerReadNmax + 1) & ~1u;
        S.caps.maxTr = (u32)params->alignTranscriptsPerReadNmax;
        S.caps.spw = c->fast.spw; S.caps.nOut = nOut; S.caps.sortMinW = c->fast.sortMinW; S.caps.binFilter = c->fast.binFilter;
        S.caps.arenaBytes = arenaSize(S.caps);
        S.lanes = envU32("STAR_B200_SLOW_LANES", 128); S.batch = envU32("STAR_B200_SLOW_BATCH", 4096);
    }
    if (devAlloc(c, &c->d_seqOff, (size_t)N * 2 + 2)) return STAR_EXIT_RUNTIME;
    if (devAlloc(c, &c->d_info, N)) return STAR_EXIT_RUNTIME;
    if (devAlloc(c, &c->d_pieces, (size_t)N * c->fast.maxP)) return STAR_EXIT_RUNTIME;
    if (devAlloc(c, &c->d_results, N)) return STAR_EXIT_RUNTIME;
    if (devAlloc(c, &c->d_staged, (size_t)N * nOut)) return STAR_EXIT_RUNTIME;
    if (devAlloc(c, &c->d_aligns, (size_t)N * nOut)) return STAR_EXIT_RUNTIME;
    if (devAlloc(c, &c->d_offsets, N)) return STAR_EXIT_RUNTIME;
    if (devAlloc(c, &c->d_total, 2)) return STAR_EXIT_RUNTIME;
    if (devAlloc(c, &c->d_scanPartial, (size_t)c->nSM * 8 + 8)) return STAR_EXIT_RUNTIME;
    if (devAlloc(c, &c->d_counter, 4)) return STAR_EXIT_RUNTIME;
    if (devAlloc(c, &c->d_list, N)) return STAR_EXIT_RUNTIME;
    if (devAlloc(c, &c->d_wc, 1)) return STAR_EXIT_RUNTIME;
    if (devAlloc(c, &c->d_keys, N)) return STAR_EXIT_RUNTIME;
    if (devAlloc(c, &c->d_keys2, N)) return STAR_EXIT_RUNTIME;
    if (devAlloc(c, &c->d_vals, N)) return STAR_EXIT_RUNTIME;
    if (devAlloc(c, &c->d_order, N)) return STAR_EXIT_RUNTIME;
    CK(cub::DeviceRadixSort::SortPairs(nullptr, c->sortTmpBytes, c->d_keys, c->d_keys2, c->d_vals, c->d_order, (int)N));
    CK(cudaMalloc(&c->d_sortTmp, c->sortTmpBytes + 64));
    c->owned.push_back(c->d_sortTmp);
    c->heavyEst = envU32("STAR_B200_HEAVY_EST", 1024);
    c->heavyNA = envU32("STAR_B200_HEAVY_NA", 4);
    if (!c->heavyEst) c->heavyNA = 0;
    c->heavyMaxTasks = envU32("STAR_B200_HEAVY_TASKS", 8192);
    c->heavyMaxBlocks = envU32("STAR_B200_HEAVY_BLOCKS", 4096);
    if (c->heavyEst) {
        c->heavyPoolBytes = (u64)envU32("STAR_B200_HEAVY_POOL_MB", 0) << 20;
        if (!c->heavyPoolBytes) c->heavyPoolBytes = std::min<u64>(8ULL << 30, std::max<u64>(64ULL << 20, (u64)N * 4096));
        CK(cudaMalloc((void**)&c->d_heavyPool, c->heavyPoolBytes));
        c->owned.push_back(c->d_heavyPool);
        if (devAlloc(c, &c->d_heavyBump, 4)) return STAR_EXIT_RUNTIME;
        if (devAlloc(c, &c->d_heavyOff, N)) return STAR_EXIT_RUNTIME;
        if (devAlloc(c, &c->d_heavyList, N)) return STAR_EXIT_RUNTIME;
    }
    if (c->heavyEst) {
        c->heavyCaps = c->fast;
        c->heavyCaps.maxW = (std::min<u32>((u32)params->alignWindowsPerReadNmax, envU32("STAR_B200_HEAVY_MAXW", 512)) + 1) & ~1u;
        c->heavyCaps.maxTr = std::min<u32>((u32)params->alignTranscriptsPerReadNmax, envU32("STAR_B200_HEAVY_MAXTR", 1024));
        c->heavyCaps.arenaBytes = arenaSize(c->heavyCaps);
    }
    // persistent grids: as many 128-lane CTAs as fit per SM (registers / shared memory decide; queried per launch config)
    c->seedWarpCtas = (int)envU32("STAR_B200_SEED_WARP", 0);
    {   // SA keys: 4 bytes per SA row (23.6 GB for GRCh38), built once per context from the resident SA and genome
        const size_t nk = (size_t)v->nSA + 8;
        CK(cudaMalloc((void**)&c->d_saKeys, nk * 4));
        c->owned.push_back(c->d_saKeys);
        CK(cudaMemsetAsync(c->d_saKeys, 0, nk * 4, c->stream));
        CK(cudaEventRecord(c->ev[0], c->stream));
        launch_build_sa_keys(c->nSM, c->stream, c->ix, c->d_saKeys);
        CK(cudaGetLastError());
        CK(cudaEventRecord(c->ev[1], c->stream));
        CK(cudaStreamSynchronize(c->stream));
        CK(cudaEventElapsedTime(&c->msKeys, c->ev[0], c->ev[1]));
        if (getenv("STAR_B200_DEBUG")) fprintf(stderr, "star_b200: SA keys of %llu rows built in %.1f ms\n", (unsigned long long)v->nSA, c->msKeys);
        KeyedArgs& ka = c->ka;
        ka.saKeys = c->d_saKeys;
        ka.maxItems = (u32)std::min<u64>(0xFFFF0000ULL, std::max<u64>(4096, (u64)N * envU32("STAR_B200_SEED_ITEMS_PER_READ", 20)));
        ka.maxRec = std::max<u32>(8, envU32("STAR_B200_SEED_RECS_PER_READ", 192));
        ka.scanMax = envU32("STAR_B200_SEED_SCAN_MAX", 2048);
        if (devAlloc(c, &ka.items, ka.maxItems)) return STAR_EXIT_RUNTIME;
        if (devAlloc(c, &ka.itemKey, ka.maxItems)) return STAR_EXIT_RUNTIME;
        if (devAlloc(c, &ka.itemIdx, ka.maxItems)) return STAR_EXIT_RUNTIME;
        if (devAlloc(c, &c->d_itemKey2, ka.maxItems)) return STAR_EXIT_RUNTIME;
        if (devAlloc(c, &c->d_itemOrder, ka.maxItems)) return STAR_EXIT_RUNTIME;
        if (devAlloc(c, &ka.itemCount, 4)) return STAR_EXIT_RUNTIME;
        if (devAlloc(c, &ka.recs, (size_t)N * ka.maxRec)) return STAR_EXIT_RUNTIME;
        if (devAlloc(c, &ka.recCount, N)) return STAR_EXIT_RUNTIME;
        CK(cub::DeviceRadixSort::SortPairs(nullptr, c->itemSortTmpBytes, ka.itemKey, c->d_itemKey2, ka.itemIdx, c->d_itemOrder, (int)ka.maxItems));
        CK(cudaMalloc(&c->d_itemSortTmp, c->itemSortTmpBytes + 64));
        c->owned.push_back(c->d_itemSortTmp);
        c->keyedCtas = (int)std::min<u32>(16, std::max<u32>(1, envU32("STAR_B200_SEED_KEYED_CTAS_PER_SM", 8)));
        c->keyedLanes = (int)envU32("STAR_B200_SEED_GROUP_LANES", 8);   // 4, 8 or 16 lanes per search
        c->seedSortBits = (int)std::min<u32>(2 * v->gSAindexNbases, envU32("STAR_B200_SEED_SORT_BITS", 0));   // 0: chains stay in read order
    }
    c->gridStitch = c->nSM * (int)envU32("STAR_B200_STITCH_CTAS_PER_SM", 2);
    {
        size_t bytes = (size_t)c->gridStitch * 128 * c->fast.arenaBytes;
        CK(cudaMalloc((void**)&c->d_arenaFast, bytes));
        c->owned.push_back(c->d_arenaFast);
    }
    if (c->heavyEst) {   // one arena per warp: the kernel indexes arenas by (first thread of the warp) * arenaBytes, so allocate with a stride of 32 arenas... no: use a dedicated stride
        size_t bytes = (size_t)c->gridStitch * 4 * c->heavyCaps.arenaBytes;
        CK(cudaMalloc((void**)&c->d_arenaHeavy, bytes));
        c->owned.push_back(c->d_arenaHeavy);
    }
    c->flat = c->heavyEst && envU32("STAR_B200_HEAVY_FLAT", 1) != 0;
    if (c->flat) {
        FlatArgs& fa = c->fa;
        // per-read sizes: with the GRCh38-sized index, 2x100 pairs use ~0.45 KB of pool, ~5 tasks, ~2 blocks and ~210 stored words (DESIGN.md §6)
        const u64 perRead = envU32("STAR_B200_FLAT_POOL_KB", 4) * 1024ULL;
        fa.poolBytes = std::min<u64>(48ULL << 30, std::max<u64>(256ULL << 20, (u64)N * perRead));
        fa.maxTasks = std::max<u64>(4ULL << 20, (u64)N * envU32("STAR_B200_FLAT_TASKS_PER_READ", 64));
        if (fa.maxTasks > 0xFFFF0000ULL) fa.maxTasks = 0xFFFF0000ULL;
        fa.maxBlocks = (u32)std::min<u64>(0xFFFF0000ULL, std::max<u64>(1ULL << 20, (u64)N * envU32("STAR_B200_FLAT_BLOCKS_PER_READ", 32)));
        fa.trWords = std::min<u64>(0xFFFF0000ULL, std::max<u64>(16ULL << 20, (u64)N * envU32("STAR_B200_FLAT_TRWORDS_PER_READ", 2048)));
        c->recCaps = c->heavyCaps;
        c->recCaps.arenaBytes = ((u64)c->recCaps.maxW * sizeof(Window) + (u64)c->recCaps.maxTr * sizeof(DevTr) + (u64)c->recCaps.maxTr * 2
                                 + (u64)c->recCaps.maxW * 4 + 255) & ~255ULL;
        c->setupCtas = (int)std::min<u32>(4, std::max<u32>(2, envU32("STAR_B200_FLAT_SETUP_CTAS_PER_SM", 3)));
        c->recCtas = (int)std::min<u32>(4, std::max<u32>(2, envU32("STAR_B200_FLAT_REC_CTAS_PER_SM", 4)));
        const u64 arenas = (u64)c->nSM * 4 * (c->setupCtas * c->heavyCaps.arenaBytes + c->recCtas * c->recCaps.arenaBytes);
        {   // The per-read pool sizes fill ~28 GB at N = 1 M pairs: more than an 80 GB device has left beside a GRCh38-sized index (~56 GB with
            // the SA keys).  The pools get what the device has free once the arenas and everything this context allocates on demand (the
            // overflow tiers, the chunk's reads; runFlatTier / ensureReads) are set aside.  Smaller pools run out sooner: every pool has an
            // exhaustion path (the reads are redone by the overflow tiers).
            const star_ctx::Tier& T0 = c->tiers[0];
            const star_ctx::Tier& T1 = c->tiers[1];
            const u64 rec0 = ((u64)T0.caps.maxW * sizeof(Window) + (u64)T0.caps.maxTr * sizeof(DevTr) + (u64)T0.caps.maxTr * 2 + (u64)T0.caps.maxW * 4 + 255) & ~255ULL;
            const u64 onDemand = ((u64)T0.batch * T0.caps.maxP + (u64)T1.batch * T1.caps.maxP) * sizeof(Piece) + (u64)c->nSM * 2 * 4 * (T0.caps.arenaBytes + rec0)
                                 + (u64)T1.lanes * T1.caps.arenaBytes + (u64)N * 1024 + (1ULL << 30);
            size_t freeB = 0, totalB = 0;
            CK(cudaMemGetInfo(&freeB, &totalB));
            const u64 want = fa.poolBytes + fa.maxTasks * (sizeof(FlatTask) + sizeof(FlatOut)) + (u64)fa.maxBlocks * sizeof(FlatBlock) + fa.trWords * 8;
            const u64 avail = freeB > onDemand + arenas ? freeB - onDemand - arenas : 0;
            if (want > avail) {
                const double s = std::max(0.01, (double)avail / (double)want);
                fa.poolBytes = (u64)(fa.poolBytes * s) & ~255ULL;
                fa.maxTasks = (u64)(fa.maxTasks * s);
                fa.maxBlocks = (u32)(fa.maxBlocks * s);
                fa.trWords = (u64)(fa.trWords * s);
            }
        }
        // absolute overrides (tests exercise the exhaustion paths with tiny pools)
        if (getenv("STAR_B200_FLAT_POOL_BYTES")) fa.poolBytes = strtoull(getenv("STAR_B200_FLAT_POOL_BYTES"), nullptr, 10);
        if (getenv("STAR_B200_FLAT_MAXTASKS")) fa.maxTasks = strtoull(getenv("STAR_B200_FLAT_MAXTASKS"), nullptr, 10);
        if (getenv("STAR_B200_FLAT_MAXBLOCKS")) fa.maxBlocks = (u32)strtoull(getenv("STAR_B200_FLAT_MAXBLOCKS"), nullptr, 10);
        if (getenv("STAR_B200_FLAT_TRWORDS")) fa.trWords = strtoull(getenv("STAR_B200_FLAT_TRWORDS"), nullptr, 10);
        fa.storeAll = envU32("STAR_B200_FLAT_STORE_ALL", 1); fa.slabByPos = 0;
        fa.maxTasksPerRead = c->heavyMaxTasks;
        fa.splitMin = envU32("STAR_B200_HEAVY_SPLIT", 48);   // windows with more seeds are cut into prefix sub-trees
        void* p = nullptr;
        CK(cudaMalloc(&p, (size_t)N * sizeof(FlatRec))); fa.recs = (FlatRec*)p; c->owned.push_back(p);
        CK(cudaMalloc(&p, fa.poolBytes)); fa.pool = (u8*)p; c->owned.push_back(p);
        CK(cudaMalloc(&p, 64)); fa.bumps = (unsigned long long*)p; c->owned.push_back(p);
        CK(cudaMalloc(&p, fa.maxTasks * sizeof(FlatTask))); fa.tasks = (FlatTask*)p; c->owned.push_back(p);
        CK(cudaMalloc(&p, fa.maxTasks * sizeof(FlatOut))); fa.outs = (FlatOut*)p; c->owned.push_back(p);
        CK(cudaMalloc(&p, (size_t)fa.maxBlocks * sizeof(FlatBlock))); fa.blocks = (FlatBlock*)p; c->owned.push_back(p);
        CK(cudaMalloc(&p, fa.trWords * 8)); fa.trStore = (u64*)p; c->owned.push_back(p);
        // recording kernel (recCaps): one lane per read, each lane with its own transcript pool; persistent grids of the three flat kernels
        CK(cudaMalloc(&p, (size_t)c->nSM * c->setupCtas * 4 * c->heavyCaps.arenaBytes)); c->d_arenaSetup = (u8*)p; c->owned.push_back(p);
        CK(cudaMalloc(&p, (size_t)c->nSM * c->recCtas * 4 * c->recCaps.arenaBytes)); c->d_arenaRec = (u8*)p; c->owned.push_back(p);   // one arena per warp
        c->dfsCtas = (int)std::min<u32>(8, std::max<u32>(2, envU32("STAR_B200_FLAT_DFS_CTAS_PER_SM", 4)));
    }
    CK(cudaFuncSetAttribute(stitch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    CK(cudaFuncSetAttribute(stitch_heavy_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    return 0;
}

static int ensureSeq(star_ctx* c, size_t bytes) {
    if (bytes + 64 <= c->seqCap) return 0;
    if (c->d_seq) cudaFree(c->d_seq);
    c->seqCap = bytes + bytes / 4 + 4096;
    CK(cudaMalloc((void**)&c->d_seq, c->seqCap));
    return 0;
}
static int ensureReads(star_ctx* c, size_t bytes) {
    if (bytes <= c->readsCap) return 0;
    if (c->d_readsBase) cudaFree(c->d_readsBase);
    c->d_readsBase = nullptr; c->d_reads = nullptr; c->readsCap = 0;
    const size_t cap = bytes + bytes / 4 + 4096;
    CK(cudaMalloc((void**)&c->d_readsBase, cap + 512));
    CK(cudaMemset(c->d_readsBase, 0, 256));
    c->d_reads = c->d_readsBase + 256;
    c->readsCap = cap;
    return 0;
}

int star_gpu_upload_chunk(star_ctx_t* c, const star_read_batch_t* in) {
    CK(cudaSetDevice(c->device));
    if (in->nReads > c->maxReads) { g_err = "star_b200: chunk larger than maxReadsPerChunk given to star_gpu_init"; return STAR_EXIT_PARAMETER; }
    if (in->nMates != 1 && in->nMates != 2) { g_err = "star_b200: nMates must be 1 or 2"; return STAR_EXIT_PARAMETER; }
    c->nReads = in->nReads; c->nMates = in->nMates;
    if (in->nReads == 0) return 0;
    const u64 nOff = (u64)in->nReads * in->nMates + 1;
    const u64 seqBytes = in->seqOff[nOff - 1];
    // longest combined read decides the row stride (host scan of the offsets; lengths were validated by the reader)
    u32 maxL = 0;
    for (u64 i = 0; i < in->nReads; i++) {
        const uint64_t* o = in->seqOff + i * in->nMates;
        u64 l0 = o[1] - o[0], l1 = in->nMates == 2 ? o[2] - o[1] : 0;
        if (in->nMates == 1 && l0 < 1) {   // (a mate of a pair may be empty: clipped to nothing before mapping)
            g_err = "EXITING because of FATAL ERROR in reads input: short read sequence line: 0\n"; return STAR_EXIT_INPUT_FILES; }
        u64 L = in->nMates == 2 ? l0 + l1 + 1 : l0;
        if (L > STAR_READ_SEQ_LENGTH_MAX) { g_err = "EXITING because of FATAL ERROR in reads input: Lread of the pair exceeds DEF_readSeqLengthMax\n"; return STAR_EXIT_INPUT_FILES; }
        if (L > maxL) maxL = (u32)L;
    }
    c->stride = (maxL + 16) & ~15u;
    u32 s = (maxL + 1 + 3) & ~3u;
    if (((s / 4) & 1) == 0) s += 4;     // odd number of 32-bit words per shared-memory row: conflict-free lane rows
    c->smemStride = s;
    if (ensureSeq(c, seqBytes)) return STAR_EXIT_RUNTIME;
    if (ensureReads(c, (size_t)in->nReads * c->stride)) return STAR_EXIT_RUNTIME;
    CK(cudaEventRecord(c->ev[0], c->stream));
    CK(cudaMemcpyAsync(c->d_seq, in->seq, seqBytes, cudaMemcpyHostToDevice, c->stream));
    CK(cudaMemcpyAsync(c->d_seqOff, in->seqOff, nOff * 8, cudaMemcpyHostToDevice, c->stream));
    CK(cudaEventRecord(c->ev[1], c->stream));
    c->last.h2d_bytes = seqBytes + nOff * 8;
    return 0;
}

// Launches the warp-per-read kernel over `nHeavy` reads of `list` (device pointer).  pool==true: reads exported by stitch_kernel
// (windows + seeds in the heavy pool); pool==false: reads routed here right after seeding (the warp does the window phases too).
static int launchHeavy(star_ctx* c, const Caps& caps, u8* arenas, int gridBlocks, const u32* list, u32 nHeavy, bool pool, const Piece* pieces) {
    if (nHeavy == 0) return 0;
    HeavyScratch hs;
    hs.maxTasks = c->heavyMaxTasks; hs.maxBlocks = c->heavyMaxBlocks; hs.maxWin = caps.maxW;
    const u32 W1 = (hs.maxWin + 2) & ~1u;
    hs.trWords = envU32("STAR_B200_HEAVY_TRWORDS", 1u << 17);   // 1 MB of stored transcripts per warp
    hs.splitMin = envU32("STAR_B200_HEAVY_SPLIT", 6);
    hs.memoSlots = envU32("STAR_B200_HEAVY_MEMO", 0);   // measured: most stitches live in windows with <10 seeds where pairs rarely repeat; off by default          // stitch memo entries per warp (power of two, 0 = off)
    if (hs.memoSlots & (hs.memoSlots - 1)) { g_err = "STAR_B200_HEAVY_MEMO must be a power of two"; return STAR_EXIT_PARAMETER; }
    hs.bytesPerWarp = ((u64)W1 * 8 + ((W1 + 7) & ~7u) + (u64)hs.maxTasks * 8 + (u64)hs.maxBlocks * 504 + (u64)hs.trWords * 8 + 8 + (u64)hs.memoSlots * 72 + 255) & ~255ULL;
    const u32 warps = (u32)gridBlocks * 4;
    const u64 need = (u64)warps * hs.bytesPerWarp;
    if (need <= c->heavyScratchBytes && hs.bytesPerWarp != c->heavyScratchStride) {
        CK(cudaMemsetAsync(c->d_heavyScratch, 0, c->heavyScratchBytes, c->stream));   // layout changed (other tier): forget memo / epochs
        c->heavyScratchStride = hs.bytesPerWarp;
    }
    if (need > c->heavyScratchBytes) {
        if (c->d_heavyScratch) cudaFree(c->d_heavyScratch);
        CK(cudaMalloc((void**)&c->d_heavyScratch, need));
        CK(cudaMemsetAsync(c->d_heavyScratch, 0, need, c->stream));   // memo keys / epochs start at zero
        c->heavyScratchBytes = need;
        c->heavyScratchStride = hs.bytesPerWarp;
    }
    CK(cudaMemsetAsync(c->d_counter, 0, 4, c->stream));
    const u32 perWarp = (2 * c->smemStride + 32 + caps.maxW * (u32)sizeof(Window) + (caps.maxW + 4) * 4 + ((caps.maxW + 3) & ~3u) + 15) & ~15u;
    const u32 smem = 4 * perWarp;
    if (smem > 200 * 1024) { g_err = "star_b200: heavy kernel shared memory exceeds the limit for this tier"; return STAR_EXIT_RUNTIME; }
    stitch_heavy_kernel<<<gridBlocks, 128, smem, c->stream>>>(c->ix, c->P, c->d_reads, c->stride, c->d_info, pieces, nHeavy, list, c->d_heavyOff,
                                                            pool ? c->d_heavyPool : nullptr, c->d_counter, arenas, caps, c->d_results, c->d_staged,
                                                            c->smemStride, c->d_heavyScratch, hs);
    g_launches++;
    CK(cudaGetLastError());
    return 0;
}

// Runs the heavy kernel over the reads the preceding stitch_kernel pass exported (if any).
static int runHeavy(star_ctx* c, const Caps& caps, u8* arenas, int gridBlocks, u32 /*smemStride*/) {
    if (!c->heavyEst) return 0;
    u32 nHeavy = 0;
    CK(cudaMemcpyAsync(&nHeavy, (u32*)(c->d_heavyBump + 1), 4, cudaMemcpyDeviceToHost, c->stream));
    CK(cudaStreamSynchronize(c->stream));
    c->lastHeavy += nHeavy;
    if (nHeavy == 0) return 0;
    // sort the exported list so that runs are reproducible (atomics produced an arbitrary order)
    std::vector<u32> list(nHeavy);
    CK(cudaMemcpy(list.data(), c->d_heavyList, (size_t)nHeavy * 4, cudaMemcpyDeviceToHost));
    std::sort(list.begin(), list.end());
    CK(cudaMemcpy(c->d_heavyList, list.data(), (size_t)nHeavy * 4, cudaMemcpyHostToDevice));
    return launchHeavy(c, caps, arenas, gridBlocks, c->d_heavyList, nHeavy, true, nullptr);
}
// Flattened heavy path, first tier.  listB = reads routed here right after seeding (head of the nA-descending order), then the
// reads stitch_kernel exported (known after a sync).  One setup launch per list, then ONE task kernel and ONE recording kernel.
static int runFlat(star_ctx* c, u32 nHeavyB) {
    const Caps& caps = c->heavyCaps;
    const u32 perWarp = (2 * c->smemStride + 32 + caps.maxW * (u32)sizeof(Window) + (caps.maxW + 4) * 4 + ((caps.maxW + 3) & ~3u) + 15) & ~15u;
    const u32 smem = 4 * perWarp;
    if (smem > 200 * 1024) { g_err = "star_b200: flat setup kernel shared memory exceeds the limit"; return STAR_EXIT_RUNTIME; }
    CK(cudaMemsetAsync(c->fa.bumps, 0, 64, c->stream));
    if (nHeavyB) {
        CK(cudaMemsetAsync(c->d_counter, 0, 4, c->stream));
        launch_flat_setup(c->setupCtas, c->nSM, smem, c->stream, c->ix, c->P, c->d_reads, c->stride, c->d_info, c->d_pieces, nHeavyB, c->d_order, c->d_heavyOff,
                          nullptr, c->d_counter, c->d_arenaSetup, caps, c->d_results, c->d_staged, c->smemStride, c->fa, 0);
        g_launches++;
        CK(cudaGetLastError());
    }
    u32 nHeavyX = 0;   // exported by stitch_kernel
    CK(cudaMemcpyAsync(&nHeavyX, (u32*)(c->d_heavyBump + 1), 4, cudaMemcpyDeviceToHost, c->stream));
    CK(cudaStreamSynchronize(c->stream));
    c->lastHeavy += nHeavyX;
    if (nHeavyX) {
        std::vector<u32> list(nHeavyX);   // deterministic order (the export order came from atomics)
        CK(cudaMemcpy(list.data(), c->d_heavyList, (size_t)nHeavyX * 4, cudaMemcpyDeviceToHost));
        std::sort(list.begin(), list.end());
        CK(cudaMemcpy(c->d_heavyList, list.data(), (size_t)nHeavyX * 4, cudaMemcpyHostToDevice));
        CK(cudaMemsetAsync(c->d_counter, 0, 4, c->stream));
        launch_flat_setup(c->setupCtas, c->nSM, smem, c->stream, c->ix, c->P, c->d_reads, c->stride, c->d_info, nullptr, nHeavyX, c->d_heavyList, c->d_heavyOff,
                          c->d_heavyPool, c->d_counter, c->d_arenaSetup, caps, c->d_results, c->d_staged, c->smemStride, c->fa, nHeavyB);
        g_launches++;
        CK(cudaGetLastError());
    }
    const u32 nRecs = nHeavyB + nHeavyX;
    if (nRecs == 0) return 0;
    CK(cudaMemsetAsync(c->d_counter, 0, 4, c->stream));
    launch_flat_dfs(c->dfsCtas, c->nSM, c->stream, c->ix, c->P, c->fa, c->d_counter, caps);
    g_launches++;
    CK(cudaGetLastError());
    CK(cudaMemsetAsync(c->d_counter, 0, 4, c->stream));
    launch_flat_record(c->recCtas, c->nSM, c->stream, c->ix, c->P, c->d_info, nRecs, c->d_counter, c->d_arenaRec, c->recCaps, c->d_results, c->d_staged, c->fa);
    g_launches++;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(c->flatUse, c->fa.bumps, 32, cudaMemcpyDeviceToHost, c->stream));
    return 0;
}

// Overflow tier on the flat path: the reads of `list` (read ids on the device; pieces re-seeded into `pieces`, one slab per list position)
// with the tier's bigger caps — cooperative window creation / assignment, sub-tree tasks, ordered recording, as the first pass.
// On the GRCh38-sized index a few reads per million overflow the first-pass window cap (reads from repeat families with hundreds of
// windows); redone by ONE LANE each they dominate the step.
static int runFlatTier(star_ctx* c, star_ctx::Tier& T, const u32* list, u32 nList) {
    const Caps& caps = T.caps;
    const u32 perWarp = (2 * c->smemStride + 32 + caps.maxW * (u32)sizeof(Window) + (caps.maxW + 4) * 4 + ((caps.maxW + 3) & ~3u) + 15) & ~15u;
    const u32 smem = 4 * perWarp;
    const int ctas = 2;
    if (!T.arenaSetup) {
        CK(cudaMalloc((void**)&T.arenaSetup, (size_t)c->nSM * ctas * 4 * caps.arenaBytes));
        c->owned.push_back(T.arenaSetup);
        T.recCaps = caps;
        T.recCaps.arenaBytes = ((u64)caps.maxW * sizeof(Window) + (u64)caps.maxTr * sizeof(DevTr) + (u64)caps.maxTr * 2 + (u64)caps.maxW * 4 + 255) & ~255ULL;
        CK(cudaMalloc((void**)&T.arenaRec, (size_t)c->nSM * ctas * 4 * T.recCaps.arenaBytes));
        c->owned.push_back(T.arenaRec);
    }
    FlatArgs fa = c->fa;
    fa.slabByPos = 1;
    CK(cudaMemsetAsync(fa.bumps, 0, 64, c->stream));
    CK(cudaMemsetAsync(c->d_counter, 0, 4, c->stream));
    launch_flat_setup(ctas, c->nSM, smem, c->stream, c->ix, c->P, c->d_reads, c->stride, c->d_info, T.pieces, nList, list, c->d_heavyOff, nullptr, c->d_counter,
                      T.arenaSetup, caps, c->d_results, c->d_staged, c->smemStride, fa, 0);
    CK(cudaMemsetAsync(c->d_counter, 0, 4, c->stream));
    launch_flat_dfs(c->dfsCtas, c->nSM, c->stream, c->ix, c->P, fa, c->d_counter, caps);
    CK(cudaMemsetAsync(c->d_counter, 0, 4, c->stream));
    launch_flat_record(ctas, c->nSM, c->stream, c->ix, c->P, c->d_info, nList, c->d_counter, T.arenaRec, T.recCaps, c->d_results, c->d_staged, fa);
    g_launches += 3;
    CK(cudaGetLastError());
    return 0;
}

static HeavyArgs heavyArgs(star_ctx* c) {
    HeavyArgs hv;
    hv.pool = c->d_heavyPool; hv.poolBytes = c->heavyPoolBytes; hv.bump = c->d_heavyBump; hv.readOff = c->d_heavyOff;
    hv.list = c->d_heavyList; hv.count = (u32*)(c->d_heavyBump + 1); hv.estLimit = c->heavyEst;
    return hv;
}

int star_gpu_map_resident(star_ctx_t* c, star_chunk_stats_t* stats) {
    CK(cudaSetDevice(c->device));
    star_chunk_stats_t& st = c->last;
    const u32 n = c->nReads;
    c->nAligns = 0;
    if (n == 0) { if (stats) { memset(stats, 0, sizeof(*stats)); } return 0; }
    const unsigned long long launches0 = g_launches;
    CK(cudaMemsetAsync(c->d_wc, 0, sizeof(WorkCounters), c->stream));
    CK(cudaEventRecord(c->ev[2], c->stream));
    {
        int grid = c->nSM * 8;
        prep_reads_kernel<<<grid, 256, 0, c->stream>>>(c->d_seq, c->d_seqOff, n, c->nMates, c->d_reads, c->stride, c->d_info, c->P);
        g_launches++;
        CK(cudaGetLastError());
    }
    CK(cudaEventRecord(c->ev[3], c->stream));
    const u32 smemStitch = 128 * 2 * c->smemStride;
    if (smemStitch > 200 * 1024) { g_err = "star_b200: read too long for the shared-memory staging"; return STAR_EXIT_RUNTIME; }
    // ---- fast path over all reads ----
    CK(cudaMemsetAsync(c->d_counter, 0, 16, c->stream));
    if (c->seedWarpCtas) {   // measurements: one read per warp, 32-ary search with genome comparisons (the tier seeder) over the whole chunk
        launch_seed_warp(c->seedWarpCtas, c->nSM, c->stream, c->ix, c->P, c->d_reads, c->stride, c->d_info, c->d_pieces, c->fast.maxP, n, nullptr, c->d_counter, c->smemStride);
    } else {                 // default: chains binned by SAindex L-mer, keyed SA windows, ordered replay (seed_keyed.cuh)
        const KeyedArgs& ka = c->ka;
        CK(cudaMemsetAsync(ka.itemCount, 0, 4, c->stream));
        launch_seed_chains(c->nSM, c->stream, c->ix, c->P, c->d_reads, c->stride, c->d_info, n, ka);
        const u32* order = nullptr;
        if (c->seedSortBits > 0) {
            u32 nItems = 0;
            CK(cudaMemcpyAsync(&nItems, ka.itemCount, 4, cudaMemcpyDeviceToHost, c->stream));
            CK(cudaStreamSynchronize(c->stream));
            if (nItems > ka.maxItems) nItems = ka.maxItems;
            if (nItems > 1) {
                const int hiBit = 2 * (int)c->ix.gSAindexNbases;
                CK(cub::DeviceRadixSort::SortPairs(c->d_itemSortTmp, c->itemSortTmpBytes, ka.itemKey, c->d_itemKey2, ka.itemIdx, c->d_itemOrder, (int)nItems,
                                                   hiBit - c->seedSortBits, hiBit, c->stream));
                g_launches += 3;
                order = c->d_itemOrder;
            }
        }
        launch_seed_keyed_search(c->keyedLanes, c->keyedCtas, c->nSM, c->stream, c->ix, c->P, c->d_reads, c->stride, c->d_info, order, ka);
        launch_seed_replay(c->nSM, c->stream, c->P, c->d_info, c->d_pieces, c->fast.maxP, n, ka);
        g_launches += 2;
    }
    g_launches++;
    CK(cudaGetLastError());
    CK(cudaEventRecord(c->ev[4], c->stream));
    CK(cudaMemsetAsync(c->d_counter, 0, 16, c->stream));
    order_keys_kernel<<<(n + 255) / 256, 256, 0, c->stream>>>(c->d_info, n, c->d_keys, c->d_vals);
    CK(cub::DeviceRadixSort::SortPairs(c->d_sortTmp, c->sortTmpBytes, c->d_keys, c->d_keys2, c->d_vals, c->d_order, (int)n, 0, 32, c->stream));
    g_launches += 4;   // key kernel + cub's histogram/onesweep passes (library kernels, not counted as ours beyond the launch)
    c->lastHeavy = 0;
    if (c->heavyEst) CK(cudaMemsetAsync(c->d_heavyBump, 0, 16, c->stream));
    // reads with many genomic loci (nA) go straight to the warp-per-read kernel: they are the head of the nA-descending order
    u32 nHeavyA = 0;
    if (c->heavyNA) {
        CK(cudaMemsetAsync(c->d_counter + 2, 0, 4, c->stream));
        count_heavy_kernel<<<(n + 255) / 256, 256, 0, c->stream>>>(c->d_info, n, c->heavyNA, c->d_counter + 2);
        g_launches++;
        CK(cudaMemcpyAsync(&nHeavyA, c->d_counter + 2, 4, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
    }
    c->lastHeavy += nHeavyA;
    CK(cudaMemsetAsync(c->d_counter, 0, 4, c->stream));
    if (n > nHeavyA) {
        stitch_kernel<<<c->gridStitch, 128, smemStitch, c->stream>>>(c->ix, c->P, c->d_reads, c->stride, c->d_info, c->d_pieces, n - nHeavyA, nullptr, c->d_counter,
                                                                      c->d_arenaFast, c->fast, c->d_results, c->d_staged, c->d_order + nHeavyA, c->smemStride, heavyArgs(c));
        g_launches++;
        CK(cudaGetLastError());
    }
    CK(cudaEventRecord(c->ev[9], c->stream));
    if (c->flat) {
        if (runFlat(c, nHeavyA)) return STAR_EXIT_RUNTIME;
    } else {
        if (launchHeavy(c, c->heavyCaps, c->d_arenaHeavy, c->gridStitch, c->d_order, nHeavyA, false, c->d_pieces)) return STAR_EXIT_RUNTIME;
        if (runHeavy(c, c->heavyCaps, c->d_arenaHeavy, c->gridStitch, c->smemStride)) return STAR_EXIT_RUNTIME;
    }
    CK(cudaEventRecord(c->ev[8], c->stream));
    // ---- overflow tiers: reads that exceeded the caps of a tier are redone in the next one; the last tier has the reference's own limits ----
    c->tierReads[0] = c->tierReads[1] = 0;
    for (int tier = 0; tier < 2; tier++) {
        CK(cudaMemsetAsync(c->d_counter + 1, 0, 4, c->stream));
        collect_flagged_kernel<<<(n + 255) / 256, 256, 0, c->stream>>>(c->d_info, n, 1u, c->d_list, c->d_counter + 1);
        g_launches++;
        u32 nSlow = 0;
        CK(cudaMemcpyAsync(&nSlow, c->d_counter + 1, 4, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        if (nSlow == 0) break;
        star_ctx::Tier& T = c->tiers[tier];
        const u32 perWarpT = (2 * c->smemStride + 32 + T.caps.maxW * (u32)sizeof(Window) + (T.caps.maxW + 4) * 4 + ((T.caps.maxW + 3) & ~3u) + 15) & ~15u;
        const bool flatTier = tier == 0 && c->flat && 4 * perWarpT <= 226 * 1024 && envU32("STAR_B200_FLAT_TIER", 1) != 0;   // (one CTA of flat_setup_kernel<2> per SM)
        if (!T.pieces) {
            CK(cudaMalloc((void**)&T.pieces, (size_t)T.batch * T.caps.maxP * sizeof(Piece)));
            c->owned.push_back(T.pieces);
        }
        if (!flatTier && !T.arena) {   // one arena per lane of the lane-per-read path (the flat tier has its own per-warp arenas)
            CK(cudaMalloc((void**)&T.arena, (size_t)T.lanes * T.caps.arenaBytes));
            c->owned.push_back(T.arena);
        }
        // heaviest first inside the tier too, deterministic order: sort (nA desc, index) on the host (the list is small)
        std::vector<u32> list(nSlow);
        CK(cudaMemcpy(list.data(), c->d_list, (size_t)nSlow * 4, cudaMemcpyDeviceToHost));
        std::sort(list.begin(), list.end());
        c->tierReads[tier] = nSlow;
        if (getenv("STAR_B200_DEBUG")) {   // why the reads of this tier left the previous one (reason in bits 8.. of ReadInfo.flags; 0 = seed stage)
            std::vector<ReadInfo> inf(n);
            CK(cudaMemcpy(inf.data(), c->d_info, (size_t)n * sizeof(ReadInfo), cudaMemcpyDeviceToHost));
            unsigned long long hist[8] = {0, 0, 0, 0, 0, 0, 0, 0};
            for (u32 r : list) hist[(inf[r].flags >> 8) & 7]++;
            fprintf(stderr, "star_b200: overflow tier %d: %u reads (seed stage %llu, windows %llu, transcripts %llu, export pool %llu, flat pools / tasks %llu)\n", tier, nSlow,
                    hist[0], hist[1], hist[3], hist[4], hist[5]);
        }
        CK(cudaMemcpy(c->d_list, list.data(), (size_t)nSlow * 4, cudaMemcpyHostToDevice));
        int grid = (int)(T.lanes / 128);
        if (grid < 1) grid = 1;
        for (u32 lo = 0; lo < nSlow; lo += T.batch) {
            u32 m = nSlow - lo < T.batch ? nSlow - lo : T.batch;
            CK(cudaMemsetAsync(c->d_counter, 0, 4, c->stream));
            launch_seed_warp(8, std::max(1, grid / 8), c->stream, c->ix, c->P, c->d_reads, c->stride, c->d_info, T.pieces, T.caps.maxP, m, c->d_list + lo, c->d_counter, c->smemStride);
            g_launches++;
            if (flatTier) {   // medium caps: the flat kernels again (warp-cooperative), not one lane per read
                if (runFlatTier(c, T, c->d_list + lo, m)) return STAR_EXIT_RUNTIME;
                continue;
            }
            CK(cudaMemsetAsync(c->d_counter, 0, 4, c->stream));
            if (c->heavyEst) CK(cudaMemsetAsync(c->d_heavyBump, 0, 16, c->stream));
            HeavyArgs hv = heavyArgs(c);
            const u32 perWarpH = (2 * c->smemStride + 32 + T.caps.maxW * (u32)sizeof(Window) + (T.caps.maxW + 4) * 4 + ((T.caps.maxW + 3) & ~3u) + 15) & ~15u;
            const bool heavyOk = c->heavyEst && 4 * perWarpH <= 200 * 1024;   // the last tier (reference limits) has no shared-memory window table
            if (!heavyOk) hv.estLimit = 0;
            stitch_kernel<<<grid, 128, smemStitch, c->stream>>>(c->ix, c->P, c->d_reads, c->stride, c->d_info, T.pieces, m, c->d_list + lo,
                                                                 c->d_counter, T.arena, T.caps, c->d_results, c->d_staged, nullptr, c->smemStride, hv);
            g_launches++;
            CK(cudaGetLastError());
            if (heavyOk && runHeavy(c, T.caps, T.arena, grid, c->smemStride)) return STAR_EXIT_RUNTIME;
        }
    }
    CK(cudaEventRecord(c->ev[5], c->stream));
    {
        const u32 nb = (u32)c->nSM * 8, per = (n + nb - 1) / nb;
        scan_partial_kernel<<<nb, 256, 0, c->stream>>>(c->d_results, n, per, c->d_scanPartial);
        scan_top_kernel<<<1, 32, 0, c->stream>>>(c->d_scanPartial, nb, c->d_total);
        scan_write_kernel<<<nb, 256, 0, c->stream>>>(c->d_results, c->d_offsets, n, per, c->d_scanPartial);
    }
    pack_kernel<<<c->nSM * 8, 256, 0, c->stream>>>(c->d_results, c->d_offsets, c->d_staged, c->fast.nOut, n, c->d_aligns);
    g_launches += 4;
    CK(cudaGetLastError());
    CK(cudaEventRecord(c->ev[6], c->stream));
    CK(cudaMemsetAsync(c->d_wc, 0, sizeof(WorkCounters), c->stream));
    reduce_counters_kernel<<<c->nSM * 4, 256, 0, c->stream>>>(c->d_info, n, c->d_wc);
    g_launches++;
    // fatal per-read conditions (reference: exitWithError inside the read loop)
    CK(cudaMemsetAsync(c->d_counter + 1, 0, 4, c->stream));
    collect_flagged_kernel<<<(n + 255) / 256, 256, 0, c->stream>>>(c->d_info, n, 3u, c->d_list, c->d_counter + 1);
    g_launches++;
    u32 nBad = 0;
    WorkCounters wc;
    CK(cudaMemcpyAsync(&nBad, c->d_counter + 1, 4, cudaMemcpyDeviceToHost, c->stream));
    CK(cudaMemcpyAsync(&wc, c->d_wc, sizeof(wc), cudaMemcpyDeviceToHost, c->stream));
    CK(cudaMemcpyAsync(&c->nAligns, c->d_total, 8, cudaMemcpyDeviceToHost, c->stream));
    CK(cudaStreamSynchronize(c->stream));
    if (c->flat && getenv("STAR_B200_FLAT_DEBUG"))
        fprintf(stderr, "star_b200 flat path: pool %.1f/%.1f MB, tasks %llu/%llu, blocks %llu/%u, stored words %llu/%llu\n", c->flatUse[0] / 1048576.0,
                c->fa.poolBytes / 1048576.0, c->flatUse[1], (unsigned long long)c->fa.maxTasks, c->flatUse[2], c->fa.maxBlocks, c->flatUse[3], (unsigned long long)c->fa.trWords);
    if (nBad > 0) {
        std::vector<ReadInfo> inf(1);
        u32 first = 0;
        CK(cudaMemcpy(&first, c->d_list, 4, cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(inf.data(), c->d_info + first, sizeof(ReadInfo), cudaMemcpyDeviceToHost));
        if (inf[0].flags & 2) {
            g_err = "EXITING because of FATAL error: too many pieces pere read\nSOLUTION: increase input parameter --seedPerReadNmax";   // ReadAlign_storeAligns.cpp:46-51
            return STAR_EXIT_RUNTIME;
        }
        g_err = "BUG: a read exceeded the slow-path capacities of star_b200";
        return STAR_EXIT_BUG;
    }
    float ms;
    cudaEventElapsedTime(&ms, c->ev[2], c->ev[3]); st.ms_prep = ms;
    cudaEventElapsedTime(&ms, c->ev[3], c->ev[4]); st.ms_seed = ms;
    cudaEventElapsedTime(&ms, c->ev[4], c->ev[8]); st.ms_stitch = ms;     // first tier: light kernel + heavy (warp-per-read) kernel
    cudaEventElapsedTime(&ms, c->ev[9], c->ev[8]); st.ms_heavy = ms;      // of which: heavy kernel
    st.heavy_reads = c->lastHeavy;
    cudaEventElapsedTime(&ms, c->ev[8], c->ev[5]); st.ms_window = ms;     // slow path (reads redone with the reference's limits)
    cudaEventElapsedTime(&ms, c->ev[5], c->ev[6]); st.ms_pack = ms;
    cudaEventElapsedTime(&ms, c->ev[2], c->ev[6]); st.ms_total = ms;
    st.n_kernel_launches = g_launches - launches0;
    st.mmp_searches = wc.searches; st.mmp_sai_words = wc.saiWords; st.mmp_compare_calls = wc.compareCalls; st.mmp_bases_examined = wc.basesExamined;
    st.sa_enumerated = wc.saEnum; st.stitch_nodes = wc.nodes; st.stitch_leaves = wc.leaves; st.slow_path_reads = wc.slowReads;
    if (stats) *stats = st;
    return 0;
}

int star_gpu_download_results(star_ctx_t* c, star_align_batch_t* out) {
    CK(cudaSetDevice(c->device));
    if (c->nAligns > out->alignsCapacity) { out->nAligns = c->nAligns; g_err = "star_b200: aligns capacity too small"; return STAR_EXIT_RUNTIME; }
    CK(cudaEventRecord(c->ev[0], c->stream));
    if (c->nReads) CK(cudaMemcpyAsync(out->reads, c->d_results, (size_t)c->nReads * sizeof(star_read_result_t), cudaMemcpyDeviceToHost, c->stream));
    if (c->nAligns) CK(cudaMemcpyAsync(out->aligns, c->d_aligns, (size_t)c->nAligns * sizeof(star_align_t), cudaMemcpyDeviceToHost, c->stream));
    CK(cudaEventRecord(c->ev[7], c->stream));
    CK(cudaStreamSynchronize(c->stream));
    out->nAligns = c->nAligns;
    float ms;
    cudaEventElapsedTime(&ms, c->ev[0], c->ev[7]);
    c->last.ms_d2h = ms;
    c->last.d2h_bytes = (u64)c->nReads * sizeof(star_read_result_t) + c->nAligns * sizeof(star_align_t);
    return 0;
}

void* star_gpu_host_alloc(size_t bytes) {
    void* p = nullptr;
    if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocPortable) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    return p;
}
void star_gpu_host_free(void* p) { if (p) cudaFreeHost(p); }

int star_gpu_map_chunk(star_ctx_t* c, const star_read_batch_t* in, star_align_batch_t* out, star_chunk_stats_t* stats) {
    memset(&c->last, 0, sizeof(c->last));
    int rc = star_gpu_upload_chunk(c, in);
    if (rc) return rc;
    star_chunk_stats_t s;
    rc = star_gpu_map_resident(c, &s);
    if (rc) return rc;
    float msH2D = 0;
    if (c->nReads) cudaEventElapsedTime(&msH2D, c->ev[0], c->ev[1]);   // before ev[0] is reused by the download
    rc = star_gpu_download_results(c, out);
    c->last.ms_h2d = msH2D;
    c->last.ms_total += msH2D + c->last.ms_d2h;
    if (stats) *stats = c->last;   // (also when the capacity was too small: the caller may fetch the results again)
    return rc;
}

// debug / analysis: copies the per-read ReadInfo records (work counters, flags) of the resident chunk
int star_gpu_debug_read_info(star_ctx_t* c, void* dst, uint64_t bytes) {
    CK(cudaSetDevice(c->device));
    uint64_t need = (uint64_t)c->nReads * sizeof(ReadInfo);
    if (bytes < need) { g_err = "star_gpu_debug_read_info: buffer too small"; return STAR_EXIT_RUNTIME; }
    CK(cudaMemcpy(dst, c->d_info, need, cudaMemcpyDeviceToHost));
    return 0;
}

// debug / analysis: cycle accounting of the stitch kernels (32 x u64; see stitch.cu g_prof); resets the counters
int star_gpu_debug_prof(star_ctx_t* c, uint64_t* out32) {
    CK(cudaSetDevice(c->device));
    unsigned long long* d = nullptr;
    CK(cudaMalloc((void**)&d, 32 * 8));
    prof_read_kernel<<<1, 32, 0, c->stream>>>(d, 1);
    CK(cudaStreamSynchronize(c->stream));
    CK(cudaMemcpy(out32, d, 32 * 8, cudaMemcpyDeviceToHost));
    cudaFree(d);
    return 0;
}

// ---- engine vtable for the host driver; the shipped CLI binds the CUDA engine and nothing else ----
static int vt_init(void** ctx, int device, const star_index_view_t* ix, const star_params_t* p, uint32_t maxReads) {
    return star_gpu_init((star_ctx_t**)ctx, device, ix, p, maxReads);
}
static int vt_map(void* ctx, const star_read_batch_t* in, star_align_batch_t* out, star_chunk_stats_t* st) {
    return star_gpu_map_chunk((star_ctx_t*)ctx, in, out, st);
}
static void vt_destroy(void* ctx) { star_gpu_destroy((star_ctx_t*)ctx); }
static int vt_sjdb_open(void** h, int device, const star_index_view_t* v) { return star_gpu_sjdb_open((star_sjdb_t**)h, device, v); }
static int vt_sjdb_search(void* h, const uint8_t* Gsj, uint64_t sjdbN, uint64_t sjdbLength, const uint8_t* skipSeq, uint64_t* ind) {
    return star_gpu_sjdb_search((star_sjdb_t*)h, Gsj, sjdbN, sjdbLength, skipSeq, ind);
}
static int vt_sjdb_merge(void* h, const uint64_t* indSorted, uint64_t nInd, uint64_t nGsj, uint64_t nGsjNew, uint64_t sjdbLength, const uint32_t* oldSJind,
                         uint8_t* SAnew, uint64_t nSAnewByte) {
    return star_gpu_sjdb_merge_sa((star_sjdb_t*)h, indSorted, nInd, nGsj, nGsjNew, sjdbLength, oldSJind, SAnew, nSAnewByte);
}
static int vt_set_sj_novel(void* c, const uint64_t* a, const uint64_t* b, uint64_t n) { return star_gpu_set_sj_novel((star_ctx_t*)c, a, b, n); }
static void vt_sjdb_close(void* h) { star_gpu_sjdb_close((star_sjdb_t*)h); }
static int vt_download(void* ctx, star_align_batch_t* out) { return star_gpu_download_results((star_ctx_t*)ctx, out); }
static int vt_signal_open(void** h, int device, uint32_t nStrands) { return star_gpu_signal_open((star_signal_t**)h, device, nStrands); }
static int vt_signal_segment(void* h, uint32_t chrLen, const star_signal_block_t* b, uint64_t nB, int mode, star_signal_track_t* tr, float* ms) {
    return star_gpu_signal_segment((star_signal_t*)h, chrLen, b, nB, mode, tr, ms);
}
static void vt_signal_close(void* h) { star_gpu_signal_close((star_signal_t*)h); }
static int vt_dedup_open(void** h, int device, uint64_t n2) { return star_gpu_dedup_open((star_dedup_t**)h, device, n2); }
static int vt_dedup_batch(void* h, const uint8_t* bytes, const uint64_t* off, const uint32_t* grp, uint64_t n, uint8_t* unmark, float* ms) {
    return star_gpu_dedup_batch((star_dedup_t*)h, bytes, off, grp, n, unmark, ms);
}
static void vt_dedup_close(void* h) { star_gpu_dedup_close((star_dedup_t*)h); }
static int vt_addref_open(void** h, int device, const star_index_view_t* v, uint64_t nG, uint64_t nG1, uint64_t nG2, float* ms) {
    return star_gpu_addref_open((star_addref_t**)h, device, v, nG, nG1, nG2, ms);
}
static int vt_addref_search(void* h, const uint8_t* seq, uint64_t* ind, float* ms) { return star_gpu_addref_search((star_addref_t*)h, seq, ind, ms); }
static int vt_addref_merge(void* h, const uint64_t* ind, uint64_t nInd, uint8_t* SAnew, uint64_t nSAnewByte, float* ms) {
    return star_gpu_addref_merge_sa((star_addref_t*)h, ind, nInd, SAnew, nSAnewByte, ms);
}
static void vt_addref_close(void* h) { star_gpu_addref_close((star_addref_t*)h); }
static const star_engine_vtbl_t g_cuda_engine = {vt_init, vt_map, vt_destroy, star_gpu_last_error, vt_sjdb_open, vt_sjdb_search, vt_sjdb_merge, vt_sjdb_close, star_gpu_sa_build, vt_set_sj_novel,
                                                 star_gpu_host_alloc, star_gpu_host_free, vt_download, vt_signal_open, vt_signal_segment, vt_signal_close,
                                                 vt_dedup_open, vt_dedup_batch, vt_dedup_close, vt_addref_open, vt_addref_search, vt_addref_merge, vt_addref_close};

int star_cli_main(int argc, char** argv) { return star_cli_main_engine(argc, argv, &g_cuda_engine); }

}  // extern "C"
