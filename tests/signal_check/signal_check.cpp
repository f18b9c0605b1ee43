// signal_check.cpp — TEST INFRASTRUCTURE ONLY: two CPU implementations of star_gpu_signal_open / _segment / _close (include/star_b200.h)
// that the tests compare the product against.
//
//   signal_oracle_*   the reference's own loop (signalFromBAM.cpp:116-202) over the decoded blocks: one double per position and track, `++`
//                     for NH == 1 and `+= 1.0/NH` in record order, then the output scan of :81-104 recording where each track changes
//                     (bedGraph) or is nonzero (wiggle)
//   signal_emul_*     the UNMODIFIED kernels and window loop of star_b200/csrc/engine/signal_kernels.cuh compiled as host code through
//                     oracle/cuda_host_shim.h: every launch is one emulated CTA of host threads, cub's scans / sort / selection are std::
//                     restatements.  Capacities: STAR_B200_SIGNAL_WINDOW / STAR_B200_SIGNAL_PAIRS as in signal.cu (defaults 2^20).
// Built with hidden visibility and -Bsymbolic (tests/signal_check/Makefile): the host-compiled starb:: code never binds to the CUDA build
// of the same names in libstar_b200.so.
#include <algorithm>
#include <cstdlib>
#include <functional>
#include <thread>
#include <vector>

#include "../../oracle/cuda_host_shim.h"

namespace cuda_shim {
thread_local Dim tIdx, bIdx, bDim, gDim;
thread_local CtaShared* cta;
}  // namespace cuda_shim

namespace starb {
static void* emAlloc(size_t bytes) { return calloc(bytes ? bytes : 1, 1); }
static void emScanU32(unsigned* a, unsigned long long n) { for (unsigned long long i = 1; i < n; i++) a[i] += a[i - 1]; }
static void emExScanU32(unsigned* a, unsigned long long n) { unsigned s = 0; for (unsigned long long i = 0; i < n; i++) { const unsigned v = a[i]; a[i] = s; s += v; } }
static void emExScanU64(unsigned long long* a, unsigned long long n) { unsigned long long s = 0; for (unsigned long long i = 0; i < n; i++) { const unsigned long long v = a[i]; a[i] = s; s += v; } }
static void emSortPairsU32(const unsigned* kIn, unsigned* kOut, const unsigned* vIn, unsigned* vOut, unsigned long long n, int endBit) {   // stable, like cub's LSD radix sort
    std::vector<unsigned long long> order(n);
    for (unsigned long long i = 0; i < n; i++) order[i] = i;
    const unsigned mask = endBit >= 32 ? ~0u : ((1u << endBit) - 1);
    std::stable_sort(order.begin(), order.end(), [&](unsigned long long a, unsigned long long b) { return (kIn[a] & mask) < (kIn[b] & mask); });
    for (unsigned long long i = 0; i < n; i++) { kOut[i] = kIn[order[i]]; vOut[i] = vIn[order[i]]; }
}
static void emSelectIndex(const unsigned char* flags, unsigned* out, unsigned long long n, unsigned long long* nSel) {
    unsigned long long k = 0;
    for (unsigned long long i = 0; i < n; i++) if (flags[i]) out[k++] = (unsigned)i;
    *nSel = k;
}
// one CTA of nThreads host threads executing `body` (a kernel call with its arguments bound); the signal kernels use no warp collectives
static void runCta(unsigned nThreads, const std::function<void()>& body) {
    cuda_shim::CtaShared c;
    c.nThreads = nThreads;
    pthread_barrier_init(&c.bar, nullptr, nThreads);
    std::vector<std::thread> th;
    for (unsigned t = 0; t < nThreads; t++)
        th.emplace_back([&, t] {
            cuda_shim::tIdx = {t, 0, 0}; cuda_shim::bIdx = {0, 0, 0}; cuda_shim::bDim = {nThreads, 1, 1}; cuda_shim::gDim = {1, 1, 1};
            cuda_shim::cta = &c;
            body();
        });
    for (auto& t : th) t.join();
    pthread_barrier_destroy(&c.bar);
}
}  // namespace starb
#define SG_ALLOC(bytes) starb::emAlloc(bytes)
#define SG_FREE(p) free(p)
#define SG_ZERO(p, bytes) memset(p, 0, bytes)
#define SG_COPY_TO(dst, src, bytes) memcpy(dst, src, bytes)
#define SG_COPY_FROM(dst, src, bytes) memcpy(dst, src, bytes)
#define SG_LAUNCH(count, kernel, ...) starb::runCta(64, [&] { kernel(__VA_ARGS__); })
#define SG_SCAN_U32(a, n) starb::emScanU32(a, n)
#define SG_EXSCAN_U32(a, n) starb::emExScanU32(a, n)
#define SG_EXSCAN_U64(a, n) starb::emExScanU64(a, n)
#define SG_SORT_PAIRS_U32(kIn, kOut, vIn, vOut, n, endBit) starb::emSortPairsU32(kIn, kOut, vIn, vOut, n, endBit)
#define SG_SELECT_INDEX(flags, out, n, nSel) starb::emSelectIndex(flags, out, n, nSel)
#define SG_SYNC() ((void)0)
#include "../../star_b200/csrc/engine/signal_kernels.cuh"

using namespace starb;

namespace {
bool blocksOk(const star_signal_block_t* b, uint64_t n, uint32_t chrLen, uint32_t nS) {
    for (uint64_t i = 0; i < n; i++)
        if ((uint64_t)b[i].start + b[i].len > chrLen || b[i].nh == 0 || b[i].strand >= nS) return false;
    return true;
}
struct Tracks {
    uint32_t nS;
    std::vector<uint32_t> pos[4];
    std::vector<double> val[4];
    void publish(star_signal_track_t* tr) const {
        for (uint32_t t = 0; t < 2 * nS; t++) { tr[t].pos = pos[t].data(); tr[t].val = val[t].data(); tr[t].n = pos[t].size(); }
    }
};
struct Emul : Tracks {
    u64 maxW, maxPairs;
    SigBufs bufs;
};
u64 envU64(const char* name, u64 dflt) { const char* e = getenv(name); const u64 v = e ? strtoull(e, nullptr, 10) : dflt; return v ? v : 1; }
}  // namespace

extern "C" {
#pragma GCC visibility push(default)

int signal_oracle_open(void** h, int, uint32_t nStrands) {
    if (nStrands != 1 && nStrands != 2) return STAR_EXIT_BUG;
    Tracks* o = new Tracks;
    o->nS = nStrands;
    *h = o;
    return 0;
}
int signal_oracle_segment(void* h, uint32_t chrLen, const star_signal_block_t* blocks, uint64_t nBlocks, int mode, star_signal_track_t* tracks, float* ms) {
    Tracks* o = (Tracks*)h;
    if (!blocksOk(blocks, nBlocks, chrLen, o->nS)) return STAR_EXIT_BUG;
    const uint32_t sigN = 2 * o->nS;
    std::vector<double> sigAll((size_t)sigN * chrLen, 0.0);
    for (uint64_t i = 0; i < nBlocks; i++) {
        const star_signal_block_t& b = blocks[i];
        for (uint32_t aG = b.start; aG < b.start + b.len; aG++) {
            if (b.nh == 1) sigAll[(size_t)aG * sigN + 0 + 2 * b.strand]++;
            sigAll[(size_t)aG * sigN + 1 + 2 * b.strand] += 1.0 / b.nh;
        }
    }
    for (uint32_t is = 0; is < sigN; is++) {
        o->pos[is].clear(); o->val[is].clear();
        double prevSig = 0;
        for (uint32_t ig = 0; ig < chrLen; ig++) {
            const double newSig = sigAll[(size_t)sigN * ig + is];
            if (mode == 0 ? newSig != prevSig : newSig != 0) { o->pos[is].push_back(ig); o->val[is].push_back(newSig); }
            prevSig = newSig;
        }
    }
    o->publish(tracks);
    if (ms) *ms = 0;
    return 0;
}
void signal_oracle_close(void* h) { delete (Tracks*)h; }

int signal_emul_open(void** h, int, uint32_t nStrands) {
    if (nStrands != 1 && nStrands != 2) return STAR_EXIT_BUG;
    Emul* e = new Emul;
    e->nS = nStrands;
    e->maxW = envU64("STAR_B200_SIGNAL_WINDOW", 1u << 20);
    e->maxPairs = envU64("STAR_B200_SIGNAL_PAIRS", 1u << 20);
    *h = e;
    return 0;
}
int signal_emul_segment(void* h, uint32_t chrLen, const star_signal_block_t* blocks, uint64_t nBlocks, int mode, star_signal_track_t* tracks, float* ms) {
    Emul* e = (Emul*)h;
    if (!blocksOk(blocks, nBlocks, chrLen, e->nS)) return STAR_EXIT_BUG;
    for (uint32_t t = 0; t < 2 * e->nS; t++) { e->pos[t].clear(); e->val[t].clear(); }
    if (signalSegmentRun(e->bufs, e->nS, chrLen, blocks, nBlocks, mode, e->maxW, e->maxPairs, e->pos, e->val)) return STAR_EXIT_MEMORY_ALLOCATION;
    e->publish(tracks);
    if (ms) *ms = 0;
    return 0;
}
void signal_emul_close(void* h) { Emul* e = (Emul*)h; e->bufs.release(); delete e; }

#pragma GCC visibility pop
}  // extern "C"
