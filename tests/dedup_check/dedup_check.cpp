// dedup_check.cpp — TEST INFRASTRUCTURE ONLY: two CPU implementations of star_gpu_dedup_open / _batch / _close (include/star_b200.h) that
// the tests compare the product against.
//
//   dedup_oracle_*   the reference's own steps per group (bamRemoveDuplicates.cpp:206-237): a stable sort of the members by funCompareNames
//                    (:13-32; glibc's qsort is a stable merge sort), adjacent members as pairs, a stable sort of the pairs by
//                    funCompareCoordFlagCigarSeq (:34-112), and the loop that keeps the highest AS of every run of equal pairs
//   dedup_emul_*     the UNMODIFIED kernels and batch loop of star_b200/csrc/engine/dedup_kernels.cuh compiled as host code through
//                    oracle/cuda_host_shim.h: every launch is one emulated CTA of host threads, cub's sort / scan / selection are std::
//                    restatements.  STAR_B200_DEDUP_BATCH_RECS (default 2^20) and STAR_B200_DEDUP_HASH_BITS as in dedup.cu.
// Built with hidden visibility and -Bsymbolic (tests/dedup_check/Makefile), like tests/signal_check.
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
static void emSortPairsU64(const unsigned long long* kIn, unsigned long long* kOut, const unsigned* vIn, unsigned* vOut, unsigned long long n, int endBit) {   // stable
    std::vector<unsigned long long> order(n);
    for (unsigned long long i = 0; i < n; i++) order[i] = i;
    const unsigned long long mask = endBit >= 64 ? ~0ULL : ((1ULL << endBit) - 1);
    std::stable_sort(order.begin(), order.end(), [&](unsigned long long a, unsigned long long b) { return (kIn[a] & mask) < (kIn[b] & mask); });
    for (unsigned long long i = 0; i < n; i++) { kOut[i] = kIn[order[i]]; vOut[i] = vIn[order[i]]; }
}
static void emMaxScanU32(unsigned* a, unsigned long long n) { for (unsigned long long i = 1; i < n; i++) a[i] = std::max(a[i], a[i - 1]); }
static void emSelectIndex(const unsigned char* flags, unsigned* out, unsigned long long n, unsigned long long* nSel) {
    unsigned long long k = 0;
    for (unsigned long long i = 0; i < n; i++) if (flags[i]) out[k++] = (unsigned)i;
    *nSel = k;
}
static void emAtomicMin(unsigned long long* p, unsigned long long v) {
    unsigned long long o = __atomic_load_n(p, __ATOMIC_SEQ_CST);
    while (v < o && !__atomic_compare_exchange_n(p, &o, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {}
}
static void emAtomicMax(unsigned long long* p, unsigned long long v) {
    unsigned long long o = __atomic_load_n(p, __ATOMIC_SEQ_CST);
    while (v > o && !__atomic_compare_exchange_n(p, &o, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {}
}
// one CTA of nThreads host threads executing `body`; the dedup kernels use no warp collectives
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
#define DD_ALLOC(bytes) starb::emAlloc(bytes)
#define DD_FREE(p) free(p)
#define DD_ZERO(p, bytes) memset(p, 0, bytes)
#define DD_COPY_TO(dst, src, bytes) memcpy(dst, src, bytes)
#define DD_COPY_FROM(dst, src, bytes) memcpy(dst, src, bytes)
#define DD_LAUNCH(count, kernel, ...) starb::runCta(16, [&] { kernel(__VA_ARGS__); })
#define DD_SORT_PAIRS_U64(kIn, kOut, vIn, vOut, n, endBit) starb::emSortPairsU64(kIn, kOut, vIn, vOut, n, endBit)
#define DD_MAXSCAN_U32(a, n) starb::emMaxScanU32(a, n)
#define DD_SELECT_INDEX(flags, out, n, nSel) starb::emSelectIndex(flags, out, n, nSel)
#define DD_ATOMIC_MIN_U64(p, v) starb::emAtomicMin((unsigned long long*)(p), (unsigned long long)(v))
#define DD_ATOMIC_MAX_U64(p, v) starb::emAtomicMax((unsigned long long*)(p), (unsigned long long)(v))
#define DD_SYNC() ((void)0)
#include "../../star_b200/csrc/engine/dedup_kernels.cuh"

using namespace starb;

namespace {
u64 envU64(const char* name, u64 dflt) { const char* e = getenv(name); return e ? strtoull(e, nullptr, 10) : dflt; }
struct Emul { u32 mate2N, hashBits; u64 maxM; DdBufs bufs; };
struct Oracle { uint64_t mate2N; };

bool orderOk(const uint64_t* offsets, const uint32_t* groups, uint64_t n) {
    for (uint64_t i = 1; i < n; i++) if (groups[i] < groups[i - 1] || offsets[i] <= offsets[i - 1]) return false;
    return true;
}

// the record fields as the reference reads them through uint32 pointers (p[k] = 32-bit word k of the record)
struct Ref {
    const uint8_t* b;
    uint32_t w(int k) const { return rd(b + 4 * k); }
    static uint32_t rd(const uint8_t* q) { uint32_t v; memcpy(&v, q, 4); return v; }
    uint32_t lName() const { return (w(3) << 24) >> 24; }
    uint32_t nCig() const { return (w(4) << 16) >> 16; }
    uint32_t flag() const { return w(4) >> 16; }
    uint32_t cig(uint32_t k) const { return rd(b + 36 + lName() + 4 * k); }
    const uint8_t* seq() const { return b + 36 + lName() + 4 * nCig(); }
};
int funCompareNames(const Ref& a, const Ref& b) {   // :13-32
    const uint32_t la = a.lName(), lb = b.lName();
    if (la != lb) return la > lb ? 1 : -1;
    const char* ca = (const char*)(a.b + 36);
    const char* cb = (const char*)(b.b + 36);
    for (uint32_t i = 0; i < la; i++) if (ca[i] != cb[i]) return ca[i] > cb[i] ? 1 : -1;   // (char is signed here, as on x86)
    const uint32_t fa = a.flag() & 0x80, fb = b.flag() & 0x80;
    return fa == fb ? 0 : fa > fb ? 1 : -1;
}
uint32_t funStartExtendS(const Ref& p) { return (p.cig(0) & 15) == 4 ? p.w(2) - (p.cig(0) >> 4) : p.w(2); }   // :34-41
uint32_t funCigarExtendS(const Ref& p, uint32_t* cout) {   // :43-59 (called on CIGARs of 1..100 operations that are not all S only)
    const uint32_t n = p.nCig();
    uint32_t n1 = n;
    if ((p.cig(0) & 15) == 4) { --n1; for (uint32_t k = 0; k < n1; k++) cout[k] = p.cig(k + 1); cout[0] += (p.cig(0) >> 4) << 4; }
    else for (uint32_t k = 0; k < n; k++) cout[k] = p.cig(k);
    if ((p.cig(n - 1) & 15) == 4) { --n1; cout[n1 - 1] += (p.cig(n - 1) >> 4) << 4; }
    return n1;
}
#define CMP(a, b) if ((a) > (b)) return 1; else if ((a) < (b)) return -1;
int funCompareCoordFlagCigarSeq(const Ref& a1, const Ref& a2, const Ref& b1, const Ref& b2, uint64_t N) {   // :72-112
    CMP(funStartExtendS(a1), funStartExtendS(b1));
    CMP(funStartExtendS(a2), funStartExtendS(b2));
    CMP(a1.flag(), b1.flag());
    CMP(a2.flag(), b2.flag());
    for (int m = 0; m < 2; m++) {
        uint32_t ca[100], cb[100];
        const uint32_t na = funCigarExtendS(m ? a2 : a1, ca), nb = funCigarExtendS(m ? b2 : b1, cb);
        CMP(na, nb);
        for (uint32_t i = 0; i < na; i++) CMP(ca[i], cb[i]);
    }
    const uint8_t *sa = a2.seq(), *sb = b2.seq();
    if ((a2.flag() & 0x10) == 0) {
        uint64_t ii = 1;
        for (; ii < N; ii += 2) CMP(sa[ii / 2], sb[ii / 2]);
        if (N % 2 > 0) { CMP(sa[ii / 2] >> 4, sb[ii / 2] >> 4); }
    } else {
        uint32_t ii = a2.w(5) - (uint32_t)N;
        if (ii % 2 > 0) { CMP(sa[ii / 2] & 15, sb[ii / 2] & 15); ++ii; }
        for (; ii < a2.w(5); ii += 2) CMP(sa[ii / 2], sb[ii / 2]);
    }
    return 0;
}
bool cigarOk(const Ref& r) {
    const uint32_t n = r.nCig();
    if (n < 1 || n > 100) return false;
    return (int)n - ((r.cig(0) & 15) == 4) - ((r.cig(n - 1) & 15) == 4) >= 1;
}
// bam_aux_get(.., "AS") + bam_aux2i: 0 found, 1 missing, 2 malformed
int auxAS(const uint8_t* rec, int& v) {
    const Ref R{rec};
    const uint8_t* s = rec + 36 + R.lName() + 4ull * R.nCig() + (R.w(5) + 1ull) / 2 + R.w(5);
    const uint8_t* end = rec + 4 + R.w(0);
    v = 0;
    auto sz = [](uint8_t t) { return t == 'A' || t == 'c' || t == 'C' ? 1 : t == 's' || t == 'S' ? 2 : t == 'i' || t == 'I' || t == 'f' ? 4 : t == 'd' ? 8 : 0; };
    while (s < end) {
        if (end - s < 3) return 2;
        const uint8_t t = s[2];
        const bool hit = s[0] == 'A' && s[1] == 'S';
        s += 3;
        if (hit) {
            if (end - s < sz(t)) return 2;
            int16_t h; uint16_t H; int32_t i;
            memcpy(&h, s, 2); memcpy(&H, s, 2); memcpy(&i, s, 4);
            v = t == 'c' ? (int8_t)s[0] : t == 'C' ? s[0] : t == 's' ? h : t == 'S' ? H : t == 'i' || t == 'I' ? i : 0;
            return 0;
        }
        if (sz(t)) s += sz(t);
        else if (t == 'Z' || t == 'H') { while (s < end && *s) ++s; ++s; }
        else if (t == 'B') {
            if (end - s < 5) return 2;
            const int b = sz(s[0]);
            if (!b) return 2;
            s += 5 + (uint64_t)Ref::rd(s + 1) * b;
        } else return 2;
    }
    return 1;
}
}  // namespace

extern "C" {
#pragma GCC visibility push(default)

int dedup_oracle_open(void** h, int, uint64_t mate2basesN) { *h = new Oracle{mate2basesN}; return 0; }
int dedup_oracle_batch(void* h, const uint8_t* bytes, const uint64_t* offsets, const uint32_t* groups, uint64_t n, uint8_t* unmark, float* ms) {
    const uint64_t N = ((Oracle*)h)->mate2N;
    if (ms) *ms = 0;
    if (!orderOk(offsets, groups, n)) return STAR_EXIT_BUG;
    memset(unmark, 0, n);
    for (uint64_t g0 = 0; g0 < n;) {
        uint64_t g1 = g0;
        while (g1 < n && groups[g1] == groups[g0]) g1++;
        std::vector<uint64_t> aD;   // members of the group in file order, then in name order (:206)
        for (uint64_t i = g0; i < g1; i++) aD.push_back(i);
        auto rec = [&](uint64_t i) { return Ref{bytes + offsets[i]}; };
        std::stable_sort(aD.begin(), aD.end(), [&](uint64_t a, uint64_t b) { return funCompareNames(rec(a), rec(b)) < 0; });
        const uint64_t nP = aD.size() / 2;
        // the inputs on which the reference is undefined, and the AS it needs: the first (kind, member) of the group
        uint64_t err = ~0ULL;
        auto note = [&](uint32_t kind, uint64_t i) { err = std::min<uint64_t>(err, (uint64_t)kind << 32 | i); };
        for (uint64_t i = g0; i < g1; i++) if (!cigarOk(rec(i))) note(DD_ERR_CIGAR, i);
        std::vector<int> as(nP);
        for (uint64_t p = 0; p < nP; p++) {
            if (N > rec(aD[2 * p + 1]).w(5)) note(DD_ERR_MATE2N, aD[2 * p + 1]);
            const int r = auxAS(bytes + offsets[aD[2 * p]], as[p]);
            if (r == 2) note(DD_ERR_AUX, aD[2 * p]);
            else if (r == 1) note(DD_ERR_AS_MISSING, aD[2 * p]);
            else if (as[p] <= -999) note(DD_ERR_AS_LOW, aD[2 * p]);
        }
        if (err != ~0ULL) return dedupReportError(unmark, n, err & 0xffffffffULL, (uint32_t)(err >> 32));
        std::vector<uint64_t> pr(nP);   // pairs, sorted (:207)
        for (uint64_t p = 0; p < nP; p++) pr[p] = p;
        auto cmp = [&](uint64_t a, uint64_t b) {
            return funCompareCoordFlagCigarSeq(rec(aD[2 * a]), rec(aD[2 * a + 1]), rec(aD[2 * b]), rec(aD[2 * b + 1]), N);
        };
        std::stable_sort(pr.begin(), pr.end(), [&](uint64_t a, uint64_t b) { return cmp(a, b) < 0; });
        int bScore = -999;
        uint64_t bP = 0;
        for (uint64_t q = 0; q < nP; q++) {   // :209-237
            if (as[pr[q]] > bScore) { bScore = as[pr[q]]; bP = q; }
            if (q == nP - 1 || cmp(pr[q], pr[q + 1]) != 0) {
                unmark[aD[2 * pr[bP]]] ^= 1;
                unmark[aD[2 * pr[bP] + 1]] ^= 1;
                bScore = -999;
            }
        }
        g0 = g1;
    }
    return 0;
}
void dedup_oracle_close(void* h) { delete (Oracle*)h; }

int dedup_emul_open(void** h, int, uint64_t mate2basesN) {
    Emul* e = new Emul;
    e->mate2N = mate2basesN > 0xffffffffULL ? 0xffffffffu : (u32)mate2basesN;
    e->maxM = std::max<u64>(1, envU64("STAR_B200_DEDUP_BATCH_RECS", 1u << 20));
    e->hashBits = (u32)std::min<u64>(64, envU64("STAR_B200_DEDUP_HASH_BITS", 64));
    *h = e;
    return 0;
}
int dedup_emul_batch(void* h, const uint8_t* bytes, const uint64_t* offsets, const uint32_t* groups, uint64_t n, uint8_t* unmark, float* ms) {
    Emul* e = (Emul*)h;
    if (ms) *ms = 0;
    if (!orderOk(offsets, groups, n)) return STAR_EXIT_BUG;
    memset(unmark, 0, n);
    if (n == 0) return 0;
    u64 errMember = 0;
    u32 errKind = 0;
    const int rc = dedupBatchRun(e->bufs, bytes, offsets, groups, n, e->mate2N, e->hashBits, e->maxM, unmark, errMember, errKind);
    if (rc == 3) return STAR_EXIT_MEMORY_ALLOCATION;
    if (rc == 1) return dedupReportError(unmark, n, errMember, errKind);
    return 0;
}
void dedup_emul_close(void* h) { Emul* e = (Emul*)h; e->bufs.release(); delete e; }

#pragma GCC visibility pop
}  // extern "C"
