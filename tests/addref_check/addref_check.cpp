// addref_check.cpp — TEST INFRASTRUCTURE ONLY: two CPU implementations of star_gpu_addref_open / _search / _merge_sa / _close
// (include/star_b200.h) that the tests compare the product against.
//
//   addref_oracle_*   the reference's own loops, sequential: the row loop of insertSeqSA.cpp:33-51, suffixArraySearch1 /
//                     compareSeqToGenome1 / compareRefEnds (SuffixArrayFuns.cpp:210-351) per suffix with the text and its complement as two
//                     arrays (insertSeqSA.cpp:53-87), and the two-pointer sweep of insertSeqSA.cpp:158-199
//   addref_oracle_sort  qsort with funCompareUintAndSuffixesMemcmp (funCompareUintAndSuffixesMemcmp.cpp:7-33) over the reference's buffer
//   addref_emul_*     the UNMODIFIED kernels of star_b200/csrc/engine/addref_kernels.cuh compiled as host code through oracle/cuda_host_shim.h:
//                     every launch is one emulated CTA of host threads, around them what addref.cu does on the host
// Built with hidden visibility and -Bsymbolic (tests/addref_check/Makefile), like tests/dedup_check.
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

#include "../../star_b200/csrc/engine/addref_kernels.cuh"

namespace starb {
alignas(128) u8 smem[256 * 1024];   // dynamic shared memory of the (single) emulated CTA

// one CTA of nThreads host threads executing `body` (warps meet at the shim's per-warp barriers)
static void runCta(unsigned nThreads, const std::function<void()>& body) {
    cuda_shim::CtaShared c;
    c.nThreads = nThreads;
    pthread_barrier_init(&c.bar, nullptr, nThreads);
    for (unsigned w = 0; w < (nThreads + 31) / 32; w++) {
        pthread_barrier_init(&c.warp[w].bar, nullptr, 32);
        for (int g = 0; g < 4; g++)
            for (int k = 0; k < 16; k++) pthread_barrier_init(&c.warp[w].gbar[g][k], nullptr, 2u << g);
    }
    std::vector<std::thread> th;
    for (unsigned t = 0; t < nThreads; t++)
        th.emplace_back([&, t] {
            cuda_shim::tIdx = {t, 0, 0}; cuda_shim::bIdx = {0, 0, 0}; cuda_shim::bDim = {nThreads, 1, 1}; cuda_shim::gDim = {1, 1, 1};
            cuda_shim::cta = &c;
            body();
        });
    for (auto& t : th) t.join();
    for (unsigned w = 0; w < (nThreads + 31) / 32; w++) {
        pthread_barrier_destroy(&c.warp[w].bar);
        for (int g = 0; g < 4; g++)
            for (int k = 0; k < 16; k++) pthread_barrier_destroy(&c.warp[w].gbar[g][k]);
    }
    pthread_barrier_destroy(&c.bar);
}
}  // namespace starb

using namespace starb;

namespace {
// ---- restatement ----------------------------------------------------------------------------------------------------------------
struct AddrefOracle {
    std::vector<uint8_t> G;    // 256 + nGenome + 256 bytes of the grown genome
    std::vector<uint8_t> SA;   // the old rows, re-based in open
    uint64_t nGenome, nSA, nG, nG1, nG2;
    uint32_t GstrandBit;
    uint64_t get(uint64_t i) const {   // PackedArray.h:24-32
        const uint64_t b = i * (GstrandBit + 1);
        uint64_t w;
        memcpy(&w, SA.data() + b / 8, 8);
        return (w >> (b % 8)) & (~0ULL >> (64 - (GstrandBit + 1)));
    }
    void put(uint64_t i, uint64_t x) {   // PackedArray::writePacked
        const uint64_t b = i * (GstrandBit + 1), S = b % 8, mask = ~0ULL >> (64 - (GstrandBit + 1));
        uint64_t w;
        memcpy(&w, SA.data() + b / 8, 8);
        w = (w & ~(mask << S)) | (x << S);
        memcpy(SA.data() + b / 8, &w, 8);
    }
    const uint8_t* g() const { return G.data() + 256; }
    int compareRefEnds(uint64_t SAstr, uint64_t gInsert, bool strG, bool strR) const {   // SuffixArrayFuns.cpp:210-220
        if (strG) return strR ? (SAstr < gInsert ? 1 : -1) : 1;
        return strR ? -1 : (gInsert == (uint64_t)-1 ? -1 : (SAstr < nGenome - gInsert ? 1 : -1));
    }
    // compareSeqToGenome1, SuffixArrayFuns.cpp:223-295
    uint64_t compare1(const uint8_t* const* s2, uint64_t S, uint64_t N, uint64_t L, uint64_t iSA, bool dirR, uint64_t gInsert, int& compRes) const {
        uint64_t SAstr = get(iSA);
        const bool dirG = (SAstr >> GstrandBit) == 0;
        SAstr &= ~(1ULL << GstrandBit);
        if (dirG) {
            const uint8_t* s = s2[0] + S + L;
            const uint8_t* gg = g() + SAstr + L;
            for (uint64_t ii = 0; ii < N - L; ii++) {
                if (s[ii] != gg[ii]) { compRes = s[ii] > gg[ii] ? 1 : -1; return ii + L; }
                else if (s[ii] == 5) { compRes = compareRefEnds(SAstr, gInsert, dirG, dirR); return ii + L; }
            }
            return N;
        }
        const uint8_t* s = s2[1] + S + L;
        const uint8_t* gg = g() + nGenome - 1 - SAstr - L;
        for (uint64_t ii = 0; ii < N - L; ii++) {
            if (s[ii] != *(gg - ii)) {
                uint8_t a = s[ii], b = *(gg - ii);
                if (a < 4) a = 3 - a;
                if (b < 4) b = 3 - b;
                compRes = a > b ? 1 : -1;
                return ii + L;
            } else if (s[ii] == 5) { compRes = compareRefEnds(SAstr, gInsert, dirG, dirR); return ii + L; }
        }
        return N;
    }
    // suffixArraySearch1, SuffixArrayFuns.cpp:297-351
    uint64_t search1(const uint8_t* const* s2, uint64_t S, uint64_t N, uint64_t gInsert, bool strR) const {
        int compRes = 0;   // (uninitialised in the reference: only read after an N-base match with row 0)
        uint64_t i1 = 0, i2 = nSA - 1;
        uint64_t L1 = compare1(s2, S, N, 0, i1, strR, gInsert, compRes);
        if (compRes < 0) return 0;
        uint64_t L2 = compare1(s2, S, N, 0, i2, strR, gInsert, compRes);
        if (compRes > 0) return (uint64_t)-2;
        uint64_t L = std::min(L1, L2);
        while (i1 + 1 < i2) {
            const uint64_t i3 = i1 / 2 + i2 / 2 + (i1 % 2 + i2 % 2) / 2;   // medianUint2
            const uint64_t L3 = compare1(s2, S, N, L, i3, strR, gInsert, compRes);
            if (L3 == N) return i3;
            if (compRes > 0) { i1 = i3; L1 = L3; } else if (compRes < 0) { i2 = i3; L2 = L3; }
            L = std::min(L1, L2);
        }
        return i2;
    }
};

const uint8_t* g_sortBase;
uint64_t g_sortEnd;
int sortCompare(const void* a, const void* b) {   // funCompareUintAndSuffixesMemcmp.cpp:7-33, bounded at the buffer's end
    const uint64_t* va = (const uint64_t*)a;
    const uint64_t* vb = (const uint64_t*)b;
    if (va[0] > vb[0]) return 1;
    if (va[0] < vb[0]) return -1;
    int comp = memcmp(g_sortBase + va[1], g_sortBase + vb[1], g_sortEnd - std::max(va[1], vb[1]));
    if (comp == 0) comp = va[1] > vb[1] ? 1 : -1;
    return comp;
}

// ---- emulation ------------------------------------------------------------------------------------------------------------------
struct AddrefHost {
    std::vector<u8> g;
    std::vector<u64> sa;
    SjdbIndex ix;
    u64 nG, nG1, nG2;
};
}  // namespace

extern "C" {
#pragma GCC visibility push(default)

int addref_oracle_open(void** h, int, const star_index_view_t* v, uint64_t nG, uint64_t nG1, uint64_t nG2, float* ms) {
    if (nG + nG1 + nG2 != v->nGenome) return STAR_EXIT_BUG;
    AddrefOracle* o = new AddrefOracle;
    o->G.assign(v->G - 256, v->G + v->nGenome + 256);
    o->SA.assign(v->SA, v->SA + v->nSAbyte);
    o->SA.resize(v->nSAbyte + 16, 0);
    o->nGenome = v->nGenome; o->nSA = v->nSA; o->GstrandBit = v->GstrandBit; o->nG = nG; o->nG1 = nG1; o->nG2 = nG2;
    const uint64_t N2bit = 1ULL << o->GstrandBit, strandMask = ~N2bit;
    for (uint64_t isa = 0; isa < o->nSA; isa++) {   // insertSeqSA.cpp:33-51
        const uint64_t ind1 = o->get(isa);
        if ((ind1 & N2bit) > 0) {
            if ((ind1 & strandMask) >= nG2) o->put(isa, ind1 + nG1);
        } else if (ind1 >= nG) o->put(isa, ind1 + nG1);
    }
    if (ms) *ms = 0;
    *h = o;
    return 0;
}

int addref_oracle_search(void* h, const uint8_t* seq, uint64_t* indArray, float* ms) {
    const AddrefOracle* o = (const AddrefOracle*)h;
    const uint64_t nG1 = o->nG1, L16 = 16;
    std::vector<uint8_t> seqq(4 * nG1 + 3 * L16, 5);   // insertSeqSA.cpp:53-70
    const uint8_t* seq1[2] = {seqq.data() + L16, seqq.data() + 2 * L16 + 2 * nG1};
    memcpy(seqq.data() + L16, seq, 2 * nG1);
    for (uint64_t ii = 0; ii < 2 * nG1; ii++) seqq[2 * L16 + 2 * nG1 + ii] = seq[ii] < 4 ? 3 - seq[ii] : seq[ii];   // complementSeqNumbers
    for (uint64_t ii = 0; ii < 2 * nG1; ii++) {   // :76-87
        if (seq1[0][ii] > 3) indArray[ii * 2] = (uint64_t)-1;
        else indArray[ii * 2] = o->search1(seq1, ii, 10000, o->nG, ii < nG1);
        indArray[ii * 2 + 1] = ii;
    }
    if (ms) *ms = 0;
    return 0;
}

int addref_oracle_merge_sa(void* h, const uint64_t* ind, uint64_t nInd, uint8_t* SAnew, uint64_t nSAnewByte, float* ms) {
    const AddrefOracle* o = (const AddrefOracle*)h;
    const uint32_t bits = o->GstrandBit + 1;
    const uint64_t mask = ~0ULL >> (64 - bits), N2bit = 1ULL << o->GstrandBit;
    std::vector<uint8_t> buf(nSAnewByte + 16, 0);
    auto put = [&](uint64_t jj, uint64_t x) {
        const uint64_t b = jj * bits, S = b % 8;
        uint64_t w;
        memcpy(&w, buf.data() + b / 8, 8);
        w = (w & ~(mask << S)) | (x << S);
        memcpy(buf.data() + b / 8, &w, 8);
    };
    auto value = [&](uint64_t ind1) { return ind1 < o->nG1 ? ind1 + o->nG : ((ind1 - o->nG1 + o->nG2) | N2bit); };
    uint64_t isa1 = 0, isa2 = 0;   // :158-199
    for (uint64_t isa = 0; isa < o->nSA; isa++) {
        while (isa1 < nInd && isa == ind[isa1 * 2]) { put(isa2, value(ind[isa1 * 2 + 1])); ++isa2; ++isa1; }
        put(isa2, o->get(isa));
        ++isa2;
    }
    for (; isa1 < nInd; isa1++) { put(isa2, value(ind[isa1 * 2 + 1])); ++isa2; }
    memcpy(SAnew, buf.data(), nSAnewByte);
    if (ms) *ms = 0;
    return 0;
}

void addref_oracle_close(void* h) { delete (AddrefOracle*)h; }

// seq = the 2*nG1 bytes of seq1[0]; ind = nInd (row, offset) pairs, sorted in place
int addref_oracle_sort(const uint8_t* seq, uint64_t nG1, uint64_t* ind, uint64_t nInd) {
    std::vector<uint8_t> seqq(4 * nG1 + 48, 5);
    memcpy(seqq.data() + 16, seq, 2 * nG1);
    for (uint64_t ii = 0; ii < 2 * nG1; ii++) seqq[32 + 2 * nG1 + ii] = seq[ii] < 4 ? 3 - seq[ii] : seq[ii];
    g_sortBase = seqq.data() + 16;
    g_sortEnd = 4 * nG1 + 32;
    qsort(ind, nInd, 2 * sizeof(uint64_t), sortCompare);
    return 0;
}

int addref_emul_open(void** h, int, const star_index_view_t* v, uint64_t nG, uint64_t nG1, uint64_t nG2, float* ms) {
    if (nG + nG1 + nG2 != v->nGenome) return STAR_EXIT_BUG;
    AddrefHost* H = new AddrefHost;
    const u32 bits = v->GstrandBit + 1;
    H->g.assign(v->G - 256, v->G + v->nGenome + 256);
    H->sa.assign((v->nSA + 63) / 64 * bits + 2, 0);
    memcpy(H->sa.data(), v->SA, v->nSAbyte);
    H->ix.G = H->g.data() + 256; H->ix.SA = H->sa.data(); H->ix.nGenome = v->nGenome; H->ix.nSA = v->nSA; H->ix.GstrandBit = v->GstrandBit; H->ix.saBits = bits;
    H->nG = nG; H->nG1 = nG1; H->nG2 = nG2;
    const AddrefRebase a{v->nSA, nG, nG1, nG2, v->GstrandBit, bits};
    runCta(128, [&] { addref_rebase_kernel(a, H->sa.data()); });
    if (ms) *ms = 0;
    *h = H;
    return 0;
}

int addref_emul_search(void* h, const uint8_t* seq, uint64_t* indArray, float* ms) {
    AddrefHost* H = (AddrefHost*)h;
    const u64 nSuf = 2 * H->nG1;
    std::vector<u8> text(nSuf + 272, 5);
    memcpy(text.data(), seq, nSuf);
    runCta(256, [&] { addref_search_kernel(H->ix, text.data(), H->nG, H->nG1, (u64*)indArray); });
    if (ms) *ms = 0;
    return 0;
}

int addref_emul_merge_sa(void* h, const uint64_t* indSorted, uint64_t nInd, uint8_t* SAnew, uint64_t nSAnewByte, float* ms) {
    AddrefHost* H = (AddrefHost*)h;
    const u64 nSAnew = H->ix.nSA + nInd;
    std::vector<u64> row(nInd + 1), val(nInd + 1);
    sjdbInsertedRows(indSorted, nInd, H->ix.nSA, H->nG1, H->nG, H->ix.GstrandBit, row.data(), val.data(), H->nG2);
    std::vector<u64> out((nSAnew + 63) / 64 * H->ix.saBits + 2, 0);
    const AddrefMerge m{row.data(), val.data(), nInd, nSAnew};
    runCta(128, [&] { sjdb_merge_sa_kernel(H->ix, m, out.data()); });
    if (nSAnewByte > out.size() * 8) return STAR_EXIT_BUG;
    memcpy(SAnew, out.data(), nSAnewByte);
    if (ms) *ms = 0;
    return 0;
}

void addref_emul_close(void* h) { delete (AddrefHost*)h; }

#pragma GCC visibility pop
}  // extern "C"
