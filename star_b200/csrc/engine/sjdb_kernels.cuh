// sjdb_kernels.cuh — device part of the on-the-fly junction insertion (SURVEY.md §8f N3; reference source/sjdbBuildIndex.cpp).
//
//   sjdb_search_kernel   one thread per suffix of the junction inserts (both strands): the SA row in front of which the suffix has to
//                        be inserted = suffixArraySearch1 (SuffixArrayFuns.cpp:309-351) with compareSeqToGenome1 (:233-306): a binary
//                        search over the whole SA in which a spacer (code 5) of the insert sorts behind the genome's (compareRefEnds,
//                        :221-231, with gInsert = -1: new rows always go behind equal old ones).
//   sjdb_merge_sa_kernel one thread per 64 rows of the NEW suffix array (= GstrandBit+1 whole 64-bit words, so no two threads share a
//                        word), a warp's 32 groups staged in shared memory and stored coalesced: old rows are re-based (reverse-strand coordinates grow with the genome, rows of old inserts move with
//                        their junction's new index) and the sorted new rows are spliced in (sjdbBuildIndex.cpp:141-214).
//                        HBM-bound: reads nSA x (GstrandBit+1)/8 bytes, writes as much plus the new rows.
// Both are grid-stride loops, so that the host emulation (oracle/engine_emul.cpp) can run them as one CTA.
#pragma once
#include "dev.cuh"

namespace starb {

struct SjdbIndex {
    const u8* G;       // base 0 of the old genome, 256 bytes of code 5 readable on both sides
    const u64* SA;     // packed words of the old suffix array
    u64 nGenome, nSA;
    u32 GstrandBit, saBits;
};

// What suffixArraySearch1 is called with besides the text: N = most bases compared, gInsert / strR = where the text goes in the genome and
// its strand, which decide a tie at a spacer (compareRefEnds, SuffixArrayFuns.cpp:210-220).  Junction inserts: N = 10000, gInsert = -1,
// strR = true (sjdbBuildIndex.cpp:80); added references: N = 10000, gInsert = nG, strR = forward half (insertSeqSA.cpp:84).
struct SaSearch1 {
    u64 N, gInsert;
    bool strR;
};

// compareRefEnds with the genome length of the index searched
__device__ __forceinline__ int compareRefEnds(const SjdbIndex& ix, const SaSearch1& q, u64 SAstr, bool dirG) {
    if (dirG) return q.strR ? (SAstr < q.gInsert ? 1 : -1) : 1;
    return q.strR ? -1 : (q.gInsert == ~0ULL ? -1 : (SAstr < ix.nGenome - q.gInsert ? 1 : -1));
}

// compareSeqToGenome1 (SuffixArrayFuns.cpp:233-295) from offset L on: +1 / -1 = the insert suffix s sorts behind / in front of SA row iSA;
// Lout = common length.  Lout = q.N (no difference in N bases) leaves compRes as it was, as the reference does.
__device__ __forceinline__ void sjdbCompare(const SjdbIndex& ix, const SaSearch1& q, const u8* __restrict__ s, u64 L, u64 iSA, u64& Lout, int& compRes) {
    u64 SAstr = packedGet(ix.SA, ix.saBits, iSA);
    const bool dirG = (SAstr >> ix.GstrandBit) == 0;
    SAstr &= ~(1ULL << ix.GstrandBit);
    if (dirG) {
        const u8* g = ix.G + SAstr;
#pragma unroll 1
        for (u64 ii = L; ii < q.N; ii++) {
            const u8 a = SB_LDG(s + ii), b = SB_LDG(g + ii);
            if (a != b) { Lout = ii; compRes = a > b ? 1 : -1; return; }
            if (a == 5) { Lout = ii; compRes = compareRefEnds(ix, q, SAstr, true); return; }
        }
    } else {   // row on the reverse strand: the genome is read backwards and complemented
        const u8* g = ix.G + (ix.nGenome - 1 - SAstr);
#pragma unroll 1
        for (u64 ii = L; ii < q.N; ii++) {
            const u8 a = SB_LDG(s + ii);
            u8 b = SB_LDG(g - (i64)ii);
            if (b < 4) b = 3 - b;
            if (a != b) { Lout = ii; compRes = a > b ? 1 : -1; return; }
            if (a == 5) { Lout = ii; compRes = compareRefEnds(ix, q, SAstr, false); return; }
        }
    }
    Lout = q.N;
}

// suffixArraySearch1 with i1 = 0, i2 = nSA-1, L = 0 (SuffixArrayFuns.cpp:297-351).  A probe that matches N bases returns its row at once,
// not the sorted position.  (compRes starts at 0 where the reference leaves it uninitialised: only an N-base match with row 0 reads it.)
__device__ __forceinline__ u64 sjdbSearchOne(const SjdbIndex& ix, const SaSearch1& q, const u8* __restrict__ s) {
    u64 L1, L2, L3;
    int compRes = 0;
    sjdbCompare(ix, q, s, 0, 0, L1, compRes);
    if (compRes < 0) return 0;
    sjdbCompare(ix, q, s, 0, ix.nSA - 1, L2, compRes);
    if (compRes > 0) return ~0ULL - 1;   // behind the last row
    u64 i1 = 0, i2 = ix.nSA - 1, L = L1 < L2 ? L1 : L2;
#pragma unroll 1
    while (i1 + 1 < i2) {
        const u64 i3 = i1 / 2 + i2 / 2 + (i1 % 2 + i2 % 2) / 2;   // medianUint2
        sjdbCompare(ix, q, s, L, i3, L3, compRes);
        if (L3 == q.N) return i3;
        if (compRes > 0) { i1 = i3; L1 = L3; }
        else if (compRes < 0) { i2 = i3; L2 = L3; }
        L = L1 < L2 ? L1 : L2;
    }
    return i2;
}

static __global__ void __launch_bounds__(256) sjdb_search_kernel(const SjdbIndex ix, const u8* __restrict__ Gsj, u64 nSeq, u64 sjdbLength,
                                                          const u8* __restrict__ skipSeq, u64* __restrict__ indArray) {
    const u64 nSuf = nSeq * sjdbLength;
#pragma unroll 1
    for (u64 k = (u64)blockIdx.x * blockDim.x + threadIdx.x; k < nSuf; k += (u64)gridDim.x * blockDim.x) {
        const u64 q = k / sjdbLength;
        u64 row = ~0ULL;                                                     // no row: junction already in the index, or suffix starts with N / spacer
        if (!SB_LDG(skipSeq + q) && SB_LDG(Gsj + k) <= 3) row = sjdbSearchOne(ix, SaSearch1{10000, ~0ULL, true}, Gsj + k);
        indArray[2 * k] = row;
        indArray[2 * k + 1] = k;
    }
}

struct SjdbMerge;
__device__ __forceinline__ u64 sjdbRebase(const SjdbMerge& m, u64 ind1, u64 N2bit);

struct SjdbMerge {
    const u64* insRow;    // nInd: row of the NEW array every inserted suffix lands in (strictly increasing)
    const u64* insVal;    // nInd: its packed value
    u64 nInd, nSAnew;
    u64 nGenomeOld, nGenomeNew, sjGstart, sjdbLength, sjdbNold, nGsjNew;
    const u32* oldSJind;  // new index of old junction j
    __device__ __forceinline__ u64 rebase(u64 ind1, u64 N2bit) const { return sjdbRebase(*this, ind1, N2bit); }
};

// an old row in the coordinates of the new index (sjdbBuildIndex.cpp:163-187)
__device__ __forceinline__ u64 sjdbRebase(const SjdbMerge& m, u64 ind1, u64 N2bit) {
    if (ind1 & N2bit) {
        u64 ind1s = m.nGenomeOld - (ind1 & ~N2bit);
        if (ind1s >= m.sjGstart) {   // inside an old insert: moves with its junction
            const u64 sj1 = (ind1s - m.sjGstart) / m.sjdbLength;
            if (sj1 < m.sjdbNold) ind1s += ((u64)SB_LDG(m.oldSJind + sj1) - sj1) * m.sjdbLength;
            ind1 = (m.nGenomeNew - ind1s) | N2bit;
        } else ind1 += m.nGsjNew;    // reverse-strand coordinates count from the (longer) end
    } else if (ind1 >= m.sjGstart) {
        const u64 sj1 = (ind1 - m.sjGstart) / m.sjdbLength;
        if (sj1 < m.sjdbNold) ind1 += ((u64)SB_LDG(m.oldSJind + sj1) - sj1) * m.sjdbLength;
    }
    return ind1;
}

// Merge = SjdbMerge, or any type with the same insRow / insVal / nInd / nSAnew members and its own rebase() of an old row.
// Tile = 32 groups of 64 rows per warp: every lane packs its group into the warp's shared-memory tile (same layout as the global
// array: group after group, `bits` words each), then the warp stores the tile with consecutive 8-byte words per lane (256 B per
// store instruction instead of 32 stores 8*bits bytes apart).  Dynamic shared memory: (blockDim.x/32) * 32 * bits * 8 bytes.
template <class Merge>
__global__ void __launch_bounds__(128) sjdb_merge_sa_kernel(const SjdbIndex ix, const Merge m, u64* __restrict__ SAnew) {
    extern __shared__ u8 smem[];
    const u32 bits = ix.saBits;
    const u32 lane = threadIdx.x & 31;
    u64* tile = (u64*)smem + (u64)(threadIdx.x >> 5) * 32 * bits;
    const u64 N2bit = 1ULL << ix.GstrandBit;
    const u64 nGroups = (m.nSAnew + 63) / 64;
    const u64 nWarps = ((u64)gridDim.x * blockDim.x) >> 5;
#pragma unroll 1
    for (u64 t = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5; t * 32 < nGroups; t += nWarps) {
        const u64 g = t * 32 + lane;
        if (g < nGroups) {
            const u64 r0 = g * 64;
            u64 lo = 0, hi = m.nInd;            // j = number of inserted rows in front of r0
            while (lo < hi) { const u64 mid = (lo + hi) >> 1; if (SB_LDG(m.insRow + mid) < r0) lo = mid + 1; else hi = mid; }
            u64 j = lo;
            u64 nextIns = j < m.nInd ? SB_LDG(m.insRow + j) : ~0ULL;
            u64* out = tile + (u64)lane * bits;
            u64 acc = 0;
            u32 sh = 0;
#pragma unroll 1
            for (u32 e = 0; e < 64; e++) {
                const u64 r = r0 + e;
                u64 val = 0;
                if (r < m.nSAnew) {
                    if (r == nextIns) { val = SB_LDG(m.insVal + j); j++; nextIns = j < m.nInd ? SB_LDG(m.insRow + j) : ~0ULL; }
                    else val = m.rebase(packedGet(ix.SA, bits, r - j), N2bit);
                }
                acc |= val << sh;
                if (sh + bits >= 64) {
                    *out++ = acc;
                    acc = sh + bits > 64 ? val >> (64 - sh) : 0;
                }
                sh = (sh + bits) & 63;
            }
        }
        __syncwarp();
        const u64 rows = nGroups - t * 32 < 32 ? nGroups - t * 32 : 32;
        u64* dst = SAnew + t * 32 * bits;
        for (u64 k = lane; k < rows * bits; k += 32) dst[k] = tile[k];
        __syncwarp();
    }
}

// Host side of the merge launch: where every inserted suffix lands in the new array and what the row holds
// (sjdbBuildIndex.cpp:143-152, 191-199).  indSorted = nInd sorted (row, offset in Gsj) pairs; rows behind the last old one are appended.
// An offset in the reverse half is a reverse-strand position counted from revBase (0 for junctions; insertSeqSA.cpp:158-199: nG2).
inline void sjdbInsertedRows(const uint64_t* indSorted, u64 nInd, u64 nSAold, u64 nGsj, u64 sjGstart, u32 GstrandBit, u64* row, u64* val, u64 revBase = 0) {
    const u64 N2bit = 1ULL << GstrandBit;
    for (u64 j = 0; j < nInd; j++) {
        const u64 r = indSorted[2 * j] < nSAold ? indSorted[2 * j] : nSAold;
        row[j] = r + j;
        const u64 ind1 = indSorted[2 * j + 1];
        val[j] = ind1 < nGsj ? ind1 + sjGstart : ((ind1 - nGsj + revBase) | N2bit);
    }
}

}  // namespace starb
