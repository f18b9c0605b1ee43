// dedup_kernels.cuh — duplicate pairs of --bamRemoveDuplicatesType (reference source/bamRemoveDuplicates.cpp:13-112, 206-237) for a batch of
// whole groups.
//
// The host hands over the NH == 1 members of consecutive groups in file order (record bytes, offset and group of every member).  Per batch:
//   dedup_decode_kernel    one thread per member: CIGAR contract (1..100 operations, not only S), name length and the 0x80 bit
//   dedup_namekey_kernel   the key of one LSD pass, gathered through the current order: the 0x80 bit, a name word (big-endian, every byte
//   (stable radix sort)    XOR 0x80: signed char order), last word first, then (group, l_read_name).  The passes start from file order, so
//                          equal names keep file order, as the stable qsort of funCompareNames does
//   dedup_pairflag_kernel  pair heads: every even position of a group that has a successor in the group ((0,1), (2,3), ...)
//   (select)               pair list, in (group, name) order
//   dedup_pairkey_kernel   one thread per pair: 64-bit hash of what funCompareCoordFlagCigarSeq compares, AS of the first record, the
//                          N <= l_seq and AS > -999 contract
//   (two stable sorts)     by hash, then by group: the pairs of a (group, hash) run stay in name order
//   dedup_runhead_kernel   run heads; a max-scan gives every pair its head
//   dedup_runcheck_kernel  every pair compared exactly with its head; a mismatch marks the run as a hash collision
//   dedup_resplit_kernel   class representative = the head, or in a collided run the first earlier pair of the run that is exactly equal
//   dedup_best_kernel      per class the maximum of (AS, -pair index) by a 64-bit atomic max: highest AS, ties to the first in name order
//   dedup_unmark_kernel    the winning pair of every class flags both of its records
// Errors go to one 64-bit word by atomic min of (group, kind, member), so the first group in file order reports, and within it the kind
// the reference would meet first.  All kernels are grid-stride loops; dedupBatchRun is compiled with the DD_* primitives of dedup.cu (cub,
// CUDA runtime) or of the host emulation (tests/dedup_check/dedup_check.cpp).
#pragma once
#include <string.h>

#include <vector>

#include "dev.cuh"

namespace starb {

// error kinds, in the order the reference meets them inside one group (CIGAR and sequence reads in the sorts, then the AS loop)
enum { DD_ERR_CIGAR = 0, DD_ERR_MATE2N = 1, DD_ERR_AUX = 2, DD_ERR_AS_MISSING = 3, DD_ERR_AS_LOW = 4 };
static const u64 DD_NO_ERROR = ~0ULL;

struct DdBatch {
    const u8* recs;          // record bytes
    const u64* moff;         // per member: offset of its record (block_size field) in recs
    const u32* grp;          // per member: group index within the batch (non-decreasing)
    u64 n;                   // members
    u32 mate2N, hashBits;
    u32* perm;               // name order -> member
    u8* meta;                // per member: l_read_name
    u64* err;                // first error (atomic min), DD_NO_ERROR if none
};

__host__ __device__ __forceinline__ u32 ddRd32(const u8* p) { return (u32)p[0] | (u32)p[1] << 8 | (u32)p[2] << 16 | (u32)p[3] << 24; }
__host__ __device__ __forceinline__ u32 ddRd16(const u8* p) { return (u32)p[0] | (u32)p[1] << 8; }

struct DdRec {   // the fields of one record that the comparison reads
    const u8* r;
    u32 pos, flag, lName, nCig, lSeq;
    __device__ __forceinline__ explicit DdRec(const u8* p) : r(p) {
        pos = ddRd32(p + 8); lName = p[12]; nCig = ddRd16(p + 16); flag = ddRd16(p + 18); lSeq = ddRd32(p + 20);
    }
    __device__ __forceinline__ u32 cig(u32 k) const { return ddRd32(r + 36 + lName + 4 * k); }
    __device__ __forceinline__ bool lead() const { return nCig > 0 && (cig(0) & 15) == 4; }
    __device__ __forceinline__ bool trail() const { return nCig > 0 && (cig(nCig - 1) & 15) == 4; }
    // funCigarExtendS: a leading S is added to the next operation, a trailing S to the one before it
    __device__ __forceinline__ int extN() const { return (int)nCig - (int)lead() - (int)trail(); }
    __device__ __forceinline__ bool cigarOk() const { return nCig >= 1 && nCig <= 100 && extN() >= 1; }
    __device__ __forceinline__ u32 extWord(u32 k) const {
        const u32 l = lead(), n1 = (u32)extN();
        u32 w = cig(k + l);
        if (k == 0 && l) w += (cig(0) >> 4) << 4;
        if (k == n1 - 1 && trail()) w += (cig(nCig - 1) >> 4) << 4;
        return w;
    }
    __device__ __forceinline__ u32 startExtS() const { return lead() ? pos - (cig(0) >> 4) : pos; }   // funStartExtendS (uint32)
    // the sequence nibbles the reference compares for a second mate: the first N (forward), or from l_seq-N up to the end of the last
    // byte (reverse; for an odd l_seq that includes the pad nibble, even for N = 0)
    __device__ __forceinline__ void nibRange(u32 N, u32& a, u32& e) const {
        if (flag & 0x10) { a = lSeq - N; e = (lSeq + 1) & ~1u; } else { a = 0; e = N; }
    }
    __device__ __forceinline__ u32 nib(u32 i) const {
        const u8 b = r[36 + lName + 4 * nCig + i / 2];
        return i & 1 ? b & 15 : b >> 4;
    }
};

__device__ __forceinline__ u64 ddMix(u64 h, u64 v) {   // splitmix64 finaliser of h ^ v
    h ^= v + 0x9E3779B97F4A7C15ULL + (h << 6) + (h >> 2);
    h ^= h >> 30; h *= 0xBF58476D1CE4E5B9ULL;
    h ^= h >> 27; h *= 0x94D049BB133111EBULL;
    return h ^ (h >> 31);
}

// htslib bam_aux_get + bam_aux2i: 0 = found (v = value; a non-integer type reads as 0), 1 = missing, 2 = malformed
__device__ __forceinline__ int ddAuxInt(const u8* rec, u8 t0, u8 t1, int& v) {
    const DdRec R(rec);
    const u8* s = rec + 36 + R.lName + 4ull * R.nCig + (R.lSeq + 1ull) / 2 + R.lSeq;
    const u8* end = rec + 4 + ddRd32(rec);
    v = 0;
    while (s < end) {
        if (end - s < 3) return 2;
        const u8 type = s[2];
        const bool hit = s[0] == t0 && s[1] == t1;
        s += 3;
        const int sz = type == 'A' || type == 'c' || type == 'C' ? 1 : type == 's' || type == 'S' ? 2 : type == 'i' || type == 'I' || type == 'f' ? 4 : type == 'd' ? 8 : 0;
        if (hit) {
            if (end - s < (sz ? sz : 0)) return 2;
            if (type == 'c') v = (int)(signed char)s[0];
            else if (type == 'C') v = s[0];
            else if (type == 's') v = (int)(short)ddRd16(s);
            else if (type == 'S') v = (int)ddRd16(s);
            else if (type == 'i' || type == 'I') v = (int)ddRd32(s);
            return 0;
        }
        if (sz) s += sz;
        else if (type == 'Z' || type == 'H') { while (s < end && *s) ++s; ++s; }
        else if (type == 'B') {
            if (end - s < 5) return 2;
            const u8 sub = s[0];
            const int bs = sub == 'c' || sub == 'C' || sub == 'A' ? 1 : sub == 's' || sub == 'S' ? 2 : sub == 'i' || sub == 'I' || sub == 'f' ? 4 : sub == 'd' ? 8 : 0;
            if (!bs) return 2;
            s += 5 + (u64)ddRd32(s + 1) * bs;
        } else return 2;
    }
    return 1;
}

__device__ __forceinline__ void ddError(const DdBatch& b, u64 member, u32 kind) {
    DD_ATOMIC_MIN_U64(b.err, (u64)b.grp[member] << 35 | (u64)kind << 32 | member);
}

__global__ void __launch_bounds__(256) dedup_decode_kernel(const DdBatch b) {
#pragma unroll 1
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < b.n; i += (u64)gridDim.x * blockDim.x) {
        const DdRec R(b.recs + b.moff[i]);
        if (!R.cigarOk()) ddError(b, i, DD_ERR_CIGAR);
        b.meta[i] = (u8)R.lName;
        b.perm[i] = (u32)i;
    }
}

// pass -1: the 0x80 bit; pass w >= 0: name word w; pass -2: (group, l_read_name)
__global__ void __launch_bounds__(256) dedup_namekey_kernel(const DdBatch b, int pass, u64* __restrict__ keys) {
#pragma unroll 1
    for (u64 k = (u64)blockIdx.x * blockDim.x + threadIdx.x; k < b.n; k += (u64)gridDim.x * blockDim.x) {
        const u32 m = b.perm[k];
        const u8* r = b.recs + b.moff[m];
        u64 key;
        if (pass == -1) key = (ddRd16(r + 18) & 0x80) ? 1 : 0;
        else if (pass == -2) key = (u64)b.grp[m] << 8 | b.meta[m];
        else {
            const u32 l = b.meta[m];
            key = 0;
            for (u32 j = 0; j < 8; j++) {
                const u32 c = (u32)pass * 8 + j;
                key = key << 8 | (c < l ? (u8)(r[36 + c] ^ 0x80) : 0);
            }
        }
        keys[k] = key;
    }
}

__global__ void __launch_bounds__(256) dedup_pairflag_kernel(const DdBatch b, const u32* __restrict__ gStart, u8* __restrict__ flags) {
#pragma unroll 1
    for (u64 k = (u64)blockIdx.x * blockDim.x + threadIdx.x; k < b.n; k += (u64)gridDim.x * blockDim.x) {
        const u32 m = b.perm[k];
        flags[k] = ((k - gStart[m]) % 2 == 0) && k + 1 < b.n && b.grp[b.perm[k + 1]] == b.grp[m];
    }
}

__global__ void __launch_bounds__(256) dedup_pairkey_kernel(const DdBatch b, const u32* __restrict__ pairA, u64 nP, u64* __restrict__ hkey, u32* __restrict__ pidx,
                                                            int* __restrict__ pas) {
#pragma unroll 1
    for (u64 p = (u64)blockIdx.x * blockDim.x + threadIdx.x; p < nP; p += (u64)gridDim.x * blockDim.x) {
        const u32 m1 = b.perm[pairA[p]], m2 = b.perm[pairA[p] + 1];
        const DdRec A(b.recs + b.moff[m1]), B(b.recs + b.moff[m2]);
        u64 h = 0;
        h = ddMix(h, (u64)A.startExtS() << 32 | B.startExtS());
        h = ddMix(h, (u64)(A.flag | 0x400) << 16 | (B.flag | 0x400));
        if (A.cigarOk() && B.cigarOk()) {
            for (const DdRec* R : {&A, &B}) {
                const u32 n1 = (u32)R->extN();
                h = ddMix(h, n1);
                for (u32 k = 0; k < n1; k++) h = ddMix(h, R->extWord(k));
            }
        }
        if ((u64)b.mate2N > B.lSeq) ddError(b, m2, DD_ERR_MATE2N);
        else {
            u32 a, e;
            B.nibRange(b.mate2N, a, e);
            u64 w = 0;
            u32 c = 0;
            for (u32 i = a; i < e; i++) {
                w = w << 4 | B.nib(i);
                if (++c == 16) { h = ddMix(h, w); w = 0; c = 0; }
            }
            h = ddMix(h, w << 8 | c);
        }
        hkey[p] = b.hashBits >= 64 ? h : b.hashBits == 0 ? 0 : h & ((1ULL << b.hashBits) - 1);
        pidx[p] = (u32)p;
        int as = 0;
        const int r = ddAuxInt(A.r, 'A', 'S', as);
        if (r == 2) ddError(b, m1, DD_ERR_AUX);
        else if (r == 1) ddError(b, m1, DD_ERR_AS_MISSING);
        else if (as <= -999) ddError(b, m1, DD_ERR_AS_LOW);
        pas[p] = as;
    }
}

// funCompareCoordFlagCigarSeq == 0, on the pairs p and q (pair heads pairA[.] in name order)
__device__ __forceinline__ bool ddPairEqual(const DdBatch& b, const u32* pairA, u32 p, u32 q) {
    const DdRec A1(b.recs + b.moff[b.perm[pairA[p]]]), A2(b.recs + b.moff[b.perm[pairA[p] + 1]]);
    const DdRec B1(b.recs + b.moff[b.perm[pairA[q]]]), B2(b.recs + b.moff[b.perm[pairA[q] + 1]]);
    if (A1.startExtS() != B1.startExtS() || A2.startExtS() != B2.startExtS()) return false;
    if ((A1.flag | 0x400) != (B1.flag | 0x400) || (A2.flag | 0x400) != (B2.flag | 0x400)) return false;
    if (!A1.cigarOk() || !A2.cigarOk() || !B1.cigarOk() || !B2.cigarOk()) return true;   // (an error is reported for these)
    for (int s = 0; s < 2; s++) {
        const DdRec& X = s ? A2 : A1;
        const DdRec& Y = s ? B2 : B1;
        const u32 n1 = (u32)X.extN();
        if ((u32)Y.extN() != n1) return false;
        for (u32 k = 0; k < n1; k++) if (X.extWord(k) != Y.extWord(k)) return false;
    }
    if ((u64)b.mate2N > A2.lSeq || (u64)b.mate2N > B2.lSeq) return true;
    u32 a, e, c, f;
    A2.nibRange(b.mate2N, a, e);
    B2.nibRange(b.mate2N, c, f);
    if (e - a != f - c) return false;
    for (u32 i = 0; i < e - a; i++) if (A2.nib(a + i) != B2.nib(c + i)) return false;
    return true;
}

__global__ void __launch_bounds__(256) dedup_classgrp_kernel(const DdBatch b, const u32* __restrict__ pairA, const u32* __restrict__ byHash, u64 nP, u64* __restrict__ keys) {
#pragma unroll 1
    for (u64 q = (u64)blockIdx.x * blockDim.x + threadIdx.x; q < nP; q += (u64)gridDim.x * blockDim.x) keys[q] = b.grp[b.perm[pairA[byHash[q]]]];
}

// cls: pair indices in class-sorted order; head[q] = q at a (group, hash) run head, else 0 (max-scanned afterwards)
__global__ void __launch_bounds__(256) dedup_runhead_kernel(const DdBatch b, const u32* __restrict__ pairA, const u32* __restrict__ cls, const u64* __restrict__ hkey,
                                                            u64 nP, u32* __restrict__ head, u8* __restrict__ collided) {
#pragma unroll 1
    for (u64 q = (u64)blockIdx.x * blockDim.x + threadIdx.x; q < nP; q += (u64)gridDim.x * blockDim.x) {
        bool h = q == 0;
        if (!h) {
            const u32 p = cls[q], o = cls[q - 1];
            h = hkey[p] != hkey[o] || b.grp[b.perm[pairA[p]]] != b.grp[b.perm[pairA[o]]];
        }
        head[q] = h ? (u32)q : 0;
        collided[q] = 0;
    }
}

__global__ void __launch_bounds__(256) dedup_runcheck_kernel(const DdBatch b, const u32* __restrict__ pairA, const u32* __restrict__ cls, const u32* __restrict__ head,
                                                             u64 nP, u8* __restrict__ collided) {
#pragma unroll 1
    for (u64 q = (u64)blockIdx.x * blockDim.x + threadIdx.x; q < nP; q += (u64)gridDim.x * blockDim.x)
        if (head[q] != q && !ddPairEqual(b, pairA, cls[q], cls[head[q]])) collided[head[q]] = 1;
}

__global__ void __launch_bounds__(256) dedup_resplit_kernel(const DdBatch b, const u32* __restrict__ pairA, const u32* __restrict__ cls, const u32* __restrict__ head,
                                                            const u8* __restrict__ collided, u64 nP, u32* __restrict__ rep, u64* __restrict__ best) {
#pragma unroll 1
    for (u64 q = (u64)blockIdx.x * blockDim.x + threadIdx.x; q < nP; q += (u64)gridDim.x * blockDim.x) {
        u32 r = head[q];
        if (collided[r])
            while (r < q && !ddPairEqual(b, pairA, cls[r], cls[q])) r++;
        rep[q] = r;
        best[q] = 0;
    }
}

__global__ void __launch_bounds__(256) dedup_best_kernel(const u32* __restrict__ cls, const u32* __restrict__ rep, const int* __restrict__ pas, u64 nP, u64* __restrict__ best) {
#pragma unroll 1
    for (u64 q = (u64)blockIdx.x * blockDim.x + threadIdx.x; q < nP; q += (u64)gridDim.x * blockDim.x) {
        const u32 p = cls[q];
        DD_ATOMIC_MAX_U64(best + rep[q], (u64)((u32)pas[p] ^ 0x80000000u) << 32 | (0xffffffffu - p));
    }
}

__global__ void __launch_bounds__(256) dedup_unmark_kernel(const DdBatch b, const u32* __restrict__ pairA, const u32* __restrict__ cls, const u32* __restrict__ rep,
                                                           const u64* __restrict__ best, u64 nP, u8* __restrict__ unmark) {
#pragma unroll 1
    for (u64 q = (u64)blockIdx.x * blockDim.x + threadIdx.x; q < nP; q += (u64)gridDim.x * blockDim.x) {
        const u32 p = cls[q];
        if ((u32)best[rep[q]] == 0xffffffffu - p) { unmark[b.perm[pairA[p]]] = 1; unmark[b.perm[pairA[p] + 1]] = 1; }
    }
}

#ifdef DD_LAUNCH
// Device buffers of a handle, grown on demand
struct DdBufs {
    u64 capM = 0, capBytes = 0, capTmp = 0;
    u8 *recs = nullptr, *meta = nullptr, *flags = nullptr, *unmark = nullptr, *collided = nullptr;
    u64 *moff = nullptr, *keys = nullptr, *keys2 = nullptr, *hkey = nullptr, *best = nullptr, *err = nullptr;
    u32 *grp = nullptr, *gStart = nullptr, *perm = nullptr, *perm2 = nullptr, *pairA = nullptr, *pidx = nullptr, *head = nullptr, *rep = nullptr;
    int* pas = nullptr;
    void release() {
        void* all[] = {recs, meta, flags, unmark, collided, moff, keys, keys2, hkey, best, err, grp, gStart, perm, perm2, pairA, pidx, head, rep, pas};
        for (void* p : all) if (p) DD_FREE(p);
        *this = DdBufs();
    }
    bool reserve(u64 m, u64 bytes) {
        if (!err) { err = (u64*)DD_ALLOC(8); if (!err) return false; }
        if (bytes > capBytes) { if (recs) DD_FREE(recs); recs = (u8*)DD_ALLOC(bytes); capBytes = bytes; if (!recs) return false; }
        if (m <= capM) return true;
        for (u8** p : {&meta, &flags, &unmark, &collided}) { if (*p) DD_FREE(*p); *p = (u8*)DD_ALLOC(m); }
        for (u64** p : {&moff, &keys, &keys2, &hkey, &best}) { if (*p) DD_FREE(*p); *p = (u64*)DD_ALLOC(m * 8); }
        for (u32** p : {&grp, &gStart, &perm, &perm2, &pairA, &pidx, &head, &rep}) { if (*p) DD_FREE(*p); *p = (u32*)DD_ALLOC(m * 4); }
        if (pas) DD_FREE(pas);
        pas = (int*)DD_ALLOC(m * 4);
        capM = m;
        for (void* p : {(void*)meta, (void*)flags, (void*)unmark, (void*)collided, (void*)moff, (void*)keys, (void*)keys2, (void*)hkey, (void*)best,
                        (void*)grp, (void*)gStart, (void*)perm, (void*)perm2, (void*)pairA, (void*)pidx, (void*)head, (void*)rep, (void*)pas})
            if (!p) return false;
        return true;
    }
};

// the error return of star_gpu_dedup_batch: unmark[] all 0 except 2 + kind at the member the error names
inline int dedupReportError(u8* unmark, u64 n, u64 member, u32 kind) {
    memset(unmark, 0, n);
    unmark[member] = (u8)(2 + kind);
    return kind == DD_ERR_AS_MISSING ? STAR_EXIT_PARAMETER : STAR_EXIT_INPUT_FILES;
}

// Members [0, n) of whole groups (groups[] non-decreasing); bytes + offsets[i] = member i's record.  Sub-batches of whole groups of at most
// maxM members (a larger group goes alone).  unmark[i] = 1 for the records to un-mark.  Returns 0; 3 when a device allocation failed; or
// 1 with errMember / errKind set (the first error of the first group that has one).
inline int dedupBatchRun(DdBufs& B, const u8* bytes, const uint64_t* offsets, const u32* groups, u64 n, u32 mate2N, u32 hashBits, u64 maxM, u8* unmark,
                         u64& errMember, u32& errKind) {
    std::vector<u64> moff;
    std::vector<u32> grp, gStart;
    for (u64 i0 = 0; i0 < n;) {
        u64 i1 = i0;   // whole groups up to maxM members
        while (i1 < n) {
            u64 j = i1;
            while (j < n && groups[j] == groups[i1]) j++;
            if (i1 > i0 && j - i0 > maxM) break;
            i1 = j;
        }
        const u64 m = i1 - i0;
        const u64 base = offsets[i0], end = offsets[i1 - 1] + 4 + ddRd32(bytes + offsets[i1 - 1]);
        moff.resize(m); grp.resize(m); gStart.resize(m);
        u32 maxL = 0;
        for (u64 i = 0; i < m; i++) {
            moff[i] = offsets[i0 + i] - base;
            grp[i] = i == 0 ? 0 : grp[i - 1] + (groups[i0 + i] != groups[i0 + i - 1]);
            gStart[i] = i == 0 || grp[i] != grp[i - 1] ? (u32)i : gStart[i - 1];
            const u32 l = bytes[offsets[i0 + i] + 12];
            maxL = l > maxL ? l : maxL;
        }
        if (!B.reserve(m, end - base)) { B.release(); return 3; }
        DD_COPY_TO(B.recs, bytes + base, end - base);
        DD_COPY_TO(B.moff, moff.data(), m * 8);
        DD_COPY_TO(B.grp, grp.data(), m * 4);
        DD_COPY_TO(B.gStart, gStart.data(), m * 4);
        const u64 noErr = DD_NO_ERROR;
        DD_COPY_TO(B.err, &noErr, 8);
        DdBatch b;
        b.recs = B.recs; b.moff = B.moff; b.grp = B.grp; b.n = m; b.mate2N = mate2N; b.hashBits = hashBits; b.perm = B.perm; b.meta = B.meta; b.err = B.err;
        DD_LAUNCH(m, dedup_decode_kernel, b);
        // name order: LSD passes, least significant key first
        int gBits = 1;
        while (gBits < 56 && (1ULL << gBits) <= grp[m - 1]) gBits++;
        std::vector<int> passes = {-1};
        for (int w = (int)((maxL + 7) / 8) - 1; w >= 0; w--) passes.push_back(w);
        passes.push_back(-2);
        for (int pass : passes) {
            DD_LAUNCH(m, dedup_namekey_kernel, b, pass, B.keys);
            DD_SORT_PAIRS_U64(B.keys, B.keys2, B.perm, B.perm2, m, pass == -1 ? 1 : pass == -2 ? 8 + gBits : 64);
            u32* t = B.perm; B.perm = B.perm2; B.perm2 = t;
            b.perm = B.perm;
        }
        DD_LAUNCH(m, dedup_pairflag_kernel, b, B.gStart, B.flags);
        u64 nP = 0;
        DD_SELECT_INDEX(B.flags, B.pairA, m, &nP);
        DD_ZERO(B.unmark, m);
        if (nP) {
            DD_LAUNCH(nP, dedup_pairkey_kernel, b, B.pairA, nP, B.hkey, B.pidx, B.pas);
            // class order: stable by hash, then stable by group (keys2 / perm2 / head are free here)
            DD_SORT_PAIRS_U64(B.hkey, B.keys2, B.pidx, B.rep, nP, hashBits >= 64 ? 64 : (hashBits ? (int)hashBits : 1));
            DD_LAUNCH(nP, dedup_classgrp_kernel, b, B.pairA, B.rep, nP, B.keys);
            DD_SORT_PAIRS_U64(B.keys, B.keys2, B.rep, B.pidx, nP, gBits);
            const u32* cls = B.pidx;
            DD_LAUNCH(nP, dedup_runhead_kernel, b, B.pairA, cls, B.hkey, nP, B.head, B.collided);
            DD_MAXSCAN_U32(B.head, nP);
            DD_LAUNCH(nP, dedup_runcheck_kernel, b, B.pairA, cls, B.head, nP, B.collided);
            DD_LAUNCH(nP, dedup_resplit_kernel, b, B.pairA, cls, B.head, B.collided, nP, B.rep, B.best);
            DD_LAUNCH(nP, dedup_best_kernel, cls, B.rep, B.pas, nP, B.best);
            DD_LAUNCH(nP, dedup_unmark_kernel, b, B.pairA, cls, B.rep, B.best, nP, B.unmark);
        }
        u64 e = 0;
        DD_COPY_FROM(&e, B.err, 8);
        if (e != DD_NO_ERROR) { errMember = i0 + (e & 0xffffffffULL); errKind = (u32)(e >> 32) & 7; return 1; }
        DD_COPY_FROM(unmark + i0, B.unmark, m);
        DD_SYNC();
        i0 = i1;
    }
    return 0;
}
#endif

}  // namespace starb
