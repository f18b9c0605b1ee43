// addref_kernels.cuh — device part of adding references at the mapping stage (--genomeFastaFiles with --runMode alignReads;
// reference source/Genome_insertSequences.cpp, insertSeqSA.cpp).
//
// The nG1 bytes of the added sequences (padded chromosomes) go into the genome at nG, the end of the old chromosomes; the nG2 bytes of the
// junction inserts move behind them.
//   addref_rebase_kernel  one thread per 64 rows of the OLD suffix array, in place (insertSeqSA.cpp:33-51): a forward row >= nG and a
//                         reverse row whose position (strand bit cleared) is >= nG2 grow by nG1.  A warp loads its 32 groups (GstrandBit+1
//                         whole words each) into shared memory with coalesced loads, every lane rewrites its own group there, the warp stores
//                         the tile back.  HBM-bound: reads and writes nSA x (GstrandBit+1)/8 bytes.
//   addref_search_kernel  one thread per suffix of the 2*nG1-byte text forward + reverse complement: the row of the re-based SA in front of
//                         which the suffix goes, suffixArraySearch1(N = 10000, gInsert = nG, strR = forward half) over the NEW genome
//                         (insertSeqSA.cpp:76-87).  Suffixes that start with a code > 3 get no row.
//   merge                 sjdb_merge_sa_kernel<AddrefMerge>: the old rows are already re-based, so they are copied as they are.
// All are grid-stride loops, so that the host emulation (tests/addref_check/addref_check.cpp) can run them as one CTA.
#pragma once
#include "sjdb_kernels.cuh"

namespace starb {

struct AddrefRebase {
    u64 nSA, nG, nG1, nG2;
    u32 GstrandBit, bits;
};

__device__ __forceinline__ u64 addrefRebaseRow(const AddrefRebase& a, u64 ind1) {
    const u64 N2bit = 1ULL << a.GstrandBit;
    if (ind1 & N2bit) return (ind1 & ~N2bit) >= a.nG2 ? ind1 + a.nG1 : ind1;
    return ind1 >= a.nG ? ind1 + a.nG1 : ind1;
}

// SA: (nSA+63)/64 * bits words (the tail of the last group is zero).  Dynamic shared memory: (blockDim.x/32) * 32 * bits * 8 bytes.
__global__ void __launch_bounds__(128) addref_rebase_kernel(const AddrefRebase a, u64* __restrict__ SA) {
    extern __shared__ u8 smem[];
    const u32 bits = a.bits;
    const u32 lane = threadIdx.x & 31;
    u64* tile = (u64*)smem + (u64)(threadIdx.x >> 5) * 32 * bits;
    const u64 mask = ~0ULL >> (64 - bits);
    const u64 nGroups = (a.nSA + 63) / 64;
    const u64 nWarps = ((u64)gridDim.x * blockDim.x) >> 5;
#pragma unroll 1
    for (u64 t = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5; t * 32 < nGroups; t += nWarps) {
        const u64 rows = nGroups - t * 32 < 32 ? nGroups - t * 32 : 32;
        u64* src = SA + t * 32 * bits;
        for (u64 k = lane; k < rows * bits; k += 32) tile[k] = src[k];
        __syncwarp();
        const u64 g = t * 32 + lane;
        if (g < nGroups) {
            u64* w = tile + (u64)lane * bits;
#pragma unroll 1
            for (u32 e = 0; e < 64 && g * 64 + e < a.nSA; e++) {
                const u64 b = (u64)e * bits, wi = b >> 6;
                const u32 sh = (u32)(b & 63);
                u64 v = w[wi] >> sh;
                if (sh + bits > 64) v |= w[wi + 1] << (64 - sh);
                v &= mask;
                const u64 nv = addrefRebaseRow(a, v);
                if (nv == v) continue;
                w[wi] = (w[wi] & ~(mask << sh)) | (nv << sh);
                if (sh + bits > 64) w[wi + 1] = (w[wi + 1] & ~(mask >> (64 - sh))) | (nv >> (64 - sh));
            }
        }
        __syncwarp();
        for (u64 k = lane; k < rows * bits; k += 32) src[k] = tile[k];
        __syncwarp();
    }
}

// seq: 2*nG1 bytes (forward, then reverse complement) followed by at least 16 bytes of code 5.  ix: the NEW genome, the re-based SA.
// indArray[2k] = row ((u64)-1: none, (u64)-2: behind the last row), indArray[2k+1] = k.
__global__ void __launch_bounds__(256) addref_search_kernel(const SjdbIndex ix, const u8* __restrict__ seq, u64 nG, u64 nG1, u64* __restrict__ indArray) {
    const u64 nSuf = 2 * nG1;
#pragma unroll 1
    for (u64 k = (u64)blockIdx.x * blockDim.x + threadIdx.x; k < nSuf; k += (u64)gridDim.x * blockDim.x) {
        u64 row = ~0ULL;
        if (SB_LDG(seq + k) <= 3) row = sjdbSearchOne(ix, SaSearch1{10000, nG, k < nG1}, seq + k);
        indArray[2 * k] = row;
        indArray[2 * k + 1] = k;
    }
}

// the inserted rows of the merge (sjdbInsertedRows with sjGstart = nG, revBase = nG2); old rows keep their (re-based) values
struct AddrefMerge {
    const u64* insRow;
    const u64* insVal;
    u64 nInd, nSAnew;
    __device__ __forceinline__ u64 rebase(u64 ind1, u64) const { return ind1; }
};

}  // namespace starb
