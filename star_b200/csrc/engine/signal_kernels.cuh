// signal_kernels.cuh — per-base signal tracks of one segment (reference source/signalFromBAM.cpp:76-202), in position windows.
//
// Per window [w0, w0+W) and strand s, two counters per position: cntU = records with NH == 1 covering it, cntM = records with NH != 1.
//   signal_scatter_kernel  one thread per block: +1 / -1 at the ends of the block's window part (u32 difference arrays; a scan sums them)
//   (scan)                 one inclusive scan over all difference arrays (each array's differences sum to 0, so they concatenate)
//   signal_mixed_kernel    flag of the "mixed" positions (cntM != 0), exclusive-scanned into ranks
//   signal_count_kernel    pairs per block = mixed positions it covers; exclusively scanned into offsets (= record order)
//   signal_emit_kernel     (key = array index of the position, value = block) for every pair of a chunk of the pair sequence
//   (stable radix sort)    by key: every position's pairs stay in record order
//   signal_fold_kernel     one thread per position of the chunk: um += 1.0/nh over its pairs, sequentially, from the partial sum the chunks
//                          before left (chunks split the pair sequence in record order, so the fold order is the reference's)
//   signal_flag_kernel     output positions: value differs from the position before (bedGraph) or is nonzero (wiggle)
//   (select)               their indices, in track-major order
//   signal_gather_kernel   their values
// Where cntM == 0 both tracks are the integer count cntU: the reference's sum of 1.0 terms from 0.0 is exact.  The UniqueMultiple value of a
// mixed position is the fold; the sum of 1/3 + 1 + 1/3 depends on the order and bedGraph splits records on exact inequality, so no atomics
// and no tree reduction touch it.  All kernels are grid-stride loops, so the host emulation (oracle/engine_emul.cpp) runs them as one CTA.
// signalSegmentRun (below) is the window / chunk loop; it is compiled with the SG_* primitives of signal.cu (cub, CUDA runtime) or of the
// emulation (std::).
#pragma once
#include <vector>

#include "dev.cuh"

namespace starb {

struct SigWin {
    const star_signal_block_t* blocks;
    u64 nBlocks;
    u32 w0, W, stride, nS;   // window [w0, w0+W); stride = W+1 entries per strand array
    u32* cntU;               // nS * stride
    u32* cntM;
    u32* rank;               // nS * stride: exclusive rank of the mixed positions
    double* um;              // nS * stride: UniqueMultiple fold at mixed positions
    u64* off;                // nBlocks + 1: pair offsets of the blocks
};

__device__ __forceinline__ bool sigClip(const SigWin& w, const star_signal_block_t& b, u32& a, u32& e) {
    const u64 s = b.start, t = (u64)b.start + b.len, lo = w.w0, hi = (u64)w.w0 + w.W;
    a = (u32)((s > lo ? s : lo) - lo);
    e = (u32)((t < hi ? t : hi) - lo);
    return s < hi && t > lo && b.len > 0;
}

__global__ void __launch_bounds__(256) signal_scatter_kernel(const SigWin w) {
#pragma unroll 1
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < w.nBlocks; i += (u64)gridDim.x * blockDim.x) {
        const star_signal_block_t b = w.blocks[i];
        u32 a, e;
        if (!sigClip(w, b, a, e)) continue;
        u32* c = (b.nh == 1 ? w.cntU : w.cntM) + (u64)b.strand * w.stride;
        atomicAdd(c + a, 1u);
        atomicAdd(c + e, 0xffffffffu);
    }
}

__global__ void __launch_bounds__(256) signal_mixed_kernel(const SigWin w) {
    const u64 n = (u64)w.nS * w.stride;
#pragma unroll 1
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        w.rank[i] = w.cntM[i] != 0;
        w.um[i] = 0.0;
    }
}

__global__ void __launch_bounds__(256) signal_count_kernel(const SigWin w) {
#pragma unroll 1
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i <= w.nBlocks; i += (u64)gridDim.x * blockDim.x) {
        u64 c = 0;
        u32 a, e;
        if (i < w.nBlocks && sigClip(w, w.blocks[i], a, e)) {
            const u32* r = w.rank + (u64)w.blocks[i].strand * w.stride;
            c = r[e] - r[a];   // (exclusive ranks: mixed positions in [a, e))
        }
        w.off[i] = c;
    }
}

// pairs [k0, k0 + cap) of the window's pair sequence (block by block, position by position)
__global__ void __launch_bounds__(256) signal_emit_kernel(const SigWin w, u64 k0, u64 cap, u32* __restrict__ keys, u32* __restrict__ vals) {
#pragma unroll 1
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < w.nBlocks; i += (u64)gridDim.x * blockDim.x) {
        const u64 o = w.off[i], n = w.off[i + 1] - o;
        if (n == 0 || o >= k0 + cap || o + n <= k0) continue;
        u32 a, e;
        sigClip(w, w.blocks[i], a, e);
        const u64 base = (u64)w.blocks[i].strand * w.stride;
        u64 k = o;
#pragma unroll 1
        for (u32 p = a; p < e && k < k0 + cap; p++) {
            if (w.cntM[base + p] == 0) continue;
            if (k >= k0) { keys[k - k0] = (u32)(base + p); vals[k - k0] = (u32)i; }
            k++;
        }
    }
}

__global__ void __launch_bounds__(256) signal_fold_kernel(const SigWin w, const u32* __restrict__ keys, const u32* __restrict__ vals, u64 n) {
#pragma unroll 1
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        const u32 key = keys[i];
        if (i > 0 && keys[i - 1] == key) continue;
        double acc = w.um[key];
#pragma unroll 1
        for (u64 j = i; j < n && keys[j] == key; j++) acc += 1.0 / (double)w.blocks[vals[j]].nh;
        w.um[key] = acc;
    }
}

// value of track t (= 2*strand + k) at window position p
__device__ __forceinline__ double sigValue(const SigWin& w, u32 t, u32 p) {
    const u64 i = (u64)(t >> 1) * w.stride + p;
    const u32 m = w.cntM[i];
    return (t & 1) && m != 0 ? w.um[i] : (double)w.cntU[i];
}

struct SigPrev { double v[4]; };   // value of every track at position w0-1 (0 before position 0)

__global__ void __launch_bounds__(256) signal_flag_kernel(const SigWin w, int mode, const SigPrev prev, u8* __restrict__ flags) {
    const u64 n = (u64)2 * w.nS * w.W;
#pragma unroll 1
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        const u32 t = (u32)(i / w.W), p = (u32)(i % w.W);
        const double v = sigValue(w, t, p);
        if (mode == 0) flags[i] = v != (p == 0 ? prev.v[t] : sigValue(w, t, p - 1));
        else flags[i] = v != 0.0;
    }
}

__global__ void __launch_bounds__(256) signal_gather_kernel(const SigWin w, const u32* __restrict__ idx, u64 n, double* __restrict__ val) {
#pragma unroll 1
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) val[i] = sigValue(w, idx[i] / w.W, idx[i] % w.W);
}

#ifdef SG_LAUNCH
// Device buffers of a handle (grown on demand); positions per window and pairs per chunk are the caller's capacities.
struct SigBufs {
    u64 capPos = 0, capPairs = 0, capBlocks = 0;
    u32 *cntU = nullptr, *cntM = nullptr, *rank = nullptr, *idx = nullptr, *keys = nullptr, *vals = nullptr, *keys2 = nullptr, *vals2 = nullptr;
    double *um = nullptr, *val = nullptr;
    u8* flags = nullptr;
    u64* off = nullptr;
    star_signal_block_t* blocks = nullptr;
    void release() {
        void* all[] = {cntU, cntM, rank, idx, keys, vals, keys2, vals2, um, val, flags, off, blocks};
        for (void* p : all) if (p) SG_FREE(p);
        *this = SigBufs();
    }
};

// One segment: windows of at most maxW positions, pair chunks of at most maxPairs.  out[t] receives (position, value) of the output
// positions of track t, appended in position order.  Returns 0, or 3 when a device allocation failed.
inline int signalSegmentRun(SigBufs& B, u32 nS, u32 chrLen, const star_signal_block_t* hostBlocks, u64 nBlocks, int mode, u64 maxW, u64 maxPairs,
                            std::vector<u32>* outPos, std::vector<double>* outVal) {
    const u32 nT = 2 * nS;
    const u64 W0 = chrLen < maxW ? chrLen : maxW;
    if (B.capPos < W0) {
        const u64 np = (u64)nS * (W0 + 1);
        for (u32** p : {&B.cntU, &B.cntM, &B.rank}) { if (*p) SG_FREE(*p); *p = (u32*)SG_ALLOC(np * 4); }
        if (B.um) SG_FREE(B.um);
        B.um = (double*)SG_ALLOC(np * 8);
        if (B.flags) SG_FREE(B.flags);
        B.flags = (u8*)SG_ALLOC((u64)nT * W0);
        if (B.idx) SG_FREE(B.idx);
        B.idx = (u32*)SG_ALLOC((u64)nT * W0 * 4);
        if (B.val) SG_FREE(B.val);
        B.val = (double*)SG_ALLOC((u64)nT * W0 * 8);
        B.capPos = W0;
        if (!B.cntU || !B.cntM || !B.rank || !B.um || !B.flags || !B.idx || !B.val) { B.release(); return 3; }
    }
    if (B.capBlocks < nBlocks + 1) {
        if (B.blocks) SG_FREE(B.blocks);
        if (B.off) SG_FREE(B.off);
        B.blocks = (star_signal_block_t*)SG_ALLOC((nBlocks + 1) * sizeof(star_signal_block_t));
        B.off = (u64*)SG_ALLOC((nBlocks + 2) * 8);
        B.capBlocks = nBlocks + 1;
        if (!B.blocks || !B.off) { B.release(); return 3; }
    }
    SG_COPY_TO(B.blocks, hostBlocks, nBlocks * sizeof(star_signal_block_t));
    SigPrev prev;
    for (u32 t = 0; t < 4; t++) prev.v[t] = 0.0;
    for (u64 w0 = 0; w0 < chrLen; w0 += W0) {
        SigWin w;
        w.blocks = B.blocks; w.nBlocks = nBlocks;
        w.w0 = (u32)w0; w.W = (u32)(chrLen - w0 < W0 ? chrLen - w0 : W0); w.stride = w.W + 1; w.nS = nS;
        w.cntU = B.cntU; w.cntM = B.cntM; w.rank = B.rank; w.um = B.um; w.off = B.off;
        const u64 nArr = (u64)nS * w.stride;
        SG_ZERO(B.cntU, nArr * 4);
        SG_ZERO(B.cntM, nArr * 4);
        SG_LAUNCH(nBlocks, signal_scatter_kernel, w);
        SG_SCAN_U32(B.cntU, nArr);
        SG_SCAN_U32(B.cntM, nArr);
        SG_LAUNCH(nArr, signal_mixed_kernel, w);
        SG_EXSCAN_U32(B.rank, nArr);
        SG_LAUNCH(nBlocks + 1, signal_count_kernel, w);
        SG_EXSCAN_U64(B.off, nBlocks + 1);
        u64 nPairs = 0;
        SG_COPY_FROM(&nPairs, B.off + nBlocks, 8);
        if (nPairs) {
            const u64 cap = nPairs < maxPairs ? nPairs : maxPairs;
            if (B.capPairs < cap) {
                for (u32** p : {&B.keys, &B.vals, &B.keys2, &B.vals2}) { if (*p) SG_FREE(*p); *p = (u32*)SG_ALLOC(cap * 4); }
                B.capPairs = cap;
                if (!B.keys || !B.vals || !B.keys2 || !B.vals2) { B.release(); return 3; }
            }
            int endBit = 1;
            while (endBit < 32 && (1ULL << endBit) < nArr) endBit++;
            for (u64 k0 = 0; k0 < nPairs; k0 += cap) {
                const u64 n = nPairs - k0 < cap ? nPairs - k0 : cap;
                SG_LAUNCH(nBlocks, signal_emit_kernel, w, k0, cap, B.keys, B.vals);
                SG_SORT_PAIRS_U32(B.keys, B.keys2, B.vals, B.vals2, n, endBit);
                SG_LAUNCH(n, signal_fold_kernel, w, B.keys2, B.vals2, n);
            }
        }
        const u64 nF = (u64)nT * w.W;
        SG_LAUNCH(nF, signal_flag_kernel, w, mode, prev, B.flags);
        u64 nSel = 0;
        SG_SELECT_INDEX(B.flags, B.idx, nF, &nSel);
        if (nSel) {
            SG_LAUNCH(nSel, signal_gather_kernel, w, B.idx, nSel, B.val);
            std::vector<u32> ix(nSel);
            std::vector<double> vx(nSel);
            SG_COPY_FROM(ix.data(), B.idx, nSel * 4);
            SG_COPY_FROM(vx.data(), B.val, nSel * 8);
            for (u64 k = 0; k < nSel; k++) {   // (track-major: every track's positions stay in order)
                const u32 t = ix[k] / w.W;
                outPos[t].push_back(w.w0 + ix[k] % w.W);
                outVal[t].push_back(vx[k]);
            }
        }
        for (u32 t = 0; t < nT; t++)   // the value at the last position of this window = the last output value (bedGraph), or not needed (wiggle)
            prev.v[t] = outVal[t].empty() ? 0.0 : outVal[t].back();
        SG_SYNC();
    }
    return 0;
}
#endif

}  // namespace starb
