// engine_emul.cpp — TEST INFRASTRUCTURE ONLY: the kernel pipeline of the CUDA engine executed on the CPU.
//
// The kernel sources of star_b200/csrc/engine (seed.cu, stitch.cu, stitch_flat.cuh) are included UNMODIFIED and compiled as host
// code through cuda_host_shim.h: every kernel runs as one emulated CTA of 128 (256 for the prep kernel) host threads, warp collectives
// meet at per-warp barriers.  This file mirrors what engine_api.cu does around the kernels for the first tier of a chunk
// (index layout, caps, arenas, pools, launch order: prep -> seed -> heaviest-first order -> stitch_kernel for reads with few loci ->
// flat_setup -> flat_dfs_warp -> flat_record_warp -> scan/pack) on host memory.  tests/ compare the produced alignments with the
// oracle's field by field, so the device logic of the whole path (every kernel of the default pipeline) is exercised lane by lane without a GPU.
// Reads that exceed a first-tier cap are reported (nOverflow) instead of being redone by the tiers.
#include "cuda_host_shim.h"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <functional>
#include <thread>
#include <vector>

namespace cuda_shim {
thread_local Dim tIdx, bIdx, bDim, gDim;
thread_local CtaShared* cta;
}

#include "../star_b200/csrc/engine/seed.cu"
#include "../star_b200/csrc/engine/stitch.cu"
#include "../star_b200/csrc/engine/sjdb_kernels.cuh"

namespace starb { alignas(128) u8 smem[256 * 1024]; }   // dynamic shared memory of the (single) emulated CTA

using namespace starb;

namespace {

// one CTA of nThreads host threads executing `body` (a kernel call with its arguments bound)
void runCta(unsigned nThreads, const std::function<void()>& body) {
    cuda_shim::CtaShared cta;
    cta.nThreads = nThreads;
    pthread_barrier_init(&cta.bar, nullptr, nThreads);
    const unsigned nWarps = (nThreads + 31) / 32;
    for (unsigned w = 0; w < nWarps; w++) {
        pthread_barrier_init(&cta.warp[w].bar, nullptr, 32); memset(cta.warp[w].slot, 0, sizeof(cta.warp[w].slot));
        for (int lg = 0; lg < 4; lg++) for (int gi = 0; gi < 16; gi++) pthread_barrier_init(&cta.warp[w].gbar[lg][gi], nullptr, 2u << lg);
    }
    std::vector<std::thread> th;
    for (unsigned t = 0; t < nThreads; t++)
        th.emplace_back([&, t] {
            cuda_shim::tIdx = {t, 0, 0}; cuda_shim::bIdx = {0, 0, 0}; cuda_shim::bDim = {nThreads, 1, 1}; cuda_shim::gDim = {1, 1, 1};
            cuda_shim::cta = &cta;
            body();
        });
    for (auto& t : th) t.join();
    for (unsigned w = 0; w < nWarps; w++) {
        pthread_barrier_destroy(&cta.warp[w].bar);
        for (int lg = 0; lg < 4; lg++) for (int gi = 0; gi < 16; gi++) pthread_barrier_destroy(&cta.warp[w].gbar[lg][gi]);
    }
    pthread_barrier_destroy(&cta.bar);
}

u64 arenaSize(const Caps& c) {   // engine_api.cu
    u64 b = 0;
    b += (u64)c.maxW * sizeof(Window);
    b += (u64)c.maxW * c.spw * sizeof(Seed);
    b += (u64)c.maxTr * sizeof(DevTr);
    b += 2 * sizeof(DevTr);
    b += (u64)(c.spw + 2) * 128;
    b += (u64)c.maxTr * 2;
    b += (u64)c.maxW * 2 * 2;
    return (b + 255) & ~255ULL;
}

// 2nd stage of --outFilterType BySJout for the next engine_emul_map_chunk calls (engine_emul_set_sj_novel)
std::vector<u64> g_sjNovelStart, g_sjNovelEnd;
bool g_sjNovelOn = false;


u32 envU32(const char* name, u32 dflt) { const char* e = getenv(name); return e ? (u32)strtoul(e, nullptr, 10) : dflt; }

// prep done: the seed stage as engine_api.cu runs it (default: keyed stage of seed_keyed.cuh; STAR_B200_SEED_WARP: the tier seeder over the whole chunk)
static void emulSeedStage(const DevIndex& ix, const star_params_t& P, u8* readsPtr, u32 stride, u32 smemStride, std::vector<ReadInfo>& info, std::vector<Piece>& pieces,
                          u32 maxP, u32 n, std::vector<u32>& counter) {
    if (envU32("STAR_B200_SEED_WARP", 0)) {
        runCta(128, [&] { seed_search_warp_kernel<6>(ix, P, readsPtr, stride, info.data(), pieces.data(), maxP, n, nullptr, counter.data(), smemStride); });
        return;
    }
    std::vector<u32> saKeys((size_t)ix.nSA + 8, 0);
    runCta(256, [&] { build_sa_keys_kernel(ix, saKeys.data()); });
    KeyedArgs ka;
    ka.saKeys = saKeys.data();
    ka.maxItems = std::max<u32>(4096, n * envU32("STAR_B200_SEED_ITEMS_PER_READ", 20));
    ka.maxRec = std::max<u32>(8, envU32("STAR_B200_SEED_RECS_PER_READ", 192));
    ka.scanMax = envU32("STAR_B200_SEED_SCAN_MAX", 2048);
    std::vector<ChainItem> items(ka.maxItems);
    std::vector<u32> itemKey(ka.maxItems), itemIdx(ka.maxItems), itemCount(4, 0), recCount(n, 0);
    std::vector<SeedRec> recs((size_t)n * ka.maxRec);
    ka.items = items.data(); ka.itemKey = itemKey.data(); ka.itemIdx = itemIdx.data(); ka.itemCount = itemCount.data(); ka.recs = recs.data(); ka.recCount = recCount.data();
    runCta(128, [&] { seed_chains_kernel(ix, P, readsPtr, stride, info.data(), n, ka); });
    const u32 nItems = std::min(itemCount[0], ka.maxItems);
    std::vector<u32> itemOrder(itemIdx.begin(), itemIdx.begin() + nItems);
    const int sortBits = (int)std::min<u32>(2 * ix.gSAindexNbases, envU32("STAR_B200_SEED_SORT_BITS", 0)), hiBit = 2 * (int)ix.gSAindexNbases;
    if (sortBits > 0)
        std::stable_sort(itemOrder.begin(), itemOrder.end(), [&](u32 a, u32 b) {
            const u32 ka_ = (itemKey[a] & (u32)((1ULL << hiBit) - 1)) >> (hiBit - sortBits), kb_ = (itemKey[b] & (u32)((1ULL << hiBit) - 1)) >> (hiBit - sortBits);
            return ka_ < kb_; });
    const u32 gl = envU32("STAR_B200_SEED_GROUP_LANES", 8);
    if (gl == 4) runCta(128, [&] { seed_keyed_search_kernel<4, 8>(ix, P, readsPtr, stride, info.data(), sortBits > 0 ? itemOrder.data() : nullptr, ka); });
    else if (gl == 16) runCta(128, [&] { seed_keyed_search_kernel<16, 8>(ix, P, readsPtr, stride, info.data(), sortBits > 0 ? itemOrder.data() : nullptr, ka); });
    else runCta(128, [&] { seed_keyed_search_kernel<8, 8>(ix, P, readsPtr, stride, info.data(), sortBits > 0 ? itemOrder.data() : nullptr, ka); });
    runCta(128, [&] { seed_replay_kernel(P, info.data(), pieces.data(), maxP, n, ka); });
}

struct HostIndex {
    DevIndex ix;
    std::vector<u64> sa, sai, thr;
    std::vector<int> val;
    std::vector<u32> chrBin;
    HostIndex(const star_index_view_t* v, const star_params_t* params) {
        memset(&ix, 0, sizeof(ix));
        ix.G = v->G; ix.nGenome = v->nGenome;
        sa.assign((v->nSAbyte + 7) / 8 + 2, 0); memcpy(sa.data(), v->SA, v->nSAbyte);
        sai.assign((v->nSAibyte + 7) / 8 + 2, 0); memcpy(sai.data(), v->SAi, v->nSAibyte);
        ix.SA = sa.data(); ix.SAi = sai.data(); ix.nSA = v->nSA; ix.nSAi = v->nSAi;
        ix.GstrandBit = v->GstrandBit; ix.saBits = v->GstrandBit + 1; ix.saiBits = v->GstrandBit + 3;
        ix.gSAindexNbases = v->gSAindexNbases; ix.gChrBinNbits = v->gChrBinNbits; ix.nChrReal = v->nChrReal;
        ix.GstrandMask = ~(1ULL << v->GstrandBit);
        ix.SAiMarkNmaskC = 1ULL << (v->GstrandBit + 1); ix.SAiMarkNmask = ~ix.SAiMarkNmaskC; ix.SAiMarkAbsentMaskC = 1ULL << (v->GstrandBit + 2);
        for (u32 i = 0; i <= v->gSAindexNbases; i++) ix.genomeSAindexStart[i] = v->genomeSAindexStart[i];
        {   // Genome::chrBinFill Genome.cpp:209-216
            const u64 nb = 1ULL << v->gChrBinNbits;
            const u64 chrBinN = v->chrStart[v->nChrReal] / nb + 1;
            chrBin.resize(chrBinN);
            for (u64 ii = 0, ichr = 1; ii < chrBinN; ++ii) {
                if (ii * nb >= v->chrStart[ichr]) ichr++;
                chrBin[ii] = (u32)(ichr - 1);
            }
            ix.chrBin = chrBin.data(); ix.chrBinN = chrBinN;
        }
        ix.chrStart = (const u64*)v->chrStart; ix.chrLength = (const u64*)v->chrLength;
        ix.sjdbN = v->sjdbN; ix.sjdbOverhang = v->sjdbOverhang; ix.sjdbLength = v->sjdbLength; ix.sjGstart = v->sjGstart;
        ix.sjdbStart = (const u64*)v->sjdbStart; ix.sjdbEnd = (const u64*)v->sjdbEnd; ix.sjDstart = (const u64*)v->sjDstart; ix.sjAstart = (const u64*)v->sjAstart;
        ix.sjdbMotif = v->sjdbMotif; ix.sjdbShiftLeft = v->sjdbShiftLeft; ix.sjdbShiftRight = v->sjdbShiftRight; ix.sjdbStrand = v->sjdbStrand;
        if (g_sjNovelOn) { ix.sjNovelStart = g_sjNovelStart.data(); ix.sjNovelEnd = g_sjNovelEnd.data(); ix.sjNovelN = g_sjNovelStart.size(); ix.sjNovelOn = 1; }
        {   // step table of the genomic-length score, host libm (engine_api.cu)
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
            ix.log2Thr = thr.data(); ix.log2Val = val.data(); ix.log2N = (int)thr.size();
        }
    }
};

// flat_record_warp_kernel restated sequentially (ONE host thread, the non-cooperative device functions): an independent consumer of the
// task outputs of the emulated flat_dfs_warp_kernel (ENGINE_EMUL_HOST_RECORD=1), used to cross-check the recording kernel.
void hostRecord(const DevIndex& ix, const star_params_t& P, ReadInfo* info, u32 nRecs, u8* arena, const Caps& caps, star_read_result_t* results,
                star_align_t* staged, const FlatArgs& fa) {
    cuda_shim::tIdx = {0, 0, 0}; cuda_shim::bIdx = {0, 0, 0}; cuda_shim::bDim = {1, 1, 1}; cuda_shim::gDim = {1, 1, 1};
    Lane ln;
    static DevTr curL, leafL;
    static Frame stackL[2];
    static u8 phL[8];
    ln.cur = &curL; ln.leaf = &leafL; ln.stack = stackL; ln.ph = phL;
    ln.ix = &ix; ln.P = &P; ln.R0 = nullptr; ln.R2 = nullptr; ln.R = nullptr; ln.caps = caps;
    u8* a = arena;
    ln.win = (Window*)a; a += (u64)caps.maxW * sizeof(Window);
    ln.pool = (DevTr*)a; a += (u64)caps.maxTr * sizeof(DevTr);
    ln.trPtr = (u16*)a; a += (u64)caps.maxTr * sizeof(u16);
    ln.winBase = (u16*)a; a += (u64)caps.maxW * sizeof(u16);
    ln.winN = (u16*)a;
    ln.wa = nullptr;
    ln.memo = nullptr; ln.memoMask = 0; ln.memoBase = 0; ln.memoHit = 0; ln.memoMiss = 0; ln.lastSeed = -1; ln.coop = 0;
    for (u32 q = 0; q < caps.maxTr; q++) ln.trPtr[q] = (u16)q;
    for (u32 k = 0; k < nRecs; k++) {
        const FlatRec rec = fa.recs[k];
        if (rec.done) continue;
        const u32 i = rec.read;
        ReadInfo ri = info[i];
        readBegin(ln, ri);
        ln.saEnum = rec.saEnum;
        if (rec.over) {
            ln.overflow = rec.over;
        } else {
            const u8* rp = fa.pool + rec.poolOff;
            const u32 rs = flatReadStride(rec.Lread);
            ln.R0 = rp; ln.R2 = rp + rs;
            const FlatWin* fw = (const FlatWin*)(rp + 2 * (u64)rs);
            const Seed* fs = (const Seed*)(fw + rec.nWin);
            u64 nd = 0, lv = 0;
            for (u32 t = 0; t < rec.nTasks; t++) { nd += fa.outs[(u64)rec.taskBase + t].nodes; lv += fa.outs[(u64)rec.taskBase + t].leaves; }
            ln.nodes = nd; ln.leaves = lv;
            for (u32 w = 0; w < rec.nWin && !ln.overflow; w++) {
                const FlatWin W = fw[w];
                u16* wTr = nullptr; u16 nWinTr = 0;
                int rc = windowBegin(ln, wTr, nWinTr);
                if (rc == 2) { ln.overflow = 3; break; }
                if (rc == 1) break;
                const u32 Chr = W.Chr, Str = W.Str, nA = W.nWA;
                const Seed* WA = fs + W.seedOff;
                ln.R = Str == 0 ? ln.R0 : ln.R2;
                const u64 tb = (u64)rec.taskBase + W.taskStart;
                for (u32 tq = 0; tq < (1u << W.depth) && !ln.overflow; tq++) {
                    const FlatOut o = fa.outs[tb + tq];
                    u32 b = o.first, inBlock = 0;
                    for (u32 q = 0; q < o.count; q++) {
                        Cand c;
                        if (q == 0) c = o.c0;
                        else {
                            if (inBlock == FLAT_CAND_PER_BLOCK) { b = fa.blocks[b].next; inBlock = 0; }
                            c = fa.blocks[b].c[inBlock++];
                        }
                        if (c.iFrag >= 0 && ln.maxScoreMate[c.iFrag] < c.score) ln.maxScoreMate[c.iFrag] = c.score;
                        const int wBest = ln.pool[wTr[0]].h.maxScore;
                        if (c.score + P.outFilterMultimapScoreRange >= wBest || (c.iFrag >= 0 && c.score + P.outFilterMultimapScoreRange >= ln.maxScoreMate[c.iFrag])) {
                            if (nWinTr > caps.maxTr - ln.trNtotal - 1) { ln.overflow = 3; break; }
                            if (c.trOff != FLAT_NONE) {
                                const u64* src = fa.trStore + c.trOff;
                                memcpy(&ln.leaf->h, src, sizeof(TrHead));
                                memcpy(ln.leaf->ex, src + sizeof(TrHead) / 8, (size_t)ln.leaf->h.nExons * sizeof(Exon));
                                recordLeaf(ln, wTr, &nWinTr);
                            } else {
                                int Score; u32 tR2; u64 tG2;
                                bool ok = replayPath(ln, WA, nA, c.mask, Score, tR2, tG2) && evalLeaf(ln, Score, tR2, tG2, Chr, Str, Str);
                                if (ok) recordLeaf(ln, wTr, &nWinTr);
                            }
                        }
                    }
                }
                windowEnd(ln, Chr, Str, wTr, nWinTr);
            }
        }
        selectExport(ln, ri, i, 0, 0, results, staged, info);
    }
}


}  // namespace

extern "C" {
#pragma GCC visibility push(default)

// Maps one chunk with the emulated kernels.  out: as star_gpu_map_chunk.  info4[4]: reads on the flat path, reads on the lane path,
// reads that overflowed a first-tier cap (their results are not valid), tasks.  Returns 0 or a STAR_EXIT code.
int engine_emul_map_chunk(const star_index_view_t* view, const star_params_t* params, const star_read_batch_t* in, star_align_batch_t* out, uint64_t* info4) {
    HostIndex H(view, params);
    const DevIndex& ix = H.ix;
    const star_params_t P = *params;
    const u32 n = in->nReads;
    const u32 nMates = in->nMates;
    const u32 nOut = (u32)(P.outFilterMultimapNmax > 0 ? P.outFilterMultimapNmax : 1);
    // ---- upload_chunk
    u32 maxL = 0;
    for (u32 i = 0; i < n; i++) {
        const uint64_t* o = in->seqOff + (u64)i * nMates;
        u64 L = nMates == 2 ? (o[1] - o[0]) + (o[2] - o[1]) + 1 : o[1] - o[0];
        if (L > maxL) maxL = (u32)L;
    }
    const u32 stride = (maxL + 16) & ~15u;
    u32 smemStride = (maxL + 1 + 3) & ~3u;
    if (((smemStride / 4) & 1) == 0) smemStride += 4;
    std::vector<u8> readsStore((size_t)n * stride + 64 + 256, 0);   // 256 bytes in front: the 8-byte gathers of the seed stage reach before a row
    u8* const readsPtr = readsStore.data() + 256;
    std::vector<ReadInfo> info(n);
    // ---- caps (engine_api.cu defaults)
    Caps fast;
    fast.maxP = std::min<u32>(128, (u32)P.seedPerReadNmax);
    fast.maxW = (std::min<u32>(128, (u32)P.alignWindowsPerReadNmax) + 1) & ~1u;
    fast.maxTr = std::min<u32>(128, (u32)P.alignTranscriptsPerReadNmax);
    fast.spw = (u32)P.seedPerWindowNmax; fast.nOut = nOut; fast.sortMinW = envU32("STAR_B200_SORTED_LOOKUP_MIN", 12); fast.binFilter = envU32("STAR_B200_BIN_FILTER", 0); fast.arenaBytes = arenaSize(fast);
    Caps heavy = fast;
    heavy.maxW = (std::min<u32>((u32)P.alignWindowsPerReadNmax, 256) + 1) & ~1u;
    heavy.maxTr = std::min<u32>((u32)P.alignTranscriptsPerReadNmax, 1024);
    heavy.arenaBytes = arenaSize(heavy);
    Caps rec = heavy;
    rec.arenaBytes = ((u64)rec.maxW * sizeof(Window) + (u64)rec.maxTr * sizeof(DevTr) + (u64)rec.maxTr * 2 + (u64)rec.maxW * 4 + 255) & ~255ULL;
    const u32 heavyNA = envU32("STAR_B200_HEAVY_NA", 4), heavyEst = envU32("STAR_B200_HEAVY_EST", 1024);
    std::vector<Piece> pieces((size_t)n * fast.maxP);
    std::vector<star_read_result_t> results(n);
    std::vector<star_align_t> staged((size_t)n * nOut);
    memset(results.data(), 0, results.size() * sizeof(star_read_result_t));
    std::vector<u32> counter(8, 0);
    // ---- prep + seed
    runCta(256, [&] { prep_reads_kernel(in->seq, (const u64*)in->seqOff, n, nMates, readsPtr, stride, info.data(), P); });
    if (getenv("ENGINE_EMUL_DEBUG")) fprintf(stderr, "emul: seqOff %llu %llu %llu seq0=%c reads0=%d,%d winBinNbits=%u\n", (unsigned long long)in->seqOff[0], (unsigned long long)in->seqOff[1], (unsigned long long)in->seqOff[2], in->seq[0], readsPtr[0], readsPtr[1], (unsigned)P.winBinNbits);
    if (getenv("ENGINE_EMUL_DEBUG")) fprintf(stderr, "emul: after prep: Lread[0]=%u stride=%u smemStride=%u n=%u\n", info[0].Lread, stride, smemStride, n);
    counter[0] = 0;
    emulSeedStage(ix, P, readsPtr, stride, smemStride, info, pieces, fast.maxP, n, counter);
    if (getenv("ENGINE_EMUL_DEBUG")) fprintf(stderr, "emul: after seed: nP[0]=%u nA[0]=%u flags=%u counter=%u\n", info[0].nP, info[0].nA, info[0].flags, counter[0]);
    // ---- heaviest-first order (stable, like the radix sort on keys ~nA)
    std::vector<u32> order(n);
    for (u32 i = 0; i < n; i++) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](u32 a, u32 b) { return info[a].nA > info[b].nA; });
    u32 nHeavyA = 0;
    if (heavyNA) for (u32 i = 0; i < n; i++) if (info[i].nA >= heavyNA) nHeavyA++;
    // ---- heavy-read hand-over pool of stitch_kernel
    std::vector<u8> heavyPool(64u << 20);
    std::vector<unsigned long long> heavyBump(4, 0);
    std::vector<u64> heavyOff(n, 0);
    std::vector<u32> heavyList(n, 0);
    HeavyArgs hv;
    hv.pool = heavyPool.data(); hv.poolBytes = heavyPool.size(); hv.bump = heavyBump.data(); hv.readOff = heavyOff.data();
    hv.list = heavyList.data(); hv.count = (u32*)(heavyBump.data() + 1); hv.estLimit = heavyEst;
    const bool dbg = getenv("ENGINE_EMUL_DEBUG") != nullptr;
    if (dbg) fprintf(stderr, "emul: nHeavyA=%u of %u, arenaFast %.1f MB\n", nHeavyA, n, 128.0 * fast.arenaBytes / 1048576);
    std::vector<u8> arenaFast((size_t)128 * fast.arenaBytes);
    if (n > nHeavyA) {
        counter[0] = 0;
        runCta(128, [&] { stitch_kernel(ix, P, readsPtr, stride, info.data(), pieces.data(), n - nHeavyA, nullptr, counter.data(), arenaFast.data(), fast,
                                        results.data(), staged.data(), order.data() + nHeavyA, smemStride, hv); });
    }
    const u32 nHeavyX = *hv.count;
    if (dbg) fprintf(stderr, "emul: stitch_kernel done, exported %u\n", nHeavyX);
    std::sort(heavyList.begin(), heavyList.begin() + nHeavyX);
    // ---- flat path
    FlatArgs fa;
    memset(&fa, 0, sizeof(fa));
    std::vector<FlatRec> recs(n + 1);
    std::vector<u8> pool(std::max<u64>(64ull << 20, (u64)n * 65536));
    std::vector<unsigned long long> bumps(8, 0);
    const u64 maxTasks = std::max<u64>(1u << 16, (u64)n * 1024);
    std::vector<FlatTask> tasks(maxTasks);
    std::vector<FlatOut> outs(maxTasks);
    std::vector<FlatBlock> blocks(std::max<u64>(1u << 14, (u64)n * 64));
    std::vector<u64> trStore(std::max<u64>(1u << 20, (u64)n * 8192));
    fa.recs = recs.data(); fa.pool = pool.data(); fa.poolBytes = pool.size(); fa.bumps = bumps.data();
    fa.tasks = tasks.data(); fa.outs = outs.data(); fa.maxTasks = maxTasks; fa.blocks = blocks.data(); fa.maxBlocks = (u32)blocks.size();
    fa.trStore = trStore.data(); fa.trWords = trStore.size(); fa.maxTasksPerRead = 8192; fa.splitMin = envU32("STAR_B200_HEAVY_SPLIT", 12);
    fa.storeAll = envU32("STAR_B200_FLAT_STORE_ALL", 1);
    std::vector<u8> arenaSetup((size_t)4 * heavy.arenaBytes), arenaRec((size_t)4 * rec.arenaBytes);
    if (nHeavyA && envU32("STAR_B200_HEAVY_FLAT", 1) != 0) {
        counter[0] = 0;
        runCta(128, [&] { flat_setup_kernel<3>(ix, P, readsPtr, stride, info.data(), pieces.data(), nHeavyA, order.data(), heavyOff.data(), nullptr, counter.data(),
                                               arenaSetup.data(), heavy, results.data(), staged.data(), smemStride, fa, 0); });
    }
    if (nHeavyX && envU32("STAR_B200_HEAVY_FLAT", 1) != 0) {
        counter[0] = 0;
        runCta(128, [&] { flat_setup_kernel<3>(ix, P, readsPtr, stride, info.data(), nullptr, nHeavyX, heavyList.data(), heavyOff.data(), heavyPool.data(),
                                               counter.data(), arenaSetup.data(), heavy, results.data(), staged.data(), smemStride, fa, nHeavyA); });
    }
    const bool oldHeavy = envU32("STAR_B200_HEAVY_FLAT", 1) == 0;   // warp-per-read kernel (the engine of the overflow tiers) instead of the flat path
    const u32 nRecs = oldHeavy ? 0 : nHeavyA + nHeavyX;
    if (dbg) fprintf(stderr, "emul: setup done, tasks %llu pool %llu\n", bumps[1], bumps[0]);
    if (nRecs) {
        counter[0] = 0;
        runCta(128, [&] { flat_dfs_warp_kernel<4>(ix, P, fa, counter.data(), heavy); });
        if (dbg) fprintf(stderr, "emul: dfs done, blocks %llu words %llu\n", bumps[2], bumps[3]);
        if (envU32("ENGINE_EMUL_HOST_RECORD", 0)) {   // cross-check: the recording restated sequentially on one host thread
            hostRecord(ix, P, info.data(), nRecs, arenaRec.data(), rec, results.data(), staged.data(), fa);
        } else {
            counter[0] = 0;
            runCta(128, [&] { flat_record_warp_kernel<4>(ix, P, info.data(), nRecs, counter.data(), arenaRec.data(), rec, results.data(), staged.data(), fa); });
        }
    }
    if (oldHeavy && (nHeavyA || nHeavyX)) {   // launchHeavy of engine_api.cu
        HeavyScratch hs;
        hs.maxTasks = 8192; hs.maxBlocks = 4096; hs.maxWin = heavy.maxW;
        const u32 W1 = (hs.maxWin + 2) & ~1u;
        hs.trWords = 1u << 17; hs.splitMin = envU32("STAR_B200_HEAVY_SPLIT", 6); hs.memoSlots = 0;
        hs.bytesPerWarp = ((u64)W1 * 8 + ((W1 + 7) & ~7u) + (u64)hs.maxTasks * 8 + (u64)hs.maxBlocks * 504 + (u64)hs.trWords * 8 + 8 + (u64)hs.memoSlots * 72 + 255) & ~255ULL;
        std::vector<u8> scratch((size_t)4 * hs.bytesPerWarp, 0);
        std::vector<u8> arenaHeavy((size_t)4 * heavy.arenaBytes);
        if (nHeavyA) {
            counter[0] = 0;
            runCta(128, [&] { stitch_heavy_kernel(ix, P, readsPtr, stride, info.data(), pieces.data(), nHeavyA, order.data(), heavyOff.data(), nullptr, counter.data(),
                                                  arenaHeavy.data(), heavy, results.data(), staged.data(), smemStride, scratch.data(), hs); });
        }
        if (nHeavyX) {
            counter[0] = 0;
            runCta(128, [&] { stitch_heavy_kernel(ix, P, readsPtr, stride, info.data(), nullptr, nHeavyX, heavyList.data(), heavyOff.data(), heavyPool.data(), counter.data(),
                                                  arenaHeavy.data(), heavy, results.data(), staged.data(), smemStride, scratch.data(), hs); });
        }
        if (dbg) fprintf(stderr, "emul: warp-per-read kernel done (%u + %u reads)\n", nHeavyA, nHeavyX);
    }
    if (dbg) fprintf(stderr, "emul: record done\n");
    // ---- overflow tier (engine_api.cu: reads that exceeded a first-tier cap are redone by stitch_kernel with bigger arenas)
    {
        std::vector<u32> list;
        for (u32 i = 0; i < n; i++) if (info[i].flags & 1) list.push_back(i);
        if (!list.empty()) {
            Caps mid;
            mid.maxP = std::min<u32>((u32)P.seedPerReadNmax, 512);
            mid.maxW = (std::min<u32>((u32)P.alignWindowsPerReadNmax, 1024) + 1) & ~1u;
            mid.maxTr = std::min<u32>((u32)P.alignTranscriptsPerReadNmax, 1024);
            mid.spw = fast.spw; mid.nOut = nOut; mid.sortMinW = fast.sortMinW; mid.binFilter = fast.binFilter; mid.arenaBytes = arenaSize(mid);
            std::vector<Piece> tp((size_t)list.size() * mid.maxP);
            std::vector<u8> arenaMid((size_t)128 * mid.arenaBytes);
            for (u32 i : list) info[i].flags &= ~1u;
            counter[0] = 0;
            runCta(128, [&] { seed_search_warp_kernel<6>(ix, P, readsPtr, stride, info.data(), tp.data(), mid.maxP, (u32)list.size(), list.data(), counter.data(), smemStride); });
            if (envU32("STAR_B200_HEAVY_FLAT", 1) != 0 && envU32("STAR_B200_FLAT_TIER", 1) != 0) {
                // runFlatTier of engine_api.cu: the flat kernels again with the tier's caps, piece slabs by list position
                Caps midRec = mid;
                midRec.arenaBytes = ((u64)mid.maxW * sizeof(Window) + (u64)mid.maxTr * sizeof(DevTr) + (u64)mid.maxTr * 2 + (u64)mid.maxW * 4 + 255) & ~255ULL;
                std::vector<u8> arenaSetupT((size_t)4 * mid.arenaBytes), arenaRecT((size_t)4 * midRec.arenaBytes);
                FlatArgs faT = fa;
                faT.slabByPos = 1;
                std::fill(bumps.begin(), bumps.end(), 0ULL);
                counter[0] = 0;
                runCta(128, [&] { flat_setup_kernel<2>(ix, P, readsPtr, stride, info.data(), tp.data(), (u32)list.size(), list.data(), heavyOff.data(), nullptr, counter.data(),
                                                       arenaSetupT.data(), mid, results.data(), staged.data(), smemStride, faT, 0); });
                counter[0] = 0;
                runCta(128, [&] { flat_dfs_warp_kernel<4>(ix, P, faT, counter.data(), mid); });
                counter[0] = 0;
                runCta(128, [&] { flat_record_warp_kernel<2>(ix, P, info.data(), (u32)list.size(), counter.data(), arenaRecT.data(), midRec, results.data(), staged.data(), faT); });
            } else {
                HeavyArgs hv0 = hv; hv0.estLimit = 0;   // (no hand-over inside the tier)
                counter[0] = 0;
                runCta(128, [&] { stitch_kernel(ix, P, readsPtr, stride, info.data(), tp.data(), (u32)list.size(), list.data(), counter.data(), arenaMid.data(), mid,
                                                results.data(), staged.data(), nullptr, smemStride, hv0); });
            }
            if (dbg) fprintf(stderr, "emul: tier redid %zu reads\n", list.size());
        }
    }
    // ---- scan + pack (host)
    u64 nAl = 0, nOver = 0;
    for (u32 i = 0; i < n; i++) {
        if (info[i].flags & 1) { nOver++; results[i].nTrOut = 0; results[i].nTr = 0; }
        results[i].trOffset = nAl;
        if (nAl + results[i].nTrOut > out->alignsCapacity) return STAR_EXIT_RUNTIME;
        for (u32 k = 0; k < results[i].nTrOut; k++) out->aligns[nAl++] = staged[(u64)i * nOut + k];
        out->reads[i] = results[i];
    }
    out->nAligns = nAl;
    if (info4) { info4[0] = oldHeavy ? nHeavyA + nHeavyX : nRecs; info4[1] = n - nHeavyA; info4[2] = nOver; info4[3] = bumps[1]; }
    return 0;
}

// ---- junction insertion: the kernels of sjdb_kernels.cuh as one emulated CTA each, around them what sjdb.cu does on the host ----
namespace {
struct SjdbHost {
    SjdbIndex ix;
    std::vector<u64> sa;
    u64 sjGstart, sjdbNold;
    explicit SjdbHost(const star_index_view_t* v) {
        sa.assign((v->nSAbyte + 7) / 8 + 2, 0);
        memcpy(sa.data(), v->SA, v->nSAbyte);
        ix.G = v->G; ix.SA = sa.data(); ix.nGenome = v->nGenome; ix.nSA = v->nSA; ix.GstrandBit = v->GstrandBit; ix.saBits = v->GstrandBit + 1;
        sjGstart = v->chrStart[v->nChrReal]; sjdbNold = v->sjdbN;
    }
};
}  // namespace

// n = (uint64)-1 switches the filter off again
// Seeding only (prep + the seed stage of the default pipeline): pc receives 8 numbers per stored piece in the oracle's dump layout
// (rStart, Length, Str=0, Dir, Nrep, SAstart, SAend, iFrag); pcOff[nReads+1]; counters[4] = searches, SAindex words, probes, flagged reads.
int engine_emul_seed_chunk(const star_index_view_t* view, const star_params_t* params, const star_read_batch_t* in, uint64_t* pcOff, uint64_t* pc, uint64_t pcCap,
                           uint64_t* counters) {
    HostIndex hix(view, params);
    const DevIndex& ix = hix.ix;
    const star_params_t P = *params;
    const u32 n = in->nReads, nMates = in->nMates;
    u32 maxL = 0;
    for (u32 i = 0; i < n; i++) {
        const uint64_t* o = in->seqOff + (u64)i * nMates;
        u64 L = nMates == 2 ? (o[1] - o[0]) + (o[2] - o[1]) + 1 : o[1] - o[0];
        if (L > maxL) maxL = (u32)L;
    }
    const u32 stride = (maxL + 16) & ~15u;
    u32 smemStride = (maxL + 1 + 3) & ~3u;
    if (((smemStride / 4) & 1) == 0) smemStride += 4;
    std::vector<u8> readsStore((size_t)n * stride + 64 + 256, 0);   // 256 bytes in front: the 8-byte gathers of the seed stage reach before a row
    u8* const readsPtr = readsStore.data() + 256;
    std::vector<ReadInfo> info(n);
    const u32 maxP = std::min<u32>(128, (u32)P.seedPerReadNmax);
    std::vector<Piece> pieces((size_t)n * maxP);
    std::vector<u32> counter(8, 0);
    runCta(256, [&] { prep_reads_kernel(in->seq, (const u64*)in->seqOff, n, nMates, readsPtr, stride, info.data(), P); });
    emulSeedStage(ix, P, readsPtr, stride, smemStride, info, pieces, maxP, n, counter);
    u64 nPieces = 0;
    pcOff[0] = 0;
    counters[0] = counters[1] = counters[2] = counters[3] = 0;
    for (u32 i = 0; i < n; i++) {
        const ReadInfo& ri = info[i];
        if (ri.flags & 1) counters[3]++;
        else {
            if (nPieces + ri.nP > pcCap) return 1;
            for (u32 k = 0; k < ri.nP; k++) {
                const Piece& p = pieces[(size_t)i * maxP + k];
                uint64_t* o = pc + (nPieces + k) * 8;
                o[0] = p.rStart; o[1] = p.Length; o[2] = 0; o[3] = p.Dir; o[4] = p.Nrep; o[5] = p.SAstart; o[6] = p.SAstart + p.Nrep - 1; o[7] = p.iFrag;
            }
            nPieces += ri.nP;
        }
        pcOff[i + 1] = nPieces;
        counters[0] += ri.cSearches; counters[1] += ri.cSaiWords; counters[2] += ri.cCompare;
    }
    return 0;
}

// The SA key of every row (build_sa_keys_kernel as one emulated CTA): keys[nSA].
int engine_emul_sa_keys(const star_index_view_t* view, const star_params_t* params, uint32_t* keys) {
    HostIndex hix(view, params);
    runCta(256, [&] { build_sa_keys_kernel(hix.ix, keys); });
    return 0;
}

int engine_emul_set_sj_novel(const uint64_t* sjStart, const uint64_t* sjEnd, uint64_t n) {
    if (n == ~0ULL) { g_sjNovelOn = false; return 0; }
    g_sjNovelStart.assign(sjStart, sjStart + n);
    g_sjNovelEnd.assign(sjEnd, sjEnd + n);
    g_sjNovelOn = true;
    return 0;
}

int engine_emul_sjdb_search(const star_index_view_t* v, const uint8_t* Gsj, uint64_t sjdbN, uint64_t sjdbLength, const uint8_t* skipSeq, uint64_t* indArray) {
    SjdbHost H(v);
    const u64 nSeq = 2 * sjdbN, nSuf = nSeq * sjdbLength;
    std::vector<u8> g(nSuf + 1 + 256, 5);
    memcpy(g.data(), Gsj, nSuf + 1);
    runCta(256, [&] { sjdb_search_kernel(H.ix, g.data(), nSeq, sjdbLength, skipSeq, (u64*)indArray); });
    return 0;
}

int engine_emul_sjdb_merge_sa(const star_index_view_t* v, const uint64_t* indSorted, uint64_t nInd, uint64_t nGsj, uint64_t nGsjNew, uint64_t sjdbLength,
                              const uint32_t* oldSJind, uint8_t* SAnew, uint64_t nSAnewByte) {
    SjdbHost H(v);
    const u64 nSAnew = H.ix.nSA + nInd;
    std::vector<u64> row(nInd + 1), val(nInd + 1);
    sjdbInsertedRows(indSorted, nInd, H.ix.nSA, nGsj, H.sjGstart, H.ix.GstrandBit, row.data(), val.data());
    std::vector<u64> out((nSAnew + 63) / 64 * H.ix.saBits + 2, 0);
    SjdbMerge m;
    m.insRow = row.data(); m.insVal = val.data(); m.nInd = nInd; m.nSAnew = nSAnew;
    m.nGenomeOld = H.ix.nGenome; m.nGenomeNew = H.sjGstart + nGsj; m.sjGstart = H.sjGstart; m.sjdbLength = sjdbLength; m.sjdbNold = H.sjdbNold;
    m.nGsjNew = nGsjNew; m.oldSJind = (const u32*)oldSJind;
    runCta(128, [&] { sjdb_merge_sa_kernel(H.ix, m, out.data()); });
    if (nSAnewByte > out.size() * 8) return STAR_EXIT_BUG;
    memcpy(SAnew, out.data(), nSAnewByte);
    return 0;
}

#pragma GCC visibility pop
}  // extern "C"

// ---- suffix-array build: the kernels and the round loop of sa_build_impl.cuh on host memory; cub's sort / scan / select replaced by std:: ----
namespace starb {
static void* emAlloc(size_t bytes) { return calloc(bytes ? bytes : 1, 1); }
static void emSortPairs(const u64* kIn, u64* kOut, const u32* vIn, u32* vOut, u64 n, int endBit) {
    std::vector<u64> order(n);
    for (u64 i = 0; i < n; i++) order[i] = i;
    const u64 mask = endBit >= 64 ? ~0ULL : ((1ULL << endBit) - 1);
    std::stable_sort(order.begin(), order.end(), [&](u64 a, u64 b) { return (kIn[a] & mask) < (kIn[b] & mask); });
    for (u64 i = 0; i < n; i++) { kOut[i] = kIn[order[i]]; vOut[i] = vIn[order[i]]; }
}
static void emMaxScan(u32* a, u64 n) { for (u64 i = 1; i < n; i++) if (a[i] < a[i - 1]) a[i] = a[i - 1]; }
static void emSortPairs64(const u64* kIn, u64* kOut, const u64* vIn, u64* vOut, u64 n, int endBit) {
    std::vector<u64> order(n);
    for (u64 i = 0; i < n; i++) order[i] = i;
    const u64 mask = endBit >= 64 ? ~0ULL : ((1ULL << endBit) - 1);
    std::stable_sort(order.begin(), order.end(), [&](u64 a, u64 b) { return (kIn[a] & mask) < (kIn[b] & mask); });
    for (u64 i = 0; i < n; i++) { kOut[i] = kIn[order[i]]; vOut[i] = vIn[order[i]]; }
}
static void emMaxScan64(u64* a, u64 n) { for (u64 i = 1; i < n; i++) if (a[i] < a[i - 1]) a[i] = a[i - 1]; }
template <class F> static void emSelectIf(F f, u64 lo, u64 hi, u64* out, u64* nSel) { u64 k = 0; for (u64 v = lo; v < hi; v++) if (f(v)) out[k++] = v; *nSel = k; }
static void emSelect(const u32* in, const u8* flag, u32* out, u64 n, u64* nSel) { u64 k = 0; for (u64 i = 0; i < n; i++) if (flag[i]) out[k++] = in[i]; *nSel = k; }
}  // namespace starb
#define SA_ALLOC(bytes) starb::emAlloc(bytes)
#define SA_FREE(p) free(p)
#define SA_LAUNCH(count, kernel, ...) runCta(256, [&] { kernel(__VA_ARGS__); })
#define SA_LAUNCH_PACK(nRows, bits, kernel, ...) runCta(128, [&] { kernel(__VA_ARGS__); })
#define SA_COPY_TO(dst, src, bytes) memcpy(dst, src, bytes)
#define SA_COPY_FROM(dst, src, bytes) memcpy(dst, src, bytes)
#define SA_SORT_PAIRS(kIn, kOut, vIn, vOut, n, endBit) starb::emSortPairs(kIn, kOut, vIn, vOut, n, endBit)
#define SA_MAX_SCAN(a, n) starb::emMaxScan(a, n)
#define SA_SELECT(in, flag, out, n, nSel) starb::emSelect(in, flag, out, n, nSel)
#define SA_SYNC() ((void)0)
#define SA_ZERO(p, bytes) memset(p, 0, bytes)
#define SA_SORT_PAIRS64(kIn, kOut, vIn, vOut, n, endBit) starb::emSortPairs64(kIn, kOut, vIn, vOut, n, endBit)
#define SA_MAX_SCAN64(a, n) starb::emMaxScan64(a, n)
#define SA_SELECT_IF(f, lo, hi, out, nSel) starb::emSelectIf(f, lo, hi, out, nSel)
#include "../star_b200/csrc/engine/sa_build_large.cuh"

extern "C" {
#pragma GCC visibility push(default)
int engine_emul_sa_build(int, const uint8_t* G, uint64_t nGenome, uint32_t GstrandBit, uint64_t nSA, uint8_t* SA, uint64_t nSAbyte) {
    if (2 * nGenome >= (1ULL << 32) - 64 && !getenv("STAR_B200_SA_LARGE_CAP")) return STAR_EXIT_PARAMETER;
    const u64 outWords = (nSA + 63) / 64 * (GstrandBit + 1) + 2;
    std::vector<u64> out(outWords, 0);
    u64 rounds = 0;
    u64 largeCap = 0;   // STAR_B200_SA_LARGE_CAP=<elements per sort>: the batched 64-bit path of sa_build_large.cuh
    if (const char* e = getenv("STAR_B200_SA_LARGE_CAP")) largeCap = strtoull(e, nullptr, 10);
    int rc;
    if (largeCap) {   // (the large path releases its genome copy early and allocates the packed output late)
        u8* Gc = (u8*)emAlloc(nGenome);
        memcpy(Gc, G, nGenome);
        u64* ow = nullptr;
        rc = saBuildRunLarge(Gc, nGenome, GstrandBit, nSA, &ow, outWords, largeCap, &rounds);
        if (!rc) memcpy(out.data(), ow, outWords * 8);
        free(ow);
    } else rc = saBuildRun(G, nGenome, GstrandBit, nSA, out.data(), &rounds);
    if (getenv("ENGINE_EMUL_DEBUG")) fprintf(stderr, "emul: sa_build rc %d after %llu rounds\n", rc, (unsigned long long)rounds);
    if (rc == 4) return STAR_EXIT_PARAMETER;   // a bin or a tied group exceeds the forced capacity
    if (rc) return STAR_EXIT_BUG;
    if (nSAbyte > outWords * 8) return STAR_EXIT_BUG;
    memcpy(SA, out.data(), nSAbyte);
    return 0;
}
#pragma GCC visibility pop
}  // extern "C"
