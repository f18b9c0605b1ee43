// driver.cpp — the drop-in command line: STAR --runMode alignReads --genomeDir .. --readFilesIn .. (SAM out).
//
// Mirrors the run orchestration of reference source/STAR.cpp:58-313 (parameters -> genomeLoad -> SAM header ->
// map all chunks -> SJ.out.tab -> Log.final.out) with the per-chunk work of
// ReadAlignChunk::processChunks/mapChunk (ReadAlignChunk_processChunks.cpp:11-282, ReadAlignChunk_mapChunk.cpp:7-128)
// replaced by one engine call per chunk through the C-ABI (include/star_b200.h).  The engine is passed in as a
// vtable so that the test-suite can drive the same host code with the CPU oracle; the shipped binary
// binds the CUDA engine (star_cli_main below) and has no other engine.
#include <sys/stat.h>

#include <cstring>
#include <ctime>
#include <fstream>
#include <iostream>
#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <deque>
#include <filesystem>
#include <memory>
#include <mutex>
#include <random>
#include <sstream>
#include <thread>

#include "host.h"

namespace starhost {

// what the reference sends to stdout goes to <prefix>Log.std.out when stdout carries alignments (--outStd SAM | BAM_*; Parameters.cpp:385-391)
static std::ostream* g_logStd = &std::cout;
static std::ofstream g_logStdFile;

static std::string timeMonthDayTime(time_t t) {
    char b[100];
    strftime(b, 80, "%b %d %H:%M:%S", localtime(&t));
    return b;
}

static void makeDirs(const std::string& prefix) {  // createDirectory, Parameters.cpp:367
    size_t p = prefix.rfind('/');
    if (p == std::string::npos) return;
    std::string dir = prefix.substr(0, p);
    std::string cur;
    for (size_t i = 0; i <= dir.size(); i++) {
        if (i == dir.size() || dir[i] == '/') {
            if (!cur.empty()) mkdir(cur.c_str(), 0700);
        }
        if (i < dir.size()) cur.push_back(dir[i]);
    }
}

// what one shard of a multi-GPU run leaves for the merge: the 24 counters, 3 times, the collapsed junction records
static void writeShardBin(const std::string& path, const Stats& stats, const std::vector<Junction>& sj) {
    std::ofstream sb(path, std::ios::binary);
    uint64_t cnt[Stats::N_COUNTERS];
    stats.toArray(cnt);
    int64_t tm[3] = {(int64_t)stats.timeStart, (int64_t)stats.timeStartMap, (int64_t)stats.timeFinish};
    uint64_t nsj = sj.size();
    sb.write((const char*)cnt, sizeof(cnt));
    sb.write((const char*)tm, sizeof(tm));
    sb.write((const char*)&nsj, 8);
    if (nsj) sb.write((const char*)sj.data(), nsj * sizeof(Junction));
}

// One mapping pass over the read files (ReadAlignChunk::processChunks / mapThreadsSpawn for all chunks): reads -> engine -> records.
// Used for the main pass and, with the outputs switched off in P, for the 1st pass of --twopassMode Basic.
// Returns 0 or a STAR_EXIT_* code with the message in err.
// State that outlives one call of mapPass when a run maps in two stages (--outFilterType BySJout, STAR.cpp:196-220): the reads held
// back by the 1st stage, the junction records of all reads, and the records waiting for the coordinate sort.
struct CoordRec { uint64_t alignG, key; uint32_t blob, size; uint64_t off; };
struct StageState {
    int bySJstage = 0;                       // 0: single stage; 1: hold reads with unannotated junctions; 2: map the held reads
    std::vector<Junction> sjAll;             // stage 1: junction records of ALL mapped reads (chunkOutSJ1)
    std::vector<ReadChunk> held;             // stage 1 -> 2: the reads to map again, in input order, chunked (never across input files)
    const TranscriptModel* trModel = nullptr;   // --quantMode TranscriptomeSAM
    std::mt19937 rngMultOrder;               // one draw per mapped, written read, in read order (ReadAlign_quantTranscriptome.cpp:69)
    const GeneModel* geneModel = nullptr;    // --quantMode GeneCounts: exons / genes, and the counts of every stage
    GeneCounts geneCounts;
    std::string streamSuffix;                // sharded 2nd stage: records go to Aligned.out<suffix>.sam|bam (the merge orders the parts)
    std::vector<std::string> coordBlobs;     // coordinate-sorted BAM: uncompressed records of every stage
    std::vector<CoordRec> coordIndex;
};

static void holdRead(std::vector<ReadChunk>& held, const ReadChunk& c, uint32_t i, uint32_t maxReads) {
    if (held.empty() || held.back().nReads >= maxReads || held.back().fileIndex != c.fileIndex) {
        held.emplace_back();
        ReadChunk& h = held.back();
        h.nMates = c.nMates; h.fastq = c.fastq; h.fileIndex = c.fileIndex;
        h.seqOff.push_back(0); h.nameOff.push_back(0);
    }
    ReadChunk& h = held.back();
    for (uint32_t m = 0; m < c.nMates; m++) {
        const uint64_t a = c.seqOff[(uint64_t)i * c.nMates + m], b = c.seqOff[(uint64_t)i * c.nMates + m + 1];
        h.seq.append(c.seq, a, b - a);
        if (!c.qual.empty()) h.qual.append(c.qual, a, b - a);
        h.seqOff.push_back(h.seq.size());
    }
    h.names.append(c.names, c.nameOff[i], c.nameOff[i + 1] - c.nameOff[i]);
    h.nameOff.push_back((uint32_t)h.names.size());
    if (c.clipped()) {
        if (h.seqOffC.empty()) h.seqOffC.push_back(0);
        for (uint32_t m = 0; m < c.nMates; m++) {
            const uint64_t a = c.seqOffC[(uint64_t)i * c.nMates + m], b = c.seqOffC[(uint64_t)i * c.nMates + m + 1];
            h.seqC.append(c.seqC, a, b - a);
            h.seqOffC.push_back(h.seqC.size());
            h.clip5.push_back(c.clip5[(uint64_t)i * c.nMates + m]); h.clip3.push_back(c.clip3[(uint64_t)i * c.nMates + m]);
        }
    }
    if (!c.nameFullOff.empty()) { h.nameFullOff.push_back((uint32_t)h.namesFull.size()); h.namesFull += c.namesFull.c_str() + c.nameFullOff[i]; h.namesFull.push_back('\0'); }
    h.readFilter.push_back(c.readFilter[i]);
    h.iReadAll.push_back(c.iReadAll[i]);
    h.nReads++;
}

// Sharded --outFilterType BySJout: what the 1st stage of a shard leaves for its 2nd stage (a separate call of the command line, after the
// junction records of all shards have been gathered): counters, the junction records of the reads written so far, the held reads.
template <class T> static void putVec(std::ofstream& o, const std::vector<T>& v) { uint64_t n = v.size(); o.write((const char*)&n, 8); if (n) o.write((const char*)v.data(), n * sizeof(T)); }
template <class T> static void getVec(std::ifstream& in, std::vector<T>& v) { uint64_t n = 0; in.read((char*)&n, 8); v.resize(n); if (n) in.read((char*)v.data(), n * sizeof(T)); }
static void putStr(std::ofstream& o, const std::string& v) { uint64_t n = v.size(); o.write((const char*)&n, 8); o.write(v.data(), n); }
static void getStr(std::ifstream& in, std::string& v) { uint64_t n = 0; in.read((char*)&n, 8); v.resize(n); if (n) in.read(&v[0], n); }
static void saveStage1(const std::string& path, const Stats& stats, const std::vector<Junction>& allSJ, const std::vector<ReadChunk>& held) {
    std::ofstream o(path, std::ios::binary);
    uint64_t cnt[Stats::N_COUNTERS];
    stats.toArray(cnt);
    int64_t tm[3] = {(int64_t)stats.timeStart, (int64_t)stats.timeStartMap, (int64_t)stats.timeFinish};
    o.write((const char*)cnt, sizeof(cnt)); o.write((const char*)tm, sizeof(tm));
    putVec(o, allSJ);
    uint64_t nh = held.size();
    o.write((const char*)&nh, 8);
    for (const ReadChunk& c : held) {
        uint32_t hd[4] = {c.nReads, c.nMates, (uint32_t)c.fastq, c.fileIndex};
        o.write((const char*)hd, sizeof(hd));
        putStr(o, c.seq); putStr(o, c.qual); putVec(o, c.seqOff); putStr(o, c.names); putVec(o, c.nameOff); putVec(o, c.readFilter); putVec(o, c.iReadAll); putStr(o, c.namesFull); putVec(o, c.nameFullOff); putVec(o, c.clip5); putVec(o, c.clip3); putStr(o, c.seqC); putVec(o, c.seqOffC);
    }
}
static bool loadStage1(const std::string& path, Stats& stats, std::vector<Junction>& allSJ, std::vector<ReadChunk>& held) {
    std::ifstream in(path, std::ios::binary);
    if (!in.good()) return false;
    uint64_t cnt[Stats::N_COUNTERS]; int64_t tm[3];
    in.read((char*)cnt, sizeof(cnt)); in.read((char*)tm, sizeof(tm));
    stats.fromArray(cnt);
    stats.timeStart = (time_t)tm[0]; stats.timeStartMap = (time_t)tm[1]; stats.timeFinish = (time_t)tm[2];
    getVec(in, allSJ);
    uint64_t nh = 0;
    in.read((char*)&nh, 8);
    held.resize(nh);
    for (ReadChunk& c : held) {
        uint32_t hd[4];
        in.read((char*)hd, sizeof(hd));
        c.nReads = hd[0]; c.nMates = hd[1]; c.fastq = hd[2] != 0; c.fileIndex = hd[3];
        getStr(in, c.seq); getStr(in, c.qual); getVec(in, c.seqOff); getStr(in, c.names); getVec(in, c.nameOff); getVec(in, c.readFilter); getVec(in, c.iReadAll); getStr(in, c.namesFull); getVec(in, c.nameFullOff); getVec(in, c.clip5); getVec(in, c.clip3); getStr(in, c.seqC); getVec(in, c.seqOffC);
    }
    return in.good();
}
// adds the counts of a ReadsPerGene table (4 summary rows, then one row per gene) to gc; N_unmapped is recomputed from the counters
static bool readGeneCounts(const std::string& path, GeneCounts& gc) {
    std::ifstream in(path);
    if (!in.good()) return false;
    std::string name;
    uint64_t v[3];
    size_t ig = 0;
    for (int row = 0; in >> name >> v[0] >> v[1] >> v[2]; row++) {
        if (row == 0) continue;
        if (row == 1) gc.cMulti += v[0];
        else if (row == 2) for (int t = 0; t < 3; t++) gc.cNone[t] += v[t];
        else if (row == 3) for (int t = 0; t < 3; t++) gc.cAmbig[t] += v[t];
        else { for (int t = 0; t < 3; t++) { if (gc.gCount[t].size() <= ig) gc.gCount[t].resize(ig + 1, 0); gc.gCount[t][ig] += v[t]; } ig++; }
    }
    return true;
}

// junction records of shard.bin-style files (24 counters, 3 times, count, records)
static bool readShardJunctions(const std::string& path, std::vector<Junction>& sj) {
    std::ifstream in(path, std::ios::binary);
    if (!in.good()) return false;
    in.seekg(8 * Stats::N_COUNTERS + 24);
    uint64_t n = 0;
    in.read((char*)&n, 8);
    const size_t old = sj.size();
    sj.resize(old + n);
    if (n) in.read((char*)(sj.data() + old), n * sizeof(Junction));
    return in.good();
}

// bamSortByCoordinate.cpp / BAMbinSortByCoordinate.cpp:49-55 / BAMbinSortUnmapped.cpp: mapped records by (refID<<32|pos, read-order key,
// emission order), then the unmapped ones (refID = -1 sorts last) in read order.  The reference bins by coordinate and sorts bin by
// bin on disk; one stable in-memory sort gives the same sequence.
static void writeSortedBam(const HostParams& P, const OutputWriter& W, const std::vector<std::string>& coordBlobs, std::vector<CoordRec>& coordIndex, int nT) {
    std::stable_sort(coordIndex.begin(), coordIndex.end(), [](const CoordRec& a, const CoordRec& b) { return a.alignG != b.alignG ? a.alignG < b.alignG : a.key < b.key; });
    std::ofstream cbFile;
    if (P.outStd != "BAM_SortedByCoordinate") cbFile.open(P.outFileNamePrefix + "Aligned.sortedByCoord.out.bam", std::ios::binary);   // Parameters.cpp:642-644
    std::ostream& cb = P.outStd == "BAM_SortedByCoordinate" ? static_cast<std::ostream&>(std::cout) : cbFile;
    { std::string z; const std::string h = W.bamHeader(true); OutputWriter::bgzfCompress(h.data(), h.size(), P.outBAMcompression, z); cb.write(z.data(), z.size()); }
    const size_t nRec = coordIndex.size();
    const size_t batch = 1u << 16;   // records per compression task
    for (size_t base = 0; base < nRec; base += batch * (size_t)nT) {
        std::vector<std::string> z(nT);
        auto cw = [&](int t) {
            const size_t lo = std::min(nRec, base + batch * (size_t)t), hi = std::min(nRec, lo + batch);
            std::string raw;
            for (size_t q = lo; q < hi; q++) raw.append(coordBlobs[coordIndex[q].blob], coordIndex[q].off, coordIndex[q].size);
            OutputWriter::bgzfCompress(raw.data(), raw.size(), P.outBAMcompression, z[t]);
        };
        std::vector<std::thread> th;
        for (int t = 0; t < nT; t++) th.emplace_back(cw, t);
        for (auto& t : th) t.join();
        for (int t = 0; t < nT; t++) cb.write(z[t].data(), z[t].size());
    }
    size_t ne; const char* e = OutputWriter::bgzfEofBlock(ne); cb.write(e, ne);
    cb.flush();
}
// sharded runs: records + keys of one shard (and stage) for the merge
static void writeCoordShard(const std::string& path, const std::vector<std::string>& coordBlobs, const std::vector<CoordRec>& coordIndex) {
    std::ofstream o(path, std::ios::binary);
    uint64_t n = coordIndex.size();
    o.write((const char*)&n, 8);
    for (const CoordRec& r : coordIndex) { o.write((const char*)&r.alignG, 8); o.write((const char*)&r.key, 8); o.write((const char*)&r.size, 4); }
    for (const CoordRec& r : coordIndex) o.write(coordBlobs[r.blob].data() + r.off, r.size);
}
static bool readCoordShard(const std::string& path, std::vector<std::string>& coordBlobs, std::vector<CoordRec>& coordIndex) {
    std::ifstream in(path, std::ios::binary);
    if (!in.good()) return false;
    uint64_t n = 0;
    in.read((char*)&n, 8);
    const uint32_t ib = (uint32_t)coordBlobs.size();
    const size_t base = coordIndex.size();
    coordIndex.resize(base + n);
    uint64_t off = 0;
    for (uint64_t i = 0; i < n; i++) {
        CoordRec& r = coordIndex[base + i];
        in.read((char*)&r.alignG, 8); in.read((char*)&r.key, 8); in.read((char*)&r.size, 4);
        r.blob = ib; r.off = off; off += r.size;
    }
    coordBlobs.emplace_back();
    coordBlobs.back().resize(off);
    if (off) in.read(&coordBlobs.back()[0], off);
    return in.good();
}

static int mapPass(const HostParams& P, const LoadedIndex& idx, const star_engine_vtbl_t* eng, void* ectx, Stats& stats, std::vector<Junction>& allSJ,
                   std::ofstream& logMain, std::string& err, StageState& stage) {
    int rc = 0;
    const bool firstStage = stage.bySJstage != 2, lastStage = stage.bySJstage != 1;
    // the 2nd BySJout stage appends only when both stages run in this process and share the files; a sharded phase-2 process owns its
    // own ".stage2" files and must not inherit what an earlier run left under the same prefix
    const std::ios::openmode outMode = (!firstStage && stage.streamSuffix.empty()) ? (std::ios::binary | std::ios::app) : (std::ios::binary | std::ios::trunc);
    ReadsReader reader;
    if (firstStage) {
        rc = reader.open(P, err);
        if (rc) return rc;
    }
    size_t heldNext = 0;   // 2nd stage: the held chunks are the input

    OutputWriter W(P, idx);
    W.geneModel = stage.geneModel;
    W.trModel = stage.trModel;
    const bool trYes = stage.trModel != nullptr;
    std::ofstream trOut;
    std::ostream& trO = P.outStd == "BAM_Quant" ? static_cast<std::ostream&>(std::cout) : trOut;   // Parameters.cpp:908-909
    if (trYes) {   // Aligned.toTranscriptome.out.bam (Parameters.cpp:911-914)
        if (P.outStd != "BAM_Quant") trOut.open(P.outFileNamePrefix + "Aligned.toTranscriptome.out" + stage.streamSuffix + ".bam", outMode);
        if (P.gpuShardIndex == 0 && firstStage) { std::string z; const std::string h = W.bamHeaderTranscriptome(); OutputWriter::bgzfCompress(h.data(), h.size(), P.quantTranscriptomeBAMcompression, z); trO.write(z.data(), z.size()); }
    }
    const bool samYes = !(P.outSAMtype[0] == "None" || P.outSAMmode == "None");
    std::ofstream samOut;
    const bool streamYes = samYes && (P.outSAMtype[0] == "SAM" || P.outBAMunsorted);   // Aligned.out.sam / Aligned.out.bam
    const bool bamYes = samYes && P.outBAMunsorted;
    const bool coordYes = samYes && P.outBAMcoord;                                        // Aligned.sortedByCoord.out.bam, sorted at the end
    const bool unmYes = P.outReadsUnmapped == "Fastx";   // Unmapped.out.mate1/2 (Parameters.cpp:838-844); both stages of BySJout append
    std::ofstream unmOut[2];
    if (unmYes) for (unsigned m = 0; m < P.readNmates; m++)
        unmOut[m].open(P.outFileNamePrefix + "Unmapped.out" + stage.streamSuffix + ".mate" + std::to_string(m + 1), outMode);
    const bool samToStdout = (P.outStd == "SAM" && streamYes && !bamYes) || (P.outStd == "BAM_Unsorted" && bamYes);   // Parameters.cpp:634-636, 669-670
    std::ostream& samO = samToStdout ? static_cast<std::ostream&>(std::cout) : samOut;
    if (streamYes) {
        if (!samToStdout) samOut.open(P.outFileNamePrefix + "Aligned.out" + stage.streamSuffix + (bamYes ? ".bam" : ".sam"), outMode);
        if (P.gpuShardIndex == 0 && firstStage) {   // shards > 0 write records only; the merge concatenates in shard order
            if (bamYes) { std::string z; const std::string h = W.bamHeader(); OutputWriter::bgzfCompress(h.data(), h.size(), P.outBAMcompression, z); samO.write(z.data(), z.size()); }
            else samO << W.samHeader();
        }
    }

    // ---- three overlapped stages, chunks flow in input order through bounded queues (3 chunk buffers in flight):
    //   reader thread   : FASTQ/FASTA text -> ReadChunk                      (ReadAlignChunk_processChunks.cpp:11-282)
    //   this thread     : one engine call per chunk through the C-ABI        (ReadAlignChunk_mapChunk.cpp:7-128)
    //   output thread   : SAM / junction / counter formatting on runThreadN threads, ordered writes
    struct Work {
        ReadChunk chunk;
        // result buffers: page-locked when the engine offers such memory (device->host copies to pageable memory run at a fraction of
        // the link rate), sized for 5/4 records per read and grown when a chunk holds more; otherwise plain memory for the worst case
        // nReads x outFilterMultimapNmax records of 496 B, allocated once and not initialised (only the part the engine fills is ever
        // touched, so the untouched pages are never faulted in)
        star_read_result_t* results = nullptr; uint64_t resultsCap = 0; bool resultsPinned = false;
        star_align_t* aligns = nullptr; uint64_t alignsCap = 0; bool alignsPinned = false;
        uint8_t* inPin = nullptr; uint64_t inPinCap = 0, inOffAt = 0; bool inStaged = false;   // page-locked copy of the chunk's sequences + offsets (the reader's strings are pageable), made by the reader thread
        star_align_batch_t out;
        long long n = 0;          // reads in the chunk; 0 = end of input; < 0 = -STAR_EXIT_* (err holds the message)
        std::string err;
    };
    struct Queue {
        std::mutex m; std::condition_variable cv; std::deque<Work*> q;
        void push(Work* w) { { std::lock_guard<std::mutex> l(m); q.push_back(w); } cv.notify_one(); }
        Work* pop() { std::unique_lock<std::mutex> l(m); cv.wait(l, [&] { return !q.empty(); }); Work* w = q.front(); q.pop_front(); return w; }
    };
    const bool canPin = eng->host_alloc && eng->host_free && eng->download_results;
    auto hostAlloc = [&](uint64_t bytes, bool pin, bool& pinned) -> void* {
        void* p = pin ? eng->host_alloc(bytes) : nullptr;
        pinned = p != nullptr;
        return p ? p : malloc(bytes ? bytes : 1);
    };
    auto hostFree = [&](void* p, bool pinned) { if (!p) return; if (pinned) eng->host_free(p); else free(p); };
    const int NBUF = 3;
    std::vector<Work> bufs(NBUF);
    struct BufRelease {   // (runs after the three threads were joined: every return below comes after the joins)
        std::vector<Work>& b; const star_engine_vtbl_t* e;
        ~BufRelease() {
            for (Work& w : b) {
                if (w.results) { if (w.resultsPinned) e->host_free(w.results); else free(w.results); }
                if (w.aligns) { if (w.alignsPinned) e->host_free(w.aligns); else free(w.aligns); }
                if (w.inPin) e->host_free(w.inPin);
            }
        }
    } bufRelease{bufs, eng};
    Queue freeQ, mapQ, outQ;
    for (auto& wk : bufs) freeQ.push(&wk);
    // coordinate-sorted BAM: all records stay in host memory (uncompressed, ~0.55 kB per record) until the end of the run
    std::vector<std::string>& coordBlobs = stage.coordBlobs;
    std::vector<CoordRec>& coordIndex = stage.coordIndex;
    const int nT = P.stageThreads();
    double msEngine = 0, msRead = 0, msFormat = 0, msWrite = 0;
    auto now = [] { return std::chrono::steady_clock::now(); };
    const auto tPass0 = now();
    auto msSince = [&](std::chrono::steady_clock::time_point t0) { return std::chrono::duration<double, std::milli>(now() - t0).count(); };
    uint64_t nChunks = 0;
    std::atomic<bool> abortRun(false);
    std::string outErr;   // set by the output thread (junction buffer bug check)

    std::thread readerThread([&] {
        for (;;) {
            Work* wk = freeQ.pop();
            if (abortRun.load()) { wk->n = 0; mapQ.push(wk); return; }
            auto t0 = now();
            wk->err.clear();
            if (firstStage) wk->n = reader.next(wk->chunk, P.gpuChunkReads, wk->err);
            else if (heldNext < stage.held.size()) { wk->chunk = std::move(stage.held[heldNext++]); wk->n = wk->chunk.nReads; }
            else wk->n = 0;
            wk->inStaged = false;
            if (canPin && wk->n > 0) {   // sequences and offsets of the chunk through one page-locked block (the engine copies from it)
                const ReadChunk& ch = wk->chunk;
                const char* sq = ch.clipped() ? ch.seqC.data() : ch.seq.data();                 // the engine maps the clipped reads
                const uint64_t* so = ch.clipped() ? ch.seqOffC.data() : ch.seqOff.data();
                const uint64_t nOff = (uint64_t)ch.nReads * ch.nMates + 1, seqBytes = so[nOff - 1], offAt = (seqBytes + 15) & ~15ULL;
                const uint64_t need = offAt + nOff * 8;
                if (wk->inPinCap >= need) {   // (the block is allocated / grown by the engine thread, whose current device is the run's)
                    memcpy(wk->inPin, sq, seqBytes);
                    memcpy(wk->inPin + offAt, so, nOff * 8);
                    wk->inOffAt = offAt; wk->inStaged = true;
                }
            }
            msRead += msSince(t0);
            const long long n = wk->n;
            mapQ.push(wk);
            if (n <= 0) return;
        }
    });
    // the alignment stream (the bulk of the output bytes) is written by its own thread, in chunk order, while the next chunk is being
    // formatted: at most two formatted chunks wait in memory
    struct WriteJob { std::vector<std::string> pieces; bool last = false; };
    std::mutex wrM; std::condition_variable wrCv; std::deque<WriteJob> wrQ;
    // the per-thread text pieces (hundreds of MB per chunk) circulate between the output thread and the writer instead of being allocated
    // and released per chunk: fresh allocations of that size are mapped, faulted in page by page and unmapped again by every chunk
    std::mutex poolM; std::vector<std::vector<std::string>> piecePool;
    std::thread writerThread([&] {
        for (;;) {
            WriteJob job;
            {
                std::unique_lock<std::mutex> l(wrM);
                wrCv.wait(l, [&] { return !wrQ.empty(); });
                job = std::move(wrQ.front());
            }
            if (!job.last) {
                auto tw0 = now();
                for (const std::string& p : job.pieces) samO.write(p.data(), p.size());
                msWrite += msSince(tw0);
                std::lock_guard<std::mutex> lp(poolM);
                piecePool.emplace_back(std::move(job.pieces));
            }
            {
                std::lock_guard<std::mutex> l(wrM);
                wrQ.pop_front();
            }
            wrCv.notify_all();
            if (job.last) return;
        }
    });
    auto pushWrite = [&](WriteJob&& job) {
        std::unique_lock<std::mutex> l(wrM);
        wrCv.wait(l, [&] { return wrQ.size() < 2; });
        wrQ.push_back(std::move(job));
        l.unlock();
        wrCv.notify_all();
    };
    std::thread outputThread([&] {
        for (;;) {
            Work* wk = outQ.pop();
            if (wk->n <= 0) { WriteJob end; end.last = true; pushWrite(std::move(end)); return; }
            if (!abortRun.load()) {
                const ReadChunk& chunk = wk->chunk;
                auto tf0 = now();
                std::vector<std::string> sam;
                {
                    std::lock_guard<std::mutex> lp(poolM);
                    if (!piecePool.empty()) { sam.swap(piecePool.back()); piecePool.pop_back(); }
                }
                sam.resize(nT);
                for (auto& piece : sam) piece.clear();   // (the capacity stays)
                std::vector<std::vector<Junction>> sj(nT);
                std::vector<Stats> st(nT);
                std::vector<std::string> cblob(coordYes ? nT : 0);
                std::vector<std::vector<uint64_t>> ckey(coordYes ? nT : 0);
                std::vector<OutputWriter::BySJoutHold> hold(stage.bySJstage == 1 ? nT : 0);
                std::vector<std::string> unm(unmYes ? 2 * nT : 0);   // [2*t + mate]
                std::vector<std::string> trb(trYes ? nT : 0);
                std::vector<double> trDraw;
                if (trYes) {   // the run's random stream is consumed read by read: draw before the ranges are formatted in parallel
                    trDraw.assign(chunk.nReads, 0.0);
                    std::uniform_real_distribution<double> u01(0.0, 1.0);
                    for (uint32_t i = 0; i < chunk.nReads; i++)
                        if (wk->out.reads[i].unmapType < 0 && !(stage.bySJstage == 1 && OutputWriter::heldBySJout(wk->out, i))) trDraw[i] = u01(stage.rngMultOrder);
                }
                std::vector<GeneCounts> gcs(stage.geneModel ? nT : 0);
                for (auto& gcT : gcs) gcT.init(stage.geneModel->geID.size());
                auto work = [&](int t) {   // contiguous read ranges; concatenated in input order below
                    uint32_t lo = (uint64_t)chunk.nReads * t / nT, hi = (uint64_t)chunk.nReads * (t + 1) / nT;
                    sam[t].reserve((size_t)(hi - lo) * 700);
                    W.formatReads(chunk, wk->out, lo, hi, sam[t], sj[t], st[t], coordYes ? &cblob[t] : nullptr, coordYes ? &ckey[t] : nullptr,
                                  stage.bySJstage == 1 ? &hold[t] : nullptr, unmYes ? &unm[2 * t] : nullptr,
                                  stage.geneModel ? &gcs[t] : nullptr, trYes ? &trb[t] : nullptr, trYes ? trDraw.data() : nullptr);
                    if (trYes) { std::string z; OutputWriter::bgzfCompress(trb[t].data(), trb[t].size(), P.quantTranscriptomeBAMcompression, z); trb[t].swap(z); }
                    if (bamYes) {   // BGZF framing in the formatting thread: complete blocks, so the per-thread pieces simply concatenate
                        std::string z;
                        z.reserve(sam[t].size() / 3);
                        OutputWriter::bgzfCompress(sam[t].data(), sam[t].size(), P.outBAMcompression, z);
                        sam[t].swap(z);
                    }
                };
                if (nT == 1) {
                    work(0);
                } else {
                    std::vector<std::thread> th;
                    for (int t = 0; t < nT; t++) th.emplace_back(work, t);
                    for (auto& t : th) t.join();
                }
                msFormat += msSince(tf0);
                for (int t = 0; t < nT; t++) {
                    allSJ.insert(allSJ.end(), sj[t].begin(), sj[t].end());
                    stats.add(st[t]);
                    if (stage.geneModel) stage.geneCounts.add(gcs[t]);
                    if (trYes) trO.write(trb[t].data(), trb[t].size());
                    if (unmYes) for (unsigned m = 0; m < P.readNmates; m++) unmOut[m].write(unm[2 * t + m].data(), unm[2 * t + m].size());
                    if (stage.bySJstage == 1) {
                        stage.sjAll.insert(stage.sjAll.end(), hold[t].sjAll.begin(), hold[t].sjAll.end());
                        for (uint32_t i : hold[t].held) holdRead(stage.held, chunk, i, P.gpuChunkReads);
                    }
                    if (coordYes && !cblob[t].empty()) {   // index the records of this piece (BAMoutput::coordOneAlign: key = refID<<32 | pos)
                        const uint32_t ib = (uint32_t)coordBlobs.size();
                        coordBlobs.emplace_back();
                        coordBlobs.back().swap(cblob[t]);
                        const std::string& b = coordBlobs.back();
                        size_t o = 0, k = 0;
                        while (o < b.size()) {
                            uint32_t w[3]; memcpy(w, b.data() + o, 12);
                            CoordRec cr; cr.alignG = ((uint64_t)w[1] << 32) | w[2]; cr.key = ckey[t][k++]; cr.blob = ib; cr.size = 4 + w[0]; cr.off = o;
                            coordIndex.push_back(cr);
                            o += cr.size;
                        }
                    }
                }
                if (streamYes) { WriteJob job; job.pieces.swap(sam); pushWrite(std::move(job)); }
                if (allSJ.size() > 4000000) {  // ReadAlignChunk_mapChunk.cpp:66-86 collapses when the buffer fills
                    std::string e2;
                    OutputWriter::collapseSJ(allSJ, e2);
                    if (!e2.empty()) { outErr = e2; abortRun.store(true); }
                }
                if (stage.sjAll.size() > 4000000) {
                    std::string e2;
                    OutputWriter::collapseSJ(stage.sjAll, e2);
                    if (!e2.empty()) { outErr = e2; abortRun.store(true); }
                }
            }
            freeQ.push(wk);
        }
    });
    int runRc = 0;
    std::string runErr;
    for (;;) {
        Work* wk = mapQ.pop();
        if (wk->n <= 0 || abortRun.load()) {
            if (wk->n < 0 && !runRc) { runRc = (int)-wk->n; runErr = wk->err; }
            abortRun.store(abortRun.load() || wk->n < 0);
            wk->n = 0;
            outQ.push(wk);      // end marker for the output thread
            break;
        }
        const ReadChunk& chunk = wk->chunk;
        star_read_batch_t in;
        in.nReads = chunk.nReads; in.nMates = chunk.nMates; in.seq = chunk.seq.data(); in.seqOff = chunk.seqOff.data();
        if (chunk.clipped()) { in.seq = chunk.seqC.data(); in.seqOff = chunk.seqOffC.data(); }   // the engine maps the clipped reads
        const uint64_t capWorst = (uint64_t)chunk.nReads * std::max<uint64_t>(1, P.hp.outFilterMultimapNmax);
        auto growAligns = [&](uint64_t cap) {   // false: out of memory
            if (wk->alignsCap >= cap) return true;
            hostFree(wk->aligns, wk->alignsPinned);
            wk->aligns = (star_align_t*)hostAlloc(cap * sizeof(star_align_t), canPin, wk->alignsPinned);
            wk->alignsCap = wk->aligns ? cap : 0;
            return wk->aligns != nullptr;
        };
        static const uint64_t pinPct = [] { const char* e = getenv("STAR_B200_PINNED_ALIGNS_PCT"); const long v = e ? atol(e) : 0; return (uint64_t)(v > 0 ? v : 125); }();   // records per 100 reads the first page-locked buffer holds
        bool memOk = growAligns(canPin ? std::min<uint64_t>(capWorst, (uint64_t)chunk.nReads * pinPct / 100 + 64) : capWorst);
        if (wk->resultsCap < chunk.nReads) {
            hostFree(wk->results, wk->resultsPinned);
            wk->resultsCap = std::max<uint64_t>(chunk.nReads, P.gpuChunkReads);
            wk->results = (star_read_result_t*)hostAlloc(wk->resultsCap * sizeof(star_read_result_t), canPin, wk->resultsPinned);
            if (!wk->results) { wk->resultsCap = 0; memOk = false; }
        }
        if (canPin && !wk->inStaged) {   // first chunk through this buffer, or a chunk larger than all before: (re)allocate the page-locked block here
            const uint64_t nOff = (uint64_t)in.nReads * in.nMates + 1, seqBytes = in.seqOff[nOff - 1], offAt = (seqBytes + 15) & ~15ULL;
            const uint64_t need = offAt + nOff * 8;
            if (wk->inPinCap < need) {
                eng->host_free(wk->inPin);
                wk->inPinCap = need + need / 8;
                wk->inPin = (uint8_t*)eng->host_alloc(wk->inPinCap);
                if (!wk->inPin) wk->inPinCap = 0;
            }
            if (wk->inPin) {
                memcpy(wk->inPin, in.seq, seqBytes);
                memcpy(wk->inPin + offAt, in.seqOff, nOff * 8);
                wk->inOffAt = offAt; wk->inStaged = true;
            }
        }
        if (wk->inStaged) { in.seq = (const char*)wk->inPin; in.seqOff = (const uint64_t*)(wk->inPin + wk->inOffAt); }   // (normally copied by the reader thread)
        wk->out.reads = wk->results; wk->out.aligns = wk->aligns; wk->out.alignsCapacity = wk->alignsCap; wk->out.nAligns = 0;
        star_chunk_stats_t cs;
        memset(&cs, 0, sizeof(cs));
        rc = memOk ? eng->map_chunk(ectx, &in, &wk->out, &cs) : STAR_EXIT_RUNTIME;
        if (rc && memOk && canPin && wk->out.nAligns > wk->alignsCap) {   // more records than the page-locked buffer holds: grow it, fetch again
            const uint64_t needed = wk->out.nAligns;
            memOk = growAligns(std::min<uint64_t>(capWorst, needed + needed / 4));
            if (memOk) {
                wk->out.aligns = wk->aligns; wk->out.alignsCapacity = wk->alignsCap; wk->out.nAligns = 0;
                rc = eng->download_results(ectx, &wk->out);
            }
        }
        if (!memOk) {
            runRc = STAR_EXIT_RUNTIME; runErr = "EXITING because of fatal ERROR: not enough memory for the chunk buffers of the mapping pass\n";
            abortRun.store(true);
            wk->n = 0;
            outQ.push(wk);
            break;
        }
        if (rc) {
            runRc = rc; runErr = eng->last_error();
            abortRun.store(true);
            wk->n = 0;
            outQ.push(wk);
            break;
        }
        msEngine += cs.ms_total;
        nChunks++;
        outQ.push(wk);
    }
    outputThread.join();
    writerThread.join();
    if (abortRun.load()) {   // release a reader that may be waiting for a free buffer
        for (auto& wk : bufs) freeQ.push(&wk);
    }
    readerThread.join();
    if (runRc) { err = runErr; return runRc; }
    if (!outErr.empty()) { err = outErr; return STAR_EXIT_BUG; }
    if (trYes && P.gpuShardCount == 1 && lastStage) { size_t ne; const char* e = OutputWriter::bgzfEofBlock(ne); trO.write(e, ne); trO.flush(); }
    if (bamYes && P.gpuShardCount == 1 && lastStage) { size_t ne; const char* e = OutputWriter::bgzfEofBlock(ne); samO.write(e, ne); }   // (sharded runs: the merge appends it)
    if (streamYes) { samO.flush(); if (!samToStdout) samOut.close(); }
    if (coordYes && P.gpuShardCount > 1) {   // one shard: the (unsorted) records and their keys go to the merge, which sorts the whole run
        writeCoordShard(P.outFileNamePrefix + "coord" + stage.streamSuffix + ".bin", coordBlobs, coordIndex);
    } else if (coordYes && lastStage) {
        time_t ts; time(&ts);
        *g_logStd << timeMonthDayTime(ts) << " ..... started sorting BAM\n" << std::flush;
        writeSortedBam(P, W, coordBlobs, coordIndex, nT);
    }
    logMain << "star-b200: engine time " << msEngine << " ms over " << nChunks << " chunks; mapping pass wall " << msSince(tPass0) << " ms\n";
    logMain << "star-b200: host stages used " << nT << " threads each (--runThreadN " << P.runThreadN << ", CPUs allowed to this process " << HostParams::allowedCpus() << ")\n";
    logMain << "star-b200: host time: reads input " << msRead << " ms, SAM/SJ formatting " << msFormat << " ms, output writes " << msWrite << " ms\n";
    return 0;
}

static int runAlign(int argc, char** argv, const star_engine_vtbl_t* eng) {
    HostParams P;
    std::string err;
    Stats stats;
    time(&stats.timeStart);
    int rc = parseCommandLine(argc, argv, P, err);
    if (rc == -1 && err == "version") { std::cout << "2.7.11b" << std::endl; return 0; }
    auto exitWithError = [&](const std::string& msg, int code, std::ofstream* logMain) {  // ErrorWarning.cpp:8-23
        time_t t; time(&t);
        if (logMain && logMain->is_open()) *logMain << "\n" << msg << "\n" << timeMonthDayTime(t) << " ...... FATAL ERROR, exiting\n" << std::flush;
        std::cerr << "\n" << msg << "\n" << timeMonthDayTime(t) << " ...... FATAL ERROR, exiting\n" << std::flush;
        return code;
    };
    if (rc) return exitWithError(err, rc, nullptr);
    makeDirs(P.outFileNamePrefix);
    std::ofstream logMain(P.outFileNamePrefix + "Log.out");
    if (logMain.fail())
        return exitWithError("EXITING because of FATAL ERROR: could not create output file: " + P.outFileNamePrefix + "Log.out\nSOLUTION: check if the path " + P.outFileNamePrefix + " exists and you have permissions to write there\n", STAR_EXIT_PARAMETER, nullptr);
    g_logStd = &std::cout;
    if (P.outStd != "Log") {
        if (g_logStdFile.is_open()) g_logStdFile.close();
        g_logStdFile.open(P.outFileNamePrefix + "Log.std.out");
        g_logStd = &g_logStdFile;
    }
    logMain << "STAR version=2.7.11b (star-b200 GPU alignment hot path)\n##### Command Line:\n" << P.commandLine << "\n##### Final effective command line:\n" << P.commandLineFull << "\n" << std::flush;
    for (const std::string& ip : P.ignoredParams) logMain << "star-b200: --" << ip << " is accepted and has no effect (no host-side buffer / temporary-file limits)\n";
    *g_logStd << "\t" << P.commandLine << "\n\tSTAR version: 2.7.11b (star-b200)\n" << timeMonthDayTime(stats.timeStart) << " ..... started STAR run\n" << std::flush;

    if (P.runMode == "inputAlignmentsFromBAM") {   // Parameters.cpp:585-607: the signal tracks if asked for, else duplicate marking
        time_t t; time(&t);
        const char* what = P.wigYes ? " ..... reading from BAM, output wiggle\n" : " ..... reading from BAM, remove duplicates, output BAM\n";
        *g_logStd << timeMonthDayTime(t) << what << std::flush;
        logMain << timeMonthDayTime(t) << what << std::flush;
        rc = P.wigYes ? signalFromBAMfile(P, eng, logMain, err) : dedupFromBAMfile(P, eng, logMain, err);
        if (rc) return exitWithError(err, rc, &logMain);
        time(&t);
        *g_logStd << timeMonthDayTime(t) << " ..... done\n" << std::flush;
        logMain << timeMonthDayTime(t) << " ..... done\n" << std::flush;
        return 0;
    }
    if (P.runMode == "genomeGenerate") {   // STAR.cpp:120-125
        rc = genomeGenerate(P, eng, logMain, err);
        if (rc) return exitWithError(err, rc, &logMain);
        logMain << "DONE: Genome generation, EXITING\n" << std::flush;
        return 0;
    }
    {
        time_t t; time(&t);
        *g_logStd << timeMonthDayTime(t) << " ..... loading genome\n" << std::flush;
    }
    LoadedIndex idx;
    std::string glog;
    rc = loadIndex(P.genomeDir, &P.hp, idx, err, &glog);
    logMain << glog << std::flush;
    if (rc) return exitWithError(err, rc, &logMain);
    // ---- references added at the mapping stage (Genome_genomeLoad.cpp:374): before any junction insertion, so that the junctions and the
    // GTF may name them; a 2-pass run maps both passes against the grown index
    rc = addReferences(P, &P.hp, idx, eng, logMain, err);
    if (rc) return exitWithError(err, rc, &logMain);

    // ---- on-the-fly junction insertion (STAR.cpp:145-150) and the 1st pass of --twopassMode Basic (twoPassRunPass1.cpp:9-96)
    SjdbLoci sjdbLoci;
    if (P.sjdbInsertYes) {
        if (idx.sjdbInfoExists && idx.sjdbInsertSaveGenome.empty())   // Genome_genomeLoad.cpp:95-101
            return exitWithError("EXITING because of FATAL ERROR: old Genome is INCOMPATIBLE with on the fly junction insertion\nSOLUTION: please re-generate genome from scratch with the latest version of STAR\n", STAR_EXIT_GENOME_FILES, &logMain);
        uint64_t ov = P.sjdbOverhang;                                  // Genome_genomeLoad.cpp:113-125
        if (!P.userSet.count("sjdbOverhang") && idx.sjdbOverhangGenome > 0) {
            ov = idx.sjdbOverhangGenome;
            logMain << "--sjdbOverhang = " << ov << " taken from the generated genome\n";
        } else if (idx.sjdbInfoExists && P.userSet.count("sjdbOverhang") && ov != idx.sjdbOverhangGenome)
            return exitWithError("EXITING because of fatal PARAMETERS error: present --sjdbOverhang=" + std::to_string(ov) + " is not equal to the value at the genome generation step =" + std::to_string(idx.sjdbOverhangGenome) + "\nSOLUTION: \n", STAR_EXIT_GENOME_FILES, &logMain);
        idx.view.sjdbOverhang = ov;
        idx.view.sjdbLength = 2 * ov + 1;
        for (const std::string* d : {&P.sjdbInsertOutDir, &P.twoPassDir}) {   // Parameters.cpp:817-825, 1027-1035: fresh run-time directories
            if (d->empty()) continue;
            if (d == &P.twoPassDir && P.gpuTwoPassPhase == 2) continue;        // holds the gathered 1st-pass junctions of all shards
            std::error_code ec;
            std::filesystem::remove_all(*d, ec);
            if (mkdir(d->c_str(), 0700) != 0)
                return exitWithError("EXITING because of fatal ERROR: could not make run-time directory: " + *d + "\nSOLUTION: please check the path and writing permissions \n", STAR_EXIT_PARAMETER, &logMain);
        }
    }
    if (P.sjdbInsertPass1) {
        rc = sjdbInsertJunctions(P, &P.hp, idx, sjdbLoci, false, "", eng, logMain, err);
        if (rc) return exitWithError(err, rc, &logMain);
    }
    void* ectx = nullptr;
    if (!(P.twoPassYes && P.gpuTwoPassPhase == 2)) {   // (phase 2 of a sharded 2-pass run goes straight to the insertion)
        rc = eng->init(&ectx, P.gpuDevice, &idx.view, &P.hp, P.gpuChunkReads);
        if (rc) return exitWithError(std::string("EXITING because of FATAL ERROR: engine initialisation failed: ") + eng->last_error() + "\n", rc, &logMain);
    }
    std::ofstream logProgress(P.outFileNamePrefix + "Log.progress.out");
    if (P.twoPassYes && P.gpuTwoPassPhase != 2) {
        HostParams P1 = P;   // outputs off, files into _STARpass1/ (twoPassRunPass1.cpp:17-47)
        P1.outSAMtype = {"None"}; P1.outBAMunsorted = false; P1.outBAMcoord = false; P1.unmappedWithin = false; P1.unmappedKeepPairs = false;
        P1.outFileNamePrefix = P.twoPassDir;
        P1.outReadsUnmapped = "None";   // twoPassRunPass1.cpp:24-33: no unmapped-read files, no quantification in the 1st pass
        const uint64_t nMax = std::min<uint64_t>(P.twopass1readsN, (uint64_t)P.readMapNumber);
        P1.readMapNumber = nMax > (uint64_t)INT64_MAX ? -1 : (long long)nMax;
        Stats st1;
        st1.timeStart = stats.timeStart;
        time(&st1.timeStartMap);
        *g_logStd << timeMonthDayTime(st1.timeStartMap) << " ..... started 1st pass mapping\n" << std::flush;
        std::vector<Junction> sj1;
        StageState stage1;
        rc = mapPass(P1, idx, eng, ectx, st1, sj1, logMain, err, stage1);
        eng->destroy(ectx);
        if (rc) return exitWithError(err, rc, &logMain);
        time(&st1.timeFinish);
        if (P.gpuTwoPassPhase == 1) {   // one shard of a multi-GPU run: the junction records go to the gather (star_b200.dist), nothing else to do here
            std::string e2;
            OutputWriter::collapseSJ(sj1, e2);
            if (!e2.empty()) return exitWithError(e2, STAR_EXIT_BUG, &logMain);
            writeShardBin(P.twoPassDir + "shard.bin", st1, sj1);
            *g_logStd << timeMonthDayTime(st1.timeFinish) << " ..... finished 1st pass of shard " << P.gpuShardIndex << " of " << P.gpuShardCount << "\n" << std::flush;
            return 0;
        }
        OutputWriter W1(P1, idx);
        std::string e2 = W1.writeSJ(sj1, P.twoPassDir + "SJ.out.tab");
        if (!e2.empty()) return exitWithError(e2, STAR_EXIT_BUG, &logMain);
        *g_logStd << timeMonthDayTime(st1.timeFinish) << " ..... finished 1st pass mapping\n" << std::flush;
        W1.writeLogFinal(st1, P.twoPassDir + "Log.final.out");
    }   // (phase 2: the 1st pass was a separate run; star_b200.dist gathered the junctions of all shards into _STARpass1/SJ.out.tab)
    if (P.twoPassYes) {
        rc = sjdbInsertJunctions(P, &P.hp, idx, sjdbLoci, true, P.twoPassDir + "SJ.out.tab", eng, logMain, err);
        if (rc) return exitWithError(err, rc, &logMain);
        rc = eng->init(&ectx, P.gpuDevice, &idx.view, &P.hp, P.gpuChunkReads);   // the index with the inserted junctions becomes resident
        if (rc) return exitWithError(std::string("EXITING because of FATAL ERROR: engine initialisation failed: ") + eng->last_error() + "\n", rc, &logMain);
    }
    time(&stats.timeStartMap);
    *g_logStd << timeMonthDayTime(stats.timeStartMap) << " ..... started mapping\n" << std::flush;
    std::vector<Junction> allSJ;
    StageState stage;
    OutputWriter W(P, idx);
    GeneModel geneModel;
    if (P.quantGeneCounts) {   // the tables of the index, or of the GTF given at the mapping stage (Transcriptome.cpp:13)
        rc = geneModel.load(P.sjdbGTFfile == "-" ? P.genomeDir : P.sjdbInsertOutDir, err);
        if (rc) { eng->destroy(ectx); return exitWithError(err, rc, &logMain); }
        stage.geneModel = &geneModel;
        stage.geneCounts.init(geneModel.geID.size());
    }
    TranscriptModel trModel;
    if (P.quantTrSAM) {
        rc = trModel.load(P.sjdbGTFfile == "-" ? P.genomeDir : P.sjdbInsertOutDir, err);
        if (rc) { eng->destroy(ectx); return exitWithError(err, rc, &logMain); }
        stage.trModel = &trModel;
        stage.rngMultOrder.seed((uint32_t)(P.runRNGseed * (P.gpuShardIndex + 1)));   // thread iChunk of the reference: runRNGseed*(iChunk+1)
    }
    const bool bySJout = P.outFilterType == "BySJout";
    stage.bySJstage = bySJout ? 1 : 0;
    const std::string stateFile = P.outFileNamePrefix + "bysj_stage1.bin";
    if (!(bySJout && P.gpuBySJoutPhase == 2)) rc = mapPass(P, idx, eng, ectx, stats, allSJ, logMain, err, stage);
    if (!rc && bySJout && P.gpuBySJoutPhase == 1) {   // one shard of a multi-GPU run: the junction records of ALL its reads go to the gather
        std::string e2;
        OutputWriter::collapseSJ(stage.sjAll, e2);
        if (e2.empty()) OutputWriter::collapseSJ(allSJ, e2);
        eng->destroy(ectx);
        if (!e2.empty()) return exitWithError(e2, STAR_EXIT_BUG, &logMain);
        time(&stats.timeFinish);
        saveStage1(stateFile, stats, allSJ, stage.held);
        if (stage.geneModel) stage.geneCounts.write(geneModel, stats, P.outFileNamePrefix + "bysj_stage1.ReadsPerGene.tab");
        writeShardBin(P.outFileNamePrefix + "bysj_sjall.bin", stats, stage.sjAll);
        *g_logStd << timeMonthDayTime(stats.timeFinish) << " ..... finished 1st BySJout stage of shard " << P.gpuShardIndex << " of " << P.gpuShardCount << "\n" << std::flush;
        return 0;
    }
    if (!rc && bySJout && P.gpuBySJoutPhase == 2) {   // ... and come back from every shard (star_b200.dist: bysj_gather<r>.bin)
        const time_t t0 = stats.timeStart;
        if (!loadStage1(stateFile, stats, allSJ, stage.held)) { rc = STAR_EXIT_RUNTIME; err = "EXITING because of FATAL ERROR: missing 1st-stage state " + stateFile + "\n"; }
        stats.timeStart = t0;
        for (unsigned r = 0; r < P.gpuShardCount && !rc; r++)
            if (!readShardJunctions(P.outFileNamePrefix + "bysj_gather" + std::to_string(r) + ".bin", stage.sjAll)) {
                rc = STAR_EXIT_RUNTIME; err = "EXITING because of FATAL ERROR: missing gathered junctions " + P.outFileNamePrefix + "bysj_gather" + std::to_string(r) + ".bin\n";
            }
        stage.streamSuffix = ".stage2";
        if (stage.geneModel && !rc) readGeneCounts(P.outFileNamePrefix + "bysj_stage1.ReadsPerGene.tab", stage.geneCounts);
    }
    if (!rc && bySJout) {   // STAR.cpp:203-220: the novel junctions that pass the filters over ALL reads, then the held reads once more
        logMain << "Completed stage 1 mapping of outFilterBySJout mapping\n" << std::flush;
        std::vector<uint64_t> njS, njE;
        std::string e2 = W.novelJunctions(stage.sjAll, njS, njE);
        if (!e2.empty()) { eng->destroy(ectx); return exitWithError(e2, STAR_EXIT_BUG, &logMain); }
        logMain << "Detected " << njS.size() << " novel junctions that passed filtering, will proceed to filter reads that contained unannotated junctions" << std::endl;
        rc = eng->set_sj_novel(ectx, njS.data(), njE.data(), njS.size());
        if (rc) err = std::string("EXITING because of FATAL ERROR: ") + eng->last_error() + "\n";
        stage.bySJstage = 2;
        if (!rc) rc = mapPass(P, idx, eng, ectx, stats, allSJ, logMain, err, stage);
    }
    eng->destroy(ectx);
    if (rc) return exitWithError(err, rc, &logMain);
    {
        time_t tFinishMap; time(&tFinishMap);
        *g_logStd << timeMonthDayTime(tFinishMap) << " ..... finished mapping\n" << std::flush;
        logMain << timeMonthDayTime(tFinishMap) << " ..... finished mapping\n";
    }
    if (P.wigYes && P.gpuShardCount == 1) {   // STAR.cpp:274-283, from the sorted records still in memory (sharded runs: star_b200.dist after the merge)
        time_t t; time(&t);
        *g_logStd << timeMonthDayTime(t) << " ..... started wiggle output\n" << std::flush;
        logMain << timeMonthDayTime(t) << " ..... started wiggle output\n" << std::flush;
        std::vector<const uint8_t*> recs(stage.coordIndex.size());
        for (size_t i = 0; i < recs.size(); i++) recs[i] = (const uint8_t*)stage.coordBlobs[stage.coordIndex[i].blob].data() + stage.coordIndex[i].off;
        std::vector<uint32_t> lens(idx.chrName.size());
        for (size_t i = 0; i < lens.size(); i++) lens[i] = (uint32_t)idx.view.chrLength[i];
        rc = signalFromRecords(P, eng, idx.chrName, lens, recs, logMain, err);
        if (rc) return exitWithError(err, rc, &logMain);
    }
    time(&stats.timeFinish);
    if (stage.geneModel) stage.geneCounts.write(geneModel, stats, P.outFileNamePrefix + "ReadsPerGene.out.tab");   // STAR.cpp:258-265 (a shard: its part)
    if (P.gpuShardCount > 1) {
        // one shard of a multi-GPU run: leave the counters and the (collapsed) junction records for the merge
        // (SURVEY.md §8e: the neighbour-distance filter of outputSJ needs the GLOBAL sorted junction list)
        std::string e2;
        OutputWriter::collapseSJ(allSJ, e2);
        if (!e2.empty()) return exitWithError(e2, STAR_EXIT_BUG, &logMain);
        writeShardBin(P.outFileNamePrefix + "shard.bin", stats, allSJ);
        *g_logStd << timeMonthDayTime(stats.timeFinish) << " ..... finished shard " << P.gpuShardIndex << " of " << P.gpuShardCount << "\n" << std::flush;
        logMain << "ALL DONE!\n" << std::flush;
        return 0;
    }
    if (P.outSJyes) {
        std::string e2 = W.writeSJ(allSJ, P.outFileNamePrefix + "SJ.out.tab", /*distFilter*/ !bySJout);
        if (!e2.empty()) return exitWithError(e2, STAR_EXIT_BUG, &logMain);
    }
    W.writeLogFinal(stats, P.outFileNamePrefix + "Log.final.out");
    *g_logStd << timeMonthDayTime(stats.timeFinish) << " ..... finished successfully\n" << std::flush;
    logMain << "ALL DONE!\n" << std::flush;
    return 0;
}

// Merge of a sharded (multi-GPU) run: shard r wrote <prefix>shard<r>.{Aligned.out.sam,shard.bin}.  counters = the 24 Log.final.out
// counters after the allreduce over ranks (NULL: sum the shard files).  Writes <prefix>Aligned.out.sam, SJ.out.tab, Log.final.out.
static int mergeShards(int argc, char** argv, int nShards, const uint64_t* counters) {
    HostParams P;
    std::string err;
    int rc = parseCommandLine(argc, argv, P, err);
    if (rc) { std::cerr << err << std::endl; return rc; }
    LoadedIndex idx;
    rc = loadIndex(P.genomeDir, &P.hp, idx, err, nullptr, true);
    if (rc) { std::cerr << err << std::endl; return rc; }
    {   // the references every shard added: names and lengths only
        std::ostringstream addLog;
        rc = addReferences(P, &P.hp, idx, nullptr, addLog, err, true);
        if (rc) { std::cerr << err << std::endl; return rc; }
    }
    OutputWriter W(P, idx);
    Stats total;
    std::vector<Junction> allSJ;
    int64_t tStart = 0, tStartMap = 0, tFinish = 0;
    const bool samYes = !(P.outSAMtype[0] == "None" || P.outSAMmode == "None");
    const bool bySJ = P.outFilterType == "BySJout";   // only then do the shards hold ".stage2" parts
    const std::string alnName = P.outBAMunsorted ? "Aligned.out.bam" : "Aligned.out.sam";
    std::ofstream samOut;
    const bool streamYes = samYes && (P.outSAMtype[0] == "SAM" || P.outBAMunsorted);
    if (streamYes) samOut.open(P.outFileNamePrefix + alnName, std::ios::binary);
    for (int r = 0; r < nShards; r++) {
        std::string sp = P.outFileNamePrefix + "shard" + std::to_string(r) + ".";
        std::ifstream sb(sp + "shard.bin", std::ios::binary);
        if (!sb.good()) { std::cerr << "EXITING because of FATAL ERROR: missing shard output " << sp << "shard.bin\n"; return STAR_EXIT_RUNTIME; }
        uint64_t cnt[Stats::N_COUNTERS]; int64_t tm[3]; uint64_t nsj = 0;
        sb.read((char*)cnt, sizeof(cnt)); sb.read((char*)tm, sizeof(tm)); sb.read((char*)&nsj, 8);
        Stats s1; s1.fromArray(cnt); total.add(s1);
        if (r == 0 || tm[0] < tStart) tStart = tm[0];
        if (r == 0 || tm[1] < tStartMap) tStartMap = tm[1];
        if (tm[2] > tFinish) tFinish = tm[2];
        size_t old = allSJ.size();
        allSJ.resize(old + nsj);
        if (nsj) sb.read((char*)(allSJ.data() + old), nsj * sizeof(Junction));
        if (streamYes) {
            std::ifstream in(sp + alnName, std::ios::binary);
            samOut << in.rdbuf();
            samOut.clear();   // an empty shard sets failbit on operator<<
        }
    }
    if (streamYes && P.outFilterType == "BySJout")   // the reference writes the reads held by the 1st stage after all others
        for (int r = 0; r < nShards; r++) {
            std::ifstream in(P.outFileNamePrefix + "shard" + std::to_string(r) + ".Aligned.out.stage2" + (P.outBAMunsorted ? ".bam" : ".sam"), std::ios::binary);
            samOut << in.rdbuf();
            samOut.clear();
        }
    if (samYes && P.outBAMunsorted) { size_t ne; const char* e = OutputWriter::bgzfEofBlock(ne); samOut.write(e, ne); }
    if (P.quantTrSAM) {   // Aligned.toTranscriptome.out.bam: header of shard 0, then the parts in the reference's order
        std::ofstream to(P.outFileNamePrefix + "Aligned.toTranscriptome.out.bam", std::ios::binary);
        for (const char* part : {"", ".stage2"})
            for (int r = 0; r < nShards && (part[0] == 0 || bySJ); r++) {
                std::ifstream in(P.outFileNamePrefix + "shard" + std::to_string(r) + ".Aligned.toTranscriptome.out" + part + ".bam", std::ios::binary);
                if (in.good()) { to << in.rdbuf(); to.clear(); }
            }
        size_t ne; const char* e = OutputWriter::bgzfEofBlock(ne); to.write(e, ne);
    }
    if (P.outReadsUnmapped == "Fastx")
        for (unsigned m = 0; m < P.readNmates; m++) {
            std::ofstream uo(P.outFileNamePrefix + "Unmapped.out.mate" + std::to_string(m + 1), std::ios::binary);
            for (const char* part : {"", ".stage2"})
                for (int r = 0; r < nShards && (part[0] == 0 || bySJ); r++) {
                    std::ifstream in(P.outFileNamePrefix + "shard" + std::to_string(r) + ".Unmapped.out" + part + ".mate" + std::to_string(m + 1), std::ios::binary);
                    if (in.good()) { uo << in.rdbuf(); uo.clear(); }
                }
        }
    if (samYes && P.outBAMcoord) {   // Aligned.sortedByCoord.out.bam of the whole run: the shards' records (both BySJout stages), one stable sort
        std::vector<std::string> blobs;
        std::vector<CoordRec> index;
        for (int r = 0; r < nShards; r++)
            for (const char* part : {"coord.bin", "coord.stage2.bin"}) {
                if (!bySJ && std::string(part) != "coord.bin") continue;   // stage-2 parts exist only in a BySJout run; never pick up leftovers
                const std::string fn = P.outFileNamePrefix + "shard" + std::to_string(r) + "." + part;
                if (!readCoordShard(fn, blobs, index) && std::string(part) == "coord.bin" && !(P.outFilterType == "BySJout")) {
                    std::cerr << "EXITING because of FATAL ERROR: missing shard output " << fn << "\n";
                    return STAR_EXIT_RUNTIME;
                }
            }
        writeSortedBam(P, W, blobs, index, std::max(1, P.runThreadN));
    }
    if (counters) total.fromArray(counters);
    total.timeStart = (time_t)tStart; total.timeStartMap = (time_t)tStartMap; total.timeFinish = (time_t)tFinish;
    if (P.outSJyes) {
        std::string e2 = W.writeSJ(allSJ, P.outFileNamePrefix + "SJ.out.tab", P.outFilterType != "BySJout");
        if (!e2.empty()) { std::cerr << e2 << std::endl; return STAR_EXIT_BUG; }
    }
    W.writeLogFinal(total, P.outFileNamePrefix + "Log.final.out");
    if (P.quantGeneCounts) {   // ReadsPerGene.out.tab of the run = the sum of the shards' tables
        GeneModel gm;
        rc = gm.load(P.sjdbGTFfile == "-" ? P.genomeDir : P.outFileNamePrefix + "shard0._STARgenome/", err);
        if (rc) { std::cerr << err << std::endl; return rc; }
        GeneCounts gc;
        gc.init(gm.geID.size());
        for (int r = 0; r < nShards; r++)
            if (!readGeneCounts(P.outFileNamePrefix + "shard" + std::to_string(r) + ".ReadsPerGene.out.tab", gc)) { std::cerr << "EXITING because of FATAL ERROR: missing gene counts of shard " << r << "\n"; return STAR_EXIT_RUNTIME; }
        gc.write(gm, total, P.outFileNamePrefix + "ReadsPerGene.out.tab");
    }
    return 0;
}

// 1st pass of a sharded 2-pass run: `dir`/gather<r>.bin (r < nShards) hold the shard.bin payloads of ALL shards, as gathered over
// the collective by star_b200.dist.  Every rank calls this with its own directory and gets the same global junction list:
// `dir`/SJ.out.tab (the collapse + filters of outputSJ.cpp:20-200 over all shards) and `dir`/Log.final.out (summed counters).
static int mergePass1(int argc, char** argv, int nShards, const char* dir) {
    HostParams P;
    std::string err;
    int rc = parseCommandLine(argc, argv, P, err);
    if (rc) { std::cerr << err << std::endl; return rc; }
    LoadedIndex idx;
    rc = loadIndex(P.genomeDir, &P.hp, idx, err, nullptr, true);
    if (rc) { std::cerr << err << std::endl; return rc; }
    {   // the references every shard added: names and lengths only
        std::ostringstream addLog;
        rc = addReferences(P, &P.hp, idx, nullptr, addLog, err, true);
        if (rc) { std::cerr << err << std::endl; return rc; }
    }
    P.outSAMtype = {"None"};
    OutputWriter W(P, idx);
    Stats total;
    std::vector<Junction> allSJ;
    int64_t tStart = 0, tStartMap = 0, tFinish = 0;
    for (int r = 0; r < nShards; r++) {
        const std::string fn = std::string(dir) + "gather" + std::to_string(r) + ".bin";
        std::ifstream sb(fn, std::ios::binary);
        if (!sb.good()) { std::cerr << "EXITING because of FATAL ERROR: missing gathered 1st-pass junctions " << fn << "\n"; return STAR_EXIT_RUNTIME; }
        uint64_t cnt[Stats::N_COUNTERS]; int64_t tm[3]; uint64_t nsj = 0;
        sb.read((char*)cnt, sizeof(cnt)); sb.read((char*)tm, sizeof(tm)); sb.read((char*)&nsj, 8);
        Stats s1; s1.fromArray(cnt); total.add(s1);
        if (r == 0 || tm[0] < tStart) tStart = tm[0];
        if (r == 0 || tm[1] < tStartMap) tStartMap = tm[1];
        if (tm[2] > tFinish) tFinish = tm[2];
        const size_t old = allSJ.size();
        allSJ.resize(old + nsj);
        if (nsj) sb.read((char*)(allSJ.data() + old), nsj * sizeof(Junction));
    }
    total.timeStart = (time_t)tStart; total.timeStartMap = (time_t)tStartMap; total.timeFinish = (time_t)tFinish;
    std::string e2 = W.writeSJ(allSJ, std::string(dir) + "SJ.out.tab");
    if (!e2.empty()) { std::cerr << e2 << std::endl; return STAR_EXIT_BUG; }
    W.writeLogFinal(total, std::string(dir) + "Log.final.out");
    return 0;
}

}  // namespace starhost

extern "C" int star_host_merge_pass1(int argc, char** argv, int nShards, const char* dir) { return starhost::mergePass1(argc, argv, nShards, dir); }

extern "C" int star_host_merge_shards(int argc, char** argv, int nShards, const uint64_t* counters24) {
    return starhost::mergeShards(argc, argv, nShards, counters24);
}

extern "C" int star_cli_main_engine(int argc, char** argv, const star_engine_vtbl_t* engine) { return starhost::runAlign(argc, argv, engine); }
