// signal.cpp — signal tracks (--outWigType) from coordinate-sorted records or from --inputBAMfile (reference source/signalFromBAM.cpp:5-209).
//
// The host decodes the records segment by segment (a segment = consecutive records with the same reference id: output is flushed whenever
// the id changes, so an unsorted BAM can give a chromosome twice) into blocks in record order: one block per counted M operation, or one
// base per read for read1_5p.  The engine (star_gpu_signal_segment) builds the per-base tracks and returns only where each track changes
// (bedGraph) or is nonzero (wiggle); the lines are formatted here on the stage threads, in order.
#include <zlib.h>

#include <atomic>
#include <chrono>
#include <cstring>
#include <functional>
#include <fstream>
#include <iostream>
#include <thread>

#include "host.h"

namespace starhost {

namespace {
inline uint32_t rd32(const uint8_t* p) { uint32_t v; memcpy(&v, p, 4); return v; }
inline uint16_t rd16(const uint8_t* p) { uint16_t v; memcpy(&v, p, 2); return v; }
}  // namespace

// bam_aux_get + bam_aux2i (htslib sam.c): NH of the record; 0 = no NH tag (then *has = false).  A non-integer type reads as 0.
bool auxNH(const uint8_t* rec, bool& has, uint32_t& nh) {
    const uint32_t len = rd32(rec) + 4;
    const uint8_t* end = rec + len;
    const uint32_t lName = rec[12], nCig = rd16(rec + 16), lSeq = rd32(rec + 20);
    const uint8_t* s = rec + 36 + lName + 4ull * nCig + (lSeq + 1ull) / 2 + lSeq;
    has = false; nh = 0;
    while (s < end) {
        if (end - s < 3) return false;
        const bool hit = s[0] == 'N' && s[1] == 'H';
        const uint8_t type = s[2];
        s += 3;
        if (hit) {
            has = true;
            const size_t need = type == 'c' || type == 'C' ? 1 : type == 's' || type == 'S' ? 2 : type == 'i' || type == 'I' ? 4 : 0;
            if ((size_t)(end - s) < need) return false;
            int32_t v = 0;
            if (type == 'c') v = (int8_t)s[0];
            else if (type == 'C') v = s[0];
            else if (type == 's') v = (int16_t)rd16(s);
            else if (type == 'S') v = rd16(s);
            else if (type == 'i' || type == 'I') v = (int32_t)rd32(s);
            nh = (uint32_t)v;
            return true;
        }
        switch (type) {   // skip_aux
            case 'A': case 'c': case 'C': s += 1; break;
            case 's': case 'S': s += 2; break;
            case 'i': case 'I': case 'f': s += 4; break;
            case 'd': s += 8; break;
            case 'Z': case 'H': while (s < end && *s) ++s; ++s; break;
            case 'B': {
                if (end - s < 5) return false;
                const uint8_t sub = s[0];
                const uint64_t n = rd32(s + 1);
                const int sz = sub == 'c' || sub == 'C' || sub == 'A' ? 1 : sub == 's' || sub == 'S' ? 2 : sub == 'i' || sub == 'I' || sub == 'f' ? 4 : sub == 'd' ? 8 : 0;
                if (!sz) return false;
                s += 5 + n * sz;
                break;
            }
            default: return false;   // (htslib aborts)
        }
    }
    return s <= end;
}

void parallelFor(int n, int nT, const std::function<void(int)>& fn) {
    if (nT <= 1 || n <= 1) { for (int i = 0; i < n; i++) fn(i); return; }
    std::vector<std::thread> th;
    std::atomic<int> next(0);
    for (int t = 0; t < std::min(n, nT); t++)
        th.emplace_back([&] { for (int i; (i = next++) < n;) fn(i); });
    for (auto& t : th) t.join();
}

namespace {
struct Fmt {   // the number formatting of the output streams: fixed / precision 5 with RPM, default otherwise (libstdc++ formats via printf)
    bool rpm;
    void num(std::string& o, double v) const {
        char b[64];
        const int n = snprintf(b, sizeof(b), rpm ? "%.5f" : "%g", v);
        o.append(b, n);
    }
    static void u(std::string& o, uint64_t v) { char b[24]; const int n = snprintf(b, sizeof(b), "%llu", (unsigned long long)v); o.append(b, n); }
};

}  // namespace

int signalFromRecords(const HostParams& P, const star_engine_vtbl_t* eng, const std::vector<std::string>& names, const std::vector<uint32_t>& lens,
                      const std::vector<const uint8_t*>& recs, std::ostream& logMain, std::string& err) {
    const auto t0 = std::chrono::steady_clock::now();
    if (!eng->signal_open || !eng->signal_segment || !eng->signal_close) { err = "EXITING because of FATAL ERROR: this engine does not build signal tracks\n"; return STAR_EXIT_RUNTIME; }
    const int nRef = (int)names.size();
    const std::string& pref = P.outWigReferencesPrefix;
    auto refOk = [&](int32_t tid) { return pref == "-" || (names[tid].size() >= pref.size() && names[tid].compare(0, pref.size(), pref) == 0); };
    auto badRef = [&](size_t i, int32_t tid) {
        err = "EXITING because of fatal INPUT ERROR: BAM record " + std::to_string(i + 1) + " has the reference id " + std::to_string(tid) + ", the header lists " +
              std::to_string(nRef) + " references\n";
        return STAR_EXIT_INPUT_FILES;
    };
    // RPM: the counts of signalFromBAM.cpp:12-33 (every record with an NH tag on an output reference, duplicates included)
    double nUniq = 0, nMult = 0;
    if (P.wigNorm == 1)
        for (size_t i = 0; i < recs.size(); i++) {
            const int32_t tid = (int32_t)rd32(recs[i] + 4);
            if (tid < 0) continue;
            if (tid >= nRef) return badRef(i, tid);
            if (!refOk(tid)) continue;
            bool has; uint32_t nh;
            if (!auxNH(recs[i], has, nh)) { err = "EXITING because of fatal INPUT ERROR: malformed optional fields in BAM record " + std::to_string(i + 1) + "\n"; return STAR_EXIT_INPUT_FILES; }
            if (has) { if (nh == 1) ++nUniq; else if (nh > 1) nMult += 1.0 / nh; }
        }
    const int sigN = P.wigStranded ? 4 : 2;
    double normFactor[4] = {1, 1, 1, 1};
    if (P.wigNorm == 1) { normFactor[0] = 1.0e6 / nUniq; normFactor[1] = 1.0e6 / (nUniq + nMult); }
    normFactor[2] = normFactor[0]; normFactor[3] = normFactor[1];
    const std::string base = P.outFileNamePrefix + "Signal";
    const char* trName[4] = {".Unique.str1.out", ".UniqueMultiple.str1.out", ".Unique.str2.out", ".UniqueMultiple.str2.out"};
    std::ofstream out[4];
    for (int t = 0; t < sigN; t++) {
        const std::string fn = base + trName[t] + (P.wigFormat == 0 ? ".bg" : ".wig");
        out[t].open(fn, std::ios::binary | std::ios::trunc);
        if (!out[t].good()) { err = "EXITING because of fatal ERROR: could not create output file " + fn + "\n"; return STAR_EXIT_PARAMETER; }
    }
    void* h = nullptr;
    int rc = eng->signal_open(&h, P.gpuDevice, P.wigStranded ? 2 : 1);
    if (rc) { err = std::string("EXITING because of FATAL ERROR: signal tracks: ") + eng->last_error() + "\n"; return rc; }
    const int nT = P.stageThreads();
    const Fmt fmt{P.wigNorm == 1};
    std::vector<star_signal_block_t> blocks;
    double msDev = 0;
    uint64_t nSeg = 0, nBlocksAll = 0;
    // one finished segment: engine call, then the lines of every track (pieces of the change-point list formatted in parallel, written in order)
    auto flush = [&](int32_t iChr, uint32_t chrLen) -> int {
        star_signal_track_t tr[4];
        memset(tr, 0, sizeof(tr));
        if (!blocks.empty()) {
            float ms = 0;
            const int r = eng->signal_segment(h, chrLen, blocks.data(), blocks.size(), P.wigFormat, tr, &ms);
            if (r) { err = std::string("EXITING because of FATAL ERROR: signal tracks: ") + eng->last_error() + "\n"; return r; }
            msDev += ms;
        }
        nSeg++;
        nBlocksAll += blocks.size();
        const std::string& name = names[iChr];
        const int nPiece = 4 * nT;
        std::vector<std::string> text((size_t)sigN * nPiece);
        parallelFor(sigN * nPiece, nT, [&](int job) {
            const int t = job / nPiece, q = job % nPiece;
            const uint64_t n = tr[t].n, lo = n * q / nPiece, hi = n * (q + 1) / nPiece;
            std::string& o = text[job];
            o.reserve((hi - lo) * (name.size() + 32));
            const double nf = normFactor[t];
            for (uint64_t k = lo; k < hi; k++) {
                const uint32_t p = tr[t].pos[k];
                const double v = tr[t].val[k];
                if (P.wigFormat == 0) {   // bedGraph: close the previous record, open one where the value is nonzero
                    const double prevSig = k == 0 ? 0.0 : tr[t].val[k - 1];
                    if (prevSig != 0) { Fmt::u(o, p); o += '\t'; fmt.num(o, prevSig * nf); o += '\n'; }
                    if (v != 0) { o += name; o += '\t'; Fmt::u(o, p); o += '\t'; }
                } else {
                    Fmt::u(o, (uint64_t)p + 1); o += '\t'; fmt.num(o, v * nf); o += '\n';
                }
            }
        });
        for (int t = 0; t < sigN; t++) {
            if (P.wigFormat == 1) out[t] << "variableStep chrom=" << name << "\n";
            for (int q = 0; q < nPiece; q++) out[t].write(text[(size_t)t * nPiece + q].data(), text[(size_t)t * nPiece + q].size());
        }
        blocks.clear();
        return 0;
    };
    // the record loop of signalFromBAM.cpp:73-202
    int32_t iChr = -999;
    uint32_t chrLen = 0;
    rc = 0;
    for (size_t i = 0; i <= recs.size() && !rc; i++) {
        const bool last = i == recs.size();
        const uint8_t* r = last ? nullptr : recs[i];
        const int32_t tid = last ? 0 : (int32_t)rd32(r + 4);
        if (last || tid != iChr) {
            if (iChr != -999 && (rc = flush(iChr, chrLen))) break;
            if (last) break;
            if (tid < -1 || tid >= nRef) { rc = badRef(i, tid); break; }
            iChr = tid;
            if (iChr == -1 || !refOk(iChr)) { iChr = -999; continue; }
            chrLen = lens[iChr] + 1;   // one extra base at the end
        }
        const uint32_t flag = rd32(r + 16) >> 16;
        if (flag & 0x400) continue;   // duplicates
        bool has; uint32_t aNH;
        if (!auxNH(r, has, aNH)) { err = "EXITING because of fatal INPUT ERROR: malformed optional fields in BAM record " + std::to_string(i + 1) + "\n"; rc = STAR_EXIT_INPUT_FILES; break; }
        if (!has) aNH = 1;
        if (aNH == 0) continue;
        uint32_t aG = rd32(r + 8);
        const uint32_t iStrand = P.wigStranded ? (((flag & 0x10) > 0) == ((flag & 0x80) == 0)) : 0;
        auto past = [&]() {
            err = "EXITING because of fatal INPUT ERROR: BAM record " + std::to_string(i + 1) + " extends past the end of reference " + names[iChr] + " (length " + std::to_string(lens[iChr]) + ")\n";
            return STAR_EXIT_INPUT_FILES;
        };
        if (P.wigType == 1) {   // 5' of read 1 only
            if (flag & 0x80) continue;
            if (iStrand == 0) {
                if (aG >= chrLen) { rc = past(); break; }
                blocks.push_back({aG, 1, aNH, iStrand});
                continue;
            }
        }
        const uint32_t lName = r[12], nCig = rd16(r + 16);
        const uint8_t* cig = r + 36 + lName;
        for (uint32_t ic = 0; ic < nCig && !rc; ic++) {
            const uint32_t c = rd32(cig + 4 * ic), op = c & 0xf, L = c >> 4;
            if (op == 2 || op == 3) aG += L;   // D, N
            else if (op == 0) {                // M (= and X neither count nor advance: the reference's switch)
                if (P.wigType == 0 || (P.wigType == 2 && (flag & 0x80))) {
                    if (L && (uint64_t)aG + L > chrLen) { rc = past(); break; }
                    if (L) blocks.push_back({aG, L, aNH, iStrand});
                }
                aG += L;
            }
        }
        if (rc) break;
        if (P.wigType == 1) {
            --aG;
            if (aG >= chrLen) { rc = past(); break; }
            blocks.push_back({aG, 1, aNH, iStrand});
        }
    }
    eng->signal_close(h);
    if (rc) return rc;
    for (int t = 0; t < sigN; t++) {
        out[t].flush();
        if (!out[t].good()) { err = "EXITING because of fatal ERROR: could not write the signal output\n"; return STAR_EXIT_RUNTIME; }
    }
    logMain << "star-b200: signal tracks: " << recs.size() << " records, " << nSeg << " segments, " << nBlocksAll << " blocks; signal kernels " << msDev
            << " ms (CUDA events); signal stage wall " << std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count() << " ms\n" << std::flush;
    return 0;
}

// --inputBAMfile: BGZF blocks (htslib bgzf.c) indexed on one thread, inflated on the stage threads into one buffer, then the BAM header and
// the record boundaries
int readBAMfile(const HostParams& P, std::string& u, std::vector<std::string>& names, std::vector<uint32_t>& lens, std::vector<const uint8_t*>& recs,
                size_t& headerEnd, std::string& err) {
    const std::string& fn = P.inputBAMfile;
    std::ifstream in(fn, std::ios::binary);
    if (!in.good()) { err = "EXITING because of fatal INPUT ERROR: could not open --inputBAMfile " + fn + "\nSOLUTION: check the path and permissions\n"; return STAR_EXIT_INPUT_FILES; }
    std::string z((std::istreambuf_iterator<char>(in)), std::istreambuf_iterator<char>());
    auto bad = [&](const std::string& why) { err = "EXITING because of fatal INPUT ERROR: --inputBAMfile " + fn + " " + why + "\n"; return STAR_EXIT_INPUT_FILES; };
    struct Blk { size_t cOff, cLen, uOff, uLen; };
    std::vector<Blk> bl;
    size_t o = 0, uTot = 0;
    const uint8_t* zb = (const uint8_t*)z.data();
    while (o < z.size()) {
        if (z.size() - o < 18 || zb[o] != 31 || zb[o + 1] != 139 || zb[o + 2] != 8 || !(zb[o + 3] & 4))
            return bad(bl.empty() ? "is not a BAM file (no BGZF block at its start)" : "is truncated or corrupt (bad BGZF block at byte " + std::to_string(o) + ")");
        const size_t xlen = rd16(zb + o + 10);
        size_t bsize = 0;
        for (size_t x = o + 12; x + 4 <= o + 12 + xlen && x + 4 <= z.size();) {
            const size_t sl = rd16(zb + x + 2);
            if (zb[x] == 'B' && zb[x + 1] == 'C' && sl == 2) bsize = (size_t)rd16(zb + x + 4) + 1;
            x += 4 + sl;
        }
        if (bsize == 0) return bad(bl.empty() ? "is not a BAM file (gzip without BGZF block sizes)" : "is corrupt (BGZF block without its size at byte " + std::to_string(o) + ")");
        if (bsize < 12 + xlen + 8 || o + bsize > z.size()) return bad("is truncated (the last BGZF block is incomplete)");
        const size_t uLen = rd32(zb + o + bsize - 4);
        bl.push_back({o + 12 + xlen, bsize - 12 - xlen - 8, uTot, uLen});
        uTot += uLen;
        o += bsize;
    }
    u.assign(uTot, '\0');
    std::vector<char> okB(bl.size(), 1);
    const int nQ = P.stageThreads() * 4;
    parallelFor(nQ, P.stageThreads(), [&](int q) {
        for (size_t b = bl.size() * q / nQ; b < bl.size() * (q + 1) / nQ; b++) {
            z_stream s;
            memset(&s, 0, sizeof(s));
            if (inflateInit2(&s, -15) != Z_OK) { okB[b] = 0; continue; }
            s.next_in = (Bytef*)zb + bl[b].cOff; s.avail_in = (uInt)bl[b].cLen;
            s.next_out = (Bytef*)&u[bl[b].uOff]; s.avail_out = (uInt)bl[b].uLen;
            const int r = inflate(&s, Z_FINISH);
            if (r != Z_STREAM_END || s.total_out != bl[b].uLen || crc32(0, (const Bytef*)&u[bl[b].uOff], (uInt)bl[b].uLen) != rd32(zb + bl[b].cOff + bl[b].cLen)) okB[b] = 0;
            inflateEnd(&s);
        }
    });
    for (size_t b = 0; b < bl.size(); b++) if (!okB[b]) return bad("is corrupt (BGZF block " + std::to_string(b) + " does not inflate)");
    std::string().swap(z);
    const uint8_t* ub = (const uint8_t*)u.data();
    // header: magic, l_text, text, n_ref, (l_name, name, l_ref) x n_ref (SAM/BAM specification 4.2)
    if (uTot < 12 || memcmp(ub, "BAM\1", 4) != 0) return bad("is not a BAM file (bad magic)");
    size_t p = 8 + (size_t)rd32(ub + 4);
    if (p + 4 > uTot) return bad("is truncated (in the header)");
    const uint32_t nRef = rd32(ub + p);
    p += 4;
    names.assign(nRef, std::string());
    lens.assign(nRef, 0);
    for (uint32_t r = 0; r < nRef; r++) {
        if (p + 4 > uTot) return bad("is truncated (in the header)");
        const uint32_t ln = rd32(ub + p);
        if (ln == 0 || p + 4 + ln + 4 > uTot) return bad("is truncated (in the header)");
        names[r].assign((const char*)ub + p + 4, strnlen((const char*)ub + p + 4, ln));
        lens[r] = rd32(ub + p + 4 + ln);
        p += 8 + ln;
    }
    headerEnd = p;
    recs.clear();
    while (p < uTot) {   // bam_read1: block_size, 32 bytes of fixed fields, then the variable part
        if (uTot - p < 4) return bad("is truncated (in a record)");
        const uint32_t bs = rd32(ub + p);
        if (bs < 32 || uTot - p - 4 < bs) return bad("is truncated (in record " + std::to_string(recs.size() + 1) + ")");
        const uint8_t* r = ub + p;
        const uint64_t fixedPart = 32ull + r[12] + 4ull * rd16(r + 16);
        const int32_t lSeq = (int32_t)rd32(r + 20);
        if (lSeq < 0 || fixedPart + (uint64_t)(lSeq + 1) / 2 + (uint64_t)lSeq > bs) return bad("is corrupt (record " + std::to_string(recs.size() + 1) + " is inconsistent)");
        recs.push_back(r);
        p += 4 + (size_t)bs;
    }
    return 0;
}

int signalFromBAMfile(const HostParams& P, const star_engine_vtbl_t* eng, std::ostream& logMain, std::string& err) {
    std::string u;
    std::vector<std::string> names;
    std::vector<uint32_t> lens;
    std::vector<const uint8_t*> recs;
    size_t headerEnd = 0;
    if (int rc = readBAMfile(P, u, names, lens, recs, headerEnd, err)) return rc;
    return signalFromRecords(P, eng, names, lens, recs, logMain, err);
}

}  // namespace starhost
