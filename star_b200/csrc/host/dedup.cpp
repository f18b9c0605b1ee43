// dedup.cpp — duplicate marking of --runMode inputAlignmentsFromBAM --bamRemoveDuplicatesType (reference source/bamRemoveDuplicates.cpp:114-271).
//
// One pass over the records in file order reads NH, sets the 0x400 bit (NH == 1, or NH > 1 with UniqueIdentical) and finds the groups:
// a group closes before a record whose reference id differs from the group's first record's, or whose position is past rightMax, the
// largest mate position of the group's NH == 1 records whose mate lies to their right (0 = none yet: the group cannot close on position).
// The NH == 1 records are the members.  The engine (star_gpu_dedup_batch) pairs the members of every group in name order, classes the pairs
// and returns the pair to un-mark in every class; the flags are patched in the inflated buffer, which is re-framed as BGZF on the stage
// threads behind the header as bam_hdr_write writes it.
#include <algorithm>
#include <chrono>
#include <cstring>
#include <fstream>
#include <thread>

#include "host.h"

namespace starhost {

namespace {
inline uint32_t rd32(const uint8_t* p) { uint32_t v; memcpy(&v, p, 4); return v; }
double msSince(std::chrono::steady_clock::time_point t) { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t).count(); }
}  // namespace

int dedupFromBAMfile(const HostParams& P, const star_engine_vtbl_t* eng, std::ostream& logMain, std::string& err) {
    const auto t0 = std::chrono::steady_clock::now();
    if (!eng->dedup_open || !eng->dedup_batch || !eng->dedup_close) { err = "EXITING because of FATAL ERROR: this engine does not remove duplicates\n"; return STAR_EXIT_RUNTIME; }
    // the device is opened (CUDA context creation) while the file is read
    void* h = nullptr;
    int openRc = 0;
    std::thread opener([&] { openRc = eng->dedup_open(&h, P.gpuDevice, P.bamRemoveDuplicatesMate2basesN); });
    std::string u;
    std::vector<std::string> names;
    std::vector<uint32_t> lens;
    std::vector<const uint8_t*> recs;
    size_t headerEnd = 0;
    int rc = readBAMfile(P, u, names, lens, recs, headerEnd, err);
    const double msRead = msSince(t0);
    auto openDone = [&]() -> int {   // joins the opener; the error of a failed open, if nothing failed before it
        opener.join();
        if (openRc && !rc) err = std::string("EXITING because of FATAL ERROR: duplicate removal: ") + eng->last_error() + "\n";
        return openRc;
    };
    if (rc) {
        if (!openDone()) eng->dedup_close(h);
        return rc;
    }
    uint8_t* ub = (uint8_t*)&u[0];
    auto recNo = [](size_t i) { return "BAM record " + std::to_string(i + 1); };

    // the loop of bamRemoveDuplicates.cpp:144-266: marks, groups, members
    std::vector<uint64_t> off;        // members: record offset in u
    std::vector<uint32_t> grp;        // members: group
    std::vector<size_t> memberRec;    // members: record index
    size_t stopRec = recs.size();     // the record whose NH error ends the loop (recs.size(): none)
    bool malformed = false;
    uint32_t g = 0, rightMax = 0, chrS = recs.empty() ? 0 : rd32(recs[0] + 4);
    for (size_t i = 0; i < recs.size(); i++) {
        uint8_t* r = ub + (recs[i] - ub);
        bool has;
        uint32_t nh;
        const bool ok = auxNH(r, has, nh);
        if (!ok || !has) { stopRec = i; malformed = !ok; break; }
        const int nMult = (int32_t)nh;
        if (nMult == 1 || (nMult > 1 && P.dedupMarkMulti)) r[19] |= 0x04;   // flag |= 0x400
        const uint32_t chrE = rd32(r + 4), leftE = rd32(r + 8), rightE = rd32(r + 28);
        if (chrE != chrS || (rightMax > 0 && leftE > rightMax)) { g++; rightMax = 0; chrS = chrE; }
        if (nMult == 1) {
            off.push_back((uint64_t)(r - ub));
            grp.push_back(g);
            memberRec.push_back(i);
            if (rightE > leftE) rightMax = std::max(rightMax, rightE);
        }
    }
    if (stopRec < recs.size())   // the group open at the failing record is never processed
        while (!grp.empty() && grp.back() == g) { off.pop_back(); grp.pop_back(); memberRec.pop_back(); }
    uint64_t nGroups = recs.empty() ? 0 : (uint64_t)g + 1, nPairs = 0;
    for (size_t k = 0; k < grp.size();) {
        size_t j = k;
        while (j < grp.size() && grp[j] == grp[k]) j++;
        nPairs += (j - k) / 2;
        k = j;
    }

    const double msPass = msSince(t0) - msRead;
    if (int orc = openDone()) return orc;
    const double msOpenWait = msSince(t0) - msRead - msPass;
    std::vector<uint8_t> unmark(off.size(), 0);
    float ms = 0;
    const auto tB = std::chrono::steady_clock::now();
    rc = eng->dedup_batch(h, ub, off.data(), grp.data(), off.size(), unmark.data(), &ms);
    const double msBatch = msSince(tB);
    const std::string engErr = rc ? eng->last_error() : "";
    eng->dedup_close(h);
    if (rc == STAR_EXIT_PARAMETER || rc == STAR_EXIT_INPUT_FILES) {
        size_t k = 0;
        while (k < unmark.size() && unmark[k] < 2) k++;
        if (k == unmark.size()) { err = "EXITING because of FATAL ERROR: duplicate removal: " + engErr + "\n"; return STAR_EXIT_BUG; }
        const size_t i = memberRec[k];
        const uint8_t* r = recs[i];
        const std::string in = "EXITING because of fatal INPUT ERROR: " + recNo(i);
        switch (unmark[k] - 2) {
            case 0: err = in + " has a CIGAR of " + std::to_string(rd32(r + 16) & 0xffff) + " operations; duplicate removal compares CIGARs of 1 to 100 operations that are not all S\n"; break;
            case 1: err = in + " has " + std::to_string(rd32(r + 20)) + " bases, fewer than --bamRemoveDuplicatesMate2basesN " + std::to_string(P.bamRemoveDuplicatesMate2basesN) + "\n"; break;
            case 2: err = "EXITING because of fatal INPUT ERROR: malformed optional fields in " + recNo(i) + "\n"; break;
            case 3: err = "EXITING because of fatal ERROR: SAM tag AS is missing from a read, but it's required for deduplication. \nSOLUTION: re-generate BAM file with NH and AS tags."; break;
            default: err = in + " has AS <= -999; the reference's choice of the pair to keep is undefined for such scores\n"; break;
        }
        return rc;
    }
    if (rc) { err = "EXITING because of FATAL ERROR: duplicate removal: " + engErr + "\n"; return rc; }
    if (stopRec < recs.size()) {
        if (malformed) { err = "EXITING because of fatal INPUT ERROR: malformed optional fields in " + recNo(stopRec) + "\n"; return STAR_EXIT_INPUT_FILES; }
        err = "EXITING because of fatal ERROR: SAM tag NH is missing from a read, but it's required for deduplication. \nSOLUTION: re-generate BAM file with NH and AS tags.";
        return STAR_EXIT_PARAMETER;
    }
    uint64_t nUnmarked = 0;
    for (size_t k = 0; k < off.size(); k++)
        if (unmark[k] == 1) { ub[off[k] + 19] &= (uint8_t)~0x04; nUnmarked++; }

    // Processed.out.bam: the header as bam_hdr_write writes it, the records, the EOF block
    const auto tO = std::chrono::steady_clock::now();
    std::string hdr(ub, ub + 8 + rd32(ub + 4));
    auto put32 = [&](uint32_t v) { hdr.append((const char*)&v, 4); };
    put32((uint32_t)names.size());
    for (size_t r = 0; r < names.size(); r++) { put32((uint32_t)names[r].size() + 1); hdr += names[r]; hdr += '\0'; put32(lens[r]); }
    const std::string fn = P.outFileNamePrefix + "Processed.out.bam";
    std::ofstream out(fn, std::ios::binary | std::ios::trunc);
    if (!out.good()) { err = "EXITING because of fatal ERROR: could not create output file " + fn + "\n"; return STAR_EXIT_PARAMETER; }
    const int nT = P.stageThreads(), nPiece = 4 * nT;
    const size_t body = u.size() - headerEnd;
    std::vector<std::string> z(nPiece + 1);
    OutputWriter::bgzfCompress(hdr.data(), hdr.size(), P.outBAMcompression, z[0]);
    parallelFor(nPiece, nT, [&](int q) {
        const size_t lo = headerEnd + body * q / nPiece, hi = headerEnd + body * (q + 1) / nPiece;
        if (hi > lo) OutputWriter::bgzfCompress(u.data() + lo, hi - lo, P.outBAMcompression, z[q + 1]);
    });
    for (const std::string& s : z) out.write(s.data(), s.size());
    size_t ne;
    const char* eof = OutputWriter::bgzfEofBlock(ne);
    out.write(eof, ne);
    out.flush();
    if (!out.good()) { err = "EXITING because of fatal ERROR: could not write " + fn + "\n"; return STAR_EXIT_RUNTIME; }
    logMain << "star-b200: duplicate removal: " << recs.size() << " records, " << off.size() << " NH==1 members, " << nGroups << " groups, " << nPairs << " pairs, "
            << nUnmarked / 2 << " classes, " << nUnmarked / 2 << " pairs un-marked; dedup kernels " << ms << " ms (CUDA events); dedup stage wall "
            << msSince(t0) << " ms (read + inflate " << msRead << ", marking pass " << msPass << ", waiting for the device " << msOpenWait << ", batch call "
            << msBatch << ", output " << msSince(tO) << ")\n" << std::flush;
    return 0;
}

}  // namespace starhost
