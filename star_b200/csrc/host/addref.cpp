// addref.cpp — references added to the loaded index at the mapping stage: --genomeFastaFiles with --runMode alignReads.
//
// Host side of reference source/Genome_insertSequences.cpp and insertSeqSA.cpp (called from Genome_genomeLoad.cpp:245-250, 374): the FASTA
// scan that sizes the insert (genomeScanFastaFiles.cpp:5-91, the scanner of genome_generate.cpp), the layout of the grown genome, the sort
// of the insertion points and the SAindex rebuild (genomeSAindex.cpp, the builder of genome_generate.cpp).  The steps that touch every SA
// row or every added suffix — the re-base of the old rows, the suffixArraySearch1 loop and the SA rewrite — run on the GPU behind
// star_gpu_addref_* (include/star_b200.h, star_b200/csrc/engine/addref.cu).
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <ostream>

#include "host.h"

namespace starhost {

int addReferences(const HostParams& P, star_params_t* hp, LoadedIndex& idx, const star_engine_vtbl_t* eng, std::ostream& logMain, std::string& err, bool chrInfoOnly) {
    if (P.genomeFastaFiles.empty() || P.genomeFastaFiles[0] == "-") return 0;
    star_index_view_t& v = idx.view;
    auto t0 = std::chrono::steady_clock::now();
    auto phase = [&](const char* what, double deviceMs = -1) {   // wall time of every phase in Log.out, with the device time of its kernel
        const auto now = std::chrono::steady_clock::now();
        logMain << "   [add references, " << what << ": " << std::chrono::duration<double>(now - t0).count() << " s";
        if (deviceMs >= 0) logMain << ", kernel " << deviceMs << " ms";
        logMain << "]" << std::endl;
        t0 = now;
    };
    const uint32_t nChrOld = v.nChrReal;
    const uint64_t binN = 1ULL << v.gChrBinNbits;
    const uint64_t nG = idx.chrStart[nChrOld];          // end of the old chromosomes: the sequences go here
    const uint64_t nG2 = chrInfoOnly ? 0 : v.nGenome - nG;   // junction inserts of the index, moved behind the sequences
    logMain << " ..... inserting extra sequences into genome indexes" << std::endl;

    // ---- 1. sizing (genomeScanFastaFiles with flagRun = false; with G, the fill of Genome_insertSequences.cpp:18-20 in the same pass)
    std::vector<uint8_t> Gnew;
    if (!chrInfoOnly) {
        Gnew.reserve(256 + v.nGenome + 256);
        Gnew.assign(idx.Gstore.begin(), idx.Gstore.begin() + 256 + nG);
    }
    int rc = scanFastaFiles(P.genomeFastaFiles, binN, idx.chrName, idx.chrStart, idx.chrLength, chrInfoOnly ? nullptr : &Gnew, 256, logMain, err);
    if (rc) return rc;
    const uint32_t nChr = (uint32_t)idx.chrName.size();
    const uint64_t nG1 = idx.chrStart[nChr] - nG;      // genomeInsertL
    idx.insertChrFirst = nChrOld;
    v.nChrReal = nChr;
    {   // chrBinFill, Genome.cpp:209-216
        const uint64_t chrBinN = idx.chrStart[nChr] / binN + 1;
        idx.chrBin.resize(chrBinN);
        for (uint64_t ii = 0, ichr = 1; ii < chrBinN; ++ii) { if (ii * binN >= idx.chrStart[ichr]) ichr++; idx.chrBin[ii] = ichr - 1; }
    }
    logMain << "Chromosome sequence lengths: \n";
    for (uint32_t i = 0; i < nChr; i++) logMain << idx.chrName[i] << "\t" << idx.chrLength[i] << "\n";
    if (chrInfoOnly) {
        v.chrStart = idx.chrStart.data(); v.chrLength = idx.chrLength.data();
        return 0;
    }
    phase("FASTA scan");

    // ---- 2. the grown genome: old chromosomes, the added ones (padded), the junction inserts
    const uint64_t nGenomeNew = nG + nG1 + nG2;
    Gnew.resize(256 + nG + nG1, 5);
    Gnew.insert(Gnew.end(), idx.Gstore.begin() + 256 + nG, idx.Gstore.begin() + 256 + nG + nG2);
    Gnew.resize(256 + nGenomeNew + 256, 5);
    idx.Gstore.swap(Gnew);                  // the old genome is not read again: at most one genome and two suffix arrays are held at a time
    std::vector<uint8_t>().swap(Gnew);
    logMain << "Genome size with added sequences=" << nGenomeNew << " = " << nG << " + " << nG1 << " + " << nG2 << "\n";

    // ---- 3. GstrandBit (insertSeqSA.cpp:21-29)
    uint32_t GstrandBit1 = (uint32_t)std::floor(std::log((double)(nG + nG1)) / std::log(2.0)) + 1;
    if (GstrandBit1 < 32) GstrandBit1 = 32;
    if (GstrandBit1 + 1 > v.GstrandBit + 1) {
        err = "EXITING because of FATAL ERROR: cannot insert sequence on the fly because of strand GstrandBit problem\nSOLUTION: please contact STAR author at https://groups.google.com/forum/#!forum/rna-star\n";
        return STAR_EXIT_GENOME_FILES;
    }
    if (!eng->addref_open) { err = "EXITING because of FATAL ERROR: this engine cannot add references\n"; return STAR_EXIT_BUG; }

    // ---- 4. device: re-base, search; host: sort of the insertion points
    star_index_view_t grown = v;
    grown.G = idx.Gstore.data() + 256;
    grown.nGenome = nGenomeNew;
    void* h = nullptr;
    float ms = 0;
    rc = eng->addref_open(&h, P.gpuDevice, &grown, nG, nG1, nG2, &ms);
    if (rc) { if (h) eng->addref_close(h); err = std::string("EXITING because of FATAL ERROR: adding references failed: ") + eng->last_error() + "\n"; return rc; }
    phase("upload + re-base of the SA rows", ms);
    // the reference's text buffer (insertSeqSA.cpp:53-70): 16 x code 5, seq1[0] = forward + reverse complement (2*nG1), 16 x code 5,
    // seq1[1] = the complement of seq1[0], 16 x code 5.  The search reads seq1[0] (and its padding); the sort compares whole tails of the buffer.
    const uint64_t L16 = 16, nText = 2 * nG1;
    std::vector<uint8_t> seqq(2 * nText + 3 * L16, 5);
    uint8_t* s0 = seqq.data() + L16;
    uint8_t* s1 = seqq.data() + 2 * L16 + nText;
    memcpy(s0, idx.Gstore.data() + 256 + nG, nG1);
    for (uint64_t ii = 0; ii < nG1; ii++) s0[nText - 1 - ii] = s0[ii] < 4 ? 3 - s0[ii] : s0[ii];
    for (uint64_t ii = 0; ii < nText; ii++) s1[ii] = s0[ii] < 4 ? 3 - s0[ii] : s0[ii];   // complementSeqNumbers
    std::vector<uint64_t> ind(2 * nText + 2);
    rc = eng->addref_search(h, s0, ind.data(), &ms);
    if (rc) { eng->addref_close(h); err = std::string("EXITING because of FATAL ERROR: adding references failed: ") + eng->last_error() + "\n"; return rc; }
    phase("SA search", ms);
    struct Ins { uint64_t row, off; };
    static_assert(sizeof(Ins) == 16, "pairs of 64-bit words");
    Ins* ia = reinterpret_cast<Ins*>(ind.data());
    uint64_t nInd = 0;
    for (uint64_t ii = 0; ii < nText; ii++) if (ia[ii].row != ~0ULL) ia[nInd++] = ia[ii];
    logMain << "   Finished SA search, number of new SA indices = " << nInd << std::endl;
    // funCompareUintAndSuffixesMemcmp.cpp:7-33: row, then memcmp of the suffixes over gSuffixLengthMax/8 bytes (unlimited by default), which
    // does not stop at a code 5 and runs from seq1[0] through the padding into seq1[1].  Where two tails are equal up to the end of the buffer
    // the reference reads past its allocation (undefined); here the comparison stops at the buffer's end and the offsets decide.
    const uint8_t* base = s0;
    const uint64_t tailEnd = 2 * nText + 2 * L16;   // bytes of the buffer from s0 on
    std::sort(ia, ia + nInd, [base, tailEnd](const Ins& x, const Ins& y) {
        if (x.row != y.row) return x.row < y.row;
        const int c = memcmp(base + x.off, base + y.off, tailEnd - std::max(x.off, y.off));
        if (c != 0) return c < 0;
        return x.off < y.off;
    });
    phase("sort of the insertion points");

    // ---- 5. the merged SA (device), then SAindex from scratch (insertSeqSA.cpp:158-199, 299-308)
    const uint64_t nSAnew = v.nSA + nInd;
    const uint64_t nSAnewByte = (nSAnew - 1) * (v.GstrandBit + 1) / 8 + 8;
    std::vector<uint8_t> SAnew(nSAnewByte + 16, 0);
    rc = eng->addref_merge_sa(h, ind.data(), nInd, SAnew.data(), nSAnewByte, &ms);
    eng->addref_close(h);
    if (rc) { err = std::string("EXITING because of FATAL ERROR: adding references failed: ") + eng->last_error() + "\n"; return rc; }
    logMain << "   Finished inserting SA indices" << std::endl;
    idx.SAstore.swap(SAnew);
    std::vector<uint8_t>().swap(SAnew);
    phase("SA merge + download", ms);
    std::vector<uint64_t> saiStart;
    std::vector<uint8_t> SAi;
    uint64_t nSAi = 0, nSAibyte = 0;
    rc = buildSAindex(idx.Gstore.data() + 256, nGenomeNew, idx.SAstore.data(), nSAnew, v.GstrandBit, v.gSAindexNbases, P.runThreadN, saiStart, SAi, nSAi, nSAibyte, err);
    if (rc) return rc;
    phase("SAindex");

    // ---- 6. the grown index; loadSJDB (Genome_genomeLoad.cpp:471-520) and the window geometry (:382-410) with the new size
    idx.SAistore.swap(SAi);
    idx.genomeSAindexStart.swap(saiStart);
    v.nGenome = nGenomeNew; v.nSA = nSAnew; v.nSAbyte = nSAnewByte; v.nSAi = nSAi; v.nSAibyte = nSAibyte;
    v.sjGstart = nG2 == 0 ? idx.chrStart[nChr] + 1 : idx.chrStart[nChr];
    idx.pointView();
    windowGeometry(hp, v.nGenome, v.gChrBinNbits, &logMain);
    logMain << " ..... finished inserting extra sequences into genome indexes" << std::endl;
    return 0;
}

}  // namespace starhost
