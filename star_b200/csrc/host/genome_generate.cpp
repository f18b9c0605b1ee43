// genome_generate.cpp — `STAR --runMode genomeGenerate` (SURVEY.md §8f N4): FASTA -> Genome, SA, SAindex (+ junction inserts).
//
// Host side of reference source/Genome_genomeGenerate.cpp:98-415: FASTA scan and chromosome padding (genomeScanFastaFiles.cpp:5-103),
// chr*.txt (writeChrInfo, :417-432), SAindex (genomeSAindex.cpp:6-220), genomeParameters.txt (genomeParametersWrite.cpp:4-46) and the
// junction insertion shared with the mapping stage (sjdb_insert.cpp).  The suffix sort — hours of qsort over 16-mer buckets in the
// reference (:213-330) — is the device step behind star_gpu_sa_build (star_b200/csrc/engine/sa_build.cu).
#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <fstream>
#include <iostream>
#include <sstream>
#include <thread>

#include "host.h"

namespace starhost {

namespace {

struct PackedRW {   // PackedArray.h:24-32, PackedArray.cpp:17-25
    uint8_t* a;
    uint32_t bits;
    uint64_t mask;
    PackedRW(uint8_t* p, uint32_t b) : a(p), bits(b), mask(~0ULL >> (64 - b)) {}
    uint64_t get(uint64_t i) const { const uint64_t b = i * bits; uint64_t w; memcpy(&w, a + b / 8, 8); return (w >> (b % 8)) & mask; }
    void set(uint64_t i, uint64_t x) {
        const uint64_t b = i * bits, S = b % 8;
        uint64_t w;
        memcpy(&w, a + b / 8, 8);
        w = (w & ~(mask << S)) | (x << S);
        memcpy(a + b / 8, &w, 8);
    }
};

// funCalcSAiFromSA, SuffixArrayFuns.cpp:353-395: prefix code of the first L bases of SA row iSA; iL4 = offset of the first base > 3 (-1: none)
uint64_t calcSAiFromSA(const uint8_t* G, const PackedRW& SA, uint64_t nGenome, uint32_t GstrandBit, uint64_t iSA, int L, int& iL4) {
    uint64_t SAstr = SA.get(iSA);
    const bool dirG = (SAstr >> GstrandBit) == 0;
    SAstr &= ~(1ULL << GstrandBit);
    iL4 = -1;
    uint64_t saind = 0;
    for (int ii = 0; ii < L; ii++) {
        const uint8_t g = dirG ? G[SAstr + ii] : G[nGenome - 1 - SAstr - ii];
        if (g > 3) { iL4 = ii; return saind << (2 * (L - ii)); }
        saind = (saind << 2) + (dirG ? g : 3 - g);
    }
    return saind;
}

}  // namespace

// genomeScanFastaFiles.cpp:5-91: the chromosomes of `files` are appended to chrName / chrStart / chrLength, every one starting at a
// multiple of binN (the first one of a file list that follows existing chromosomes at the old end, chrStart.back()); gaps are code 5.
// With G, the codes go to G[pad + position] (G grows as needed, new bytes are code 5).  The lists are "closed" before and after: chrStart
// holds one more entry, the padded end.
int scanFastaFiles(const std::vector<std::string>& files, uint64_t binN, std::vector<std::string>& chrName, std::vector<uint64_t>& chrStart,
                   std::vector<uint64_t>& chrLength, std::vector<uint8_t>* G, size_t pad, std::ostream& logMain, std::string& err) {
    uint64_t N = 0;
    if (!chrLength.empty()) {   // previous chromosomes: continue behind the last one (:7-12)
        chrStart.pop_back();
        N = chrStart.back() + chrLength.back();
        chrLength.pop_back();
    }
    auto padTo = [&](uint64_t n) { if (G && G->size() < pad + n) G->resize(pad + n, 5); };
    uint8_t lut[256];   // convertNucleotidesToNumbersRemoveControls (SequenceFuns.cpp:170-192): 0..3, 4 = any other printable, 255 = control character
    for (int c = 0; c < 256; c++) lut[c] = c < 32 ? 255 : 4;
    lut['A'] = lut['a'] = 0; lut['C'] = lut['c'] = 1; lut['G'] = lut['g'] = 2; lut['T'] = lut['t'] = 3;
    for (const std::string& fn : files) {
        // the file is mapped and walked line by line (the reference reads it with getline, genomeScanFastaFiles.cpp:24-78)
        const int fd = open(fn.c_str(), O_RDONLY);
        if (fd < 0) { err = "EXITING because of INPUT ERROR: could not open genomeFastaFile: " + fn + "\n"; return STAR_EXIT_INPUT_FILES; }
        struct stat sb;
        if (fstat(fd, &sb) != 0 || sb.st_size == 0) { close(fd); err = "EXITING because of INPUT ERROR: could not read from genomeFastaFile: " + fn + "\n"; return STAR_EXIT_INPUT_FILES; }
        const size_t fsize = (size_t)sb.st_size;
        const char* text = (const char*)mmap(nullptr, fsize, PROT_READ, MAP_PRIVATE, fd, 0);
        close(fd);
        if (text == MAP_FAILED) { err = "EXITING because of INPUT ERROR: could not read from genomeFastaFile: " + fn + "\n"; return STAR_EXIT_INPUT_FILES; }
        madvise((void*)text, fsize, MADV_SEQUENTIAL);
        const int cc = (unsigned char)text[0];
        if (cc != '>') {
            munmap((void*)text, fsize);
            err = "EXITING because of INPUT ERROR: the file format of the genomeFastaFile: " + fn + " is not fasta: the first character is '" + std::string(1, (char)cc) + "' (" + std::to_string(cc) +
                  "), not '>'.\n Solution: check formatting of the fasta file. Make sure the file is uncompressed (unzipped).\n";
            return STAR_EXIT_INPUT_FILES;
        }
        for (size_t off = 0; off < fsize;) {
            const char* nl = (const char*)memchr(text + off, '\n', fsize - off);
            const size_t len = nl ? (size_t)(nl - (text + off)) : fsize - off;
            const char* line = text + off;
            off += len + 1;
            if (len > 0 && line[0] == '>') {
                std::istringstream ls(std::string(line, len));
                ls.ignore(1, ' ');
                std::string name;
                ls >> name;
                chrName.push_back(name);
                if (!chrStart.empty()) chrLength.push_back(N - chrStart.back());
                if (N > 0) N = ((N + 1) / binN + 1) * binN;
                chrStart.push_back(N);
                padTo(N);
                logMain << fn << " : chr # " << chrStart.size() - 1 << "  \"" << name << "\" chrStart: " << N << "\n";
            } else {   // control characters are dropped from the COUNT only (the reference's quirk): a code lands at the character's column
                if (!G) { for (size_t jj = 0; jj < len; jj++) N += lut[(unsigned char)line[jj]] != 255; continue; }
                padTo(N + len);
                uint8_t* dst = G->data() + pad + N;
                uint64_t kept = 0;
                for (size_t jj = 0; jj < len; jj++) {
                    const uint8_t v = lut[(unsigned char)line[jj]];
                    if (v == 255) continue;
                    dst[jj] = v;
                    kept++;
                }
                N += kept;
            }
        }
        munmap((void*)text, fsize);
    }
    if (chrStart.empty()) { err = "EXITING because of INPUT ERROR: no sequences in --genomeFastaFiles\n"; return STAR_EXIT_INPUT_FILES; }
    chrLength.push_back(N - chrStart.back());
    N = ((N + 1) / binN + 1) * binN;
    chrStart.push_back(N);
    return 0;
}

// genomeSAindex.cpp:6-220 over a whole suffix array: genomeSAindexStart (Lmax+1 entries) and the packed table SAistore (nSAibyte bytes,
// GstrandBit+3 bits per entry, 16 bytes of slack).  Used by genomeGenerate and after references are added at the mapping stage.
int buildSAindex(const uint8_t* Gp, uint64_t nGenome, const uint8_t* SAbytes, uint64_t nSA, uint32_t GstrandBit, uint32_t Lmax, int runThreadN,
                 std::vector<uint64_t>& genomeSAindexStart, std::vector<uint8_t>& SAistore, uint64_t& nSAi, uint64_t& nSAibyte, std::string& err) {
    genomeSAindexStart.assign(Lmax + 1, 0);
    for (uint32_t i = 1; i <= Lmax; i++) genomeSAindexStart[i] = genomeSAindexStart[i - 1] + (1ULL << (2 * i));
    nSAi = genomeSAindexStart[Lmax];
    nSAibyte = (nSAi - 1) * (GstrandBit + 3) / 8 + 8;
    SAistore.assign(nSAibyte + 16, 0);
    {
        // The reference walks the rows once, from run to run of equal (prefix, offset of the first base > 3), jump + bisect
        // (funSAiFindNextIndex), keeping per prefix length the last prefix seen.  The same walk is cut into row ranges that start at run
        // heads, one per host thread: what a range needs from the rows before it — the last prefix present at every length — is read off
        // the rows in front of its first row, the entries are collected unpacked (threads own disjoint entries but share packed words),
        // the "contains N" marks are applied after the join, and the table is packed by 64-entry groups (whole words) in parallel.
        const uint8_t* G = Gp;
        const PackedRW SA(const_cast<uint8_t*>(SAbytes), GstrandBit + 1);
        const uint64_t nC = 1ULL << (GstrandBit + 1), absentC = 1ULL << (GstrandBit + 2);
        const uint64_t* start = genomeSAindexStart.data();
        std::vector<uint64_t> tab(nSAi, 0);
        const uint64_t NONE = ~0ULL;
        auto keyOf = [&](uint64_t isa, int& iL4) { return calcSAiFromSA(G, SA, nGenome, GstrandBit, isa, (int)Lmax, iL4); };
        int nT = std::max(1, std::min(runThreadN, 256));
        if (nSA < 4096 * (uint64_t)nT) nT = 1;
        std::vector<uint64_t> lo(nT + 1, nSA);
        lo[0] = 0;
        for (int t = 1; t < nT; t++) {   // first run head at or after the even split
            uint64_t r = std::max<uint64_t>(lo[t - 1], nSA / nT * t);
            if (r == 0) r = 1;
            int a4, b4;
            while (r < nSA) { const uint64_t ka = keyOf(r - 1, a4), kb = keyOf(r, b4); if (ka != kb || a4 != b4) break; r++; }
            lo[t] = r;
        }
        struct Mark { uint32_t iL; uint64_t ind; };
        std::vector<std::vector<Mark>> marks(nT);
        std::vector<int> bug(nT, 0);
        std::vector<std::vector<uint64_t>> lastInd(nT);
        auto work = [&](int t) {
            const uint64_t r0 = lo[t], r1 = lo[t + 1];
            std::vector<uint64_t> ind0(Lmax, NONE);
            if (r0 > 0) {   // last prefix present at every length among the rows before r0
                uint32_t need = Lmax;
                for (uint64_t r = r0; r-- > 0 && need > 0;) {
                    int iL4;
                    const uint64_t ind = keyOf(r, iL4);
                    const uint32_t valid = iL4 < 0 ? Lmax : (uint32_t)iL4;   // lengths 1..valid hold bases only
                    for (uint32_t iL = 0; iL < valid; iL++) if (ind0[iL] == NONE) { ind0[iL] = ind >> (2 * (Lmax - 1 - iL)); need--; }
                }
            }
            const uint64_t isaStep = nSA / (1ULL << (2 * Lmax)) + 1;
            for (uint64_t isa = r0; isa < r1;) {
                int iL4;
                const uint64_t indFull = keyOf(isa, iL4);
                for (uint32_t iL = 0; iL < Lmax; iL++) {
                    const uint64_t indPref = indFull >> (2 * (Lmax - 1 - iL));
                    if ((int)iL == iL4) {   // a base > 3 inside the prefix: mark the last present prefix of every longer length
                        for (uint32_t iL1 = iL; iL1 < Lmax; iL1++) marks[t].push_back({iL1, ind0[iL1]});   // (ind0 = -1 wraps to the entry in front, as in the reference)
                        break;
                    }
                    if (indPref > ind0[iL] || isa == 0) {   // (unsigned compare: a length without any prefix so far, ind0 = -1, fails both tests unless isa == 0 ...
                        tab[start[iL] + indPref] = isa;
                        for (uint64_t ii = ind0[iL] + 1; ii < indPref; ii++) tab[start[iL] + ii] = isa | absentC;
                        ind0[iL] = indPref;
                    } else if (indPref < ind0[iL]) { bug[t] = 1; return; }   // ... and ends here like the reference)
                }
                // first row of the next run: gallop in steps of isaStep, then bisect (rows of a run are contiguous)
                uint64_t a = isa, b = isa + isaStep;
                int b4;
                while (b < r1 && keyOf(b, b4) == indFull && b4 == iL4) { a = b; b += isaStep; }
                if (b > r1) b = r1;   // (r1 is a run head or nSA: the run ends at or before it)
                while (a + 1 < b) {
                    const uint64_t m = a + (b - a) / 2;
                    if (keyOf(m, b4) == indFull && b4 == iL4) a = m; else b = m;
                }
                isa = b;
            }
            lastInd[t] = ind0;
        };
        {
            std::vector<std::thread> th;
            for (int t = 1; t < nT; t++) th.emplace_back(work, t);
            work(0);
            for (auto& x : th) x.join();
        }
        for (int t = 0; t < nT; t++) if (bug[t]) { err = "BUG: next index is smaller than previous, EXITING\n"; return STAR_EXIT_INPUT_FILES; }
        for (int t = 0; t < nT; t++) for (const Mark& m : marks[t]) { const uint64_t e = start[m.iL] + m.ind; if (e < nSAi) tab[e] |= nC; }
        {   // prefixes behind the last present one
            const std::vector<uint64_t>& ind0 = lastInd[nT - 1];
            for (uint32_t iL = 0; iL < Lmax; iL++)
                for (uint64_t ii = start[iL] + ind0[iL] + 1; ii < start[iL + 1]; ii++) tab[ii] = nSA | absentC;
        }
        {   // pack: 64 entries = (GstrandBit+3) whole words
            const uint32_t bits = GstrandBit + 3;
            uint64_t* out = reinterpret_cast<uint64_t*>(SAistore.data());   // (vector storage is suitably aligned; nSAibyte + 16 bytes)
            const uint64_t nGroups = (nSAi + 63) / 64;
            auto packRange = [&](uint64_t g0, uint64_t g1) {
                for (uint64_t g = g0; g < g1; g++) {
                    const uint64_t e0 = g * 64, e1 = std::min<uint64_t>(nSAi, e0 + 64);
                    uint8_t* base = SAistore.data() + g * bits * 8;
                    if (e1 - e0 == 64) {
                        uint64_t* o = reinterpret_cast<uint64_t*>(base);
                        uint64_t acc = 0; uint32_t sh = 0;
                        for (uint64_t e = e0; e < e1; e++) {
                            const uint64_t val = tab[e];
                            acc |= val << sh;
                            if (sh + bits >= 64) { *o++ = acc; acc = sh + bits > 64 ? val >> (64 - sh) : 0; }
                            sh = (sh + bits) & 63;
                        }
                    } else {   // last, partial group: entry by entry (the buffer is zero-filled)
                        PackedRW w(SAistore.data(), bits);
                        for (uint64_t e = e0; e < e1; e++) w.set(e, tab[e]);
                    }
                }
            };
            (void)out;
            std::vector<std::thread> th;
            const uint64_t per = (nGroups + nT - 1) / nT;
            for (int t = 1; t < nT; t++) if (per * t < nGroups) th.emplace_back(packRange, per * t, std::min(nGroups, per * (t + 1)));
            packRange(0, std::min(nGroups, per));
            for (auto& x : th) x.join();
        }
    }

    return 0;
}

int genomeGenerate(HostParams& P, const star_engine_vtbl_t* eng, std::ostream& logMain, std::string& err) {
    const std::string& gDir = P.genomeDir;
    auto tPhase = std::chrono::steady_clock::now();
    auto phaseDone = [&](const char* what) {   // wall time of every phase in Log.out (the build is minutes for a mammalian genome: say where they go)
        const auto now = std::chrono::steady_clock::now();
        logMain << "   [" << what << ": " << std::chrono::duration<double>(now - tPhase).count() << " s]" << std::endl;
        tPhase = now;
    };
    // Genome_genomeGenerate.cpp:113-133
    const bool annot = P.sjdbFileChrStartEnd[0] != "-" || P.sjdbGTFfile != "-";
    uint64_t sjdbOverhang = P.sjdbOverhang;
    if (annot && (long long)sjdbOverhang <= 0) {
        err = "EXITING because of FATAL INPUT PARAMETER ERROR: for generating genome with annotations (--sjdbFileChrStartEnd or --sjdbGTFfile options)\nyou need to specify >0 --sjdbOverhang\nSOLUTION: re-run genome generation specifying non-zero --sjdbOverhang, which ideally should be equal to OneMateLength-1, or could be chosen generically as ~100\n";
        return STAR_EXIT_INPUT_FILES;
    }
    if (!annot) {
        if (P.userSet.count("sjdbOverhang") && sjdbOverhang > 0) {
            err = "EXITING because of FATAL INPUT PARAMETER ERROR: when generating genome without annotations (--sjdbFileChrStartEnd or --sjdbGTFfile options)\ndo not specify >0 --sjdbOverhang\nSOLUTION: re-run genome generation without --sjdbOverhang option\n";
            return STAR_EXIT_INPUT_FILES;
        }
        sjdbOverhang = 0;
    }
    const uint64_t sjdbLength = sjdbOverhang == 0 ? 0 : 2 * sjdbOverhang + 1;
    { time_t t; time(&t); char b[100]; strftime(b, 80, "%b %d %H:%M:%S", localtime(&t)); std::cout << b << " ... starting to generate Genome files\n" << std::flush; }

    // ---- genomeScanFastaFiles.cpp:5-103: chromosomes start at multiples of 2^genomeChrBinNbits, gaps are code 5
    LoadedIndex idx;
    const uint64_t binN = 1ULL << P.genomeChrBinNbits;
    const size_t PAD = 256;
    std::vector<uint8_t>& Gs = idx.Gstore;
    Gs.assign(PAD, 5);
    {
        uint64_t total = 0;
        for (const std::string& fn : P.genomeFastaFiles) { struct stat sb; if (stat(fn.c_str(), &sb) == 0) total += (uint64_t)sb.st_size; }
        Gs.reserve(PAD + total + total / 8 + 2 * binN * 64 + 2 * PAD);
    }
    int rc = scanFastaFiles(P.genomeFastaFiles, binN, idx.chrName, idx.chrStart, idx.chrLength, &Gs, PAD, logMain, err);
    if (rc) return rc;
    phaseDone("FASTA scan");
    const uint32_t nChr = (uint32_t)idx.chrName.size();
    const uint64_t nGenome = idx.chrStart[nChr];
    Gs.resize(PAD + nGenome, 5);
    Gs.resize(PAD + nGenome + PAD, 5);
    uint64_t nGenomeTrue = 0;
    logMain << "Chromosome sequence lengths: \n";
    for (uint32_t i = 0; i < nChr; i++) { nGenomeTrue += idx.chrLength[i]; logMain << idx.chrName[i] << "\t" << idx.chrLength[i] << "\n"; }
    logMain << "Genome sequence total length = " << nGenomeTrue << "\nGenome size with padding = " << nGenome << "\n";
    if ((double)P.genomeSAindexNbases > std::log2((double)nGenomeTrue) / 2 - 1)
        logMain << "!!!!! WARNING: --genomeSAindexNbases " << P.genomeSAindexNbases << " is too large for the genome size=" << nGenomeTrue
                << ", which may cause seg-fault at the mapping step. Re-run genome generation with recommended --genomeSAindexNbases " << int(std::log2((double)nGenomeTrue) / 2 - 1) << "\n";
    mkdir(gDir.c_str(), 0755);
    {   // writeChrInfo, Genome_genomeGenerate.cpp:417-432
        std::ofstream cn(gDir + "chrName.txt"), cs(gDir + "chrStart.txt"), cl(gDir + "chrLength.txt"), cnl(gDir + "chrNameLength.txt");
        if (!cn.good()) { err = "EXITING because of fatal ERROR: could not create output file " + gDir + "chrName.txt\nSOLUTION: check the path and permissions of --genomeDir\n"; return STAR_EXIT_PARAMETER; }
        for (uint32_t i = 0; i < nChr; i++) {
            cn << idx.chrName[i] << "\n"; cs << idx.chrStart[i] << "\n"; cl << idx.chrLength[i] << "\n"; cnl << idx.chrName[i] << "\t" << idx.chrLength[i] << "\n";
        }
        cs << idx.chrStart[nChr] << "\n";
    }
    // ---- suffix array: every position of G + reverse complement that starts with a base (Genome_genomeGenerate.cpp:178-330)
    uint64_t nSA = 0;
    for (uint64_t i = 0; i < nGenome; i++) nSA += Gs[PAD + i] < 4;
    nSA *= 2;
    uint32_t GstrandBit = (uint32_t)std::floor(std::log((double)(nGenome + P.limitSjdbInsertNsj * sjdbLength)) / std::log(2.0)) + 1;
    if (GstrandBit < 32) GstrandBit = 32;
    logMain << "Estimated genome size with padding and SJs: total=genome+SJ=" << nGenome + P.limitSjdbInsertNsj * sjdbLength << " = " << nGenome << " + " << P.limitSjdbInsertNsj * sjdbLength
            << "\nGstrandBit=" << GstrandBit << "\nNumber of SA indices: " << nSA << "\n";
    if (nSA == 0) { err = "EXITING because of INPUT ERROR: the genome contains no A/C/G/T bases\n"; return STAR_EXIT_INPUT_FILES; }
    const uint64_t nSAbyte = (nSA - 1) * (GstrandBit + 1) / 8 + 8;
    idx.SAstore.assign(nSAbyte + 16, 0);
    { time_t t; time(&t); char b[100]; strftime(b, 80, "%b %d %H:%M:%S", localtime(&t)); std::cout << b << " ... starting to sort Suffix Array. This may take a long time...\n" << std::flush; }
    rc = eng->sa_build(P.gpuDevice, Gs.data() + PAD, nGenome, GstrandBit, nSA, idx.SAstore.data(), nSAbyte);
    if (rc) { err = std::string("EXITING because of FATAL ERROR: suffix array generation failed: ") + eng->last_error() + "\n"; return rc; }
    phaseDone("suffix array (device sort + copies)");

    // ---- SAindex, genomeSAindex.cpp:6-220
    { time_t t; time(&t); char b[100]; strftime(b, 80, "%b %d %H:%M:%S", localtime(&t)); std::cout << b << " ... generating Suffix Array index\n" << std::flush; }
    const uint32_t Lmax = (uint32_t)P.genomeSAindexNbases;
    uint64_t nSAi = 0, nSAibyte = 0;
    rc = buildSAindex(Gs.data() + PAD, nGenome, idx.SAstore.data(), nSA, GstrandBit, Lmax, P.runThreadN, idx.genomeSAindexStart, idx.SAistore, nSAi, nSAibyte, err);
    if (rc) return rc;

    phaseDone("SAindex");
    // ---- the loaded-index view, then the junction inserts (Genome_genomeGenerate.cpp:337-345)
    star_index_view_t& v = idx.view;
    memset(&v, 0, sizeof(v));
    v.nGenome = nGenome; v.nSA = nSA; v.nSAbyte = nSAbyte; v.nSAi = nSAi; v.nSAibyte = nSAibyte;
    v.GstrandBit = GstrandBit; v.gSAindexNbases = Lmax; v.gSAsparseD = 1; v.gChrBinNbits = (uint32_t)P.genomeChrBinNbits; v.nChrReal = nChr;
    v.sjdbOverhang = sjdbOverhang; v.sjdbLength = sjdbLength; v.sjGstart = nGenome;
    idx.genomeDir = gDir;
    {
        const uint64_t chrBinN = idx.chrStart[nChr] / binN + 1;   // chrBinFill, Genome.cpp:209-216
        idx.chrBin.resize(chrBinN);
        for (uint64_t ii = 0, ichr = 1; ii < chrBinN; ++ii) { if (ii * binN >= idx.chrStart[ichr]) ichr++; idx.chrBin[ii] = ichr - 1; }
    }
    idx.pointView();
    if (annot) {
        HostParams Pi = P;
        Pi.sjdbInsertOutDir = gDir;
        Pi.sjdbInsertSave = "Basic";   // the index files are written below
        SjdbLoci loci;
        rc = sjdbInsertJunctions(Pi, &P.hp, idx, loci, false, "", eng, logMain, err, /*generateMode*/ true);
        if (rc) return rc;
    }
    if (annot) phaseDone("junction insertion");
    // ---- genomeParameters.txt (genomeParametersWrite.cpp:4-46), Genome, SA, SAindex
    {
        std::ofstream gp(gDir + "genomeParameters.txt");
        gp << "### " << P.commandLineFull << "\n### GstrandBit " << GstrandBit << "\nversionGenome\t2.7.4a\ngenomeType\tFull\ngenomeFastaFiles\t";
        for (auto& f : P.genomeFastaFiles) gp << f << " ";
        gp << "\ngenomeSAindexNbases\t" << Lmax << "\ngenomeChrBinNbits\t" << P.genomeChrBinNbits << "\ngenomeSAsparseD\t1\ngenomeTransformType\tNone\ngenomeTransformVCF\t-\n";
        gp << "sjdbOverhang\t" << sjdbOverhang << "\nsjdbFileChrStartEnd\t";
        for (auto& f : P.sjdbFileChrStartEnd) gp << f << " ";
        gp << "\nsjdbGTFfile\t" << P.sjdbGTFfile << "\nsjdbGTFchrPrefix\t" << P.sjdbGTFchrPrefix << "\nsjdbGTFfeatureExon\t" << P.sjdbGTFfeatureExon
           << "\nsjdbGTFtagExonParentTranscript\t" << P.sjdbGTFtagExonParentTranscript << "\nsjdbGTFtagExonParentGene\t" << P.sjdbGTFtagExonParentGene
           << "\nsjdbInsertSave\t" << P.sjdbInsertSave << "\ngenomeFileSizes\t" << v.nGenome << " " << v.nSAbyte << "\n";
    }
    std::ofstream(gDir + "Genome", std::ios::binary).write((const char*)v.G, v.nGenome);
    std::ofstream(gDir + "SA", std::ios::binary).write((const char*)v.SA, v.nSAbyte);
    {
        std::ofstream sai(gDir + "SAindex", std::ios::binary);
        const uint64_t nb = Lmax;
        sai.write((const char*)&nb, 8);
        sai.write((const char*)idx.genomeSAindexStart.data(), 8 * (nb + 1));
        sai.write((const char*)v.SAi, v.nSAibyte);
    }
    phaseDone("index files written");
    { time_t t; time(&t); char b[100]; strftime(b, 80, "%b %d %H:%M:%S", localtime(&t)); std::cout << b << " ..... finished successfully\n" << std::flush; }
    return 0;
}

}  // namespace starhost
