// genome_load.cpp — reads a STAR genomeDir unchanged (SURVEY.md Appendix A).
//
// Follows Genome::genomeLoad (reference source/Genome_genomeLoad.cpp:18-420), Genome::chrInfoLoad
// (Genome.cpp:139-206), Genome::chrBinFill (Genome.cpp:209-216) and Genome::loadSJDB
// (Genome_genomeLoad.cpp:471-520).  Shared-memory loading is not built: GPU HBM residency replaces it.
#include <sys/stat.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <fstream>
#include <ostream>
#include <sstream>

#include "host.h"

namespace starhost {

static bool readWhole(const std::string& path, std::vector<uint8_t>& dst, size_t padFront, size_t padBack, uint8_t padVal, uint64_t& nBytes) {
    FILE* f = fopen(path.c_str(), "rb");
    if (!f) return false;
    struct stat st;
    if (fstat(fileno(f), &st) != 0) { fclose(f); return false; }
    nBytes = (uint64_t)st.st_size;
    dst.assign(padFront + nBytes + padBack, padVal);
    size_t got = 0;
    while (got < nBytes) {
        size_t r = fread(dst.data() + padFront + got, 1, nBytes - got, f);
        if (r == 0) break;
        got += r;
    }
    fclose(f);
    return got == nBytes;
}

int loadIndex(const std::string& gDirIn, star_params_t* p, LoadedIndex& L, std::string& err, std::string* log, bool chrInfoOnly) {
    std::string gDir = gDirIn;
    std::ostringstream lg;
    auto fail = [&](int code, const std::string& m) { err = m; if (log) *log = lg.str(); return code; };
    // ---- genomeParameters.txt :34-62
    uint32_t GstrandBit = 0;
    uint32_t gSAindexNbases = 14, gChrBinNbits = 18, gSAsparseD = 1;
    uint64_t sjdbOverhangGen = 0;
    std::string genomeType = "Full", transformType = "None";
    {
        std::ifstream pf(gDir + "/genomeParameters.txt");
        if (!pf.good())
            return fail(STAR_EXIT_GENOME_FILES, "EXITING because of FATAL ERROR: could not open genome file " + gDir + "/genomeParameters.txt\n" +
                        "SOLUTION: check that the path to genome files, specified in --genomeDir is correct and the files are present, and have user read permsissions\n");
        std::string line;
        while (std::getline(pf, line)) {
            std::istringstream ls(line);
            std::string w1;
            ls >> w1;
            if (w1 == "###") {
                ls >> w1;
                if (w1 == "GstrandBit") { uint32_t g = 0; ls >> g; GstrandBit = (uint8_t)g; }
                continue;
            }
            if (w1 == "versionGenome") ls >> L.versionGenome;
            else if (w1 == "genomeSAindexNbases") ls >> gSAindexNbases;
            else if (w1 == "genomeChrBinNbits") ls >> gChrBinNbits;
            else if (w1 == "genomeSAsparseD") ls >> gSAsparseD;
            else if (w1 == "sjdbOverhang") ls >> sjdbOverhangGen;
            else if (w1 == "genomeType") ls >> genomeType;
            else if (w1 == "genomeTransformType") ls >> transformType;
            else if (w1 == "sjdbInsertSave") ls >> L.sjdbInsertSaveGenome;
        }
    }
    L.genomeDir = gDir;
    L.sjdbOverhangGenome = sjdbOverhangGen;
    { struct stat st1; L.sjdbInfoExists = stat((gDir + "/sjdbInfo.txt").c_str(), &st1) == 0; }
    if (L.versionGenome.empty())
        return fail(STAR_EXIT_GENOME_FILES, "EXITING because of FATAL ERROR: read no value for the versionGenome parameter from genomeParameters.txt file\nSOLUTION: please re-generate genome from scratch with the latest version of STAR\n");
    if (L.versionGenome != "2.7.4a")  // Parameters.versionGenome of 2.7.11b (parametersDefault)
        return fail(STAR_EXIT_GENOME_FILES, "EXITING because of FATAL ERROR: Genome version: " + L.versionGenome + " is INCOMPATIBLE with running STAR version: 2.7.11b\nSOLUTION: please re-generate genome from scratch with running version of STAR, or with version: 2.7.4a\n");
    if (genomeType != "Full" || transformType != "None")
        return fail(STAR_EXIT_GENOME_FILES, "EXITING because of FATAL ERROR: star-b200 supports --genomeType Full without genome transformation only\n");
    if (gSAsparseD != 1)
        return fail(STAR_EXIT_GENOME_FILES, "EXITING because of FATAL ERROR: star-b200 supports --genomeSAsparseD 1 indices only\n");

    // ---- chrInfoLoad Genome.cpp:139-206
    {
        std::ifstream cn(gDir + "/chrName.txt");
        if (cn.fail()) return fail(STAR_EXIT_INPUT_FILES, "EXITING because of FATAL error, could not open file " + gDir + "/chrName.txt\nSOLUTION: re-generate genome files with STAR --runMode genomeGenerate\n");
        std::string s;
        while (std::getline(cn, s)) { if (s.empty()) break; L.chrName.push_back(s); }
        uint32_t n = (uint32_t)L.chrName.size();
        L.chrStart.resize(n + 1); L.chrLength.resize(n);
        std::ifstream cl(gDir + "/chrLength.txt");
        if (cl.fail()) return fail(STAR_EXIT_INPUT_FILES, "EXITING because of FATAL error, could not open file " + gDir + "/chrLength.txt\nSOLUTION: re-generate genome files with STAR --runMode genomeGenerate\n");
        for (uint32_t i = 0; i < n; i++) cl >> L.chrLength[i];
        std::ifstream cs(gDir + "/chrStart.txt");
        if (cs.fail()) return fail(STAR_EXIT_INPUT_FILES, "EXITING because of FATAL error, could not open file " + gDir + "/chrStart.txt\nSOLUTION: re-generate genome files with STAR --runMode genomeGenerate\n");
        for (uint32_t i = 0; i <= n; i++) cs >> L.chrStart[i];
        lg << "Number of real (reference) chromosomes= " << n << "\n";
    }
    if (chrInfoOnly) {   // enough for SAM headers / SJ.out.tab of a shard merge: names, starts, lengths, chrBin
        star_index_view_t& v0 = L.view;
        memset(&v0, 0, sizeof(v0));
        uint32_t nChr = (uint32_t)L.chrName.size();
        uint64_t nb = 1ULL << gChrBinNbits;
        uint64_t chrBinN = L.chrStart[nChr] / nb + 1;
        L.chrBin.resize(chrBinN);
        for (uint64_t ii = 0, ichr = 1; ii < chrBinN; ++ii) {
            if (ii * nb >= L.chrStart[ichr]) ichr++;
            L.chrBin[ii] = ichr - 1;
        }
        v0.gChrBinNbits = gChrBinNbits; v0.nChrReal = nChr; v0.chrStart = L.chrStart.data(); v0.chrLength = L.chrLength.data();
        if (log) *log = lg.str();
        return 0;
    }
    // ---- Genome / SA / SAindex :303-345
    uint64_t nGenome = 0, nSAbyte = 0, nSAiFile = 0;
    const size_t PAD = 256;  // the reference pads 200 bytes of code 5 (K-1) on both sides, :27,320-323
    if (!readWhole(gDir + "/Genome", L.Gstore, PAD, PAD, 5, nGenome))
        return fail(STAR_EXIT_GENOME_FILES, "EXITING because of FATAL ERROR: could not open genome file " + gDir + "/Genome\nSOLUTION: check that the path to genome files, specified in --genomeDir is correct and the files are present, and have user read permsissions\n");
    if (!readWhole(gDir + "/SA", L.SAstore, 0, 16, 0, nSAbyte))
        return fail(STAR_EXIT_GENOME_FILES, "EXITING because of FATAL ERROR: could not open genome file " + gDir + "/SA\nSOLUTION: check that the path to genome files, specified in --genomeDir is correct and the files are present, and have user read permsissions\n");
    std::vector<uint8_t> saiFile;
    if (!readWhole(gDir + "/SAindex", saiFile, 0, 16, 0, nSAiFile))
        return fail(STAR_EXIT_GENOME_FILES, "EXITING because of FATAL ERROR: could not open genome file " + gDir + "/SAindex\nSOLUTION: check that the path to genome files, specified in --genomeDir is correct and the files are present, and have user read permsissions\n");
    uint64_t nb64 = 0;
    memcpy(&nb64, saiFile.data(), 8);
    gSAindexNbases = (uint32_t)nb64;
    L.genomeSAindexStart.resize(gSAindexNbases + 1);
    memcpy(L.genomeSAindexStart.data(), saiFile.data() + 8, 8 * (gSAindexNbases + 1));
    uint64_t nSAi = L.genomeSAindexStart[gSAindexNbases];
    size_t saiHeader = 8 + 8 * (gSAindexNbases + 1);
    L.SAistore.assign(saiFile.begin() + saiHeader, saiFile.end());
    saiFile.clear(); saiFile.shrink_to_fit();
    if (GstrandBit == 0) {  // :147-151
        GstrandBit = (uint32_t)std::floor(std::log((double)nGenome) / std::log(2.0)) + 1;
        if (GstrandBit < 32) GstrandBit = 32;
    }
    uint64_t nSA = (nSAbyte * 8) / (GstrandBit + 1);
    uint64_t nSAibyte = (nSAi - 1) * (GstrandBit + 3) / 8 + 8;  // PackedArray.cpp:13
    if (L.SAistore.size() < nSAibyte)
        return fail(STAR_EXIT_GENOME_FILES, "EXITING because of FATAL ERROR: SAindex file is shorter than its header implies\n");
    lg << "nGenome=" << nGenome << ";  nSAbyte=" << nSAbyte << "\nGstrandBit=" << GstrandBit << "   SA number of indices=" << nSA << "\n";

    // ---- loadSJDB :471-520
    star_index_view_t& v = L.view;
    memset(&v, 0, sizeof(v));
    uint32_t nChrReal = (uint32_t)L.chrName.size();
    if (nGenome == L.chrStart[nChrReal]) {
        v.sjdbN = 0;
        v.sjGstart = L.chrStart[nChrReal] + 1;
        v.sjdbOverhang = sjdbOverhangGen;
    } else {
        std::ifstream sj(gDir + "/sjdbInfo.txt");
        if (sj.fail()) return fail(STAR_EXIT_INPUT_FILES, "EXITING because of FATAL error, could not open file " + gDir + "/sjdbInfo.txt\nSOLUTION: check that the path to genome files, specified in --genomeDir is correct and the files are present, and have user read permsissions\n");
        uint64_t n = 0, ov = 0;
        sj >> n >> ov;
        v.sjdbN = n; v.sjdbOverhang = ov;
        v.sjGstart = L.chrStart[nChrReal];
        L.sjdbStart.resize(n); L.sjdbEnd.resize(n); L.sjDstart.resize(n); L.sjAstart.resize(n);
        L.sjdbMotif.resize(n); L.sjdbShiftLeft.resize(n); L.sjdbShiftRight.resize(n); L.sjdbStrand.resize(n);
        for (uint64_t i = 0; i < n; i++) {
            uint16_t d1, d2, d3, d4;
            sj >> L.sjdbStart[i] >> L.sjdbEnd[i] >> d1 >> d2 >> d3 >> d4;
            L.sjdbMotif[i] = (uint8_t)d1; L.sjdbShiftLeft[i] = (uint8_t)d2; L.sjdbShiftRight[i] = (uint8_t)d3; L.sjdbStrand[i] = (uint8_t)d4;
            L.sjDstart[i] = L.sjdbStart[i] - ov;
            L.sjAstart[i] = L.sjdbEnd[i] + 1;
            if (L.sjdbMotif[i] == 0) { L.sjDstart[i] += L.sjdbShiftLeft[i]; L.sjAstart[i] += L.sjdbShiftLeft[i]; }
        }
        lg << "Processing splice junctions database sjdbN=" << n << ",   pGe.sjdbOverhang=" << ov << " \n";
    }
    v.sjdbLength = v.sjdbOverhang == 0 ? 0 : v.sjdbOverhang * 2 + 1;  // :126-127

    // ---- chrBinFill Genome.cpp:209-216 (host copy for SJ.out.tab; the engine builds its own)
    {
        uint64_t nb = 1ULL << gChrBinNbits;
        uint64_t chrBinN = L.chrStart[nChrReal] / nb + 1;
        L.chrBin.resize(chrBinN);
        for (uint64_t ii = 0, ichr = 1; ii < chrBinN; ++ii) {
            if (ii * nb >= L.chrStart[ichr]) ichr++;
            L.chrBin[ii] = ichr - 1;
        }
    }
    windowGeometry(p, nGenome, gChrBinNbits);

    v.nGenome = nGenome;
    v.nSA = nSA; v.nSAbyte = nSAbyte;
    v.nSAi = nSAi; v.nSAibyte = nSAibyte;
    v.GstrandBit = GstrandBit; v.gSAindexNbases = gSAindexNbases; v.gSAsparseD = gSAsparseD; v.gChrBinNbits = gChrBinNbits;
    v.nChrReal = nChrReal;
    L.pointView();
    if (log) *log = lg.str();
    return 0;
}

// Genome_genomeLoad.cpp:382-410; recomputed from scratch on every call (after references are added, with the grown genome)
void windowGeometry(star_params_t* p, uint64_t nGenome, uint32_t gChrBinNbits, std::ostream* logMain) {
    if (p->alignIntronMax == 0 && p->alignMatesGapMax == 0) {
    } else {
        p->winBinNbits = (uint64_t)std::floor(std::log2((double)(std::max(std::max(4ULL, (unsigned long long)p->alignIntronMax),
                                                                          (p->alignMatesGapMax == 0 ? 1000ULL : (unsigned long long)p->alignMatesGapMax)) / 4)) + 0.5);
        p->winBinNbits = std::max((uint64_t)p->winBinNbits, (uint64_t)std::floor(std::log2((double)(nGenome / 40000 + 1)) + 0.5));
        if (logMain) *logMain << "To accommodate alignIntronMax=" << p->alignIntronMax << " redefined winBinNbits=" << p->winBinNbits << "\n";
    }
    if (p->winBinNbits > gChrBinNbits) p->winBinNbits = gChrBinNbits;
    if (p->alignIntronMax == 0 && p->alignMatesGapMax == 0) {
    } else {
        p->winFlankNbins = std::max(p->alignIntronMax, p->alignMatesGapMax) / (1ULL << p->winBinNbits) + 1;
        p->winAnchorDistNbins = 2 * p->winFlankNbins;
    }
    p->winBinChrNbits = gChrBinNbits - p->winBinNbits;
    p->winBinN = nGenome / (1ULL << p->winBinNbits) + 1;
}

void LoadedIndex::pointView() {
    star_index_view_t& v = view;
    v.G = Gstore.data() + 256;   // PAD of loadIndex
    v.SA = SAstore.data();
    v.SAi = SAistore.data();
    v.genomeSAindexStart = genomeSAindexStart.data();
    v.chrStart = chrStart.data(); v.chrLength = chrLength.data();
    v.sjdbStart = sjdbStart.data(); v.sjdbEnd = sjdbEnd.data(); v.sjDstart = sjDstart.data(); v.sjAstart = sjAstart.data();
    v.sjdbMotif = sjdbMotif.data(); v.sjdbShiftLeft = sjdbShiftLeft.data(); v.sjdbShiftRight = sjdbShiftRight.data(); v.sjdbStrand = sjdbStrand.data();
}

}  // namespace starhost

// ---- C API ---------------------------------------------------------------------------------
struct star_index {
    starhost::LoadedIndex L;
};
static thread_local std::string g_host_err;

extern "C" {
int star_index_load(const char* genomeDir, star_params_t* p, star_index_t** out) {
    star_index* s = new star_index;
    std::string err;
    int rc = starhost::loadIndex(genomeDir, p, s->L, err, nullptr);
    if (rc) { g_host_err = err; delete s; *out = nullptr; return rc; }
    *out = s;
    return 0;
}
const star_index_view_t* star_index_get(const star_index_t* idx) { return &idx->L.view; }
void star_index_free(star_index_t* idx) { delete idx; }
const char* star_host_last_error(void) { return g_host_err.c_str(); }
}
