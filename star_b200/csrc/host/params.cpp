// params.cpp — command-line parameters of the drop-in CLI.
//
// Mirrors the reference's parameter machinery for the subset the alignment path uses
// (reference source/Parameters.cpp:19-305 registry, :310-470 input levels, :944-1124 derived values,
// defaults from source/parametersDefault).  Every other STAR parameter is recognised by name and
// rejected with a clear message when given: config breadth is outside the hot-path scope (SURVEY.md §2).
#include <cstdio>
#include <thread>
#include <sched.h>
#include <cmath>
#include <cstring>
#include <fstream>
#include <functional>
#include <limits>
#include <sstream>

#include "host.h"

namespace starhost {

int HostParams::allowedCpus() {
    int n = (int)std::thread::hardware_concurrency();
    cpu_set_t set;
    CPU_ZERO(&set);
    if (sched_getaffinity(0, sizeof(set), &set) == 0 && CPU_COUNT(&set) > 0) n = CPU_COUNT(&set);
    // cgroup v2: "<quota> <period>" or "max <period>"; cgroup v1: two files
    double quota = -1, period = -1;
    if (FILE* f = fopen("/sys/fs/cgroup/cpu.max", "r")) {
        char q[64] = {0};
        double p = 0;
        if (fscanf(f, "%63s %lf", q, &p) == 2 && strcmp(q, "max") != 0) { quota = atof(q); period = p; }
        fclose(f);
    } else {
        FILE* fq = fopen("/sys/fs/cgroup/cpu/cpu.cfs_quota_us", "r");
        FILE* fp = fopen("/sys/fs/cgroup/cpu/cpu.cfs_period_us", "r");
        if (fq && fp) { if (fscanf(fq, "%lf", &quota) != 1) quota = -1; if (fscanf(fp, "%lf", &period) != 1) period = -1; }
        if (fq) fclose(fq);
        if (fp) fclose(fp);
    }
    if (quota > 0 && period > 0) {
        const int q = (int)((quota + period - 1) / period);
        if (q >= 1 && q < n) n = q;
    }
    return n < 1 ? 1 : n;
}

void paramsDefault(star_params_t* p) {  // source/parametersDefault
    memset(p, 0, sizeof(*p));
    p->seedSearchStartLmax = 50;
    p->seedSearchStartLmaxOverLread = 1.0;
    p->seedSearchLmax = 0;
    p->seedMapMin = 5;
    p->seedSplitMin = 12;
    p->seedMultimapNmax = 10000;
    p->seedPerReadNmax = 1000;
    p->seedPerWindowNmax = 50;
    p->maxNsplit = 10;  // Parameters.cpp:473
    p->winAnchorMultimapNmax = 50;
    p->winBinNbits = 16;
    p->winAnchorDistNbins = 9;
    p->winFlankNbins = 4;
    p->alignWindowsPerReadNmax = 10000;
    p->alignTranscriptsPerWindowNmax = 100;
    p->alignTranscriptsPerReadNmax = 10000;
    p->alignIntronMin = 21;
    p->alignIntronMax = 0;
    p->alignMatesGapMax = 0;
    p->alignSJoverhangMin = 5;
    p->alignSJDBoverhangMin = 3;
    p->alignSJstitchMismatchNmax[0] = 0; p->alignSJstitchMismatchNmax[1] = -1; p->alignSJstitchMismatchNmax[2] = 0; p->alignSJstitchMismatchNmax[3] = 0;
    p->alignSplicedMateMapLmin = 0;
    p->alignSplicedMateMapLminOverLmate = 0.66;
    p->alignEndsProtrudeNbasesMax = 0;
    p->alignEndsProtrudeConcordantPair = 0;
    p->alignSoftClipAtReferenceEnds = 1;
    p->alignInsertionFlushRight = 0;
    p->scoreGap = 0; p->scoreGapNoncan = -8; p->scoreGapGCAG = -4; p->scoreGapATAC = -8;
    p->scoreGenomicLengthLog2scale = -0.25;
    p->scoreDelOpen = -2; p->scoreDelBase = -2; p->scoreInsOpen = -2; p->scoreInsBase = -2; p->scoreStitchSJshift = 1;
    p->sjdbScore = 2;
    p->outFilterMismatchNmax = 10;
    p->outFilterMismatchNoverLmax = 0.3;
    p->outFilterMismatchNoverReadLmax = 1.0;
    p->outFilterMultimapScoreRange = 1;
    p->outFilterMultimapNmax = 10;
    p->outFilterScoreMin = 0;
    p->outFilterScoreMinOverLread = 0.66;
    p->outFilterMatchNmin = 0;
    p->outFilterMatchNminOverLread = 0.66;
    p->outFilterIntronMotifs = 0;
    p->outFilterIntronStrandsRemoveInconsistent = 1;
    p->outSAMstrandFieldType = 0;
    p->outSAMprimaryFlagAllBestScore = 0;
    p->outSAMmultNmax = (uint64_t)-1;
}

namespace {

typedef std::vector<std::string> Vals;
struct Setter {
    std::function<bool(const Vals&)> fn;
};

template <class T>
bool parseNum(const std::string& s, T& out) {
    std::istringstream is(s);
    is >> out;
    return !is.fail() && is.eof();
}
// the reference reads unsigned parameters through operator>> which accepts "-1" as 2^64-1
bool parseU64(const std::string& s, uint64_t& out) {
    if (!s.empty() && s[0] == '-') { long long v; if (!parseNum(s, v)) return false; out = (uint64_t)v; return true; }
    return parseNum(s, out);
}

// STAR parameters that exist in the reference but belong to subsystems outside the hot path (SURVEY.md §2)
const char* kUnsupported[] = {
    "genomeChainFiles", "genomeFileSizes", "genomeTransformOutput", "genomeChrSetMitochondrial", "genomeSuffixLengthMax",
    "genomeTransformType", "genomeTransformVCF", "genomeType", "varVCFfile", "readFilesType", "readFilesSAMattrKeep",
    "peOverlapNbasesMin", "peOverlapMMp", "chimOutType",
    "chimSegmentMin", "chimScoreMin", "chimScoreDropMax", "chimScoreSeparation", "chimScoreJunctionNonGTAG", "chimJunctionOverhangMin",
    "chimSegmentReadGapMax", "chimFilter", "chimMainSegmentMultNmax", "chimMultimapNmax", "chimMultimapScoreRange",
    "chimNonchimScoreDropMin", "chimOutJunctionFormat", "waspOutputMode", "soloType", "soloCBtype", "soloCBwhitelist", "soloCBstart",
    "soloCBlen", "soloUMIstart", "soloUMIlen", "soloBarcodeReadLength", "soloBarcodeMate", "soloCBposition", "soloUMIposition",
    "soloAdapterSequence", "soloAdapterMismatchesNmax", "soloCBmatchWLtype", "soloInputSAMattrBarcodeSeq",
    "soloInputSAMattrBarcodeQual", "soloStrand", "soloFeatures", "soloMultiMappers", "soloUMIdedup", "soloUMIfiltering",
    "soloOutFileNames", "soloCellFilter", "soloOutFormatFeaturesGeneField3", "soloCellReadStats", "soloClusterCBfile", "sjdbScoreX",
    "clip5pAdapterSeq", "clip5pAdapterMMp", "clip5pAfterAdapterNbases"};

// resource / housekeeping knobs of the reference that cannot change any output here (buffers are sized from the chunk, the BAM sort is in
// memory, there are no temporary files): accepted and ignored, so that existing command lines keep working
const char* kIgnored[] = {"sysShell", "runDirPerm", "limitIObufferSize", "limitOutSAMoneReadBytes", "limitOutSJoneRead", "limitOutSJcollapsed",
                          "limitBAMsortRAM", "limitNreadsSoft", "outTmpDir", "outTmpKeep", "outBAMsortingThreadN", "outBAMsortingBinsN",
                          // read by the long-read stitcher / solo statistics only: no effect in the short-read build of the reference either
                          "seedNoneLociPerWindow", "winReadCoverageRelativeMin", "winReadCoverageBasesMin", "readQualityScoreBase"};

}  // namespace

int parseCommandLine(int argc, char** argv, HostParams& P, std::string& err) {
    paramsDefault(&P.hp);
    star_params_t& h = P.hp;
    std::map<std::string, Setter> tab;
    auto U64 = [&](const char* name, uint64_t* dst) {
        tab[name] = Setter{[dst](const Vals& v) { return v.size() == 1 && parseU64(v[0], *dst); }};
    };
    auto I32 = [&](const char* name, int32_t* dst) {
        tab[name] = Setter{[dst](const Vals& v) { return v.size() == 1 && parseNum(v[0], *dst); }};
    };
    auto DBL = [&](const char* name, double* dst) {
        tab[name] = Setter{[dst](const Vals& v) { return v.size() == 1 && parseNum(v[0], *dst); }};
    };
    auto STR = [&](const char* name, std::string* dst) {
        tab[name] = Setter{[dst](const Vals& v) { if (v.size() != 1) return false; *dst = v[0]; return true; }};
    };
    auto VSTR = [&](const char* name, std::vector<std::string>* dst) {
        tab[name] = Setter{[dst](const Vals& v) { if (v.empty()) return false; *dst = v; return true; }};
    };
    auto VI32 = [&](const char* name, std::vector<int32_t>* dst) {
        tab[name] = Setter{[dst](const Vals& v) {
            if (v.empty()) return false;
            std::vector<int32_t> t(v.size());
            for (size_t i = 0; i < v.size(); i++) if (!parseNum(v[i], t[i])) return false;
            *dst = t;
            return true;
        }};
    };
    U64("seedSearchStartLmax", &h.seedSearchStartLmax); DBL("seedSearchStartLmaxOverLread", &h.seedSearchStartLmaxOverLread);
    U64("seedSearchLmax", &h.seedSearchLmax); U64("seedMapMin", &h.seedMapMin); U64("seedSplitMin", &h.seedSplitMin);
    U64("seedMultimapNmax", &h.seedMultimapNmax); U64("seedPerReadNmax", &h.seedPerReadNmax); U64("seedPerWindowNmax", &h.seedPerWindowNmax);
    U64("winAnchorMultimapNmax", &h.winAnchorMultimapNmax); U64("winBinNbits", &h.winBinNbits); U64("winAnchorDistNbins", &h.winAnchorDistNbins);
    U64("winFlankNbins", &h.winFlankNbins); U64("alignWindowsPerReadNmax", &h.alignWindowsPerReadNmax);
    U64("alignTranscriptsPerWindowNmax", &h.alignTranscriptsPerWindowNmax); U64("alignTranscriptsPerReadNmax", &h.alignTranscriptsPerReadNmax);
    U64("alignIntronMin", &h.alignIntronMin); U64("alignIntronMax", &h.alignIntronMax); U64("alignMatesGapMax", &h.alignMatesGapMax);
    U64("alignSJoverhangMin", &h.alignSJoverhangMin); U64("alignSJDBoverhangMin", &h.alignSJDBoverhangMin);
    U64("alignSplicedMateMapLmin", &h.alignSplicedMateMapLmin); DBL("alignSplicedMateMapLminOverLmate", &h.alignSplicedMateMapLminOverLmate);
    tab["alignSJstitchMismatchNmax"] = Setter{[&h](const Vals& v) {
        if (v.size() != 4) return false;
        for (int i = 0; i < 4; i++) if (!parseNum(v[i], h.alignSJstitchMismatchNmax[i])) return false;
        return true;
    }};
    I32("scoreGap", &h.scoreGap); I32("scoreGapNoncan", &h.scoreGapNoncan); I32("scoreGapGCAG", &h.scoreGapGCAG); I32("scoreGapATAC", &h.scoreGapATAC);
    DBL("scoreGenomicLengthLog2scale", &h.scoreGenomicLengthLog2scale);
    I32("scoreDelOpen", &h.scoreDelOpen); I32("scoreDelBase", &h.scoreDelBase); I32("scoreInsOpen", &h.scoreInsOpen); I32("scoreInsBase", &h.scoreInsBase);
    I32("scoreStitchSJshift", &h.scoreStitchSJshift); I32("sjdbScore", &h.sjdbScore);
    STR("sjdbGTFfile", &P.sjdbGTFfile); STR("sjdbGTFchrPrefix", &P.sjdbGTFchrPrefix); STR("sjdbGTFfeatureExon", &P.sjdbGTFfeatureExon);
    STR("sjdbGTFtagExonParentTranscript", &P.sjdbGTFtagExonParentTranscript); STR("sjdbGTFtagExonParentGene", &P.sjdbGTFtagExonParentGene);
    VSTR("sjdbGTFtagExonParentGeneName", &P.sjdbGTFtagExonParentGeneName); VSTR("sjdbGTFtagExonParentGeneType", &P.sjdbGTFtagExonParentGeneType);
    VSTR("genomeFastaFiles", &P.genomeFastaFiles); VSTR("outSAMfilter", &P.outSAMfilter); U64("genomeSAindexNbases", &P.genomeSAindexNbases); U64("genomeChrBinNbits", &P.genomeChrBinNbits);
    U64("genomeSAsparseD", &P.genomeSAsparseD); U64("limitGenomeGenerateRAM", &P.limitGenomeGenerateRAM);
    VSTR("sjdbFileChrStartEnd", &P.sjdbFileChrStartEnd); U64("sjdbOverhang", &P.sjdbOverhang); STR("sjdbInsertSave", &P.sjdbInsertSave);
    U64("limitSjdbInsertNsj", &P.limitSjdbInsertNsj); STR("twopassMode", &P.twopassMode); U64("twopass1readsN", &P.twopass1readsN);
    U64("outFilterMismatchNmax", &h.outFilterMismatchNmax); DBL("outFilterMismatchNoverLmax", &h.outFilterMismatchNoverLmax);
    DBL("outFilterMismatchNoverReadLmax", &h.outFilterMismatchNoverReadLmax); I32("outFilterMultimapScoreRange", &h.outFilterMultimapScoreRange);
    U64("outFilterMultimapNmax", &h.outFilterMultimapNmax); I32("outFilterScoreMin", &h.outFilterScoreMin);
    DBL("outFilterScoreMinOverLread", &h.outFilterScoreMinOverLread); U64("outFilterMatchNmin", &h.outFilterMatchNmin);
    DBL("outFilterMatchNminOverLread", &h.outFilterMatchNminOverLread); U64("outSAMmultNmax", &h.outSAMmultNmax);
    STR("runMode", &P.runMode); STR("genomeDir", &P.genomeDir); STR("genomeLoad", &P.genomeLoad); VSTR("readFilesIn", &P.readFilesIn); STR("readFilesPrefix", &P.readFilesPrefix); STR("readFilesManifest", &P.readFilesManifest);
    VSTR("readFilesCommand", &P.readFilesCommand); VSTR("readNameSeparator", &P.readNameSeparator); STR("outFileNamePrefix", &P.outFileNamePrefix);
    STR("outStd", &P.outStd); VSTR("outSAMtype", &P.outSAMtype); STR("outSAMmode", &P.outSAMmode); STR("outSAMstrandField", &P.outSAMstrandField);
    VSTR("outSAMattributes", &P.outSAMattributes); VSTR("outSAMunmapped", &P.outSAMunmapped); STR("outReadsUnmapped", &P.outReadsUnmapped); VSTR("clip5pNbases", &P.clip5pNbases); VSTR("clip3pNbases", &P.clip3pNbases); VSTR("clip3pAdapterSeq", &P.clip3pAdapterSeq);
    VSTR("clip3pAdapterMMp", &P.clip3pAdapterMMp); VSTR("clip3pAfterAdapterNbases", &P.clip3pAfterAdapterNbases); VSTR("clipAdapterType", &P.clipAdapterType);
    VSTR("quantMode", &P.quantMode); I32("outSAMtlen", &P.outSAMtlen); I32("outQSconversionAdd", &P.outQSconversionAdd); VSTR("outSAMheaderHD", &P.outSAMheaderHD); VSTR("outSAMheaderPG", &P.outSAMheaderPG);
    STR("outSAMheaderCommentFile", &P.outSAMheaderCommentFile); STR("quantTranscriptomeSAMoutput", &P.quantTranscriptomeSAMoutput);
    I32("quantTranscriptomeBAMcompression", &P.quantTranscriptomeBAMcompression); U64("runRNGseed", &P.runRNGseed); STR("outSAMorder", &P.outSAMorder);
    STR("outSAMprimaryFlag", &P.outSAMprimaryFlag); STR("outSAMreadID", &P.outSAMreadID); VSTR("outSAMattrRGline", &P.outSAMattrRGline);
    STR("outFilterType", &P.outFilterType); STR("outFilterIntronMotifs", &P.outFilterIntronMotifs); STR("outFilterIntronStrands", &P.outFilterIntronStrands);
    VSTR("outSJtype", &P.outSJtype); STR("outSJfilterReads", &P.outSJfilterReads); VI32("outSJfilterOverhangMin", &P.outSJfilterOverhangMin);
    VI32("outSJfilterCountUniqueMin", &P.outSJfilterCountUniqueMin); VI32("outSJfilterCountTotalMin", &P.outSJfilterCountTotalMin);
    VI32("outSJfilterDistToOtherSJmin", &P.outSJfilterDistToOtherSJmin); VI32("outSJfilterIntronMaxVsReadN", &P.outSJfilterIntronMaxVsReadN);
    STR("alignEndsType", &P.alignEndsType); VSTR("alignEndsProtrude", &P.alignEndsProtrude);
    STR("alignSoftClipAtReferenceEnds", &P.alignSoftClipAtReferenceEnds); STR("alignInsertionFlush", &P.alignInsertionFlush);
    STR("outMultimapperOrder", &P.outMultimapperOrder);
    VSTR("outWigType", &P.outWigType); VSTR("outWigStrand", &P.outWigStrand); VSTR("outWigNorm", &P.outWigNorm);
    STR("outWigReferencesPrefix", &P.outWigReferencesPrefix); STR("inputBAMfile", &P.inputBAMfile);
    STR("bamRemoveDuplicatesType", &P.bamRemoveDuplicatesType); U64("bamRemoveDuplicatesMate2basesN", &P.bamRemoveDuplicatesMate2basesN);
    tab["runThreadN"] = Setter{[&P](const Vals& v) { return v.size() == 1 && parseNum(v[0], P.runThreadN) && P.runThreadN > 0; }};
    tab["readMapNumber"] = Setter{[&P](const Vals& v) { return v.size() == 1 && parseNum(v[0], P.readMapNumber); }};
    tab["outSAMattrIHstart"] = Setter{[&P](const Vals& v) { return v.size() == 1 && parseNum(v[0], P.outSAMattrIHstart); }};
    tab["outBAMcompression"] = Setter{[&P](const Vals& v) { return v.size() == 1 && parseNum(v[0], P.outBAMcompression); }};
    tab["outSAMmapqUnique"] = Setter{[&P](const Vals& v) { return v.size() == 1 && parseNum(v[0], P.outSAMmapqUnique); }};
    tab["outSAMflagOR"] = Setter{[&P](const Vals& v) { return v.size() == 1 && parseNum(v[0], P.outSAMflagOR); }};
    tab["outSAMflagAND"] = Setter{[&P](const Vals& v) { return v.size() == 1 && parseNum(v[0], P.outSAMflagAND); }};
    tab["gpuDevice"] = Setter{[&P](const Vals& v) { return v.size() == 1 && parseNum(v[0], P.gpuDevice); }};
    tab["gpuShardIndex"] = Setter{[&P](const Vals& v) { return v.size() == 1 && parseNum(v[0], P.gpuShardIndex); }};
    tab["gpuBySJoutPhase"] = Setter{[&P](const Vals& v) { return v.size() == 1 && parseNum(v[0], P.gpuBySJoutPhase) && P.gpuBySJoutPhase <= 2; }};
    tab["gpuTwoPassPhase"] = Setter{[&P](const Vals& v) { return v.size() == 1 && parseNum(v[0], P.gpuTwoPassPhase) && P.gpuTwoPassPhase <= 2; }};
    tab["gpuShardCount"] = Setter{[&P](const Vals& v) { return v.size() == 1 && parseNum(v[0], P.gpuShardCount) && P.gpuShardCount > 0; }};
    tab["gpuChunkReads"] = Setter{[&P](const Vals& v) { return v.size() == 1 && parseNum(v[0], P.gpuChunkReads) && P.gpuChunkReads > 0; }};

    // Parameters.cpp:331-365: "--name v1 v2", "--name=value"
    std::vector<std::pair<std::string, Vals>> given;
    P.commandLine = argc > 0 ? argv[0] : "STAR";
    for (int i = 1; i < argc; i++) {
        std::string a = argv[i];
        P.commandLine += " " + a;
        if (a == "--version") { err = "version"; return -1; }
        size_t eq = a.find('=');
        if (a.size() > 2 && a.substr(0, 2) == "--" && eq != std::string::npos) {
            given.push_back({a.substr(2, eq - 2), Vals{a.substr(eq + 1)}});
        } else if (a.size() > 2 && a.substr(0, 2) == "--") {
            given.push_back({a.substr(2), Vals{}});
        } else {
            if (given.empty()) { err = "EXITING: FATAL INPUT ERROR: value \"" + a + "\" given before any parameter name\n"; return STAR_EXIT_PARAMETER; }
            given.back().second.push_back(a);
        }
    }
    // --parametersFiles (Parameters.cpp:331-365, 400-440): "name value(s)" lines, '#' comments; the command line overrides them
    std::vector<std::pair<std::string, Vals>> fromFile;
    for (auto& g : given)
        if (g.first == "parametersFiles") {
            for (const std::string& fn : g.second) {
                if (fn == "-") continue;
                std::ifstream pf(fn);
                if (pf.fail()) { err = "EXITING because of fatal input ERROR: could not open user-defined parameters file " + fn + "\n"; return STAR_EXIT_PARAMETER; }
                std::string line;
                while (std::getline(pf, line)) {
                    std::istringstream ls(line);
                    std::string name, v;
                    if (!(ls >> name) || name[0] == '#') continue;
                    Vals vals;
                    while (ls >> v) vals.push_back(v);   // (no inline comments: the reference takes everything after the name as values)
                    fromFile.push_back({name, vals});
                }
            }
        }
    std::map<std::string, int> levelOf;   // 1 = parameters file, 2 = command line
    std::vector<std::pair<std::string, Vals>> ordered;
    std::vector<int> levels;
    for (auto& g : fromFile) { ordered.push_back(g); levels.push_back(1); }
    for (auto& g : given) if (g.first != "parametersFiles") { ordered.push_back(g); levels.push_back(2); }
    std::ostringstream full;
    full << (argc > 0 ? argv[0] : "STAR");
    for (size_t ig = 0; ig < ordered.size(); ig++) {
        auto& g = ordered[ig];
        const int level = levels[ig];
        const char* source = level == 1 ? "parametersFiles" : "Command-Line";
        auto it = tab.find(g.first);
        if (it == tab.end()) {
            bool ignored = false;
            for (const char* u : kIgnored) if (g.first == u) ignored = true;
            if (ignored && !g.second.empty() && !(levelOf.count(g.first) && levelOf[g.first] == level)) {
                P.userSet[g.first] = 2; levelOf[g.first] = level;
                P.ignoredParams.push_back(g.first);
                full << "   --" << g.first;
                for (auto& v : g.second) full << " " << v;
                continue;
            }
            bool known = false;
            for (const char* u : kUnsupported) if (g.first == u) known = true;
            if (known)
                err = "EXITING: FATAL INPUT ERROR: parameter --" + g.first +
                      " belongs to a STAR subsystem that is outside the scope of star-b200 (the GPU alignment hot path); remove it\n";
            else
                err = "EXITING: FATAL INPUT ERROR: unrecognized parameter name \"" + g.first + "\" in input \"" + source + "\"\n" +
                      "SOLUTION: use correct parameter name (check the manual)\n";  // Parameters.cpp:1245-1250
            return STAR_EXIT_PARAMETER;
        }
        if (levelOf.count(g.first) && levelOf[g.first] == level) {
            err = "EXITING: FATAL INPUT ERROR: duplicate parameter \"" + g.first + "\" in input \"" + source + "\"\nSOLUTION: keep only one definition of input parameters in each input source\n";
            return STAR_EXIT_PARAMETER;
        }
        if (g.second.empty()) {
            err = "EXITING: FATAL INPUT ERROR: empty value for parameter \"" + g.first + "\" in input \"" + source + "\"\nSOLUTION: use non-empty value for this parameter\n";
            return STAR_EXIT_PARAMETER;
        }
        if (!it->second.fn(g.second)) {
            err = "EXITING: FATAL INPUT ERROR: could not parse the value of parameter \"" + g.first + "\"\n";
            return STAR_EXIT_PARAMETER;
        }
        P.userSet[g.first] = 2; levelOf[g.first] = level;
        if (level == 2) { full << "   --" << g.first; for (auto& v : g.second) full << " " << v; }
    }
    // duplicate marking exists in --runMode inputAlignmentsFromBAM only; in the other modes (where the reference ignores them) both names
    // stay outside the scope
    if (P.runMode != "inputAlignmentsFromBAM")
        for (auto& g : ordered)
            if (g.first == "bamRemoveDuplicatesType" || g.first == "bamRemoveDuplicatesMate2basesN") {
                err = "EXITING: FATAL INPUT ERROR: parameter --" + g.first +
                      " belongs to a STAR subsystem that is outside the scope of star-b200 (the GPU alignment hot path); remove it\n";
                return STAR_EXIT_PARAMETER;
            }
    P.commandLineFull = full.str();
    return finalizeParams(P, err);
}

int finalizeParams(HostParams& P, std::string& err) {
    star_params_t& h = P.hp;
    auto bad = [&](const std::string& m) { err = m; return STAR_EXIT_PARAMETER; };
    // Parameters.cpp:511-562
    if (P.outWigType[0] == "None") P.wigYes = false;
    else if (P.outWigType[0] == "bedGraph") { P.wigYes = true; P.wigFormat = 0; }
    else if (P.outWigType[0] == "wiggle") { P.wigYes = true; P.wigFormat = 1; }
    else return bad("EXITING because of FATAL INPUT ERROR: unrecognized option in --outWigType=" + P.outWigType[0] + "\nSOLUTION: use one of the allowed values of --outWigType : 'None' or 'bedGraph' \n");
    if (P.outWigStrand[0] == "Stranded") P.wigStranded = true;
    else if (P.outWigStrand[0] == "Unstranded") P.wigStranded = false;
    else return bad("EXITING because of FATAL INPUT ERROR: unrecognized option in --outWigStrand=" + P.outWigStrand[0] + "\nSOLUTION: use one of the allowed values of --outWigStrand : 'Stranded' or 'Unstranded' \n");
    if (P.outWigType.size() == 1) P.wigType = 0;
    else if (P.outWigType[1] == "read1_5p") P.wigType = 1;
    else if (P.outWigType[1] == "read2") P.wigType = 2;
    else return bad("EXITING because of FATAL INPUT ERROR: unrecognized second option in --outWigType=" + P.outWigType[1] + "\nSOLUTION: use one of the allowed values of --outWigType : 'read1_5p' \n");
    if (P.outWigNorm[0] == "None") P.wigNorm = 0;
    else if (P.outWigNorm[0] == "RPM") P.wigNorm = 1;
    else return bad("EXITING because of fatal parameter ERROR: unrecognized option in --outWigNorm=" + P.outWigNorm[0] + "\nSOLUTION: use one of the allowed values of --outWigNorm : 'None' or 'RPM' \n");
    // Parameters.cpp:740-760 (the message names only two of the three values)
    if (P.outSAMfilter[0] == "KeepOnlyAddedReferences") P.outSAMfilterKeepOnly = true;
    else if (P.outSAMfilter[0] == "KeepAllAddedReferences") P.outSAMfilterKeepAll = true;
    else if (P.outSAMfilter[0] != "None")
        return bad("EXITING because of FATAL INPUT ERROR: unknown/unimplemented value for --outSAMfilter: " + P.outSAMfilter[0] + "\nSOLUTION: specify one of the allowed values: KeepOnlyAddedReferences or None\n");
    if ((P.outSAMfilterKeepOnly || P.outSAMfilterKeepAll) && P.genomeFastaFiles[0] == "-")
        return bad("EXITING because of FATAL INPUT ERROR: --outSAMfilter KeepOnlyAddedReferences OR KeepAllAddedReferences options can only be used if references are added on-the-fly with --genomeFastaFiles\nSOLUTION: use default --outSAMfilter None, OR add references with --genomeFataFiles\n");
    if (P.runMode == "inputAlignmentsFromBAM") {   // Parameters.cpp:566-607: no genome, no reads
        if (P.bamRemoveDuplicatesType == "UniqueIdentical") { P.dedupYes = true; P.dedupMarkMulti = true; }
        else if (P.bamRemoveDuplicatesType == "UniqueIdenticalNotMulti") { P.dedupYes = true; P.dedupMarkMulti = false; }
        else if (P.bamRemoveDuplicatesType != "-")
            return bad("EXITING because of fatal PARAMETERS error: unrecognized option in of --bamRemoveDuplicatesType=" + P.bamRemoveDuplicatesType +
                       "\nSOLUTION: use allowed option: - or UniqueIdentical or UniqueIdenticalNotMulti");
        if (!P.wigYes && !P.dedupYes)
            return bad("EXITING because of fatal INPUT ERROR: at the moment --runMode inputFromBAM only works with --outWigType bedGraph OR --bamRemoveDuplicatesType Identical\n");
        return 0;
    }
    if (P.runMode == "genomeGenerate") {   // index generation (genome_generate.cpp): only the genome / junction parameters matter
        if (P.genomeFastaFiles.empty() || P.genomeFastaFiles[0] == "-")
            return bad("EXITING because of fatal PARAMETERS error: --runMode genomeGenerate needs --genomeFastaFiles\n");
        if (P.genomeSAsparseD != 1) return bad("EXITING because of fatal PARAMETERS error: star-b200 builds --genomeSAsparseD 1 indices only\n");
        if (P.genomeSAindexNbases < 1 || P.genomeSAindexNbases > 18) return bad("EXITING because of fatal PARAMETERS error: --genomeSAindexNbases must be in 1..18\n");
        if (P.twopassMode != "None") return bad("EXITING because of fatal PARAMETERS error: 2-pass mapping option  can only be used with --runMode alignReads\nSOLUTION: remove --twopassMode option");
        if (P.sjdbFileChrStartEnd[0] != "-" || P.sjdbGTFfile != "-") { P.sjdbInsertPass1 = true; P.sjdbInsertYes = true; }
        if (P.genomeDir.empty() || P.genomeDir.back() != '/') P.genomeDir += "/";
        return 0;
    }
    if (P.runMode != "alignReads")
        return bad("EXITING because of fatal input ERROR: star-b200 implements --runMode alignReads, genomeGenerate and inputAlignmentsFromBAM only\n");
    if (P.genomeLoad == "LoadAndKeep" || P.genomeLoad == "LoadAndRemove") {   // the index lives in this process' HBM; nothing is shared or kept
        if (P.twopassMode != "None" || P.sjdbFileChrStartEnd[0] != "-" || P.sjdbGTFfile != "-")   // Parameters.cpp:809-814, 1012-1017
            return bad("EXITING because of fatal PARAMETERS error: on the fly junction insertion and 2-pass mappng cannot be used with shared memory genome \nSOLUTION: run STAR with --genomeLoad NoSharedMemory to avoid using shared memory\n");
        // the reference does not size the insert on its shared-memory path (Genome_genomeLoad.cpp:245-250 is the NoSharedMemory branch only)
        if (P.genomeFastaFiles[0] != "-")
            return bad("EXITING because of fatal PARAMETERS error: references cannot be added with --genomeFastaFiles to a shared memory genome (--genomeLoad " + P.genomeLoad + ")\nSOLUTION: run STAR with --genomeLoad NoSharedMemory to add references at the mapping stage\n");
        P.genomeLoad = "NoSharedMemory";
    }
    if (P.genomeLoad != "NoSharedMemory")
        return bad("EXITING because of fatal input ERROR: --genomeLoad " + P.genomeLoad + " is not supported: the index is resident in GPU HBM instead of host shared memory\n");
    if (P.outStd != "Log" && P.outStd != "SAM" && P.outStd != "BAM_Unsorted" && P.outStd != "BAM_SortedByCoordinate" && P.outStd != "BAM_Quant")   // Parameters.cpp:385-396
        return bad("EXITING because of FATAL PARAMETER error: outStd=" + P.outStd + " is not a valid value of the parameter\nSOLUTION: provide a valid value fot outStd: Log / SAM / BAM_Unsorted / BAM_SortedByCoordinate");
    if (P.outStd != "Log" && P.gpuShardCount > 1)
        return bad("EXITING because of fatal input ERROR: --outStd " + P.outStd + " is not supported for sharded (multi-GPU) runs: the shards' outputs are merged from files\n");
    if (P.readFilesManifest != "-") {   // Parameters_readFilesInit.cpp:96-137: Read1 <tab> Read2 (or -) <tab> read group line, one input file (pair) per line
        std::ifstream rfM(P.readFilesManifest);
        if (rfM.fail()) return bad("EXITING because of fatal INPUT error: could not open input file " + P.readFilesManifest + "\nSOLUTION: check the path and permissions for readFilesManifest = " + P.readFilesManifest + "\n");
        std::string m1, m2, line;
        std::vector<std::string> rg;
        bool first = true;
        while (std::getline(rfM, line)) {
            if (line.find_first_not_of(" \t") == std::string::npos) continue;
            const size_t t1 = line.find('\t'), t2 = t1 == std::string::npos ? t1 : line.find('\t', t1 + 1);
            if (t1 == std::string::npos || t2 == std::string::npos) {
                err = "EXITING because of FATAL INPUT FILE error: readFileManifest file " + P.readFilesManifest + " has to contain at least 3 tab separated columns\nSOLUTION: fix the formatting of the readFileManifest file: Read1 <tab> Read2 <tab> ReadGroup. For single-end reads, use - in the 2nd column.\n";
                return STAR_EXIT_INPUT_FILES;
            }
            m1 += (first ? "" : ",") + line.substr(0, t1);
            m2 += (first ? "" : ",") + line.substr(t1 + 1, t2 - t1 - 1);
            std::string g = line.substr(t2 + 1);
            if (g.substr(0, 3) != "ID:") g.insert(0, "ID:");
            if (!first) rg.push_back(",");
            size_t a = 0;
            for (;;) { const size_t b = g.find('\t', a); rg.push_back(g.substr(a, b == std::string::npos ? b : b - a)); if (b == std::string::npos) break; a = b + 1; }
            first = false;
        }
        if (first) return bad("EXITING because of FATAL INPUT FILE error: readFileManifest file " + P.readFilesManifest + " is empty\n");
        P.readFilesIn = {m1};
        if (m2.empty() || m2.back() != '-') P.readFilesIn.push_back(m2);   // (the reference looks at the last character of the first Read2 entry)
        P.outSAMattrRGline = rg;
        P.rgFromManifest = true;
    }
    if (P.readFilesIn.size() > 2 || P.readFilesIn.empty() || P.readFilesIn[0] == "Read1")
        return bad("EXITING: because of fatal input ERROR: --readFilesIn must name 1 or 2 FASTQ/FASTA files\n");
    P.readFilesNames.assign(P.readFilesIn.size(), {});
    for (size_t imate = 0; imate < P.readFilesIn.size(); imate++) {   // Parameters_readFilesInit.cpp:43-62
        std::string cur;
        for (char ch : P.readFilesIn[imate]) { if (ch == ',') { P.readFilesNames[imate].push_back(cur); cur.clear(); } else cur.push_back(ch); }
        if (!cur.empty() || P.readFilesNames[imate].empty()) P.readFilesNames[imate].push_back(cur);   // (an extra comma at the end is ignored)
        if (P.readFilesPrefix != "-") for (auto& fn : P.readFilesNames[imate]) fn = P.readFilesPrefix + fn;   // Parameters_readFilesInit.cpp:40,59
        if (imate > 0 && P.readFilesNames[imate].size() != P.readFilesNames[imate - 1].size())
            return bad("EXITING: because of fatal INPUT ERROR: number of input files for mate" + std::to_string(imate + 1) + "=" + std::to_string(P.readFilesNames[imate].size()) +
                       " is not equal to that for mate" + std::to_string(imate - 1) + "=" + std::to_string(P.readFilesNames[imate - 1].size()) + "\nMake sure that the number of files in --readFilesIn is the same for both mates\n");
    }
    P.readNmates = (unsigned)P.readFilesIn.size();
    if (P.outFilterType != "Normal" && P.outFilterType != "BySJout")   // Parameters.cpp:1176-1190
        return bad("EXITING because of FATAL input ERROR: unknown value of parameter outFilterType: " + P.outFilterType + "\nSOLUTION: re-run STAR with --outFilterType Normal OR BySJout\n");
    if (P.outFilterType == "BySJout" && P.gpuShardCount > 1 && P.gpuBySJoutPhase == 0 && P.gpuTwoPassPhase != 1)   // (the 1st pass of a 2-pass run does not filter)
        return bad("EXITING because of fatal input ERROR: --outFilterType BySJout of a sharded (multi-GPU) run needs the junctions of all shards between its two stages: run it through `python -m star_b200.dist` (which gathers them between --gpuBySJoutPhase 1 and 2)\n");
    if (P.gpuBySJoutPhase != 0 && !(P.outFilterType == "BySJout" && P.gpuShardCount > 1))
        return bad("EXITING because of fatal PARAMETERS error: --gpuBySJoutPhase is only meaningful for a sharded --outFilterType BySJout run\n");
    if (P.outMultimapperOrder != "Old_2.4") return bad("EXITING because of fatal PARAMETERS error: --outMultimapperOrder " + P.outMultimapperOrder + " is not supported by star-b200 (only Old_2.4)\n");
    {   // ParametersClip_initialize.cpp:6-99: one value per mate; a single default value is repeated
        if (P.clipAdapterType[0] != "Hamming")
            return bad(P.clipAdapterType[0] == "CellRanger4" ? "EXITING because of fatal PARAMETER error: --clipAdapterType CellRanger4 is outside the scope of star-b200\n"
                       : "EXITING because of fatal PARAMETER error: --clipAdapterType = " + P.clipAdapterType[0] + " is not a valid option\nSOLUTION: use valid --clipAdapterType options: Hamming OR CellRanger4\n");
        auto spread = [&](std::vector<std::string>& v, const char* dflt) { if (v[0] == dflt && v.size() == 1) v.assign(P.readNmates, dflt); };
        spread(P.clip5pNbases, "0"); spread(P.clip3pNbases, "0"); spread(P.clip3pAfterAdapterNbases, "0");
        if (P.clip3pAdapterSeq[0] == "-" && P.clip3pAdapterSeq.size() == 1) { P.clip3pAdapterSeq.assign(P.readNmates, "-"); P.clip3pAdapterMMp.assign(P.readNmates, "0"); }
        const std::pair<const std::vector<std::string>*, const char*> chk[] = {{&P.clip5pNbases, "--clip5pNbases"}, {&P.clip3pNbases, "--clip3pNbases"}, {&P.clip3pAdapterSeq, "--clip3pAdapterSeq"},
                                                                               {&P.clip3pAdapterMMp, "--clip3pAdapterMMp"}, {&P.clip3pAfterAdapterNbases, "--clip3pAfterAdapterNbases"}};
        for (auto& c : chk)
            if (c.first->size() != P.readNmates)
                return bad(std::string("EXITING because of fatal PARAMETER error: ") + c.second + " has to contain " + std::to_string(P.readNmates) + " values to match the number of mates.\n");
        for (unsigned m = 0; m < P.readNmates; m++) {
            unsigned long long v5 = 0, v3 = 0, va = 0;
            double mm = 0;
            if (!parseNum(P.clip5pNbases[m], v5) || !parseNum(P.clip3pNbases[m], v3) || !parseNum(P.clip3pAfterAdapterNbases[m], va) || !parseNum(P.clip3pAdapterMMp[m], mm))
                return bad("EXITING: FATAL INPUT ERROR: could not parse the value of a --clip* parameter\n");
            P.clip5N[m] = (uint32_t)v5; P.clip3N[m] = (uint32_t)v3; P.clip3After[m] = (uint32_t)va; P.clip3MMp[m] = mm;
            P.clip3Ad[m].clear();
            if (P.clip3pAdapterSeq[m] == "polyA") P.clip3Ad[m].assign(STAR_READ_SEQ_LENGTH_MAX, (char)0);   // ClipMate_initialize.cpp:13-15
            else if (P.clip3pAdapterSeq[m] != "-")
                for (char ch : P.clip3pAdapterSeq[m]) { char v; switch (ch) { case 'A': case 'a': v = 0; break; case 'C': case 'c': v = 1; break; case 'G': case 'g': v = 2; break; case 'T': case 't': v = 3; break; default: v = 4; } P.clip3Ad[m].push_back(v); }
            if (v5 || v3 || va || !P.clip3Ad[m].empty()) P.clipYes = true;
        }
    }
    // Parameters.cpp:944-955
    if (P.outSAMstrandField == "None") h.outSAMstrandFieldType = 0;
    else if (P.outSAMstrandField == "intronMotif") h.outSAMstrandFieldType = 1;
    else return bad("EXITING because of fatal INPUT error: unrecognized option in outSAMstrandField=" + P.outSAMstrandField + "\nSOLUTION: use one of the allowed values of --outSAMstrandField : None or intronMotif \n");
    // Parameters.cpp:966-989
    memset(h.alignEndsTypeExt, 0, sizeof(h.alignEndsTypeExt));
    if (P.alignEndsType == "EndToEnd") { h.alignEndsTypeExt[0][0] = h.alignEndsTypeExt[0][1] = h.alignEndsTypeExt[1][0] = h.alignEndsTypeExt[1][1] = 1; }
    else if (P.alignEndsType == "Extend5pOfRead1") { h.alignEndsTypeExt[0][0] = 1; }
    else if (P.alignEndsType == "Extend5pOfReads12") { h.alignEndsTypeExt[0][0] = 1; h.alignEndsTypeExt[1][0] = 1; }
    else if (P.alignEndsType == "Extend3pOfRead1") { h.alignEndsTypeExt[0][1] = 1; }
    else if (P.alignEndsType == "Local") {}
    else return bad("EXITING because of FATAL INPUT ERROR: unknown/unimplemented value for --alignEndsType: " + P.alignEndsType + "\nSOLUTION: re-run STAR with --alignEndsType Local OR EndToEnd OR Extend5pOfRead1 OR Extend3pOfRead1\n");
    // Parameters.cpp:1047-1060
    for (auto& s : P.readNameSeparator) {
        if (s == "space") P.readNameSeparatorChar.push_back(' ');
        else if (s == "none") {}
        else if (s.size() == 1) P.readNameSeparatorChar.push_back(s[0]);
        else return bad("EXITING because of fatal PARAMETERS error: unrecognized value of --readNameSeparator=" + s + "\nSOLUTION: use allowed values: space OR single characters");
    }
    // Parameters.cpp:1062-1082
    if (P.outSAMunmapped[0] == "None" && P.outSAMunmapped.size() == 1) {}
    else if (P.outSAMunmapped[0] == "Within" && P.outSAMunmapped.size() == 1) { P.unmappedWithin = true; }
    else if (P.outSAMunmapped[0] == "Within" && P.outSAMunmapped.size() > 1 && P.outSAMunmapped[1] == "KeepPairs") {
        P.unmappedWithin = true;
        if (P.readNmates == 2) P.unmappedKeepPairs = true;
    } else return bad("EXITING because of fatal PARAMETERS error: unrecognized option for --outSAMunmapped\nSOLUTION: use allowed options: None OR Within OR Within KeepPairs");
    // Parameters.cpp:1084-1097
    {
        int nb = 0;
        if (!parseNum(P.alignEndsProtrude[0], nb)) return bad("EXITING because of fatal PARAMETERS error: bad --alignEndsProtrude\n");
        h.alignEndsProtrudeNbasesMax = nb;
        h.alignEndsProtrudeConcordantPair = 0;
        if (nb > 0) {
            if (P.alignEndsProtrude.size() > 1 && P.alignEndsProtrude[1] == "ConcordantPair") h.alignEndsProtrudeConcordantPair = 1;
            else if (P.alignEndsProtrude.size() > 1 && P.alignEndsProtrude[1] == "DiscordantPair") h.alignEndsProtrudeConcordantPair = 0;
            else return bad("EXITING because of fatal PARAMETERS error: unrecognized option in of --alignEndsProtrude\nSOLUTION: use allowed options: ConcordantPair or DiscordantPair");
        }
    }
    if (P.alignInsertionFlush == "None") h.alignInsertionFlushRight = 0;
    else if (P.alignInsertionFlush == "Right") h.alignInsertionFlushRight = 1;
    else return bad("EXITING because of fatal PARAMETERS error: unrecognized option in of --alignInsertionFlush=" + P.alignInsertionFlush + "\nSOLUTION: use allowed options: None or Right");
    if (P.alignSoftClipAtReferenceEnds == "Yes") h.alignSoftClipAtReferenceEnds = 1;
    else if (P.alignSoftClipAtReferenceEnds == "No") h.alignSoftClipAtReferenceEnds = 0;
    else return bad("EXITING because of fatal PARAMETERS error: unrecognized option in --alignSoftClipAtReferenceEnds   " + P.alignSoftClipAtReferenceEnds + "\nSOLUTION: use allowed options: Yes or No");
    if (P.outFilterIntronMotifs == "None") h.outFilterIntronMotifs = 0;
    else if (P.outFilterIntronMotifs == "RemoveNoncanonical") h.outFilterIntronMotifs = 1;
    else if (P.outFilterIntronMotifs == "RemoveNoncanonicalUnannotated") h.outFilterIntronMotifs = 2;
    else return bad("EXITING because of FATAL INPUT error: unrecognized value of --outFilterIntronMotifs=" + P.outFilterIntronMotifs + "\nSOLUTION: re-run STAR with --outFilterIntronMotifs = None -OR- RemoveNoncanonical -OR- RemoveNoncanonicalUnannotated\n");
    h.outFilterIntronStrandsRemoveInconsistent = P.outFilterIntronStrands == "RemoveInconsistentStrands";
    h.outSAMprimaryFlagAllBestScore = P.outSAMprimaryFlag == "AllBestScore";
    if (P.outSAMprimaryFlag != "AllBestScore" && P.outSAMprimaryFlag != "OneBestScore")
        return bad("EXITING because of FATAL INPUT error: unknown value for the option --outSAMprimaryFlag=" + P.outSAMprimaryFlag + "\nSOLUTION: re-run STAR with --outSAMprimaryFlag OneBestScore -OR- AllBestScore\n");
    // output type
    if (P.outSAMtype[0] == "None" || P.outSAMmode == "None") {}
    else if (P.outSAMtype[0] == "BAM") {   // Parameters.cpp:613-660
        if (P.outSAMtype.size() < 2)
            return bad("EXITING because of fatal PARAMETER error: missing BAM option\nSOLUTION: re-run STAR with one of the allowed values of --outSAMtype BAM Unsorted OR SortedByCoordinate OR both\n");
        for (size_t ii = 1; ii < P.outSAMtype.size(); ii++) {
            if (P.outSAMtype[ii] == "Unsorted") P.outBAMunsorted = true;
            else if (P.outSAMtype[ii] == "SortedByCoordinate") P.outBAMcoord = true;
            else
                return bad("EXITING because of fatal input ERROR: unknown value for the word " + std::to_string(ii + 1) + " of outSAMtype: " + P.outSAMtype[ii] + "\nSOLUTION: re-run STAR with one of the allowed values of --outSAMtype BAM Unsorted or SortedByCoordinate or both\n");
        }
    } else if (P.outSAMtype[0] != "SAM")
        return bad("EXITING because of fatal input ERROR: unknown value for the first word of outSAMtype: " + P.outSAMtype[0] + "\nSOLUTION: re-run STAR with one of the allowed values of outSAMtype: BAM or SAM \n");
    if (!P.outBAMcoord && P.wigYes)   // Parameters.cpp:685-690
        return bad("EXITING because of fatal PARAMETER error: generating signal with --outWigType requires sorted BAM\nSOLUTION: re-run STAR with with --outSAMtype BAM SortedByCoordinate, or, id you also need unsroted BAM, with --outSAMtype BAM SortedByCoordinate Unsorted\n");
    if (P.wigYes && P.outStd == "BAM_SortedByCoordinate")   // (the reference would read the signal back from "-", i.e. standard input)
        return bad("EXITING because of fatal PARAMETER error: --outWigType cannot be combined with --outStd BAM_SortedByCoordinate: the signal is made from the sorted BAM file\nSOLUTION: re-run STAR with --outStd Log, or make the signal from the BAM with --runMode inputAlignmentsFromBAM\n");
    if (P.outSAMmode != "Full" && P.outSAMmode != "NoQS" && P.outSAMmode != "None")
        return bad("EXITING because of FATAL input ERROR: unknown value for the option --outSAMmode=" + P.outSAMmode + "\nSOLUTION: use one of the allowed values: None or Full or NoQS\n");
    if (P.outSAMorder != "Paired" && P.outSAMorder != "PairedKeepInputOrder")   // (records are always written in input order, which both values allow)
        return bad("EXITING because of fatal input ERROR: --outSAMorder " + P.outSAMorder + ": star-b200 always writes records in input order (the reference's --runThreadN 1 order)\n");
    if (P.quantMode[0] != "-")   // Parameters.cpp:898-935
        for (const std::string& m : P.quantMode) {
            if (m == "GeneCounts") P.quantGeneCounts = true;
            else if (m == "TranscriptomeSAM") P.quantTrSAM = true;
            else return bad("EXITING because of fatal INPUT error: unrecognized option in --quantMode=" + m + "\nSOLUTION: use one of the allowed values of --quantMode : TranscriptomeSAM or GeneCounts or - .\n");
        }
    if (P.quantTrSAM) {   // Parameters.cpp:905-927
        if (P.quantTranscriptomeSAMoutput == "BanSingleEnd_BanIndels_ExtendSoftclip") { P.quantTrIndel = false; P.quantTrSoftClip = false; P.quantTrSingleEnd = false; }
        else if (P.quantTranscriptomeSAMoutput == "BanSingleEnd") { P.quantTrIndel = true; P.quantTrSoftClip = true; P.quantTrSingleEnd = false; }
        else if (P.quantTranscriptomeSAMoutput == "BanSingleEnd_ExtendSoftclip") { P.quantTrIndel = true; P.quantTrSoftClip = false; P.quantTrSingleEnd = false; }
        else return bad("EXITING because of fatal INPUT error: unrecognized option in --quantTranscriptomeSAMoutput=" + P.quantTranscriptomeSAMoutput + "\nSOLUTION: use one of the allowed values: BanSingleEnd_BanIndels_ExtendSoftclip OR BanSingleEnd OR BanSingleEnd_ExtendSoftclip\n");
        if (P.quantTranscriptomeBAMcompression < -1) P.quantTrSAM = false;   // -2: no BAM output (Parameters.cpp:906-908)
    }
    if (P.outSAMtlen != 1 && P.outSAMtlen != 2)   // Parameters.cpp (outSAMtlen)
        return bad("EXITING because of FATAL INPUT ERROR: --outSAMtlen can only be 1 or 2\nSOLUTION: re-run STAR with --outSAMtlen 1 OR 2\n");
    if (P.outReadsUnmapped != "None" && P.outReadsUnmapped != "Fastx")   // Parameters.cpp (outReadsUnmapped)
        return bad("EXITING because of FATAL INPUT ERROR: unknown value of --outReadsUnmapped: " + P.outReadsUnmapped + "\nSOLUTION: use allowed values: None OR Fastx\n");
    // SJ
    if (P.outSJtype[0] == "None") P.outSJyes = false;
    else if (P.outSJtype[0] == "Standard") P.outSJyes = true;
    else return bad("EXITING because of FATAL input ERROR: unrecognized option in --outSJtype   " + P.outSJtype[0] + "\nSOLUTION: use one of the allowed options: --outSJtype   Standard   OR   None\n");
    if (P.outFilterType == "BySJout" && !P.outSJyes)   // Parameters.cpp:1179-1183
        return bad("EXITING because of FATAL input ERROR: --outFilterType BySJout requires --outSJtype Standard\nSOLUTION: --outFilterType Normal    OR   --outFilterType BySJout --outSJtype Standard\n");
    if (P.outSJfilterReads != "All" && P.outSJfilterReads != "Unique")
        return bad("EXITING because of FATAL INPUT error: unknown value for the option --outSJfilterReads=" + P.outSJfilterReads + "\nSOLUTION: re-run STAR with --outSJfilterReads All -OR- Unique\n");
    for (auto* v : {&P.outSJfilterOverhangMin, &P.outSJfilterCountUniqueMin, &P.outSJfilterCountTotalMin, &P.outSJfilterDistToOtherSJmin}) {
        if (v->size() != 4) return bad("EXITING because of fatal PARAMETERS error: outSJfilter* parameters need 4 values\n");
        for (auto& x : *v) if (x < 0) x = std::numeric_limits<int32_t>::max();  // Parameters.cpp:722-728
    }
    // SAM attributes: Parameters_samAttributes.cpp:47-60
    {
        std::vector<std::string> a;
        if (P.outSAMattributes[0] == "None") {}
        else if (P.outSAMattributes[0] == "All") a = {"NH", "HI", "AS", "nM", "NM", "MD", "jM", "jI", "MC", "ch"};
        else if (P.outSAMattributes[0] == "Standard") a = {"NH", "HI", "AS", "nM"};
        else a = P.outSAMattributes;
        static const std::map<std::string, int> code = {{"NH", 1}, {"HI", 2}, {"AS", 3}, {"NM", 4}, {"MD", 5}, {"nM", 6}, {"jM", 7}, {"jI", 8}, {"XS", 9},
                                                        {"RG", 10}, {"ch", 14}, {"MC", 15}};
        for (auto& s : a) {
            auto it = code.find(s);
            if (it == code.end()) return bad("EXITING because of FATAL INPUT ERROR: unknown/unimplemented SAM atrribute (tag): " + s + "\nSOLUTION: star-b200 supports NH HI AS nM NM MD jM jI XS MC RG ch\n");
            if (s == "RG" && P.outSAMattrRGline[0] == "-") continue;
            P.outSAMattrOrder.push_back(it->second);
            if (s == "XS") h.outSAMstrandFieldType = 1;   // Parameters_samAttributes.cpp:172-179: XS implies --outSAMstrandField intronMotif
        }
        for (int c : P.outSAMattrOrder)   // Parameters_samAttributes.cpp:226, 252-260
            if (c == 14 && !P.outBAMunsorted && !P.outBAMcoord)
                return bad("EXITING because of fatal PARAMETER error: --outSAMattributes contains ch tag, which requires BAM output.\nSOLUTION: re-run STAR with --outSAMtype BAM Unsorted (and/or) SortedByCoordinate option, or without ch tag in --outSAMattributes\n");
        if (h.outSAMstrandFieldType == 1) {  // Parameters_samAttributes.cpp: XS added for intronMotif
            bool has = false;
            for (int c : P.outSAMattrOrder) if (c == 9) has = true;
            if (!has) P.outSAMattrOrder.push_back(9);
        }
    }
    if (P.outSAMattrRGline[0] != "-") {  // Parameters_readFilesInit.cpp:65-95: entries separated by the word ","
        for (size_t ii = 0; ii < P.outSAMattrRGline.size(); ii++) {
            if (ii == 0 || P.outSAMattrRGline[ii] == ",") {
                if (ii > 0) ++ii;   // skip the comma
                if (ii >= P.outSAMattrRGline.size()) break;
                P.outSAMattrRGlineSplit.push_back(P.outSAMattrRGline[ii]);
                if (P.outSAMattrRGlineSplit.back().substr(0, 3) != "ID:") return bad("EXITING because of FATAL INPUT ERROR: the first word of a line from --outSAMattrRGline=" + P.outSAMattrRGlineSplit.back() + " does not start with ID:xxx read group identifier\nSOLUTION: re-run STAR with all lines in --outSAMattrRGline starting with ID:xxx\n");
                P.outSAMattrRGs.push_back(P.outSAMattrRGlineSplit.back().substr(3));
            } else {
                P.outSAMattrRGlineSplit.back() += "\t" + P.outSAMattrRGline[ii];
            }
        }
        const size_t nFiles = P.readFilesNames.empty() ? 1 : P.readFilesNames[0].size();
        if (P.outSAMattrRGs.size() > 1 && P.outSAMattrRGs.size() != nFiles)
            return bad("EXITING: because of fatal INPUT ERROR: number of input read files: " + std::to_string(nFiles) + " does not agree with number of read group RG entries: " + std::to_string(P.outSAMattrRGs.size()) + "\nMake sure that the number of RG lines in --outSAMattrRGline is equal to either 1, or the number of input read files in --readFilesIn\n");
        while (P.outSAMattrRGs.size() < nFiles) P.outSAMattrRGs.push_back(P.outSAMattrRGs[0]);   // the same read group for all files
        P.outSAMattrRG = P.outSAMattrRGs[0];
        bool has = false;
        for (int c : P.outSAMattrOrder) if (c == 10) has = true;
        if (!has && !P.rgFromManifest) P.outSAMattrOrder.push_back(10);   // (Parameters_samAttributes.cpp:201-205: only --outSAMattrRGline adds the tag by itself)
    }
    // 2-pass and on-the-fly junction insertion: Parameters.cpp:779-825, 1000-1035 (the directories are made by the run driver)
    if (P.userSet.count("twopass1readsN") && P.twopassMode == "None")
        return bad("EXITING because of fatal PARAMETERS error: --twopass1readsN is defined, but --twoPassMode is not defined\nSOLUTION: to activate the 2-pass mode, use --twopassMode Basic");
    if (P.twopassMode != "None") {
        if (P.twopassMode != "Basic")
            return bad("EXITING because of fatal PARAMETERS error: unrecognized value of --twopassMode=" + P.twopassMode + "\nSOLUTION: for the 2-pass mode, use allowed values --twopassMode: Basic");
        if (P.twopass1readsN == 0)
            return bad("EXITING because of fatal PARAMETERS error: --twopass1readsN = 0 in the 2-pass mode\nSOLUTION: for the 2-pass mode, specify --twopass1readsN > 0. Use a very large number or -1 to map all reads in the 1st pass.\n");
        P.twoPassYes = true;
        P.twoPassDir = P.outFileNamePrefix + "_STARpass1/";
    }
    if (P.sjdbFileChrStartEnd[0] != "-" || P.sjdbGTFfile != "-") { P.sjdbInsertPass1 = true; P.sjdbInsertYes = true; }
    if (P.twoPassYes) { P.sjdbInsertPass2 = true; P.sjdbInsertYes = true; }
    if (P.sjdbInsertYes) {
        if (P.sjdbOverhang == 0 || (long long)P.sjdbOverhang < 0)
            return bad("EXITING because of fatal PARAMETERS error: pGe.sjdbOverhang <=0 while junctions are inserted on the fly with --sjdbFileChrStartEnd or/and --sjdbGTFfile\nSOLUTION: specify pGe.sjdbOverhang>0, ideally readmateLength-1");
        if (P.sjdbInsertSave != "Basic" && P.sjdbInsertSave != "All")
            return bad("EXITING because of fatal PARAMETERS error: unrecognized value of --sjdbInsertSave=" + P.sjdbInsertSave + "\nSOLUTION: use allowed values: Basic or All\n");
        P.sjdbInsertOutDir = P.outFileNamePrefix + "_STARgenome/";
        if (P.twoPassYes && P.gpuShardCount > 1 && P.gpuTwoPassPhase == 0)
            return bad("EXITING because of fatal input ERROR: --twopassMode Basic of a sharded (multi-GPU) run needs the junctions of all shards after the 1st pass: run it through `python -m star_b200.dist` (which gathers them between --gpuTwoPassPhase 1 and 2)\n");
    }
    if (P.gpuTwoPassPhase != 0 && !(P.twoPassYes && P.gpuShardCount > 1))
        return bad("EXITING because of fatal PARAMETERS error: --gpuTwoPassPhase is only meaningful for a sharded --twopassMode Basic run\n");
    if (P.gpuShardIndex >= P.gpuShardCount) return bad("EXITING because of fatal PARAMETERS error: --gpuShardIndex must be < --gpuShardCount\n");
    // geometry the sparse window map of the GPU engine relies on (DESIGN.md, "windows")
    if (2 * h.winFlankNbins > h.winAnchorDistNbins && P.userSet.count("winFlankNbins"))
        return bad("EXITING because of fatal PARAMETERS error: star-b200 requires 2*winFlankNbins <= winAnchorDistNbins (flanks of neighbouring windows must not overlap)\n");
    return 0;
}

}  // namespace starhost

extern "C" void star_params_default(star_params_t* p) { starhost::paramsDefault(p); }

extern "C" size_t star_abi_sizeof(int which) {
    switch (which) {
        case 0: return sizeof(star_params_t);
        case 1: return sizeof(star_index_view_t);
        case 2: return sizeof(star_read_batch_t);
        case 3: return sizeof(star_align_t);
        case 4: return sizeof(star_read_result_t);
        case 5: return sizeof(star_align_batch_t);
        case 6: return sizeof(star_chunk_stats_t);
        default: return 0;
    }
}
