// host.h — internal declarations of the host side (C++) that sits above the C-ABI engine.
//
// The host side mirrors the parts of STAR that stay on the CPU around the replaced hot path:
// parameter parsing (reference source/Parameters.cpp), index loading (Genome_genomeLoad.cpp),
// FASTQ chunking (ReadAlignChunk_processChunks.cpp), SAM / SJ.out.tab / Log.final.out emission
// (ReadAlign_outputAlignments.cpp, ReadAlign_outputTranscriptSAM.cpp, outputSJ.cpp, Stats.cpp)
// and the run driver (STAR.cpp).  It never computes an alignment.
#pragma once
#include <cstdint>
#include <cstdio>
#include <map>
#include <cstdlib>
#include <functional>
#include <string>
#include <vector>

#include "../../../include/star_b200.h"

namespace starhost {

struct HostParams {
    star_params_t hp;                       // what the engine reads
    // run / IO
    std::string commandLine, commandLineFull;
    std::string runMode = "alignReads";
    int runThreadN = 1;                     // host threads used for FASTQ parsing / SAM formatting
    // Threads each host stage of the mapping pass (chunk parsing, record formatting) uses.  The stages run concurrently next to the thread that
    // drives the GPU; what they may use is the CPU time the process is ALLOWED, which in a container is the cgroup quota, not the number
    // of logical CPUs it sees.  With many more threads per stage than the quota allows, the bursts of runnable threads exhaust the quota of a
    // scheduling period and the whole process, including the thread that feeds the GPU, is frozen until the next one.  Per stage: --runThreadN, at most 32, at most half
    // of the allowed CPUs (at least 2).  STAR_B200_HOST_STAGE_THREADS sets the number directly.
    static int allowedCpus();   // min(logical CPUs of the affinity mask, cgroup CPU quota); params.cpp
    int stageThreads() const {
        static const int fixed = [] { const char* e = getenv("STAR_B200_HOST_STAGE_THREADS"); const int v = e ? atoi(e) : 0; return v > 0 ? v : 0; }();
        static const int cap = [] { const int half = allowedCpus() / 2; return half < 2 ? 2 : (half > 32 ? 32 : half); }();
        const int t = runThreadN < 1 ? 1 : runThreadN;
        if (fixed) return t < fixed ? t : fixed;
        return t < cap ? t : cap;
    }
    std::string genomeDir = "./GenomeDir/";
    std::string genomeLoad = "NoSharedMemory";
    std::vector<std::string> readFilesIn = {"Read1", "Read2"};
    std::vector<std::vector<std::string>> readFilesNames;   // [mate][file]: --readFilesIn a1,a2 b1,b2 (Parameters_readFilesInit.cpp:43-62)
    // read clipping before mapping (ParametersClip_initialize.cpp, ClipMate_clip.cpp): fixed numbers of bases at either end, a 3' adapter
    // found by ungapped search with a mismatch ratio, bases after the adapter; per mate
    std::vector<std::string> clip5pNbases = {"0"}, clip3pNbases = {"0"}, clip3pAdapterSeq = {"-"}, clip3pAdapterMMp = {"0.1"}, clip3pAfterAdapterNbases = {"0"},
                             clip5pAdapterSeq = {"-"}, clipAdapterType = {"Hamming"};
    bool clipYes = false;
    uint32_t clip5N[2] = {0, 0}, clip3N[2] = {0, 0}, clip3After[2] = {0, 0};
    std::string clip3Ad[2];                  // adapter as codes 0..4
    double clip3MMp[2] = {0.1, 0.1};
    std::string readFilesPrefix = "-", readFilesManifest = "-";
    bool rgFromManifest = false;             // read groups came from --readFilesManifest: @RG header lines, RG tag only on request
    std::vector<std::string> ignoredParams;  // accepted reference parameters without effect here (resource limits, temporary directories)
    std::vector<std::string> readFilesCommand = {"-"};
    long long readMapNumber = -1;
    std::vector<std::string> readNameSeparator = {"/"};
    std::vector<char> readNameSeparatorChar;
    std::string outFileNamePrefix = "./";
    std::string outStd = "Log";
    std::vector<std::string> outSAMtype = {"SAM"};
    bool outBAMunsorted = false;            // --outSAMtype BAM Unsorted  -> Aligned.out.bam (SURVEY.md §8f N1)
    bool outBAMcoord = false;               // --outSAMtype BAM SortedByCoordinate -> Aligned.sortedByCoord.out.bam (sorted in host memory)
    int outBAMcompression = 1;              // --outBAMcompression (zlib level of the BGZF blocks; -1 = zlib default)
    std::string outSAMmode = "Full";
    std::string outSAMstrandField = "None";
    std::vector<std::string> outSAMattributes = {"Standard"};
    std::vector<int> outSAMattrOrder;       // ATTR_* codes
    unsigned outSAMattrIHstart = 1;
    std::vector<std::string> quantMode = {"-"};   // GeneCounts only (ReadsPerGene.out.tab); TranscriptomeSAM is out of scope
    bool quantGeneCounts = false, quantTrSAM = false;
    int32_t quantTranscriptomeBAMcompression = 1;
    uint64_t runRNGseed = 777;               // seeds the primary-flag draw of Aligned.toTranscriptome.out.bam (ReadAlign.cpp:11)
    std::string quantTranscriptomeSAMoutput = "BanSingleEnd_BanIndels_ExtendSoftclip";
    bool quantTrIndel = false, quantTrSoftClip = false, quantTrSingleEnd = false;   // what Aligned.toTranscriptome.out.bam may contain
    std::vector<std::string> outSAMheaderHD = {"-"}, outSAMheaderPG = {"-"};
    std::string outSAMheaderCommentFile = "-";
    int32_t outSAMtlen = 1;                 // 2: leftmost base of any mate to rightmost base of any mate, + for the leftmost mate (BAM records; ReadAlign_alignBAM.cpp:84-88)
    int32_t outQSconversionAdd = 0;         // added to every quality value, clamped to 33..126 (readLoad.cpp:71-81)
    std::string outReadsUnmapped = "None";  // Fastx: Unmapped.out.mate1/2 (ReadAlign::outReadsUnmapped)
    std::vector<std::string> outSAMunmapped = {"None"};
    bool unmappedWithin = false, unmappedKeepPairs = false;
    std::string outSAMorder = "Paired";
    std::string outSAMprimaryFlag = "OneBestScore";
    std::string outSAMreadID = "Standard";
    int outSAMmapqUnique = 255;
    unsigned outSAMflagOR = 0, outSAMflagAND = 65535;
    std::vector<std::string> outSAMattrRGline = {"-"};
    std::string outSAMattrRG;               // ID of the first read group (if any)
    std::vector<std::string> outSAMattrRGs;        // read group ID per input file (Parameters_readFilesInit.cpp:65-95)
    std::vector<std::string> outSAMattrRGlineSplit; // one @RG header line per read group (tab-joined fields)
    std::string outFilterType = "Normal";
    std::string outFilterIntronMotifs = "None";
    std::string outFilterIntronStrands = "RemoveInconsistentStrands";
    std::vector<std::string> outSJtype = {"Standard"};
    bool outSJyes = true;
    std::string outSJfilterReads = "All";
    std::vector<int32_t> outSJfilterOverhangMin = {30, 12, 12, 12};
    std::vector<int32_t> outSJfilterCountUniqueMin = {3, 1, 1, 1};
    std::vector<int32_t> outSJfilterCountTotalMin = {3, 1, 1, 1};
    std::vector<int32_t> outSJfilterDistToOtherSJmin = {10, 0, 5, 10};
    std::vector<int32_t> outSJfilterIntronMaxVsReadN = {50000, 100000, 200000};
    std::string alignEndsType = "Local";
    std::vector<std::string> alignEndsProtrude = {"0", "ConcordantPair"};
    std::string alignSoftClipAtReferenceEnds = "Yes";
    std::string alignInsertionFlush = "None";
    std::string outMultimapperOrder = "Old_2.4";
    unsigned readNmates = 1;
    // --runMode genomeGenerate (Parameters.cpp:230-256)
    std::vector<std::string> genomeFastaFiles = {"-"};   // with --runMode alignReads: references added to the loaded index (addref.cpp)
    std::vector<std::string> outSAMfilter = {"None"};    // KeepOnlyAddedReferences / KeepAllAddedReferences (ReadAlign_outputAlignments.cpp:140-164)
    bool outSAMfilterKeepOnly = false, outSAMfilterKeepAll = false;
    uint64_t genomeSAindexNbases = 14, genomeChrBinNbits = 18, genomeSAsparseD = 1, limitGenomeGenerateRAM = 31000000000ULL;
    // on-the-fly junction insertion / 2-pass (Parameters.cpp:240-269, 779-825, 1000-1035)
    std::vector<std::string> sjdbFileChrStartEnd = {"-"};
    std::string sjdbGTFfile = "-", sjdbGTFchrPrefix = "-", sjdbGTFfeatureExon = "exon", sjdbGTFtagExonParentTranscript = "transcript_id",
                sjdbGTFtagExonParentGene = "gene_id";
    std::vector<std::string> sjdbGTFtagExonParentGeneName = {"gene_name"}, sjdbGTFtagExonParentGeneType = {"gene_type", "gene_biotype"};
    uint64_t sjdbOverhang = 100;
    std::string sjdbInsertSave = "Basic";
    uint64_t limitSjdbInsertNsj = 1000000;
    std::string twopassMode = "None";
    uint64_t twopass1readsN = ~0ULL;
    bool twoPassYes = false, sjdbInsertPass1 = false, sjdbInsertPass2 = false, sjdbInsertYes = false;
    std::string twoPassDir, sjdbInsertOutDir;
    // signal tracks (Parameters.cpp:511-562, 585-607, 685-690): --outWigType bedGraph|wiggle [read1_5p|read2], after the coordinate sort of
    // a mapping run or from --inputBAMfile with --runMode inputAlignmentsFromBAM
    std::vector<std::string> outWigType = {"None"}, outWigStrand = {"Stranded"}, outWigNorm = {"RPM"};
    std::string outWigReferencesPrefix = "-", inputBAMfile = "-";
    bool wigYes = false, wigStranded = true;
    int wigFormat = 0, wigType = 0, wigNorm = 1;   // format 0 bedGraph / 1 wiggle; type 0 all M bases / 1 read1_5p / 2 read2; norm 0 None / 1 RPM
    // duplicate marking (Parameters.cpp:566-580; --runMode inputAlignmentsFromBAM only): -> <prefix>Processed.out.bam
    std::string bamRemoveDuplicatesType = "-";
    uint64_t bamRemoveDuplicatesMate2basesN = 0;
    bool dedupYes = false, dedupMarkMulti = false;
    // star-b200 extensions (not in the reference)
    int gpuDevice = 0;
    unsigned gpuChunkReads = 65536;         // reads (pairs) per engine call (3 chunks are in flight); larger contexts do not fit an 80 GB H100 beside a GRCh38-sized index
    unsigned gpuBySJoutPhase = 0;           // sharded --outFilterType BySJout (star_b200.dist): 1 = 1st stage of this shard, 2 = 2nd stage with the gathered junctions
    unsigned gpuTwoPassPhase = 0;           // sharded --twopassMode Basic (star_b200.dist): 1 = 1st pass of this shard only, 2 = insertion of the gathered junctions + 2nd pass
    unsigned gpuShardIndex = 0, gpuShardCount = 1;   // multi-GPU: this process maps reads [n*i/N, n*(i+1)/N) (contiguous slices keep input order)
    std::map<std::string, int> userSet;     // parameter name -> input level (for --sjdbOverhang style checks)
};

// Parses argv exactly like Parameters::inputParameters (Parameters.cpp:310-470) for the supported subset.
// Returns 0 or a STAR_EXIT_* code with the message in err.
int parseCommandLine(int argc, char** argv, HostParams& P, std::string& err);
void paramsDefault(star_params_t* p);
// derived values that need the other parameters (Parameters.cpp:944-1124)
int finalizeParams(HostParams& P, std::string& err);

struct LoadedIndex {
    std::vector<uint8_t> Gstore, SAstore, SAistore;
    std::vector<uint64_t> genomeSAindexStart, chrStart, chrLength, sjdbStart, sjdbEnd, sjDstart, sjAstart;
    std::vector<uint8_t> sjdbMotif, sjdbShiftLeft, sjdbShiftRight, sjdbStrand;
    std::vector<std::string> chrName;
    std::vector<uint64_t> chrBin;
    star_index_view_t view;
    std::string versionGenome;
    uint64_t sjdbOverhangGenome = 0;      // sjdbOverhang of genomeParameters.txt
    bool sjdbInfoExists = false;
    std::string sjdbInsertSaveGenome;     // sjdbInsertSave of genomeParameters.txt ("" = index older than on-the-fly insertion)
    std::string genomeDir;
    uint32_t insertChrFirst = ~0u;        // first chromosome added at the mapping stage (genomeInsertChrIndFirst; ~0: none added)
    void pointView();                     // re-points view.* at the vectors (after they were replaced)
};

// ---- on-the-fly junction insertion (sjdb_insert.cpp) ---------------------------------------------------------------------------
struct SjdbLoci {   // sjdbClass.h
    std::vector<std::string> chr;
    std::vector<uint64_t> start, end;
    std::vector<char> str;
    std::vector<uint8_t> priority;
};
void sjdbLoadFromStream(std::istream& in, SjdbLoci& loci);   // sjdbLoadFromStream.cpp:2-28
// sjdbInsertJunctions.cpp:11-102: loads the junction lists, prepares the inserts, rebuilds G / SA / SAi of `idx` in place (the device part
// through eng->sjdb_*), writes sjdbInfo.txt / sjdbList.out.tab (and the whole index with --sjdbInsertSave All) to P.sjdbInsertOutDir and
// re-computes hp->winBinN.  pass2: the junctions of `pass1sjFile` are added.  Returns 0 or a STAR_EXIT_* code with the message in err.
// --runMode genomeGenerate (genome_generate.cpp): FASTA -> Genome, SA (eng->sa_build), SAindex, junction inserts, index files in P.genomeDir
int genomeGenerate(HostParams& P, const star_engine_vtbl_t* eng, std::ostream& logMain, std::string& err);
int sjdbInsertJunctions(const HostParams& P, star_params_t* hp, LoadedIndex& idx, SjdbLoci& loci, bool pass2, const std::string& pass1sjFile,
                        const star_engine_vtbl_t* eng, std::ostream& logMain, std::string& err, bool generateMode = false);
int loadIndex(const std::string& genomeDir, star_params_t* p, LoadedIndex& L, std::string& err, std::string* log, bool chrInfoOnly = false);
// the index-dependent window geometry (Genome_genomeLoad.cpp:382-410): winBinNbits, winFlankNbins, winAnchorDistNbins, winBinChrNbits, winBinN
void windowGeometry(star_params_t* p, uint64_t nGenome, uint32_t gChrBinNbits, std::ostream* logMain = nullptr);
// genomeScanFastaFiles.cpp:5-91 (genome_generate.cpp): appends the chromosomes of `files` behind the ones in the (closed) lists, codes into
// G[pad + position] when G is given.  Returns 0 or STAR_EXIT_INPUT_FILES with the message in err.
int scanFastaFiles(const std::vector<std::string>& files, uint64_t binN, std::vector<std::string>& chrName, std::vector<uint64_t>& chrStart,
                   std::vector<uint64_t>& chrLength, std::vector<uint8_t>* G, size_t pad, std::ostream& logMain, std::string& err);
// genomeSAindex.cpp:6-220 over a whole suffix array (genome_generate.cpp)
int buildSAindex(const uint8_t* G, uint64_t nGenome, const uint8_t* SA, uint64_t nSA, uint32_t GstrandBit, uint32_t Lmax, int runThreadN,
                 std::vector<uint64_t>& genomeSAindexStart, std::vector<uint8_t>& SAistore, uint64_t& nSAi, uint64_t& nSAibyte, std::string& err);
// --genomeFastaFiles at the mapping stage (addref.cpp; Genome_insertSequences.cpp, insertSeqSA.cpp): adds the sequences to the loaded index
// before any junction insertion (device part through eng->addref_*), then re-runs windowGeometry.  chrInfoOnly: an index loaded with
// loadIndex(..., chrInfoOnly) gets the added chromosomes' names, starts and lengths only.  Returns 0 or a STAR_EXIT_* code with the message in err.
int addReferences(const HostParams& P, star_params_t* hp, LoadedIndex& idx, const star_engine_vtbl_t* eng, std::ostream& logMain, std::string& err,
                  bool chrInfoOnly = false);

// ---- signal tracks (signal.cpp; signalFromBAM.cpp:5-209): <prefix>Signal.{Unique,UniqueMultiple}.str{1,2}.out.{bg,wig} ----------------
// recs: the BAM records in file order, each pointing at its block_size field; names / lens: the references of the header.
int signalFromRecords(const HostParams& P, const star_engine_vtbl_t* eng, const std::vector<std::string>& names, const std::vector<uint32_t>& lens,
                      const std::vector<const uint8_t*>& recs, std::ostream& logMain, std::string& err);
// --runMode inputAlignmentsFromBAM: reads --inputBAMfile (BGZF, inflated on the host stage threads)
int signalFromBAMfile(const HostParams& P, const star_engine_vtbl_t* eng, std::ostream& logMain, std::string& err);
// reads --inputBAMfile into u (inflated on the host stage threads): the header's references, recs = the records in file order (each at its
// block_size field, inside u), headerEnd = the size of the header in u.  Returns 0 or STAR_EXIT_INPUT_FILES with the message in err.
int readBAMfile(const HostParams& P, std::string& u, std::vector<std::string>& names, std::vector<uint32_t>& lens, std::vector<const uint8_t*>& recs,
                size_t& headerEnd, std::string& err);
// htslib bam_aux_get + bam_aux2i of the NH tag (has = false when there is none); false: malformed optional fields
bool auxNH(const uint8_t* rec, bool& has, uint32_t& nh);
void parallelFor(int n, int nT, const std::function<void(int)>& fn);
// ---- duplicate marking (dedup.cpp; bamRemoveDuplicates.cpp:114-271): --inputBAMfile -> <prefix>Processed.out.bam
int dedupFromBAMfile(const HostParams& P, const star_engine_vtbl_t* eng, std::ostream& logMain, std::string& err);

// one chunk of reads in host memory
struct ReadChunk {
    uint32_t nReads = 0, nMates = 1;
    std::string seq, qual;                   // all mates back to back
    std::vector<uint64_t> seqOff;            // nReads*nMates+1 (same offsets index qual)
    std::string names;                       // read names (without '@', cut at the separator), '\0'-separated
    std::vector<uint32_t> nameOff;           // nReads+1
    std::string namesFull;                   // only with --outReadsUnmapped Fastx: the read IDs as in the file ('@'/'>' included, not cut), '\0'-separated
    std::vector<uint32_t> nameFullOff;       // nReads: start of read i's ID in namesFull
    std::vector<char> readFilter;            // 'Y'/'N'
    std::vector<uint64_t> iReadAll;
    // clipping: seq / qual / seqOff hold the reads as they are in the file (what the output prints); clip5 / clip3 = bases cut at the ends of
    // every mate (empty vectors: no clipping in this run); seqC / seqOffC = the clipped sequences handed to the engine (a mate clipped
    // to nothing stays empty in a pair and is passed as one N for single-end reads)
    std::vector<uint16_t> clip5, clip3;
    std::string seqC;
    std::vector<uint64_t> seqOffC;
    bool clipped() const { return !clip5.empty(); }
    uint64_t lenOrig(uint64_t i, uint32_t m) const { return seqOff[i * nMates + m + 1] - seqOff[i * nMates + m]; }
    uint64_t lenTrue(uint64_t i, uint32_t m) const { return clipped() ? lenOrig(i, m) - clip5[i * nMates + m] - clip3[i * nMates + m] : lenOrig(i, m); }   // readLength of the reference
    uint64_t len(uint64_t i, uint32_t m) const { const uint64_t l = lenTrue(i, m); return l || nMates == 2 ? l : 1; }                              // what the engine mapped
    uint64_t c5(uint64_t i, uint32_t m) const { return clipped() ? clip5[i * nMates + m] : 0; }
    uint64_t c3(uint64_t i, uint32_t m) const { return clipped() ? lenOrig(i, m) - c5(i, m) - len(i, m) : 0; }
    char base(uint64_t i, uint32_t m, uint64_t k) const { return clipped() && lenTrue(i, m) == 0 ? 'N' : seq[seqOff[i * nMates + m] + c5(i, m) + k]; }   // base k of the clipped mate
    bool fastq = true;
    uint32_t fileIndex = 0;                  // input file (of a comma-separated list) this chunk came from: a chunk never spans files
    void clear() {
        nReads = 0; seq.clear(); qual.clear(); seqOff.clear(); names.clear(); nameOff.clear(); readFilter.clear(); iReadAll.clear();
        namesFull.clear(); nameFullOff.clear(); clip5.clear(); clip3.clear(); seqC.clear(); seqOffC.clear();
    }
};

class ReadsReader {
   public:
    ~ReadsReader();
    int open(const HostParams& P, std::string& err);
    // fills at most maxReads reads; returns number read (0 at EOF) or -STAR_EXIT_* on error
    long long next(ReadChunk& c, uint32_t maxReads, std::string& err);
    uint64_t iReadAll = 0;
    uint64_t shardLo = 0, shardHi = ~0ULL;   // reads (0-based) this process maps
    uint32_t fileIdx = 0;                    // current file of the --readFilesIn lists

   private:
    FILE* f[2] = {nullptr, nullptr};
    bool piped[2] = {false, false};
    unsigned nMates = 1;
    const HostParams* P = nullptr;
    std::vector<char> buf[2];
    size_t bpos[2] = {0, 0}, blen[2] = {0, 0};
    int openFile(uint32_t idx, std::string& err);   // opens file `idx` of every mate (mapped or stream); closes the previous one
    void closeFiles();
    bool getLine(int m, std::string& line);
    int peekChar(int m);
    // fast path: plain (not piped) 4-line FASTQ files are memory-mapped; a chunk is line-indexed per mate and parsed by runThreadN threads
    bool fast = false;
    const char* map[2] = {nullptr, nullptr};
    size_t mapSize[2] = {0, 0}, mapOff[2] = {0, 0};
    long long nextFast(ReadChunk& c, uint32_t maxReads, std::string& err);
    long long nextStream(ReadChunk& c, uint32_t maxReads, std::string& err);   // line-by-line parser (piped input, FASTA)
    std::vector<ReadChunk> parts_;                       // per-thread pieces, kept between chunks (their buffers stay mapped)
    std::vector<const char*> lineSt_[2], lineEn_[2];     // line index of the current chunk
    std::vector<std::vector<const char*>> idxFound_[2];  // newlines found by each indexing thread
    double lineBytes_[2] = {64.0, 64.0};                  // mean line length seen so far (sizes the range the next index scans)
    // parses one FASTQ record given its four lines of each mate (pointers into the mapped files); appends to `c`; returns 0 or -STAR_EXIT_*
    int parseRecord(ReadChunk& c, uint64_t iRead, const char* const* ls, const char* const* le, std::string& err) const;
};

// Stats.h:11-24
struct Stats {
    uint64_t readN = 0, readBases = 0, mappedReadsU = 0, mappedReadsM = 0, mappedBases = 0, mappedMismatchesN = 0, mappedInsN = 0,
             mappedDelN = 0, mappedInsL = 0, mappedDelL = 0;
    uint64_t splicesN[STAR_SJ_MOTIF_SIZE] = {0, 0, 0, 0, 0, 0, 0};
    uint64_t splicesNsjdb = 0;
    uint64_t unmappedOther = 0, unmappedShort = 0, unmappedMismatch = 0, unmappedMulti = 0, unmappedAll = 0, chimericAll = 0;
    time_t timeStart = 0, timeStartMap = 0, timeFinish = 0;
    void add(const Stats& s);
    // the 24 counters as a flat array (for the multi-GPU allreduce, SURVEY.md §8e)
    static const int N_COUNTERS = 24;
    void toArray(uint64_t* a) const;
    void fromArray(const uint64_t* a);
};

// OutSJ.h:9-25 junction record (27 bytes in the reference; plain struct here)
struct Junction {
    uint64_t start;
    uint32_t gap;
    char strand, motif, annot;
    uint32_t countUnique, countMultiple;
    uint16_t overhangLeft, overhangRight;
};

// --quantMode GeneCounts: exons by locus with their genes (exonGeTrInfo.tab, geneInfo.tab; Transcriptome.cpp:18-98) and the counters of
// Quantifications.h (3 strandedness types: unstranded, read strand = gene strand, reverse)
struct GeneModel {
    std::vector<uint64_t> s, e, eMax;
    std::vector<uint8_t> str;
    std::vector<uint32_t> g;
    std::vector<std::string> geID;
    int load(const std::string& dir, std::string& err);
};
struct GeneCounts {
    uint64_t cMulti = 0, cNone[3] = {0, 0, 0}, cAmbig[3] = {0, 0, 0};
    std::vector<uint64_t> gCount[3];
    void init(size_t nGe) { for (auto& v : gCount) v.assign(nGe, 0); }
    void add(const GeneCounts& o);
    void addAlign(const GeneModel& gm, uint64_t nTr, const star_align_t* trs);   // Transcriptome::geneCountsAddAlign
    void write(const GeneModel& gm, const Stats& st, const std::string& path) const;   // Transcriptome::quantsOutput
};

// --quantMode TranscriptomeSAM: transcripts and their exons (transcriptInfo.tab, exonInfo.tab; Transcriptome.cpp:32-75)
struct TranscriptModel {
    std::vector<uint64_t> trS, trE, trEmax;
    std::vector<uint32_t> trExI, trLen;
    std::vector<uint16_t> trExN;
    std::vector<uint8_t> trStr;
    std::vector<std::string> trID;
    std::vector<uint32_t> exSE, exLenCum;
    int load(const std::string& dir, std::string& err);
    // Transcriptome::quantAlign (Transcriptome_quantAlign.cpp:94-114): the projections of a genomic alignment onto every transcript it fits
    uint32_t quantAlign(const star_align_t& aG, uint64_t Lread, std::vector<star_align_t>& out) const;
};

// Formats everything the reference writes per read: SAM records, junction records, counters.
class OutputWriter {
   public:
    OutputWriter(const HostParams& P, const LoadedIndex& idx) : P(P), idx(idx) {}
    // appends SAM text for reads [lo,hi) of the chunk to `sam`, junctions to `sj`, counters to `st`
    // coord / coordKey (may be NULL): the records for the coordinate-sorted BAM (uncompressed) and, per record, the read-order key
    // (iReadAll<<32 | iTr<<8 | mate) of BAMoutput::coordOneAlign
    // by (1st stage of --outFilterType BySJout): reads with an unannotated junction are neither counted nor written but listed in
    // by->held; the junction records of ALL mapped reads are appended to by->sjAll
    struct BySJoutHold { std::vector<uint32_t> held; std::vector<Junction> sjAll; };
    // unm (--outReadsUnmapped Fastx): text for Unmapped.out.mate1 / mate2
    void formatReads(const ReadChunk& c, const star_align_batch_t& out, uint32_t lo, uint32_t hi, std::string& sam,
                     std::vector<Junction>& sj, Stats& st, std::string* coord = nullptr, std::vector<uint64_t>* coordKey = nullptr,
                     BySJoutHold* by = nullptr, std::string* unm = nullptr, GeneCounts* gc = nullptr, std::string* trBam = nullptr,
                     const double* trDraw = nullptr) const;
    const GeneModel* geneModel = nullptr;   // set for --quantMode GeneCounts
    const TranscriptModel* trModel = nullptr;   // set for --quantMode TranscriptomeSAM
    std::string bamHeaderTranscriptome() const;   // samHeaders.cpp:8-20
    // true when read i of stage 1 of BySJout is held back (ReadAlign::outFilterBySJout)
    static bool heldBySJout(const star_align_batch_t& out, uint32_t i);
    std::string samHeader(bool sortedCoord = false) const;            // samHeaders.cpp:5-113
    std::string bamHeader(bool sortedCoord = false) const;           // outBAMwriteHeader, BAMfunctions.cpp:77-92 (uncompressed bytes)
    // BGZF framing (htslib bgzf.c: 0xff00-byte payload blocks, raw deflate, crc32 + isize trailer); appends to `out`
    static void bgzfCompress(const char* data, size_t n, int level, std::string& out);
    static const char* bgzfEofBlock(size_t& n);
    // outputSJ.cpp:20-200: collapse + filters + SJ.out.tab text; returns error text (empty = ok)
    std::string writeSJ(std::vector<Junction>& all, const std::string& path, bool distFilter = true) const;
    std::string novelJunctions(std::vector<Junction>& all, std::vector<uint64_t>& sjStart, std::vector<uint64_t>& sjEnd) const;
    static void collapseSJ(std::vector<Junction>& v, std::string& err);
    void writeLogFinal(const Stats& st, const std::string& path) const;  // Stats.cpp:99-145

   private:
    const HostParams& P;
    const LoadedIndex& idx;
    void bamMapped(const ReadChunk& c, uint32_t i, const star_read_result_t& r, const star_align_t& tr, uint64_t nTrOut, uint64_t iTrOut,
                   std::string& bam, bool transcriptomic = false) const;                          // ReadAlign_alignBAM.cpp:47-614, mapped branch
    void quantTranscriptome(const ReadChunk& c, uint32_t i, const star_read_result_t& r, const star_align_t* trs, uint64_t nTr, double draw, std::string& bam) const;
    void bamUnmapped(const ReadChunk& c, uint32_t i, const star_read_result_t& r, const star_align_t* trBest, int unmapType,
                     const bool* mateMap, std::string& bam) const;    // ReadAlign_alignBAM.cpp, alignType>=0 branch
    void samMapped(const ReadChunk& c, uint32_t i, const star_read_result_t& r, const star_align_t& tr, uint64_t nTrOut, uint64_t iTrOut,
                   std::string& sam) const;
    void samUnmapped(const ReadChunk& c, uint32_t i, const star_read_result_t& r, const star_align_t* trBest, int unmapType,
                     const bool* mateMap, std::string& sam) const;
    void recordSJ(const star_align_t& tr, uint64_t nTrOut, std::vector<Junction>& sj, size_t sjReadStartN) const;
};

}  // namespace starhost
