/*
 * star_b200.h — C-ABI of the H100-native STAR alignment hot path.
 *
 * STAR (alexdobin/STAR 2.7.11b) has no plugin/FFI interface; the seam this library replaces is
 * internal C++:
 *     void ReadAlignChunk::mapChunk()            reference source/ReadAlignChunk_mapChunk.cpp:7-128
 *       -> int ReadAlign::oneRead()              reference source/ReadAlign_oneRead.cpp:8-121
 *         -> int ReadAlign::mapOneRead()         reference source/ReadAlign_mapOneRead.cpp:6-118
 *         -> void ReadAlign::multMapSelect()     reference source/ReadAlign_multMapSelect.cpp:8-95
 *         -> void ReadAlign::mappedFilter()      reference source/ReadAlign_mappedFilter.cpp:3-20
 * i.e. "take one chunk of reads, return for every read the selected alignments (trMult[0..nTr),
 * unmapType, trBest)".  Everything in this header is plain C: pointers, sizes and POD structs.
 * INTEGRATION.md shows the binding a STAR maintainer would add inside mapChunk().
 *
 * The engine entry points (star_gpu_*) are implemented ONLY by hand-written sm_90a CUDA kernels
 * (star_b200/csrc/engine/).  There is no CPU fallback: without a CUDA device star_gpu_init fails
 * with STAR_EXIT_RUNTIME and star_gpu_last_error() says why.
 */
#ifndef STAR_B200_H
#define STAR_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- exit codes: reference source/IncludeDefine.h:149-160 ------------------------------------ */
#define STAR_EXIT_OK 0
#define STAR_EXIT_BUG 101
#define STAR_EXIT_PARAMETER 102
#define STAR_EXIT_RUNTIME 103
#define STAR_EXIT_INPUT_FILES 104
#define STAR_EXIT_GENOME_FILES 105
#define STAR_EXIT_MEMORY_ALLOCATION 108

/* ---- per-read markers: reference source/IncludeDefine.h:217-226 ------------------------------ */
#define STAR_MARKER_ALL_PIECES_EXCEED_seedMultimapNmax 999901u
#define STAR_MARKER_NO_GOOD_WINDOW 999903u
#define STAR_MARKER_NO_GOOD_PIECES 999904u
#define STAR_MARKER_TOO_MANY_ANCHORS_PER_WINDOW 999905u
#define STAR_MARKER_READ_TOO_SHORT 999910u

#define STAR_MAX_N_EXONS 20        /* reference IncludeDefine.h:131 (short-read build) */
#define STAR_READ_SEQ_LENGTH_MAX 650 /* reference IncludeDefine.h:140 DEF_readSeqLengthMax */
#define STAR_MARK_FRAG_SPACER_BASE 11 /* reference IncludeDefine.h:172 */
#define STAR_SJ_MOTIF_SIZE 7

/*
 * Parameters read by the hot path (SURVEY.md §8 row a-7'); names are the reference's
 * (source/parametersDefault, Parameters.h).  Derived values are computed by the caller exactly as
 * the reference does (Parameters.cpp:966-1124, Genome_genomeLoad.cpp:382-410).
 */
typedef struct star_params {
    /* seeding: ReadAlign_mapOneRead.cpp, ReadAlign_storeAligns.cpp */
    uint64_t seedSearchStartLmax;
    double   seedSearchStartLmaxOverLread;
    uint64_t seedSearchLmax;          /* 0 (default): off; > 0: one more search of at most this length from every start */
    uint64_t seedMapMin;
    uint64_t seedSplitMin;
    uint64_t seedMultimapNmax;
    uint64_t seedPerReadNmax;
    uint64_t seedPerWindowNmax;
    uint64_t maxNsplit;               /* hard-coded 10, Parameters.cpp:473 */
    /* windows: ReadAlign_stitchPieces.cpp, ReadAlign_createExtendWindowsWithAlign.cpp */
    uint64_t winAnchorMultimapNmax;
    uint64_t winBinNbits;
    uint64_t winBinChrNbits;          /* = genomeChrBinNbits - winBinNbits */
    uint64_t winAnchorDistNbins;
    uint64_t winFlankNbins;
    uint64_t winBinN;                 /* = nGenome/2^winBinNbits + 1 */
    uint64_t alignWindowsPerReadNmax;
    uint64_t alignTranscriptsPerWindowNmax;
    uint64_t alignTranscriptsPerReadNmax;
    /* stitching: stitchAlignToTranscript.cpp, stitchWindowAligns.cpp, extendAlign.cpp */
    uint64_t alignIntronMin;
    uint64_t alignIntronMax;
    uint64_t alignMatesGapMax;
    uint64_t alignSJoverhangMin;
    uint64_t alignSJDBoverhangMin;
    int32_t  alignSJstitchMismatchNmax[4];
    uint64_t alignSplicedMateMapLmin;
    double   alignSplicedMateMapLminOverLmate;
    uint8_t  alignEndsTypeExt[2][2];  /* alignEndsType.ext, Parameters.cpp:966-989 */
    int32_t  alignEndsProtrudeNbasesMax;
    uint8_t  alignEndsProtrudeConcordantPair;
    uint8_t  alignSoftClipAtReferenceEnds; /* .yes */
    uint8_t  alignInsertionFlushRight;
    int32_t  scoreGap, scoreGapNoncan, scoreGapGCAG, scoreGapATAC;
    double   scoreGenomicLengthLog2scale;
    int32_t  scoreDelOpen, scoreDelBase, scoreInsOpen, scoreInsBase, scoreStitchSJshift;
    int32_t  sjdbScore;
    /* filters: ReadAlign_oneRead.cpp:78, ReadAlign_multMapSelect.cpp, ReadAlign_mappedFilter.cpp */
    uint64_t outFilterMismatchNmax;
    double   outFilterMismatchNoverLmax;
    double   outFilterMismatchNoverReadLmax;
    int32_t  outFilterMultimapScoreRange;
    uint64_t outFilterMultimapNmax;
    int32_t  outFilterScoreMin;
    double   outFilterScoreMinOverLread;
    uint64_t outFilterMatchNmin;
    double   outFilterMatchNminOverLread;
    uint8_t  outFilterIntronMotifs;   /* 0 None, 1 RemoveNoncanonical, 2 RemoveNoncanonicalUnannotated */
    uint8_t  outFilterIntronStrandsRemoveInconsistent; /* outFilterIntronStrands=="RemoveInconsistentStrands" */
    uint8_t  outSAMstrandFieldType;   /* 0 None, 1 intronMotif */
    uint8_t  outSAMprimaryFlagAllBestScore;
    uint64_t outSAMmultNmax;          /* (uint64)-1 = all */
    /* --outFilterType BySJout: the 2nd stage's junction list is set with star_gpu_set_sj_novel; --outMultimapperOrder Random is not built
       (rejected by the host parser) */
} star_params_t;

/*
 * Read-only view of a loaded STAR genome index (the arrays of `class Genome`, reference
 * source/Genome.h:26-56, filled by Genome_genomeLoad.cpp).  All pointers are HOST pointers owned
 * by the caller; star_gpu_init copies them to the device once.
 */
typedef struct star_index_view {
    const uint8_t* G;        /* nGenome bytes, 1 B/base codes 0..5 (Genome file); caller guarantees that
                                G[-256..-1] and G[nGenome..nGenome+255] are readable and hold code 5
                                (reference pads 200, Genome_genomeLoad.cpp:27,320-323) */
    uint64_t nGenome;
    const uint8_t* SA;       /* bit-packed, (GstrandBit+1) bits per entry, nSAbyte bytes (+8 readable) */
    uint64_t nSA, nSAbyte;
    const uint8_t* SAi;      /* bit-packed, (GstrandBit+3) bits per entry (+8 readable) */
    uint64_t nSAi, nSAibyte;
    uint32_t GstrandBit;
    uint32_t gSAindexNbases;
    uint32_t gSAsparseD;     /* must be 1 */
    uint32_t gChrBinNbits;
    const uint64_t* genomeSAindexStart; /* gSAindexNbases+1 entries */
    uint32_t nChrReal;
    const uint64_t* chrStart;  /* nChrReal+1 */
    const uint64_t* chrLength; /* nChrReal */
    /* splice junction database, Genome_genomeLoad.cpp:471-520 */
    uint64_t sjdbN, sjdbOverhang, sjdbLength, sjGstart;
    const uint64_t* sjdbStart;
    const uint64_t* sjdbEnd;
    const uint64_t* sjDstart;
    const uint64_t* sjAstart;
    const uint8_t* sjdbMotif;
    const uint8_t* sjdbShiftLeft;
    const uint8_t* sjdbShiftRight;
    const uint8_t* sjdbStrand;
} star_index_view_t;

/*
 * One chunk of reads (what processChunks() hands to mapChunk(), ReadAlignChunk_processChunks.cpp:130-157,
 * minus names and qualities which never go to the device).
 * Mate m of read i occupies seq[seqOff[i*nMates+m] .. seqOff[i*nMates+m+1]) as ASCII (ACGTacgt, anything
 * else is N: SequenceFuns.cpp:131-146).  A mate of a PAIR may be empty (a read clipped to nothing before mapping, ClipMate_clip.cpp);
 * a single-end read has at least one base.
 */
typedef struct star_read_batch {
    uint32_t nReads;
    uint32_t nMates;          /* 1 or 2 */
    const char* seq;
    const uint64_t* seqOff;   /* nReads*nMates + 1 */
} star_read_batch_t;

/* One selected alignment = the fields of `class Transcript` (Transcript.h:10-81) that
 * multMapSelect / outputTranscriptSAM / outputTranscriptSJ / Stats::transcriptStats read. */
typedef struct star_align {
    uint64_t exG[STAR_MAX_N_EXONS];      /* exons[][EX_G] */
    uint16_t exR[STAR_MAX_N_EXONS];      /* exons[][EX_R] */
    uint16_t exL[STAR_MAX_N_EXONS];      /* exons[][EX_L] */
    uint8_t  exFrag[STAR_MAX_N_EXONS];   /* exons[][EX_iFrag] */
    int8_t   canonSJ[STAR_MAX_N_EXONS];
    uint8_t  sjAnnot[STAR_MAX_N_EXONS];
    uint8_t  sjStr[STAR_MAX_N_EXONS];
    uint16_t shiftSJ[STAR_MAX_N_EXONS][2];
    uint32_t nExons;
    uint32_t Chr;
    uint8_t  Str, roStr, primaryFlag, sjMotifStrand;
    int32_t  iFrag;
    int32_t  maxScore;
    uint32_t nMatch, nMM;
    uint32_t nGap, lGap, nDel, lDel, nIns, lIns;
    uint32_t nUnique, nAnchor;
    uint32_t rStart, rLength, roStart;
    uint64_t gStart, gLength, cStart;
} star_align_t;

typedef struct star_read_result {
    int32_t  unmapType;    /* -1 mapped; 0 other, 1 too short, 2 too many mismatches, 3 too many loci
                              (ReadAlign_mappedFilter.cpp:5-17) */
    uint32_t nTr;          /* number of multimapping alignments found by multMapSelect (may exceed
                              outFilterMultimapNmax; then unmapType==3 and nothing is returned) */
    uint32_t nTrOut;       /* alignments returned for this read: nTr if unmapType<0 else 0 */
    uint32_t mapMarker;    /* STAR_MARKER_* or 0 */
    uint64_t trOffset;     /* index of the first of nTrOut entries in star_align_batch.aligns */
    int32_t  bestScore;    /* trBest->maxScore  (printed for unmapped reads, outputTranscriptSAM.cpp:44) */
    uint32_t bestNMM;      /* trBest->nMM */
    uint32_t bestRLength;  /* trBest->rLength */
    uint32_t Lread;        /* length of the combined read incl. spacer */
    uint32_t bestTr;       /* index (0..nTrOut) of trBest among the returned alignments (writeSAM's trBestSAM,
                              ReadAlign_outputAlignments.cpp:207-209) */
} star_read_result_t;

typedef struct star_align_batch {
    star_read_result_t* reads;   /* caller-owned, capacity >= nReads */
    star_align_t* aligns;        /* caller-owned */
    uint64_t alignsCapacity;     /* entries available in aligns */
    uint64_t nAligns;            /* OUT: entries written (input order, read by read) */
} star_align_batch_t;

/* per-call timing / work counters filled by the engine (all device times from CUDA events) */
typedef struct star_chunk_stats {
    float ms_h2d, ms_prep, ms_seed, ms_window /* slow-path re-run */, ms_stitch /* fast path */, ms_pack, ms_d2h, ms_total;
    uint64_t h2d_bytes, d2h_bytes;
    uint64_t n_kernel_launches;
    /* algorithmic work counters of the MMP search (SURVEY.md §8(d)): */
    uint64_t mmp_searches, mmp_sai_words, mmp_compare_calls, mmp_bases_examined;
    uint64_t sa_enumerated;
    uint64_t stitch_nodes, stitch_leaves;
    uint64_t slow_path_reads;
    uint64_t heavy_reads;   /* reads stitched by the warp-per-read kernel */
    float ms_heavy;         /* time of that kernel inside ms_stitch */
    float pad_;
} star_chunk_stats_t;

typedef struct star_ctx star_ctx_t;

/* star_gpu_init: replaces the per-thread construction of ReadAlignChunk/ReadAlign (reference
 * source/ReadAlignChunk.cpp:5-70, ReadAlign.cpp:6-110) plus making the index resident (the reference keeps
 * it in host RAM / SysV shm, Genome_genomeLoad.cpp:177-243; here: HBM).  device = CUDA ordinal.
 * maxReadsPerChunk bounds the batch size of later star_gpu_map_chunk calls. */
int star_gpu_init(star_ctx_t** ctx, int device, const star_index_view_t* index, const star_params_t* params,
                  uint32_t maxReadsPerChunk);

/* star_gpu_map_chunk: replaces ReadAlignChunk::mapChunk() + the ReadAlign::oneRead() loop (reference
 * source/ReadAlignChunk_mapChunk.cpp:29-39).  `in` and `out` are HOST buffers (pinned or pageable);
 * host->device and device->host copies happen inside.  Results are returned in input order.
 * Returns 0 or a STAR_EXIT_* code (the reference calls exitWithError -> exit(code), ErrorWarning.cpp:8-23). */
int star_gpu_map_chunk(star_ctx_t* ctx, const star_read_batch_t* in, star_align_batch_t* out,
                       star_chunk_stats_t* stats /* may be NULL */);

/* Same hot path with the chunk already resident in device memory (bench "value" leg): uploads `in` once. */
int star_gpu_upload_chunk(star_ctx_t* ctx, const star_read_batch_t* in);
/* Runs all kernels on the uploaded chunk; results stay on the device.  stats->ms_* are filled. */
int star_gpu_map_resident(star_ctx_t* ctx, star_chunk_stats_t* stats);
/* Copies the results of the last star_gpu_map_resident / star_gpu_map_chunk to host buffers.  When out->alignsCapacity is smaller than
 * the number of records, nothing is copied: STAR_EXIT_RUNTIME is returned with out->nAligns = the capacity needed (the results stay
 * resident; the call can be repeated with a larger buffer).  star_gpu_map_chunk behaves the same way. */
int star_gpu_download_results(star_ctx_t* ctx, star_align_batch_t* out);

/* Page-locked host memory for the chunk buffers (`in->seq`, `out->reads`, `out->aligns`): copies from / to pageable memory reach a
 * fraction of the link rate.  Optional: every entry point accepts pageable buffers.  NULL when the allocation fails. */
void* star_gpu_host_alloc(size_t bytes);
void star_gpu_host_free(void* p);

/* 2nd stage of --outFilterType BySJout (reference source/stitchWindowAligns.cpp:169-177, outputSJ.cpp:139-160): from now on an alignment
 * with an unannotated junction is only kept when the junction (first / last intron base, 0-based genome coordinates) is in this list, which
 * must be sorted by start, then end.  n = 0 drops every alignment with an unannotated junction. */
int star_gpu_set_sj_novel(star_ctx_t* ctx, const uint64_t* sjStart, const uint64_t* sjEnd, uint64_t n);

/* analysis helper: per-read records of the resident chunk (44 bytes each: Lread u32, readLength u16[2], nP u16, pad u16, nA, mapMarker,
 * multNminL u32, Nsplit u16, split1_0 u16, mmTotal u32, flags u32, then 8 x u32 work counters: searches, saiWords, compareCalls,
 * basesExamined, saEnumerated, stitchNodes, stitchLeaves, slowPath) */
int star_gpu_debug_read_info(star_ctx_t* ctx, void* dst, uint64_t bytes);
/* analysis helper: per-phase cycle sums of the stitch kernels (32 x uint64), reset on read */
int star_gpu_debug_prof(star_ctx_t* ctx, uint64_t* out32);

void star_gpu_destroy(star_ctx_t* ctx);
const char* star_gpu_last_error(void);
/* number of kernels this library has launched in this process (bench.py "gpu_launches") */
uint64_t star_gpu_launch_count(void);

/* ---- host-side helpers (no device needed) ----------------------------------------------------------- */

/* Fills *p with the reference's defaults (source/parametersDefault) and the derived values. */
void star_params_default(star_params_t* p);

/* Loads a STAR genomeDir (Genome, SA, SAindex, chr*.txt, sjdbInfo.txt, genomeParameters.txt) exactly as
 * Genome::genomeLoad does (Genome_genomeLoad.cpp:18-420) and finishes the index-dependent parameters in *p
 * (winBinNbits.. winBinN).  Returns an opaque handle; star_index_get gives the view. */
typedef struct star_index star_index_t;
int star_index_load(const char* genomeDir, star_params_t* p, star_index_t** out);
const star_index_view_t* star_index_get(const star_index_t* idx);
void star_index_free(star_index_t* idx);
const char* star_host_last_error(void);

/* sizeof() of the ABI structs, so that foreign-language bindings can verify their layout:
 * which = 0 star_params_t, 1 star_index_view_t, 2 star_read_batch_t, 3 star_align_t, 4 star_read_result_t,
 * 5 star_align_batch_t, 6 star_chunk_stats_t */
size_t star_abi_sizeof(int which);

/* The drop-in command line: `STAR --runMode alignReads --genomeDir .. --readFilesIn ..` (reference
 * source/STAR.cpp:58-313).  Returns the process exit code. */
int star_cli_main(int argc, char** argv);

/* Multi-GPU (SURVEY.md §8e): every rank runs the command line with --gpuShardIndex r --gpuShardCount R --outFileNamePrefix <prefix>shard<r>.
 * and maps a contiguous slice of the reads; after an allreduce(sum) of the 24 Log.final.out counters (Stats.h:11-24) rank 0 calls
 * this with the ORIGINAL command line (prefix <prefix>) to concatenate the SAM shards in order, run the reference's global junction
 * collapse + filters (outputSJ.cpp:20-200) over all shards' junction records and write SJ.out.tab / Log.final.out.
 * counters24 may be NULL (then the shard files are summed). */
int star_host_merge_shards(int argc, char** argv, int nShards, const uint64_t* counters24);

/* ---- on-the-fly junction insertion (SURVEY.md §8f N3: --sjdbFileChrStartEnd at the mapping stage, --twopassMode Basic) -------
 * The device part of sjdbBuildIndex (reference source/sjdbBuildIndex.cpp:16-333).  The host side (star_b200/csrc/host/sjdb_insert.cpp)
 * prepares the junction inserts (sjdbPrepare.cpp:5-225), sorts the insertion points and patches SAindex; the two steps that touch
 * every new suffix / every SA row run on the GPU:
 *   star_gpu_sjdb_search   = the suffixArraySearch1 loop (sjdbBuildIndex.cpp:50-87, SuffixArrayFuns.cpp:233-351): for every suffix of
 *                            every insert (both strands) the SA row it has to be inserted in front of;
 *   star_gpu_sjdb_merge_sa = the SA rewrite (sjdbBuildIndex.cpp:141-214): old rows re-based to the new genome length / new junction
 *                            order, new rows spliced in, packed at GstrandBit+1 bits.
 * All pointers are HOST pointers. */
typedef struct star_sjdb star_sjdb_t;
/* uploads G and SA of the index the junctions are inserted into */
int star_gpu_sjdb_open(star_sjdb_t** h, int device, const star_index_view_t* oldIndex);
/* Gsj: 2*nGsj+1 bytes, nGsj = sjdbN*sjdbLength: the sjdbN inserts (donor flank, acceptor flank, one code 5), then their reverse
 * complement, then one code 5 (sjdbBuildIndex.cpp:32-40).  skipSeq[q], q in [0, 2*sjdbN): sequence q belongs to a junction that is
 * already in the index (no rows are added for it).  indArray: 2 * (2*sjdbN*sjdbLength) words; for k = q*sjdbLength + start:
 * indArray[2k] = SA row in front of which the suffix goes ((uint64)-1: none, (uint64)-2: after the last row), indArray[2k+1] = k. */
int star_gpu_sjdb_search(star_sjdb_t* h, const uint8_t* Gsj, uint64_t sjdbN, uint64_t sjdbLength, const uint8_t* skipSeq, uint64_t* indArray);
/* indSorted: nInd pairs (row, offset in Gsj) in insertion order (funCompareUintAndSuffixes.cpp:6-43).  nGsj = total insert bytes of
 * the NEW junction set, nGsjNew = bytes of the junctions that were not in the old index, oldSJind[j] = new index of old junction j
 * (oldIndex->sjdbN entries).  SAnew receives nSAnewByte bytes = PackedArray of oldIndex->nSA + nInd rows. */
int star_gpu_sjdb_merge_sa(star_sjdb_t* h, const uint64_t* indSorted, uint64_t nInd, uint64_t nGsj, uint64_t nGsjNew, uint64_t sjdbLength,
                           const uint32_t* oldSJind, uint8_t* SAnew, uint64_t nSAnewByte);
void star_gpu_sjdb_close(star_sjdb_t* h);

/* ---- index generation (SURVEY.md §8f N4: --runMode genomeGenerate) --------------------------------------------------------------
 * star_gpu_sa_build replaces the suffix sort of Genome::genomeGenerate (reference source/Genome_genomeGenerate.cpp:178-330,
 * funCompareSuffixes :29-89).  G: nGenome bytes, codes 0..5, at least 100 bytes of code 5 readable on both sides (HOST pointer).
 * The text is G followed by its reverse complement; every position holding a code < 4 is a suffix; order = lexicographic by code,
 * a code 5 met at the same offset in both suffixes ends the comparison and the smaller text position goes first.
 * SA receives nSAbyte bytes: nSA entries of GstrandBit+1 bits, forward positions as they are, reverse ones as (pos - nGenome) | 1<<GstrandBit. */
int star_gpu_sa_build(int device, const uint8_t* G, uint64_t nGenome, uint32_t GstrandBit, uint64_t nSA, uint8_t* SA, uint64_t nSAbyte);

/* Sharded --twopassMode Basic: between the two phases (--gpuTwoPassPhase 1 / 2 of every rank) the collapsed 1st-pass junction records of
 * all shards are all-gathered (star_b200.dist: sizes, then payload, over NCCL / gloo); every rank stores them as <dir>gather<r>.bin and
 * calls this with the ORIGINAL command line to get the same global <dir>SJ.out.tab (collapse + filters of outputSJ.cpp:20-200 over all
 * shards) and <dir>Log.final.out; dir = <shard prefix>_STARpass1/. */
int star_host_merge_pass1(int argc, char** argv, int nShards, const char* dir);

/* ---- signal tracks (--outWigType, --runMode inputAlignmentsFromBAM; reference source/signalFromBAM.cpp:5-209) ------------------------
 * The host decodes the BAM records of one segment (a run of records with the same reference, signalFromBAM.cpp:78-120) into blocks in
 * record order; the device builds the per-base tracks of the segment and returns only the positions where a track's output changes.
 * Track t = 2*strand + k: k = 0 "Unique" (number of NH==1 records covering the base), k = 1 "UniqueMultiple" (left fold, in record order,
 * of 1.0/NH over the records covering the base, as the reference's `sigAll[..] += 1.0/aNH` sums it).  All pointers are HOST pointers. */
typedef struct star_signal_block {
    uint32_t start;   /* first position (0-based) of the segment this record adds to */
    uint32_t len;     /* positions start .. start+len-1 (start+len <= chrLen) */
    uint32_t nh;      /* NH of the record, >= 1 */
    uint32_t strand;  /* 0 or 1; always 0 for an unstranded run */
} star_signal_block_t;
typedef struct star_signal_track {
    const uint32_t* pos;   /* positions (0-based, increasing) ... */
    const double* val;     /* ... and the track's value there (owned by the handle; valid until its next call) */
    uint64_t n;
} star_signal_track_t;
typedef struct star_signal star_signal_t;
/* nStrands = 1 (2 tracks) or 2 (4 tracks) */
int star_gpu_signal_open(star_signal_t** h, int device, uint32_t nStrands);
/* One segment of chrLen positions.  mode 0 (bedGraph): every position whose value differs from the position before (0 before position 0);
 * mode 1 (wiggle): every position with a nonzero value.  tracks: 2*nStrands entries.  ms (may be NULL) receives the device time of the
 * call's kernels (CUDA events).  Returns 0 or a STAR_EXIT_* code. */
int star_gpu_signal_segment(star_signal_t* h, uint32_t chrLen, const star_signal_block_t* blocks, uint64_t nBlocks, int mode,
                            star_signal_track_t* tracks, float* ms);
void star_gpu_signal_close(star_signal_t* h);

/* ---- duplicate marking (--bamRemoveDuplicatesType with --runMode inputAlignmentsFromBAM; reference source/bamRemoveDuplicates.cpp) ----
 * The host marks the records and finds the groups; the device pairs the NH == 1 members of each group in name order, classes the pairs by
 * start, flags, S-extended CIGARs and the compared mate-2 bases, and picks the pair of every class whose first record has the highest AS
 * (ties: the first in name order).  All pointers are HOST pointers. */
typedef struct star_dedup star_dedup_t;
int star_gpu_dedup_open(star_dedup_t** h, int device, uint64_t mate2basesN);
/* n members in file order: member i's record (its block_size field) is at bytes + offsets[i] (offsets increasing), groups[i] its group
 * (non-decreasing; a batch holds whole groups).  unmark[i] (n bytes) receives 1 for every record of a winning pair, else 0.  ms (may be
 * NULL) receives the device time (CUDA events).  Returns 0, or STAR_EXIT_INPUT_FILES (a record the reference cannot compare: a CIGAR
 * without 1..100 operations that are not all S, fewer bases than mate2basesN, malformed optional fields, AS <= -999) or
 * STAR_EXIT_PARAMETER (AS missing) with unmark[] all 0 except 2 + kind at the member named (kind 0 CIGAR, 1 bases, 2 optional fields,
 * 3 AS missing, 4 AS <= -999): the first such member of the first group that has one. */
int star_gpu_dedup_batch(star_dedup_t* h, const uint8_t* bytes, const uint64_t* offsets, const uint32_t* groups, uint64_t n, uint8_t* unmark, float* ms);
void star_gpu_dedup_close(star_dedup_t* h);

/* ---- adding references at the mapping stage (--genomeFastaFiles with --runMode alignReads; reference source/Genome_insertSequences.cpp,
 * insertSeqSA.cpp) ------------------------------------------------------------------------------------------------------------------
 * The host (star_b200/csrc/host/addref.cpp) scans the FASTA files, lays out the grown genome (the nG1 bytes of the added, padded
 * chromosomes at nG = the old end of the chromosomes, the nG2 bytes of junction inserts moved behind them), sorts the insertion points and
 * rebuilds SAindex; the steps that touch every SA row or every added suffix run on the GPU:
 *   star_gpu_addref_open     uploads the grown G and the OLD SA and re-bases every old row in place (insertSeqSA.cpp:33-51): a forward row
 *                            >= nG and a reverse row whose position is >= nG2 grow by nG1;
 *   star_gpu_addref_search   for every suffix k of the 2*nG1-byte text (added sequences, then their reverse complement) the re-based row
 *                            in front of which it goes: suffixArraySearch1(N = 10000, gInsert = nG, strR = k < nG1) (SuffixArrayFuns.cpp:210-351);
 *   star_gpu_addref_merge_sa the new SA: inserted rows k + nG (forward) or (k - nG1 + nG2) | 1<<GstrandBit spliced in (insertSeqSA.cpp:158-199).
 * ms (may be NULL) receives the device time of the call's kernel (CUDA events).  All pointers are HOST pointers. */
typedef struct star_addref star_addref_t;
/* grown: G = the grown genome (nGenome = nG + nG1 + nG2, 256 readable bytes of code 5 on both sides), SA / nSA / nSAbyte / GstrandBit = the
 * OLD suffix array.  Fails with STAR_EXIT_MEMORY_ALLOCATION when G, the SA and the merged SA do not fit the free device memory. */
int star_gpu_addref_open(star_addref_t** h, int device, const star_index_view_t* grown, uint64_t nG, uint64_t nG1, uint64_t nG2, float* ms);
/* seq: 2*nG1 bytes, the added region forward then reverse complement.  indArray: 2 * (2*nG1) words; indArray[2k] = row ((uint64)-1: the
 * suffix starts with a code > 3, (uint64)-2: behind the last row), indArray[2k+1] = k. */
int star_gpu_addref_search(star_addref_t* h, const uint8_t* seq, uint64_t* indArray, float* ms);
/* indSorted: nInd pairs (row, k) in insertion order.  SAnew receives nSAnewByte bytes = PackedArray of nSA + nInd rows.  Releases the
 * device copy of G first (the merge does not read it); search cannot be called afterwards. */
int star_gpu_addref_merge_sa(star_addref_t* h, const uint64_t* indSorted, uint64_t nInd, uint8_t* SAnew, uint64_t nSAnewByte, float* ms);
void star_gpu_addref_close(star_addref_t* h);

/* Engine indirection used by star_cli_main; tests drive the same host code with the CPU oracle. */
typedef struct star_engine_vtbl {
    int (*init)(void** ctx, int device, const star_index_view_t*, const star_params_t*, uint32_t maxReads);
    int (*map_chunk)(void* ctx, const star_read_batch_t*, star_align_batch_t*, star_chunk_stats_t*);
    void (*destroy)(void* ctx);
    const char* (*last_error)(void);
    /* junction insertion (same meaning as star_gpu_sjdb_*; the handle is opaque to the host code) */
    int (*sjdb_open)(void** h, int device, const star_index_view_t* oldIndex);
    int (*sjdb_search)(void* h, const uint8_t* Gsj, uint64_t sjdbN, uint64_t sjdbLength, const uint8_t* skipSeq, uint64_t* indArray);
    int (*sjdb_merge_sa)(void* h, const uint64_t* indSorted, uint64_t nInd, uint64_t nGsj, uint64_t nGsjNew, uint64_t sjdbLength,
                         const uint32_t* oldSJind, uint8_t* SAnew, uint64_t nSAnewByte);
    void (*sjdb_close)(void* h);
    /* index generation (same meaning as star_gpu_sa_build) */
    int (*sa_build)(int device, const uint8_t* G, uint64_t nGenome, uint32_t GstrandBit, uint64_t nSA, uint8_t* SA, uint64_t nSAbyte);
    /* 2nd stage of --outFilterType BySJout (same meaning as star_gpu_set_sj_novel) */
    int (*set_sj_novel)(void* ctx, const uint64_t* sjStart, const uint64_t* sjEnd, uint64_t n);
    /* optional (may be NULL): page-locked chunk buffers (star_gpu_host_alloc / star_gpu_host_free) and a second fetch of the last
     * chunk's results after map_chunk reported a too small out->alignsCapacity (star_gpu_download_results) */
    void* (*host_alloc)(size_t bytes);
    void (*host_free)(void* p);
    int (*download_results)(void* ctx, star_align_batch_t* out);
    /* signal tracks (same meaning as star_gpu_signal_*) */
    int (*signal_open)(void** h, int device, uint32_t nStrands);
    int (*signal_segment)(void* h, uint32_t chrLen, const star_signal_block_t* blocks, uint64_t nBlocks, int mode, star_signal_track_t* tracks, float* ms);
    void (*signal_close)(void* h);
    /* duplicate marking (same meaning as star_gpu_dedup_*); may be NULL */
    int (*dedup_open)(void** h, int device, uint64_t mate2basesN);
    int (*dedup_batch)(void* h, const uint8_t* bytes, const uint64_t* offsets, const uint32_t* groups, uint64_t n, uint8_t* unmark, float* ms);
    void (*dedup_close)(void* h);
    /* adding references (same meaning as star_gpu_addref_*) */
    int (*addref_open)(void** h, int device, const star_index_view_t* grown, uint64_t nG, uint64_t nG1, uint64_t nG2, float* ms);
    int (*addref_search)(void* h, const uint8_t* seq, uint64_t* indArray, float* ms);
    int (*addref_merge_sa)(void* h, const uint64_t* indSorted, uint64_t nInd, uint8_t* SAnew, uint64_t nSAnewByte, float* ms);
    void (*addref_close)(void* h);
} star_engine_vtbl_t;
int star_cli_main_engine(int argc, char** argv, const star_engine_vtbl_t* engine);

#ifdef __cplusplus
}
#endif
#endif
