// output.cpp — per-read output records built from the engine's POD alignments.
//
// Restates (host side, text formatting only):
//   ReadAlign::outputAlignments / writeSAM / recordSJ   reference source/ReadAlign_outputAlignments.cpp:5-260
//   ReadAlign::outputTranscriptSAM                       source/ReadAlign_outputTranscriptSAM.cpp:5-359
//   ReadAlign::outputTranscriptSJ                        source/ReadAlign_outputTranscriptSJ.cpp:4-56
//   Stats::transcriptStats / reportFinal                 source/Stats.cpp:35-56,99-145
//   outputSJ + OutSJ::collapseSJ + Junction::outputStream source/outputSJ.cpp:20-200, OutSJ.cpp:34-90
//   samHeaders                                           source/samHeaders.cpp:5-113
#include <algorithm>
#include <cstring>
#include <ctime>
#include <fstream>
#include <iomanip>
#include <sstream>

#include <zlib.h>

#include "host.h"

namespace starhost {

enum { ATTR_NH = 1, ATTR_HI, ATTR_AS, ATTR_NM, ATTR_MD, ATTR_nM, ATTR_jM, ATTR_jI, ATTR_XS, ATTR_RG, ATTR_ch = 14, ATTR_MC = 15 };

static inline void putU(std::string& s, uint64_t v) {
    char b[24];
    int n = 0;
    do { b[n++] = (char)('0' + v % 10); v /= 10; } while (v);
    while (n) s.push_back(b[--n]);
}
static inline void putI(std::string& s, long long v) {
    if (v < 0) { s.push_back('-'); putU(s, (uint64_t)(-(v + 1)) + 1); } else putU(s, (uint64_t)v);
}

static const char* revComplementTable() {   // SequenceFuns.cpp:16-54
    struct Tab {   // built once, thread-safely (function-local static): the formatting threads call this concurrently
        char t[256];
        Tab() {
            for (int i = 0; i < 256; i++) t[i] = (char)i;
            const char* a = "ACGTNRYKMSWBDVHacgtnrykmswbdvh";
            const char* b = "TGCANYRMKSWVHBDtgcanyrmkswvhbd";
            for (int i = 0; a[i]; i++) t[(unsigned char)a[i]] = b[i];
        }
    };
    static const Tab T;
    return T.t;
}
static void revComplementAppend(const char* in, size_t L, std::string& s) {   // appends the reverse complement to s (no temporary)
    const char* tab = revComplementTable();
    const size_t o = s.size();
    s.resize(o + L);
    char* d = &s[o];
    for (size_t j = 0; j < L; j++) d[j] = tab[(unsigned char)in[L - 1 - j]];
}
static void revComplement(const char* in, size_t L, std::string& out) {  // SequenceFuns.cpp:16-54
    struct Tab {   // built once, thread-safely (function-local static): the formatting threads call this concurrently
        char t[256];
        Tab() {
            for (int i = 0; i < 256; i++) t[i] = (char)i;
            const char* a = "ACGTNRYKMSWBDVHacgtnrykmswbdvh";
            const char* b = "TGCANYRMKSWVHBDtgcanyrmkswvhbd";
            for (int i = 0; a[i]; i++) t[(unsigned char)a[i]] = b[i];
        }
    };
    static const Tab T;
    const char* tab = T.t;
    out.resize(L);
    for (size_t j = 0; j < L; j++) out[j] = tab[(unsigned char)in[L - 1 - j]];
}

void Stats::add(const Stats& s) {
    readN += s.readN; readBases += s.readBases; mappedReadsU += s.mappedReadsU; mappedReadsM += s.mappedReadsM; mappedBases += s.mappedBases;
    mappedMismatchesN += s.mappedMismatchesN; mappedInsN += s.mappedInsN; mappedDelN += s.mappedDelN; mappedInsL += s.mappedInsL; mappedDelL += s.mappedDelL;
    for (int i = 0; i < STAR_SJ_MOTIF_SIZE; i++) splicesN[i] += s.splicesN[i];
    splicesNsjdb += s.splicesNsjdb;
    unmappedOther += s.unmappedOther; unmappedShort += s.unmappedShort; unmappedMismatch += s.unmappedMismatch; unmappedMulti += s.unmappedMulti;
    unmappedAll += s.unmappedAll; chimericAll += s.chimericAll;
}
void Stats::toArray(uint64_t* a) const {
    uint64_t t[N_COUNTERS] = {readN, readBases, mappedReadsU, mappedReadsM, mappedBases, mappedMismatchesN, mappedInsN, mappedDelN, mappedInsL, mappedDelL,
                              splicesN[0], splicesN[1], splicesN[2], splicesN[3], splicesN[4], splicesN[5], splicesN[6], splicesNsjdb,
                              unmappedOther, unmappedShort, unmappedMismatch, unmappedMulti, unmappedAll, chimericAll};
    memcpy(a, t, sizeof(t));
}
void Stats::fromArray(const uint64_t* a) {
    readN = a[0]; readBases = a[1]; mappedReadsU = a[2]; mappedReadsM = a[3]; mappedBases = a[4]; mappedMismatchesN = a[5]; mappedInsN = a[6];
    mappedDelN = a[7]; mappedInsL = a[8]; mappedDelL = a[9];
    for (int i = 0; i < 7; i++) splicesN[i] = a[10 + i];
    splicesNsjdb = a[17]; unmappedOther = a[18]; unmappedShort = a[19]; unmappedMismatch = a[20]; unmappedMulti = a[21]; unmappedAll = a[22]; chimericAll = a[23];
}

// ReadAlign_outputTranscriptSJ.cpp:4-56
void OutputWriter::recordSJ(const star_align_t& tr, uint64_t nTrOut, std::vector<Junction>& sj, size_t sjReadStartN) const {
    if (tr.nExons == 0) return;
    for (uint32_t iex = 0; iex + 1 < tr.nExons; iex++) {
        if (tr.canonSJ[iex] >= 0) {
            Junction j;
            j.start = tr.exG[iex] + tr.exL[iex];
            j.gap = (uint32_t)(tr.exG[iex + 1] - j.start);
            j.overhangLeft = (uint16_t)std::min((uint32_t)tr.exL[iex], (uint32_t)tr.exL[iex + 1]);
            j.overhangRight = j.overhangLeft;
            bool dup = false;
            for (size_t ii = sjReadStartN; ii < sj.size(); ii++) {
                if (j.start == sj[ii].start && j.gap == sj[ii].gap) {
                    dup = true;
                    if (sj[ii].overhangLeft < j.overhangLeft) { sj[ii].overhangLeft = j.overhangLeft; sj[ii].overhangRight = j.overhangLeft; }
                    break;
                }
            }
            if (dup) continue;
            j.motif = (char)tr.canonSJ[iex];
            j.strand = (char)(tr.canonSJ[iex] == 0 ? 0 : (tr.canonSJ[iex] + 1) % 2 + 1);
            j.annot = (char)tr.sjAnnot[iex];
            if (nTrOut == 1) { j.countUnique = 1; j.countMultiple = 0; } else { j.countMultiple = 1; j.countUnique = 0; }
            sj.push_back(j);
        }
    }
}

// ReadAlign_outputTranscriptSAM.cpp:13-53 (unmapType>=0 branch)
void OutputWriter::samUnmapped(const ReadChunk& c, uint32_t i, const star_read_result_t& r, const star_align_t* tr, int unmapType,
                               const bool* mateMap, std::string& s) const {
    const char* name = c.names.data() + c.nameOff[i];
    for (unsigned imate = 0; imate < c.nMates; imate++) {
        if (mateMap[imate]) continue;
        unsigned flag = 0x4;
        if (c.nMates == 2) {
            flag |= 0x1 + (imate == 0 ? 0x40 : 0x80);
            if (mateMap[1 - imate]) {
                if (tr->Str != (1 - imate)) flag |= 0x20;
            } else {
                flag |= 0x8;
            }
        }
        if (c.readFilter[i] == 'Y') flag |= 0x200;
        if (mateMap[1 - imate] && tr && !tr->primaryFlag && P.unmappedKeepPairs) flag |= 0x100;
        s += name; s.push_back('\t'); putU(s, flag);
        s += "\t*\t0\t0\t*";
        if (c.nMates == 2 && mateMap[1 - imate]) {
            s.push_back('\t'); s += idx.chrName[tr->Chr]; s.push_back('\t'); putU(s, tr->exG[0] + 1 - idx.chrStart[tr->Chr]);
        } else {
            s += "\t*\t0";
        }
        uint64_t a = c.seqOff[(uint64_t)i * c.nMates + imate], b = c.seqOff[(uint64_t)i * c.nMates + imate + 1];
        s += "\t0\t";
        s.append(c.seq, a, b - a);
        s.push_back('\t');
        if (c.fastq) s.append(c.qual, a, b - a); else s.push_back('*');
        s += "\tNH:i:0\tHI:i:0\tAS:i:"; putI(s, tr ? tr->maxScore : r.bestScore);
        s += "\tnM:i:"; putU(s, tr ? tr->nMM : r.bestNMM);
        s += "\tuT:A:"; putI(s, unmapType);
        if (!P.outSAMattrRGs.empty()) { s += "\tRG:Z:"; s += P.outSAMattrRGs[c.fileIndex]; }
        s.push_back('\n');
    }
}

// ReadAlign_outputTranscriptSAM.cpp:56-359 (mapped branch)
void OutputWriter::samMapped(const ReadChunk& c, uint32_t i, const star_read_result_t& r, const star_align_t& tr, uint64_t nTrOut, uint64_t iTrOut,
                             std::string& s) const {
    const char* name = c.names.data() + c.nameOff[i];
    const bool flagPaired = c.nMates == 2;
    const uint64_t Lread = r.Lread;
    uint64_t readLength[2];
    readLength[0] = c.len(i, 0);   // the lengths that were mapped (after clipping)
    readLength[1] = flagPaired ? c.len(i, 1) : 0;
    const uint64_t readLengthOriginal[2] = {c.lenOrig(i, 0), flagPaired ? c.lenOrig(i, 1) : 0};
    uint32_t iExMate;
    unsigned nMates = 1;
    for (iExMate = 0; iExMate + 1 < tr.nExons; iExMate++) {
        if (tr.canonSJ[iExMate] == -3) { nMates = 2; break; }
    }
    unsigned samFlagCommon = 0;
    if (flagPaired) {
        samFlagCommon = 0x0001;
        if (iExMate == tr.nExons - 1) {
            samFlagCommon += 0x0008;  // mateChr == (uint)-1 > nChrReal
        } else {
            if (P.hp.alignEndsProtrudeConcordantPair ||
                ((tr.exG[0] <= tr.exG[iExMate + 1] + tr.exR[0]) &&
                 (tr.exG[iExMate] + tr.exL[iExMate] <= tr.exG[tr.nExons - 1] + Lread - tr.exR[tr.nExons - 1]))) {
                samFlagCommon += 0x0002;
            }
        }
    }
    if (c.readFilter[i] == 'Y') samFlagCommon += 0x200;
    const unsigned Str = tr.Str;
    unsigned leftMate = flagPaired ? Str : 0;

    std::string cigars[2], sjMotif[2], sjIntron[2];
    unsigned mateOf[2] = {0, 0};
    uint32_t ex1[2], ex2[2];
    for (unsigned imate = 0; imate < nMates; imate++) {  // also ReadAlign_calcCIGAR.cpp:3-60 (MC needs both CIGARs first)
        uint32_t iEx1 = (imate == 0 ? 0 : iExMate + 1);
        uint32_t iEx2 = (imate == 0 ? iExMate : tr.nExons - 1);
        ex1[imate] = iEx1; ex2[imate] = iEx2;
        unsigned Mate = tr.exFrag[iEx1];
        mateOf[imate] = Mate;
        std::string& cg = cigars[imate];
        // bases clipped before mapping come back as soft clips (ReadAlign_outputTranscriptSAM.cpp:134-146, 184-186)
        const uint64_t trimL = (Str == 0) == (Mate == 0) ? c.c5(i, Mate) : c.c3(i, Mate);
        uint64_t trimL1 = trimL + (uint64_t)tr.exR[iEx1] - (tr.exR[iEx1] < readLength[leftMate] ? 0 : readLength[leftMate] + 1);
        if (trimL1 > 0) { putU(cg, trimL1); cg.push_back('S'); }
        for (uint32_t ii = iEx1; ii <= iEx2; ii++) {
            if (ii > iEx1) {
                uint64_t gapG = tr.exG[ii] - (tr.exG[ii - 1] + tr.exL[ii - 1]);
                uint64_t gapR = (uint64_t)tr.exR[ii] - tr.exR[ii - 1] - tr.exL[ii - 1];
                if (gapR > 0) { putU(cg, gapR); cg.push_back('I'); }
                if (tr.canonSJ[ii - 1] >= 0 || tr.sjAnnot[ii - 1] == 1) {
                    putU(cg, gapG); cg.push_back('N');
                    sjMotif[imate].push_back(','); putI(sjMotif[imate], tr.canonSJ[ii - 1] + (tr.sjAnnot[ii - 1] == 0 ? 0 : 20));
                    sjIntron[imate].push_back(','); putU(sjIntron[imate], tr.exG[ii - 1] + tr.exL[ii - 1] + 1 - idx.chrStart[tr.Chr]);
                    sjIntron[imate].push_back(','); putU(sjIntron[imate], tr.exG[ii] - idx.chrStart[tr.Chr]);
                } else if (gapG > 0) {
                    putU(cg, gapG); cg.push_back('D');
                }
            }
            putU(cg, tr.exL[ii]); cg.push_back('M');
        }
        if (sjMotif[imate].empty()) { sjMotif[imate] = ",-1"; sjIntron[imate] = ",-1"; }
        uint64_t trimR1 = (tr.exR[iEx1] < readLength[leftMate] ? readLengthOriginal[leftMate] : readLength[leftMate] + 1 + readLengthOriginal[Mate]) - tr.exR[iEx2] - tr.exL[iEx2] - trimL;
        if (trimR1 > 0) { putU(cg, trimR1); cg.push_back('S'); }
    }

    for (unsigned imate = 0; imate < nMates; imate++) {
        unsigned samFLAG = samFlagCommon;
        uint32_t iEx1 = ex1[imate], iEx2 = ex2[imate];
        unsigned Mate = mateOf[imate];
        if (Mate == 0) {
            samFLAG |= Str * 0x10;
            if (nMates == 2) samFLAG |= (1 - Str) * 0x20;
        } else {
            samFLAG |= (1 - Str) * 0x10;
            if (nMates == 2) samFLAG |= Str * 0x20;
        }
        if (flagPaired) samFLAG |= (Mate == 0 ? 0x0040 : 0x0080);
        if (!tr.primaryFlag) samFLAG |= 0x100;
        int MAPQ = P.outSAMmapqUnique;
        if (nTrOut >= 5) MAPQ = 0; else if (nTrOut >= 3) MAPQ = 1; else if (nTrOut == 2) MAPQ = 3;
        s += name; s.push_back('\t'); putU(s, (samFLAG & P.outSAMflagAND) | P.outSAMflagOR); s.push_back('\t');
        s += idx.chrName[tr.Chr]; s.push_back('\t'); putU(s, tr.exG[iEx1] + 1 - idx.chrStart[tr.Chr]); s.push_back('\t');
        putI(s, MAPQ); s.push_back('\t'); s += cigars[imate];
        if (nMates > 1) {
            s += "\t=\t"; putU(s, tr.exG[(imate == 0 ? iExMate + 1 : 0)] + 1 - idx.chrStart[tr.Chr]);
            s.push_back('\t'); if (imate != 0) s.push_back('-');
            putU(s, tr.exG[tr.nExons - 1] + tr.exL[tr.nExons - 1] - tr.exG[0]);
        } else {
            s += "\t*\t0\t0";
        }
        uint64_t a = c.seqOff[(uint64_t)i * c.nMates + Mate], b = c.seqOff[(uint64_t)i * c.nMates + Mate + 1];
        s.push_back('\t');
        if (Mate == Str) {
            s.append(c.seq, a, b - a);
        } else {
            revComplementAppend(c.seq.data() + a, b - a, s);
        }
        s.push_back('\t');
        if (c.fastq && P.outSAMmode != "NoQS") {
            if (Mate == Str) s.append(c.qual, a, b - a);
            else {   // reversed, written in place (one resize instead of a capacity check per character)
                const size_t o = s.size(), L = b - a;
                s.resize(o + L);
                char* d = &s[o];
                const char* q = c.qual.data() + a;
                for (size_t k = 0; k < L; k++) d[k] = q[L - 1 - k];
            }
        } else {
            s.push_back('*');
        }
        uint64_t tagNM = 0;
        std::string tagMD;
        bool needNM = false;
        for (int code : P.outSAMattrOrder) if (code == ATTR_NM || code == ATTR_MD) needNM = true;
        if (needNM) {  // :252-288; R = Read1[roStr==0?0:2], built here from the original mates
            std::string R(Lread, (char)4);
            auto conv = [](char ch) -> char { switch (ch) { case 'A': case 'a': return 0; case 'C': case 'c': return 1; case 'G': case 'g': return 2; case 'T': case 't': return 3; default: return 4; } };
            for (uint64_t k = 0; k < readLength[0]; k++) R[k] = conv(c.base(i, 0, k));
            if (flagPaired) {
                R[readLength[0]] = STAR_MARK_FRAG_SPACER_BASE;
                for (uint64_t k = 0; k < readLength[1]; k++) { char ch = conv(c.base(i, 1, readLength[1] - 1 - k)); R[readLength[0] + 1 + k] = ch < 4 ? 3 - ch : ch; }
            }
            if (tr.roStr != 0) {
                std::string R2(Lread, (char)4);
                for (uint64_t k = 0; k < Lread; k++) { char ch = R[k]; R2[Lread - 1 - k] = ch < 4 ? 3 - ch : ch; }
                R.swap(R2);
            }
            static const char numToNT[6] = {'A', 'C', 'G', 'T', 'N', 'N'};
            uint64_t matchN = 0;
            for (uint32_t iex = iEx1; iex <= iEx2; iex++) {
                for (uint64_t ii = 0; ii < tr.exL[iex]; ii++) {
                    char r1 = R[ii + tr.exR[iex]];
                    char g1 = (char)idx.view.G[ii + tr.exG[iex]];
                    if (r1 != g1 || r1 == 4 || g1 == 4) {
                        ++tagNM;
                        tagMD += std::to_string(matchN);
                        tagMD.push_back(numToNT[(uint8_t)g1 < 6 ? (uint8_t)g1 : 5]);
                        matchN = 0;
                    } else {
                        matchN++;
                    }
                }
                if (iex < iEx2) {
                    if (tr.canonSJ[iex] == -1) {
                        tagNM += tr.exG[iex + 1] - (tr.exG[iex] + tr.exL[iex]);
                        tagMD += std::to_string(matchN) + "^";
                        for (uint64_t ii = tr.exG[iex] + tr.exL[iex]; ii < tr.exG[iex + 1]; ii++) tagMD.push_back(numToNT[idx.view.G[ii] < 6 ? idx.view.G[ii] : 5]);
                        matchN = 0;
                    } else if (tr.canonSJ[iex] == -2) {
                        tagNM += (uint64_t)tr.exR[iex + 1] - tr.exR[iex] - tr.exL[iex];
                    }
                }
            }
            tagMD += std::to_string(matchN);
        }
        for (int code : P.outSAMattrOrder) {
            switch (code) {
                case ATTR_NH: s += "\tNH:i:"; putU(s, nTrOut); break;
                case ATTR_HI: s += "\tHI:i:"; putU(s, iTrOut + P.outSAMattrIHstart); break;
                case ATTR_AS: s += "\tAS:i:"; putI(s, tr.maxScore); break;
                case ATTR_nM: s += "\tnM:i:"; putU(s, tr.nMM); break;
                case ATTR_jM: s += "\tjM:B:c"; s += sjMotif[imate]; break;
                case ATTR_jI: s += "\tjI:B:i"; s += sjIntron[imate]; break;
                case ATTR_XS:
                    if (tr.sjMotifStrand == 1) s += "\tXS:A:+";
                    else if (tr.sjMotifStrand == 2) s += "\tXS:A:-";
                    break;
                case ATTR_NM: s += "\tNM:i:"; putU(s, tagNM); break;
                case ATTR_MD: s += "\tMD:Z:"; s += tagMD; break;
                case ATTR_RG: s += "\tRG:Z:"; s += P.outSAMattrRGs[c.fileIndex]; break;
                case ATTR_MC: if (nMates > 1) { s += "\tMC:Z:"; s += cigars[1 - imate]; } break;
                default: break;  // ch: BAM-only
            }
        }
        s.push_back('\n');
    }
}

// ------------------------------------------------------------------------------------------------------------------
// BAM records (SURVEY.md §8f N1): restatement of ReadAlign::alignBAM (ReadAlign_alignBAM.cpp:47-614) for the path's
// alignment types (-1 mapped, >=0 unmapped), the typed attribute writers of BAMfunctions.cpp / BAMfunctions.h:44-77 and
// nuclPackBAM (SequenceFuns.cpp:99-129).  Records are appended uncompressed; the caller frames them into BGZF blocks.
namespace {
inline void put32(std::string& s, uint32_t v) { s.append((const char*)&v, 4); }
inline void attrInt(std::string& s, const char* tag, long long x) {  // bamAttrArrayWriteInt: smallest fitting type
    s.push_back(tag[0]); s.push_back(tag[1]);
    if (x < 0) {
        if (x >= -127) { s.push_back('c'); int8_t v = (int8_t)x; s.append((const char*)&v, 1); }
        else if (x >= -32767) { s.push_back('s'); int16_t v = (int16_t)x; s.append((const char*)&v, 2); }
        else { s.push_back('i'); int32_t v = (int32_t)x; s.append((const char*)&v, 4); }
    } else {
        if (x <= 255) { s.push_back('C'); uint8_t v = (uint8_t)x; s.append((const char*)&v, 1); }
        else if (x <= 65535) { s.push_back('S'); uint16_t v = (uint16_t)x; s.append((const char*)&v, 2); }
        else { s.push_back('I'); uint32_t v = (uint32_t)x; s.append((const char*)&v, 4); }
    }
}
inline void attrChar(std::string& s, const char* tag, char c) { s.push_back(tag[0]); s.push_back(tag[1]); s.push_back('A'); s.push_back(c); }
inline void attrStr(std::string& s, const char* tag, const std::string& v) { s.push_back(tag[0]); s.push_back(tag[1]); s.push_back('Z'); s.append(v.c_str(), v.size() + 1); }
inline int reg2bin(int beg, int end) {  // BAMfunctions.cpp:95-104
    --end;
    if (beg >> 14 == end >> 14) return ((1 << 15) - 1) / 7 + (beg >> 14);
    if (beg >> 17 == end >> 17) return ((1 << 12) - 1) / 7 + (beg >> 17);
    if (beg >> 20 == end >> 20) return ((1 << 9) - 1) / 7 + (beg >> 20);
    if (beg >> 23 == end >> 23) return ((1 << 6) - 1) / 7 + (beg >> 23);
    if (beg >> 26 == end >> 26) return ((1 << 3) - 1) / 7 + (beg >> 26);
    return 0;
}
inline uint8_t nuclToNumBAM(char cc) {  // =ACMGRSVTWYHKDBN
    switch (cc) {
        case '=': return 0; case 'A': case 'a': return 1; case 'C': case 'c': return 2; case 'M': case 'm': return 3;
        case 'G': case 'g': return 4; case 'R': case 'r': return 5; case 'S': case 's': return 6; case 'V': case 'v': return 7;
        case 'T': case 't': return 8; case 'W': case 'w': return 9; case 'Y': case 'y': return 10; case 'H': case 'h': return 11;
        case 'K': case 'k': return 12; case 'D': case 'd': return 13; case 'B': case 'b': return 14; default: return 15;
    }
}
// name | cigar | packed seq | qual | attributes after the 9-word core; block_size is patched at the end
void bamFinish(std::string& bam, size_t rec0) {
    uint32_t sz = (uint32_t)(bam.size() - rec0 - 4);
    memcpy(&bam[rec0], &sz, 4);
}
void bamSeqQual(std::string& bam, const char* seq, const char* qual, size_t L, bool fastqQual) {
    for (size_t jj = 0; jj < L / 2; jj++) bam.push_back((char)(nuclToNumBAM(seq[2 * jj]) << 4 | nuclToNumBAM(seq[2 * jj + 1])));
    if (L % 2 == 1) bam.push_back((char)(nuclToNumBAM(seq[L - 1]) << 4));
    if (fastqQual) for (size_t ii = 0; ii < L; ii++) bam.push_back((char)(qual[ii] - 33));
    else bam.append(L, (char)0xFF);
}
}  // namespace

void OutputWriter::bamUnmapped(const ReadChunk& c, uint32_t i, const star_read_result_t& r, const star_align_t* tr, int unmapType,
                               const bool* mateMap, std::string& bam) const {
    const char* name = c.names.data() + c.nameOff[i];
    const size_t nameLen = strlen(name);
    for (unsigned imate = 0; imate < c.nMates; imate++) {
        if (mateMap[imate]) continue;   // this mate was mapped, do not record it as unmapped (:121)
        unsigned flag = 0x4;
        uint32_t mateChr = 0xFFFFFFFFu, mateStart = 0xFFFFFFFFu;
        if (c.nMates == 2) {
            flag |= 0x1 + (imate == 0 ? 0x40 : 0x80);
            if (mateMap[1 - imate]) {
                if (tr->Str != (1 - imate)) flag |= 0x20;
                mateChr = tr->Chr;
                mateStart = (uint32_t)(tr->exG[0] - idx.chrStart[tr->Chr]);
                if (!tr->primaryFlag && P.unmappedKeepPairs) flag |= 0x100;
            } else {
                flag |= 0x8;
            }
        }
        if (c.readFilter[i] == 'Y') flag |= 0x200;
        std::string at;
        attrInt(at, "NH", 0); attrInt(at, "HI", 0);
        attrInt(at, "AS", tr ? tr->maxScore : r.bestScore);
        attrInt(at, "nM", tr ? (long long)tr->nMM : (long long)r.bestNMM);
        attrChar(at, "uT", std::to_string((unsigned)unmapType).at(0));
        if (!P.outSAMattrRGs.empty()) attrStr(at, "RG", P.outSAMattrRGs[c.fileIndex]);
        const uint64_t a = c.seqOff[(uint64_t)i * c.nMates + imate], b = c.seqOff[(uint64_t)i * c.nMates + imate + 1];
        const size_t rec0 = bam.size();
        put32(bam, 0);
        put32(bam, 0xFFFFFFFFu);                                         // refID
        put32(bam, 0xFFFFFFFFu);                                         // pos
        put32(bam, (uint32_t)(reg2bin(-1, 0) << 16 | (uint32_t)(nameLen + 1)));
        put32(bam, (((flag & P.outSAMflagAND) | P.outSAMflagOR) << 16) | 0u);
        put32(bam, (uint32_t)(b - a));
        put32(bam, mateChr < idx.chrName.size() ? mateChr : 0xFFFFFFFFu);
        put32(bam, mateChr < idx.chrName.size() ? mateStart : 0xFFFFFFFFu);
        put32(bam, 0);
        bam.append(name, nameLen + 1);
        bamSeqQual(bam, c.seq.data() + a, c.qual.data() + a, b - a, c.fastq && P.outSAMmode != "NoQS");
        bam += at;
        bamFinish(bam, rec0);
    }
}

void OutputWriter::bamMapped(const ReadChunk& c, uint32_t i, const star_read_result_t& r, const star_align_t& tr, uint64_t nTrOut, uint64_t iTrOut,
                             std::string& bam, bool transcriptomic) const {
    // transcriptomic (ReadAlign_quantTranscriptome.cpp:72: alignBAM(..., trChrStart = 0, ..., outSAMattrOrderQuant)): tr.Chr is a transcript,
    // coordinates are transcript coordinates, attributes NH HI (+ RG, MC when requested)
    std::vector<int> quantAttr;
    if (transcriptomic) {
        quantAttr = {ATTR_NH, ATTR_HI};
        for (int code : P.outSAMattrOrder) if (code == ATTR_RG || code == ATTR_MC) quantAttr.push_back(code);
    }
    const std::vector<int>& attrOrder = transcriptomic ? quantAttr : P.outSAMattrOrder;
    const char* name = c.names.data() + c.nameOff[i];
    const size_t nameLen = strlen(name);
    const bool flagPaired = c.nMates == 2;
    const uint64_t Lread = r.Lread;
    uint64_t readLength[2];
    readLength[0] = c.len(i, 0);   // the lengths that were mapped (after clipping)
    readLength[1] = flagPaired ? c.len(i, 1) : 0;
    const uint64_t readLengthOriginal[2] = {c.lenOrig(i, 0), flagPaired ? c.lenOrig(i, 1) : 0};
    uint32_t iExMate;
    unsigned nMates = 1;
    for (iExMate = 0; iExMate + 1 < tr.nExons; iExMate++) {
        if (tr.canonSJ[iExMate] == -3) { nMates = 2; break; }
    }
    const unsigned Str = tr.Str;
    const unsigned leftMate = flagPaired ? Str : 0;
    const uint64_t chrStart = transcriptomic ? 0 : idx.chrStart[tr.Chr];
    // CIGARs of both mates first (MC needs the other mate's), packed and as text (ReadAlign_calcCIGAR.cpp:3-60)
    std::vector<uint32_t> packed[2];
    std::string cigarText[2];
    std::vector<char> sjMotif[2];
    std::vector<int32_t> sjIntron[2];
    uint32_t ex1[2] = {0, 0}, ex2[2] = {0, 0};
    unsigned mateOf[2] = {0, 0};
    for (unsigned imate = 0; imate < nMates; imate++) {
        const uint32_t iEx1 = (imate == 0 ? 0 : iExMate + 1), iEx2 = (imate == 0 ? iExMate : tr.nExons - 1);
        ex1[imate] = iEx1; ex2[imate] = iEx2;
        const unsigned Mate = tr.exFrag[iEx1];
        mateOf[imate] = Mate;
        auto op = [&](uint64_t len, unsigned code, char ch) { packed[imate].push_back((uint32_t)(len << 4 | code)); putU(cigarText[imate], len); cigarText[imate].push_back(ch); };
        const uint64_t trimL = (Str == 0) == (Mate == 0) ? c.c5(i, Mate) : c.c3(i, Mate);   // ReadAlign_alignBAM.cpp:222-233, 268-271
        const uint64_t trimL1 = trimL + (uint64_t)tr.exR[iEx1] - (tr.exR[iEx1] < readLength[leftMate] ? 0 : readLength[leftMate] + 1);
        if (trimL1 > 0) op(trimL1, 4, 'S');
        for (uint32_t ii = iEx1; ii <= iEx2; ii++) {
            if (ii > iEx1) {
                const uint64_t gapG = tr.exG[ii] - (tr.exG[ii - 1] + tr.exL[ii - 1]);
                const uint64_t gapR = (uint64_t)tr.exR[ii] - tr.exR[ii - 1] - tr.exL[ii - 1];
                if (gapR > 0) op(gapR, 1, 'I');
                if (tr.canonSJ[ii - 1] >= 0 || tr.sjAnnot[ii - 1] == 1) {
                    op(gapG, 3, 'N');
                    sjMotif[imate].push_back((char)(tr.canonSJ[ii - 1] + (tr.sjAnnot[ii - 1] == 0 ? 0 : 20)));
                    sjIntron[imate].push_back((int32_t)(tr.exG[ii - 1] + tr.exL[ii - 1] + 1 - chrStart));
                    sjIntron[imate].push_back((int32_t)(tr.exG[ii] - chrStart));
                } else if (gapG > 0) {
                    op(gapG, 2, 'D');
                }
            }
            if (tr.exL[ii] > 0) op(tr.exL[ii], 0, 'M');   // 0-length blocks are not recorded in BAM (:276)
        }
        if (sjMotif[imate].empty()) { sjMotif[imate].push_back(-1); sjIntron[imate].push_back(-1); }
        const uint64_t trimR1 = (tr.exR[iEx1] < readLength[leftMate] ? readLengthOriginal[leftMate] : readLength[leftMate] + 1 + readLengthOriginal[Mate]) - tr.exR[iEx2] - tr.exL[iEx2] - trimL;
        if (trimR1 > 0) op(trimR1, 4, 'S');
    }
    std::string rc, rq;
    for (unsigned imate = 0; imate < nMates; imate++) {
        const uint32_t iEx1 = ex1[imate], iEx2 = ex2[imate];
        const unsigned Mate = mateOf[imate];
        unsigned samFLAG = 0;
        if (flagPaired) {
            samFLAG = 0x0001;
            if (iExMate == tr.nExons - 1) samFLAG |= 0x0008;   // single mate: mateChr = (uint)-1 > nChrReal
            else samFLAG |= 0x0002;                             // (alignBAM marks every two-mate transcript as proper pair, :187-189)
        }
        if (c.readFilter[i] == 'Y') samFLAG |= 0x200;
        if (!tr.primaryFlag) samFLAG |= 0x100;
        if (Mate == 0) {
            samFLAG |= Str * 0x10;
            if (nMates == 2) samFLAG |= (1 - Str) * 0x20;
        } else {
            samFLAG |= (1 - Str) * 0x10;
            if (nMates == 2) samFLAG |= Str * 0x20;
        }
        if (flagPaired) samFLAG |= (Mate == 0 ? 0x0040 : 0x0080);
        int MAPQ = P.outSAMmapqUnique;
        if (nTrOut >= 5) MAPQ = 0; else if (nTrOut >= 3) MAPQ = 1; else if (nTrOut == 2) MAPQ = 3;
        // attributes
        uint64_t tagNM = 0;
        std::string tagMD;
        bool needNM = false;
        for (int code : attrOrder) if (code == ATTR_NM || code == ATTR_MD) needNM = true;
        if (needNM) {  // samAttrNM_MD, ReadAlign_alignBAM.cpp:9-45
            std::string R(Lread, (char)4);
            auto conv = [](char ch) -> char { switch (ch) { case 'A': case 'a': return 0; case 'C': case 'c': return 1; case 'G': case 'g': return 2; case 'T': case 't': return 3; default: return 4; } };
            for (uint64_t k = 0; k < readLength[0]; k++) R[k] = conv(c.base(i, 0, k));
            if (flagPaired) {
                R[readLength[0]] = STAR_MARK_FRAG_SPACER_BASE;
                for (uint64_t k = 0; k < readLength[1]; k++) { char ch = conv(c.base(i, 1, readLength[1] - 1 - k)); R[readLength[0] + 1 + k] = ch < 4 ? 3 - ch : ch; }
            }
            if (tr.roStr != 0) {
                std::string R2(Lread, (char)4);
                for (uint64_t k = 0; k < Lread; k++) { char ch = R[k]; R2[Lread - 1 - k] = ch < 4 ? 3 - ch : ch; }
                R.swap(R2);
            }
            static const char numToNT[6] = {'A', 'C', 'G', 'T', 'N', 'N'};
            uint64_t matchN = 0, nMM = 0, nI = 0, nD = 0;
            for (uint32_t iex = iEx1; iex <= iEx2; iex++) {
                for (uint64_t ii = 0; ii < tr.exL[iex]; ii++) {
                    const char r1 = R[ii + tr.exR[iex]];
                    const char g1 = (char)idx.view.G[ii + tr.exG[iex]];
                    if (r1 != g1 || r1 == 4 || g1 == 4) {
                        ++nMM;
                        tagMD += std::to_string(matchN);
                        tagMD.push_back(numToNT[(uint8_t)g1 < 6 ? (uint8_t)g1 : 5]);
                        matchN = 0;
                    } else {
                        matchN++;
                    }
                }
                if (iex < iEx2) {
                    if (tr.canonSJ[iex] < 0) nD += tr.exG[iex + 1] - (tr.exG[iex] + tr.exL[iex]);   // indels; junctions are not in the edit distance
                    nI += (uint64_t)tr.exR[iex + 1] - tr.exR[iex] - tr.exL[iex];
                    if (tr.canonSJ[iex] == -1) {
                        tagMD += std::to_string(matchN) + "^";
                        for (uint64_t ii = tr.exG[iex] + tr.exL[iex]; ii < tr.exG[iex + 1]; ii++) tagMD.push_back(numToNT[idx.view.G[ii] < 6 ? idx.view.G[ii] : 5]);
                        matchN = 0;
                    }
                }
            }
            tagMD += std::to_string(matchN);
            tagNM = nMM + nI + nD;
        }
        std::string at;
        for (int code : attrOrder) {
            switch (code) {
                case ATTR_NH: attrInt(at, "NH", (long long)nTrOut); break;
                case ATTR_HI: attrInt(at, "HI", (long long)(iTrOut + P.outSAMattrIHstart)); break;
                case ATTR_AS: attrInt(at, "AS", tr.maxScore); break;
                case ATTR_nM: attrInt(at, "nM", (long long)tr.nMM); break;
                case ATTR_jM: {
                    at += "jMBc"; put32(at, (uint32_t)sjMotif[imate].size()); at.append(sjMotif[imate].data(), sjMotif[imate].size());
                    break;
                }
                case ATTR_jI: {
                    at += "jIBi"; put32(at, (uint32_t)sjIntron[imate].size()); at.append((const char*)sjIntron[imate].data(), 4 * sjIntron[imate].size());
                    break;
                }
                case ATTR_XS:
                    if (tr.sjMotifStrand == 1) attrChar(at, "XS", '+');
                    else if (tr.sjMotifStrand == 2) attrChar(at, "XS", '-');
                    break;
                case ATTR_NM: attrInt(at, "NM", (long long)tagNM); break;
                case ATTR_MD: attrStr(at, "MD", tagMD); break;
                case ATTR_RG: attrStr(at, "RG", P.outSAMattrRGs[c.fileIndex]); break;
                case ATTR_MC: if (nMates > 1) attrStr(at, "MC", cigarText[1 - imate]); break;
                default: break;   // ch: chimeric alignments only
            }
        }
        // sequence / qualities in alignment orientation
        const uint64_t a = c.seqOff[(uint64_t)i * c.nMates + Mate], b = c.seqOff[(uint64_t)i * c.nMates + Mate + 1];
        const char* seqOut = c.seq.data() + a;
        const char* qualOut = c.qual.data() + a;
        if (Mate != Str) {
            revComplement(c.seq.data() + a, b - a, rc);
            rq.assign(b - a, 'A');
            if (c.fastq) for (uint64_t k = 0; k < b - a; k++) rq[k] = c.qual[b - 1 - k];
            seqOut = rc.data(); qualOut = rq.data();
        }
        const uint64_t gBeg = tr.exG[iEx1] - chrStart, gEnd = tr.exG[iEx2] + tr.exL[iEx2] - chrStart;
        const size_t rec0 = bam.size();
        put32(bam, 0);
        put32(bam, tr.Chr);
        put32(bam, (uint32_t)gBeg);
        put32(bam, (uint32_t)(reg2bin((int)gBeg, (int)gEnd) << 16) | (uint32_t)(MAPQ << 8) | (uint32_t)(nameLen + 1));
        put32(bam, (((samFLAG & P.outSAMflagAND) | P.outSAMflagOR) << 16) | (uint32_t)packed[imate].size());
        put32(bam, (uint32_t)(b - a));
        if (nMates > 1) {
            put32(bam, tr.Chr);
            put32(bam, (uint32_t)(tr.exG[(imate == 0 ? iExMate + 1 : 0)] - chrStart));
            if (P.outSAMtlen == 2) {   // ReadAlign_alignBAM.cpp:84-88, 571-573
                const uint64_t hi = std::max(tr.exG[tr.nExons - 1] + tr.exL[tr.nExons - 1], tr.exG[iExMate] + tr.exL[iExMate]), lo = std::min(tr.exG[0], tr.exG[iExMate + 1]);
                const int32_t tlen = (int32_t)(hi - lo);
                const unsigned leftMostMate = tr.exG[0] <= tr.exG[iExMate + 1] ? 0 : 1;
                put32(bam, (uint32_t)(imate == leftMostMate ? tlen : -tlen));
            } else {
                const int32_t tlen = (int32_t)(tr.exG[tr.nExons - 1] + tr.exL[tr.nExons - 1] - tr.exG[0]);
                put32(bam, (uint32_t)(imate == 0 ? tlen : -tlen));
            }
        } else {
            put32(bam, 0xFFFFFFFFu); put32(bam, 0xFFFFFFFFu); put32(bam, 0);
        }
        bam.append(name, nameLen + 1);
        bam.append((const char*)packed[imate].data(), 4 * packed[imate].size());
        bamSeqQual(bam, seqOut, qualOut, b - a, c.fastq && P.outSAMmode != "NoQS");
        bam += at;
        bamFinish(bam, rec0);
    }
}

std::string OutputWriter::bamHeader(bool sortedCoord) const {  // BAMfunctions.cpp:77-92
    std::string h = "BAM\001";
    std::string text = samHeader(sortedCoord);   // samHeaderSortedCoord, samHeaders.cpp:99
    put32(h, (uint32_t)text.size());
    h += text;
    put32(h, (uint32_t)idx.chrName.size());
    for (size_t ii = 0; ii < idx.chrName.size(); ii++) {
        put32(h, (uint32_t)(idx.chrName[ii].size() + 1));
        h.append(idx.chrName[ii].c_str(), idx.chrName[ii].size() + 1);
        put32(h, (uint32_t)idx.chrLength[ii]);
    }
    return h;
}

// BGZF: gzip members with the 'BC' extra field holding the block size; payload <= 0xff00 bytes so that a block always fits 64 KB
void OutputWriter::bgzfCompress(const char* data, size_t n, int level, std::string& out) {
    const size_t BLOCK = 0xff00;
    std::vector<unsigned char> buf(0x10000 + 1024);
    for (size_t off = 0; off < n || (n == 0 && off == 0); off += BLOCK) {
        if (n == 0) break;
        const size_t len = std::min(BLOCK, n - off);
        z_stream zs;
        memset(&zs, 0, sizeof(zs));
        deflateInit2(&zs, level, Z_DEFLATED, -15, 8, Z_DEFAULT_STRATEGY);
        zs.next_in = (Bytef*)(data + off); zs.avail_in = (uInt)len;
        zs.next_out = buf.data(); zs.avail_out = (uInt)buf.size();
        deflate(&zs, Z_FINISH);
        const size_t clen = zs.total_out;
        deflateEnd(&zs);
        const uint32_t crc = (uint32_t)crc32(crc32(0L, Z_NULL, 0), (const Bytef*)(data + off), (uInt)len);
        const uint16_t bsize = (uint16_t)(clen + 25);   // total block size - 1 (18 header + clen + 8 trailer - 1)
        static const unsigned char hdr[16] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 'B', 'C', 2, 0};
        out.append((const char*)hdr, 16);
        out.append((const char*)&bsize, 2);
        out.append((const char*)buf.data(), clen);
        out.append((const char*)&crc, 4);
        const uint32_t isize = (uint32_t)len;
        out.append((const char*)&isize, 4);
    }
}

const char* OutputWriter::bgzfEofBlock(size_t& n) {
    static const unsigned char eof[28] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 'B', 'C', 2, 0, 0x1b, 0, 3, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    n = 28;
    return (const char*)eof;
}

// ReadAlign_oneRead.cpp:74-75, ReadAlign_mappedFilter.cpp, ReadAlign_outputAlignments.cpp:18-90,133-260
void OutputWriter::formatReads(const ReadChunk& c, const star_align_batch_t& out, uint32_t lo, uint32_t hi, std::string& sam,
                               std::vector<Junction>& sj, Stats& st, std::string* coord, std::vector<uint64_t>* coordKey, BySJoutHold* by, std::string* unm, GeneCounts* gc, std::string* trBam, const double* trDraw) const {
    const bool samYes = !(P.outSAMtype[0] == "None" || P.outSAMmode == "None");
    const bool coordYes = samYes && P.outBAMcoord && coord && coordKey;
    // records appended to `dst` since `from` also go to the coordinate-sorted set with read-order key `key` (one key per record)
    auto toCoord = [&](const std::string& dst, size_t from, uint64_t key) {
        size_t o = from;
        while (o < dst.size()) {
            uint32_t bs; memcpy(&bs, dst.data() + o, 4);
            coord->append(dst, o, 4 + (size_t)bs);
            coordKey->push_back(key);
            o += 4 + (size_t)bs;
        }
    };
    std::string scratch;
    std::vector<star_align_t> keptTr;   // --outSAMfilter KeepAllAddedReferences: the alignments written
    star_align_t bestCopy;
    for (uint32_t i = lo; i < hi; i++) {
        const star_read_result_t& r = out.reads[i];
        uint64_t L0 = c.lenTrue(i, 0);   // readLength after clipping (ReadAlign_oneRead.cpp: statsRA.readBases)
        uint64_t L1 = c.nMates == 2 ? c.lenTrue(i, 1) : 0;
        if (by && r.unmapType < 0) {   // ReadAlign::outFilterBySJout (ReadAlign_outputAlignments.cpp:90-130), 1st stage of --outFilterType BySJout
            const star_align_t* tr1 = out.aligns + r.trOffset;
            const bool pass = !heldBySJout(out, i);
            if (P.outSJyes && (P.outSJfilterReads == "All" || r.nTrOut == 1)) {   // the junctions of ALL reads decide which novel ones survive
                size_t s0 = by->sjAll.size();
                for (uint64_t k = 0; k < r.nTrOut; k++) recordSJ(tr1[k], r.nTrOut, by->sjAll, s0);
            }
            if (!pass) { by->held.push_back(i); continue; }   // not counted, not written: mapped again in the 2nd stage
        }
        st.readN++;
        st.readBases += L0 + L1;
        int unmapType = r.unmapType;
        bool mateMappedOut[2] = {false, false};
        switch (unmapType) { case 0: st.unmappedOther++; break; case 1: st.unmappedShort++; break; case 2: st.unmappedMismatch++; break; case 3: st.unmappedMulti++; break; default: break; }
        const star_align_t* trs = out.aligns + r.trOffset;
        if (unmapType < 0) {
            uint64_t nTr = r.nTrOut;
            if (nTr > 1) {
                st.mappedReadsM++;
            } else if (nTr == 1) {
                st.mappedReadsU++;
                const star_align_t& T = trs[0];  // Stats::transcriptStats Stats.cpp:35-56
                st.mappedMismatchesN += T.nMM; st.mappedInsN += T.nIns; st.mappedDelN += T.nDel; st.mappedInsL += T.lIns; st.mappedDelL += T.lDel;
                if (T.nExons > 0) {
                    uint64_t mappedL = 0;
                    for (uint32_t ii = 0; ii < T.nExons; ii++) mappedL += T.exL[ii];
                    for (uint32_t ii = 0; ii + 1 < T.nExons; ii++) {
                        if (T.canonSJ[ii] >= 0) st.splicesN[T.canonSJ[ii]]++;
                        if (T.sjAnnot[ii] == 1) st.splicesNsjdb++;
                    }
                    st.mappedBases += mappedL;
                }
            }
            if (gc && geneModel) gc->addAlign(*geneModel, nTr, trs);   // ReadAlign::alignedAnnotation :296-308
            if (trBam && trModel) quantTranscriptome(c, i, r, trs, nTr, trDraw ? trDraw[i] : 0.0, *trBam);   // ReadAlign_outputAlignments.cpp:50-57
            if (P.outSJyes && (P.outSJfilterReads == "All" || nTr == 1)) {  // recordSJ :76-87
                size_t sjReadStartN = sj.size();
                for (uint64_t k = 0; k < nTr; k++) recordSJ(trs[k], nTr, sj, sjReadStartN);
            }
            // writeSAM :133-230
            const star_align_t* trsAll = trs;
            const star_align_t* bestP = &trsAll[r.bestTr];
            if (P.outSAMfilterKeepOnly || P.outSAMfilterKeepAll) {   // --outSAMfilter :140-164, after the counters, junctions and quantifications
                if (P.outSAMfilterKeepOnly) {   // an alignment on an old reference: nothing at all is written (unmapType stays < 0)
                    bool old = false;
                    for (uint64_t k = 0; k < nTr; k++) old = old || trs[k].Chr < idx.insertChrFirst;
                    if (old) continue;
                } else {   // only the alignments on added references; the first of them is primary; NH / HI / MAPQ count these
                    keptTr.clear();
                    int64_t bestKept = -1;
                    for (uint64_t k = 0; k < nTr; k++)
                        if (trs[k].Chr >= idx.insertChrFirst) {
                            if (k == r.bestTr) bestKept = (int64_t)keptTr.size();
                            keptTr.push_back(trs[k]);
                            keptTr.back().primaryFlag = 0;
                        }
                    if (keptTr.empty()) continue;
                    keptTr[0].primaryFlag = 1;
                    // the best alignment (whose mates decide the unmapped-mate record) is not filtered, but it is the same object as its copy in
                    // the list, so it carries the primary flag the filter gave that copy
                    bestCopy = trsAll[r.bestTr];
                    if (bestKept >= 0) bestCopy.primaryFlag = keptTr[bestKept].primaryFlag;
                    bestP = &bestCopy;
                    trs = keptTr.data();
                    nTr = keptTr.size();
                }
            }
            bool mateMapped[2] = {false, false};
            uint64_t nWrite = std::min<uint64_t>(P.hp.outSAMmultNmax, nTr);
            for (uint64_t k = 0; k < nWrite; k++) {
                bool mm1[2] = {false, false};
                mm1[trs[k].exFrag[0]] = true;
                mm1[trs[k].exFrag[trs[k].nExons - 1]] = true;
                if (samYes && P.outSAMtype[0] == "SAM") {
                    samMapped(c, i, r, trs[k], nTr, k, sam);
                    if (P.unmappedKeepPairs && c.nMates > 1 && (!mm1[0] || !mm1[1])) samUnmapped(c, i, r, &trs[k], 4, mm1, sam);
                } else if (samYes) {   // ReadAlign_outputAlignments.cpp:183-203
                    std::string& dst = P.outBAMunsorted ? sam : scratch;
                    if (!P.outBAMunsorted) scratch.clear();
                    const size_t from = dst.size();
                    bamMapped(c, i, r, trs[k], nTr, k, dst);
                    if (coordYes) toCoord(dst, from, (c.iReadAll[i] << 32) | (k << 8) | trs[k].exFrag[0]);
                    if (P.outBAMunsorted && P.unmappedKeepPairs && c.nMates > 1 && (!mm1[0] || !mm1[1])) bamUnmapped(c, i, r, &trs[k], 4, mm1, sam);   // (unsorted stream only)
                }
            }
            const star_align_t& best = *bestP;
            mateMapped[best.exFrag[0]] = true;
            mateMapped[best.exFrag[best.nExons - 1]] = true;
            if (c.nMates > 1 && !(mateMapped[0] && mateMapped[1])) unmapType = 4;
            mateMappedOut[0] = mateMapped[0]; mateMappedOut[1] = mateMapped[1];
            if (unmapType == 4 && P.unmappedWithin && samYes) {   // :214-232 (KeepPairs does not affect the sorted BAM)
                if (P.outSAMtype[0] == "SAM") { if (!P.unmappedKeepPairs) samUnmapped(c, i, r, &best, 4, mateMapped, sam); }
                else {
                    scratch.clear();
                    bamUnmapped(c, i, r, &best, 4, mateMapped, scratch);
                    if (P.outBAMunsorted && !P.unmappedKeepPairs) sam += scratch;
                    if (coordYes) toCoord(scratch, 0, c.iReadAll[i] << 32);
                }
            }
        } else if (P.unmappedWithin && (samYes || trBam)) {
            bool mateMapped[2] = {false, false};
            if (samYes && P.outSAMtype[0] == "SAM") samUnmapped(c, i, r, nullptr, unmapType, mateMapped, sam);
            if ((samYes && P.outSAMtype[0] != "SAM") || trBam) {   // :236-248: the unmapped record also goes to Aligned.toTranscriptome.out.bam
                scratch.clear();
                bamUnmapped(c, i, r, nullptr, unmapType, mateMapped, scratch);
                if (samYes && P.outBAMunsorted) sam += scratch;
                if (trBam) *trBam += scratch;
                if (coordYes) toCoord(scratch, 0, c.iReadAll[i] << 32);
            }
        }
        if (unmapType >= 0) {
            st.unmappedAll++;
            if (unm) {   // ReadAlign::outReadsUnmapped (ReadAlign_outputAlignments.cpp:259-274): unmapped reads and pairs with one mapped mate
                for (uint32_t m = 0; m < c.nMates; m++) {
                    std::string& u = unm[m];
                    u += c.namesFull.c_str() + c.nameFullOff[i];
                    u.push_back(' '); u.push_back((char)('0' + m)); u.push_back(':'); u.push_back(c.readFilter[i]); u += ": ";
                    if (c.nMates > 1) { u.push_back(' '); u.push_back(mateMappedOut[0] ? '1' : '0'); u.push_back(mateMappedOut[1] ? '1' : '0'); }
                    u.push_back('\n');
                    const uint64_t a = c.seqOff[(uint64_t)i * c.nMates + m], b = c.seqOff[(uint64_t)i * c.nMates + m + 1];
                    u.append(c.seq, a, b - a); u.push_back('\n');
                    if (c.fastq) { u += "+\n"; u.append(c.qual, a, b - a); u.push_back('\n'); }
                }
            }
        }
    }
}

std::string OutputWriter::samHeader(bool sortedCoord) const {  // samHeaders.cpp:27-113
    std::ostringstream h;
    if (P.outSAMheaderHD[0] != "-") { for (size_t ii = 0; ii < P.outSAMheaderHD.size(); ii++) h << (ii ? "\t" : "") << P.outSAMheaderHD[ii]; }
    else h << "@HD\tVN:1.4";
    if (sortedCoord) h << "\tSO:coordinate";   // (appended to a user-given @HD line too, as the reference does)
    h << "\n";
    for (size_t ii = 0; ii < idx.chrName.size(); ii++) h << "@SQ\tSN:" << idx.chrName[ii] << "\tLN:" << idx.chrLength[ii] << "\n";
    if (P.outSAMheaderPG[0] != "-") { for (size_t ii = 0; ii < P.outSAMheaderPG.size(); ii++) h << (ii ? "\t" : "") << P.outSAMheaderPG[ii]; h << "\n"; }
    h << "@PG\tID:STAR\tPN:STAR\tVN:2.7.11b\tCL:" << P.commandLineFull << "\n";
    if (P.outSAMheaderCommentFile != "-") {
        std::ifstream com(P.outSAMheaderCommentFile);
        std::string line1;
        while (std::getline(com, line1)) if (line1.find_first_not_of(" \t\n\v\f\r") != std::string::npos) h << line1 << "\n";
    }
    for (auto& l : P.outSAMattrRGlineSplit) h << "@RG\t" << l << "\n";   // samHeaders.cpp:83-85
    h << "@CO\tuser command line: " << P.commandLine << "\n";
    return h.str();
}

void OutputWriter::collapseSJ(std::vector<Junction>& v, std::string& err) {  // OutSJ.cpp:34-62,89-125
    if (v.empty()) return;
    std::sort(v.begin(), v.end(), [](const Junction& a, const Junction& b) { return a.start != b.start ? a.start < b.start : a.gap < b.gap; });
    size_t k = 0;
    for (size_t i = 1; i < v.size(); i++) {
        if (v[i].start == v[k].start && v[i].gap == v[k].gap) {
            v[k].countUnique += v[i].countUnique;
            v[k].countMultiple += v[i].countMultiple;
            if (v[k].overhangLeft < v[i].overhangLeft) v[k].overhangLeft = v[i].overhangLeft;
            if (v[k].overhangRight < v[i].overhangRight) v[k].overhangRight = v[i].overhangRight;
            if (v[k].motif != v[i].motif) err = "EXITING because of BUG: different motifs for the same junction while collapsing junctions\n";
            if (v[k].annot < v[i].annot) err = "EXITING because  of BUG: different annotation status for the same junction while collapsing junctions:\n";
        } else {
            v[++k] = v[i];
        }
    }
    v.resize(k + 1);
}

// outputSJ.cpp:20-124: collapse, the count / overhang / intron-size filters (kept), then the distance-to-neighbour filters (sjFilter);
// distFilter = false is the 2nd stage of --outFilterType BySJout, where every kept junction is written (outputSJ.cpp:86, 130)
static std::string filterSJ(const HostParams& P, std::vector<Junction>& all, std::vector<Junction>& kept, std::vector<char>& sjFilter, bool distFilter) {
    std::string err;
    OutputWriter::collapseSJ(all, err);
    if (!err.empty()) return err;
    kept.clear();
    for (auto& j : all) {
        int mi = (j.motif + 1) / 2;
        uint32_t tot = j.countMultiple + j.countUnique;
        bool f = j.annot > 0 ||
                 ((j.countUnique >= (uint32_t)P.outSJfilterCountUniqueMin[mi] || tot >= (uint32_t)P.outSJfilterCountTotalMin[mi]) &&
                  j.overhangLeft >= (uint32_t)P.outSJfilterOverhangMin[mi] && j.overhangRight >= (uint32_t)P.outSJfilterOverhangMin[mi] &&
                  (tot > P.outSJfilterIntronMaxVsReadN.size() || j.gap <= (uint32_t)P.outSJfilterIntronMaxVsReadN[tot - 1]));
        if (f) kept.push_back(j);
    }
    size_t N = kept.size();
    sjFilter.assign(N, distFilter ? 0 : 1);
    if (!distFilter) return std::string();
    std::vector<uint64_t> sjA(N * 3);
    for (size_t ii = 0; ii < N; ii++) {
        uint64_t x1 = 0, x2 = (uint64_t)-1;
        if (ii > 0) x1 = kept[ii - 1].start;
        if (ii + 1 < N) x2 = kept[ii + 1].start;
        uint64_t minDist = std::min(kept[ii].start - x1, x2 - kept[ii].start);
        sjFilter[ii] = minDist >= (uint64_t)P.outSJfilterDistToOtherSJmin[(kept[ii].motif + 1) / 2];
        sjA[ii * 3] = kept[ii].start + (uint64_t)kept[ii].gap;
        sjA[ii * 3 + 1] = ii;
        sjA[ii * 3 + 2] = kept[ii].annot == 0 ? (uint64_t)kept[ii].motif : STAR_SJ_MOTIF_SIZE + 1;
    }
    std::vector<size_t> ord(N);
    for (size_t i = 0; i < N; i++) ord[i] = i;
    std::stable_sort(ord.begin(), ord.end(), [&](size_t a, size_t b) { return sjA[a * 3] < sjA[b * 3]; });
    for (size_t oi = 0; oi < N; oi++) {
        size_t ii = ord[oi];
        if (sjA[ii * 3 + 2] == STAR_SJ_MOTIF_SIZE + 1) {
            sjFilter[sjA[ii * 3 + 1]] = 1;
        } else {
            uint64_t x1 = 0, x2 = (uint64_t)-1;
            if (oi > 0) x1 = sjA[ord[oi - 1] * 3];
            if (oi + 1 < N) x2 = sjA[ord[oi + 1] * 3];
            uint64_t minDist = std::min(sjA[ii * 3] - x1, x2 - sjA[ii * 3]);
            sjFilter[sjA[ii * 3 + 1]] = sjFilter[sjA[ii * 3 + 1]] && (minDist >= (uint64_t)P.outSJfilterDistToOtherSJmin[(sjA[ii * 3 + 2] + 1) / 2]);
        }
    }
    return std::string();
}

std::string OutputWriter::writeSJ(std::vector<Junction>& all, const std::string& path, bool distFilter) const {  // outputSJ.cpp:20-165
    std::vector<Junction> kept;
    std::vector<char> sjFilter;
    std::string err = filterSJ(P, all, kept, sjFilter, distFilter);
    if (!err.empty()) return err;
    const size_t N = kept.size();
    std::string txt;
    for (size_t ii = 0; ii < N; ii++) {
        if (!sjFilter[ii]) continue;
        const Junction& j = kept[ii];  // Junction::outputStream OutSJ.cpp:85-90
        uint64_t sjChr = idx.chrBin[j.start >> idx.view.gChrBinNbits];
        txt += idx.chrName.at(sjChr); txt.push_back('\t'); putU(txt, j.start + 1 - idx.chrStart[sjChr]); txt.push_back('\t');
        putU(txt, j.start + j.gap - idx.chrStart[sjChr]); txt.push_back('\t'); putI(txt, (int)j.strand); txt.push_back('\t'); putI(txt, (int)j.motif);
        txt.push_back('\t'); putI(txt, (int)j.annot); txt.push_back('\t'); putU(txt, j.countUnique); txt.push_back('\t'); putU(txt, j.countMultiple);
        txt.push_back('\t'); putU(txt, j.overhangLeft); txt.push_back('\n');
    }
    std::ofstream o(path);
    o << txt;
    return std::string();
}

// 1st stage of --outFilterType BySJout (outputSJ.cpp:139-160): the unannotated junctions of ALL reads that pass every filter, as
// (first, last) intron base, in collapsed (start, gap) order
std::string OutputWriter::novelJunctions(std::vector<Junction>& all, std::vector<uint64_t>& sjStart, std::vector<uint64_t>& sjEnd) const {
    std::vector<Junction> kept;
    std::vector<char> sjFilter;
    std::string err = filterSJ(P, all, kept, sjFilter, true);
    if (!err.empty()) return err;
    sjStart.clear(); sjEnd.clear();
    for (size_t ii = 0; ii < kept.size(); ii++)
        if (sjFilter[ii] && kept[ii].annot == 0) { sjStart.push_back(kept[ii].start); sjEnd.push_back(kept[ii].start + (uint64_t)kept[ii].gap - 1); }
    return std::string();
}

bool OutputWriter::heldBySJout(const star_align_batch_t& out, uint32_t i) {
    const star_read_result_t& r = out.reads[i];
    if (r.unmapType >= 0) return false;
    const star_align_t* tr1 = out.aligns + r.trOffset;
    for (uint64_t k = 0; k < r.nTrOut; k++)
        for (uint32_t iex = 0; iex + 1 < tr1[k].nExons; iex++)
            if (tr1[k].canonSJ[iex] >= 0 && tr1[k].sjAnnot[iex] == 0) return true;
    return false;
}

// ---- --quantMode TranscriptomeSAM ----------------------------------------------------------------------------------------------------
int TranscriptModel::load(const std::string& dir, std::string& err) {   // Transcriptome.cpp:32-75
    const char* sol = "SOLUTION: utilize --sjdbGTFfile /path/to/annotantions.gtf option at the genome generation step or mapping step\n";
    std::ifstream tr(dir + "/transcriptInfo.tab");
    if (tr.fail()) { err = "EXITING because of fatal INPUT error: could not open input file " + dir + "/transcriptInfo.tab\n" + sol; return STAR_EXIT_INPUT_FILES; }
    uint64_t nTr = 0;
    tr >> nTr;
    trS.resize(nTr); trE.resize(nTr); trEmax.resize(nTr); trExI.resize(nTr); trExN.resize(nTr); trStr.resize(nTr); trID.resize(nTr); trLen.resize(nTr);
    for (uint64_t i = 0; i < nTr; i++) {
        uint32_t str1, gene;
        tr >> trID[i] >> trS[i] >> trE[i] >> trEmax[i] >> str1 >> trExN[i] >> trExI[i] >> gene;
        trStr[i] = (uint8_t)str1;
        if (!tr.good()) { err = "EXITING because of FATAL GENOME INDEX FILE error: transcriptInfo.tab is corrupt, or is incompatible with the current STAR version\nSOLUTION: re-generate genome index"; return STAR_EXIT_GENOME_FILES; }
    }
    std::ifstream ex(dir + "/exonInfo.tab");
    if (ex.fail()) { err = "EXITING because of fatal INPUT error: could not open input file " + dir + "/exonInfo.tab\n" + sol; return STAR_EXIT_INPUT_FILES; }
    uint64_t nEx = 0;
    ex >> nEx;
    exSE.resize(2 * nEx); exLenCum.resize(nEx);
    for (uint64_t i = 0; i < nEx; i++) ex >> exSE[2 * i] >> exSE[2 * i + 1] >> exLenCum[i];
    for (uint64_t i = 0; i < nTr; i++) { const uint32_t l = trExI[i] + trExN[i] - 1; trLen[i] = exLenCum[l] + exSE[2 * l + 1] - exSE[2 * l] + 1; }
    return 0;
}

namespace {
uint32_t bsearch1(uint32_t x, const uint32_t* X, uint32_t N) {   // binarySearch1, serviceFuns.cpp:192-209: last element <= x, (uint32)-1 outside the range
    if (x > X[N - 1] || x < X[0]) return (uint32_t)-1;
    uint32_t i1 = 0, i2 = N - 1;
    while (i2 > i1 + 1) { const uint32_t i3 = (i1 + i2) / 2; if (X[i3] > x) i2 = i3; else i1 = i3; }
    while (i1 < N - 1 && x == X[i1 + 1]) ++i1;
    return i1;
}
// alignToTranscript, Transcriptome_quantAlign.cpp:5-92
int alignToTranscript(star_align_t aG, uint64_t Lread, uint64_t trS1, uint8_t trStr1, const uint32_t* exSE1, const uint32_t* exLenCum1, uint16_t exN1, star_align_t& aT) {
    const uint32_t g1 = (uint32_t)(aG.exG[0] - trS1);
    uint32_t ex1 = bsearch1(g1, exSE1, 2 * (uint32_t)exN1);
    if (ex1 >= 2 * (uint32_t)exN1) return 0;
    if (ex1 % 2 == 1) { if (exSE1[ex1] == g1) --ex1; else return 0; }
    ex1 /= 2;
    aT.nExons = 0;
    aT.primaryFlag = 0;
    const int LAST = -99;
    aG.canonSJ[aG.nExons - 1] = LAST;
    for (uint32_t iab = 0; iab < aG.nExons; iab++) {
        if (aG.exG[iab] + aG.exL[iab] > (uint64_t)exSE1[2 * ex1 + 1] + trS1 + 1) return 0;   // block runs past the exon
        if (iab == 0 || aG.canonSJ[iab - 1] < 0) {
            aT.exR[aT.nExons] = aG.exR[iab];
            aT.exG[aT.nExons] = aG.exG[iab] - trS1 - exSE1[2 * ex1] + exLenCum1[ex1];
            aT.exL[aT.nExons] = aG.exL[iab];
            aT.exFrag[aT.nExons] = aG.exFrag[iab];
            if (aT.nExons > 0) aT.canonSJ[aT.nExons - 1] = aG.canonSJ[iab - 1];
            ++aT.nExons;
        } else aT.exL[aT.nExons - 1] = (uint16_t)(aT.exL[aT.nExons - 1] + aG.exL[iab]);
        switch (aG.canonSJ[iab]) {
            case LAST:
                if (trStr1 == 2) {   // transcript on the - strand: mirror the coordinates
                    const uint32_t trlength = exLenCum1[exN1 - 1] + exSE1[2 * exN1 - 1] - exSE1[2 * exN1 - 2] + 1;
                    for (uint32_t iex = 0; iex < aT.nExons; iex++) {
                        aT.exR[iex] = (uint16_t)(Lread - (aT.exR[iex] + aT.exL[iex]));
                        aT.exG[iex] = trlength - (aT.exG[iex] + aT.exL[iex]);
                    }
                    for (uint32_t iex = 0; iex < aT.nExons / 2; iex++) {
                        std::swap(aT.exR[iex], aT.exR[aT.nExons - 1 - iex]); std::swap(aT.exG[iex], aT.exG[aT.nExons - 1 - iex]);
                        std::swap(aT.exL[iex], aT.exL[aT.nExons - 1 - iex]); std::swap(aT.exFrag[iex], aT.exFrag[aT.nExons - 1 - iex]);
                    }
                    for (uint32_t iex = 0; iex < (aT.nExons - 1) / 2; iex++) std::swap(aT.canonSJ[iex], aT.canonSJ[aT.nExons - 2 - iex]);
                }
                for (uint32_t iex = 0; iex < aT.nExons; iex++) { aT.sjAnnot[iex] = 0; aT.shiftSJ[iex][0] = 0; aT.shiftSJ[iex][1] = 0; aT.sjStr[iex] = 0; }
                return 1;
            case -3:   // mate connection
                ex1 = bsearch1((uint32_t)(aG.exG[iab + 1] - trS1), exSE1, 2 * (uint32_t)exN1);
                if (ex1 % 2 == 1) return 0;
                ex1 /= 2;
                break;
            case -2: case -1: break;   // insertion, deletion
            default:   // junction: has to be the transcript's
                if (aG.exG[iab] + aG.exL[iab] == (uint64_t)exSE1[2 * ex1 + 1] + trS1 + 1 && aG.exG[iab + 1] == (uint64_t)exSE1[2 * (ex1 + 1)] + trS1) ++ex1;
                else return 0;
        }
    }
    return 0;
}
}  // namespace

uint32_t TranscriptModel::quantAlign(const star_align_t& aG, uint64_t Lread, std::vector<star_align_t>& out) const {
    const int64_t nTr = (int64_t)trS.size();
    if (nTr == 0) return 0;
    const uint64_t g0 = aG.exG[0];
    int64_t tr1;   // binarySearch1a: last transcript start <= align start
    if (g0 > trS[nTr - 1]) tr1 = nTr - 1;
    else if (g0 < trS[0]) return 0;
    else {
        int64_t i1 = 0, i2 = nTr - 1;
        while (i2 > i1 + 1) { const int64_t i3 = (i1 + i2) / 2; if (trS[i3] > g0) i2 = i3; else i1 = i3; }
        while (i1 < nTr - 1 && g0 == trS[i1 + 1]) ++i1;
        tr1 = i1;
    }
    const uint64_t aGend = aG.exG[aG.nExons - 1];
    uint32_t n = 0;
    ++tr1;
    do {
        --tr1;
        if (aGend <= trE[tr1]) {
            star_align_t aT = aG;   // the scalars (maxScore, nMM, ...) of the genomic alignment stay
            if (alignToTranscript(aG, Lread, trS[tr1], trStr[tr1], exSE.data() + 2 * trExI[tr1], exLenCum.data() + trExI[tr1], trExN[tr1], aT) == 1) {
                aT.Chr = (uint32_t)tr1;
                aT.Str = trStr[tr1] == 1 ? aG.Str : 1 - aG.Str;
                out.push_back(aT);
                ++n;
            }
        }
    } while (trEmax[tr1] >= aGend && tr1 > 0);
    return n;
}

// ReadAlign::quantTranscriptome, ReadAlign_quantTranscriptome.cpp:7-91.  draw = this read's number of the run's random stream (uniform in [0,1))
void OutputWriter::quantTranscriptome(const ReadChunk& c, uint32_t i, const star_read_result_t& r, const star_align_t* trs, uint64_t nTr, double draw, std::string& bam) const {
    std::vector<star_align_t> alignT;
    const uint64_t Lread = r.Lread;
    uint64_t readLength[2];
    readLength[0] = c.len(i, 0);
    readLength[1] = c.nMates == 2 ? c.len(i, 1) : 0;
    std::string R;   // Read1[0]: mate 1, spacer, reverse complement of mate 2 (numeric); reversed-complemented for roStr = 1
    for (uint64_t iag = 0; iag < nTr; iag++) {
        const star_align_t* a1 = &trs[iag];
        if (!P.quantTrIndel && (a1->nDel > 0 || a1->nIns > 0)) continue;
        if (!P.quantTrSingleEnd && c.nMates == 2 && a1->exFrag[0] == a1->exFrag[a1->nExons - 1]) continue;
        star_align_t a2;
        if (!P.quantTrSoftClip) {   // soft clips are extended to the read ends if the mismatches allow it
            if (R.empty()) {
                auto conv = [](char ch) -> char { switch (ch) { case 'A': case 'a': return 0; case 'C': case 'c': return 1; case 'G': case 'g': return 2; case 'T': case 't': return 3; default: return 4; } };
                R.assign(Lread, (char)4);
                for (uint64_t k = 0; k < readLength[0]; k++) R[k] = conv(c.base(i, 0, k));
                if (c.nMates == 2) {
                    R[readLength[0]] = STAR_MARK_FRAG_SPACER_BASE;
                    for (uint64_t k = 0; k < readLength[1]; k++) { char ch = conv(c.base(i, 1, readLength[1] - 1 - k)); R[readLength[0] + 1 + k] = ch < 4 ? 3 - ch : ch; }
                }
            }
            std::string Rr;
            const std::string* Rp = &R;
            if (a1->roStr != 0) {
                Rr.assign(Lread, (char)4);
                for (uint64_t k = 0; k < Lread; k++) { char ch = R[k]; Rr[Lread - 1 - k] = ch < 4 ? 3 - ch : ch; }
                Rp = &Rr;
            }
            a2 = *a1;
            uint64_t nMM1 = 0;
            for (uint32_t iab = 0; iab < a2.nExons; iab++) {
                uint64_t left1 = 0, right1 = 0;
                if (iab == 0) left1 = a2.exR[iab];
                else if (a2.canonSJ[iab - 1] == -3) left1 = a2.exR[iab] - readLength[a2.exFrag[iab - 1]] - 1;
                if (iab == a2.nExons - 1) right1 = Lread - a2.exR[iab] - a2.exL[iab];
                else if (a2.canonSJ[iab] == -3) right1 = readLength[a2.exFrag[iab]] - a2.exR[iab] - a2.exL[iab];
                for (uint64_t b = 1; b <= left1; b++) {
                    const char r1 = (*Rp)[a2.exR[iab] - b], g1 = (char)idx.view.G[a2.exG[iab] - b];
                    if (r1 != g1 && r1 < 4 && g1 < 4) ++nMM1;
                }
                for (uint64_t b = 0; b < right1; b++) {
                    const char r1 = (*Rp)[a2.exR[iab] + a2.exL[iab] + b], g1 = (char)idx.view.G[a2.exG[iab] + a2.exL[iab] + b];
                    if (r1 != g1 && r1 < 4 && g1 < 4) ++nMM1;
                }
                a2.exR[iab] = (uint16_t)(a2.exR[iab] - left1);
                a2.exG[iab] -= left1;
                a2.exL[iab] = (uint16_t)(a2.exL[iab] + left1 + right1);
            }
            const uint64_t mmTotal = std::min<uint64_t>(P.hp.outFilterMismatchNmax, (uint64_t)(P.hp.outFilterMismatchNoverReadLmax * (double)(readLength[0] + readLength[1])));
            if (a2.nMM + nMM1 > std::min<uint64_t>(mmTotal, (uint64_t)(P.hp.outFilterMismatchNoverLmax * (double)(Lread - 1)))) continue;
            a1 = &a2;
        }
        trModel->quantAlign(*a1, Lread, alignT);
    }
    const uint64_t nAlignT = alignT.size();
    if (nAlignT == 0) return;
    alignT[(size_t)(draw * (double)nAlignT)].primaryFlag = 1;
    for (uint64_t k = 0; k < nAlignT; k++) bamMapped(c, i, r, alignT[k], nAlignT, k, bam, true);
}

std::string OutputWriter::bamHeaderTranscriptome() const {   // samHeaders.cpp:8-20, outBAMwriteHeader
    std::string text;
    for (size_t ii = 0; ii < trModel->trID.size(); ii++) text += "@SQ\tSN:" + trModel->trID[ii] + "\tLN:" + std::to_string(trModel->trLen[ii]) + "\n";
    for (const std::string& rg : P.outSAMattrRGlineSplit) text += "@RG\t" + rg + "\n";
    std::string h = "BAM\001";
    put32(h, (uint32_t)text.size());
    h += text;
    put32(h, (uint32_t)trModel->trID.size());
    for (size_t ii = 0; ii < trModel->trID.size(); ii++) {
        put32(h, (uint32_t)(trModel->trID[ii].size() + 1));
        h.append(trModel->trID[ii].c_str(), trModel->trID[ii].size() + 1);
        put32(h, trModel->trLen[ii]);
    }
    return h;
}

// ---- --quantMode GeneCounts --------------------------------------------------------------------------------------------------------
int GeneModel::load(const std::string& dir, std::string& err) {   // Transcriptome.cpp:18-31, 78-98
    const char* sol = "SOLUTION: utilize --sjdbGTFfile /path/to/annotations.gtf option at the genome generation step or mapping step\n";
    std::ifstream ge(dir + "/geneInfo.tab");
    if (ge.fail()) { err = "EXITING because of fatal INPUT error: could not open input file " + dir + "/geneInfo.tab\n" + sol; return STAR_EXIT_INPUT_FILES; }
    uint64_t nGe = 0;
    ge >> nGe;
    geID.resize(nGe);
    std::string line;
    std::getline(ge, line);
    for (uint64_t i = 0; i < nGe; i++) { std::getline(ge, line); std::istringstream ls(line); ls >> geID[i]; }
    std::ifstream ex(dir + "/exonGeTrInfo.tab");
    if (ex.fail()) { err = "EXITING because of fatal INPUT error: could not open input file " + dir + "/exonGeTrInfo.tab\n" + sol; return STAR_EXIT_INPUT_FILES; }
    uint64_t nEx = 0;
    ex >> nEx;
    s.resize(nEx); e.resize(nEx); eMax.resize(nEx); str.resize(nEx); g.resize(nEx);
    for (uint64_t i = 0; i < nEx; i++) { int st1; uint32_t t1; ex >> s[i] >> e[i] >> st1 >> g[i] >> t1; str[i] = (uint8_t)st1; }
    for (uint64_t i = 0; i < nEx; i++) eMax[i] = i == 0 ? e[0] : std::max(eMax[i - 1], e[i]);
    return 0;
}

void GeneCounts::add(const GeneCounts& o) {
    cMulti += o.cMulti;
    for (int t = 0; t < 3; t++) {
        cNone[t] += o.cNone[t]; cAmbig[t] += o.cAmbig[t];
        for (size_t i = 0; i < gCount[t].size() && i < o.gCount[t].size(); i++) gCount[t][i] += o.gCount[t][i];
    }
}

// Transcriptome_geneCountsAddAlign.cpp:4-63: a uniquely mapped read counts for the one gene whose exons its blocks overlap
void GeneCounts::addAlign(const GeneModel& gm, uint64_t nTr, const star_align_t* trs) {
    if (nTr > 1) { cMulti++; return; }
    const star_align_t& a = trs[0];
    int64_t gene1[3] = {-1, -1, -1};
    const int64_t nEx = (int64_t)gm.s.size();
    for (int ib = (int)a.nExons - 1; ib >= 0 && nEx > 0; ib--) {
        const uint64_t g1 = a.exG[ib] + a.exL[ib] - 1;   // end of the block
        int64_t e1;                                        // binarySearch1a: last exon start <= g1
        if (g1 > gm.s[nEx - 1]) e1 = nEx - 1;
        else if (g1 < gm.s[0]) e1 = -1;
        else {
            int64_t i1 = 0, i2 = nEx - 1;
            while (i2 > i1 + 1) { const int64_t i3 = (i1 + i2) / 2; if (gm.s[i3] > g1) i2 = i3; else i1 = i3; }
            while (i1 < nEx - 1 && g1 == gm.s[i1 + 1]) ++i1;
            e1 = i1;
        }
        while (e1 >= 0 && gm.eMax[e1] >= a.exG[ib]) {
            if (gm.e[e1] >= a.exG[ib]) {
                const unsigned str1 = (unsigned)gm.str[e1] - 1;
                for (int itype = 0; itype < 3; itype++) {
                    if (itype == 1 && a.Str != str1 && str1 < 2) continue;
                    if (itype == 2 && a.Str == str1 && str1 < 2) continue;
                    if (gene1[itype] == -1) gene1[itype] = gm.g[e1];
                    else if (gene1[itype] == -2) continue;
                    else if (gene1[itype] != (int64_t)gm.g[e1]) gene1[itype] = -2;
                }
            }
            --e1;
        }
    }
    for (int itype = 0; itype < 3; itype++) {
        if (gene1[itype] == -1) cNone[itype]++;
        else if (gene1[itype] == -2) cAmbig[itype]++;
        else gCount[itype][gene1[itype]]++;
    }
}

void GeneCounts::write(const GeneModel& gm, const Stats& st, const std::string& path) const {   // Transcriptome.cpp:156-190
    std::ofstream q(path);
    const uint64_t unm = st.unmappedMismatch + st.unmappedShort + st.unmappedOther + st.unmappedMulti;
    q << "N_unmapped"; for (int t = 0; t < 3; t++) q << "\t" << unm; q << "\n";
    q << "N_multimapping"; for (int t = 0; t < 3; t++) q << "\t" << cMulti; q << "\n";
    q << "N_noFeature"; for (int t = 0; t < 3; t++) q << "\t" << cNone[t]; q << "\n";
    q << "N_ambiguous"; for (int t = 0; t < 3; t++) q << "\t" << cAmbig[t]; q << "\n";
    for (size_t ig = 0; ig < gm.geID.size(); ig++) {
        q << gm.geID[ig];
        for (int t = 0; t < 3; t++) q << "\t" << gCount[t][ig];
        q << "\n";
    }
}

static std::string timeMonthDayTime(time_t t) {  // TimeFunctions.cpp:14-20
    char b[100];
    strftime(b, 80, "%b %d %H:%M:%S", localtime(&t));
    return b;
}

void OutputWriter::writeLogFinal(const Stats& s, const std::string& path) const {  // Stats.cpp:99-145
    std::ofstream o(path);
    const int w1 = 50;
    auto pct = [&](uint64_t a) { return s.readN > 0 ? double(a) / double(s.readN) * 100 : 0.0; };
    double dt = difftime(s.timeFinish, s.timeStartMap);
    o << std::setiosflags(std::ios::fixed) << std::setprecision(2)
      << std::setw(w1) << "Started job on |\t" << timeMonthDayTime(s.timeStart) << "\n"
      << std::setw(w1) << "Started mapping on |\t" << timeMonthDayTime(s.timeStartMap) << "\n"
      << std::setw(w1) << "Finished on |\t" << timeMonthDayTime(s.timeFinish) << "\n"
      << std::setw(w1) << "Mapping speed, Million of reads per hour |\t" << double(s.readN) / 1e6 / dt * 3600 << "\n"
      << "\n"
      << std::setw(w1) << "Number of input reads |\t" << s.readN << "\n"
      << std::setw(w1) << "Average input read length |\t" << (s.readN > 0 ? s.readBases / s.readN : 0) << "\n"
      << std::setw(w1) << "UNIQUE READS:\n"
      << std::setw(w1) << "Uniquely mapped reads number |\t" << s.mappedReadsU << "\n"
      << std::setw(w1) << "Uniquely mapped reads % |\t" << pct(s.mappedReadsU) << '%' << "\n"
      << std::setw(w1) << "Average mapped length |\t" << (s.mappedReadsU > 0 ? double(s.mappedBases) / double(s.mappedReadsU) : 0) << "\n";
    o << std::setw(w1) << "Number of splices: Total |\t" << s.splicesN[0] + s.splicesN[1] + s.splicesN[2] + s.splicesN[3] + s.splicesN[4] + s.splicesN[5] + s.splicesN[6] << "\n"
      << std::setw(w1) << "Number of splices: Annotated (sjdb) |\t" << s.splicesNsjdb << "\n"
      << std::setw(w1) << "Number of splices: GT/AG |\t" << s.splicesN[1] + s.splicesN[2] << "\n"
      << std::setw(w1) << "Number of splices: GC/AG |\t" << s.splicesN[3] + s.splicesN[4] << "\n"
      << std::setw(w1) << "Number of splices: AT/AC |\t" << s.splicesN[5] + s.splicesN[6] << "\n"
      << std::setw(w1) << "Number of splices: Non-canonical |\t" << s.splicesN[0] << "\n";
    o << std::setw(w1) << "Mismatch rate per base, % |\t" << double(s.mappedMismatchesN) / double(s.mappedBases) * 100 << '%' << "\n"
      << std::setw(w1) << "Deletion rate per base |\t" << (s.mappedBases > 0 ? double(s.mappedDelL) / double(s.mappedBases) * 100 : 0) << '%' << "\n"
      << std::setw(w1) << "Deletion average length |\t" << (s.mappedDelN > 0 ? double(s.mappedDelL) / double(s.mappedDelN) : 0) << "\n"
      << std::setw(w1) << "Insertion rate per base |\t" << (s.mappedBases > 0 ? double(s.mappedInsL) / double(s.mappedBases) * 100 : 0) << '%' << "\n"
      << std::setw(w1) << "Insertion average length |\t" << (s.mappedInsN > 0 ? double(s.mappedInsL) / double(s.mappedInsN) : 0) << "\n"
      << std::setw(w1) << "MULTI-MAPPING READS:\n"
      << std::setw(w1) << "Number of reads mapped to multiple loci |\t" << s.mappedReadsM << "\n"
      << std::setw(w1) << "% of reads mapped to multiple loci |\t" << pct(s.mappedReadsM) << '%' << "\n"
      << std::setw(w1) << "Number of reads mapped to too many loci |\t" << s.unmappedMulti << "\n"
      << std::setw(w1) << "% of reads mapped to too many loci |\t" << pct(s.unmappedMulti) << '%' << "\n"
      << std::setw(w1) << "UNMAPPED READS:\n"
      << std::setw(w1) << "Number of reads unmapped: too many mismatches |\t" << s.unmappedMismatch << "\n"
      << std::setw(w1) << "% of reads unmapped: too many mismatches |\t" << pct(s.unmappedMismatch) << '%' << "\n"
      << std::setw(w1) << "Number of reads unmapped: too short |\t" << s.unmappedShort << "\n"
      << std::setw(w1) << "% of reads unmapped: too short |\t" << pct(s.unmappedShort) << '%' << "\n"
      << std::setw(w1) << "Number of reads unmapped: other |\t" << s.unmappedOther << "\n"
      << std::setw(w1) << "% of reads unmapped: other |\t" << pct(s.unmappedOther) << '%' << "\n"
      << std::setw(w1) << "CHIMERIC READS:\n"
      << std::setw(w1) << "Number of chimeric reads |\t" << s.chimericAll << "\n"
      << std::setw(w1) << "% of chimeric reads |\t" << pct(s.chimericAll) << '%' << "\n"
      << std::flush;
}

}  // namespace starhost
