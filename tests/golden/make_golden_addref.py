#!/usr/bin/env python3
"""Regenerates tests/golden/addref.tar.xz — run in the BUILD container only (needs oracle/_ref/STAR, i.e. /root/reference).

Golden outputs of the UNMODIFIED reference binary for references added at the mapping stage (--genomeFastaFiles with --runMode
alignReads, --outSAMfilter), on the indexes of tiny.tar.gz (tiny/idx: annotated, with a junction region) and twopass.tar.gz
(twopass/idx0: no junction region):

  addref/addA.fa          92 ERCC-like spikes (seeded): 6 of them end in the same 40-base poly-A tail, one is shorter than a read; N runs,
                          IUPAC codes, lowercase, CRLF line ends, a header with a description
  addref/addB.fa          a 12 kb copy of chr1 (more than the 10 000 bases the insertion search compares) and the reverse complement of
                          3 kb of chr2 (multimappers across strands)
  addref/add.gtf          annot.gtf + genes on two spikes;  addref/addsj.tab  junctions on a spike and on chr2
  addref/{pe_1,pe_2,se_1}.fq   reads from the spikes, the copies and the genome, some spliced at the added junctions, with mismatches
  addref/scenarios.json   name -> argument list (IDX = tiny/idx, IDX0 = twopass/idx0, AR/ = the unpacked addref/ directory)
  addref/<name>/          what the reference wrote: Aligned.out.sam or the BAM files, SJ.out.tab, Log.final.out, header.txt (the @SQ lines
                          of the SAM / BAM header), Unmapped.out.mate*, ReadsPerGene.out.tab, Aligned.toTranscriptome.out.bam,
                          _STARpass1/{SJ.out.tab,Log.final.out}, _STARgenome/{sjdbInfo.txt,sjdbList.out.tab,sha256.txt} (digests of the
                          Genome, SA and SAindex written with --sjdbInsertSave All)

The generator asserts what the fixture has to pin: the chr1 copy repeats more than 10 000 bases, at least two spikes share their last 12
bases, and the grown genome changes winBinNbits for --alignIntronMax 1000 --alignMatesGapMax 1000.
"""
import gzip
import hashlib
import json
import math
import os
import random
import subprocess
import tarfile
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
STAR = os.path.join(ROOT, "oracle", "_ref", "STAR")
COMP = str.maketrans("ACGTNacgtn", "TGCANtgcan")

COMMON = ["--outSAMattributes", "NH", "HI", "AS", "nM", "--runThreadN", "1"]
SCENARIOS = {
    "A_pe": ["--genomeDir", "IDX", "--genomeFastaFiles", "AR/addA.fa", "AR/addB.fa", "--readFilesIn", "AR/pe_1.fq", "AR/pe_2.fq"],
    "B_se_noannot": ["--genomeDir", "IDX0", "--genomeFastaFiles", "AR/addA.fa", "AR/addB.fa", "--readFilesIn", "AR/se_1.fq"],
    "C_keeponly_within_keeppairs": ["--genomeDir", "IDX", "--genomeFastaFiles", "AR/addA.fa", "AR/addB.fa", "--readFilesIn", "AR/pe_1.fq", "AR/pe_2.fq",
                                    "--outSAMfilter", "KeepOnlyAddedReferences", "--outSAMunmapped", "Within", "KeepPairs", "--outReadsUnmapped", "Fastx"],
    "D_keepall_sorted_bam": ["--genomeDir", "IDX", "--genomeFastaFiles", "AR/addA.fa", "AR/addB.fa", "--readFilesIn", "AR/pe_1.fq", "AR/pe_2.fq",
                             "--outSAMfilter", "KeepAllAddedReferences", "--outSAMunmapped", "Within", "--outSAMtype", "BAM", "Unsorted", "SortedByCoordinate",
                             "--outReadsUnmapped", "Fastx"],
    "E_keepall_sam_keeppairs_allbest": ["--genomeDir", "IDX0", "--genomeFastaFiles", "AR/addB.fa", "AR/addA.fa", "--readFilesIn", "AR/pe_1.fq", "AR/pe_2.fq",
                                        "--outSAMfilter", "KeepAllAddedReferences", "--outSAMunmapped", "Within", "KeepPairs", "--outSAMprimaryFlag", "AllBestScore"],
    "F_sjfile_save_noannot": ["--genomeDir", "IDX0", "--genomeFastaFiles", "AR/addA.fa", "AR/addB.fa", "--readFilesIn", "AR/pe_1.fq", "AR/pe_2.fq",
                              "--sjdbFileChrStartEnd", "AR/addsj.tab", "--sjdbOverhang", "60", "--sjdbInsertSave", "All"],
    "G_sjfile_save_annot": ["--genomeDir", "IDX", "--genomeFastaFiles", "AR/addA.fa", "AR/addB.fa", "--readFilesIn", "AR/pe_1.fq", "AR/pe_2.fq",
                            "--sjdbFileChrStartEnd", "AR/addsj.tab", "--sjdbInsertSave", "All"],
    "H_gtf_quant_twopass": ["--genomeDir", "IDX", "--genomeFastaFiles", "AR/addA.fa", "AR/addB.fa", "--readFilesIn", "AR/pe_1.fq", "AR/pe_2.fq",
                            "--sjdbGTFfile", "AR/add.gtf", "--quantMode", "GeneCounts", "TranscriptomeSAM", "--twopassMode", "Basic", "--sjdbInsertSave", "All"],
    "I_bysjout_keepall": ["--genomeDir", "IDX", "--genomeFastaFiles", "AR/addA.fa", "AR/addB.fa", "--readFilesIn", "AR/pe_1.fq", "AR/pe_2.fq",
                          "--outFilterType", "BySJout", "--outSAMfilter", "KeepAllAddedReferences", "--outSAMunmapped", "Within"],
    "J_intron_window": ["--genomeDir", "IDX0", "--genomeFastaFiles", "AR/addA.fa", "AR/addB.fa", "--readFilesIn", "AR/pe_1.fq", "AR/pe_2.fq",
                        "--alignIntronMax", "1000", "--alignMatesGapMax", "1000"],
}
SAVED = ["Aligned.out.sam", "Aligned.out.bam", "Aligned.sortedByCoord.out.bam", "SJ.out.tab", "Log.final.out", "Unmapped.out.mate1", "Unmapped.out.mate2",
         "ReadsPerGene.out.tab", "Aligned.toTranscriptome.out.bam", "_STARpass1/SJ.out.tab", "_STARpass1/Log.final.out", "_STARgenome/sjdbInfo.txt",
         "_STARgenome/sjdbList.out.tab"]


def read_fasta(path):
    seqs, name = {}, None
    for line in open(path):
        line = line.strip()
        if line.startswith(">"):
            name = line[1:].split()[0]
            seqs[name] = []
        elif name:
            seqs[name].append(line)
    return {k: "".join(v).upper() for k, v in seqs.items()}


def rc(s):
    return s.translate(COMP)[::-1]


def wrap(s, w=60, eol="\n"):
    return "".join(s[i:i + w] + eol for i in range(0, len(s), w))


def make_inputs(d, genome, gtf_src, rng):
    spikes = []
    tail = "A" * 40
    for i in range(92):
        L = 40 if i == 7 else rng.randint(300, 1200)   # spike 7 is shorter than a read
        s = "".join(rng.choice("ACGT") for _ in range(L))
        if i in (3, 11, 19, 27, 35, 43):
            s = s[:-40] + tail
        spikes.append(("ERCC-%05d" % (i + 1), s))
    # N runs, IUPAC codes and lowercase in the FASTA text (the sequences used for reads keep A/C/G/T)
    text = []
    for i, (nm, s) in enumerate(spikes):
        t = s
        if i == 5:
            t = t[:100] + "N" * 30 + t[130:]
        if i == 6:
            t = t[:50] + "RYKM" + t[54:200].lower() + t[200:]
        hdr = ">%s ERCC-like spike %d" % (nm, i) if i == 0 else ">" + nm
        eol = "\r\n" if i in (1, 2) else "\n"
        text.append(hdr + eol + wrap(t, 70 if i % 2 else 60, eol))
    open(os.path.join(d, "addA.fa"), "w", newline="").write("".join(text))
    copy = genome["chr1"][10000:22000]
    rcseg = rc(genome["chr2"][5000:8000])
    assert len(copy) > 10000 and "N" not in copy
    open(os.path.join(d, "addB.fa"), "w").write(">dupchr1 copy of chr1:10001-22000\n" + wrap(copy) + ">rcchr2\n" + wrap(rcseg))
    added = dict(spikes)
    added["dupchr1"] = copy
    added["rcchr2"] = rcseg
    # at least two spikes share their last 12 bases (equal rows whose memcmp order differs from offset order)
    ends = [s[-12:] for _, s in spikes]
    assert max(ends.count(e) for e in ends) >= 2
    # junctions on an added reference and on chr2, genes on two spikes
    s1 = spikes[10][1]
    open(os.path.join(d, "addsj.tab"), "w").write("%s\t201\t400\t+\nchr2\t20001\t20500\t+\n" % spikes[10][0])
    gtf = open(gtf_src).read()
    gtf += '%s\tsynth\texon\t1\t200\t.\t+\t.\tgene_id "GS1"; transcript_id "GS1.1";\n' % spikes[10][0]
    gtf += '%s\tsynth\texon\t401\t%d\t.\t+\t.\tgene_id "GS1"; transcript_id "GS1.1";\n' % (spikes[10][0], len(s1))
    gtf += '%s\tsynth\texon\t1\t%d\t.\t-\t.\tgene_id "GS2"; transcript_id "GS2.1";\n' % (spikes[20][0], len(spikes[20][1]))
    open(os.path.join(d, "add.gtf"), "w").write(gtf)
    # reads
    def mutate(s):
        s = list(s)
        for _ in range(rng.choice([0, 0, 1, 2])):
            p = rng.randrange(len(s))
            s[p] = rng.choice("ACGT")
        return "".join(s)

    sources = [(nm, s) for nm, s in spikes if len(s) >= 300] + [("dupchr1", copy), ("rcchr2", rcseg), ("chr1", genome["chr1"]), ("chr2", genome["chr2"])]
    spliced = s1[:200] + s1[400:]
    sources.append(("spliced", spliced))
    r1, r2, se = [], [], []
    for i in range(500):
        nm, s = sources[rng.randrange(len(sources))] if i % 5 else ("spliced", spliced)
        frag = rng.randint(180, min(300, len(s)))
        p = rng.randrange(len(s) - frag + 1)
        f = s[p:p + frag]
        if "N" in f:
            continue
        if rng.random() < 0.5:
            f = rc(f)
        a, b = mutate(f[:100]), mutate(rc(f)[:100])
        if i % 23 == 0:   # one mate from a random place: pairs with one mapped mate
            b = "".join(rng.choice("ACGT") for _ in range(100))
        r1.append(("r%d" % i, a))
        r2.append(("r%d" % i, b))
    for nm, s in spikes[7:8]:   # the short spike, as 40-base reads
        r1.append(("short", s)); r2.append(("short", rc(s)))
    for i in range(300):
        nm, s = sources[rng.randrange(len(sources))]
        p = rng.randrange(len(s) - 100 + 1)
        f = s[p:p + 100]
        if "N" in f:
            continue
        se.append(("s%d" % i, mutate(f if rng.random() < 0.5 else rc(f))))
    for fn, rr in (("pe_1.fq", r1), ("pe_2.fq", r2), ("se_1.fq", se)):
        with open(os.path.join(d, fn), "w") as f:
            for nm, s in rr:
                f.write("@%s\n%s\n+\n%s\n" % (nm, s, "I" * len(s)))
    return added


def win_bits(nGenome, intron=1000, gap=1000, chrBin=18):
    b = int(math.floor(math.log2(max(max(4, intron), gap) / 4) + 0.5))
    b = max(b, int(math.floor(math.log2(nGenome // 40000 + 1) + 0.5)))
    return min(b, chrBin)


def main():
    out_tar = os.path.join(ROOT, "tests", "golden", "addref.tar.xz")
    rng = random.Random(20261019)
    with tempfile.TemporaryDirectory() as tmp:
        for t in ("tiny.tar.gz", "twopass.tar.gz"):
            with tarfile.open(os.path.join(ROOT, "tests", "golden", t)) as tf:
                tf.extractall(tmp)
        d = os.path.join(tmp, "addref")
        os.makedirs(d)
        genome = read_fasta(os.path.join(tmp, "tiny", "genome.fa"))
        make_inputs(d, genome, os.path.join(tmp, "tiny", "annot.gtf"), rng)
        json.dump(SCENARIOS, open(os.path.join(d, "scenarios.json"), "w"), indent=1)
        subst = {"IDX": os.path.join(tmp, "tiny", "idx"), "IDX0": os.path.join(tmp, "twopass", "idx0")}
        for name, args in SCENARIOS.items():
            od = os.path.join(d, name) + "/"
            os.makedirs(od)
            a = [subst.get(x, os.path.join(d, x[3:]) if x.startswith("AR/") else x) for x in args]
            subprocess.check_call([STAR] + a + COMMON + ["--outFileNamePrefix", od], stdout=subprocess.DEVNULL)
            logout = open(od + "Log.out").read()
            if name == "J_intron_window":   # the grown genome decides winBinNbits
                old = int(open(os.path.join(subst["IDX0"], "chrStart.txt")).read().split()[-1])
                starts = [l for l in logout.split("\n") if "chrStart:" in l]
                new = max(int(l.split("chrStart:")[1]) for l in starts) + (1 << 18)   # the last (short) chromosome fills one 2^18 bin
                assert win_bits(old) != win_bits(new), (win_bits(old), win_bits(new))
                assert "redefined winBinNbits=%d" % win_bits(new) in logout
            sam = od + "Aligned.out.sam"
            hdr = []
            if os.path.exists(sam):
                hdr = [l for l in open(sam) if l.startswith("@SQ")]
            else:
                for f in ("Aligned.out.bam", "Aligned.sortedByCoord.out.bam"):
                    if os.path.exists(od + f):
                        txt = gzip.decompress(open(od + f, "rb").read())
                        hdr = [l + "\n" for l in txt.decode("latin-1").split("\n") if l.startswith("@SQ")]
                        break
            open(od + "header.txt", "w").write("".join(hdr))
            if os.path.exists(od + "_STARgenome/SA"):
                with open(od + "_STARgenome/sha256.txt", "w") as f:
                    for fn in ("Genome", "SA", "SAindex"):
                        f.write("%s %s\n" % (fn, hashlib.sha256(open(od + "_STARgenome/" + fn, "rb").read()).hexdigest()))
            keep = set(SAVED + ["header.txt", "_STARgenome/sha256.txt"])
            for root, dirs, files in os.walk(od, topdown=False):
                for fn in files:
                    rel = os.path.relpath(os.path.join(root, fn), od)
                    if rel not in keep:
                        os.remove(os.path.join(root, fn))
                for dn in dirs:
                    p = os.path.join(root, dn)
                    if not os.listdir(p):
                        os.rmdir(p)
        # the @PG / @CO lines name temporary paths: keep only records and @SQ/@HD lines in the SAM files
        for name in SCENARIOS:
            sam = os.path.join(d, name, "Aligned.out.sam")
            if os.path.exists(sam):
                lines = [l for l in open(sam) if not l.startswith("@PG") and not l.startswith("@CO")]
                open(sam, "w").write("".join(lines))
        with tarfile.open(out_tar, "w:xz") as tf:
            tf.add(d, arcname="addref")
    print("wrote", out_tar, os.path.getsize(out_tar))


if __name__ == "__main__":
    main()
