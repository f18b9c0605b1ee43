#!/usr/bin/env python3
"""Regenerates tests/golden/signal.tar.gz — needs oracle/_ref/STAR (the unmodified reference, built by __graft_entry__.build()).

Golden signal tracks (--outWigType) of the UNMODIFIED reference binary:

  signal/scenarios.json        name -> argument list; in mapping runs relative to the unpacked tiny/ directory, SG = the unpacked signal/
  signal/bam{1,2,3}.bam        hand-built BAMs (tools/bam_synth.py, seeded): unsorted with reference ids that come back, NH absent / as
                               c C s S i I / as f, duplicates, unmapped mates with a reference id, tid = -1 records at the end, I S H D N = X,
                               a record ending on the last base of a reference and one running one base past it, a reference that
                               --outWigReferencesPrefix chr excludes, piles of NH 2..7 records interleaved with unique ones
  signal/<name>/Signal.*       the reference's Signal.{Unique,UniqueMultiple}.str{1,2}.out.{bg,wig}

The generator asserts that the fixtures pin the fold order: at least one position's UniqueMultiple value changes when its 1/NH terms are
summed in another order.
"""
import json
import os
import shutil
import subprocess
import sys
import tarfile
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bam_synth  # noqa: E402

STAR = os.path.join(ROOT, "oracle", "_ref", "STAR")
SORTED = ["--outSAMtype", "BAM", "SortedByCoordinate"]
ENCODE = ["--outFilterType", "BySJout", "--outSAMattributes", "NH", "HI", "AS", "NM", "MD", "--outFilterMultimapNmax", "20", "--outFilterMismatchNmax", "999",
          "--outFilterMismatchNoverReadLmax", "0.04", "--alignIntronMin", "20", "--alignIntronMax", "1000000", "--alignMatesGapMax", "1000000",
          "--alignSJoverhangMin", "8", "--alignSJDBoverhangMin", "1", "--sjdbScore", "1", "--outSAMtype", "BAM", "Unsorted", "SortedByCoordinate",
          "--quantMode", "TranscriptomeSAM", "GeneCounts", "--outSAMunmapped", "Within", "--outSAMstrandField", "intronMotif",
          "--outSAMheaderHD", "@HD", "VN:1.4", "SO:unsorted", "--outSAMheaderPG", "@PG", "ID:x", "PN:y", "--limitBAMsortRAM", "10000000000"]
HARD = ["--genomeDir", "idx", "--readFilesIn", "hard_1.fq", "hard_2.fq"]
SCENARIOS = {
    # mapping runs on the tiny index with the multimapper-rich reads
    "M1_bg_stranded_rpm": HARD + SORTED + ["--outWigType", "bedGraph"],
    "M2_wig_read1_5p_unstranded_none": HARD + SORTED + ["--outWigType", "wiggle", "read1_5p", "--outWigStrand", "Unstranded", "--outWigNorm", "None"],
    "M3_bg_read2": HARD + SORTED + ["--outWigType", "bedGraph", "read2"],
    "M4_bg_single_end": ["--genomeDir", "idx", "--readFilesIn", "se_1.fq"] + SORTED + ["--outWigType", "bedGraph", "--outWigNorm", "None"],
    "M5_encode_full": HARD + ENCODE + ["--outWigType", "bedGraph"],
    "M6_unmapped_within": HARD + SORTED + ["--outSAMunmapped", "Within", "--outWigType", "bedGraph", "--outWigStrand", "Unstranded"],
    "M7_multimap20": HARD + SORTED + ["--outFilterMultimapNmax", "20", "--outWigType", "wiggle", "--outWigNorm", "None"],
    # --runMode inputAlignmentsFromBAM on the hand-built BAMs
    "B1_bg_stranded_rpm": ["--inputBAMfile", "SG/bam1.bam", "--outWigType", "bedGraph"],
    "B2_bg_none_prefix": ["--inputBAMfile", "SG/bam1.bam", "--outWigType", "bedGraph", "--outWigNorm", "None", "--outWigReferencesPrefix", "chr"],
    "B3_wig_read1_5p": ["--inputBAMfile", "SG/bam2.bam", "--outWigType", "wiggle", "read1_5p", "--outWigNorm", "None"],
    "B4_wig_unstranded_rpm_prefix": ["--inputBAMfile", "SG/bam2.bam", "--outWigType", "wiggle", "--outWigStrand", "Unstranded", "--outWigReferencesPrefix", "chr"],
    "B5_bg_read2_unstranded": ["--inputBAMfile", "SG/bam3.bam", "--outWigType", "bedGraph", "read2", "--outWigStrand", "Unstranded", "--outWigNorm", "None"],
    "B6_bg_read1_5p_rpm": ["--inputBAMfile", "SG/bam3.bam", "--outWigType", "bedGraph", "read1_5p"],
}
SEEDS = {"bam1.bam": 11, "bam2.bam": 12, "bam3.bam": 13}


def run_args(name, args, sg):
    a = [x.replace("SG/", sg + "/") for x in args]
    if name.startswith("B"):
        a = ["--runMode", "inputAlignmentsFromBAM"] + a
    return a


def main():
    tmp = tempfile.mkdtemp(prefix="golden_sig_")
    with tarfile.open(os.path.join(ROOT, "tests", "golden", "tiny.tar.gz")) as t:
        t.extractall(tmp)
    tiny = os.path.join(tmp, "tiny")
    sg = os.path.join(tmp, "signal")
    os.makedirs(sg)
    pinned = False
    for fn, seed in SEEDS.items():
        refs, recs = bam_synth.random_bam(seed)
        with open(os.path.join(sg, fn), "wb") as f:
            f.write(bam_synth.bam_bytes(refs, recs))
        pinned |= bam_synth.fold_order_matters(bam_synth.um_terms(refs, recs))
    assert pinned, "no fixture position depends on the order of its 1/NH terms"
    for name, args in SCENARIOS.items():
        out = os.path.join(tmp, "run_" + name) + "/"
        os.makedirs(out)
        subprocess.check_call([STAR] + run_args(name, args, sg) + ["--outFileNamePrefix", out, "--runThreadN", "1"], cwd=tiny, stdout=subprocess.DEVNULL)
        dst = os.path.join(sg, name)
        os.makedirs(dst)
        files = sorted(f for f in os.listdir(out) if f.startswith("Signal."))
        assert files, name
        for f in files:
            shutil.copy(out + f, os.path.join(dst, f))
    with open(os.path.join(sg, "scenarios.json"), "w") as f:
        json.dump(SCENARIOS, f, indent=1)
    dst = os.path.join(ROOT, "tests", "golden", "signal.tar.gz")
    with tarfile.open(dst, "w:gz", compresslevel=9) as t:
        t.add(sg, arcname="signal")
    print("wrote", dst, os.path.getsize(dst), "bytes")
    shutil.rmtree(tmp)


if __name__ == "__main__":
    main()
