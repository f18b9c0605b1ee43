#!/usr/bin/env python3
"""Regenerates tests/golden/dedup.tar.gz — needs oracle/_ref/STAR (the unmodified reference, built by __graft_entry__.build()).

Golden duplicate marking (--runMode inputAlignmentsFromBAM --bamRemoveDuplicatesType) of the UNMODIFIED reference binary:

  dedup/scenarios.json          name -> argument list; DG = the unpacked dedup/ directory
  dedup/pe{1,2}.bam             hand-built coordinate-sorted paired BAMs (tools/bam_synth.py, seeded): pairs duplicated under new names
                                with other AS values, mate-2 differences at the forward start and the reverse end, S-clipped CIGARs, an
                                N gap, an insertion, names occurring 1 and 3 times, signed-char names, multimappers with and without a
                                preset 0x400, unmapped records at the end, groups closed by reference and by position, a group held open
                                by rightMax == 0, and the pinned cases of bam_synth.dedup_pinned_records
  dedup/se.bam                  single-end records (every reference one group; pairs of unrelated reads)
  dedup/map.bam, map_unm.bam    the reference's sorted BAMs of the tiny fixture's first 800 std pairs with a seeded fifth of the pairs duplicated
                                under new names (a tenth of those with mate 2 changed at its first base); map_unm.bam with
                                --outSAMunmapped Within
  dedup/<name>/Processed.out.bam the reference's output

The generator asserts that the fixtures pin the tie order (a class whose best pairs differ in name and file order keeps the first in name
order), the pad nibble of an odd l_seq (pairs that differ only there stay two classes with N = 0) and the S extension (3S47M at p is the
same as 50M at p-3).
"""
import json
import os
import random
import shutil
import subprocess
import sys
import tarfile
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bam_synth  # noqa: E402

STAR = os.path.join(ROOT, "oracle", "_ref", "STAR")
UI, UINM = ["--bamRemoveDuplicatesType", "UniqueIdentical"], ["--bamRemoveDuplicatesType", "UniqueIdenticalNotMulti"]


def N(n):
    return ["--bamRemoveDuplicatesMate2basesN", str(n)]


SCENARIOS = {
    "P1_ui_n0": ["--inputBAMfile", "DG/pe1.bam"] + UI,
    "P2_uinm_n1": ["--inputBAMfile", "DG/pe1.bam"] + UINM + N(1),
    "P3_ui_n7": ["--inputBAMfile", "DG/pe2.bam"] + UI + N(7),
    "P4_uinm_n8": ["--inputBAMfile", "DG/pe2.bam"] + UINM + N(8),
    "S1_ui_single_end": ["--inputBAMfile", "DG/se.bam"] + UI,
    "M1_ui_n0": ["--inputBAMfile", "DG/map.bam"] + UI,
    "M2_uinm_n8": ["--inputBAMfile", "DG/map.bam"] + UINM + N(8),
    "M3_unmapped_within_ui_n1": ["--inputBAMfile", "DG/map_unm.bam"] + UI + N(1),
}


def run_args(args, dg):
    return ["--runMode", "inputAlignmentsFromBAM"] + [x.replace("DG/", dg + "/") for x in args]


def dup_reads(tiny, out, seed=31, n=800):
    """The first n pairs of std_{1,2}.fq with a seeded fifth of the pairs repeated under new names; a tenth of the copies with mate 2 changed at base 1."""
    rng = random.Random(seed)
    fq = [open(os.path.join(tiny, "std_%d.fq" % m)).read().split("\n") for m in (1, 2)]
    w = [open(os.path.join(out, "dup_%d.fq" % m), "w") for m in (1, 2)]
    for i in range(n):
        rec = [fq[m][4 * i:4 * i + 4] for m in (0, 1)]
        for m in (0, 1):
            w[m].write("\n".join(rec[m]) + "\n")
        if rng.random() < 0.2:
            alt = rng.random() < 0.1
            for m in (0, 1):
                h, s, p, q = rec[m]
                if alt and m == 1:
                    s = ("A" if s[0] != "A" else "C") + s[1:]
                w[m].write("\n".join(["@dup%d_%s" % (i, h[1:]), s, p, q]) + "\n")
    for f in w:
        f.close()


def flags_by_name(path):
    st = {}
    for r in bam_synth.read_bam(open(path, "rb").read())[1]:
        n, f = bam_synth.rec_name_flag(r)
        st.setdefault(n, []).append(not f & 0x400)
    return st


def main():
    tmp = tempfile.mkdtemp(prefix="golden_dedup_")
    with tarfile.open(os.path.join(ROOT, "tests", "golden", "tiny.tar.gz")) as t:
        t.extractall(tmp)
    tiny = os.path.join(tmp, "tiny")
    dg = os.path.join(tmp, "dedup")
    os.makedirs(dg)
    for fn, seed in (("pe1.bam", 21), ("pe2.bam", 22)):
        refs, recs = bam_synth.dedup_pe_bam(seed, n_pairs=200)
        open(os.path.join(dg, fn), "wb").write(bam_synth.bam_bytes(refs, recs))
    refs, recs = bam_synth.dedup_se_bam(23)
    open(os.path.join(dg, "se.bam"), "wb").write(bam_synth.bam_bytes(refs, recs))
    dup_reads(tiny, tmp)
    for fn, extra in (("map.bam", []), ("map_unm.bam", ["--outSAMunmapped", "Within"])):
        out = os.path.join(tmp, "map_" + fn) + "/"
        subprocess.check_call([STAR, "--genomeDir", "idx", "--readFilesIn", os.path.join(tmp, "dup_1.fq"), os.path.join(tmp, "dup_2.fq"), "--outSAMtype", "BAM",
                               "SortedByCoordinate", "--runThreadN", "1", "--outFileNamePrefix", out] + extra, cwd=tiny, stdout=subprocess.DEVNULL)
        shutil.copy(out + "Aligned.sortedByCoord.out.bam", os.path.join(dg, fn))
    for name, args in SCENARIOS.items():
        out = os.path.join(tmp, "run_" + name) + "/"
        os.makedirs(out)
        subprocess.check_call([STAR] + run_args(args, dg) + ["--outFileNamePrefix", out], cwd=tmp, stdout=subprocess.DEVNULL)
        os.makedirs(os.path.join(dg, name))
        shutil.copy(out + "Processed.out.bam", os.path.join(dg, name, "Processed.out.bam"))
    st = flags_by_name(os.path.join(dg, "P1_ui_n0", "Processed.out.bam"))
    for case, expect in bam_synth.dedup_pinned_records()[1].items():
        for qname, kept in expect:
            assert st[qname] == [kept, kept], (case, qname, st[qname])
    with open(os.path.join(dg, "scenarios.json"), "w") as f:
        json.dump(SCENARIOS, f, indent=1)
    dst = os.path.join(ROOT, "tests", "golden", "dedup.tar.gz")
    with tarfile.open(dst, "w:gz", compresslevel=9) as t:
        t.add(dg, arcname="dedup")
    print("wrote", dst, os.path.getsize(dst), "bytes")
    shutil.rmtree(tmp)


if __name__ == "__main__":
    main()
