#!/usr/bin/env python3
"""Duplicate-marking timing: one coordinate-sorted BAM of synthetic read pairs, a seeded share of them repeated under new names (a few of
the copies with mate 2 changed at its first base), mapped by star_b200/bin/STAR on the bench genome (bench.prepare_genome, GRCh38-sized by
default), then

  STAR --runMode inputAlignmentsFromBAM --inputBAMfile Aligned.sortedByCoord.out.bam --bamRemoveDuplicatesType UniqueIdentical

with ours and with the unmodified reference (oracle/_ref/STAR), on the same file, one run each.  Prints one JSON line: wall clock of both
arms, the device time of our dedup kernels (CUDA events, from Log.out), the GPU's name and power limit.  The decompressed
Processed.out.bam files are compared; a difference exits non-zero.  Work files go to STAR_B200_BENCH_DIR (default /tmp/star_b200_bench).

  python tools/bench_dedup.py [--preset grch38|chr21] [--pairs 131072] [--dup 0.2] [--gpu 0]
"""
import argparse
import gzip
import json
import os
import random
import shutil
import subprocess
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)


def dup_pairs(f1, f2, o1, o2, frac, seed, mismatch=0.05):
    """o1/o2 = f1/f2 with a seeded share `frac` of the pairs repeated under new names; a share `mismatch` of the copies has mate 2 changed
    at its first base."""
    rng = random.Random(seed)
    src = [open(f).read().split("\n") for f in (f1, f2)]
    out = [[], []]
    for i in range(len(src[0]) // 4):
        rec = [src[m][4 * i:4 * i + 4] for m in (0, 1)]
        for m in (0, 1):
            out[m] += rec[m]
        if rng.random() < frac:
            alt = rng.random() < mismatch
            for m in (0, 1):
                h, s, p, q = rec[m]
                if alt and m == 1:
                    s = ("A" if s[0] != "A" else "C") + s[1:]
                out[m] += ["@dup%d_%s" % (i, h[1:]), s, p, q]
    for m, o in ((0, o1), (1, o2)):
        with open(o, "w") as f:
            f.write("\n".join(out[m]) + "\n")


def decompressed_equal(a, b):
    return gzip.decompress(open(a, "rb").read()) == gzip.decompress(open(b, "rb").read())


def main():
    import bench  # noqa: E402
    import synth  # noqa: E402
    ap = argparse.ArgumentParser()
    ap.add_argument("--preset", default="grch38")
    ap.add_argument("--pairs", type=int, default=1 << 17)
    ap.add_argument("--dup", type=float, default=0.2)
    ap.add_argument("--gpu", type=int, default=0)
    ap.add_argument("--workdir", default=os.environ.get("STAR_B200_BENCH_DIR", "/tmp/star_b200_bench"))
    a = ap.parse_args()
    wd = os.path.join(a.workdir, a.preset)
    os.makedirs(wd, exist_ok=True)
    chrs, trs, idx, _ = bench.prepare_genome(wd, a.preset, a.gpu)
    m1, m2 = synth.make_reads(chrs, trs, a.pairs, read_len=100, mm=0.005, seed=1000)   # the reads of bench.py's step
    fq1, fq2 = os.path.join(wd, "dd_1.fq"), os.path.join(wd, "dd_2.fq")
    synth.write_fastq(m1, fq1)
    synth.write_fastq(m2, fq2)
    dup_pairs(fq1, fq2, fq1 + ".dup", fq2 + ".dup", a.dup, 7)
    threads = max(8, min(32, bench.allowed_cpus() // 4))
    out_b = os.path.join(wd, "dd_bam")
    shutil.rmtree(out_b, ignore_errors=True)
    os.makedirs(out_b)
    subprocess.check_call([bench.OUR_STAR, "--genomeDir", idx, "--readFilesIn", fq1 + ".dup", fq2 + ".dup", "--outFileNamePrefix", out_b + "/", "--runThreadN",
                           str(threads), "--outSAMtype", "BAM", "SortedByCoordinate", "--gpuDevice", str(a.gpu)], stdout=subprocess.DEVNULL)
    bam = os.path.join(out_b, "Aligned.sortedByCoord.out.bam")
    dd_args = ["--runMode", "inputAlignmentsFromBAM", "--inputBAMfile", bam, "--bamRemoveDuplicatesType", "UniqueIdentical"]
    arms = {}
    for arm, exe in (("ours", [bench.OUR_STAR, "--runThreadN", str(threads), "--gpuDevice", str(a.gpu)]), ("reference", [bench.REF_STAR])):
        if arm == "reference" and not os.path.exists(bench.REF_STAR):
            continue
        out_s = os.path.join(wd, "dd_" + arm)
        shutil.rmtree(out_s, ignore_errors=True)
        os.makedirs(out_s)
        t0 = time.time()
        subprocess.check_call(exe + dd_args + ["--outFileNamePrefix", out_s + "/"], stdout=subprocess.DEVNULL)
        arms[arm] = {"wall_s": time.time() - t0, "dir": out_s}
    kernel_ms = stage_ms = log = parts = None
    for line in open(os.path.join(arms["ours"]["dir"], "Log.out")):
        if "dedup kernels" in line:
            log = line.split("duplicate removal: ")[1].split(";")[0]
            kernel_ms = float(line.split("dedup kernels")[1].split("ms")[0])
            stage_ms = float(line.split("dedup stage wall")[1].split("ms")[0])
            parts = line.split("ms (", 2)[-1].rstrip(")\n")
    res = {"metric": "duplicate marking wall clock (s)", "preset": a.preset, "pairs": a.pairs, "dup_share": a.dup, "bam_bytes": os.path.getsize(bam),
           "ours_log": log, "ours_wall_s": arms["ours"]["wall_s"], "ours_dedup_stage_ms": stage_ms, "ours_dedup_kernels_ms": kernel_ms,
           "ours_dedup_stage_parts_ms": parts,
           "reference_wall_s": arms.get("reference", {}).get("wall_s"), "device": bench.device_info(a.gpu),
           "scope": "one run each; ours: BAM read + inflate + marking pass + CUDA kernels + BGZF output, kernels from CUDA events"}
    rc = 0
    if "reference" in arms:
        same = decompressed_equal(os.path.join(arms["ours"]["dir"], "Processed.out.bam"), os.path.join(arms["reference"]["dir"], "Processed.out.bam"))
        res["files_equal"] = bool(same)
        rc = 0 if same else 3
    print(json.dumps(res), flush=True)
    for d in ("dd_bam", "dd_ours", "dd_reference"):
        shutil.rmtree(os.path.join(wd, d), ignore_errors=True)
    return rc


if __name__ == "__main__":
    sys.exit(main())
