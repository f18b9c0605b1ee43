#!/usr/bin/env python3
"""Signal-track timing (the ENCODE pipeline's second STAR call): one coordinate-sorted BAM of synthetic read pairs mapped by
star_b200/bin/STAR on the bench genome (bench.prepare_genome, GRCh38-sized by default), then

  STAR --runMode inputAlignmentsFromBAM --inputBAMfile Aligned.sortedByCoord.out.bam --outWigType bedGraph --outWigStrand Stranded

with ours and with the unmodified reference (oracle/_ref/STAR), on the same file, one run each.  Prints one JSON line: wall clock of both
arms, the device time of our signal kernels (CUDA events, from Log.out), the GPU's name and power limit.  The four Signal files are
compared byte for byte; a difference exits non-zero.  Work files go to STAR_B200_BENCH_DIR (default /tmp/star_b200_bench).

  python tools/bench_signal.py [--preset grch38|chr21] [--pairs 131072] [--gpu 0]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
import bench  # noqa: E402
import synth  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--preset", default="grch38")
    ap.add_argument("--pairs", type=int, default=1 << 17)
    ap.add_argument("--gpu", type=int, default=0)
    ap.add_argument("--workdir", default=os.environ.get("STAR_B200_BENCH_DIR", "/tmp/star_b200_bench"))
    a = ap.parse_args()
    wd = os.path.join(a.workdir, a.preset)
    os.makedirs(wd, exist_ok=True)
    chrs, trs, idx, _ = bench.prepare_genome(wd, a.preset, a.gpu)
    m1, m2 = synth.make_reads(chrs, trs, a.pairs, read_len=100, mm=0.005, seed=1000)   # the reads of bench.py's step
    fq1, fq2 = os.path.join(wd, "sig_1.fq"), os.path.join(wd, "sig_2.fq")
    synth.write_fastq(m1, fq1)
    synth.write_fastq(m2, fq2)
    threads = max(8, min(32, bench.allowed_cpus() // 4))
    out_b = os.path.join(wd, "sig_bam")
    shutil.rmtree(out_b, ignore_errors=True)
    os.makedirs(out_b)
    subprocess.check_call([bench.OUR_STAR, "--genomeDir", idx, "--readFilesIn", fq1, fq2, "--outFileNamePrefix", out_b + "/", "--runThreadN", str(threads),
                           "--outSAMtype", "BAM", "SortedByCoordinate", "--gpuDevice", str(a.gpu)], stdout=subprocess.DEVNULL)
    bam = os.path.join(out_b, "Aligned.sortedByCoord.out.bam")
    sig_args = ["--runMode", "inputAlignmentsFromBAM", "--inputBAMfile", bam, "--outWigType", "bedGraph", "--outWigStrand", "Stranded"]
    arms = {}
    for arm, exe in (("ours", [bench.OUR_STAR, "--runThreadN", str(threads), "--gpuDevice", str(a.gpu)]), ("reference", [bench.REF_STAR])):
        if arm == "reference" and not os.path.exists(bench.REF_STAR):
            continue
        out_s = os.path.join(wd, "sig_" + arm)
        shutil.rmtree(out_s, ignore_errors=True)
        os.makedirs(out_s)
        t0 = time.time()
        subprocess.check_call(exe + sig_args + ["--outFileNamePrefix", out_s + "/"], stdout=subprocess.DEVNULL)
        arms[arm] = {"wall_s": time.time() - t0, "dir": out_s}
    kernel_ms = stage_ms = None
    for line in open(os.path.join(arms["ours"]["dir"], "Log.out")):
        if "signal kernels" in line:
            kernel_ms = float(line.split("signal kernels")[1].split("ms")[0])
            stage_ms = float(line.split("signal stage wall")[1].split("ms")[0])
    files = ["Signal.%s.str%d.out.bg" % (k, s) for s in (1, 2) for k in ("Unique", "UniqueMultiple")]
    res = {"metric": "signal tracks wall clock (s)", "preset": a.preset, "bam_pairs": a.pairs, "bam_bytes": os.path.getsize(bam),
           "ours_wall_s": arms["ours"]["wall_s"], "ours_signal_stage_ms": stage_ms, "ours_signal_kernels_ms": kernel_ms,
           "reference_wall_s": arms.get("reference", {}).get("wall_s"), "device": bench.device_info(a.gpu),
           "scope": "one run each; ours: BAM read + inflate + decode + CUDA kernels + formatting, kernels from CUDA events"}
    rc = 0
    if "reference" in arms:
        same = all(open(os.path.join(arms["ours"]["dir"], f), "rb").read() == open(os.path.join(arms["reference"]["dir"], f), "rb").read() for f in files)
        res["files_byte_equal_to_reference"] = bool(same)
        rc = 0 if same else 3
    print(json.dumps(res), flush=True)
    for d in ("sig_bam", "sig_ours", "sig_reference"):
        shutil.rmtree(os.path.join(wd, d), ignore_errors=True)
    return rc


if __name__ == "__main__":
    sys.exit(main())
