#!/usr/bin/env python3
"""Timing of adding references at the mapping stage: the bench genome (bench.prepare_genome, GRCh38-sized by default, cached under
STAR_B200_BENCH_DIR) with 92 seeded ERCC-like spikes and a 20 kb copy of a chromosome added (synth.make_spikes), mapping a small set of
pairs from the spikes and the genome:

  STAR --genomeDir idx --genomeFastaFiles spikes.fa --readFilesIn r_1.fq r_2.fq

Prints one JSON line: the wall clock of the run, the phases of the insertion from Log.out (FASTA scan; upload + device re-base, SA search
and SA merge + download, each with the kernel's CUDA-event time; the host sort of the insertion points; the SAindex rebuild), the wall
clock up to the start of mapping, the GPU's name and power limit.  With --reference the unmodified reference (oracle/_ref/STAR) runs the
same command once more for a comparison time, and the SAM records of both are compared (a difference exits non-zero).

  python tools/bench_addref.py [--preset grch38|chr21] [--pairs 20000] [--gpu 0] [--reference]
"""
import argparse
import json
import os
import re
import shutil
import subprocess
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)


def phases(log_path):
    """'[add references, <phase>: <s> s(, kernel <ms> ms)]' lines of Log.out -> {phase: {"wall_s", "kernel_ms"}}."""
    out = {}
    for line in open(log_path):
        m = re.search(r"\[add references, (.+?): ([0-9.e+-]+) s(?:, kernel ([0-9.e+-]+) ms)?\]", line)
        if m:
            out[m.group(1)] = {"wall_s": float(m.group(2)), "kernel_ms": float(m.group(3)) if m.group(3) else None}
    return out


def sam_records(path):
    with open(path, "rb") as f:
        return [l for l in f.read().split(b"\n") if l and not l.startswith(b"@")]


def main():
    import bench  # noqa: E402
    import numpy as np  # noqa: E402
    import synth  # noqa: E402
    ap = argparse.ArgumentParser()
    ap.add_argument("--preset", default="grch38")
    ap.add_argument("--pairs", type=int, default=20000)
    ap.add_argument("--gpu", type=int, default=0)
    ap.add_argument("--reference", action="store_true", help="also run oracle/_ref/STAR (slow at GRCh38 size) and compare the SAM records")
    ap.add_argument("--workdir", default=os.environ.get("STAR_B200_BENCH_DIR", "/tmp/star_b200_bench"))
    a = ap.parse_args()
    wd = os.path.join(a.workdir, a.preset)
    os.makedirs(wd, exist_ok=True)
    chrs, trs, idx, _ = bench.prepare_genome(wd, a.preset, a.gpu)
    spikes = synth.make_spikes(chrs)
    fa = os.path.join(wd, "ar_spikes.fa")
    synth.write_fasta(spikes, fa)
    m1, m2 = synth.make_reads(chrs, trs, a.pairs // 2, read_len=100, mm=0.005, seed=2000)
    s1, s2 = synth.make_reads(spikes, [], a.pairs - a.pairs // 2, read_len=100, mm=0.005, seed=2001, tx_frac=0.0)
    fq1, fq2 = os.path.join(wd, "ar_1.fq"), os.path.join(wd, "ar_2.fq")
    synth.write_fastq(np.concatenate([m1, s1]), fq1)
    synth.write_fastq(np.concatenate([m2, s2]), fq2)
    threads = max(8, min(32, bench.allowed_cpus() // 4))
    args = ["--genomeDir", idx, "--genomeFastaFiles", fa, "--readFilesIn", fq1, fq2]
    arms = {}
    for arm, exe in (("ours", [bench.OUR_STAR, "--runThreadN", str(threads), "--gpuDevice", str(a.gpu)]), ("reference", [bench.REF_STAR, "--runThreadN", str(threads)])):
        if arm == "reference" and (not a.reference or not os.path.exists(bench.REF_STAR)):
            continue
        out = os.path.join(wd, "ar_" + arm)
        shutil.rmtree(out, ignore_errors=True)
        os.makedirs(out)
        t0 = time.time()
        subprocess.check_call(exe + args + ["--outFileNamePrefix", out + "/"], stdout=subprocess.DEVNULL)
        arms[arm] = {"wall_s": time.time() - t0, "dir": out}
    log = os.path.join(arms["ours"]["dir"], "Log.out")
    ph = phases(log)
    res = {"metric": "adding references at the mapping stage", "preset": a.preset, "added_sequences": len(spikes),
           "added_bases": int(sum(len(s) for _, s in spikes)), "pairs": a.pairs, "ours_wall_s": arms["ours"]["wall_s"], "ours_insertion_phases": ph,
           "ours_insertion_wall_s": sum(p["wall_s"] for p in ph.values()), "reference_wall_s": arms.get("reference", {}).get("wall_s"),
           "device": bench.device_info(a.gpu),
           "scope": "one run each; ours_wall_s is the whole command (index load, insertion, engine upload, mapping, output)"}
    rc = 0
    if "reference" in arms:
        same = sam_records(os.path.join(arms["ours"]["dir"], "Aligned.out.sam")) == sam_records(os.path.join(arms["reference"]["dir"], "Aligned.out.sam"))
        res["sam_records_equal"] = bool(same)
        rc = 0 if same else 3
    print(json.dumps(res), flush=True)
    for arm in arms.values():
        shutil.rmtree(arm["dir"], ignore_errors=True)
    return rc


if __name__ == "__main__":
    sys.exit(main())
