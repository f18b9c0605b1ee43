#!/usr/bin/env python3
"""Differential fuzz of duplicate marking: seeded random BAMs (tools/bam_synth.py) through --runMode inputAlignmentsFromBAM
--bamRemoveDuplicatesType of the unmodified reference (oracle/_ref/STAR) and of ours, every option set; the decompressed
Processed.out.bam files must be equal.

  python tools/fuzz_dedup.py [first_seed] [n_seeds] [--gpu]      (default: build/dedup_check/star_cli_dedup, the CPU checker; --gpu: star_b200/bin/STAR)
"""
import gzip
import os
import subprocess
import sys

import bam_synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref", "STAR")
OPTION_SETS = [
    ["--bamRemoveDuplicatesType", "UniqueIdentical"],
    ["--bamRemoveDuplicatesType", "UniqueIdenticalNotMulti", "--bamRemoveDuplicatesMate2basesN", "1"],
    ["--bamRemoveDuplicatesType", "UniqueIdentical", "--bamRemoveDuplicatesMate2basesN", "7"],
    ["--bamRemoveDuplicatesType", "UniqueIdenticalNotMulti", "--bamRemoveDuplicatesMate2basesN", "30"],
]


def check(seed, work, ours, cwd=None, env=None):
    """Returns the list of differences (empty: equal) for one seed: a paired BAM, and a single-end one for every third seed."""
    refs, recs = bam_synth.dedup_se_bam(seed, n=150 + seed % 5 * 50) if seed % 3 == 0 else bam_synth.dedup_pe_bam(seed, n_pairs=80 + seed % 7 * 30)
    bam = os.path.join(work, "fuzz%d.bam" % seed)
    with open(bam, "wb") as f:
        f.write(bam_synth.bam_bytes(refs, recs))
    diffs = []
    for k, opt in enumerate(OPTION_SETS):
        outs = []
        for tag, exe in (("ref", [REF]), ("ours", ours)):
            pre = os.path.join(work, "d%d_%d_%s." % (seed, k, tag))
            r = subprocess.run(exe + ["--runMode", "inputAlignmentsFromBAM", "--inputBAMfile", bam, "--outFileNamePrefix", pre] + opt, cwd=cwd or work,
                               capture_output=True, text=True, env=dict(os.environ, **(env or {})))
            if r.returncode:
                diffs.append("seed %d %s %s: exit %d %s" % (seed, opt, tag, r.returncode, r.stderr[-300:]))
            outs.append(pre + "Processed.out.bam")
        if not diffs and gzip.decompress(open(outs[0], "rb").read()) != gzip.decompress(open(outs[1], "rb").read()):
            diffs.append("seed %d %s: Processed.out.bam differs" % (seed, opt))
    return diffs


def main():
    import tempfile
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    first, n = (int(args[0]) if args else 1), (int(args[1]) if len(args) > 1 else 50)
    ours = [os.path.join(ROOT, "star_b200", "bin", "STAR")] if "--gpu" in sys.argv else [os.path.join(ROOT, "build", "dedup_check", "star_cli_dedup")]
    work = tempfile.mkdtemp(prefix="fuzz_dedup_")
    bad = 0
    for seed in range(first, first + n):
        d = check(seed, work, ours)
        bad += bool(d)
        for x in d:
            print(x)
    print("%d of %d seeds differ" % (bad, n))
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
