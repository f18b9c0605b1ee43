#!/usr/bin/env python3
"""Differential fuzz of the signal tracks: seeded random BAMs (tools/bam_synth.py) through --runMode inputAlignmentsFromBAM of the
unmodified reference (oracle/_ref/STAR) and of ours, every option set; the Signal files must be byte-equal.

  python tools/fuzz_signal.py [first_seed] [n_seeds] [--gpu]      (default: build/signal_check/star_cli_signal, the CPU checker; --gpu: star_b200/bin/STAR)
"""
import os
import subprocess
import sys

import bam_synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref", "STAR")
OPTION_SETS = [
    ["--outWigType", "bedGraph"],
    ["--outWigType", "bedGraph", "--outWigNorm", "None", "--outWigStrand", "Unstranded"],
    ["--outWigType", "wiggle", "read1_5p", "--outWigNorm", "None"],
    ["--outWigType", "wiggle", "read2", "--outWigReferencesPrefix", "chr"],
    ["--outWigType", "bedGraph", "read1_5p", "--outWigReferencesPrefix", "chr"],
]


def check(seed, work, ours, cwd=None):
    """Returns the list of differences (empty: equal) for one seed."""
    refs, recs = bam_synth.random_bam(seed, n=200 + seed % 7 * 60)
    bam = os.path.join(work, "fuzz%d.bam" % seed)
    with open(bam, "wb") as f:
        f.write(bam_synth.bam_bytes(refs, recs))
    diffs = []
    for k, opt in enumerate(OPTION_SETS):
        outs = []
        for tag, exe in (("ref", [REF]), ("ours", ours)):
            pre = os.path.join(work, "f%d_%d_%s." % (seed, k, tag))
            r = subprocess.run(exe + ["--runMode", "inputAlignmentsFromBAM", "--inputBAMfile", bam, "--outFileNamePrefix", pre] + opt, cwd=cwd or work,
                               capture_output=True, text=True)
            if r.returncode:
                diffs.append("seed %d %s %s: exit %d %s" % (seed, opt, tag, r.returncode, r.stderr[-300:]))
            outs.append(pre)
        d = os.path.dirname(outs[0])
        for f in sorted(os.listdir(d)):
            if f.startswith(os.path.basename(outs[0]) + "Signal"):
                tail = f[len(os.path.basename(outs[0])):]
                a, b = open(outs[0] + tail, "rb").read(), open(outs[1] + tail, "rb").read() if os.path.exists(outs[1] + tail) else None
                if a != b:
                    diffs.append("seed %d %s: %s differs" % (seed, opt, tail))
    return diffs


def main():
    import tempfile
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    first, n = (int(args[0]) if args else 1), (int(args[1]) if len(args) > 1 else 50)
    ours = [os.path.join(ROOT, "star_b200", "bin", "STAR")] if "--gpu" in sys.argv else [os.path.join(ROOT, "build", "signal_check", "star_cli_signal")]
    work = tempfile.mkdtemp(prefix="fuzz_signal_")
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
