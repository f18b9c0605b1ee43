#!/usr/bin/env python3
"""Regenerates tests/golden/edges.tar.xz — needs oracle/_ref/STAR (the unmodified reference, built by oracle/Makefile.ref).

Mapping at the edges of the genome and of the read, where the kernels have special cases that the synthetic reads of tools/synth.py
never reach.  Everything is seeded; only data goes into the archive.

  edges/genome.fa      266 kb, 12 chromosomes (make_genome): chromosomes of 40 and 150 bp, one of exactly 1024 bp (one bin of index
                       A), N runs of 1, 5, 137 and 800 bases (at a chromosome start and at a chromosome end), IUPAC codes, lowercase,
                       two identical chromosomes, a chromosome that is the reverse complement of another, a 3 kb segment with 4 exact
                       copies (one reverse-complemented), a 1 kb segment with 3, a 200 bp element with 20 and a 300 bp element with 60
                       (more than --winAnchorMultimapNmax 50), a 3.5 kb poly-A run and a 5 kb (AC)n run (SA windows > 2048 rows)
  edges/annot.gtf      5 transcripts: junctions next to chromosome starts and ends, inside the 150 bp and the 1024 bp chromosome, and
                       exons of 10-40 bases (shorter than --sjdbOverhang 60)
  edges/idx{A,B}.sha256  digests of every file of the two indexes the reference generated (genomeParameters.txt without its command
                       line); the tests regenerate the indexes with our genomeGenerate and check them against these digests, which keeps
                       4.5 MB of suffix arrays out of the archive:
                       A: --genomeSAindexNbases 8 --genomeChrBinNbits 10 (no annotation; winBinNbits is clamped to 10)
                       B: --genomeSAindexNbases 5 --sjdbGTFfile annot.gtf --sjdbOverhang 60
  edges/se.fq          single-end reads of every category (make_reads), all lengths in one file, read name = <category>.<number>
  edges/pe_{1,2}.fq    pairs of every category, unequal mates included
  edges/ref_<idx>_<set>_<opt>/Aligned.out.sam|SJ.out.tab|Log.final.out   reference outputs, --runThreadN 1, for OPTSETS; the @PG and @CO
                       header lines name the binary "STAR" instead of its path (the tests compare the records, not the header)

The archive is xz-compressed: the 24 SAM files repeat the same reads, which xz's large window finds and gzip's 32 kB window does not
(260 kB instead of 1.3 MB).

Categories: reads at both ends of every chromosome and on both strands, starting every 9 bases from one read length before the
boundary to one read length after it, the part beyond the boundary filled with random bases, the neighbouring chromosome's sequence
or nothing; pairs with a mate over a chromosome end and pairs whose mates protrude past each other by 1-20 bases; reads across every
N run, reads with N at the first, the last and a middle base, all-N reads; reads from the identical chromosomes, the reverse-
complement copy and the repeats; poly-A and (AC)n reads; the length sweep; reads over annotated junctions with overhangs of 1-10
bases.  Every category also comes with mutated copies: a mismatch at the first or the last base, or a 1-base indel 2 bases from an end.

Read-length limit.  The reference reads the sequence line into DEF_readSeqLengthMax+1 = 651 bytes but the quality line into 650
(readLoad.cpp:31, 64): a FASTQ record of 650 bases fails with "quality string length is not equal to sequence length".  The longest
single-end read it accepts is therefore LMAX_SE = 649, and a pair must satisfy l1 + l2 + 1 <= 650 (ReadAlign_oneRead.cpp:38), so the
longest pairs are 324 + 325.  probe_read_limit() checks both facts on every run of this script.  Longer reads are tested against
the engine's own limit (L <= 650 accepted, 651 rejected) through the C-ABI only.

Option sets: every set in OPTSETS is accepted by our parameter parser, so none was dropped.  --outSAMunmapped Within is added to all of
them so that every read has a record.
"""
import hashlib
import io
import lzma
import os
import random
import re
import shutil
import subprocess
import tarfile
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
STAR = os.path.join(ROOT, "oracle", "_ref", "STAR")

LMAX_SE = 649
LMAX_PAIR = (324, 325)
SWEEP = list(range(1, 41)) + [49, 50, 51, 99, 100, 101, 149, 150, 151, 255, 256, 257, 300, 400, 500, 600, LMAX_SE]
PAIR_SWEEP = [(1, 100), (100, 1), (20, 300), (300, 20), (150, 150), (49, 600), (600, 49), LMAX_PAIR, LMAX_PAIR[::-1]]
INDEXES = {"A": ["--genomeSAindexNbases", "8", "--genomeChrBinNbits", "10"],
           "B": ["--genomeSAindexNbases", "5", "--sjdbGTFfile", "annot.gtf", "--sjdbOverhang", "60"]}
OPTSETS = {
    "def": [],
    "noclip": ["--alignSoftClipAtReferenceEnds", "No"],
    "protrude": ["--alignEndsType", "EndToEnd", "--alignEndsProtrude", "10", "ConcordantPair"],
    "multi": ["--outFilterMultimapNmax", "100", "--winAnchorMultimapNmax", "200", "--outSAMattributes", "NH", "HI", "AS", "nM", "NM", "MD"],
    "lmax": ["--seedSearchStartLmax", "12", "--seedSearchLmax", "30"],
    "gap": ["--alignIntronMax", "500", "--alignMatesGapMax", "500"],
}
COMMON = ["--outSAMunmapped", "Within"]
READ_SEED = 21

_COMP = str.maketrans("ACGTNacgtnRYKMSWBDHV", "TGCANtgcanYRMKSWVHDB")


def rc(s):
    return s.translate(_COMP)[::-1]


def make_genome(seed=17):
    """Returns (chroms, transcripts, runs): chroms = [(name, seq)], transcripts = [(chrom index, strand, [(start, end) 0-based half-open])],
    runs = {name: (chrom index, start, end)} of the N runs and the low-complexity runs."""
    rng = random.Random(seed)
    rnd = lambda n: "".join(rng.choices("ACGT", k=n))
    seg4, seg3, el20, el60 = rnd(3000), rnd(1000), rnd(200), rnd(300)

    def body(n, pastes):
        s = list(rnd(n))
        for p, x in pastes:
            s[p:p + len(x)] = x
        return "".join(s)

    def spread(el, k, start, step):
        return [(start + i * step, el) for i in range(k)]

    chr1 = body(60000, [(10000, seg4), (20000, seg3)] + spread(el20, 8, 24000, 600) + spread(el60, 25, 30000, 700))
    chr1 = chr1[:3000] + chr1[3000:3500].lower() + chr1[3500:4000] + "R" + chr1[4001:4500] + "YKM" + chr1[4503:5000] + "SWBDHV" + chr1[5006:]
    ns = body(30000, spread(el60, 10, 3000, 700))
    ns = "N" * 5 + ns[5:9000] + "N" + ns[9001:15000] + "N" * 137 + ns[15137:29200] + "N" * 800
    dup = body(8000, [(4000, seg3)])
    fwd = body(8000, [])
    homo = rnd(2000) + "A" * 3500 + rnd(2000) + "AC" * 2500 + rnd(2000)
    m2 = body(90000, [(20000, seg4), (40000, rc(seg4))] + spread(el20, 8, 50000, 600) + spread(el60, 25, 60000, 700))
    last = body(40000, [(10000, seg4)] + spread(el20, 4, 20000, 600))
    chroms = [("chr1", chr1), ("chrTiny", rnd(40)), ("chrS150", rnd(150)), ("chrBin", rnd(1024)), ("chrNs", ns), ("chrDupA", dup),
              ("chrDupB", dup), ("chrFwd", fwd), ("chrRev", rc(fwd)), ("chrHomo", homo), ("chrM2", m2), ("chrLast", last)]
    L = len(last)
    trs = [(0, "+", [(0, 30), (200, 400), (600, 640), (1000, 1200)]),
           (11, "-", [(L - 1200, L - 1000), (L - 700, L - 660), (L - 400, L - 370), (L - 25, L)]),
           (2, "+", [(0, 50), (100, 150)]),
           (3, "+", [(0, 300), (500, 520), (700, 1024)]),
           (10, "+", [(5000, 5200), (5400, 5410), (5600, 5800)])]
    seqs = [list(s) for _, s in chroms]
    for ci, strand, ex in trs:   # canonical motifs: GT..AG on + (CT..AC in genome orientation on -)
        for (a0, b0), (a1, b1) in zip(ex, ex[1:]):
            d, a = ("GT", "AG") if strand == "+" else ("CT", "AC")
            seqs[ci][b0:b0 + 2] = d
            seqs[ci][a1 - 2:a1] = a
    chroms = [(n, "".join(s)) for (n, _), s in zip(chroms, seqs)]
    runs = {"N5": (4, 0, 5), "N1": (4, 9000, 9001), "N137": (4, 15000, 15137), "N800": (4, 29200, 30000),
            "IUPAC1": (0, 4000, 4001), "IUPAC3": (0, 4500, 4503), "IUPAC6": (0, 5000, 5006),
            "polyA": (9, 2000, 5500), "AC": (9, 7500, 12500)}
    repeats = {"seg4": [(0, 10000, 13000), (10, 20000, 23000), (10, 40000, 43000), (11, 10000, 13000)],
               "seg3": [(0, 20000, 21000), (5, 4000, 5000), (6, 4000, 5000)],
               "el20": [(0, 24000 + i * 600, 24200 + i * 600) for i in range(8)],
               "el60": [(0, 30000 + i * 700, 30300 + i * 700) for i in range(25)]}
    return chroms, trs, dict(runs, **{"rep_" + k: v[0] for k, v in repeats.items()})


class ReadSets:
    def __init__(self, chroms, seed):
        self.chroms = chroms
        self.rng = random.Random(seed)
        self.se, self.pe = [], []

    def rnd(self, n):
        return "".join(self.rng.choices("ACGT", k=n))

    def window(self, ci, p, n, fill):
        """Bases [p, p+n) of chromosome ci; the part outside the chromosome is random ('rand'), the neighbouring chromosome's sequence
        ('nbr') or left out ('cut')."""
        s = self.chroms[ci][1]
        left, mid, right = "", s[max(0, p):max(0, min(len(s), p + n))], ""
        nl, nr = max(0, min(n, -p)), max(0, p + n - max(len(s), p))
        if fill == "rand":
            left, right = self.rnd(nl), self.rnd(nr)
        elif fill == "nbr":
            prv = self.chroms[ci - 1][1] if ci > 0 else ""
            nxt = self.chroms[ci + 1][1] if ci + 1 < len(self.chroms) else ""
            left = (self.rnd(nl) + prv)[-nl:] if nl else ""
            right = (nxt + self.rnd(nr))[:nr] if nr else ""
        return left + mid + right

    def mutate(self, s, grow=True):
        k = self.rng.randrange(4) if len(s) >= 6 else self.rng.randrange(2)
        if k == 2 and not grow:   # (no insertion at the read-length limit)
            k = 3
        other = lambda c: self.rng.choice([b for b in "ACGT" if b != c.upper()])
        if k == 0:
            return other(s[0]) + s[1:]
        if k == 1:
            return s[:-1] + other(s[-1])
        if k == 2:
            return s[:2] + self.rng.choice("ACGT") + s[2:]
        return s[:-3] + s[-2:]

    def add(self, cat, s, m2=None, mut=True):
        s = s.upper()
        if not s or (m2 is not None and not m2):
            return
        if m2 is None:
            self.se.append((cat, s))
            if mut:
                self.se.append((cat + "M", self.mutate(s, len(s) < LMAX_SE)))
        else:
            m2 = m2.upper()
            self.pe.append((cat, s, m2))
            if mut:
                grow = len(s) + len(m2) + 2 < sum(LMAX_PAIR)
                self.pe.append((cat + "M", self.mutate(s, grow), self.mutate(m2, False)))

    def interior(self, n):
        """A window of unique sequence, away from repeats, runs and transcripts."""
        ci, a, b = self.rng.choice(((0, 48000, 59000), (10, 6000, 19000), (11, 23000, 38000)))
        return ci, self.rng.randrange(a, b - n)


def make_reads(chroms, trs, runs, seed=READ_SEED, step=9):
    """Returns (se, pe): se = [(category, seq)], pe = [(category, seq1, seq2)]."""
    R = ReadSets(chroms, seed)
    fills = ("rand", "nbr", "cut")
    k = 0
    # ---- chromosome ends, both strands, three fills
    for ci, (_, s) in enumerate(chroms):
        n = 100
        starts = sorted(set(list(range(-n + 10, n + 1, step)) + [0]))
        ends = sorted(set(list(range(len(s) - 2 * n, len(s) + 1 - 10, step)) + [len(s) - n]))
        for p in starts + ends:
            for strand in (0, 1):
                w = R.window(ci, p, n, fills[k % 3])
                k += 1
                R.add("end", w if strand == 0 else rc(w), mut=(k % 3 == 0))
    # ---- pairs with a mate over a chromosome end; mates protruding past each other
    for ci, (_, s) in enumerate(chroms):
        for d in range(-60, 41, 10):
            f = fills[k % 3]
            k += 1
            m1, m2 = R.window(ci, d, 100, f), rc(R.window(ci, d + 150, 100, f))
            R.add("pend", m1, m2, mut=(k % 2 == 0))
            R.add("pend", m2, m1, mut=False)
            q = len(s) - 100 + d + 20
            m1, m2 = R.window(ci, q - 150, 100, f), rc(R.window(ci, q, 100, f))
            R.add("pend", m1, m2, mut=(k % 2 == 1))
            R.add("pend", m2, m1, mut=False)
    for d in range(1, 21):
        ci, p = R.interior(200)
        p += 30
        R.add("prot", R.window(ci, p, 100, "rand"), rc(R.window(ci, p - d, 100, "rand")), mut=(d % 2 == 0))
        R.add("prot", R.window(ci, p, 100, "rand"), rc(R.window(ci, p - d, 80, "rand")), mut=False)
        R.add("prot", R.window(0, d, 100, "rand"), rc(R.window(0, 0, 100, "rand")), mut=False)   # at the genome's first base
        L11 = len(chroms[11][1])
        R.add("prot", R.window(11, L11 - 100, 100, "rand"), rc(R.window(11, L11 - 100 + d, 100, "rand")), mut=False)
    # ---- N runs, IUPAC codes, N inside reads, all-N reads
    for name, (ci, a, b) in runs.items():
        if not (name.startswith("N") or name.startswith("IUPAC")):
            continue
        for p in (a - 95, a - 50, a - 10, b - 90, b - 50, b - 5):
            for strand in (0, 1):
                w = R.window(ci, p, 100, "nbr")
                R.add("nrun", w if strand == 0 else rc(w))
        ci2 = ci
        R.add("nrun", R.window(ci2, a - 100, 100, "rand"), rc(R.window(ci2, b + 20, 100, "rand")))
    for i in range(12):
        ci, p = R.interior(150)
        w = list(chroms[ci][1][p:p + 100].upper())
        pos = [0, 99, 50, 1 + i * 7][i % 4]
        w[pos] = "N"
        w = "".join(w)
        R.add("nread", w if i % 2 == 0 else rc(w))
        m2 = rc(chroms[ci][1][p + 150:p + 250])
        R.add("nread", w, m2[:-1] + "N" if i % 2 else "N" + m2[1:])
    for n in (100, 30, 1):
        R.add("alln", "N" * n, mut=False)
        R.add("alln", "N" * n, "N" * n, mut=False)
    ci, p = R.interior(400)
    R.add("alln", chroms[ci][1][p:p + 100], "N" * 100, mut=False)
    # ---- repeats: identical chromosomes, reverse-complement copy, exact repeats with 2, 3, 4, 20, 60 loci
    for name, (ci, a, b) in [("dup", (5, 0, 8000)), ("rev", (7, 0, 8000)), ("rev", (8, 0, 8000)), ("seg3", runs["rep_seg3"]),
                             ("seg4", runs["rep_seg4"]), ("el20", runs["rep_el20"]), ("el60", runs["rep_el60"])]:
        for i in range(10):
            n = 100 if i < 7 else (50 if i == 7 else min(b - a, 150))
            p = a + R.rng.randrange(0, max(1, b - a - n + 1))
            w = chroms[ci][1][p:p + n]
            R.add("rep" + name, w if i % 2 == 0 else rc(w))
        for i in range(4):   # both mates inside the repeat, then one mate outside it
            n = 80 if b - a <= 300 else 100
            p = a + R.rng.randrange(0, max(1, b - a - 2 * n + 1))
            q = min(b - n, p + 150)
            R.add("rep" + name, chroms[ci][1][p:p + n], rc(chroms[ci][1][q:q + n]))
            R.add("rep" + name, chroms[ci][1][p:p + n], rc(R.window(ci, b + 50, n, "rand")), mut=False)
    # ---- poly-A and (AC)n
    for name in ("polyA", "AC"):
        ci, a, b = runs[name]
        for p in (a - 90, a - 40, a, a + 1, a + 500, b - 100, b - 99, b - 60, b - 10):
            for n in (50, 100, 150):
                w = R.window(ci, p, n, "rand")
                R.add("homo", w if p % 2 == 0 else rc(w), mut=(n == 100))
        R.add("homo", R.window(ci, a + 300, 100, "rand"), rc(R.window(ci, a + 500, 100, "rand")))
        R.add("homo", R.window(ci, a - 60, 100, "rand"), rc(R.window(ci, b - 40, 100, "rand")))
    # ---- length sweep (all lengths in one file) and pairs of unequal mates
    for n in SWEEP:
        for strand in (0, 1):
            ci, p = R.interior(n)
            w = chroms[ci][1][p:p + n]
            R.add("len%d" % n, w if strand == 0 else rc(w), mut=(n >= 8 and strand == 0))
    for l1, l2 in PAIR_SWEEP:
        frag = max(l1, l2) + 60
        ci, p = R.interior(frag)
        s = chroms[ci][1]
        R.add("plen%d_%d" % (l1, l2), s[p:p + l1], rc(s[p + frag - l2:p + frag]), mut=(min(l1, l2) >= 8))
    # ---- annotated junctions with overhangs of 1-10 bases (transcript sequence: short exons make reads span several junctions)
    for ci, strand, ex in trs:
        t = "".join(chroms[ci][1][a:b] for a, b in ex)
        acc = 0
        for a, b in ex[:-1]:
            acc += b - a
            for o in range(1, 11):
                for side in (0, 1):
                    n = 100
                    p = acc - o if side == 0 else acc + o - n
                    w = t[max(0, p):max(0, p + n)]
                    R.add("junc", w if o % 2 == 0 else rc(w), mut=(o == 5))
            R.add("junc", t[max(0, acc - 50):acc + 50], rc(t[-100:]), mut=False)
    return R.se, R.pe


def write_fasta(chroms, path):
    with open(path, "w") as f:
        for name, s in chroms:
            f.write(">" + name + "\n")
            for i in range(0, len(s), 60):
                f.write(s[i:i + 60] + "\n")


def write_gtf(chroms, trs, path):
    with open(path, "w") as f:
        for k, (ci, strand, ex) in enumerate(trs):
            for j, (a, b) in enumerate(ex):
                f.write('%s\tedge\texon\t%d\t%d\t.\t%s\t.\tgene_id "G%d"; transcript_id "T%d";\n' % (chroms[ci][0], a + 1, b, strand, k, k))


def write_reads(se, pe, d, prefix=""):
    with open(os.path.join(d, prefix + "se.fq"), "w") as f:
        for i, (cat, s) in enumerate(se):
            f.write("@%s.%05d\n%s\n+\n%s\n" % (cat, i, s, "I" * len(s)))
    with open(os.path.join(d, prefix + "pe_1.fq"), "w") as f1, open(os.path.join(d, prefix + "pe_2.fq"), "w") as f2:
        for i, (cat, a, b) in enumerate(pe):
            f1.write("@%s.%05d\n%s\n+\n%s\n" % (cat, i, a, "I" * len(a)))
            f2.write("@%s.%05d\n%s\n+\n%s\n" % (cat, i, b, "I" * len(b)))


def run(cmd, cwd, check=True):
    r = subprocess.run(cmd, cwd=cwd, stdout=subprocess.DEVNULL, stderr=subprocess.PIPE)
    if check and r.returncode:
        raise RuntimeError("%s failed (%d): %s" % (" ".join(cmd), r.returncode, r.stderr.decode()[-2000:]))
    return r.returncode


def align(d, idx, files, out, extra):
    os.makedirs(os.path.join(d, out))
    run([STAR, "--genomeDir", idx, "--readFilesIn"] + files + ["--outFileNamePrefix", out + "/", "--runThreadN", "1"] + COMMON + extra, d)
    sam = os.path.join(d, out, "Aligned.out.sam")
    with open(sam) as f:
        lines = f.read().split("\n")
    with open(sam, "w") as f:
        f.write("\n".join(l.replace(STAR, "STAR") if l.startswith("@PG") or l.startswith("@CO") else l for l in lines))
    for f in os.listdir(os.path.join(d, out)):
        if f not in ("Aligned.out.sam", "SJ.out.tab", "Log.final.out"):
            p = os.path.join(d, out, f)
            shutil.rmtree(p) if os.path.isdir(p) else os.remove(p)


def probe_read_limit(d, chroms):
    """The longest read and pair the reference accepts (module docstring)."""
    s = chroms[0][1][6000:7000].upper()
    out = {}
    for tag, mates in (("se649", [s[:649]]), ("se650", [s[:650]]), ("pe324_325", [s[:324], rc(s[400:725])]), ("pe325_325", [s[:325], rc(s[400:725])])):
        files = []
        for m, x in enumerate(mates):
            fn = os.path.join(d, "probe_%s_%d.fq" % (tag, m))
            open(fn, "w").write("@p\n%s\n+\n%s\n" % (x, "I" * len(x)))
            files.append(fn)
        pd = os.path.join(d, "probe_" + tag)
        os.makedirs(pd)
        out[tag] = run([STAR, "--genomeDir", "idxA", "--readFilesIn"] + files + ["--outFileNamePrefix", pd + "/", "--runThreadN", "1"], d, check=False)
        shutil.rmtree(pd)
        for fn in files:
            os.remove(fn)
    assert out["se649"] == 0 and out["pe324_325"] == 0, out
    assert out["se650"] != 0 and out["pe325_325"] != 0, out


def sam_records(path):
    recs = []
    for l in open(path):
        if l.startswith("@"):
            continue
        f = l.rstrip("\n").split("\t")
        tags = dict((t[:2], t[5:]) for t in f[11:])
        recs.append((f[0], int(f[1]), f[2], int(f[3]), f[5], tags))
    return recs


def ref_end(pos, cigar):
    return pos - 1 + sum(int(n) for n, op in re.findall(r"(\d+)([MDN=X])", cigar))


def check_coverage(d, chroms):
    """The fixture reaches the edges it is for (module docstring); asserts on the reference's own output."""
    clen = {n: len(s) for n, s in chroms}

    def recs(idx, rs, opt):
        return sam_records(os.path.join(d, "ref_%s_%s_%s" % (idx, rs, opt), "Aligned.out.sam"))

    for idx in INDEXES:
        for rs in ("se", "pe"):
            r = [x for x in recs(idx, rs, "def") if not x[1] & 4]
            assert any(x[3] == 1 for x in r), (idx, rs, "POS 1")
            assert any(ref_end(x[3], x[4]) == clen[x[2]] for x in r), (idx, rs, "chromosome's last base")
            assert any(x[3] == 1 and re.match(r"^\d+S", x[4]) for x in r), (idx, rs, "soft clip at a chromosome start")
            assert any(ref_end(x[3], x[4]) == clen[x[2]] and x[4].endswith("S") for x in r), (idx, rs, "soft clip at a chromosome end")
            mapped = {x[0] for x in r}
            unm_noclip = {x[0] for x in recs(idx, rs, "noclip") if x[1] & 4}
            assert mapped & unm_noclip, (idx, rs, "reads unmapped only without soft clips at reference ends")
            for nh, chrs in ((2, {"chrDupA", "chrDupB"}), (2, {"chrFwd", "chrRev"}), (3, None), (4, None)):
                assert any(x[5].get("NH") == str(nh) and (chrs is None or x[2] in chrs) for x in r), (idx, rs, "NH", nh, chrs)
            assert any(x[1] & 4 and x[5].get("uT") == "3" for x in recs(idx, rs, "def")), (idx, rs, "too many loci")
            assert any(int(x[5].get("NH", 0)) > 50 for x in recs(idx, rs, "multi") if not x[1] & 4), (idx, rs, "more than 50 loci")
    r = [x for x in recs("A", "se", "def") if not x[1] & 4]
    mapped_len = {int(x[0].split(".")[0][3:]) for x in r if re.match(r"len\d+\.", x[0])}
    missing = [n for n in SWEEP if n >= 20 and n not in mapped_len]
    assert not missing, ("sweep lengths never mapped", missing)
    rb = [x for x in recs("B", "se", "def") if not x[1] & 4 and x[0].startswith("junc")]
    assert any("N" in x[4] for x in rb), "no junction read spliced on index B"


def index_digests(idx):
    """name -> sha256 of every file of a genome directory (genomeParameters.txt without its command line)."""
    out = {}
    for name in sorted(os.listdir(idx)):
        data = open(os.path.join(idx, name), "rb").read()
        if name == "genomeParameters.txt":
            data = data.split(b"\n", 1)[1]
        out[name] = hashlib.sha256(data).hexdigest()
    return out


def _tar_filter(ti):
    ti.mtime, ti.uid, ti.gid, ti.uname, ti.gname = 0, 0, 0, "", ""
    return ti


def main():
    tmp = tempfile.mkdtemp(prefix="golden_edges_")
    d = os.path.join(tmp, "edges")
    os.makedirs(d)
    chroms, trs, runs = make_genome()
    write_fasta(chroms, os.path.join(d, "genome.fa"))
    write_gtf(chroms, trs, os.path.join(d, "annot.gtf"))
    for name, args in INDEXES.items():
        run([STAR, "--runMode", "genomeGenerate", "--genomeDir", "idx" + name, "--genomeFastaFiles", "genome.fa", "--runThreadN", "4",
             "--outFileNamePrefix", "gen_"] + args, d)
        os.remove(os.path.join(d, "idx" + name, "Log.out"))
    for f in os.listdir(d):
        if f.startswith("gen_"):
            p = os.path.join(d, f)
            shutil.rmtree(p) if os.path.isdir(p) else os.remove(p)
    probe_read_limit(d, chroms)
    se, pe = make_reads(chroms, trs, runs)
    write_reads(se, pe, d)
    for idx in INDEXES:
        for opt, extra in OPTSETS.items():
            align(d, "idx" + idx, ["se.fq"], "ref_%s_se_%s" % (idx, opt), extra)
            align(d, "idx" + idx, ["pe_1.fq", "pe_2.fq"], "ref_%s_pe_%s" % (idx, opt), extra)
    check_coverage(d, chroms)
    for idx in INDEXES:
        with open(os.path.join(d, "idx%s.sha256" % idx), "w") as f:
            for name, h in index_digests(os.path.join(d, "idx" + idx)).items():
                f.write("%s\t%s\n" % (name, h))
        shutil.rmtree(os.path.join(d, "idx" + idx))
    dst = os.path.join(ROOT, "tests", "golden", "edges.tar.xz")
    buf = io.BytesIO()
    with tarfile.open(fileobj=buf, mode="w", format=tarfile.GNU_FORMAT) as t:
        for base, dirs, files in sorted(os.walk(d)):
            dirs.sort()
            for f in sorted(files):
                p = os.path.join(base, f)
                t.add(p, arcname=os.path.relpath(p, tmp), filter=_tar_filter)
    with open(dst, "wb") as f:
        f.write(lzma.compress(buf.getvalue(), format=lzma.FORMAT_XZ, preset=9 | lzma.PRESET_EXTREME))
    print("wrote %s: %d bytes, %d single-end reads, %d pairs" % (dst, os.path.getsize(dst), len(se), len(pe)))
    shutil.rmtree(tmp)


if __name__ == "__main__":
    main()
