#!/usr/bin/env python3
"""Seeded synthetic genome / annotation / paired-end read generator (SURVEY.md §8(d), self-contained tier).

No real genome (chr21 / GRCh38 / GENCODE) exists in the build container or on the GPU box and
there is no network, so every parity fixture and every bench workload is produced by this
script from fixed seeds.  It only produces INPUT files (FASTA, GTF, FASTQ); indices are built
from them by the reference's own `--runMode genomeGenerate` (oracle/_ref/STAR) because index
construction is out of scope for this repository (SURVEY.md §2, row "Index build").

Presets
    tiny   : 3 chromosomes (60/40/25 kb), 40 genes            -> committed golden fixture
    small  : 3 chromosomes (2.0/1.2/0.8 Mb), 300 genes        -> fast GPU parity runs
    chr21  : 3 chromosomes (28/12/6.7 Mb = 46.7 Mb), 2000 genes, repeat families, N block
             (the survey's chr21-sized stand-in; BASELINE.json configs[0] analogue)
    grch38 : 24 chromosomes with the GRCh38 primary-assembly lengths (3.09 Gb), ~27 k multi-exon genes -> ~350 k annotated
             junctions, the chr21 repeat families scaled x66, one 100 kb N block per chromosome
             (SURVEY.md §8(d) tier 2: the GRCh38 + GENCODE sized stand-in for BASELINE.json configs[1..4]; index ~29 GB)

Reads: fragment length 300 (fixed), 50 % from spliced transcripts / 50 % from the genome,
random strand, mate1 = first L bases, mate2 = reverse complement of the last L bases,
substitution rate --mm, optional indels / N bases / junk pairs, constant quality 'I',
names r%09d so that records are fixed-width and can be written vectorised.
"""
import argparse
import os
import random
import sys

import numpy as np

ACGT = np.frombuffer(b"ACGT", dtype=np.uint8)
COMP = np.zeros(256, dtype=np.uint8)
for a, b in zip(b"ACGTN", b"TGCAN"):
    COMP[a] = b

PRESETS = {
    #            chromosome lengths             genes  repeat families (len, copies, divergence)     N block
    "tiny":  dict(chrs=[60_000, 40_000, 25_000], genes=40,
                  reps=[(300, 20, 0.05), (1000, 6, 0.02)], nblock=(30_000, 500)),
    "small": dict(chrs=[2_000_000, 1_200_000, 800_000], genes=300,
                  reps=[(300, 200, 0.05), (6000, 12, 0.02), (1000, 60, 0.10)], nblock=(1_000_000, 5_000)),
    "chr21": dict(chrs=[28_000_000, 12_000_000, 6_700_000], genes=2000,
                  reps=[(300, 3000, 0.05), (6000, 200, 0.02), (1000, 1000, 0.10)], nblock=(10_000_000, 50_000)),
    # GRCh38 primary assembly chromosome lengths (chr1..22, X, Y)
    "grch38": dict(chrs=[248956422, 242193529, 198295559, 190214555, 181538259, 170805979, 159345973, 145138636, 138394717,
                         133797422, 135086622, 133275309, 114364328, 107043718, 101991189, 90338345, 83257441, 80373285,
                         58617616, 64444167, 46709983, 50818468, 156040895, 57227415], genes=27000,
                   reps=[(300, 200_000, 0.05), (6000, 13_000, 0.02), (1000, 66_000, 0.10)], nblock=None, big=True),
    # a 1/8 scale model of the same construction (386 Mb): used to exercise the large-genome code paths quickly
    "grch38_8th": dict(chrs=[x // 8 for x in [248956422, 242193529, 198295559, 190214555, 181538259, 170805979, 159345973, 145138636,
                                              138394717, 133797422, 135086622, 133275309, 114364328, 107043718, 101991189, 90338345,
                                              83257441, 80373285, 58617616, 64444167, 46709983, 50818468, 156040895, 57227415]],
                       genes=3400, reps=[(300, 25_000, 0.05), (6000, 1_600, 0.02), (1000, 8_000, 0.10)], nblock=None, big=True),
}


def _make_genome_big(p, seed):
    """Large presets: same construction as make_genome, generated in blocks / whole families at a time (seconds per Gb)."""
    rng = np.random.default_rng(seed)
    total = sum(p["chrs"])
    g = np.empty(total, dtype=np.uint8)
    lut = np.tile(ACGT, 64)   # byte -> base
    step = 1 << 28
    for lo in range(0, total, step):
        hi = min(total, lo + step)
        g[lo:hi] = lut[rng.integers(0, 256, size=hi - lo, dtype=np.uint8)]
    for (rlen, copies, div) in p["reps"]:
        cons = ACGT[rng.integers(0, 4, size=rlen, dtype=np.uint8)]
        batch = max(1, (64 << 20) // rlen)
        for c0 in range(0, copies, batch):
            nb = min(batch, copies - c0)
            starts = rng.integers(0, total - rlen, size=nb)
            m = np.broadcast_to(cons, (nb, rlen)).copy()
            mut = rng.random((nb, rlen)) < div
            m[mut] = ACGT[rng.integers(0, 4, size=int(mut.sum()), dtype=np.uint8)]
            flip = rng.random(nb) < 0.5
            m[flip] = COMP[m[flip][:, ::-1]]
            for k in range(nb):
                s = int(starts[k])
                g[s:s + rlen] = m[k]
    chrs = []
    off = 0
    for i, L in enumerate(p["chrs"]):
        name = "chr%d" % (i + 1) if i < 22 else ("chrX" if i == 22 else "chrY")
        seq = g[off:off + L]
        nb_start = int(L * 0.4)
        seq[nb_start:nb_start + min(100_000, L // 50)] = ord("N")   # one N block per chromosome (centromere stand-in)
        chrs.append((name, seq))
        off += L
    return chrs


def _make_annotation_big(chrs, p, seed):
    """Large presets: genes laid out left to right on every chromosome (random gaps), 4-24 exons of 80-400 bp, introns 200-8000 bp."""
    rnd = random.Random(seed)
    total = sum(len(c[1]) for c in chrs)
    avg_span = 13 * 4100 + 14 * 240
    gap_avg = max(2000, total // p["genes"] - avg_span)
    dcode = {"GTAG": (b"GT", b"AG"), "GCAG": (b"GC", b"AG"), "ATAC": (b"AT", b"AC")}
    trs = []
    for ci, (_, seq) in enumerate(chrs):
        L = len(seq)
        pos = 1000 + rnd.randint(0, gap_avg)
        while True:
            n_ex = rnd.randint(4, 24)
            ex_len = [rnd.randint(80, 400) for _ in range(n_ex)]
            in_len = [rnd.randint(200, 8000) for _ in range(n_ex - 1)]
            span = sum(ex_len) + sum(in_len)
            s = pos
            e = s + span
            if e + 1000 >= L:
                break
            pos = e + 500 + rnd.randint(0, 2 * gap_avg)
            if (seq[s:e:97] == ord("N")).any() or (seq[s:e] == ord("N")).any():
                continue
            exons = []
            q = s
            for k in range(n_ex):
                exons.append((q, q + ex_len[k]))
                q += ex_len[k]
                if k < n_ex - 1:
                    q += in_len[k]
            strand = "+" if rnd.random() < 0.5 else "-"
            for k in range(n_ex - 1):
                i0 = exons[k][1]
                i1 = exons[k + 1][0]
                r = rnd.random()
                if r < 0.80:
                    d, a = dcode["GTAG"]
                elif r < 0.88:
                    d, a = dcode["GCAG"]
                elif r < 0.92:
                    d, a = dcode["ATAC"]
                else:
                    continue
                if strand == "+":
                    seq[i0:i0 + 2] = np.frombuffer(d, dtype=np.uint8)
                    seq[i1 - 2:i1] = np.frombuffer(a, dtype=np.uint8)
                else:
                    seq[i0:i0 + 2] = COMP[np.frombuffer(a, dtype=np.uint8)[::-1]]
                    seq[i1 - 2:i1] = COMP[np.frombuffer(d, dtype=np.uint8)[::-1]]
            trs.append(dict(chr=ci, strand=strand, exons=exons, gid="G%06d" % len(trs)))
    return trs


def make_genome(preset, seed=7):
    """Returns list of (name, uint8 ASCII array)."""
    p = PRESETS[preset]
    if p.get("big"):
        return _make_genome_big(p, seed)
    rng = np.random.default_rng(seed)
    total = sum(p["chrs"])
    g = ACGT[rng.integers(0, 4, size=total, dtype=np.uint8)]
    # repeat families: one consensus each, pasted with per-copy divergence at random places
    for (rlen, copies, div) in p["reps"]:
        cons = ACGT[rng.integers(0, 4, size=rlen, dtype=np.uint8)]
        starts = rng.integers(0, total - rlen, size=copies)
        for s in starts:
            c = cons.copy()
            mut = rng.random(rlen) < div
            c[mut] = ACGT[rng.integers(0, 4, size=int(mut.sum()), dtype=np.uint8)]
            if rng.random() < 0.5:
                c = COMP[c[::-1]]
            g[s:s + rlen] = c
    nb_start, nb_len = p["nblock"]
    g[nb_start:nb_start + nb_len] = ord("N")
    chrs = []
    off = 0
    for i, L in enumerate(p["chrs"]):
        chrs.append(("chr%d" % (i + 1), g[off:off + L]))
        off += L
    return chrs


def make_annotation(chrs, preset, seed=3):
    """Returns list of transcripts: dict(chr index, strand, exons=[(start0, end0_exclusive)...] ascending)."""
    p = PRESETS[preset]
    if p.get("big"):
        return _make_annotation_big(chrs, p, seed)
    rnd = random.Random(seed)
    intron_max = 20_000 if preset != "tiny" else 3_000
    trs = []
    tries = 0
    occupied = [[] for _ in chrs]
    while len(trs) < p["genes"] and tries < 100 * p["genes"]:
        tries += 1
        ci = rnd.choices(range(len(chrs)), weights=[len(c[1]) for c in chrs])[0]
        n_ex = rnd.randint(3, 8)
        ex_len = [rnd.randint(80, 400) for _ in range(n_ex)]
        in_len = [rnd.randint(200, intron_max) for _ in range(n_ex - 1)]
        span = sum(ex_len) + sum(in_len)
        L = len(chrs[ci][1])
        if span + 2000 >= L:
            continue
        s = rnd.randint(1000, L - span - 1000)
        e = s + span
        if any(not (e + 500 < a or b + 500 < s) for a, b in occupied[ci]):
            continue
        seq = chrs[ci][1]
        if (seq[s:e] == ord("N")).any():
            continue
        occupied[ci].append((s, e))
        exons = []
        pos = s
        for k in range(n_ex):
            exons.append((pos, pos + ex_len[k]))
            pos += ex_len[k]
            if k < n_ex - 1:
                pos += in_len[k]
        strand = "+" if rnd.random() < 0.5 else "-"
        # plant canonical motifs in most introns so that the junctions look real:
        # + strand GT..AG, - strand CT..AC; ~8 % GC-AG, ~4 % AT-AC, ~8 % left as random (non-canonical)
        for k in range(n_ex - 1):
            i0 = exons[k][1]
            i1 = exons[k + 1][0]
            r = rnd.random()
            if r < 0.80:
                d, a = (b"GT", b"AG")
            elif r < 0.88:
                d, a = (b"GC", b"AG")
            elif r < 0.92:
                d, a = (b"AT", b"AC")
            else:
                continue
            if strand == "+":
                seq[i0:i0 + 2] = np.frombuffer(d, dtype=np.uint8)
                seq[i1 - 2:i1] = np.frombuffer(a, dtype=np.uint8)
            else:
                seq[i0:i0 + 2] = COMP[np.frombuffer(a, dtype=np.uint8)[::-1]]
                seq[i1 - 2:i1] = COMP[np.frombuffer(d, dtype=np.uint8)[::-1]]
        trs.append(dict(chr=ci, strand=strand, exons=exons, gid="G%05d" % len(trs)))
    return trs


def make_spikes(chrs, n=92, seed=92, copy_len=20000):
    """References to add at the mapping stage: n ERCC-like spikes of 400-2000 random bases (a third end in the same 30-base poly-A tail) and
    a copy of copy_len bases of the first chromosome.  Returns list of (name, uint8 ASCII array), the copy last."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        s = ACGT[rng.integers(0, 4, size=int(rng.integers(400, 2001)), dtype=np.uint8)]
        if i % 3 == 0:
            s[-30:] = ord("A")
        out.append(("ERCC-%05d" % (i + 1), s))
    seq = chrs[0][1]
    p = int(rng.integers(0, len(seq) - copy_len))
    while np.any(seq[p:p + copy_len] == ord("N")):
        p = int(rng.integers(0, len(seq) - copy_len))
    out.append(("copy_%s_%d" % (chrs[0][0], p + 1), seq[p:p + copy_len].copy()))
    return out


def write_fasta(chrs, path):
    with open(path, "wb") as f:
        for name, seq in chrs:
            f.write(b">" + name.encode() + b"\n")
            n = len(seq)
            full = (n // 60) * 60
            if full:
                block = np.empty((full // 60, 61), dtype=np.uint8)
                block[:, :60] = seq[:full].reshape(-1, 60)
                block[:, 60] = 10
                f.write(block.tobytes())
            if n > full:
                f.write(seq[full:].tobytes() + b"\n")


def write_gtf(chrs, trs, path):
    with open(path, "w") as f:
        for t in trs:
            cname = chrs[t["chr"]][0]
            for k, (a, b) in enumerate(t["exons"]):
                f.write('%s\tsynth\texon\t%d\t%d\t.\t%s\t.\tgene_id "%s"; transcript_id "%s.1"; exon_number "%d";\n'
                        % (cname, a + 1, b, t["strand"], t["gid"], t["gid"], k + 1))


def _mutate(frag, rng, mm):
    """frag: (n, L) uint8 ASCII ACGT/N.  Substitute with probability mm to a different base."""
    if mm <= 0:
        return frag
    mask = (rng.random(frag.shape) < mm) & (frag != ord("N"))
    n = int(mask.sum())
    if n:
        old = frag[mask]
        # code of old base 0..3
        code = np.zeros(256, dtype=np.uint8)
        code[ord("C")] = 1
        code[ord("G")] = 2
        code[ord("T")] = 3
        new = (code[old] + rng.integers(1, 4, size=n, dtype=np.uint8)) % 4
        frag[mask] = ACGT[new]
    return frag


def make_reads(chrs, trs, n_pairs, read_len=100, frag_len=300, mm=0.005, seed=1,
               indel=0.0, nrate=0.0, junk=0.0, tx_frac=0.5):
    """Returns (mate1, mate2): two (n_pairs, read_len) uint8 ASCII arrays."""
    rng = np.random.default_rng(seed)
    frag_len = max(frag_len, read_len)
    # transcriptome: concatenate transcript sequences (in genome orientation; strand handled by random flip)
    tx_seqs = []
    for t in trs:
        s = np.concatenate([chrs[t["chr"]][1][a:b] for a, b in t["exons"]])
        if len(s) >= frag_len:
            tx_seqs.append(s)
    n_tx = int(n_pairs * tx_frac) if tx_seqs else 0
    n_gn = n_pairs - n_tx
    frags = np.empty((n_pairs, frag_len), dtype=np.uint8)
    ar = np.arange(frag_len)
    # genome fragments
    lens = np.array([len(c[1]) for c in chrs], dtype=np.int64)
    usable = lens - frag_len
    ci = rng.choice(len(chrs), size=n_gn, p=usable / usable.sum())
    st = (rng.random(n_gn) * usable[ci]).astype(np.int64)
    for k, (_, seq) in enumerate(chrs):
        sel = np.nonzero(ci == k)[0]
        for lo in range(0, len(sel), 1 << 18):
            ss = sel[lo:lo + (1 << 18)]
            frags[ss] = seq[st[ss, None] + ar[None, :]]
    # transcript fragments
    if n_tx:
        tl = np.array([len(s) for s in tx_seqs], dtype=np.int64)
        toff = np.concatenate([[0], np.cumsum(tl)[:-1]])
        tcat = np.concatenate(tx_seqs)
        ti = rng.integers(0, len(tx_seqs), size=n_tx)
        ts = (rng.random(n_tx) * (tl[ti] - frag_len + 1)).astype(np.int64)
        base = toff[ti] + ts
        for lo in range(0, n_tx, 1 << 18):
            frags[n_gn + lo:n_gn + lo + (1 << 18)] = tcat[base[lo:lo + (1 << 18), None] + ar[None, :]]
    # shuffle pair order so transcript and genome reads interleave
    perm = rng.permutation(n_pairs)
    frags = frags[perm]
    # random strand
    flip = rng.random(n_pairs) < 0.5
    frags[flip] = COMP[frags[flip][:, ::-1]]
    m1 = frags[:, :read_len].copy()
    m2 = COMP[frags[:, frag_len - read_len:][:, ::-1]].copy()
    m1 = _mutate(m1, rng, mm)
    m2 = _mutate(m2, rng, mm)
    if indel > 0:
        # per-read indel events (one small insertion or deletion); rows handled in a python loop, rate is small
        for m in (m1, m2):
            rows = np.nonzero(rng.random(n_pairs) < indel * read_len)[0]
            for r in rows:
                pos = int(rng.integers(15, read_len - 15))
                k = int(rng.integers(1, 4))
                row = m[r].copy()
                if rng.random() < 0.5:   # insertion of k random bases (read keeps length: tail drops)
                    ins = ACGT[rng.integers(0, 4, size=k, dtype=np.uint8)]
                    m[r] = np.concatenate([row[:pos], ins, row[pos:]])[:read_len]
                else:                    # deletion of k bases (pad tail with random bases)
                    pad = ACGT[rng.integers(0, 4, size=k, dtype=np.uint8)]
                    m[r] = np.concatenate([row[:pos], row[pos + k:], pad])
    if nrate > 0:
        for m in (m1, m2):
            m[rng.random(m.shape) < nrate] = ord("N")
    if junk > 0:
        rows = np.nonzero(rng.random(n_pairs) < junk)[0]
        m1[rows] = ACGT[rng.integers(0, 4, size=(len(rows), read_len), dtype=np.uint8)]
        m2[rows] = ACGT[rng.integers(0, 4, size=(len(rows), read_len), dtype=np.uint8)]
    return m1, m2


def write_fastq(m, path, first_index=0):
    n, L = m.shape
    names = np.char.add("@r", np.char.zfill(np.arange(first_index, first_index + n).astype(str), 9))
    nm = np.frombuffer("".join(names.tolist()).encode(), dtype=np.uint8).reshape(n, 11)
    rec = np.empty((n, 11 + 1 + L + 1 + 2 + L + 1), dtype=np.uint8)
    rec[:, :11] = nm
    rec[:, 11] = 10
    rec[:, 12:12 + L] = m
    rec[:, 12 + L] = 10
    rec[:, 13 + L] = ord("+")
    rec[:, 14 + L] = 10
    rec[:, 15 + L:15 + 2 * L] = ord("I")
    rec[:, 15 + 2 * L] = 10
    rec.tofile(path)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--preset", default="tiny", choices=sorted(PRESETS))
    ap.add_argument("--out", required=True)
    ap.add_argument("--pairs", type=int, default=2000)
    ap.add_argument("--read-len", type=int, default=100)
    ap.add_argument("--mm", type=float, default=0.005)
    ap.add_argument("--indel", type=float, default=0.0)
    ap.add_argument("--nrate", type=float, default=0.0)
    ap.add_argument("--junk", type=float, default=0.0)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--reads-only", action="store_true")
    ap.add_argument("--tag", default="reads")
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    chrs = make_genome(a.preset)
    trs = make_annotation(chrs, a.preset)
    if not a.reads_only:
        write_fasta(chrs, os.path.join(a.out, "genome.fa"))
        write_gtf(chrs, trs, os.path.join(a.out, "annot.gtf"))
    m1, m2 = make_reads(chrs, trs, a.pairs, read_len=a.read_len, mm=a.mm, seed=a.seed,
                        indel=a.indel, nrate=a.nrate, junk=a.junk)
    write_fastq(m1, os.path.join(a.out, a.tag + "_1.fq"))
    write_fastq(m2, os.path.join(a.out, a.tag + "_2.fq"))
    print("genome %d bp in %d chrs, %d transcripts, %d pairs" %
          (sum(len(c[1]) for c in chrs), len(chrs), len(trs), a.pairs), file=sys.stderr)


if __name__ == "__main__":
    main()
