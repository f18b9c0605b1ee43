"""Hand-built BAM files for the signal-track tests (--runMode inputAlignmentsFromBAM): a BGZF writer (zlib) and a seeded generator of
records that exercise what signalFromBAM reads: reference ids that come back (unsorted input), NH as every aux type or absent, duplicates,
unmapped mates that carry a reference id, tid = -1 records, every CIGAR operation, records ending on the last base of a reference or one
past it, references a --outWigReferencesPrefix excludes, and piles of multimappers (NH 2..7) interleaved with unique records.
"""
import random
import struct
import zlib

OPS = "MIDNSHP=X"


def bgzf(data, level=6):
    """BGZF framing (SAM/BAM specification 4.1): blocks of <= 0xff00 payload bytes, raw deflate, then the empty EOF block."""
    out = bytearray()
    for o in range(0, len(data), 0xFF00):
        chunk = data[o:o + 0xFF00]
        c = zlib.compressobj(level, zlib.DEFLATED, -15)
        cdata = c.compress(chunk) + c.flush()
        bsize = 18 + len(cdata) + 8
        out += struct.pack("<BBBBIBBHBBHH", 31, 139, 8, 4, 0, 0, 255, 6, 66, 67, 2, bsize - 1)
        out += cdata + struct.pack("<II", zlib.crc32(chunk) & 0xFFFFFFFF, len(chunk))
    out += bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")
    return bytes(out)


def nh_aux(nh_type, nh):
    if nh_type is None:
        return b""
    if nh_type == "f":
        return b"NHf" + struct.pack("<f", float(nh))
    fmt = {"c": "<b", "C": "<B", "s": "<h", "S": "<H", "i": "<i", "I": "<I"}[nh_type]
    return b"NH" + nh_type.encode() + struct.pack(fmt, nh)


def record(tid, pos, flag, cigar, aux=b"", name=b"r"):
    """cigar: list of (op char, length)."""
    lseq = sum(l for op, l in cigar if op in "MIS=X")
    cig = b"".join(struct.pack("<I", (l << 4) | OPS.index(op)) for op, l in cigar)
    qname = name + b"\0"
    body = struct.pack("<iiBBHHHiiii", tid, pos, len(qname), 255, 4680, len(cigar), flag, lseq, -1, -1, 0)
    body += qname + cig + b"\x11" * ((lseq + 1) // 2) + b"\x1e" * lseq + aux
    return struct.pack("<i", len(body)) + body


def bam_bytes(refs, records):
    text = b"@HD\tVN:1.4\n" + b"".join(b"@SQ\tSN:%s\tLN:%d\n" % (n.encode(), l) for n, l in refs)
    h = b"BAM\1" + struct.pack("<i", len(text)) + text + struct.pack("<i", len(refs))
    for n, l in refs:
        h += struct.pack("<i", len(n) + 1) + n.encode() + b"\0" + struct.pack("<i", l)
    return bgzf(h + b"".join(records))


REFS = [("chr1", 700), ("chr2", 400), ("chrM", 120), ("scaffold_7", 300), ("chr3", 250)]


def random_bam(seed, n=400, refs=REFS):
    """Records in an order that returns to earlier references; returns (refs, list of encoded records)."""
    rng = random.Random(seed)
    recs = []
    tids = [rng.randrange(len(refs)) for _ in range(6)] + [0, 2]
    for seg, tid in enumerate(tids):
        L = refs[tid][1]
        hot = [rng.randrange(0, L - 60) for _ in range(3)]   # pile-up centres (multimappers stacked with uniques)
        for k in range(n // len(tids)):
            flag = rng.choice([0, 16, 0x40 | 0x1, 0x80 | 0x1, 0x50 | 0x1, 0x90 | 0x1, 0x400, 0x4 | 0x1 | 0x40, 0x10 | 0x400])
            nh_type = rng.choice([None, "c", "C", "s", "S", "I", "i", "i", "i", "C", "f"])
            nh = rng.choice([1, 1, 1, 2, 3, 4, 5, 6, 7]) if nh_type not in (None, "f") else 1
            if rng.random() < 0.02 and nh_type in ("i", "c"):
                nh = 0
            start = rng.choice(hot) + rng.randrange(-8, 8) if rng.random() < 0.6 else rng.randrange(1, L - 40)
            start = max(1, start)
            if flag & 0x4:
                cigar = []
            else:
                cigar = []
                if rng.random() < 0.3:
                    cigar.append((rng.choice("SH"), rng.randrange(1, 6)))
                room = L - start
                for _ in range(rng.randrange(1, 5)):
                    op = rng.choice("MMMMDNI=X")
                    ln = rng.randrange(1, 15)
                    if op in "MDN=X":
                        ln = min(ln, max(0, room - 2))
                        if ln == 0:
                            continue
                        room -= ln if op in "MDN" else 0
                    cigar.append((op, ln))
                if rng.random() < 0.2:
                    cigar.append(("S", rng.randrange(1, 5)))
            aux = b""
            if rng.random() < 0.4:
                aux += b"XSA+"
            if rng.random() < 0.3:
                aux += b"ZZZtext\0"
            if rng.random() < 0.2:
                aux += b"BBBc" + struct.pack("<I", 3) + b"\1\2\3"
            aux += nh_aux(nh_type, nh)
            if rng.random() < 0.3:
                aux += b"HIi" + struct.pack("<i", 1)
            recs.append(record(tid, start, flag, cigar, aux))
    # a record ending on the last base of chr1, and one running one base past it (the extra position every segment has)
    recs.append(record(0, refs[0][1] - 10, 0, [("M", 10)], nh_aux("C", 1)))
    recs.append(record(0, refs[0][1] - 5, 0, [("M", 6)], nh_aux("C", 3)))
    # unmapped records without a reference at the end
    recs += [record(-1, -1, 0x4, []) for _ in range(3)]
    return refs, recs


def um_terms(refs, recs, prefix="-"):
    """The 1/NH terms per (segment, strand, position) of the full-signal stranded tracks, in file order (signalFromBAM.cpp restated)."""
    terms = {}
    seg, itid = -1, None
    for r in recs:
        tid, pos, lqn, _, _, ncig, flag, _ = struct.unpack("<iiBBHHHi", r[4:24])
        if tid != itid:
            seg += 1
            itid = tid
        if tid < 0 or flag & 0x400 or (prefix != "-" and not refs[tid][0].startswith(prefix)):
            continue
        aux = r[36 + lqn + 4 * ncig:]
        nh = 1
        i = aux.find(b"NH")
        # (the fixtures put NH after fixed-size or NUL-terminated tags only; good enough for the order check)
        if i >= 0:
            t = aux[i + 2:i + 3]
            nh = {b"c": lambda s: struct.unpack("<b", s[:1])[0], b"C": lambda s: s[0], b"s": lambda s: struct.unpack("<h", s[:2])[0],
                  b"S": lambda s: struct.unpack("<H", s[:2])[0], b"i": lambda s: struct.unpack("<i", s[:4])[0],
                  b"I": lambda s: struct.unpack("<I", s[:4])[0]}.get(t, lambda s: 0)(aux[i + 3:])
        if nh <= 0:
            continue
        strand = int(bool(flag & 0x10) == (not flag & 0x80))
        g = pos
        for k in range(ncig):
            c = struct.unpack("<I", r[36 + lqn + 4 * k:40 + lqn + 4 * k])[0]
            op, ln = c & 15, c >> 4
            if op in (2, 3):
                g += ln
            elif op == 0:
                for p in range(g, g + ln):
                    terms.setdefault((seg, strand, p), []).append(1.0 / nh)
                g += ln
    return terms


def fold_order_matters(terms):
    """True when some position's left fold of its terms differs from the fold of the same terms in another order."""
    for t in terms.values():
        a = 0.0
        for x in t:
            a += x
        for perm in (sorted(t), sorted(t, reverse=True)):
            b = 0.0
            for x in perm:
                b += x
            if a != b:
                return True
    return False
