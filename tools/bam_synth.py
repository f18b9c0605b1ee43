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


# ---- duplicate marking (--bamRemoveDuplicatesType) ---------------------------------------------------------------------------------
def dd_record(tid, pos, flag, cigar, name, nib, mtid=-1, mpos=-1, nh=1, as_=None, pad=0, extra=b""):
    """A record for the duplicate-marking fixtures: name (bytes), packed sequence nibbles `nib` (len = l_seq; `pad` = the pad nibble of an
    odd l_seq), mate reference / position, NH (None: no tag) and AS (None: no tag) as aux fields."""
    lseq = len(nib)
    cig = b"".join(struct.pack("<I", (l << 4) | OPS.index(op)) for op, l in cigar)
    qname = name + b"\0"
    n = list(nib) + ([pad] if lseq % 2 else [])
    seq = bytes((n[i] << 4) | n[i + 1] for i in range(0, len(n), 2))
    aux = extra
    if nh is not None:
        aux += b"NHC" + struct.pack("<B", nh) if 0 <= nh < 256 else b"NHi" + struct.pack("<i", nh)
    if as_ is not None:
        aux += b"ASs" + struct.pack("<h", as_) if -32768 <= as_ < 32768 else b"ASi" + struct.pack("<i", as_)
    body = struct.pack("<iiBBHHHiiii", tid, pos, len(qname), 255, 4680, len(cigar), flag, lseq, mtid, mpos, 0)
    body += qname + cig + seq + b"\x1e" * lseq + aux
    return struct.pack("<i", len(body)) + body


def _qlen(cigar):
    return sum(l for op, l in cigar if op in "MIS=X")


def _rlen(cigar):
    return sum(l for op, l in cigar if op in "MDN=X")


DD_REFS = [("chr1", 5000), ("chr2", 3000), ("chrM", 1500)]


def _pair(rng, recs, tid, pos, name, isize=None, as_=None, mate2_first=False, cig1=None, cig2=None, nib2=None, pad2=0):
    """Two records of a proper pair: mate 1 forward at pos, mate 2 reverse to its right (or, mate2_first, mate 2 forward at pos and mate 1
    reverse to its right).  Returns the nibbles of mate 2 (for duplicates)."""
    cig1 = cig1 or [("M", 50)]
    cig2 = cig2 or [("M", 50)]
    isize = isize or rng.randrange(60, 300)
    as_ = rng.randrange(60, 99) if as_ is None else as_
    p2 = pos + isize
    nib1 = [rng.choice([1, 2, 4, 8]) for _ in range(_qlen(cig1))]
    nib2 = nib2 or [rng.choice([1, 2, 4, 8]) for _ in range(_qlen(cig2))]
    if not mate2_first:
        recs.append(dd_record(tid, pos, 0x1 | 0x2 | 0x20 | 0x40, cig1, name, nib1, tid, p2, 1, as_))
        recs.append(dd_record(tid, p2, 0x1 | 0x2 | 0x10 | 0x80, cig2, name, nib2, tid, pos, 1, as_, pad2))
    else:
        recs.append(dd_record(tid, pos, 0x1 | 0x2 | 0x20 | 0x80, cig2, name, nib2, tid, p2, 1, as_, pad2))
        recs.append(dd_record(tid, p2, 0x1 | 0x2 | 0x10 | 0x40, cig1, name, nib1, tid, pos, 1, as_))
    return nib2


def _sorted(recs):
    key = lambda r: (struct.unpack("<I", r[4:8])[0], struct.unpack("<i", r[8:12])[0])
    return sorted(recs, key=key)


def dedup_pe_bam(seed, n_pairs=300, refs=DD_REFS):
    """A coordinate-sorted paired-end BAM for duplicate marking: random pairs, a quarter duplicated under new names with other AS values,
    plus the cases listed in tests/golden/make_golden_dedup.py.  Returns (refs, records)."""
    rng = random.Random(seed)
    recs = []
    k = 0

    def nm(tag=b"p"):
        nonlocal k
        k += 1
        return tag + b":%05d:%d" % (rng.randrange(100000), k)

    for _ in range(n_pairs):   # (chr2 holds the cases of dedup_pinned_records)
        tid = rng.choice([0, 0, 2])
        pos = rng.randrange(1, refs[tid][1] - 400)
        c1 = rng.choice([[("M", 50)], [("S", 3), ("M", 47)], [("M", 20), ("N", 100), ("M", 30)], [("M", 45), ("S", 5)], [("M", 30), ("I", 2), ("M", 18)]])
        first = rng.random() < 0.3
        name = nm()
        nib2 = _pair(rng, recs, tid, pos, name, cig1=c1, mate2_first=first)
        for _ in range(rng.choice([0, 0, 0, 1, 2, 3])):   # duplicates under new names
            n2 = list(nib2)
            r = rng.random()
            if r < 0.15:
                n2[0] ^= 3       # mate 2 differs at the forward start / reverse start
            elif r < 0.3:
                n2[-1] ^= 3      # ... at the end
            _pair(rng, recs, tid, pos, nm(), isize=_isize_of(recs, name), cig1=c1, mate2_first=first, nib2=n2)
    # multimappers (NH 2), some with 0x400 already set
    for _ in range(40):
        tid = rng.choice([0, 1])
        pos = rng.randrange(1, refs[tid][1] - 100)
        recs.append(dd_record(tid, pos, rng.choice([0, 0x400, 0x10, 0x410]), [("M", 50)], nm(b"m"), [1] * 50, -1, -1, 2, 70))
    # names occurring 1 and 3 times (single records / a pair plus a stray mate)
    for _ in range(6):
        tid = 0
        pos = rng.randrange(1, refs[tid][1] - 400)
        name = nm(b"odd")
        recs.append(dd_record(tid, pos, 0x1 | 0x40 | 0x8, [("M", 50)], name, [2] * 50, tid, pos, 1, 80))
        if rng.random() < 0.5:
            _pair(rng, recs, tid, pos + 3, name)
    # signed-char names: bytes >= 0x80 sort before ASCII
    for b in (b"\xe9t\xe9", b"et\xe9", b"\x80x", b"zz"):
        pos = rng.randrange(1, refs[0][1] - 400)
        nib2 = _pair(rng, recs, 0, pos, b + b":%d" % k, as_=77)
        _pair(rng, recs, 0, pos, b + b":%d:dup" % k, as_=77, isize=_isize_of(recs, b + b":%d" % k), nib2=nib2)
    recs = _sorted(recs + dedup_pinned_records()[0]) + [dd_record(-1, -1, 0x4 | 0x1 | 0x40 | 0x8, [], nm(b"u"), [4] * 30, -1, -1, 0) for _ in range(3)]
    return refs, recs


def _isize_of(recs, name):
    for r in reversed(recs):
        lq = r[12]
        if r[36:36 + lq - 1] == name:
            return abs(struct.unpack("<i", r[28:32])[0] - struct.unpack("<i", r[8:12])[0])
    raise KeyError(name)


def dedup_pinned_records():
    """The cases the goldens must pin, at fixed places of chr2 (before any random record there): S extension, the tie order, mate-2
    differences at the forward start and the reverse end, odd l_seq with different pad nibbles, and a group held open by rightMax == 0.
    Returns (records, {case: [(name, expect_unmarked)]}) for N = 0 runs."""
    recs = []
    nib = [1, 2, 4, 8, 1, 2, 4, 8, 1] * 5 + [2, 4, 8, 1, 2]    # 50 bases
    # S extension: 3S47M at 1003 equals 50M at 1000 (and its mate the same); the 2nd has the higher AS
    recs.append(dd_record(1, 1003, 0x63, [("S", 3), ("M", 47)], b"sext:a", nib, 1, 1200, 1, 60))
    recs.append(dd_record(1, 1200, 0x93, [("M", 50)], b"sext:a", nib, 1, 1003, 1, 60))
    recs.append(dd_record(1, 1000, 0x63, [("M", 50)], b"sext:b", nib, 1, 1200, 1, 61))
    recs.append(dd_record(1, 1200, 0x93, [("M", 50)], b"sext:b", nib, 1, 1000, 1, 61))
    # tie: equal AS; file order tie:z before tie:a, name order tie:a first -> tie:a is kept
    for nmz in (b"tie:z", b"tie:a"):
        recs.append(dd_record(1, 1600, 0x63, [("M", 50)], nmz, nib, 1, 1750, 1, 70))
    for nmz in (b"tie:z", b"tie:a"):
        recs.append(dd_record(1, 1750, 0x93, [("M", 50)], nmz, nib, 1, 1600, 1, 70))
    # odd l_seq (49 bases), reverse mate 2, identical but the pad nibble: two classes even with N = 0
    n49 = nib[:49]
    for nmz, pad in ((b"pad:a", 0), (b"pad:b", 5)):
        recs.append(dd_record(1, 2100, 0x63, [("M", 49)], nmz, n49, 1, 2250, 1, 50))
        recs.append(dd_record(1, 2250, 0x93, [("M", 49)], nmz, n49, 1, 2100, 1, 50, pad))
    # a group held open by rightMax == 0 at the start of chrM: both mates at the same position (the random pairs after them join it)
    for nmz in (b"same:a", b"same:b"):
        recs.append(dd_record(2, 0, 0x63, [("M", 50)], nmz, nib, 2, 0, 1, 40))
        recs.append(dd_record(2, 0, 0x93, [("M", 50)], nmz, nib, 2, 0, 1, 40))
    expect = {"s_extension": [(b"sext:a", False), (b"sext:b", True)], "tie_order": [(b"tie:a", True), (b"tie:z", False)],
              "pad_nibble": [(b"pad:a", True), (b"pad:b", True)]}
    return recs, expect


def dedup_se_bam(seed, n=400, refs=DD_REFS):
    """Single-end records (mpos = -1: every chromosome is one group; pairs are formed from unrelated reads)."""
    rng = random.Random(seed)
    recs = []
    for i in range(n):
        tid = rng.choice([0, 1])
        pos = rng.randrange(1, 300)
        cig = rng.choice([[("M", 40)], [("S", 2), ("M", 38)], [("M", 38), ("S", 2)]])
        recs.append(dd_record(tid, pos, rng.choice([0, 16]), cig, b"se%d" % rng.randrange(60), [rng.choice([1, 2]) for _ in range(40)], -1, -1,
                              rng.choice([1, 1, 1, 3]), rng.randrange(30, 40)))
    return refs, _sorted(recs)


def read_bam(data):
    """(header bytes, [records]) of a BAM file (BGZF = concatenated gzip members)."""
    import gzip
    u = gzip.decompress(data)
    lt = struct.unpack("<i", u[4:8])[0]
    p = 8 + lt
    nref = struct.unpack("<i", u[p:p + 4])[0]
    p += 4
    for _ in range(nref):
        p += 8 + struct.unpack("<i", u[p:p + 4])[0]
    hdr, recs = u[:p], []
    while p < len(u):
        bs = struct.unpack("<i", u[p:p + 4])[0]
        recs.append(u[p:p + 4 + bs])
        p += 4 + bs
    return hdr, recs


def rec_name_flag(r):
    return r[36:36 + r[12] - 1], struct.unpack("<H", r[18:20])[0]
