"""Duplicate marking (--runMode inputAlignmentsFromBAM --bamRemoveDuplicatesType) against the goldens of the unmodified reference
(tests/golden/dedup.tar.gz, make_golden_dedup.py).

CPU (tests/dedup_check/: the product's host code driven by the oracle engine): the pair selection by the sequential restatement of
bamRemoveDuplicates and by the emulated kernels of dedup_kernels.cuh, also with 3-member batches and with hashes cut to 0 and 3 bits so
that the collision re-split runs; the emulated batch call against the restatement on random member sets; parameter errors; the NH / AS
errors; the inputs on which the reference is undefined; bad files; a header-only BAM; a differential fuzz against the live reference.
GPU (-m gpu): star_b200/bin/STAR on every golden; the device batch call against the restatement, with forced collisions and one group of
a million members; a chr21-sized mapping run with duplicated pairs, our Processed.out.bam against the reference's.
"""
import ctypes as C
import gzip
import json
import os
import struct
import subprocess
import sys
import tarfile

import numpy as np
import pytest

import conftest as cf
import oracle_capi as oc

ROOT = cf.ROOT
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bam_synth  # noqa: E402

DEDUP_DIR = os.path.join(ROOT, "build", "dedup_check")
DEDUP_CLI = os.path.join(DEDUP_DIR, "star_cli_dedup")
OURS = os.path.join(ROOT, "star_b200", "bin", "STAR")
EMUL = {"STAR_DEDUP_EMUL": "1"}
EOF_BLOCK = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")
NH_MISSING = "SAM tag NH is missing from a read, but it's required for deduplication."
AS_MISSING = "SAM tag AS is missing from a read, but it's required for deduplication."


@pytest.fixture(scope="module")
def checkers(oracle, lib):
    """build/dedup_check/ (tests/dedup_check/Makefile; __graft_entry__.build() makes it): the test CLI and the CPU implementations."""
    if not os.path.exists(DEDUP_CLI):
        subprocess.check_call(["make", "-s", "-f", os.path.join(ROOT, "tests", "dedup_check", "Makefile")], cwd=ROOT)
    return C.CDLL(os.path.join(DEDUP_DIR, "libdedup_check.so"))


@pytest.fixture(scope="module")
def dd_golden(tmp_path_factory):
    d = tmp_path_factory.mktemp("golden_dedup")
    with tarfile.open(os.path.join(ROOT, "tests", "golden", "dedup.tar.gz")) as t:
        t.extractall(d)
    dg = str(d / "dedup")
    return dg, json.load(open(os.path.join(dg, "scenarios.json")))


def _run(exe, args, out, env=None, cwd=None, threads=2):
    return subprocess.run([exe, "--runMode", "inputAlignmentsFromBAM"] + args + ["--outFileNamePrefix", out, "--runThreadN", str(threads)], cwd=cwd or ROOT,
                          env=dict(os.environ, **(env or {})), capture_output=True, text=True)


def _same_bam(ours, ref):
    z = open(ours, "rb").read()
    assert z.endswith(EOF_BLOCK)
    assert gzip.decompress(z) == gzip.decompress(open(ref, "rb").read())


def _golden_runs(exe, dg, sc, tmp_path, env=None, names=None):
    for name in names or sc:
        args = [x.replace("DG/", dg + "/") for x in sc[name]]
        out = str(tmp_path / (name + "_" + str(bool(env)))) + "."
        r = _run(exe, args, out, env)
        assert r.returncode == 0, (name, r.stderr)
        _same_bam(out + "Processed.out.bam", os.path.join(dg, name, "Processed.out.bam"))


def test_oracle_and_emulated_kernels_equal_golden(checkers, dd_golden, tmp_path):
    dg, sc = dd_golden
    _golden_runs(DEDUP_CLI, dg, sc, tmp_path)
    _golden_runs(DEDUP_CLI, dg, sc, tmp_path, EMUL)


@pytest.mark.parametrize("env", [{"STAR_B200_DEDUP_BATCH_RECS": "3"}, {"STAR_B200_DEDUP_HASH_BITS": "0"}, {"STAR_B200_DEDUP_HASH_BITS": "3"}])
def test_emulated_kernels_small_batches_and_short_hashes(checkers, dd_golden, tmp_path, env):
    dg, sc = dd_golden
    _golden_runs(DEDUP_CLI, dg, sc, tmp_path, dict(EMUL, **env), ["P1_ui_n0", "P4_uinm_n8", "S1_ui_single_end", "M2_uinm_n8"])


# ---- the batch call on member sets ------------------------------------------------------------------------------------------------
def random_members(rng, n_groups, per_group, n_names=None, lseq=40):
    """Members of n_groups groups (0x400 set, as the host leaves them): few distinct starts, CIGARs, flags and sequences, so that classes
    have several pairs; names drawn from a small pool so that some repeat.  Returns (bytes, offsets, groups)."""
    recs, groups = [], []
    n_names = n_names or max(4, per_group // 2)
    for g in range(n_groups):
        for _ in range(int(rng.integers(1, per_group + 1))):
            cig = [[("M", lseq)], [("S", 2), ("M", lseq - 2)], [("M", lseq - 3), ("S", 3)], [("M", 10), ("N", 50), ("M", lseq - 10)]][rng.integers(0, 4)]
            pos = int(rng.integers(100, 104)) + (2 if cig[0][0] == "S" else 0)
            flag = int(rng.choice([0x463, 0x493, 0x4a3, 0x453, 0x400, 0x410]))
            nib = [int(x) for x in rng.choice([1, 2], lseq)] if rng.random() < 0.3 else [1] * lseq
            name = b"n%d" % rng.integers(0, n_names) if rng.random() < 0.8 else bytes([0x80 + int(rng.integers(0, 3))]) + b"x"
            recs.append(bam_synth.dd_record(0, pos, flag, cig, name, nib, 0, pos + 100, 1, int(rng.integers(0, 4)), pad=int(rng.integers(0, 3))))
            groups.append(g)
    offsets = np.cumsum([0] + [len(r) for r in recs[:-1]]).astype(np.uint64)
    return np.frombuffer(b"".join(recs), np.uint8), offsets, np.array(groups, np.uint32)


def _batch(checkers, impl, data, offsets, groups, n2=0):
    op, ba, cl = (getattr(checkers, "dedup_%s_%s" % (impl, f)) for f in ("open", "batch", "close"))
    op.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.c_uint64]
    ba.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]
    cl.argtypes = [C.c_void_p]
    cl.restype = None
    h = C.c_void_p()
    assert op(C.byref(h), 0, n2) == 0
    un = np.zeros(len(offsets), np.uint8)
    rc = ba(h, data.ctypes.data, offsets.ctypes.data, groups.ctypes.data, len(offsets), un.ctypes.data, None)
    cl(h)
    return rc, un


def test_emulated_batch_equal_to_restatement(checkers, monkeypatch):
    rng = np.random.default_rng(11)
    for bits, recs in (("64", "1048576"), ("2", "1048576"), ("0", "7"), ("64", "1")):
        monkeypatch.setenv("STAR_B200_DEDUP_HASH_BITS", bits)
        monkeypatch.setenv("STAR_B200_DEDUP_BATCH_RECS", recs)
        for n_groups, per_group, n2 in ((40, 12, 0), (5, 60, 3), (2, 200, 40)):
            data, off, grp = random_members(rng, n_groups, per_group)
            o = _batch(checkers, "oracle", data, off, grp, n2)
            e = _batch(checkers, "emul", data, off, grp, n2)
            assert o[0] == e[0] == 0 and np.array_equal(o[1], e[1]), (bits, recs, n_groups)
            assert o[1].sum() > 0


def test_emulated_batch_errors_equal_to_restatement(checkers):
    """The error a batch reports (code, and the member it names) is the restatement's: N > l_seq, AS missing and AS <= -999 in later
    groups than an earlier clean one."""
    rng = np.random.default_rng(5)
    data, off, grp = random_members(rng, 6, 10)
    for n2, patch, code in ((41, None, 104), (0, "as_missing", 102), (0, "as_low", 104)):
        d = data.copy()
        if patch:   # the AS of every member of groups >= 3 (its last aux field, "ASs" + int16)
            for i in np.nonzero(grp >= 3)[0]:
                s = int(off[i]) + 4 + struct.unpack("<i", d[int(off[i]):int(off[i]) + 4].tobytes())[0]
                if patch == "as_missing":
                    d[s - 5:s - 3] = np.frombuffer(b"XS", np.uint8)
                else:
                    d[s - 2:s] = np.frombuffer(struct.pack("<h", -999), np.uint8)
        o, e = _batch(checkers, "oracle", d, off, grp, n2), _batch(checkers, "emul", d, off, grp, n2)
        assert o[0] == e[0] == code and np.array_equal(o[1], e[1]) and (o[1] >= 2).sum() == 1, (n2, patch)


# ---- command line: parameters, errors ---------------------------------------------------------------------------------------------
def _pe(tmp_path, fn="pe.bam", seed=3, extra=(), drop=None):
    refs, recs = bam_synth.dedup_pe_bam(seed, n_pairs=60)
    recs = [r for r in recs if not (drop and drop(r))] + list(extra)
    p = str(tmp_path / fn)
    open(p, "wb").write(bam_synth.bam_bytes(refs, recs))
    return p, refs, recs


def test_parameter_errors(checkers, golden, tmp_path):
    bam, _, _ = _pe(tmp_path)
    base = ["--runMode", "inputAlignmentsFromBAM", "--inputBAMfile", bam, "--outFileNamePrefix", str(tmp_path) + "/"]
    cases = [
        (["--bamRemoveDuplicatesType", "Identical"], "unrecognized option in of --bamRemoveDuplicatesType=Identical"),
        (["--bamRemoveDuplicatesType", "-"], "only works with --outWigType bedGraph OR --bamRemoveDuplicatesType Identical"),
        (["--bamRemoveDuplicatesType", "UniqueIdentical", "--bamRemoveDuplicatesMate2basesN", "x"], "bamRemoveDuplicatesMate2basesN"),
    ]
    for extra, text in cases:
        r = subprocess.run([DEDUP_CLI] + base + extra, cwd=golden, capture_output=True, text=True)
        assert r.returncode == 102 and text in r.stderr, (extra, r.stderr)
    if os.path.exists(oc.REF_STAR):
        for extra, text in cases[:2]:
            r = subprocess.run([oc.REF_STAR] + base + extra, cwd=golden, capture_output=True, text=True)
            assert r.returncode == 102 and text in r.stderr, (extra, r.stderr)
    # outside inputAlignmentsFromBAM both names stay outside the scope
    for extra in (["--bamRemoveDuplicatesType", "UniqueIdentical"], ["--bamRemoveDuplicatesMate2basesN", "3"]):
        r = subprocess.run([DEDUP_CLI, "--genomeDir", "idx", "--readFilesIn", "se_1.fq", "--outFileNamePrefix", str(tmp_path) + "/"] + extra, cwd=golden,
                           capture_output=True, text=True)
        assert r.returncode == 102 and "outside the scope" in r.stderr, (extra, r.stderr)


def test_signal_and_dedup_make_only_signal(checkers, tmp_path):
    """(tests/signal_check's CLI has signal tracks and no duplicate marking: it fails if the run goes to duplicate marking.)"""
    bam, _, _ = _pe(tmp_path)
    signal_cli = os.path.join(ROOT, "build", "signal_check", "star_cli_signal")
    if not os.path.exists(signal_cli):
        subprocess.check_call(["make", "-s", "-f", os.path.join(ROOT, "tests", "signal_check", "Makefile")], cwd=ROOT)
    for exe, tag in ((signal_cli, "ours"), (oc.REF_STAR, "ref")):
        if not os.path.exists(exe):
            continue
        out = str(tmp_path / tag) + "/"
        r = _run(exe, ["--inputBAMfile", bam, "--outWigType", "bedGraph", "--bamRemoveDuplicatesType", "UniqueIdentical"], out)
        assert r.returncode == 0, r.stderr
        files = os.listdir(out)
        assert "Processed.out.bam" not in files and any(f.startswith("Signal.") for f in files), files
        assert "reading from BAM, output wiggle" in open(out + "Log.out").read()


def test_nh_and_as_errors_in_reference_order(checkers, tmp_path):
    """NH is read before the group closes: a record without NH that closes a group whose pair lacks AS reports NH; one record later, AS."""
    nib = [1] * 30
    def rec(tid, pos, flag, name, nh=1, as_=None, mpos=-1):
        return bam_synth.dd_record(tid, pos, flag, [("M", 30)], name, nib, tid, mpos, nh, as_)
    no_as = [rec(0, 100, 0x63, b"a", mpos=200), rec(0, 200, 0x93, b"a", mpos=100)]
    cases = {"nh": (no_as + [rec(1, 50, 0x63, b"b", None, 40)], NH_MISSING),
             "as": (no_as + [rec(1, 50, 0x63, b"b", 1, 40, 90), rec(1, 60, 0x63, b"c", None, 40)], AS_MISSING),
             "nh_first": ([rec(0, 10, 0, b"z", None, 40)] + no_as, NH_MISSING),
             "as_at_end": (no_as, AS_MISSING)}
    for k, (rs, text) in cases.items():
        p = str(tmp_path / (k + ".bam"))
        open(p, "wb").write(bam_synth.bam_bytes(bam_synth.DD_REFS, rs))
        for exe, env in ((DEDUP_CLI, None), (DEDUP_CLI, EMUL), (oc.REF_STAR, None)):
            if not os.path.exists(exe):
                continue
            r = _run(exe, ["--inputBAMfile", p, "--bamRemoveDuplicatesType", "UniqueIdentical"], str(tmp_path / k) + ".", env)
            assert r.returncode == 102 and text in r.stderr, (k, exe, r.stderr)


def test_undefined_inputs_exit_104(checkers, tmp_path):
    """Inputs on which the reference reads out of bounds or depends on the order of classes: exit 104 naming the record."""
    nib = [1] * 30
    def pair(cig2, as1=50, n2=None, name=b"q"):
        return [bam_synth.dd_record(0, 100, 0x63, [("M", 30)], name, nib, 0, 200, 1, as1),
                bam_synth.dd_record(0, 200, 0x93, cig2, name, n2 or nib, 0, 100, 1, as1)]
    refs = bam_synth.DD_REFS
    cases = {"no_cigar": (pair([]), [], "CIGAR of 0 operations"), "only_s": (pair([("S", 30)]), [], "CIGAR of 1 operations"),
             "ss": (pair([("S", 10), ("S", 20)]), [], "CIGAR of 2 operations"),
             "101_ops": (pair([("M", 1), ("I", 1)] * 14 + [("M", 1)] + [("M", 1)] * 72), [], "CIGAR of 101 operations"),
             "n_gt_lseq": (pair([("M", 30)]), ["--bamRemoveDuplicatesMate2basesN", "31"], "fewer than --bamRemoveDuplicatesMate2basesN 31"),
             "as_low": (pair([("M", 30)], as1=-999), [], "AS <= -999")}
    for k, (rs, extra, text) in cases.items():
        rs = rs + pair([("M", 30)], name=b"r")
        p = str(tmp_path / (k + ".bam"))
        open(p, "wb").write(bam_synth.bam_bytes(refs, rs))
        for env in (None, EMUL):
            r = _run(DEDUP_CLI, ["--inputBAMfile", p, "--bamRemoveDuplicatesType", "UniqueIdentical"] + extra, str(tmp_path / k) + ".", env)
            assert r.returncode == 104 and text in r.stderr and "BAM record " in r.stderr, (k, env, r.stderr)
    good = open(_pe(tmp_path)[0], "rb").read()
    for fn, data in {"text.bam": b"@HD\tVN:1.4\nnot a BAM\n", "trunc.bam": good[: len(good) // 2]}.items():
        p = str(tmp_path / fn)
        open(p, "wb").write(data)
        r = _run(DEDUP_CLI, ["--inputBAMfile", p, "--bamRemoveDuplicatesType", "UniqueIdentical"], p + ".")
        assert r.returncode == 104 and "--inputBAMfile" in r.stderr, (fn, r.stderr)


def test_header_only_bam(checkers, tmp_path):
    p = str(tmp_path / "empty.bam")
    open(p, "wb").write(bam_synth.bam_bytes(bam_synth.DD_REFS, []))
    for env in (None, EMUL):
        r = _run(DEDUP_CLI, ["--inputBAMfile", p, "--bamRemoveDuplicatesType", "UniqueIdentical"], p + ".", env)
        assert r.returncode == 0, r.stderr
        z = open(p + ".Processed.out.bam", "rb").read()
        assert z.endswith(EOF_BLOCK) and gzip.decompress(z) == gzip.decompress(open(p, "rb").read())


@pytest.mark.skipif(not os.path.exists(oc.REF_STAR), reason="oracle/_ref/STAR not built (needs /root/reference)")
@pytest.mark.parametrize("seed", [201, 202, 203, 204])
def test_fuzz_against_live_reference(checkers, tmp_path, seed):
    import fuzz_dedup
    assert fuzz_dedup.check(seed, str(tmp_path), [DEDUP_CLI]) == []
    assert fuzz_dedup.check(seed, str(tmp_path), [DEDUP_CLI], env=EMUL) == []


# ---- GPU ----------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_gpu_cli_equals_golden(lib, dd_golden, tmp_path):
    dg, sc = dd_golden
    _golden_runs(OURS, dg, sc, tmp_path)


@pytest.mark.gpu
def test_gpu_batch_equal_to_restatement(lib, checkers, monkeypatch):
    import star_b200
    rng = np.random.default_rng(17)
    for bits, recs in (("64", None), ("3", None), ("0", "50")):
        monkeypatch.setenv("STAR_B200_DEDUP_HASH_BITS", bits)
        if recs:
            monkeypatch.setenv("STAR_B200_DEDUP_BATCH_RECS", recs)
        for n_groups, per_group, n2 in ((400, 30, 0), (20, 300, 5), (3, 2000, 40)):
            if bits == "0" and per_group > 300:
                continue   # (every pair of a group in one run: quadratic re-split)
            data, off, grp = random_members(rng, n_groups, per_group)
            d = star_b200.capi.Dedup(lib, n2)
            rc, g, _ = d.batch(data, off, grp)
            d.close()
            o = _batch(checkers, "oracle", data, off, grp, n2)
            assert rc == o[0] == 0 and np.array_equal(g, o[1]), (bits, n_groups)


@pytest.mark.gpu
def test_gpu_batch_one_group_of_a_million_members(lib, checkers):
    """Single-end data makes a chromosome one group: 2^20 members, names from a pool of 2^18 (so most repeat)."""
    import star_b200
    rng = np.random.default_rng(23)
    n = 1 << 20
    recs = []
    for i in range(n):
        cig = [("M", 30)] if i % 3 else [("S", 2), ("M", 28)]
        recs.append(bam_synth.dd_record(0, 1000 + int(i % 50), 0x400 | (16 if i % 7 == 0 else 0), cig, b"r%06d" % rng.integers(0, 1 << 18), [1 + i % 2] * 30,
                                        -1, -1, 1, int(i % 11)))
    data = np.frombuffer(b"".join(recs), np.uint8)
    off = np.cumsum([0] + [len(r) for r in recs[:-1]]).astype(np.uint64)
    grp = np.zeros(n, np.uint32)
    d = star_b200.capi.Dedup(lib, 2)
    rc, g, ms = d.batch(data, off, grp)
    d.close()
    o = _batch(checkers, "oracle", data, off, grp, 2)
    assert rc == o[0] == 0 and np.array_equal(g, o[1]) and g.sum() > 0


@pytest.mark.gpu
@pytest.mark.skipif(not os.path.exists(oc.REF_STAR), reason="oracle/_ref/STAR not built")
def test_gpu_dedup_of_config_size_bam_equals_reference(lib, tmp_path):
    """chr21-sized index (tests/test_gpu_config_gate.py), 100 k pairs with a fifth of them repeated under new names: our CLI's sorted BAM
    through our duplicate marking and the reference's must give the same Processed.out.bam."""
    import test_gpu_config_gate as gate
    import bench
    import bench_dedup
    import synth
    wd = os.path.join(os.environ.get("STAR_B200_BENCH_DIR", "/tmp/star_b200_bench"), "chr21")
    os.makedirs(wd, exist_ok=True)
    chrs, trs, idx, _ = bench.prepare_genome(wd, "chr21")
    c = {"dir": wd, "chrs": chrs, "trs": trs, "idx": idx, "synth": synth}
    _, _, r1, r2 = gate._reads(c, 100000, 100, 0.005, 21, "dd")
    bench_dedup.dup_pairs(r1, r2, r1 + ".dup", r2 + ".dup", 0.2, 5)
    out = str(tmp_path / "map") + "/"
    subprocess.check_call([OURS, "--genomeDir", idx, "--readFilesIn", r1 + ".dup", r2 + ".dup", "--outSAMtype", "BAM", "SortedByCoordinate", "--runThreadN", "8",
                           "--outFileNamePrefix", out], stdout=subprocess.DEVNULL)
    bam = out + "Aligned.sortedByCoord.out.bam"
    for exe, d in ((OURS, "ours"), (oc.REF_STAR, "ref")):
        subprocess.check_call([exe, "--runMode", "inputAlignmentsFromBAM", "--inputBAMfile", bam, "--bamRemoveDuplicatesType", "UniqueIdentical",
                               "--bamRemoveDuplicatesMate2basesN", "4", "--outFileNamePrefix", str(tmp_path / d) + "/"], stdout=subprocess.DEVNULL)
    _same_bam(str(tmp_path / "ours" / "Processed.out.bam"), str(tmp_path / "ref" / "Processed.out.bam"))
    log = open(str(tmp_path / "ours" / "Log.out")).read()
    assert "pairs un-marked" in log
