"""Signal tracks (--outWigType; --runMode inputAlignmentsFromBAM) against the goldens of the unmodified reference (tests/golden/signal.tar.gz,
make_golden_signal.py).

CPU (tests/signal_check/: the product's host code driven by the oracle engine): the signal tracks by the sequential restatement of
signalFromBAM and by the emulated kernels of signal_kernels.cuh, also with tiny window / pair capacities so that the window loop and the chunked fold of deep piles run; parameter
errors; bad input files; a 2-shard run and its merge; a differential fuzz against the live reference binary.
GPU (-m gpu): star_b200/bin/STAR on every golden scenario; the device segment call against the oracle restatement on random blocks, bit
for bit; the signal of a config-size mapping run against the reference's signal of the same BAM.
"""
import ctypes as C
import json
import os
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

SIGNAL_DIR = os.path.join(ROOT, "build", "signal_check")
SIGNAL_CLI = os.path.join(SIGNAL_DIR, "star_cli_signal")
EMUL = {"STAR_SIGNAL_EMUL": "1"}


@pytest.fixture(scope="module")
def checkers(oracle, lib):
    """build/signal_check/ (tests/signal_check/Makefile; __graft_entry__.build() makes it): the test CLI and the CPU implementations."""
    if not os.path.exists(SIGNAL_CLI):
        subprocess.check_call(["make", "-s", "-f", os.path.join(ROOT, "tests", "signal_check", "Makefile")], cwd=ROOT)
    return C.CDLL(os.path.join(SIGNAL_DIR, "libsignal_check.so"))
OURS = os.path.join(ROOT, "star_b200", "bin", "STAR")


@pytest.fixture(scope="module")
def sig_golden(tmp_path_factory, golden):
    d = tmp_path_factory.mktemp("golden_sig")
    with tarfile.open(os.path.join(ROOT, "tests", "golden", "signal.tar.gz")) as t:
        t.extractall(d)
    sg = str(d / "signal")
    return sg, json.load(open(os.path.join(sg, "scenarios.json")))


def _args(name, args, sg):
    a = [x.replace("SG/", sg + "/") for x in args]
    return (["--runMode", "inputAlignmentsFromBAM"] + a) if name.startswith("B") else a


def _run(exe, name, args, sg, golden, out, env=None, threads=2):
    r = subprocess.run([exe] + _args(name, args, sg) + ["--outFileNamePrefix", out, "--runThreadN", str(threads)], cwd=golden,
                       env=dict(os.environ, **(env or {})), capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return out


def _same_signal(out, ref):
    files = sorted(f for f in os.listdir(ref) if f.startswith("Signal."))
    assert files and sorted(f for f in os.listdir(out) if f.startswith("Signal.")) == files
    for f in files:
        assert open(os.path.join(out, f), "rb").read() == open(os.path.join(ref, f), "rb").read(), f


def test_oracle_and_emulated_kernels_equal_golden(checkers, sig_golden, golden, tmp_path):
    sg, sc = sig_golden
    for name, args in sc.items():
        _same_signal(_run(SIGNAL_CLI, name, args, sg, golden, str(tmp_path / ("o_" + name)) + "/"), os.path.join(sg, name))
        _same_signal(_run(SIGNAL_CLI, name, args, sg, golden, str(tmp_path / ("e_" + name)) + "/", EMUL), os.path.join(sg, name))


@pytest.mark.parametrize("name", ["B1_bg_stranded_rpm", "B3_wig_read1_5p", "M1_bg_stranded_rpm"])
def test_emulated_kernels_tiny_windows_and_pair_chunks(checkers, sig_golden, golden, tmp_path, name):
    sg, sc = sig_golden
    env = dict(EMUL, STAR_B200_SIGNAL_WINDOW="97", STAR_B200_SIGNAL_PAIRS="7")
    _same_signal(_run(SIGNAL_CLI, name, sc[name], sg, golden, str(tmp_path) + "/", env), os.path.join(sg, name))


def test_emulated_segment_bit_equal_to_restatement(checkers, monkeypatch):
    """The emulated kernels against the sequential restatement on random blocks, bit for bit, also with windows and pair chunks far
    smaller than the segment and its deepest pile."""
    rng = np.random.default_rng(3)
    for window, pairs in (("1048576", "1048576"), ("333", "50")):
        monkeypatch.setenv("STAR_B200_SIGNAL_WINDOW", window)
        monkeypatch.setenv("STAR_B200_SIGNAL_PAIRS", pairs)
        for n_strands, chr_len, n in ((2, 3000, 3000), (1, 1500, 2000)):
            b = np.zeros(n, BLOCK)
            b["start"] = rng.integers(0, chr_len - 100, n) if n_strands == 2 else rng.integers(0, 300, n)
            b["len"] = rng.integers(1, 100, n)
            b["nh"] = rng.choice([1, 1, 2, 3, 5, 7], n)
            b["strand"] = rng.integers(0, n_strands, n)
            for mode in (0, 1):
                e = _segment(checkers.signal_emul_open, checkers.signal_emul_segment, checkers.signal_emul_close, n_strands, chr_len, b, mode)
                o = _segment(checkers.signal_oracle_open, checkers.signal_oracle_segment, checkers.signal_oracle_close, n_strands, chr_len, b, mode)
                for (ep, ev), (op, ov) in zip(e, o):
                    assert np.array_equal(ep, op) and np.array_equal(ev.view(np.uint64), ov.view(np.uint64))


def _rc(exe, args, cwd):
    return subprocess.run([exe] + args, cwd=cwd, capture_output=True, text=True)


def test_parameter_errors(checkers, golden, tmp_path):
    base = ["--genomeDir", "idx", "--readFilesIn", "se_1.fq", "--outFileNamePrefix", str(tmp_path) + "/"]
    cases = [
        (["--outWigType", "bigWig", "--outSAMtype", "BAM", "SortedByCoordinate"], "unrecognized option in --outWigType=bigWig"),
        (["--outWigType", "bedGraph", "read3", "--outSAMtype", "BAM", "SortedByCoordinate"], "unrecognized second option in --outWigType=read3"),
        (["--outWigType", "bedGraph", "--outWigStrand", "Both", "--outSAMtype", "BAM", "SortedByCoordinate"], "unrecognized option in --outWigStrand=Both"),
        (["--outWigType", "bedGraph", "--outWigNorm", "CPM", "--outSAMtype", "BAM", "SortedByCoordinate"], "unrecognized option in --outWigNorm=CPM"),
        (["--outWigType", "bedGraph"], "generating signal with --outWigType requires sorted BAM"),
        (["--outWigType", "bedGraph", "--outSAMtype", "BAM", "Unsorted"], "generating signal with --outWigType requires sorted BAM"),
        (["--outWigType", "bedGraph", "--outSAMtype", "BAM", "SortedByCoordinate", "--outStd", "BAM_SortedByCoordinate"], "cannot be combined with --outStd"),
        (["--runMode", "inputAlignmentsFromBAM", "--inputBAMfile", "x.bam"], "only works with --outWigType bedGraph"),
        (["--bamRemoveDuplicatesType", "UniqueIdentical"], "outside the scope"),
    ]
    for extra, text in cases:
        r = _rc(SIGNAL_CLI, base + extra, golden)
        assert r.returncode == 102 and text in r.stderr, (extra, r.stderr)
    if os.path.exists(oc.REF_STAR):   # the texts and codes the reference gives for the same mistakes
        for extra, text in cases[:6] + cases[7:8]:
            r = _rc(oc.REF_STAR, base + extra, golden)
            assert r.returncode == 102 and text in r.stderr, (extra, r.stderr)


def test_bad_input_files(checkers, golden, tmp_path):
    refs, recs = bam_synth.random_bam(5, n=50)
    good = bam_synth.bam_bytes(refs, recs)
    cases = {"missing.bam": None, "text.bam": b"@HD\tVN:1.4\nnot a BAM\n", "trunc.bam": good[: len(good) // 2],
             "gzip_only.bam": __import__("gzip").compress(b"BAM\1" + b"\0" * 40), "nomagic.bam": bam_synth.bgzf(b"SAM\1" + b"\0" * 40),
             "cut_record.bam": bam_synth.bgzf(_raw_bam(refs, recs)[:-7])}
    for fn, data in cases.items():
        p = str(tmp_path / fn)
        if data is not None:
            open(p, "wb").write(data)
        r = _rc(SIGNAL_CLI, ["--runMode", "inputAlignmentsFromBAM", "--inputBAMfile", p, "--outWigType", "bedGraph", "--outFileNamePrefix", str(tmp_path / fn) + "."], golden)
        assert r.returncode == 104 and "--inputBAMfile" in r.stderr, (fn, r.stderr)
    # a record that runs past the extra base at the end of its reference: the reference's "BUG ... extends past chromosome" exit
    past = bam_synth.bam_bytes(refs, [bam_synth.record(1, refs[1][1] - 3, 0, [("M", 5)])])
    open(str(tmp_path / "past.bam"), "wb").write(past)
    r = _rc(SIGNAL_CLI, ["--runMode", "inputAlignmentsFromBAM", "--inputBAMfile", str(tmp_path / "past.bam"), "--outWigType", "bedGraph",
                            "--outFileNamePrefix", str(tmp_path / "past.")], golden)
    assert r.returncode == 104 and "extends past the end of reference chr2" in r.stderr, r.stderr


def _raw_bam(refs, recs):
    import gzip
    return gzip.decompress(bam_synth.bam_bytes(refs, recs))


def test_two_shards_and_merge_equal_single_process(checkers, lib, golden, tmp_path):
    """Shards leave their records to the merge; the tracks are made once from the merged BAM (what star_b200.dist does on rank 0)."""
    args = ["--genomeDir", "idx", "--readFilesIn", "hard_1.fq", "hard_2.fq", "--outSAMtype", "BAM", "SortedByCoordinate", "--outWigType", "bedGraph"]
    one = str(tmp_path / "one") + "/"
    subprocess.check_call([SIGNAL_CLI] + args + ["--outFileNamePrefix", one], cwd=golden, stdout=subprocess.DEVNULL)
    pre = str(tmp_path / "sh") + "/"
    for r in range(2):
        subprocess.check_call([SIGNAL_CLI] + args + ["--outFileNamePrefix", pre + "shard%d." % r, "--gpuShardIndex", str(r), "--gpuShardCount", "2"],
                              cwd=golden, stdout=subprocess.DEVNULL)
    assert not [f for f in os.listdir(pre) if "Signal" in f]   # shards write no tracks
    argv = [b"STAR"] + [os.path.join(golden, a).encode() if a in ("idx", "hard_1.fq", "hard_2.fq") else a.encode() for a in args] + [b"--outFileNamePrefix", pre.encode()]
    arr = (C.c_char_p * len(argv))(*argv)
    lib.star_host_merge_shards.argtypes = [C.c_int, C.POINTER(C.c_char_p), C.c_int, C.c_void_p]
    assert lib.star_host_merge_shards(len(argv), arr, 2, None) == 0
    import star_b200.dist as sd
    subprocess.check_call([SIGNAL_CLI] + sd.signal_args(args, pre), cwd=golden, stdout=subprocess.DEVNULL)
    _same_signal(pre, one)


@pytest.mark.skipif(not os.path.exists(oc.REF_STAR), reason="oracle/_ref/STAR not built (needs /root/reference)")
@pytest.mark.parametrize("seed", [101, 102, 103])
def test_fuzz_against_live_reference(checkers, golden, tmp_path, seed):
    import fuzz_signal
    assert fuzz_signal.check(seed, str(tmp_path), [SIGNAL_CLI], golden) == []


# ---- GPU ----------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_gpu_cli_equals_golden(lib, sig_golden, golden, tmp_path):
    sg, sc = sig_golden
    for name, args in sc.items():
        _same_signal(_run(OURS, name, args, sg, golden, str(tmp_path / name) + "/"), os.path.join(sg, name))


class _Track(C.Structure):
    _fields_ = [("pos", C.POINTER(C.c_uint32)), ("val", C.POINTER(C.c_double)), ("n", C.c_uint64)]


BLOCK = np.dtype([("start", "<u4"), ("len", "<u4"), ("nh", "<u4"), ("strand", "<u4")])


def _segment(open_, seg, close, n_strands, chr_len, blocks, mode):
    open_.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.c_uint32]
    seg.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.c_int, C.POINTER(_Track), C.POINTER(C.c_float)]
    close.argtypes = [C.c_void_p]
    close.restype = None
    h = C.c_void_p()
    assert open_(C.byref(h), 0, n_strands) == 0
    tr = (_Track * 4)()
    ms = C.c_float()
    assert seg(h, chr_len, blocks.ctypes.data, len(blocks), mode, tr, C.byref(ms)) == 0
    out = [(np.ctypeslib.as_array(tr[t].pos, (tr[t].n,)).copy() if tr[t].n else np.zeros(0, np.uint32),
            np.ctypeslib.as_array(tr[t].val, (tr[t].n,)).copy() if tr[t].n else np.zeros(0)) for t in range(2 * n_strands)]
    close(h)
    return out


@pytest.mark.gpu
def test_gpu_segment_bit_equal_to_oracle(lib, checkers):
    rng = np.random.default_rng(7)
    for n_strands, chr_len, n, deep in ((2, 5000, 20000, False), (1, 300000, 200000, False), (2, 2000, 60000, True)):
        b = np.zeros(n, BLOCK)
        if deep:   # one deep pile (chrM-like): every block covers the same few hundred bases
            b["start"] = rng.integers(0, 400, n)
        else:
            b["start"] = rng.integers(0, chr_len - 200, n)
        b["len"] = rng.integers(1, 150, n)
        b["nh"] = rng.choice([1, 1, 1, 2, 3, 5, 7, 11], n)
        b["strand"] = rng.integers(0, n_strands, n)
        for mode in (0, 1):
            import star_b200
            sig = star_b200.capi.Signal(lib, n_strands)
            g, _ = sig.segment(chr_len, b, mode)
            sig.close()
            o = _segment(checkers.signal_oracle_open, checkers.signal_oracle_segment, checkers.signal_oracle_close, n_strands, chr_len, b, mode)
            for (gp, gv), (op, ov) in zip(g, o):
                assert np.array_equal(gp, op) and np.array_equal(gv.view(np.uint64), ov.view(np.uint64))


@pytest.mark.gpu
@pytest.mark.skipif(not os.path.exists(oc.REF_STAR), reason="oracle/_ref/STAR not built")
def test_gpu_signal_of_config_size_bam_equals_reference(lib, tmp_path):
    """chr21-sized index (tests/test_gpu_config_gate.py) and 100 k pairs: our CLI's sorted BAM through our inputAlignmentsFromBAM and the
    reference's must give the same tracks; the tracks of the mapping run itself too."""
    import test_gpu_config_gate as gate
    import bench
    import synth
    wd = os.path.join(os.environ.get("STAR_B200_BENCH_DIR", "/tmp/star_b200_bench"), "chr21")
    os.makedirs(wd, exist_ok=True)
    chrs, trs, idx, _ = bench.prepare_genome(wd, "chr21")
    c = {"dir": wd, "chrs": chrs, "trs": trs, "idx": idx, "synth": synth}
    _, _, r1, r2 = gate._reads(c, 100000, 100, 0.005, 21, "sig")
    out = str(tmp_path / "map") + "/"
    subprocess.check_call([OURS, "--genomeDir", idx, "--readFilesIn", r1, r2, "--outSAMtype", "BAM", "SortedByCoordinate", "--outWigType", "bedGraph",
                           "--runThreadN", "8", "--outFileNamePrefix", out], stdout=subprocess.DEVNULL)
    bam = out + "Aligned.sortedByCoord.out.bam"
    for exe, d in ((OURS, "ours"), (oc.REF_STAR, "ref")):
        subprocess.check_call([exe, "--runMode", "inputAlignmentsFromBAM", "--inputBAMfile", bam, "--outWigType", "bedGraph", "--outWigStrand", "Stranded",
                               "--outFileNamePrefix", str(tmp_path / d) + "/"], stdout=subprocess.DEVNULL)
    _same_signal(str(tmp_path / "ours"), str(tmp_path / "ref"))
    _same_signal(out, str(tmp_path / "ref"))
