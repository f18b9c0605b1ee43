"""References added at the mapping stage (--genomeFastaFiles with --runMode alignReads, --outSAMfilter) against outputs of the UNMODIFIED
reference (tests/golden/addref.tar.xz, make_golden_addref.py): SAM / BAM records and @SQ lines, SJ.out.tab, Log.final.out, unmapped reads,
gene counts, the transcriptome BAM and, with --sjdbInsertSave All, the bytes of the grown Genome / SA / SAindex (by digest).

CPU (checkers of tests/addref_check/, built by build()): the repository's host code (star_b200/csrc/host/addref.cpp + driver + output
filter) with the oracle engine for mapping and (a) the sequential restatement of the three device steps or (b) the EMULATED CUDA kernels of
addref_kernels.cuh, through the test-only CLI build/addref_check/star_cli_addref; the emulated steps against the restatement on seeded
random inserts; parameter and file errors; a two-rank gloo run.
GPU: the drop-in CLI, the C-ABI calls against the restatement, and a chr21-sized run against the reference binary.
"""
import ctypes
import gzip
import json
import os
import subprocess
import tarfile

import numpy as np
import pytest

import conftest as cf
import oracle_capi as oc

ROOT = cf.ROOT
NAMES = ["A_pe", "B_se_noannot", "C_keeponly_within_keeppairs", "D_keepall_sorted_bam", "E_keepall_sam_keeppairs_allbest", "F_sjfile_save_noannot",
         "G_sjfile_save_annot", "H_gtf_quant_twopass", "I_bysjout_keepall", "J_intron_window"]
DIGEST_NAMES = ["F_sjfile_save_noannot", "G_sjfile_save_annot", "H_gtf_quant_twopass"]
CHECK_LIB = os.path.join(ROOT, "build", "addref_check", "libaddref_check.so")
CLI = os.path.join(ROOT, "build", "addref_check", "star_cli_addref")
COMMON = ["--outSAMattributes", "NH", "HI", "AS", "nM", "--runThreadN", "2"]


@pytest.fixture(scope="session")
def checkers(oracle, lib):
    """build/addref_check/ (tests/addref_check/Makefile; build() makes it)."""
    subprocess.check_call(["make", "-s", "-f", os.path.join("tests", "addref_check", "Makefile")], cwd=ROOT)
    return ctypes.CDLL(CHECK_LIB)


@pytest.fixture(scope="session")
def addref_golden(tmp_path_factory):
    """tiny/ and twopass/ (the indexes) and addref/ (inputs + reference outputs) unpacked side by side."""
    d = tmp_path_factory.mktemp("golden_addref")
    for t in ("tiny.tar.gz", "twopass.tar.gz"):
        with tarfile.open(os.path.join(ROOT, "tests", "golden", t)) as tf:
            tf.extractall(d)
    with tarfile.open(os.path.join(ROOT, "tests", "golden", "addref.tar.xz")) as tf:
        tf.extractall(d)
    return str(d)


def _args(g, name):
    sc = json.load(open(os.path.join(g, "addref", "scenarios.json")))[name]
    sub = {"IDX": os.path.join(g, "tiny", "idx"), "IDX0": os.path.join(g, "twopass", "idx0")}
    return [sub.get(a, os.path.join(g, "addref", a[3:]) if a.startswith("AR/") else a) for a in sc] + COMMON


def _sq(path):
    if path.endswith(".sam"):
        return [l for l in open(path).read().split("\n") if l.startswith("@SQ")]
    txt = gzip.decompress(open(path, "rb").read()).decode("latin-1")
    return [l for l in txt.split("\n") if l.startswith("@SQ")]


def check_outputs(out, ref):
    cf.check_twopass_outputs(out, ref)
    sq = [l for l in open(os.path.join(ref, "header.txt")).read().split("\n") if l]
    for f in ("Aligned.out.sam", "Aligned.out.bam", "Aligned.sortedByCoord.out.bam"):
        if os.path.exists(os.path.join(ref, f)):
            assert _sq(out + f) == sq, f
    for f in ("Unmapped.out.mate1", "Unmapped.out.mate2"):   # present exactly when the reference wrote them
        assert os.path.exists(out + f) == os.path.exists(os.path.join(ref, f)), f


def _run(cli, g, name, out, env=None):
    subprocess.check_call([cli] + _args(g, name) + ["--outFileNamePrefix", out], stdout=subprocess.DEVNULL, env=env)


@pytest.mark.parametrize("name", NAMES)
def test_oracle_cli_addref_matches_reference(checkers, addref_golden, tmp_path, name):
    out = str(tmp_path) + "/"
    _run(CLI, addref_golden, name, out)
    check_outputs(out, os.path.join(addref_golden, "addref", name))


@pytest.mark.parametrize("name", DIGEST_NAMES)
def test_emulated_addref_kernels_match_reference(checkers, addref_golden, tmp_path, name):
    """addref_rebase_kernel / addref_search_kernel / sjdb_merge_sa_kernel<AddrefMerge> compiled for the host, inside the whole run."""
    out = str(tmp_path) + "/"
    _run(CLI, addref_golden, name, out, env=dict(os.environ, STAR_ADDREF_EMUL="1"))
    check_outputs(out, os.path.join(addref_golden, "addref", name))


def test_keepall_counts_only_added_alignments(addref_golden):
    """KeepAll: a read that maps to chr1 and to its copy is written once, NH:i:1 and MAPQ 255 (the reference's own output)."""
    sam = [l.split("\t") for l in open(os.path.join(addref_golden, "addref", "E_keepall_sam_keeppairs_allbest", "Aligned.out.sam")) if not l.startswith("@")]
    dup = [r for r in sam if r[2] == "dupchr1"]
    assert dup and all(r[4] == "255" and "NH:i:1" in r for r in dup)
    allpe = [l.split("\t") for l in open(os.path.join(addref_golden, "addref", "A_pe", "Aligned.out.sam")) if not l.startswith("@")]
    assert any(r[2] == "dupchr1" and "NH:i:2" in r for r in allpe)   # unfiltered: the same reads are multimappers


# ---- the device steps against the sequential restatement ------------------------------------------------------------------------
def _sa_build(G, nGenome, GstrandBit):
    """A suffix array of G by the oracle's restatement of the suffix sort (star_oracle_sa_build)."""
    lib = oc.load_oracle()
    nSA = 2 * int(np.count_nonzero(G[256:256 + nGenome] < 4))
    nSAbyte = (nSA - 1) * (GstrandBit + 1) // 8 + 8
    SA = np.zeros(nSAbyte + 16, np.uint8)
    lib.star_oracle_sa_build.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_uint64, ctypes.c_uint32, ctypes.c_uint64, ctypes.c_void_p, ctypes.c_uint64]
    assert lib.star_oracle_sa_build(0, G.ctypes.data + 256, nGenome, GstrandBit, nSA, SA.ctypes.data, nSAbyte) == 0
    return SA, nSA, nSAbyte


def random_case(seed, nOld, nIns, nJunc):
    """A grown genome: nOld bases of old chromosomes (with a repeat and an N run), an insert of nIns bases (partly copied from the old
    text, forward and reverse complement, poly-A tails, N runs) and nJunc bytes of a junction region behind it; the old suffix array is
    the suffix array of old + junction region."""
    rng = np.random.default_rng(seed)
    old = rng.integers(0, 4, nOld).astype(np.uint8)
    if nOld > 400:
        old[nOld // 2:nOld // 2 + 150] = old[10:160]
        old[100:120] = 4
    nG = ((nOld + 1) // 256 + 1) * 256
    ins = rng.integers(0, 4, nIns).astype(np.uint8)
    k = 0
    while k + 60 < nIns:   # copies of old text, reverse complements, poly-A, N
        kind = rng.integers(0, 4)
        L = int(rng.integers(20, 60))
        p = int(rng.integers(0, max(1, nOld - L)))
        if kind == 0:
            ins[k:k + L] = old[p:p + L]
        elif kind == 1:
            ins[k:k + L] = 3 - old[p:p + L][::-1]
        elif kind == 2:
            ins[k:k + L] = 0
        else:
            ins[k:k + 5] = 4
        k += L + int(rng.integers(0, 80))
    nG1 = ((nIns + 1) // 256 + 1) * 256
    junc = rng.integers(0, 4, nJunc).astype(np.uint8)
    if nJunc:
        junc[30::31] = 5
    G0 = np.full(256 + nG + nJunc + 256, 5, np.uint8)
    G0[256:256 + nOld] = old
    G0[256 + nG:256 + nG + nJunc] = junc
    G1 = np.full(256 + nG + nG1 + nJunc + 256, 5, np.uint8)
    G1[256:256 + nOld] = old
    G1[256 + nG:256 + nG + nIns] = ins
    G1[256 + nG + nG1:256 + nG + nG1 + nJunc] = junc
    return G0, G1, nG, nG1, nJunc


def _view(G, nGenome, SA, nSA, nSAbyte, GstrandBit):
    """A star_index_view_t with the fields the addref calls read."""
    import star_b200.capi as capi
    v = capi.IndexView()
    v.G = G.ctypes.data + 256
    v.nGenome = nGenome
    v.SA = SA.ctypes.data
    v.nSA = nSA
    v.nSAbyte = nSAbyte
    v.GstrandBit = GstrandBit
    return v


def _steps(lib, prefix, v, nG, nG1, nG2, text):
    """open / search / the sort of the insertion points (the restatement's qsort) / merge through one library; returns (indArray, merged SA)."""
    import star_b200.capi as capi
    a = capi.AddRef(lib, v, nG, nG1, nG2, prefix=prefix)
    ind, _ = a.search(text)
    keep = np.ascontiguousarray(ind[ind[:, 0] != np.uint64(2**64 - 1)])
    clib = ctypes.CDLL(CHECK_LIB)
    clib.addref_oracle_sort.argtypes = [ctypes.c_void_p, ctypes.c_uint64, ctypes.c_void_p, ctypes.c_uint64]
    assert clib.addref_oracle_sort(text.ctypes.data, nG1, keep.ctypes.data, len(keep)) == 0
    sa, _ = a.merge_sa(keep)
    a.close()
    return ind.copy(), sa.copy()


def _text(G1, nG, nG1):
    fwd = G1[256 + nG:256 + nG + nG1]
    rcv = np.where(fwd[::-1] < 4, 3 - fwd[::-1], fwd[::-1]).astype(np.uint8)
    return np.concatenate([fwd, rcv]).astype(np.uint8)


CASES = [(1, 700, 300, 0), (2, 900, 500, 124), (3, 300, 1200, 62), (4, 500, 2000, 0)]   # inserts larger than the genome: long tie runs


@pytest.mark.parametrize("seed,nOld,nIns,nJunc", CASES)
def test_emulated_addref_steps_match_restatement(checkers, seed, nOld, nIns, nJunc):
    G0, G1, nG, nG1, nG2 = random_case(seed, nOld, nIns, nJunc)
    GstrandBit = 32
    SA, nSA, nSAbyte = _sa_build(G0, nG + nG2, GstrandBit)
    v = _view(G1, nG + nG1 + nG2, SA, nSA, nSAbyte, GstrandBit)
    text = _text(G1, nG, nG1)
    ref = _steps(checkers, "addref_oracle", v, nG, nG1, nG2, text)
    emu = _steps(checkers, "addref_emul", v, nG, nG1, nG2, text)
    assert np.array_equal(ref[0], emu[0])
    assert np.array_equal(ref[1], emu[1])


def test_addref_parameter_and_file_errors(checkers, addref_golden, tmp_path):
    """Parameters.cpp:740-760 and genomeScanFastaFiles.cpp:15-36: the reference's exit codes and texts."""
    g = addref_golden
    base = [CLI, "--genomeDir", os.path.join(g, "twopass", "idx0"), "--readFilesIn", os.path.join(g, "addref", "se_1.fq"), "--outFileNamePrefix", str(tmp_path) + "/"]
    fa = os.path.join(g, "addref", "addB.fa")

    def run(extra):
        p = subprocess.run(base + extra, stdout=subprocess.DEVNULL, stderr=subprocess.PIPE)
        return p.returncode, p.stderr.decode()
    rc, e = run(["--outSAMfilter", "KeepSome", "--genomeFastaFiles", fa])
    assert rc == 102 and "unknown/unimplemented value for --outSAMfilter: KeepSome" in e and "KeepOnlyAddedReferences or None" in e
    rc, e = run(["--outSAMfilter", "KeepAllAddedReferences"])
    assert rc == 102 and "--genomeFataFiles" in e
    rc, e = run(["--outSAMfilter", "KeepOnlyAddedReferences"])
    assert rc == 102
    rc, e = run(["--genomeFastaFiles", fa, "--genomeLoad", "LoadAndKeep"])
    assert rc == 102 and "shared memory genome" in e
    rc, e = run(["--genomeFastaFiles", os.path.join(str(tmp_path), "missing.fa")])
    assert rc == 104 and "could not open genomeFastaFile" in e
    empty = os.path.join(str(tmp_path), "empty.fa")
    open(empty, "w").close()
    rc, e = run(["--genomeFastaFiles", empty])
    assert rc == 104 and "could not read from genomeFastaFile" in e
    notfa = os.path.join(str(tmp_path), "x.fa")
    open(notfa, "w").write("ACGT\n")
    rc, e = run(["--genomeFastaFiles", fa, notfa])
    assert rc == 104 and "is not fasta: the first character is 'A' (65)" in e
    assert run(["--outSAMfilter", "None"])[0] == 0


def test_two_rank_gloo_equals_single_process(checkers, addref_golden, tmp_path):
    """star_b200.dist over gloo with the oracle-driven CLI: every rank adds the references to its replica, the merge sees them as well; the
    merged SAM (@SQ lines included), junctions and counters equal one process's output."""
    import sys
    out = str(tmp_path / "two") + "/"
    env = dict(os.environ)
    env["PYTHONPATH"] = ROOT + os.pathsep + env.get("PYTHONPATH", "")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1", "--master-port", "29619",
           "-m", "star_b200.dist", "--cli", CLI, "--"] + _args(addref_golden, "C_keeponly_within_keeppairs") + ["--outFileNamePrefix", out]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    one = str(tmp_path / "one") + "/"
    _run(CLI, addref_golden, "C_keeponly_within_keeppairs", one)
    assert cf.sam_body(out + "Aligned.out.sam") == cf.sam_body(one + "Aligned.out.sam")
    assert _sq(out + "Aligned.out.sam") == _sq(one + "Aligned.out.sam")
    assert open(out + "SJ.out.tab").read() == open(one + "SJ.out.tab").read()
    assert cf.log_counters(out + "Log.final.out") == cf.log_counters(one + "Log.final.out")


# ---- GPU -------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_gpu_cli_addref_matches_reference(lib, addref_golden, tmp_path, name):
    out = str(tmp_path) + "/"
    _run(os.path.join(ROOT, "star_b200", "bin", "STAR"), addref_golden, name, out)
    check_outputs(out, os.path.join(addref_golden, "addref", name))


@pytest.mark.gpu
@pytest.mark.parametrize("seed,nOld,nIns,nJunc", CASES + [(11, 200000, 1 << 20, 5000), (12, 1 << 20, 2 << 20, 0)])
def test_gpu_addref_calls_match_restatement(lib, checkers, seed, nOld, nIns, nJunc):
    """star_gpu_addref_* (through star_b200.capi.AddRef) against the oracle's restatement, up to a 2 Mb insert."""
    G0, G1, nG, nG1, nG2 = random_case(seed, nOld, nIns, nJunc)
    GstrandBit = 32
    SA, nSA, nSAbyte = _sa_build(G0, nG + nG2, GstrandBit)
    v = _view(G1, nG + nG1 + nG2, SA, nSA, nSAbyte, GstrandBit)
    text = _text(G1, nG, nG1)
    ref = _steps(checkers, "addref_oracle", v, nG, nG1, nG2, text)
    gpu = _steps(lib, "star_gpu_addref", v, nG, nG1, nG2, text)
    assert np.array_equal(ref[0], gpu[0])
    assert np.array_equal(ref[1], gpu[1])


@pytest.mark.gpu
def test_gpu_cli_equals_reference_at_chr21_size(lib, tmp_path):
    """The chr21-sized genome of test_gpu_config_gate.py (index built by the reference's genomeGenerate) with 92 ERCC-like spikes and a 20 kb
    copy of a chromosome added, 100 k pairs of genome / transcript reads plus 5 k pairs from the added references, a junction on a spike and
    --sjdbInsertSave All: the drop-in CLI and oracle/_ref/STAR --runThreadN 1 write the same SAM records (and @SQ lines), SJ.out.tab,
    counters and grown Genome / SA / SAindex."""
    import hashlib
    import bench
    import synth
    ref_star = os.path.join(ROOT, "oracle", "_ref", "STAR")
    if not os.path.exists(ref_star):
        pytest.skip("the reference binary was not built (no reference checkout)")
    wd = os.path.join(os.environ.get("STAR_B200_BENCH_DIR", "/tmp/star_b200_bench"), "chr21")
    os.makedirs(wd, exist_ok=True)
    chrs, trs, idx, _ = bench.prepare_genome(wd, "chr21")
    spikes = synth.make_spikes(chrs)
    fa = str(tmp_path / "spikes.fa")
    synth.write_fasta(spikes, fa)
    m1, m2 = synth.make_reads(chrs, trs, 100_000, read_len=100, mm=0.005, seed=91)
    s1, s2 = synth.make_reads(spikes, [], 5_000, read_len=100, mm=0.005, seed=93, tx_frac=0.0)
    f1, f2 = str(tmp_path / "r_1.fq"), str(tmp_path / "r_2.fq")
    synth.write_fastq(np.concatenate([m1, s1]), f1)
    synth.write_fastq(np.concatenate([m2, s2]), f2)
    sj = str(tmp_path / "sj.tab")
    open(sj, "w").write("%s\t201\t300\t+\n" % spikes[0][0])
    outs = {}
    for tag, binary, threads in (("ours", os.path.join(ROOT, "star_b200", "bin", "STAR"), "16"), ("ref", ref_star, "1")):
        out = str(tmp_path / tag) + "/"
        subprocess.check_call([binary, "--genomeDir", idx, "--genomeFastaFiles", fa, "--readFilesIn", f1, f2, "--sjdbFileChrStartEnd", sj,
                               "--sjdbInsertSave", "All", "--runThreadN", threads, "--outFileNamePrefix", out], stdout=subprocess.DEVNULL, timeout=3000)
        outs[tag] = out
    a, b = cf.sam_body(outs["ours"] + "Aligned.out.sam"), cf.sam_body(outs["ref"] + "Aligned.out.sam")
    assert len(a) == len(b)
    bad = [i for i in range(len(a)) if a[i] != b[i]]
    assert not bad, "%d of %d SAM records differ, first:\n%s\n%s" % (len(bad), len(a), a[bad[0]], b[bad[0]])
    assert _sq(outs["ours"] + "Aligned.out.sam") == _sq(outs["ref"] + "Aligned.out.sam")
    assert sum(1 for r in a if r.split(b"\t")[2].startswith(b"ERCC-")) > 1000
    assert open(outs["ours"] + "SJ.out.tab", "rb").read() == open(outs["ref"] + "SJ.out.tab", "rb").read()
    assert cf.log_counters(outs["ours"] + "Log.final.out") == cf.log_counters(outs["ref"] + "Log.final.out")
    for f in ("Genome", "SA", "SAindex", "sjdbInfo.txt", "sjdbList.out.tab"):
        d = [hashlib.sha256(open(outs[t] + "_STARgenome/" + f, "rb").read()).hexdigest() for t in ("ours", "ref")]
        assert d[0] == d[1], f
