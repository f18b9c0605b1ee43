"""ctypes binding of the C-ABI in include/star_b200.h (star_b200/lib/libstar_b200.so).

The library is the product: hand-written sm_90a CUDA kernels behind plain C entry points.  This
module only moves pointers; it contains no alignment logic and no fallback: if the shared library
is missing, import fails loudly, and without a CUDA device `Engine()` raises.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("STAR_B200_LIB", os.path.join(_HERE, "lib", "libstar_b200.so"))   # the override is for A/B builds of the same ABI

MAX_EX = 20


class Params(C.Structure):
    _fields_ = [
        ("seedSearchStartLmax", C.c_uint64), ("seedSearchStartLmaxOverLread", C.c_double), ("seedSearchLmax", C.c_uint64),
        ("seedMapMin", C.c_uint64), ("seedSplitMin", C.c_uint64), ("seedMultimapNmax", C.c_uint64), ("seedPerReadNmax", C.c_uint64),
        ("seedPerWindowNmax", C.c_uint64), ("maxNsplit", C.c_uint64),
        ("winAnchorMultimapNmax", C.c_uint64), ("winBinNbits", C.c_uint64), ("winBinChrNbits", C.c_uint64), ("winAnchorDistNbins", C.c_uint64),
        ("winFlankNbins", C.c_uint64), ("winBinN", C.c_uint64), ("alignWindowsPerReadNmax", C.c_uint64),
        ("alignTranscriptsPerWindowNmax", C.c_uint64), ("alignTranscriptsPerReadNmax", C.c_uint64),
        ("alignIntronMin", C.c_uint64), ("alignIntronMax", C.c_uint64), ("alignMatesGapMax", C.c_uint64), ("alignSJoverhangMin", C.c_uint64),
        ("alignSJDBoverhangMin", C.c_uint64), ("alignSJstitchMismatchNmax", C.c_int32 * 4), ("alignSplicedMateMapLmin", C.c_uint64),
        ("alignSplicedMateMapLminOverLmate", C.c_double), ("alignEndsTypeExt", (C.c_uint8 * 2) * 2), ("alignEndsProtrudeNbasesMax", C.c_int32),
        ("alignEndsProtrudeConcordantPair", C.c_uint8), ("alignSoftClipAtReferenceEnds", C.c_uint8), ("alignInsertionFlushRight", C.c_uint8),
        ("scoreGap", C.c_int32), ("scoreGapNoncan", C.c_int32), ("scoreGapGCAG", C.c_int32), ("scoreGapATAC", C.c_int32),
        ("scoreGenomicLengthLog2scale", C.c_double),
        ("scoreDelOpen", C.c_int32), ("scoreDelBase", C.c_int32), ("scoreInsOpen", C.c_int32), ("scoreInsBase", C.c_int32),
        ("scoreStitchSJshift", C.c_int32), ("sjdbScore", C.c_int32),
        ("outFilterMismatchNmax", C.c_uint64), ("outFilterMismatchNoverLmax", C.c_double), ("outFilterMismatchNoverReadLmax", C.c_double),
        ("outFilterMultimapScoreRange", C.c_int32), ("outFilterMultimapNmax", C.c_uint64), ("outFilterScoreMin", C.c_int32),
        ("outFilterScoreMinOverLread", C.c_double), ("outFilterMatchNmin", C.c_uint64), ("outFilterMatchNminOverLread", C.c_double),
        ("outFilterIntronMotifs", C.c_uint8), ("outFilterIntronStrandsRemoveInconsistent", C.c_uint8), ("outSAMstrandFieldType", C.c_uint8),
        ("outSAMprimaryFlagAllBestScore", C.c_uint8), ("outSAMmultNmax", C.c_uint64),
    ]


class IndexView(C.Structure):
    _fields_ = [
        ("G", C.c_void_p), ("nGenome", C.c_uint64), ("SA", C.c_void_p), ("nSA", C.c_uint64), ("nSAbyte", C.c_uint64),
        ("SAi", C.c_void_p), ("nSAi", C.c_uint64), ("nSAibyte", C.c_uint64), ("GstrandBit", C.c_uint32), ("gSAindexNbases", C.c_uint32),
        ("gSAsparseD", C.c_uint32), ("gChrBinNbits", C.c_uint32), ("genomeSAindexStart", C.c_void_p), ("nChrReal", C.c_uint32),
        ("chrStart", C.c_void_p), ("chrLength", C.c_void_p), ("sjdbN", C.c_uint64), ("sjdbOverhang", C.c_uint64), ("sjdbLength", C.c_uint64),
        ("sjGstart", C.c_uint64), ("sjdbStart", C.c_void_p), ("sjdbEnd", C.c_void_p), ("sjDstart", C.c_void_p), ("sjAstart", C.c_void_p),
        ("sjdbMotif", C.c_void_p), ("sjdbShiftLeft", C.c_void_p), ("sjdbShiftRight", C.c_void_p), ("sjdbStrand", C.c_void_p),
    ]


class ReadBatch(C.Structure):
    _fields_ = [("nReads", C.c_uint32), ("nMates", C.c_uint32), ("seq", C.c_void_p), ("seqOff", C.c_void_p)]


class AlignBatch(C.Structure):
    _fields_ = [("reads", C.c_void_p), ("aligns", C.c_void_p), ("alignsCapacity", C.c_uint64), ("nAligns", C.c_uint64)]


class ChunkStats(C.Structure):
    _fields_ = [(n, C.c_float) for n in ("ms_h2d", "ms_prep", "ms_seed", "ms_window", "ms_stitch", "ms_pack", "ms_d2h", "ms_total")] + \
               [(n, C.c_uint64) for n in ("h2d_bytes", "d2h_bytes", "n_kernel_launches", "mmp_searches", "mmp_sai_words", "mmp_compare_calls",
                                          "mmp_bases_examined", "sa_enumerated", "stitch_nodes", "stitch_leaves", "slow_path_reads", "heavy_reads")] + \
               [("ms_heavy", C.c_float), ("pad_", C.c_float)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


ALIGN_DTYPE = np.dtype([
    ("exG", "<u8", (MAX_EX,)), ("exR", "<u2", (MAX_EX,)), ("exL", "<u2", (MAX_EX,)), ("exFrag", "u1", (MAX_EX,)), ("canonSJ", "i1", (MAX_EX,)),
    ("sjAnnot", "u1", (MAX_EX,)), ("sjStr", "u1", (MAX_EX,)), ("shiftSJ", "<u2", (MAX_EX, 2)), ("nExons", "<u4"), ("Chr", "<u4"),
    ("Str", "u1"), ("roStr", "u1"), ("primaryFlag", "u1"), ("sjMotifStrand", "u1"), ("iFrag", "<i4"), ("maxScore", "<i4"),
    ("nMatch", "<u4"), ("nMM", "<u4"), ("nGap", "<u4"), ("lGap", "<u4"), ("nDel", "<u4"), ("lDel", "<u4"), ("nIns", "<u4"), ("lIns", "<u4"),
    ("nUnique", "<u4"), ("nAnchor", "<u4"), ("rStart", "<u4"), ("rLength", "<u4"), ("roStart", "<u4"),
    ("gStart", "<u8"), ("gLength", "<u8"), ("cStart", "<u8"),
])
assert ALIGN_DTYPE.itemsize == 496
RESULT_DTYPE = np.dtype({
    "names": ["unmapType", "nTr", "nTrOut", "mapMarker", "trOffset", "bestScore", "bestNMM", "bestRLength", "Lread", "bestTr"],
    "formats": ["<i4", "<u4", "<u4", "<u4", "<u8", "<i4", "<u4", "<u4", "<u4", "<u4"],
    "offsets": [0, 4, 8, 12, 16, 24, 28, 32, 36, 40],
    "itemsize": 48,
})


class SignalTrack(C.Structure):
    _fields_ = [("pos", C.POINTER(C.c_uint32)), ("val", C.POINTER(C.c_double)), ("n", C.c_uint64)]


SIGNAL_BLOCK_DTYPE = np.dtype([("start", "<u4"), ("len", "<u4"), ("nh", "<u4"), ("strand", "<u4")])   # star_signal_block_t


def load_library(path=LIB_PATH):
    if not os.path.exists(path):
        raise ImportError("star_b200: %s is missing; run `python -c 'import __graft_entry__ as g; g.build()'` (or `make`) first — "
                          "there is no Python/CPU fallback" % path)
    lib = C.CDLL(path, mode=C.RTLD_GLOBAL)
    lib.star_gpu_init.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.POINTER(IndexView), C.POINTER(Params), C.c_uint32]
    lib.star_gpu_init.restype = C.c_int
    lib.star_gpu_map_chunk.argtypes = [C.c_void_p, C.POINTER(ReadBatch), C.POINTER(AlignBatch), C.POINTER(ChunkStats)]
    lib.star_gpu_map_chunk.restype = C.c_int
    lib.star_gpu_upload_chunk.argtypes = [C.c_void_p, C.POINTER(ReadBatch)]
    lib.star_gpu_upload_chunk.restype = C.c_int
    lib.star_gpu_map_resident.argtypes = [C.c_void_p, C.POINTER(ChunkStats)]
    lib.star_gpu_map_resident.restype = C.c_int
    lib.star_gpu_download_results.argtypes = [C.c_void_p, C.POINTER(AlignBatch)]
    lib.star_gpu_download_results.restype = C.c_int
    lib.star_gpu_destroy.argtypes = [C.c_void_p]
    lib.star_gpu_destroy.restype = None
    lib.star_gpu_last_error.restype = C.c_char_p
    lib.star_gpu_launch_count.restype = C.c_uint64
    lib.star_params_default.argtypes = [C.POINTER(Params)]
    lib.star_index_load.argtypes = [C.c_char_p, C.POINTER(Params), C.POINTER(C.c_void_p)]
    lib.star_index_load.restype = C.c_int
    lib.star_index_get.argtypes = [C.c_void_p]
    lib.star_index_get.restype = C.POINTER(IndexView)
    lib.star_index_free.argtypes = [C.c_void_p]
    lib.star_host_last_error.restype = C.c_char_p
    lib.star_cli_main.argtypes = [C.c_int, C.POINTER(C.c_char_p)]
    lib.star_cli_main.restype = C.c_int
    lib.star_gpu_signal_open.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.c_uint32]
    lib.star_gpu_signal_open.restype = C.c_int
    lib.star_gpu_signal_segment.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.c_int, C.POINTER(SignalTrack), C.POINTER(C.c_float)]
    lib.star_gpu_signal_segment.restype = C.c_int
    lib.star_gpu_signal_close.argtypes = [C.c_void_p]
    lib.star_gpu_signal_close.restype = None
    lib.star_gpu_dedup_open.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.c_uint64]
    lib.star_gpu_dedup_open.restype = C.c_int
    lib.star_gpu_dedup_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.POINTER(C.c_float)]
    lib.star_gpu_dedup_batch.restype = C.c_int
    lib.star_gpu_dedup_close.argtypes = [C.c_void_p]
    lib.star_gpu_dedup_close.restype = None
    return lib


class Signal:
    """star_gpu_signal_open / _segment / _close: the per-base tracks of one segment from its blocks (SIGNAL_BLOCK_DTYPE, record order)."""

    def __init__(self, lib, n_strands, device=0):
        self.lib = lib
        self.n_tracks = 2 * n_strands
        h = C.c_void_p()
        rc = lib.star_gpu_signal_open(C.byref(h), device, n_strands)
        if rc:
            raise StarError(rc, lib.star_gpu_last_error().decode())
        self.h = h

    def segment(self, chr_len, blocks, mode=0):
        """mode 0 (bedGraph): positions where a track changes; 1 (wiggle): nonzero positions.  Returns [(pos, val)] per track, device ms."""
        blocks = np.ascontiguousarray(blocks, dtype=SIGNAL_BLOCK_DTYPE)
        tr = (SignalTrack * 4)()
        ms = C.c_float()
        rc = self.lib.star_gpu_signal_segment(self.h, chr_len, blocks.ctypes.data, len(blocks), mode, tr, C.byref(ms))
        if rc:
            raise StarError(rc, self.lib.star_gpu_last_error().decode())
        out = [(np.ctypeslib.as_array(t.pos, (t.n,)).copy(), np.ctypeslib.as_array(t.val, (t.n,)).copy()) if t.n else
               (np.zeros(0, np.uint32), np.zeros(0)) for t in tr[:self.n_tracks]]
        return out, ms.value

    def close(self):
        if self.h:
            self.lib.star_gpu_signal_close(self.h)
            self.h = None


class Dedup:
    """star_gpu_dedup_open / _batch / _close: the pairs to un-mark among the NH == 1 members of whole groups (bamRemoveDuplicates)."""

    def __init__(self, lib, mate2_bases_n=0, device=0):
        self.lib = lib
        h = C.c_void_p()
        rc = lib.star_gpu_dedup_open(C.byref(h), device, mate2_bases_n)
        if rc:
            raise StarError(rc, lib.star_gpu_last_error().decode())
        self.h = h

    def batch(self, data, offsets, groups):
        """data: the record bytes (uint8); offsets: uint64 offset of every member's record in data (increasing); groups: uint32 group of
        every member (non-decreasing).  Returns (rc, unmark uint8 per member, device ms); rc != 0 is an input error, and unmark then holds
        2 + kind at the member it names (include/star_b200.h)."""
        data = np.ascontiguousarray(data, dtype=np.uint8)
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        groups = np.ascontiguousarray(groups, dtype=np.uint32)
        unmark = np.zeros(len(offsets), np.uint8)
        ms = C.c_float()
        rc = self.lib.star_gpu_dedup_batch(self.h, data.ctypes.data, offsets.ctypes.data, groups.ctypes.data, len(offsets), unmark.ctypes.data, C.byref(ms))
        if rc not in (0, 102, 104):
            raise StarError(rc, self.lib.star_gpu_last_error().decode())
        return rc, unmark, ms.value

    def close(self):
        if self.h:
            self.lib.star_gpu_dedup_close(self.h)
            self.h = None


class AddRef:
    """star_gpu_addref_open / _search / _merge_sa / _close: the device steps of adding references (include/star_b200.h).  prefix names
    another library's functions with the same signatures (the CPU restatement and the emulated kernels of the tests)."""

    def __init__(self, lib, view, nG, nG1, nG2, device=0, prefix="star_gpu_addref"):
        self.lib, self.nG1, self.view = lib, nG1, view
        self.f = {k: getattr(lib, prefix + "_" + k) for k in ("open", "search", "merge_sa", "close")}
        self.f["open"].argtypes = [C.POINTER(C.c_void_p), C.c_int, C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, C.c_void_p]
        self.f["search"].argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        self.f["merge_sa"].argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p]
        self.f["close"].argtypes = [C.c_void_p]
        self.f["close"].restype = None
        h = C.c_void_p()
        ms = C.c_float()
        rc = self.f["open"](C.byref(h), device, C.addressof(view), nG, nG1, nG2, C.addressof(ms))
        if rc:
            raise StarError(rc, "addref open failed")
        self.h, self.ms_open = h, ms.value

    def search(self, text):
        """text: the 2*nG1 bytes forward + reverse complement.  Returns (indArray uint64 [2*nG1, 2], device ms)."""
        text = np.ascontiguousarray(text, dtype=np.uint8)
        ind = np.zeros(4 * self.nG1 + 2, np.uint64)
        ms = C.c_float()
        rc = self.f["search"](self.h, text.ctypes.data, ind.ctypes.data, C.addressof(ms))
        if rc:
            raise StarError(rc, "addref search failed")
        return ind[:4 * self.nG1].reshape(-1, 2), ms.value

    def merge_sa(self, ind_sorted):
        """ind_sorted: (nInd, 2) uint64 in insertion order.  Returns (the merged SA bytes, device ms)."""
        ind_sorted = np.ascontiguousarray(ind_sorted, dtype=np.uint64)
        nInd = len(ind_sorted)
        nSAnew = self.view.nSA + nInd
        nbyte = (nSAnew - 1) * (self.view.GstrandBit + 1) // 8 + 8
        out = np.zeros(nbyte + 16, np.uint8)
        ms = C.c_float()
        rc = self.f["merge_sa"](self.h, ind_sorted.ctypes.data, nInd, out.ctypes.data, nbyte, C.addressof(ms))
        if rc:
            raise StarError(rc, "addref merge failed")
        return out[:nbyte], ms.value

    def close(self):
        if self.h:
            self.f["close"](self.h)
            self.h = None


class StarError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("star_b200 error %d: %s" % (code, msg))
        self.code = code


class Index:
    """A STAR genomeDir loaded into host memory (star_index_load)."""

    def __init__(self, lib, genome_dir, params=None):
        self.lib = lib
        self.params = params if params is not None else default_params(lib)
        h = C.c_void_p()
        rc = lib.star_index_load(genome_dir.encode(), C.byref(self.params), C.byref(h))
        if rc:
            raise StarError(rc, lib.star_host_last_error().decode())
        self.handle = h
        self.view = lib.star_index_get(h)

    def close(self):
        if self.handle:
            self.lib.star_index_free(self.handle)
            self.handle = None


def default_params(lib):
    p = Params()
    lib.star_params_default(C.byref(p))
    return p


def pack_reads(mates):
    """mates: list (per mate) of lists of bytes objects, or (n, L) uint8 arrays -> (seq uint8 array, off uint64 array, nReads, nMates)."""
    n_mates = len(mates)
    if isinstance(mates[0], np.ndarray) and mates[0].ndim == 2:
        n = mates[0].shape[0]
        lens = np.stack([np.full(n, m.shape[1], dtype=np.uint64) for m in mates], axis=1).reshape(-1)
        off = np.zeros(n * n_mates + 1, dtype=np.uint64)
        np.cumsum(lens, out=off[1:])
        if n_mates == 1:
            seq = np.ascontiguousarray(mates[0]).reshape(-1)
        else:
            seq = np.concatenate([mates[0], mates[1]], axis=1).reshape(-1)
        return np.ascontiguousarray(seq, dtype=np.uint8), off, n, n_mates
    n = len(mates[0])
    parts = []
    lens = np.empty(n * n_mates, dtype=np.uint64)
    for i in range(n):
        for m in range(n_mates):
            parts.append(mates[m][i])
            lens[i * n_mates + m] = len(mates[m][i])
    off = np.zeros(n * n_mates + 1, dtype=np.uint64)
    np.cumsum(lens, out=off[1:])
    seq = np.frombuffer(b"".join(parts), dtype=np.uint8).copy()
    return seq, off, n, n_mates


class _EngineBase:
    """Shared call plumbing of the CUDA engine (and, in tests only, of the oracle which exports the same shapes)."""

    def _batch(self, seq, off, n, n_mates):
        b = ReadBatch()
        b.nReads = n
        b.nMates = n_mates
        b.seq = seq.ctypes.data
        b.seqOff = off.ctypes.data
        return b

    def _out(self, n, n_out):
        res = np.zeros(n, dtype=RESULT_DTYPE)
        al = np.zeros(max(1, n * n_out), dtype=ALIGN_DTYPE)
        ab = AlignBatch()
        ab.reads = res.ctypes.data
        ab.aligns = al.ctypes.data
        ab.alignsCapacity = al.shape[0]
        ab.nAligns = 0
        return res, al, ab


class Engine(_EngineBase):
    """star_gpu_init / star_gpu_map_chunk / star_gpu_destroy."""

    def __init__(self, lib, index, max_reads, device=0):
        self.lib = lib
        self.index = index
        self.n_out = max(1, int(index.params.outFilterMultimapNmax))
        ctx = C.c_void_p()
        rc = lib.star_gpu_init(C.byref(ctx), device, index.view, C.byref(index.params), max_reads)
        if rc:
            raise StarError(rc, lib.star_gpu_last_error().decode())
        self.ctx = ctx

    def map_chunk(self, seq, off, n, n_mates, out=None):
        b = self._batch(seq, off, n, n_mates)
        res, al, ab = out if out is not None else self._out(n, self.n_out)
        st = ChunkStats()
        rc = self.lib.star_gpu_map_chunk(self.ctx, C.byref(b), C.byref(ab), C.byref(st))
        if rc:
            raise StarError(rc, self.lib.star_gpu_last_error().decode())
        return res, al[:ab.nAligns], st

    def upload(self, seq, off, n, n_mates):
        b = self._batch(seq, off, n, n_mates)
        rc = self.lib.star_gpu_upload_chunk(self.ctx, C.byref(b))
        if rc:
            raise StarError(rc, self.lib.star_gpu_last_error().decode())

    def map_resident(self):
        st = ChunkStats()
        rc = self.lib.star_gpu_map_resident(self.ctx, C.byref(st))
        if rc:
            raise StarError(rc, self.lib.star_gpu_last_error().decode())
        return st

    def download(self, n, out=None):
        res, al, ab = out if out is not None else self._out(n, self.n_out)
        rc = self.lib.star_gpu_download_results(self.ctx, C.byref(ab))
        if rc:
            raise StarError(rc, self.lib.star_gpu_last_error().decode())
        return res, al[:ab.nAligns]

    def close(self):
        if self.ctx:
            self.lib.star_gpu_destroy(self.ctx)
            self.ctx = None
