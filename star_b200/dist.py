"""Multi-GPU driver: one process per GPU (torchrun), reads sharded by contiguous slices, index replicated per GPU.

There is no collective on the data path of a pass (SURVEY.md §8e).  Collectives:
  * allreduce(sum) of the 24 Log.final.out counters after mapping (NCCL on GPUs; gloo in the CPU test-suite),
  * a barrier; the junction records and SAM shards are files on the node's filesystem and are merged by rank 0 through the
    C-ABI helper star_host_merge_shards (global collapse + the neighbour-distance filter need the complete sorted list),
  * --twopassMode Basic: the one real exchange step of the program.  Every rank maps its slice in the 1st pass
    (--gpuTwoPassPhase 1), the collapsed junction records of all shards are ALL-GATHERED (sizes, then padded payload), every rank
    derives the same global junction list from them (star_host_merge_pass1) and inserts it into its replica of the index
    (--gpuTwoPassPhase 2) before mapping its slice again.
  * --outFilterType BySJout: the same kind of exchange between its two stages (--gpuBySJoutPhase 1 / 2): the junction records of all
    reads of all shards are all-gathered, every rank derives the same list of surviving novel junctions and maps its held reads again.

  torchrun --nproc-per-node 8 --master-addr 127.0.0.1 -m star_b200.dist -- --genomeDir idx --readFilesIn r_1.fq r_2.fq --outFileNamePrefix out/
"""
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

N_COUNTERS = 24


def _prefix(argv):
    for i, a in enumerate(argv):
        if a == "--outFileNamePrefix" and i + 1 < len(argv):
            return argv[i + 1]
    return "./"


def shard_args(argv, rank, world, device=None):
    """Command line of shard `rank`: same arguments, shard slice, shard output prefix."""
    pre = _prefix(argv)
    out = [a for a in argv]
    if "--outFileNamePrefix" in out:
        i = out.index("--outFileNamePrefix")
        out[i + 1] = pre + "shard%d." % rank
    else:
        out += ["--outFileNamePrefix", pre + "shard%d." % rank]
    out += ["--gpuShardIndex", str(rank), "--gpuShardCount", str(world)]
    if device is not None:
        out += ["--gpuDevice", str(device)]
    return out


def signal_args(argv, prefix):
    """--outWigType of a sharded run: the command line that makes the tracks from the merged Aligned.sortedByCoord.out.bam (rank 0, after
    the merge), or None.  The shards write no tracks: the reference builds them from the whole sorted BAM (STAR.cpp:274-283)."""
    keep = ("outWigType", "outWigStrand", "outWigNorm", "outWigReferencesPrefix", "runThreadN", "gpuDevice")
    groups, cur = [], None
    for a in argv:
        if a.startswith("--"):
            cur = [a]
            groups.append(cur)
        elif cur is not None:
            cur.append(a)
    out = [x for g in groups if g[0][2:].split("=")[0] in keep for x in g]
    if not any(x.startswith("--outWigType") for x in out) or "None" in [g[1] for g in groups if g[0] == "--outWigType" and len(g) > 1]:
        return None
    return ["--runMode", "inputAlignmentsFromBAM", "--inputBAMfile", prefix + "Aligned.sortedByCoord.out.bam", "--outFileNamePrefix", prefix] + out


def read_shard_counters(prefix, rank):
    with open(prefix + "shard%d.shard.bin" % rank, "rb") as f:
        return np.frombuffer(f.read(8 * N_COUNTERS), dtype=np.uint64).copy()


def two_pass(argv):
    return "--twopassMode" in argv and argv[argv.index("--twopassMode") + 1] != "None"


def by_sjout(argv):
    return "--outFilterType" in argv and argv[argv.index("--outFilterType") + 1] == "BySJout"


TIMING = {}   # phase -> seconds on this rank (rank 0 writes <prefix>dist_timing.json: the product path's own measurement)


def _timed(name, t0):
    TIMING[name] = TIMING.get(name, 0.0) + time.time() - t0


def all_gather_bytes(blob, world, device):
    """Variable-length all-gather: sizes first, then the payload padded to the longest.  Returns the list of every rank's bytes."""
    import torch
    import torch.distributed as dist
    TIMING["gather_bytes_this_rank"] = TIMING.get("gather_bytes_this_rank", 0) + len(blob)
    n = torch.tensor([len(blob)], dtype=torch.int64, device=device)
    sizes = [torch.zeros(1, dtype=torch.int64, device=device) for _ in range(world)]
    dist.all_gather(sizes, n)
    sizes = [int(x.item()) for x in sizes]
    cap = max(max(sizes), 1)
    mine = torch.zeros(cap, dtype=torch.uint8, device=device)
    if blob:
        mine[:len(blob)] = torch.frombuffer(bytearray(blob), dtype=torch.uint8).to(device)
    parts = [torch.zeros(cap, dtype=torch.uint8, device=device) for _ in range(world)]
    dist.all_gather(parts, mine)
    return [bytes(p[:sz].cpu().numpy().tobytes()) for p, sz in zip(parts, sizes)]


def run_sharded(argv, cli=None, backend=None):
    """Runs under torchrun (RANK/WORLD_SIZE/LOCAL_RANK set).  cli: None = the CUDA engine in-process (star_cli_main);
    or the path of an executable with the same command line (the test-suite passes the oracle-driven CLI)."""
    import torch
    import torch.distributed as dist
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    use_cuda = cli is None
    if world == 1:   # nothing to shard, gather or merge: the plain command line on this rank's device (it writes the final files itself)
        t0 = time.time()
        a = list(argv) + (["--gpuDevice", str(local_rank)] if use_cuda and "--gpuDevice" not in argv else [])
        if cli is None:
            import star_b200 as sb
            lib = sb.load_library()
            arr = (C.c_char_p * (len(a) + 1))(*([b"STAR"] + [x.encode() for x in a]))
            rc = lib.star_cli_main(len(a) + 1, arr)
        else:
            rc = subprocess.call([cli] + a, stdout=subprocess.DEVNULL)
        TIMING["map_s"] = TIMING["total_s"] = time.time() - t0
        TIMING["world"] = 1
        try:
            json.dump(TIMING, open(_prefix(argv) + "dist_timing.json", "w"))
        except OSError:
            pass
        return rc
    if backend is None:
        backend = "nccl" if use_cuda else "gloo"
    if use_cuda:
        torch.cuda.set_device(local_rank)
        dist.init_process_group(backend, device_id=torch.device("cuda", local_rank))
    else:
        dist.init_process_group(backend)
    import star_b200 as sb
    lib = sb.load_library()
    lib.star_host_merge_shards.argtypes = [C.c_int, C.POINTER(C.c_char_p), C.c_int, C.c_void_p]
    prog = "STAR"
    sargv = shard_args(argv, rank, world, device=local_rank if use_cuda else None)
    os.makedirs(os.path.dirname(_prefix(argv)) or ".", exist_ok=True)
    dev = "cuda" if use_cuda else "cpu"

    def run_cli(extra):
        a = sargv + extra
        if cli is None:
            arr = (C.c_char_p * (len(a) + 1))(*([prog.encode()] + [x.encode() for x in a]))
            return lib.star_cli_main(len(a) + 1, arr)
        return subprocess.call([cli] + a, stdout=subprocess.DEVNULL)

    def all_ok(rc):
        ok = torch.tensor([1 if rc == 0 else 0], dtype=torch.int64, device=dev)
        dist.all_reduce(ok, op=dist.ReduceOp.MIN)
        return int(ok.item()) == 1

    t_all = time.time()
    if two_pass(argv):
        t0 = time.time()
        rc = run_cli(["--gpuTwoPassPhase", "1"])
        _timed("pass1_map_s", t0)
        if not all_ok(rc):
            dist.destroy_process_group()
            return rc or 1
        p1dir = _prefix(sargv) + "_STARpass1/"
        t0 = time.time()
        gathered = all_gather_bytes(open(p1dir + "shard.bin", "rb").read(), world, dev)
        _timed("junction_allgather_s", t0)
        t0 = time.time()
        for r, blob in enumerate(gathered):
            with open(p1dir + "gather%d.bin" % r, "wb") as f:
                f.write(blob)
        lib.star_host_merge_pass1.argtypes = [C.c_int, C.POINTER(C.c_char_p), C.c_int, C.c_char_p]
        margv = [prog] + list(argv)
        arr = (C.c_char_p * len(margv))(*[a.encode() for a in margv])
        rc = lib.star_host_merge_pass1(len(margv), arr, world, p1dir.encode())
        _timed("pass1_junction_merge_s", t0)
        if rank == 0 and rc == 0:   # the run's own _STARpass1/ as the reference leaves it
            os.makedirs(_prefix(argv) + "_STARpass1", exist_ok=True)
            for f in ("SJ.out.tab", "Log.final.out"):
                with open(p1dir + f, "rb") as src, open(_prefix(argv) + "_STARpass1/" + f, "wb") as dst:
                    dst.write(src.read())
        if not all_ok(rc):
            dist.destroy_process_group()
            return rc or 1
        phase = ["--gpuTwoPassPhase", "2"]
    else:
        phase = []
    if by_sjout(argv):   # two stages: the junctions of ALL reads of ALL shards decide which reads with novel junctions survive
        t0 = time.time()
        rc = run_cli(phase + ["--gpuBySJoutPhase", "1"])
        _timed("map_s", t0)
        if not all_ok(rc):
            dist.destroy_process_group()
            return rc or 1
        sp = _prefix(sargv)
        t0 = time.time()
        gathered = all_gather_bytes(open(sp + "bysj_sjall.bin", "rb").read(), world, dev)
        _timed("junction_allgather_s", t0)
        for r, blob in enumerate(gathered):
            with open(sp + "bysj_gather%d.bin" % r, "wb") as f:
                f.write(blob)
        t0 = time.time()
        rc = run_cli(phase + ["--gpuBySJoutPhase", "2"])
        _timed("map_s", t0)
    else:
        t0 = time.time()
        rc = run_cli(phase)
        _timed("map_s", t0)   # (2-pass: junction insertion into this rank's index replica + the 2nd mapping pass)
    if not all_ok(rc):
        dist.destroy_process_group()
        return rc or 1
    # the one collective of the path: the Log.final.out counters
    cnt = read_shard_counters(_prefix(argv), rank).astype(np.int64)
    t = torch.from_numpy(cnt)
    if use_cuda:
        t = t.cuda()
    t0 = time.time()
    dist.all_reduce(t, op=dist.ReduceOp.SUM)
    dist.barrier()
    _timed("counter_allreduce_and_barrier_s", t0)   # (includes waiting for the slowest rank's mapping)
    rc = 0
    if rank == 0:
        t0 = time.time()
        total = t.cpu().numpy().astype(np.uint64)
        margv = [prog] + list(argv)
        arr = (C.c_char_p * len(margv))(*[a.encode() for a in margv])
        rc = lib.star_host_merge_shards(len(margv), arr, world, total.ctypes.data)
        _timed("merge_shards_s", t0)
        sig = signal_args(argv, _prefix(argv))
        if rc == 0 and sig is not None:   # the tracks of the whole run, once, from the merged sorted BAM
            t0 = time.time()
            if cli is None:
                sarr = (C.c_char_p * (len(sig) + 1))(*([prog.encode()] + [x.encode() for x in sig]))
                rc = lib.star_cli_main(len(sig) + 1, sarr)
            else:
                rc = subprocess.call([cli] + sig, stdout=subprocess.DEVNULL)
            _timed("signal_s", t0)
        TIMING["total_s"] = time.time() - t_all
        TIMING["world"] = world
        try:
            json.dump(TIMING, open(_prefix(argv) + "dist_timing.json", "w"))
        except OSError:
            pass
    dist.barrier()
    dist.destroy_process_group()
    return rc


def main():
    args = sys.argv[1:]
    cli = None
    if args and args[0] == "--cli":
        cli = args[1]
        args = args[2:]
    if args and args[0] == "--":
        args = args[1:]
    sys.exit(run_sharded(args, cli=cli))


if __name__ == "__main__":
    main()
