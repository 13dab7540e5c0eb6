#!/usr/bin/env python3
"""Multi-GPU parity check, run under torchrun with one rank per GPU (tests/test_multi_gpu.py launches it on 2 ranks
when the box has at least two GPUs):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29533 tests/multi_gpu_check.py

Every rank scans its record range; the results are exchanged through libfeiscan's multi-GPU paths and rank 0 compares the
gathered GLOBAL ordered lists with the oracle on the whole corpus:
  * fei_comm_allgather_hits   : adaptive all-gatherv after a scan (sparse = grouped ncclBroadcast of the lists, dense = masks);
  * fei_comm_scan_gather      : scan with the mask all-gather folded in (peer stores from inside the scan kernel, peer-memory
                                copies over CUDA IPC after the scan with FEI_COMM_KERNEL_PUSH=0, or a grouped ncclBroadcast
                                with FEI_COMM_P2P=0): totals, order-sensitive checksums and the materialised global lists;
  * fei_comm_allreduce_first_bad : 8-byte min-reduce of a range-sharded chain."""
import ctypes as C
import os
import re
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
os.environ.setdefault("TZ", "UTC")
M64 = (1 << 64) - 1


def checksum(lst):
    a = s = 0
    for k, v in enumerate(lst):
        a = (a + (k + 1) * int(v)) & M64
        s = (s + int(v)) & M64
    return a, s


def main():
    import torch
    import torch.distributed as dist
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    from fei_b200 import _abi, shard, synth
    from fei_b200.corpus import Corpus
    from fei_b200.program import C_BODY, C_FLAGS, Cond, ProgramBuilder
    from fei_b200.regexc import Pattern
    from oracle import chain_oracle as co, memdir_oracle as mo
    lib = _abi.lib()
    _abi.init(local)
    idbuf = np.zeros(_abi.NCCL_ID_BYTES, dtype=np.uint8)
    if rank == 0:
        _abi.check(lib.fei_comm_unique_id(_abi.ptr(idbuf)))
    t = torch.from_numpy(idbuf).cuda(); dist.broadcast(t, 0); idbuf = t.cpu().numpy()
    _abi.check(lib.fei_comm_init(_abi.ptr(idbuf), world, rank))

    n = 9001                                               # uneven shards on purpose, more than one 4096-record window each
    a, b = shard.shard_ranges(n, world)[rank]
    corpus = Corpus().synth(0xFE1, a, b - a)
    mems = None
    if rank == 0:
        recs = [synth.record(0xFE1, i) for i in range(n)]
        mems = [mo.make_memory(r["filename"], r["folder"], r["status"], synth.file_text(r), True) for r in recs]
    cases = (("sparse", ["zebra", r"kubernetes.*docker.*terraform", "rust.*python.*go"]), ("dense", ["python", "docker|kubernetes", "react", "e"]))
    for name, pats in cases:
        pb = ProgramBuilder()
        for p in pats:
            pb.add_query([Cond(C_BODY, pattern=Pattern("regex", p, re.IGNORECASE))])
        prog = pb.build(); nq = len(pats)
        want = None
        if rank == 0:
            want = [mo.run_search(mems, [{"field": "content", "operator": "matches", "value": p}]) for p in pats]
        # ---- scan, then the adaptive all-gatherv
        corpus.scan_count(prog, nq)
        bufs = [np.zeros(n, dtype=np.uint64) for _ in range(nq)]
        ptrs = (C.c_void_p * 32)(*[x.ctypes.data for x in bufs])
        cap = np.zeros(32, dtype=np.uint64); cap[:nq] = n
        tot = np.zeros(32, dtype=np.uint64); counts = np.zeros(world * nq, dtype=np.uint64)
        _abi.check(lib.fei_comm_allgather_hits(corpus.handle, nq, ptrs, _abi.ptr(cap), _abi.ptr(tot), _abi.ptr(counts)))
        gt = np.zeros(32, dtype=np.uint64); ga = np.zeros(32, dtype=np.uint64); gs = np.zeros(32, dtype=np.uint64)
        _abi.check(lib.fei_comm_gathered_checksum(nq, _abi.ptr(gt), _abi.ptr(ga), _abi.ptr(gs)))
        if rank == 0:
            for q, p in enumerate(pats):
                got = bufs[q][:int(tot[q])].tolist()
                assert got == want[q], (name, p, len(got), len(want[q]))
                assert (int(gt[q]),) + checksum(want[q]) == (len(want[q]), int(ga[q]), int(gs[q])), (name, p, "checksum")
            print(f"[multi_gpu_check] {name}: all-gatherv over {world} ranks ok ({[int(x) for x in tot[:nq]]} hits)", flush=True)
        dist.barrier()
        # ---- the scan with the gather folded in, over peer memory and over NCCL
        for p2p, push in (("1", "1"), ("1", "0"), ("0", "1")):
            os.environ["FEI_COMM_P2P"] = p2p                 # peer memory (CUDA IPC) or NCCL
            os.environ["FEI_COMM_KERNEL_PUSH"] = push        # peer stores from inside the scan kernel, or copy engines after it
            _abi.check(lib.fei_comm_bind_corpus(corpus.handle))
            tot2 = np.zeros(32, dtype=np.uint64)
            _abi.check(lib.fei_comm_scan_gather(corpus.handle, prog, len(prog), _abi.ptr(tot2)))
            _abi.check(lib.fei_comm_gathered_checksum(nq, _abi.ptr(gt), _abi.ptr(ga), _abi.ptr(gs)))
            gl = np.zeros(32, dtype=np.uint64); ms = C.c_float()
            _abi.check(lib.fei_comm_global_lists(nq, _abi.ptr(gl), C.byref(ms)))
            la, ls = corpus.list_checksums(nq)             # the local ordered lists are still built (same work as one GPU)
            if rank == 0:
                for q, p in enumerate(pats):
                    assert int(tot2[q]) == len(want[q]) == int(gt[q]) == int(gl[q]), (name, p, int(tot2[q]), len(want[q]))
                    assert checksum(want[q]) == (int(ga[q]), int(gs[q])), (name, p, "checksum of the gathered masks")
                    mine = [i for i in want[q] if a <= i < b]
                    assert checksum(mine) == (int(la[q]), int(ls[q])), (name, p, "local lists")
                how = "NCCL" if not lib.fei_comm_is_p2p() else "peer stores inside the scan kernel" if lib.fei_comm_last_exchange_in_kernel() else "peer copies after the scan"
                print(f"[multi_gpu_check] {name}: scan+gather ({how}) ok", flush=True)
            if lib.fei_comm_is_p2p():
                assert bool(lib.fei_comm_last_exchange_in_kernel()) == (push == "1"), "which path moved the masks"
            dist.barrier()
        os.environ.pop("FEI_COMM_P2P"); os.environ.pop("FEI_COMM_KERNEL_PUSH")
    # a query with header predicates: the head pass runs first, then the content pass
    pb = ProgramBuilder()
    pb.add_query([Cond(C_FLAGS, pattern=Pattern("exact_contains", "F")), Cond(C_BODY, pattern=Pattern("regex", "python|rust", re.IGNORECASE))])
    prog = pb.build()
    _abi.check(lib.fei_comm_bind_corpus(corpus.handle))
    tot2 = np.zeros(32, dtype=np.uint64)
    _abi.check(lib.fei_comm_scan_gather(corpus.handle, prog, len(prog), _abi.ptr(tot2)))
    gt = np.zeros(32, dtype=np.uint64); ga = np.zeros(32, dtype=np.uint64); gs = np.zeros(32, dtype=np.uint64)
    _abi.check(lib.fei_comm_gathered_checksum(1, _abi.ptr(gt), _abi.ptr(ga), _abi.ptr(gs)))
    if rank == 0:
        want = mo.run_search(mems, [{"field": "flags", "operator": "has_flag", "value": "F"}, {"field": "content", "operator": "matches", "value": "python|rust"}])
        assert (len(want),) + checksum(want) == (int(tot2[0]), int(ga[0]), int(gs[0])), "head + body scan+gather"
        print(f"[multi_gpu_check] flags + content query: scan+gather ok ({len(want)} hits)", flush=True)
    dist.barrier()

    # the library is called from a worker thread of the caller (CUDA's current device is per thread: it must follow fei_init's)
    import threading
    box = {}

    def worker():
        try:
            c2 = Corpus().synth(0xFE1, a, b - a)
            pb2 = ProgramBuilder(); pb2.add_query([Cond(C_BODY, pattern=Pattern("regex", "python", re.IGNORECASE))])
            box["got"] = c2.scan_hits(pb2.build(), 1)[0]
            c2.close()
        except Exception as e:  # noqa: BLE001
            box["err"] = e
    th = threading.Thread(target=worker); th.start(); th.join()
    assert "err" not in box, box.get("err")
    pb2 = ProgramBuilder(); pb2.add_query([Cond(C_BODY, pattern=Pattern("regex", "python", re.IGNORECASE))])
    assert np.array_equal(box["got"], corpus.scan_hits(pb2.build(), 1)[0]), "scan from a worker thread"
    if rank == 0:
        print("[multi_gpu_check] calls from a worker thread land on the bound device: ok", flush=True)
    dist.barrier()

    # range-sharded chain with a one-block halo; first failure = min over ranks
    nb, bad_at = 4000, 2777
    ch = C.c_void_p(); _abi.check(lib.fei_chain_create(C.byref(ch)))
    lo, hi = shard.chain_shard_ranges(nb, world)[rank]
    _abi.check(lib.fei_chain_synth(ch, 0xC4A1, lo, hi - lo, bad_at))
    fb, kind = C.c_int64(), C.c_int32()
    _abi.check(lib.fei_chain_validate(ch, C.byref(fb), C.byref(kind), None, None))
    _abi.check(lib.fei_comm_allreduce_first_bad(C.byref(fb), C.byref(kind)))
    assert (fb.value, kind.value) == (bad_at, 1), (fb.value, kind.value)
    if rank == 0:
        print(f"[multi_gpu_check] sharded chain: first bad block {fb.value} kind {kind.value}: ok", flush=True)
        print("[multi_gpu_check] ALL OK", flush=True)
    lib.fei_chain_destroy(ch)
    lib.fei_comm_destroy()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
